// C-ABI calls of libzopfli.so.1 whose input and result live in device memory (include/zopfli_b200.h,
// "input and output in device memory"): the deflate pieces are the ones ZopfliCompress produces, the stream
// is emitted behind the container header in a device allocation, and the checksum is computed on the device.
// Also the device half of the block-emission seam (ZopfliB200DeviceEmitBlocks) and the device staging of
// ZopfliB200Compressor, which need engine calls the host-only test build of api.cpp does not have.
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/zopfli_b200.h"
#include "api.hpp"
#include "checksum.hpp"
#include "dist_layout.hpp"
#include "driver.hpp"
#include "emit_bits.hpp"
#include "engine.hpp"

using namespace zb;

namespace {

int compress_device_to_device(const ZopfliOptions* options, ZopfliFormat fmt, const unsigned char* dev_in,
                              size_t insize, void* stream, unsigned char** dev_out, size_t* outsize) {
  const int ck = trailer_kind(fmt);
  if (!dev_out || !outsize || ck < 0) return 1;
  const int dev = (insize == 0 && !dev_in) ? Engine::current_device() : Engine::pointer_device(dev_in);
  if (dev < 0) return 1;
  const double t0 = now_ms();
  Engine::Lease eng(dev);
  eng->set_input_device_copy(dev_in, insize, stream, ck);
  std::vector<Piece> pieces;
  deflate_units(*eng, options, 2, true, master_blocks(0, insize), 0, pieces);
  std::vector<Engine::EmitPiece> ep;
  std::vector<uint64_t> layout;
  const uint64_t total = place_pieces(pieces, 0, 0, ep, &layout, options->verbose != 0);
  unsigned char hdr[10];
  const int hdr_len = container_header(fmt, hdr);
  size_t n = 0;
  unsigned char* out = eng->emit_to_device(ep, total, hdr, hdr_len, ck, stream, &n);
  if (options->verbose) report_sizes(fmt, insize, (size_t)((total + 7) / 8), n);
  *dev_out = out;
  *outsize = n;
  api_call_done(layout, t0);
  return 0;
}

int device_checksum(const unsigned char* dev_in, size_t size, void* stream, int kind, uint32_t* out) {
  if (!out) return 1;
  if (size == 0) { *out = kind == kCkCrc32 ? 0u : 1u; return 0; }
  const int dev = Engine::pointer_device(dev_in);
  if (dev < 0) return 1;
  Engine::Lease eng(dev);
  *out = eng->checksum_device(dev_in, size, stream, kind);
  return 0;
}

// A compressor's waves in device memory (chunks of one device): one stream-ordered allocation per slot, grown
// as bytes arrive up to one wave and its dictionary.  Each chunk is copied device to device after the work
// queued on the caller's stream; a wave's engine adopts its slot as input (no host copy).  The stream stays on
// the device too: each wave's runs of compressed blocks are emitted into an allocation of their own, and k_splice
// places them and the stored blocks (read from the slot) on the pending stream, so only the bytes a caller asks
// for on the host are downloaded.
struct DeviceWaveStaging : WaveStaging {
  DeviceStaging ds;
  void* user_stream;
  unsigned char* slot[kSlots] = {};
  size_t cap[kSlots] = {}, len[kSlots] = {};
  static constexpr size_t kPad = 64;  // the kernels read up to 16 bytes past the input; zeroed as set_input_host does
  // the stream not yet returned: pend_bits bits from bit 0 of pend, which is zero past them
  unsigned char* pend = nullptr;
  size_t pend_cap = 0;
  uint64_t pend_bits = 0;

  DeviceWaveStaging(int dev, void* stream) : ds(dev), user_stream(stream) {}
  ~DeviceWaveStaging() override {
    for (int s = 0; s < kSlots; s++) ds.release(slot[s]);
    ds.release(pend);
  }
  int device() const override { return ds.device(); }
  bool accepts(const void* p, size_t n) const override { return n == 0 || Engine::pointer_device(p) == ds.device(); }
  void grow(int s, size_t need) {  // keeps the slot's len[s] bytes
    if (need + kPad <= cap[s]) return;
    const size_t want = std::max(need, std::min(2 * cap[s], slot_bytes)) + kPad;
    unsigned char* p = (unsigned char*)ds.alloc(want);
    if (slot[s]) {
      ds.copy(p, slot[s], len[s], ds.stream());
      ds.release(slot[s]);
    }
    slot[s] = p;
    cap[s] = want;
  }
  void put(int s, size_t off, const unsigned char* chunk, size_t n) override {
    len[s] = off;
    grow(s, off + n);
    ds.copy(slot[s] + off, chunk, n, user_stream);
    len[s] = off + n;
  }
  void carry(int from, size_t off, int to, size_t n) override {
    len[to] = 0;
    grow(to, n);
    ds.copy(slot[to], slot[from] + off, n, ds.stream());
    len[to] = n;
  }
  void stage(Engine& eng, int s, size_t n) override {
    grow(s, n);
    ds.zero(slot[s] + n, kPad);
    eng.set_input_device(slot[s], n);
  }
  uint32_t checksum(Engine& eng, int s, size_t off, size_t n, int kind) override {
    return eng.checksum_device(slot[s] + off, n, ds.stream(), kind);
  }
  // The records point into sr.runs and slot s until the wave is spliced: only the filling slot is written or
  // regrown (put, carry; stage grew slot s before this), and slot s is not filling again before its wave is retired.
  void take_records(Engine& eng, int s, size_t base, SpanRecords& sr) override {
    if (sr.run_bits) {
      const void* bits = eng.emit_device(sr.ep, sr.run_bits, 0);  // done when it returns
      const size_t n = (size_t)(sr.run_bits / 8);  // whole 8-byte words: every run starts on one
      sr.runs = (unsigned char*)ds.alloc(n);
      ds.copy(sr.runs, bits, n, ds.stream());
    }
    point_records(sr, sr.runs, slot[s], base);
  }
  void drop_records(SpanRecords& sr) override {
    ds.release(sr.runs);
    sr.runs = nullptr;
  }
  uint32_t checksum_of(const unsigned char* p, size_t n, int kind) override {  // k_crc32 / k_adler32: no PCIe copy
    Engine::Lease eng(ds.device());
    return eng->checksum_device(p, n, user_stream, kind);
  }

  unsigned phase() const override { return (unsigned)(pend_bits & 7); }
  // room for a stream of end_bits bits in whole 4-byte words (k_splice's unit), zero past the current stream
  void pend_grow(uint64_t end_bits) {
    const size_t need = (size_t)((end_bits + 31) / 32) * 4;
    if (need <= pend_cap) return;
    const size_t want = std::max(need, 2 * pend_cap);
    unsigned char* p = (unsigned char*)ds.alloc(want);
    ds.zero(p, want);
    if (pend) {
      ds.copy(p, pend, (size_t)((pend_bits + 7) / 8), ds.stream());
      ds.release(pend);
    }
    pend = p;
    pend_cap = want;
  }
  void put(const std::vector<Engine::SpanRecord>& recs, uint64_t end) {
    pend_grow(end);
    Engine::Lease eng(ds.device());  // for this splice only: the compressor holds no context between calls
    eng->splice(recs, pend, ds.stream());
    pend_bits = end;
  }
  void put_bytes(const unsigned char* p, size_t n) override {
    if (n == 0) return;
    Engine::SpanRecord r;
    r.bit_start = (pend_bits + 7) & ~(uint64_t)7;
    r.n = (uint64_t)n * 8;
    r.src = p;
    r.literal = true;
    put({r}, r.bit_start + r.n);
  }
  void splice(SpanRecords& sr) override { put(sr.recs, span_positions(sr.recs, pend_bits)); }
  size_t hand_out(bool all, bool to_device, unsigned char** out, size_t* outsize) override {
    const size_t used = (size_t)((pend_bits + 7) / 8), n = all ? used : (size_t)(pend_bits / 8);
    if (to_device) {
      *out = nullptr;
      *outsize = 0;
    }
    if (n && to_device) {
      *out = (unsigned char*)ds.alloc_on(n, user_stream);
      ds.copy(*out, pend, n, user_stream);  // after the allocation; done when it returns
      *outsize = n;
    } else if (n) {
      Engine::Lease eng(ds.device());
      eng->download(pend, append_reserve(n, out, outsize), n);
    }
    // the partly filled last byte, if it stays, moves to byte 0; the rest is zero again
    const size_t keep = used - n;
    if (keep && n) ds.copy(pend, pend + n, 1, ds.stream());
    if (used > keep) ds.zero(pend + keep, used - keep);
    pend_bits -= (uint64_t)n * 8;
    return n;
  }
};

// ZopfliB200AppendSpan with the splice done by k_splice: the records' bytes (each from a 4-byte boundary) and the
// caller's partly filled last byte are uploaded, spliced on the device, and the new bytes downloaded
int device_append_span(const unsigned char* span, size_t spansize, unsigned char* bp, unsigned char** out,
                       size_t* outsize) {
  std::vector<Engine::SpanRecord> recs;
  if (!bp || !out || !outsize || !parse_span(span, spansize, recs)) return 1;
  const unsigned phase = (*outsize > 0) ? *bp : 0u;  // splice_pieces' bit0
  if (phase > 7) return 1;
  const uint64_t end = span_positions(recs, phase);
  const size_t nbytes = (size_t)((end + 7) / 8);
  if (recs.empty() || nbytes == 0) {
    *bp = (unsigned char)(end & 7);
    return 0;
  }
  std::vector<size_t> at(recs.size());
  std::vector<unsigned char> src;
  for (size_t i = 0; i < recs.size(); i++) {
    const Engine::SpanRecord& r = recs[i];
    at[i] = src.size();
    src.insert(src.end(), r.src, r.src + (r.stored ? r.n : (r.n + 7) / 8));
    src.resize((src.size() + 3) & ~(size_t)3);
  }
  const int dev = Engine::current_device();
  DeviceStaging ds(dev);
  const size_t cap = (nbytes + 3) & ~(size_t)3;
  unsigned char* d_src = (unsigned char*)ds.alloc(src.size() + 4);
  unsigned char* d_out = (unsigned char*)ds.alloc(cap);
  ds.zero(d_out, cap);
  Engine::Lease eng(dev);
  if (!src.empty()) eng->upload(d_src, src.data(), src.size());
  if (phase) eng->upload(d_out, *out + *outsize - 1, 1);
  for (size_t i = 0; i < recs.size(); i++) recs[i].src = d_src + at[i];
  eng->splice(recs, d_out, ds.stream());
  append_stream(nbytes, phase, out, outsize, [&](unsigned char* dst) { eng->download(d_out, dst, nbytes); });
  ds.release(d_src);
  ds.release(d_out);
  *bp = (unsigned char)(end & 7);
  return 0;
}

WaveStaging* device_staging(int dev, void* stream) {
  if (dev < 0 || dev >= Engine::device_count()) return nullptr;
  return new DeviceWaveStaging(dev, stream);
}

// ZopfliB200CompressorNew (api.cpp) reaches device memory through these
const bool g_registered = [] {
  g_device_staging = device_staging;
  g_pointer_device = Engine::pointer_device;
  return true;
}();

}  // namespace

extern "C" {

int ZopfliB200CompressDeviceToDevice(const ZopfliOptions* options, ZopfliFormat output_type, const unsigned char* dev_in,
                                     size_t insize, void* cuda_stream, unsigned char** dev_out, size_t* outsize) {
  return compress_device_to_device(options, output_type, dev_in, insize, cuda_stream, dev_out, outsize);
}

void ZopfliB200FreeDevice(void* dev_ptr, void* cuda_stream) { Engine::free_device(dev_ptr, cuda_stream); }

int ZopfliB200Crc32Device(const unsigned char* dev_in, size_t size, void* cuda_stream, uint32_t* crc) {
  return device_checksum(dev_in, size, cuda_stream, kCkCrc32, crc);
}

int ZopfliB200Adler32Device(const unsigned char* dev_in, size_t size, void* cuda_stream, uint32_t* adler) {
  return device_checksum(dev_in, size, cuda_stream, kCkAdler32, adler);
}

int ZopfliB200DeviceAppendSpan(const unsigned char* span, size_t spansize, unsigned char* bp, unsigned char** out,
                               size_t* outsize) {
  return device_append_span(span, spansize, bp, out, outsize);
}

int ZopfliB200DeviceProbeParts(const uint32_t* hists, size_t nhist, uint32_t* smoothed, unsigned char* lengths,
                               uint32_t* tree_bits, uint64_t* dyn_bits) {
  Engine::Lease eng;
  eng->device_probe_parts(hists, nhist, smoothed, lengths, tree_bits, dyn_bits);
  return 0;
}

int ZopfliB200DeviceEmitBlocks(const unsigned char* in, size_t insize, const unsigned short* litlens,
                               const unsigned short* dists, size_t n, size_t npieces, const size_t* lstart,
                               const size_t* lend, const int* btype, const int* final, unsigned bp0,
                               unsigned char* out, size_t cap, uint64_t* nbits, unsigned char* plan_len,
                               uint64_t* plan_val) {
  std::vector<Piece> pieces;
  if (!seam_pieces(insize, litlens, dists, n, npieces, lstart, lend, btype, final, bp0, pieces)) return 1;
  Engine::Lease eng;
  eng->set_input_host(in, insize);
  eng->load_symbols(Engine::kFin, litlens, dists, n);
  std::vector<Engine::PlanReq> rq(npieces);
  for (size_t i = 0; i < npieces; i++) rq[i] = {pieces[i].off, pieces[i].n, (uint32_t)Engine::kFin};
  std::vector<Engine::PlanCost> costs;
  std::vector<uint64_t> handles;
  eng->plan_blocks(rq, costs, handles);
  for (size_t i = 0; i < npieces; i++) {
    BlockPlan b;
    eng->download((const void*)(uintptr_t)handles[i], (uint8_t*)&b, sizeof(b));
    pieces[i].plan = handles[i];
    seam_plan_out(b, pieces[i], plan_len + i * 320, plan_val + i * 6);
  }
  std::vector<Engine::EmitPiece> ep;
  *nbits = layout_pieces(pieces, 0, bp0, ep, nullptr);  // the driver's placement: prefix sum, stored_end
  if ((*nbits + 7) / 8 > cap) return 1;
  eng->emit(ep, *nbits, out);
  return 0;
}

}  // extern "C"

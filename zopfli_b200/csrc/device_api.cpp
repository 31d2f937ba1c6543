// C-ABI calls of libzopfli.so.1 whose input and result live in device memory (include/zopfli_b200.h,
// "input and output in device memory"): the deflate pieces are the ones ZopfliCompress produces, the stream
// is emitted behind the container header in a device allocation, and the checksum is computed on the device.
// Also the device half of the block-emission seam (ZopfliB200DeviceEmitBlocks) and the device staging of
// ZopfliB200Compressor, which need engine calls the host-only test build of api.cpp does not have.
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
// queued on the caller's stream; a wave's engine adopts its slot as input (no host copy), and only the bytes of
// stored blocks come back to the host.
struct DeviceWaveStaging : WaveStaging {
  DeviceStaging ds;
  void* user_stream;
  unsigned char* slot[kSlots] = {};
  size_t cap[kSlots] = {}, len[kSlots] = {};
  static constexpr size_t kPad = 64;  // the kernels read up to 16 bytes past the input; zeroed as set_input_host does

  DeviceWaveStaging(int dev, void* stream) : ds(dev), user_stream(stream) {}
  ~DeviceWaveStaging() override {
    for (int s = 0; s < kSlots; s++) ds.release(slot[s]);
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
  void read(Engine& eng, int s, size_t off, size_t n, unsigned char* dst) override { eng.download(slot[s] + off, dst, n); }
  uint32_t checksum_of(const unsigned char* p, size_t n, int kind) override {  // k_crc32 / k_adler32: no PCIe copy
    Engine::Lease eng(ds.device());
    return eng->checksum_device(p, n, user_stream, kind);
  }
};

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

// C-ABI calls of libzopfli.so.1 whose input and result live in device memory (include/zopfli_b200.h,
// "input and output in device memory"): the deflate pieces are the ones ZopfliCompress produces, the stream
// is emitted behind the container header in a device allocation, and the checksum is computed on the device.
// Also the device half of the block-emission seam (ZopfliB200DeviceEmitBlocks), which needs engine calls
// the host-only test build of api.cpp does not have.
#include <stdio.h>

#include <vector>

#include "../../include/zopfli_b200.h"
#include "api.hpp"
#include "checksum.hpp"
#include "driver.hpp"
#include "emit_bits.hpp"
#include "engine.hpp"

using namespace zb;

namespace {

int compress_device_to_device(const ZopfliOptions* options, ZopfliFormat fmt, const unsigned char* dev_in,
                              size_t insize, void* stream, unsigned char** dev_out, size_t* outsize) {
  if (!dev_out || !outsize || (fmt != ZOPFLI_FORMAT_GZIP && fmt != ZOPFLI_FORMAT_ZLIB && fmt != ZOPFLI_FORMAT_DEFLATE))
    return 1;
  const int dev = (insize == 0 && !dev_in) ? Engine::current_device() : Engine::pointer_device(dev_in);
  if (dev < 0) return 1;
  const double t0 = api_now_ms();
  const int ck = fmt == ZOPFLI_FORMAT_GZIP ? kCkCrc32 : (fmt == ZOPFLI_FORMAT_ZLIB ? kCkAdler32 : kCkNone);
  Engine::Lease eng(dev);
  eng->set_input_device_copy(dev_in, insize, stream, ck);
  std::vector<Piece> pieces;
  deflate_units(*eng, options, 2, true, nullptr, api_master_units(insize), 0, pieces);
  std::vector<Engine::EmitPiece> ep;
  std::vector<uint64_t> layout;
  const uint64_t total = place_pieces(pieces, 0, 0, ep, &layout, options->verbose != 0);
  unsigned char hdr[10];
  const int hdr_len = container_header(fmt, hdr);
  size_t n = 0;
  unsigned char* out = eng->emit_to_device(ep, total, hdr, hdr_len, ck, stream, &n);
  if (options->verbose) {  // the reports ZopfliCompress prints after the deflate body and after the container
    const size_t deflated = (size_t)((total + 7) / 8);
    fprintf(stderr, "Original Size: %lu, Deflate: %lu, Compression: %f%% Removed\n", (unsigned long)insize,
            (unsigned long)deflated, 100.0 * (double)(insize - deflated) / (double)insize);
    if (fmt != ZOPFLI_FORMAT_DEFLATE)
      fprintf(stderr, "Original Size: %d, %s: %d, Compression: %f%% Removed\n", (int)insize,
              fmt == ZOPFLI_FORMAT_GZIP ? "Gzip" : "Zlib", (int)n, 100.0 * (double)(insize - n) / (double)insize);
  }
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

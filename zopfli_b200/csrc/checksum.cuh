// CRC-32 and Adler-32 of device bytes (checksum.hpp has the slice algebra), plus the kernel that writes a
// gzip / zlib header and trailer around a stream that lives in device memory.
//
// Layout: the head (up to 15 bytes before the first 16-byte boundary) and the tail (the last n - head mod
// 16 bytes) are slices of their own, summed by thread 0 of CTA 0.  The body between them is cut into 4 KiB
// tiles; warp w takes tiles w, w + W, w + 2W, ... (W warps in the grid).  Each lane reads 128 contiguous
// bytes of the tile with 16-byte loads and reduces them to its slice's contribution; the warp reduces the
// lanes, carries the running sum of its tiles in registers and adds it to the global accumulator with one
// atomic per kernel.  Every byte in [in, in + n) is read once and nothing outside it is read.
#pragma once
#include <stdint.h>

#include "checksum.hpp"

namespace zb {

constexpr int kCkThreads = 256;
constexpr uint32_t kCkTile = 4096;
constexpr uint32_t kCkLaneBytes = kCkTile / 32;

struct CkArgs {
  const uint8_t* in;
  uint64_t n;
  ChecksumAcc* acc;
  CrcShiftTable tab;
};

struct CkLayout {
  uint64_t head, body_end, ntiles;  // body = [head, body_end), a multiple of 16 bytes at a 16-byte address
  __device__ explicit CkLayout(const uint8_t* in, uint64_t n) {
    head = (16 - ((uintptr_t)in & 15)) & 15;
    if (head > n) head = n;
    body_end = head + ((n - head) & ~(uint64_t)15);
    ntiles = (body_end - head + kCkTile - 1) / kCkTile;
  }
};

// loads lane `lane`'s part [la, lb) of tile t (la, lb relative to the tile start; lb - la a multiple of 16)
__device__ __forceinline__ uint32_t ck_load(const uint8_t* in, const CkLayout& L, uint64_t t, uint32_t lane,
                                            uint4 (&v)[kCkLaneBytes / 16], uint32_t& tile_len, uint32_t& lb) {
  const uint64_t start = L.head + t * kCkTile;
  tile_len = L.body_end - start < kCkTile ? (uint32_t)(L.body_end - start) : kCkTile;
  const uint32_t la = min(lane * kCkLaneBytes, tile_len);
  lb = min(la + kCkLaneBytes, tile_len);
  const uint4* p = (const uint4*)(in + start + la);
#pragma unroll
  for (uint32_t k = 0; k < kCkLaneBytes / 16; k++)
    if (la + 16 * k < lb) v[k] = p[k];
  return la;
}

__global__ void __launch_bounds__(kCkThreads) k_crc32(CkArgs a) {
  __shared__ uint32_t T[8][256];  // slicing-by-8 tables (the host checksum uses the same)
  for (uint32_t i = threadIdx.x; i < 256; i += kCkThreads) T[0][i] = crc_table_entry(0, i);
  __syncthreads();
  for (int t = 1; t < 8; t++) {
    for (uint32_t i = threadIdx.x; i < 256; i += kCkThreads) T[t][i] = (T[t - 1][i] >> 8) ^ T[0][T[t - 1][i] & 255];
    __syncthreads();
  }
  const CkLayout L(a.in, a.n);
  const uint32_t lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) {  // head and tail slices
    uint32_t c = 0;
    for (uint64_t i = 0; i < L.head; i++) c = T[0][(c ^ a.in[i]) & 255] ^ (c >> 8);
    uint32_t r = crc_shift(c, a.n - L.head, a.tab);
    c = 0;
    for (uint64_t i = L.body_end; i < a.n; i++) c = T[0][(c ^ a.in[i]) & 255] ^ (c >> 8);
    r ^= c;
    if (r) atomicXor(&a.acc->crc0, r);
  }
  const uint64_t nwarps = (uint64_t)gridDim.x * (kCkThreads / 32);
  const uint64_t w = (uint64_t)blockIdx.x * (kCkThreads / 32) + threadIdx.x / 32;
  if (w >= L.ntiles) return;
  // lane contribution of a whole tile: shifted past the lanes after it; running sum: shifted past W tiles
  const uint32_t k_lane = crc_shift(0x80000000u, kCkTile - (lane + 1) * kCkLaneBytes, a.tab);
  const uint32_t k_stride = crc_shift(0x80000000u, nwarps * kCkTile, a.tab);
  uint32_t run = 0;
  uint64_t run_end = 0;
  for (uint64_t t = w; t < L.ntiles; t += nwarps) {
    uint4 v[kCkLaneBytes / 16];
    uint32_t tile_len, lb;
    const uint32_t la = ck_load(a.in, L, t, lane, v, tile_len, lb);
    uint32_t c = 0;
#pragma unroll
    for (uint32_t k = 0; k < kCkLaneBytes / 16; k++)
      if (la + 16 * k < lb) { c = crc_slice8(c, v[k].x, v[k].y, T); c = crc_slice8(c, v[k].z, v[k].w, T); }
    c = tile_len == kCkTile ? crc_mulmod(c, k_lane) : crc_shift(c, tile_len - lb, a.tab);
#pragma unroll
    for (int o = 16; o; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
    const uint64_t end = L.head + t * kCkTile + tile_len;
    if (t == w) run = c;
    else run = (end - run_end == nwarps * kCkTile ? crc_mulmod(run, k_stride) : crc_shift(run, end - run_end, a.tab)) ^ c;
    run_end = end;
  }
  if (lane == 0) {
    run = crc_shift(run, a.n - run_end, a.tab);
    if (run) atomicXor(&a.acc->crc0, run);
  }
}

__device__ __forceinline__ void adler_word(uint32_t x, uint32_t& s1, uint32_t& s2) {
  s2 += 4 * s1 + __dp4a(x, 0x01020304u, 0u);  // bytes d0..d3 (little endian) weigh 4, 3, 2, 1
  s1 += __dp4a(x, 0x01010101u, 0u);
}

__global__ void __launch_bounds__(kCkThreads) k_adler32(CkArgs a) {
  const CkLayout L(a.in, a.n);
  const uint32_t lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) {  // head and tail slices
    uint64_t sa = 0, sb = 0;
    uint32_t s1 = 0, s2 = 0;
    for (uint64_t i = 0; i < L.head; i++) { s1 += a.in[i]; s2 += s1; }
    sa += s1;
    sb += s2 + ((a.n - L.head) % kAdlerMod) * s1;
    s1 = s2 = 0;
    for (uint64_t i = L.body_end; i < a.n; i++) { s1 += a.in[i]; s2 += s1; }
    sa += s1;
    sb += s2;
    atomicAdd(&a.acc->a, (unsigned long long)sa);
    atomicAdd(&a.acc->b, (unsigned long long)sb);
  }
  const uint64_t nwarps = (uint64_t)gridDim.x * (kCkThreads / 32);
  const uint64_t w = (uint64_t)blockIdx.x * (kCkThreads / 32) + threadIdx.x / 32;
  if (w >= L.ntiles) return;
  uint64_t sa = 0, sb = 0;  // sa < 255 n; sb < tiles x 2^36
  for (uint64_t t = w; t < L.ntiles; t += nwarps) {
    uint4 v[kCkLaneBytes / 16];
    uint32_t tile_len, lb;
    const uint32_t la = ck_load(a.in, L, t, lane, v, tile_len, lb);
    uint32_t s1 = 0, s2 = 0;  // 128 bytes: s1 < 2^15, s2 < 2^23
#pragma unroll
    for (uint32_t k = 0; k < kCkLaneBytes / 16; k++)
      if (la + 16 * k < lb) { adler_word(v[k].x, s1, s2); adler_word(v[k].y, s1, s2); adler_word(v[k].z, s1, s2); adler_word(v[k].w, s1, s2); }
    uint32_t t2 = (s2 + (tile_len - lb) * s1) % kAdlerMod;  // relative to the tile's end: < 2^28 before the mod
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      t2 += __shfl_xor_sync(0xffffffffu, t2, o);
    }
    const uint64_t end = L.head + t * kCkTile + tile_len;
    sa += s1;
    sb += t2 + ((a.n - end) % kAdlerMod) * s1;
  }
  if (lane == 0) {
    atomicAdd(&a.acc->a, (unsigned long long)sa);
    atomicAdd(&a.acc->b, (unsigned long long)(sb % kAdlerMod));
  }
}

// gzip (gzip_container.c:84-124) / zlib (zlib_container.c:50-79) framing of a stream of body_bytes bytes that
// already sits at out + hdr_len: the header, and the trailer from the device checksum and ISIZE.
struct ContainerArgs {
  uint8_t* out;
  uint64_t body_bytes, isize;
  const ChecksumAcc* acc;
  CrcShiftTable tab;
  uint8_t hdr[12];
  uint32_t hdr_len;
  int kind;
};

__global__ void k_container(ContainerArgs a) {
  const uint32_t lane = threadIdx.x;
  if (lane < a.hdr_len) a.out[lane] = a.hdr[lane];
  if (lane != 0) return;
  const uint32_t c = a.kind == kCkCrc32     ? crc_finish(a.acc->crc0, a.isize, a.tab)
                     : a.kind == kCkAdler32 ? adler_finish(a.acc->a, a.acc->b, a.isize)
                                            : 0u;
  container_trailer(a.kind, c, a.isize, a.out + a.hdr_len + a.body_bytes);
}

}  // namespace zb

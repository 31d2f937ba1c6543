// DEFLATE symbol arithmetic shared by host code and sm_90a kernels.
// Same values as the reference's tables (/root/reference/src/zopfli/symbols.h:38-237), computed
// in closed form (bit tricks instead of 259-entry tables) so they cost no memory traffic on
// the device.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define ZB_HD __host__ __device__ __forceinline__
#else
#define ZB_HD inline
#endif
#if defined(__CUDA_ARCH__)
#define ZB_UNROLL _Pragma("unroll")
#else
#define ZB_UNROLL
#endif

namespace zb {

constexpr int kNumLL = 288;        // util.h:31
constexpr int kNumD = 32;          // util.h:32
constexpr int kWindow = 32768;     // util.h:41
constexpr int kMaxMatch = 258;     // util.h:28
constexpr int kMinMatch = 3;       // util.h:29
constexpr int kMaxChainHits = 8192;  // util.h:84
constexpr int kMasterBlock = 1000000;  // util.h:60

ZB_HD int ilog2(uint32_t x) {  // floor(log2(x)), x > 0
#if defined(__CUDA_ARCH__)
  return 31 - __clz((int)x);
#else
  return 31 - __builtin_clz(x);
#endif
}

// symbols.h:138-176
ZB_HD int length_symbol(int l) {
  if (l < 11) return l < 3 ? 0 : 254 + l;
  if (l == 258) return 285;
  int x = l - 3;
  int hb = ilog2((uint32_t)x);
  return 257 + 4 * (hb - 1) + ((x >> (hb - 2)) & 3);
}
// symbols.h:88-110
ZB_HD int length_extra_bits(int l) {
  if (l < 11 || l == 258) return 0;
  return ilog2((uint32_t)(l - 3)) - 2;
}
// symbols.h:113-135
ZB_HD int length_extra_bits_value(int l) {
  if (l < 11 || l == 258) return 0;
  int x = l - 3;
  int eb = ilog2((uint32_t)x) - 2;
  return x & ((1 << eb) - 1);
}
// symbols.h:222-228
ZB_HD int length_symbol_extra_bits(int s) {
  if (s < 265 || s == 285) return 0;
  return (s - 261) >> 2;
}
// symbols.h:62-86
ZB_HD int dist_symbol(int dist) {
  if (dist < 5) return dist - 1;
  int l = ilog2((uint32_t)(dist - 1));
  return l * 2 + (((dist - 1) >> (l - 1)) & 1);
}
// symbols.h:38-41
ZB_HD int dist_extra_bits(int dist) {
  if (dist < 5) return 0;
  return ilog2((uint32_t)(dist - 1)) - 1;
}
// symbols.h:44-59
ZB_HD int dist_extra_bits_value(int dist) {
  if (dist < 5) return 0;
  int l = ilog2((uint32_t)(dist - 1));
  return (dist - (1 + (1 << l))) & ((1 << (l - 1)) - 1);
}
// symbols.h:231-237
ZB_HD int dist_symbol_extra_bits(int s) { return s < 4 ? 0 : (s - 2) >> 1; }

}  // namespace zb

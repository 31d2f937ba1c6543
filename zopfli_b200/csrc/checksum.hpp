// CRC-32 (gzip trailer, gzip_container.c:27-81) and Adler-32 (zlib trailer, zlib_container.c:29-48) written
// as sums of per-slice contributions that commute, shared by the sm_90a kernels (checksum.cuh) and the host
// checksum of api.cpp.
//
// CRC-32: crc0(s) is the CRC register after slice s starting from 0, without the final inversion.  crc0 is
// linear over GF(2), so for an n-byte input cut into slices [a, b):
//   crc0(input) = XOR over slices of crc0(slice) * x^(8(n - b))  mod P
//   crc32       = crc0(input) ^ (0xFFFFFFFF * x^(8n) mod P) ^ 0xFFFFFFFF
// Adler-32: with s1 = sum d_i and s2 = sum (b - i) d_i over a slice [a, b):
//   A = 1 + sum s1,  B = n + sum (s2 + (n - b) s1)   (both mod 65521)
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "symbols.hpp"

namespace zb {

constexpr uint32_t kCrcPoly = 0xEDB88320u;   // reflected: bit 31 is x^0
constexpr uint32_t kAdlerMod = 65521;
// which trailer a checksum feeds; the values are the ZopfliFormat of that container
enum ChecksumKind { kCkCrc32 = 0, kCkAdler32 = 1, kCkNone = 2 };

// entry i of slicing table t: the register after byte i followed by t zero bytes
ZB_HD uint32_t crc_table_entry(int t, uint32_t i) {
  uint32_t c = i;
  for (int k = 0; k < 8 * (t + 1); k++) c = (c & 1) ? kCrcPoly ^ (c >> 1) : c >> 1;
  return c;
}

// slicing-by-8: the register c after the eight bytes lo (bytes 0-3, little-endian) and hi (bytes 4-7), with
// T[t][i] = crc_table_entry(t, i)
ZB_HD uint32_t crc_slice8(uint32_t c, uint32_t lo, uint32_t hi, const uint32_t (*T)[256]) {
  lo ^= c;
  return T[7][lo & 255] ^ T[6][(lo >> 8) & 255] ^ T[5][(lo >> 16) & 255] ^ T[4][lo >> 24] ^ T[3][hi & 255] ^
         T[2][(hi >> 8) & 255] ^ T[1][(hi >> 16) & 255] ^ T[0][hi >> 24];
}

// a * b mod P in the reflected representation (32 fixed steps, no data-dependent exit)
ZB_HD uint32_t crc_mulmod(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (int k = 0; k < 32; k++) {
    p ^= b & (0u - ((a >> (31 - k)) & 1u));
    b = (b >> 1) ^ (kCrcPoly & (0u - (b & 1u)));
  }
  return p;
}

// x^(8 * 2^j) mod P, j = 0..63: multiplying by x^(8L) takes one crc_mulmod per set bit of L
struct CrcShiftTable { uint32_t x8pow2[64]; };
ZB_HD CrcShiftTable crc_shift_table() {
  CrcShiftTable t;
  t.x8pow2[0] = 0x80000000u >> 8;  // x^8
  for (int j = 1; j < 64; j++) t.x8pow2[j] = crc_mulmod(t.x8pow2[j - 1], t.x8pow2[j - 1]);
  return t;
}
// c * x^(8L) mod P: the register c followed by L zero bytes
ZB_HD uint32_t crc_shift(uint32_t c, uint64_t L, const CrcShiftTable& t) {
  for (int j = 0; L; j++, L >>= 1)
    if (L & 1) c = crc_mulmod(c, t.x8pow2[j]);
  return c;
}
ZB_HD uint32_t crc_finish(uint32_t crc0, uint64_t n, const CrcShiftTable& t) {
  return crc0 ^ crc_shift(0xFFFFFFFFu, n, t) ^ 0xFFFFFFFFu;
}

// The zlib crc32_combine construction: crc32 of A|B from crc32(A), crc32(B) and |B|.  The initial and final
// inversions cancel, leaving crc1 * x^(8 len2) ^ crc2.
inline uint32_t crc32_combine(uint32_t crc1, uint32_t crc2, uint64_t len2) {
  if (len2 == 0) return crc1;
  static const CrcShiftTable t = crc_shift_table();
  return crc_shift(crc1, len2, t) ^ crc2;
}

// Adler-32 of A|B from adler32(A), adler32(B) and |B| (the zlib adler32_combine construction).  With s1 = 1 + sum
// of bytes and s2 = sum of the s1 after each byte: s1(A|B) = s1(A) + s1(B) - 1, s2(A|B) = s2(A) + s2(B) + |B| (s1(A) - 1).
inline uint32_t adler32_combine(uint32_t adler1, uint32_t adler2, uint64_t len2) {
  const uint64_t a1 = adler1 & 0xffff, b1 = adler1 >> 16, a2 = adler2 & 0xffff, b2 = adler2 >> 16;
  const uint64_t s1 = (a1 + a2 + kAdlerMod - 1) % kAdlerMod;
  const uint64_t s2 = (b1 + b2 + (len2 % kAdlerMod) * ((a1 + kAdlerMod - 1) % kAdlerMod)) % kAdlerMod;
  return (uint32_t)((s2 << 16) | s1);
}

// s1 = sum of bytes, s2 = sum of (n - i) * d_i over p[0, n), both mod 65521.  5552 bytes is the largest run
// whose 32-bit running sums cannot overflow (the zlib bound the reference also relies on with 5550).
struct AdlerPart { uint64_t s1, s2, len; };
inline AdlerPart adler_chunk(const unsigned char* p, size_t n) {
  uint32_t a = 0, b = 0;
  size_t left = n;
  while (left) {
    const size_t k = left > 5552 ? 5552 : left;
    for (size_t i = 0; i < k; i++) { a += p[i]; b += a; }
    a %= kAdlerMod;
    b %= kAdlerMod;
    p += k;
    left -= k;
  }
  return {a, b, n};
}
// a = sum of s1, b = sum of (s2 + (n - b) s1) over the slices (any size below 2^64, reduced here)
ZB_HD uint32_t adler_finish(uint64_t a, uint64_t b, uint64_t n) {
  const uint64_t s1 = (1 + a % kAdlerMod) % kAdlerMod, s2 = (b % kAdlerMod + n % kAdlerMod) % kAdlerMod;
  return (uint32_t)((s2 << 16) | s1);
}

// The container trailer at tr: gzip (gzip_container.c:106-116) CRC-32 then ISIZE, both little-endian; zlib
// (zlib_container.c:67-71) Adler-32, big-endian.  Returns its length, 0 for kCkNone.
ZB_HD int container_trailer(int kind, uint32_t checksum, uint64_t isize, uint8_t* tr) {
  if (kind == kCkCrc32) {
    for (int k = 0; k < 4; k++) tr[k] = (uint8_t)(checksum >> (8 * k));
    for (int k = 0; k < 4; k++) tr[4 + k] = (uint8_t)(isize >> (8 * k));
    return 8;
  }
  if (kind == kCkAdler32) {
    for (int k = 0; k < 4; k++) tr[k] = (uint8_t)(checksum >> (24 - 8 * k));
    return 4;
  }
  return 0;
}

// slices' contributions added up: crc0 XORed, a and b summed (what crc_finish / adler_finish take)
struct ChecksumAcc {
  uint32_t crc0, pad;
  unsigned long long a, b;
};

}  // namespace zb

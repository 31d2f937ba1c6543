// Exact DEFLATE block-size arithmetic, shared by host code (block splitter, emitter) and by the
// sm_90a kernels (per-iteration block cost inside the iterate loop, split-cost evaluation).
//
// What the reference computes here (citations relative to /root/reference/src/zopfli/):
//   ZopfliLengthLimitedCodeLengths  katajainen.c:172-262   -> length_limited()
//   PatchDistanceCodesForBuggyDecoders deflate.c:86-99     -> patch_distance_codes()
//   EncodeTree(size_only)           deflate.c:105-249      -> encode_tree_size()
//   CalculateTreeSize               deflate.c:277-290      -> best_tree_size()
//   OptimizeHuffmanForRle           deflate.c:434-518      -> optimize_for_rle()
//   CalculateBlockSymbolSize*       deflate.c:348-420      -> symbol_bits()
//   GetDynamicLengths / TryOptimizeHuffmanForRle deflate.c:525-582 -> dynamic_lengths()
//
// The reference's boundary package-merge (a recursive node-pool algorithm) is replaced by the
// classic level-by-level package-merge over flat arrays -- no pointers, no recursion, O(n*L)
// words of scratch -- with the reference's tie rule (a leaf precedes a package only when it is
// STRICTLY lighter, katajainen.c:93-104).  Bit-identical lengths; checked against the compiled
// reference in tests/test_host_logic.py.
#pragma once
#include <stdint.h>

#include "symbols.hpp"

namespace zb {

template <int NMAX, int LMAX>
struct PmScratch {
  uint32_t key[NMAX];                     // leaves sorted by (weight << 9 | symbol)
  uint32_t row[2][2 * NMAX - 2];          // item weights of the previous / current level
  uint32_t mask[LMAX][(2 * NMAX + 29) / 32];  // bit = item is a leaf
};

// freq: n counts (< 2^22, as katajainen.c:168-170's int comparator also requires);
// out: n code lengths (0 for unused symbols).
template <int NMAX, int LMAX, typename FreqT, typename OutT>
ZB_HD void length_limited(const FreqT* freq, int n, int maxbits, OutT* out,
                          PmScratch<NMAX, LMAX>& s) {
  int ns = 0;
  for (int i = 0; i < n; i++) {
    out[i] = 0;
    if (freq[i]) s.key[ns++] = ((uint32_t)freq[i] << 9) | (uint32_t)i;
  }
  if (ns == 0) return;                                     // katajainen.c:208-211
  if (ns == 1) { out[s.key[0] & 511] = 1; return; }        // :212-216
  if (ns == 2) { out[s.key[0] & 511] = 1; out[s.key[1] & 511] = 1; return; }  // :217-222
  // katajainen.c:224-235: sort by weight, symbol index breaking ties (keys are unique).
  // Shell sort: no recursion, in place.
  for (int gap = ns >> 1; gap > 0; gap = (gap == 2) ? 1 : (gap * 5) / 11) {
    for (int i = gap; i < ns; i++) {
      uint32_t k = s.key[i];
      int j = i;
      while (j >= gap && s.key[j - gap] > k) { s.key[j] = s.key[j - gap]; j -= gap; }
      s.key[j] = k;
    }
  }
  if (ns - 1 < maxbits) maxbits = ns - 1;                  // :238-240
  const int maxitems = 2 * ns - 2;  // only the first 2n-2 items of any level can be selected
  const int mwords = (maxitems + 31) >> 5;
  // level 0: the leaves
  int prevlen = ns;
  for (int i = 0; i < ns; i++) s.row[0][i] = s.key[i] >> 9;
  for (int w = 0; w < mwords; w++) s.mask[0][w] = 0;
  for (int i = 0; i < ns; i++) s.mask[0][i >> 5] |= 1u << (i & 31);
  int cur = 1;
  for (int lev = 1; lev < maxbits; lev++, cur ^= 1) {
    const uint32_t* prev = s.row[cur ^ 1];
    uint32_t* row = s.row[cur];
    uint32_t* mk = s.mask[lev];
    for (int w = 0; w < mwords; w++) mk[w] = 0;
    const int npk = prevlen >> 1;
    int li = 0, pi = 0, len = 0;
    while (len < maxitems && (li < ns || pi < npk)) {
      bool leaf;
      uint32_t sum = 0;
      if (pi < npk) {
        sum = prev[2 * pi] + prev[2 * pi + 1];
        leaf = li < ns && sum > (s.key[li] >> 9);
      } else {
        leaf = true;
      }
      if (leaf) { row[len] = s.key[li] >> 9; mk[len >> 5] |= 1u << (len & 31); li++; }
      else { row[len] = sum; pi++; }
      len++;
    }
    prevlen = len;
  }
  // Selection (ExtractBitLengths katajainen.c:145-163): take the first 2n-2 items of the last
  // level; p selected packages pull in the first 2p items of the level below.  A leaf of
  // sorted rank r gets one bit per level whose selected-leaf count exceeds r.
  int need = maxitems;
  for (int lev = maxbits - 1; lev >= 0; lev--) {
    const uint32_t* mk = s.mask[lev];
    int c = 0, full = need >> 5, rem = need & 31;
    for (int w = 0; w < full; w++) {
#if defined(__CUDA_ARCH__)
      c += __popc(mk[w]);
#else
      c += __builtin_popcount(mk[w]);
#endif
    }
    if (rem) {
      uint32_t v = mk[full] & ((1u << rem) - 1);
#if defined(__CUDA_ARCH__)
      c += __popc(v);
#else
      c += __builtin_popcount(v);
#endif
    }
    for (int i = 0; i < c; i++) out[s.key[i] & 511]++;
    need = 2 * (need - c);
  }
}

template <typename LenT>
ZB_HD void patch_distance_codes(LenT* d_lengths) {  // deflate.c:86-99
  int num = 0;
  for (int i = 0; i < 30; i++) {
    if (d_lengths[i]) num++;
    if (num >= 2) return;
  }
  if (num == 0) d_lengths[0] = d_lengths[1] = 1;
  else if (num == 1) d_lengths[d_lengths[0] ? 1 : 0] = 1;
}

// ---- code-length RLE of the tree header (deflate.c:105-249) ----
// The transmitted sequence is ll_len[0 .. hlit+257) followed by d_len[0 .. hdist+1).  tok(sym, extra)
// is called for every token in stream order: sym 0..15 = a literal code length, 16/17/18 = repeat
// codes with their extra value.  Token counts per run come from closed forms (quotient / remainder
// by the repeat capacity) -- the same function serves size evaluation (counting functor) and
// emission (emit_bits.hpp, writing functor), so the two can never disagree.
struct TreeShape { unsigned hlit, hdist, total; };

template <typename LenT>
ZB_HD TreeShape tree_shape(const LenT* ll_len, const LenT* d_len) {
  TreeShape s;
  s.hlit = 29;
  s.hdist = 29;
  while (s.hlit > 0 && ll_len[256 + s.hlit] == 0) s.hlit--;   // trailing zeros are not sent (deflate.c:133-136)
  while (s.hdist > 0 && d_len[s.hdist] == 0) s.hdist--;
  s.total = s.hlit + 257 + s.hdist + 1;
  return s;
}

template <typename LenT, typename Tok>
ZB_HD void tree_tokens(const LenT* ll_len, const LenT* d_len, const TreeShape& sh, unsigned flags, Tok tok) {
  const bool use_16 = (flags & 1) != 0, use_17 = (flags & 2) != 0, use_18 = (flags & 4) != 0;
  const unsigned nll = sh.hlit + 257;
  auto at = [&](unsigned i) -> unsigned { return i < nll ? ll_len[i] : d_len[i - nll]; };
  unsigned i = 0;
  while (i < sh.total) {
    const unsigned v = at(i);
    unsigned j = i + 1;
    if (use_16 || (v == 0 && (use_17 || use_18)))   // runs are only looked for where a repeat code could use them
      while (j < sh.total && at(j) == v) j++;
    unsigned c = j - i;   // c equal lengths v
    i = j;
    if (v == 0) {
      if (use_18 && c >= 11) {           // 11..138 zeros per token
        for (unsigned k = c / 138; k; k--) tok(18u, 127u);
        c %= 138;
        if (c >= 11) { tok(18u, c - 11); c = 0; }
      }
      if (use_17 && c >= 3) {            // 3..10 zeros per token
        for (unsigned k = c / 10; k; k--) tok(17u, 7u);
        c %= 10;
        if (c >= 3) { tok(17u, c - 3); c = 0; }
      }
    }
    if (use_16 && c >= 4) {              // the length itself, then "repeat previous" 3..6 times per token
      tok(v, 0u);
      c--;
      for (unsigned k = c / 6; k; k--) tok(16u, 3u);
      c %= 6;
      if (c >= 3) { tok(16u, c - 3); c = 0; }
    }
    for (; c; c--) tok(v, 0u);
  }
}

ZB_HD unsigned clcl_rank_symbol(unsigned k) {  // RFC1951 3.2.7 transmission order of the code-length alphabet
  // 16 17 18 0 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15
  if (k < 3) return 16 + k;
  if (k == 3) return 0;
  const unsigned h = (k - 4) >> 1;
  return (k & 1) ? 7 - h : 8 + h;
}

// Bits of the tree header given the code-length-code counts and clcode_bits = sum of clcl[i] * clcounts[i]
// over their 7-limited code: HCLEN, the code-length code itself, the tokens and their extra bits
ZB_HD uint32_t tree_header_bits_from(const uint32_t* clcounts, uint32_t clcode_bits) {
  unsigned hclen = 15;
  while (hclen > 0 && clcounts[clcl_rank_symbol(hclen + 3)] == 0) hclen--;
  return 14 + (hclen + 4) * 3 + clcode_bits + clcounts[16] * 2 + clcounts[17] * 3 + clcounts[18] * 7;
}

// The rest of EncodeTree(size_only) once the code-length-code counts are known (deflate.c:205-241):
// their length-limited code, HCLEN, and the bits of the header
ZB_HD uint32_t tree_header_bits(const uint32_t* clcounts) {
  uint8_t clcl[19];
  PmScratch<19, 7> s;
  length_limited<19, 7>(clcounts, 19, 7, clcl, s);
  uint32_t r = 0;
  for (int i = 0; i < 19; i++) r += clcl[i] * clcounts[i];
  return tree_header_bits_from(clcounts, r);
}

// The header uses the code-length code only through sum(clcl[i] * clcounts[i]), and every optimal 7-limited
// code has the same sum, so an unconstrained Huffman code no deeper than 7 gives it too.  Builds one in
// registers (19 keys weight << 10 | height << 5 | slot; the lowest height wins among equal weights, which
// keeps the tree shallow) and returns false when it comes out deeper than 7: the caller then takes the
// package-merge (length_limited), which is exact in every case.  0, 1 or 2 used symbols get length 1 each
// (katajainen.c:208-222).  The counts must sum to less than 2^22 (a header has at most 320 tokens).
ZB_HD bool clcode_bits_unlimited(const uint32_t* clcounts, uint32_t* clcode_bits) {
  const uint32_t kNone = 0xffffffffu;
  uint32_t k[19];
  uint32_t ns = 0, total = 0;
ZB_UNROLL
  for (int i = 0; i < 19; i++) {
    const uint32_t c = clcounts[i];
    k[i] = c ? (c << 10) | (uint32_t)i : kNone;
    ns += c ? 1u : 0u;
    total += c;
  }
  if (ns <= 2) { *clcode_bits = total; return true; }
  uint32_t bits = 0, height = 0;
  for (uint32_t m = 1; m < ns; m++) {
    uint32_t m1 = kNone, m2 = kNone;
ZB_UNROLL
    for (int i = 0; i < 19; i++) m1 = k[i] < m1 ? k[i] : m1;
ZB_UNROLL
    for (int i = 0; i < 19; i++) k[i] = k[i] == m1 ? kNone : k[i];
ZB_UNROLL
    for (int i = 0; i < 19; i++) m2 = k[i] < m2 ? k[i] : m2;
    const uint32_t w = (m1 >> 10) + (m2 >> 10), h1 = (m1 >> 5) & 31u, h2 = (m2 >> 5) & 31u;
    height = (h1 > h2 ? h1 : h2) + 1;
    const uint32_t merged = (w << 10) | (height << 5) | (m2 & 31u);
ZB_UNROLL
    for (int i = 0; i < 19; i++) k[i] = k[i] == m2 ? merged : k[i];
    bits += w;   // every leaf under the new node is one bit deeper
  }
  *clcode_bits = bits;
  return height <= 7;
}

// tree_header_bits by clcode_bits_unlimited where its tree fits in 7 bits (the device's way, CPU-testable)
ZB_HD uint32_t tree_header_bits_huffman(const uint32_t* clcounts) {
  uint32_t bits;
  if (clcode_bits_unlimited(clcounts, &bits)) return tree_header_bits_from(clcounts, bits);
  return tree_header_bits(clcounts);
}

// EncodeTree with out == NULL (deflate.c:105-249): bits of the tree header for one flag choice
template <typename LenT>
ZB_HD uint32_t encode_tree_size(const LenT* ll_lengths, const LenT* d_lengths, bool use_16,
                                bool use_17, bool use_18) {
  uint32_t clcounts[19];
  for (int i = 0; i < 19; i++) clcounts[i] = 0;
  const TreeShape sh = tree_shape(ll_lengths, d_lengths);
  tree_tokens(ll_lengths, d_lengths, sh, (use_16 ? 1u : 0u) | (use_17 ? 2u : 0u) | (use_18 ? 4u : 0u),
              [&](unsigned sym, unsigned) { clcounts[sym]++; });
  return tree_header_bits(clcounts);
}

// Code-length-code counts that tree_tokens produces for one maximal run of c equal lengths v (a run
// in the transmitted sequence ll_len[0 .. hlit+257) ++ d_len[0 .. hdist+1)) under `flags`, added
// through add(sym, count).  tree_tokens only extends a run where a repeat code could use it; where it
// does not, each length of the run is a token of its own, which is the c literal tokens below.
template <typename Add>
ZB_HD void run_token_counts(unsigned v, unsigned c, unsigned flags, Add add) {
  const bool use_16 = (flags & 1) != 0, use_17 = (flags & 2) != 0, use_18 = (flags & 4) != 0;
  if (!(use_16 || (v == 0 && (use_17 || use_18)))) { add(v, c); return; }
  if (v == 0) {
    if (use_18 && c >= 11) {
      unsigned n = c / 138;
      c %= 138;
      if (c >= 11) { n++; c = 0; }
      add(18u, n);
    }
    if (use_17 && c >= 3) {
      unsigned n = c / 10;
      c %= 10;
      if (c >= 3) { n++; c = 0; }
      add(17u, n);
    }
  }
  if (use_16 && c >= 4) {
    add(v, 1u);
    c--;
    unsigned n = c / 6;
    c %= 6;
    if (c >= 3) { n++; c = 0; }
    add(16u, n);
  }
  if (c) add(v, c);
}

// deflate.c:277-290 / 251-272: first minimum over the 8 flag combinations.
template <typename LenT>
ZB_HD uint32_t best_tree_size(const LenT* ll_lengths, const LenT* d_lengths, int* best_flags) {
  uint32_t best = 0;
  int bf = 0;
  for (int i = 0; i < 8; i++) {
    uint32_t size = encode_tree_size(ll_lengths, d_lengths, (i & 1) != 0, (i & 2) != 0, (i & 4) != 0);
    if (best == 0 || size < best) { best = size; bf = i; }
  }
  if (best_flags) *best_flags = bf;
  return best;
}

// deflate.c:379-401 (the `Small` variant :348-374 adds up the same integers symbol by symbol)
template <typename CntT, typename LenT>
ZB_HD uint64_t symbol_bits(const CntT* llc, const CntT* dc, const LenT* ll, const LenT* d) {
  uint64_t r = 0;
  for (int i = 0; i < 256; i++) r += (uint64_t)ll[i] * llc[i];
  for (int i = 257; i < 286; i++) r += (uint64_t)(ll[i] + length_symbol_extra_bits(i)) * llc[i];
  for (int i = 0; i < 30; i++) r += (uint64_t)(d[i] + dist_symbol_extra_bits(i)) * dc[i];
  return r + ll[256];
}

// OptimizeHuffmanForRle (deflate.c:434-518) as three passes over RUNS instead of one flag-driven
// scan: (1) drop trailing zeros; (2) every maximal run of equal counts that is long enough for an
// RLE code (>= 5 zeros, >= 7 non-zeros) is pinned; (3) greedy segmentation: a segment grows while the
// next count is unpinned and within 4 of `limit`, a finished segment of >= 4 counts (>= 3 when all zero)
// is flattened to its rounded mean, and the next segment's limit is the mean of the four counts ahead.
// `good` is caller scratch of `length` bytes.
template <typename CntT>
ZB_HD void optimize_for_rle(int length, CntT* counts, uint8_t* good) {
  while (length > 0 && counts[length - 1] == 0) length--;
  if (length == 0) return;
  for (int a = 0; a < length;) {                       // pass 2: pin long runs
    int b = a + 1;
    while (b < length && counts[b] == counts[a]) b++;
    const uint8_t pin = (b - a) >= (counts[a] == 0 ? 5 : 7) ? 1 : 0;
    for (int k = a; k < b; k++) good[k] = pin;
    a = b;
  }
  auto ahead = [&](int i) -> uint64_t {                  // limit for a segment starting at i
    if (i < length - 3) return ((uint64_t)counts[i] + counts[i + 1] + counts[i + 2] + counts[i + 3] + 2) / 4;
    return i < length ? (uint64_t)counts[i] : 0;
  };
  uint64_t limit = good[0] ? ahead(0) : (uint64_t)counts[0];
  for (int a = 0; a < length;) {                       // pass 3: segment, flatten
    int b = a + 1;
    uint64_t sum = counts[a];
    while (b < length && !good[b]) {
      const uint64_t c = counts[b];
      if ((c > limit ? c - limit : limit - c) >= 4) break;
      sum += c;
      b++;
    }
    const int stride = b - a;
    if (stride >= 4 || (stride >= 3 && sum == 0)) {
      uint64_t mean = (sum + (uint64_t)(stride / 2)) / (uint64_t)stride;
      if (mean < 1) mean = 1;
      if (sum == 0) mean = 0;
      for (int k = a; k < b; k++) counts[k] = (CntT)mean;
    }
    limit = ahead(b);
    a = b;
  }
}

// Pass 3 of optimize_for_rle as a function of the segment start.  Pass 3 reads only original counts (a
// segment is flattened after the next limit has been read from the counts at and after its end), and a
// segment that starts at a > 0 always has limit ahead(a); only a = 0 takes counts[0] when position 0 is
// not pinned.  So where the segment that starts at `a` ends is a pure function of a: the device evaluates
// it with one ballot per 32 positions and hops from start to start (warp_optimize_for_rle, iterate.cuh).
// The limit never exceeds the largest count, so it fits the count type.
template <typename CntT>
ZB_HD uint32_t rle_segment_limit(const CntT* counts, int length, bool good0, int a) {
  if (a == 0 && !good0) return (uint32_t)counts[0];
  if (a < length - 3) return (uint32_t)(((uint64_t)counts[a] + counts[a + 1] + counts[a + 2] + counts[a + 3] + 2) / 4);
  return a < length ? (uint32_t)counts[a] : 0u;
}
ZB_HD bool rle_extends(uint32_t c, uint32_t limit) { return (c > limit ? c - limit : limit - c) < 4; }
template <typename CntT>
ZB_HD int rle_segment_end(const CntT* counts, const uint8_t* good, int length, int a) {
  const uint32_t limit = rle_segment_limit(counts, length, good[0] != 0, a);
  int b = a + 1;
  while (b < length && !good[b] && rle_extends((uint32_t)counts[b], limit)) b++;
  return b;
}
// whether a finished segment of `stride` counts summing to `sum` is flattened, and to what value
ZB_HD bool rle_flatten(uint64_t sum, int stride, uint32_t* mean) {
  if (stride < 3 || (stride == 3 && sum != 0)) return false;
  uint64_t m = (sum + (uint64_t)(stride / 2)) / (uint64_t)stride;
  if (m < 1) m = 1;
  if (sum == 0) m = 0;
  *mean = (uint32_t)m;
  return true;
}

// optimize_for_rle in the device's order (CPU model of warp_optimize_for_rle): pinned runs, then every
// segment start found by hopping through rle_segment_end, then each segment flattened.  `good` is caller
// scratch of `length` bytes; length <= 288.
template <typename CntT>
ZB_HD void optimize_for_rle_by_segments(int length, CntT* counts, uint8_t* good) {
  while (length > 0 && counts[length - 1] == 0) length--;
  if (length == 0) return;
  for (int a = 0; a < length;) {
    int b = a + 1;
    while (b < length && counts[b] == counts[a]) b++;
    for (int k = a; k < b; k++) good[k] = (b - a) >= (counts[a] == 0 ? 5 : 7) ? 1 : 0;
    a = b;
  }
  uint32_t starts[(288 + 31) / 32] = {0};
  for (int a = 0; a < length; a = rle_segment_end(counts, good, length, a)) starts[a >> 5] |= 1u << (a & 31);
  for (int a = 0; a < length;) {
    int b = a + 1;
    while (b < length && !((starts[b >> 5] >> (b & 31)) & 1u)) b++;
    uint64_t sum = 0;
    for (int k = a; k < b; k++) sum += counts[k];
    uint32_t mean;
    if (rle_flatten(sum, b - a, &mean))
      for (int k = a; k < b; k++) counts[k] = (CntT)mean;
    a = b;
  }
}

struct DynScratch {
  PmScratch<kNumLL, 15> pm;
  uint32_t llc2[kNumLL];
  uint32_t dc2[kNumD];
  uint8_t ll2[kNumLL];
  uint8_t d2[kNumD];
  uint8_t good[kNumLL];
};

// GetDynamicLengths (deflate.c:569-582): code lengths minimising tree + data bits between the
// plain and the RLE-smoothed histograms.  llc[256] must already be 1.  Returns the bit count
// without the 3 block-header bits.
ZB_HD uint64_t dynamic_lengths(const uint32_t* llc, const uint32_t* dc, uint8_t* ll, uint8_t* d,
                               DynScratch& s) {
  length_limited<kNumLL, 15>(llc, kNumLL, 15, ll, s.pm);
  length_limited<kNumLL, 15>(dc, kNumD, 15, d, s.pm);
  patch_distance_codes(d);
  uint64_t size1 = best_tree_size(ll, d, nullptr) + symbol_bits(llc, dc, ll, d);
  for (int i = 0; i < kNumLL; i++) s.llc2[i] = llc[i];
  for (int i = 0; i < kNumD; i++) s.dc2[i] = dc[i];
  optimize_for_rle(kNumLL, s.llc2, s.good);
  optimize_for_rle(kNumD, s.dc2, s.good);
  length_limited<kNumLL, 15>(s.llc2, kNumLL, 15, s.ll2, s.pm);
  length_limited<kNumLL, 15>(s.dc2, kNumD, 15, s.d2, s.pm);
  patch_distance_codes(s.d2);
  uint64_t size2 = best_tree_size(s.ll2, s.d2, nullptr) + symbol_bits(llc, dc, s.ll2, s.d2);
  if (size2 < size1) {  // deflate.c:553-557
    for (int i = 0; i < kNumLL; i++) ll[i] = s.ll2[i];
    for (int i = 0; i < kNumD; i++) d[i] = s.d2[i];
    return size2;
  }
  return size1;
}

// GetFixedTree deflate.c:335-342
ZB_HD int fixed_ll_length(int i) { return i < 144 ? 8 : (i < 256 ? 9 : (i < 280 ? 7 : 8)); }

template <typename CntT>
ZB_HD uint64_t fixed_symbol_bits(const CntT* llc, const CntT* dc) {
  uint64_t r = 0;
  for (int i = 0; i < 256; i++) r += (uint64_t)fixed_ll_length(i) * llc[i];
  for (int i = 257; i < 286; i++) r += (uint64_t)(fixed_ll_length(i) + length_symbol_extra_bits(i)) * llc[i];
  for (int i = 0; i < 30; i++) r += (uint64_t)(5 + dist_symbol_extra_bits(i)) * dc[i];
  return r + 7;  // end symbol
}

// ZopfliCalculateBlockSize btype 0 (deflate.c:590-597)
ZB_HD uint64_t stored_bits(uint64_t nbytes) {
  uint64_t rem = nbytes % 65535;
  uint64_t blocks = nbytes / 65535 + (rem ? 1 : 0);
  return blocks * 5 * 8 + nbytes * 8;
}

}  // namespace zb

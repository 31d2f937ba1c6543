/*
 * zopfli_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C CPU restatement of google/zopfli's LZ77 optimal-parse hot path, written as
 * PURE FUNCTIONS of (input bytes, block range) -- the same formulation the sm_90a kernels
 * use -- so that every kernel can be diffed against a readable sequential statement of what
 * the reference computes.  Nothing in the product (zopfli_b200/, include/) may include, link
 * or call this; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg do.
 *
 * Parity status: PINNED.  Every function here is checked in tests/test_oracle.py against the
 * unmodified reference compiled from /root/reference by oracle/Makefile (oracle/_ref/), at the
 * three seams SURVEY.md section 4 names (match table, LZ77 store, final bytes).  The reference
 * ships no golden byte vectors of its own (only the Go size bounds, go/zopfli/zopfli_test.go:35-69,
 * restated in tests/test_go_cases.py).
 *
 * Citations are file:line relative to /root/reference/src/zopfli/.
 */
#ifndef ZOPFLI_ORACLE_H_
#define ZOPFLI_ORACLE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* LZ77 symbol list: dists[i]==0 -> literal litlens[i]; else (length, distance). lz77.h:44-62 */
typedef struct ZoStore {
  uint16_t* litlens;
  uint16_t* dists;
  uint32_t* pos;
  size_t size, cap;
} ZoStore;

void zo_store_init(ZoStore* s);
void zo_store_free(ZoStore* s);

/* One parse range [instart, inend) with its 32 KiB history: hash keys, `same` run lengths and
 * both hash chains laid out as position-sorted buckets (hash.c:29-143 as closed forms). */
typedef struct ZoSegment ZoSegment;
ZoSegment* zo_segment_new(const uint8_t* in, size_t instart, size_t inend);
void zo_segment_free(ZoSegment* seg);

/* Closed forms of the per-position hash state (SURVEY App. A.1); p in [winstart, inend). */
unsigned zo_segment_hv(const ZoSegment* seg, size_t p);
unsigned zo_segment_same(const ZoSegment* seg, size_t p);
unsigned zo_segment_hv2(const ZoSegment* seg, size_t p);
/* nearest earlier position on chain 1 / chain 2, or (size_t)-1 */
size_t zo_segment_prev1(const ZoSegment* seg, size_t p);
size_t zo_segment_prev2(const ZoSegment* seg, size_t p);

/* ZopfliFindLongestMatch without the cache (lz77.c:407-542). sublen may be NULL. */
void zo_find_longest_match(const ZoSegment* seg, size_t pos, unsigned limit,
                           uint16_t* sublen, uint16_t* distance, uint16_t* length);

/* ZopfliLZ77Greedy (lz77.c:544-630). */
void zo_lz77_greedy(const uint8_t* in, size_t instart, size_t inend, ZoStore* out);

/* ZopfliLZ77Optimal (squeeze.c:446-526) / ZopfliLZ77OptimalFixed (squeeze.c:528-560). */
void zo_lz77_optimal(const uint8_t* in, size_t instart, size_t inend, int numiterations,
                     ZoStore* out);
/* the same, and the largest statistics sum and count it hands to the entropy (max_sum and max_count are both NULL or both set) */
void zo_lz77_optimal_stats(const uint8_t* in, size_t instart, size_t inend, int numiterations,
                           ZoStore* out, size_t* max_sum, size_t* max_count);
void zo_lz77_optimal_fixed(const uint8_t* in, size_t instart, size_t inend, ZoStore* out);

/* ZopfliLengthLimitedCodeLengths (katajainen.c:172-262), restated as the classic
 * level-by-level package-merge with the reference's tie rule. Returns 0 on success. */
int zo_length_limited_code_lengths(const size_t* frequencies, int n, int maxbits,
                                   unsigned* bitlengths);

/* ZopfliCalculateEntropy (tree.c:71-94). */
void zo_calculate_entropy(const size_t* count, size_t n, double* bitlengths);

/* ZopfliCalculateBlockSize(lz77, 0, size, btype=2) as a function of the histogram only
 * (deflate.c:569-608); ll_counts[256] is forced to 1 like deflate.c:575. */
double zo_dynamic_block_size(const size_t* ll_counts, const size_t* d_counts,
                             unsigned* ll_lengths_out, unsigned* d_lengths_out);

/* OptimizeHuffmanForRle (deflate.c:434-518) */
void zo_optimize_huffman_for_rle(int length, size_t* counts);

#ifdef __cplusplus
}
#endif
#endif

/*
 * zopfli_oracle.c -- TEST INFRASTRUCTURE ONLY (see zopfli_oracle.h).
 *
 * CPU restatement of the zopfli hot path in the pure-function formulation of SURVEY.md
 * Appendix A.  It deliberately does NOT mirror the reference's data structures (rolling hash
 * rings, longest-match cache, boundary package-merge node pool); it restates WHAT they compute:
 *
 *   hash rings (hash.c)            -> closed-form per-position keys + position-sorted buckets
 *   FindLongestMatch (lz77.c:407)  -> walk over bucket slices, same visiting order / stop rules
 *   longest-match cache (cache.c)  -> per-block match table (pure function, computed once)
 *   GetBestLengths (squeeze.c:217) -> push-form DP over the table, fp64 add / fp32 store
 *   FollowPath (squeeze.c:338)     -> table lookup sublen[pos][len]
 *   katajainen.c                   -> classic package-merge with leaf-vs-package tie rule
 *
 * Citations are file:line relative to /root/reference/src/zopfli/.
 */
#include "zopfli_oracle.h"

#include <assert.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define ZO_WINDOW 32768u      /* util.h:41 */
#define ZO_MAX_MATCH 258u     /* util.h:28 */
#define ZO_MIN_MATCH 3u       /* util.h:29 */
#define ZO_MAX_CHAIN_HITS 8192 /* util.h:84 */
#define ZO_NUM_LL 288
#define ZO_NUM_D 32
#define ZO_LARGE 1e30         /* util.h:65 */

/* ------------------------------------------------------------------ symbols.h tables */

static int length_symbol(int l) { /* symbols.h:138-176 */
  if (l < 3) return 0;
  if (l == 258) return 285;
  if (l < 11) return 254 + l;
  {
    int x = l - 3, hb = 0;
    while ((x >> (hb + 1)) != 0) hb++; /* highest bit */
    return 257 + 4 * (hb - 1) + ((x >> (hb - 2)) & 3);
  }
}
static int length_extra_bits(int l) { /* symbols.h:88-110 */
  int s;
  if (l < 11 || l == 258) return 0;
  s = length_symbol(l);
  return (s - 261) / 4;
}
static int length_symbol_extra_bits(int s) { /* symbols.h:222-228 */
  if (s < 265 || s == 285) return 0;
  return (s - 261) / 4;
}
static int dist_symbol(int dist) { /* symbols.h:62-86 */
  if (dist < 5) return dist - 1;
  {
    int x = dist - 1, l = 0, r;
    while ((x >> (l + 1)) != 0) l++;
    r = (x >> (l - 1)) & 1;
    return l * 2 + r;
  }
}
static int dist_extra_bits(int dist) { /* symbols.h:38-41 */
  int x, l = 0;
  if (dist < 5) return 0;
  x = dist - 1;
  while ((x >> (l + 1)) != 0) l++;
  return l - 1;
}
static int dist_symbol_extra_bits(int s) { /* symbols.h:231-237 */
  return s < 4 ? 0 : (s - 2) / 2;
}

/* ------------------------------------------------------------------ store */

void zo_store_init(ZoStore* s) { memset(s, 0, sizeof(*s)); }
void zo_store_free(ZoStore* s) {
  free(s->litlens); free(s->dists); free(s->pos);
  memset(s, 0, sizeof(*s));
}
static void store_push(ZoStore* s, unsigned litlen, unsigned dist, size_t pos) {
  if (s->size == s->cap) {
    s->cap = s->cap ? s->cap * 2 : 1024;
    s->litlens = (uint16_t*)realloc(s->litlens, s->cap * sizeof(uint16_t));
    s->dists = (uint16_t*)realloc(s->dists, s->cap * sizeof(uint16_t));
    s->pos = (uint32_t*)realloc(s->pos, s->cap * sizeof(uint32_t));
  }
  s->litlens[s->size] = (uint16_t)litlen;
  s->dists[s->size] = (uint16_t)dist;
  s->pos[s->size] = (uint32_t)pos;
  s->size++;
}
static void store_copy(const ZoStore* a, ZoStore* b) {
  size_t i;
  b->size = 0;
  for (i = 0; i < a->size; i++) store_push(b, a->litlens[i], a->dists[i], a->pos[i]);
}

/* ------------------------------------------------------------------ segment (hash.c) */

struct ZoSegment {
  const uint8_t* in;
  size_t instart, inend, winstart, n;
  uint16_t *hv, *same, *hv2;   /* index p - winstart */
  uint32_t *idx1, *idx2;       /* positions (relative) sorted by (key, position) */
  uint32_t *rank1, *rank2;     /* inverse permutation */
  uint32_t *bstart1, *bstart2; /* bucket starts, 32769 entries */
};

/* Stable counting sort of positions by 15-bit key == the hash chains of hash.c:110-114,131-135
 * laid out contiguously: walking a bucket downwards from rank[p]-1 visits exactly prev[p],
 * prev[prev[p]], ... (SURVEY App. A.1). */
static void build_chain(const uint16_t* key, size_t n, uint32_t** idx, uint32_t** rank,
                        uint32_t** bstart) {
  size_t i;
  uint32_t* cnt = (uint32_t*)calloc(32769, sizeof(uint32_t));
  *idx = (uint32_t*)malloc((n + 1) * sizeof(uint32_t));
  *rank = (uint32_t*)malloc((n + 1) * sizeof(uint32_t));
  *bstart = (uint32_t*)malloc(32769 * sizeof(uint32_t));
  for (i = 0; i < n; i++) cnt[key[i] + 1]++;
  for (i = 0; i < 32768; i++) cnt[i + 1] += cnt[i];
  memcpy(*bstart, cnt, 32769 * sizeof(uint32_t));
  for (i = 0; i < n; i++) {
    uint32_t d = cnt[key[i]]++;
    (*idx)[d] = (uint32_t)i;
    (*rank)[i] = d;
  }
  free(cnt);
}

ZoSegment* zo_segment_new(const uint8_t* in, size_t instart, size_t inend) {
  ZoSegment* s = (ZoSegment*)calloc(1, sizeof(*s));
  size_t i;
  s->in = in;
  s->instart = instart;
  s->inend = inend;
  s->winstart = instart > ZO_WINDOW ? instart - ZO_WINDOW : 0; /* squeeze.c:229-230 */
  s->n = inend - s->winstart;
  s->hv = (uint16_t*)malloc((s->n + 1) * sizeof(uint16_t));
  s->same = (uint16_t*)malloc((s->n + 1) * sizeof(uint16_t));
  s->hv2 = (uint16_t*)malloc((s->n + 1) * sizeof(uint16_t));
  /* same(p): hash.c:116-126 -- count of following bytes equal to in[p], clipped at `end`
   * and at 65535.  Backward recurrence. */
  for (i = s->n; i-- > 0;) {
    size_t p = s->winstart + i;
    unsigned v = 0;
    if (p + 1 < inend && in[p + 1] == in[p]) {
      v = (unsigned)s->same[i + 1] + 1;
      if (v > 65535) v = 65535;
    }
    s->same[i] = (uint16_t)v;
  }
  for (i = 0; i < s->n; i++) {
    size_t p = s->winstart + i;
    /* hash.c:96-98,107-108: three-byte rolling hash, zero padded past `end` */
    unsigned b0 = in[p], b1 = p + 1 < inend ? in[p + 1] : 0, b2 = p + 2 < inend ? in[p + 2] : 0;
    unsigned hv = ((b0 << 10) ^ (b1 << 5) ^ b2) & 32767u;
    s->hv[i] = (uint16_t)hv;
    /* hash.c:129 */
    s->hv2[i] = (uint16_t)((((int)s->same[i] - (int)ZO_MIN_MATCH) & 255) ^ (int)hv);
  }
  build_chain(s->hv, s->n, &s->idx1, &s->rank1, &s->bstart1);
  build_chain(s->hv2, s->n, &s->idx2, &s->rank2, &s->bstart2);
  return s;
}

void zo_segment_free(ZoSegment* s) {
  if (!s) return;
  free(s->hv); free(s->same); free(s->hv2);
  free(s->idx1); free(s->idx2); free(s->rank1); free(s->rank2);
  free(s->bstart1); free(s->bstart2);
  free(s);
}

unsigned zo_segment_hv(const ZoSegment* s, size_t p) { return s->hv[p - s->winstart]; }
unsigned zo_segment_same(const ZoSegment* s, size_t p) { return s->same[p - s->winstart]; }
unsigned zo_segment_hv2(const ZoSegment* s, size_t p) { return s->hv2[p - s->winstart]; }
size_t zo_segment_prev1(const ZoSegment* s, size_t p) {
  size_t i = p - s->winstart;
  uint32_t r = s->rank1[i];
  if (r == s->bstart1[s->hv[i]]) return (size_t)-1;
  return s->winstart + s->idx1[r - 1];
}
size_t zo_segment_prev2(const ZoSegment* s, size_t p) {
  size_t i = p - s->winstart;
  uint32_t r = s->rank2[i];
  if (r == s->bstart2[s->hv2[i]]) return (size_t)-1;
  return s->winstart + s->idx2[r - 1];
}

/* ------------------------------------------------------------------ lz77.c:407-542 */

void zo_find_longest_match(const ZoSegment* s, size_t pos, unsigned limit, uint16_t* sublen,
                           uint16_t* distance, uint16_t* length) {
  const uint8_t* in = s->in;
  size_t ip = pos - s->winstart;
  unsigned best = 1, bestdist = 0;
  int hops = ZO_MAX_CHAIN_HITS;
  int chain = 1;
  const uint32_t* idx = s->idx1;
  uint32_t lo = s->bstart1[s->hv[ip]];
  uint32_t cur = s->rank1[ip];
  unsigned same0 = s->same[ip], v2 = s->hv2[ip];

  if (s->inend - pos < ZO_MIN_MATCH) { /* lz77.c:440-446 */
    *length = 0;
    *distance = 0;
    return;
  }
  if (pos + limit > s->inend) limit = (unsigned)(s->inend - pos); /* lz77.c:448-450 */

  while (cur > lo) { /* `p == pp` self link (lz77.c:523) == bucket exhausted */
    size_t iq = idx[cur - 1];
    size_t q = s->winstart + iq;
    unsigned dist = (unsigned)(pos - q);
    unsigned m = 0;
    if (dist >= ZO_WINDOW) break; /* lz77.c:464 */
    while (m < limit && in[q + m] == in[pos + m]) m++; /* GetMatch lz77.c:297-331 */
    if (m > best) { /* lz77.c:495-505 */
      if (sublen) {
        unsigned j;
        for (j = best + 1; j <= m; j++) sublen[j] = (uint16_t)dist;
      }
      bestdist = dist;
      best = m;
      if (m >= limit) break;
    }
    cur--;
    /* lz77.c:509-519: the switch test uses the candidate just processed; the next hop is
     * taken on chain 2 from that candidate. */
    if (chain == 1 && best >= same0 && s->hv2[iq] == v2) {
      chain = 2;
      idx = s->idx2;
      lo = s->bstart2[v2];
      cur = s->rank2[iq];
    }
    if (--hops <= 0) break; /* lz77.c:527-530 */
  }
  *distance = (uint16_t)bestdist;
  *length = (uint16_t)best;
}

/* ------------------------------------------------------------------ lz77.c:544-630 */

static int length_score(int length, int distance) { /* lz77.c:265-271 */
  return distance > 1024 ? length - 1 : length;
}

static void greedy_segment(const ZoSegment* seg, ZoStore* store) {
  const uint8_t* in = seg->in;
  size_t i, inend = seg->inend;
  uint16_t sub[259];
  unsigned prev_length = 0, prev_match = 0;
  int match_available = 0;
  for (i = seg->instart; i < inend; i++) {
    uint16_t leng, dist;
    int lengthscore, prevlengthscore;
    zo_find_longest_match(seg, i, ZO_MAX_MATCH, sub, &dist, &leng);
    lengthscore = length_score(leng, dist);
    prevlengthscore = length_score((int)prev_length, (int)prev_match);
    if (match_available) { /* lz77.c:584-609 */
      match_available = 0;
      if (lengthscore > prevlengthscore + 1) {
        store_push(store, in[i - 1], 0, i - 1);
        if (lengthscore >= (int)ZO_MIN_MATCH && leng < ZO_MAX_MATCH) {
          match_available = 1;
          prev_length = leng;
          prev_match = dist;
          continue;
        }
      } else {
        leng = (uint16_t)prev_length;
        dist = (uint16_t)prev_match;
        store_push(store, leng, dist, i - 1);
        i += leng - 2; /* loop `for (j = 2; j < leng; j++) i++` lz77.c:603-607 */
        continue;
      }
    } else if (lengthscore >= (int)ZO_MIN_MATCH && leng < ZO_MAX_MATCH) { /* lz77.c:610-615 */
      match_available = 1;
      prev_length = leng;
      prev_match = dist;
      continue;
    }
    if (lengthscore >= (int)ZO_MIN_MATCH) { /* lz77.c:619-625 */
      store_push(store, leng, dist, i);
    } else {
      leng = 1;
      store_push(store, in[i], 0, i);
    }
    i += leng - 1;
  }
}

void zo_lz77_greedy(const uint8_t* in, size_t instart, size_t inend, ZoStore* out) {
  ZoSegment* seg;
  if (instart == inend) return;
  seg = zo_segment_new(in, instart, inend);
  greedy_segment(seg, out);
  zo_segment_free(seg);
}

/* ------------------------------------------------------------------ tree.c:71-94 */

void zo_calculate_entropy(const size_t* count, size_t n, double* bitlengths) {
  static const double kInvLog2 = 1.4426950408889; /* tree.c:72 (truncated constant) */
  unsigned sum = 0, i;
  double log2sum;
  for (i = 0; i < n; ++i) sum += (unsigned)count[i];
  log2sum = (sum == 0 ? log((double)n) : log((double)sum)) * kInvLog2;
  for (i = 0; i < n; ++i) {
    if (count[i] == 0) bitlengths[i] = log2sum;
    else bitlengths[i] = log2sum - log((double)count[i]) * kInvLog2;
    if (bitlengths[i] < 0 && bitlengths[i] > -1e-5) bitlengths[i] = 0; /* tree.c:91 */
  }
}

/* ------------------------------------------------------------------ katajainen.c */

typedef struct { size_t w; int sym; } ZoLeaf;
static int leaf_cmp(const void* a, const void* b) {
  const ZoLeaf* x = (const ZoLeaf*)a; const ZoLeaf* y = (const ZoLeaf*)b;
  if (x->w != y->w) return x->w < y->w ? -1 : 1;
  return x->sym - y->sym; /* katajainen.c:224-235: (weight << 9) | symbol keys */
}

int zo_length_limited_code_lengths(const size_t* freq, int n, int maxbits, unsigned* bl) {
  ZoLeaf* leaves = (ZoLeaf*)malloc((size_t)n * sizeof(ZoLeaf));
  int ns = 0, i, lev, need;
  size_t *prev, *cur, prevlen, curlen;
  unsigned char* isleaf; /* [maxbits][2*ns] */
  int maxitems;
  for (i = 0; i < n; i++) bl[i] = 0;
  for (i = 0; i < n; i++) if (freq[i]) { leaves[ns].w = freq[i]; leaves[ns].sym = i; ns++; }
  if ((1 << maxbits) < ns) { free(leaves); return 1; } /* katajainen.c:204-207 */
  if (ns == 0) { free(leaves); return 0; }
  if (ns == 1) { bl[leaves[0].sym] = 1; free(leaves); return 0; } /* :212-216 */
  if (ns == 2) { bl[leaves[0].sym]++; bl[leaves[1].sym]++; free(leaves); return 0; } /* :217-222 */
  qsort(leaves, (size_t)ns, sizeof(ZoLeaf), leaf_cmp);
  if (ns - 1 < maxbits) maxbits = ns - 1; /* katajainen.c:238-240 */

  /* Level 0 holds the sorted leaves only.  Level L+1 merges the leaves with the packages
   * (consecutive pairs) of level L; a leaf goes first only when it is STRICTLY lighter than
   * the pending package (BoundaryPM, katajainen.c:93-104: `sum > leaves[lastcount].weight`).
   * Only the first 2*ns-2 items of any level can ever be selected. */
  maxitems = 2 * ns - 2;
  prev = (size_t*)malloc((size_t)maxitems * sizeof(size_t));
  cur = (size_t*)malloc((size_t)maxitems * sizeof(size_t));
  isleaf = (unsigned char*)malloc((size_t)maxbits * (size_t)maxitems);
  prevlen = (size_t)ns;
  for (i = 0; i < ns; i++) { prev[i] = leaves[i].w; isleaf[i] = 1; }
  for (lev = 1; lev < maxbits; lev++) {
    unsigned char* row = isleaf + (size_t)lev * (size_t)maxitems;
    size_t npk = prevlen / 2, li = 0, pi = 0;
    size_t* t;
    curlen = 0;
    while ((int)curlen < maxitems && (li < (size_t)ns || pi < npk)) {
      if (pi < npk) {
        size_t sum = prev[2 * pi] + prev[2 * pi + 1];
        if (li < (size_t)ns && sum > leaves[li].w) { cur[curlen] = leaves[li].w; row[curlen] = 1; li++; }
        else { cur[curlen] = sum; row[curlen] = 0; pi++; }
      } else { cur[curlen] = leaves[li].w; row[curlen] = 1; li++; }
      curlen++;
    }
    t = prev; prev = cur; cur = t;
    prevlen = curlen;
  }
  /* Selection: the first 2*ns-2 items of the last level; each selected package pulls in the
   * first 2*p items of the level below (ExtractBitLengths, katajainen.c:145-163). */
  need = maxitems;
  for (lev = maxbits - 1; lev >= 0; lev--) {
    unsigned char* row = isleaf + (size_t)lev * (size_t)maxitems;
    int c = 0;
    for (i = 0; i < need; i++) c += row[i];
    for (i = 0; i < c; i++) bl[leaves[i].sym]++;
    need = 2 * (need - c);
  }
  free(prev); free(cur); free(isleaf); free(leaves);
  return 0;
}

/* ------------------------------------------------------------------ deflate.c size estimators */

static void patch_distance_codes(unsigned* d_lengths) { /* deflate.c:86-99 */
  int num = 0, i;
  for (i = 0; i < 30; i++) {
    if (d_lengths[i]) num++;
    if (num >= 2) return;
  }
  if (num == 0) d_lengths[0] = d_lengths[1] = 1;
  else if (num == 1) d_lengths[d_lengths[0] ? 1 : 0] = 1;
}

/* EncodeTree(size_only) deflate.c:105-249 */
static size_t encode_tree_size(const unsigned* ll_lengths, const unsigned* d_lengths, int use_16,
                               int use_17, int use_18) {
  unsigned lld_total, hlit = 29, hdist = 29, hclen, hlit2, i, j;
  size_t clcounts[19];
  unsigned clcl[19];
  static const unsigned order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  size_t result = 0;
  for (i = 0; i < 19; i++) clcounts[i] = 0;
  while (hlit > 0 && ll_lengths[257 + hlit - 1] == 0) hlit--;
  while (hdist > 0 && d_lengths[1 + hdist - 1] == 0) hdist--;
  hlit2 = hlit + 257;
  lld_total = hlit2 + hdist + 1;
  for (i = 0; i < lld_total; i++) {
    unsigned char symbol = (unsigned char)(i < hlit2 ? ll_lengths[i] : d_lengths[i - hlit2]);
    unsigned count = 1;
    if (use_16 || (symbol == 0 && (use_17 || use_18))) {
      for (j = i + 1; j < lld_total && symbol == (j < hlit2 ? ll_lengths[j] : d_lengths[j - hlit2]); j++) count++;
    }
    i += count - 1;
    if (symbol == 0 && count >= 3) {
      if (use_18) while (count >= 11) { unsigned c2 = count > 138 ? 138 : count; clcounts[18]++; count -= c2; }
      if (use_17) while (count >= 3) { unsigned c2 = count > 10 ? 10 : count; clcounts[17]++; count -= c2; }
    }
    if (use_16 && count >= 4) {
      count--;
      clcounts[symbol]++;
      while (count >= 3) { unsigned c2 = count > 6 ? 6 : count; clcounts[16]++; count -= c2; }
    }
    clcounts[symbol] += count;
  }
  zo_length_limited_code_lengths(clcounts, 19, 7, clcl);
  hclen = 15;
  while (hclen > 0 && clcounts[order[hclen + 4 - 1]] == 0) hclen--;
  result += 14;
  result += (hclen + 4) * 3;
  for (i = 0; i < 19; i++) result += clcl[i] * clcounts[i];
  result += clcounts[16] * 2;
  result += clcounts[17] * 3;
  result += clcounts[18] * 7;
  return result;
}

static size_t tree_size(const unsigned* ll, const unsigned* d) { /* deflate.c:277-290 */
  size_t result = 0;
  int i;
  for (i = 0; i < 8; i++) {
    size_t size = encode_tree_size(ll, d, i & 1, i & 2, i & 4);
    if (result == 0 || size < result) result = size;
  }
  return result;
}

static size_t symbol_size(const size_t* llc, const size_t* dc, const unsigned* ll, const unsigned* d) {
  /* CalculateBlockSymbolSizeGivenCounts deflate.c:379-401 (the `Small` variant :348-374 sums
   * the same integers symbol by symbol) */
  size_t result = 0;
  int i;
  for (i = 0; i < 256; i++) result += ll[i] * llc[i];
  for (i = 257; i < 286; i++) result += (ll[i] + (unsigned)length_symbol_extra_bits(i)) * llc[i];
  for (i = 0; i < 30; i++) result += (d[i] + (unsigned)dist_symbol_extra_bits(i)) * dc[i];
  result += ll[256];
  return result;
}

void zo_optimize_huffman_for_rle(int length, size_t* counts) { /* deflate.c:434-518 */
  int i, k, stride;
  size_t symbol, sum, limit;
  unsigned char good[ZO_NUM_LL];
  for (; length >= 0; --length) {
    if (length == 0) return;
    if (counts[length - 1] != 0) break;
  }
  for (i = 0; i < length; ++i) good[i] = 0;
  symbol = counts[0];
  stride = 0;
  for (i = 0; i < length + 1; ++i) {
    if (i == length || counts[i] != symbol) {
      if ((symbol == 0 && stride >= 5) || (symbol != 0 && stride >= 7))
        for (k = 0; k < stride; ++k) good[i - k - 1] = 1;
      stride = 1;
      if (i != length) symbol = counts[i];
    } else {
      ++stride;
    }
  }
  stride = 0;
  limit = counts[0];
  sum = 0;
  for (i = 0; i < length + 1; ++i) {
    size_t ad = 0;
    if (i != length) ad = counts[i] > limit ? counts[i] - limit : limit - counts[i];
    if (i == length || good[i] || ad >= 4) {
      if (stride >= 4 || (stride >= 3 && sum == 0)) {
        int count = (int)((sum + (size_t)stride / 2) / (size_t)stride);
        if (count < 1) count = 1;
        if (sum == 0) count = 0;
        for (k = 0; k < stride; ++k) counts[i - k - 1] = (size_t)count;
      }
      stride = 0;
      sum = 0;
      if (i < length - 3) limit = (counts[i] + counts[i + 1] + counts[i + 2] + counts[i + 3] + 2) / 4;
      else if (i < length) limit = counts[i];
      else limit = 0;
    }
    ++stride;
    if (i != length) sum += counts[i];
  }
}

double zo_dynamic_block_size(const size_t* ll_in, const size_t* d_in, unsigned* ll_out,
                             unsigned* d_out) {
  /* GetDynamicLengths deflate.c:569-582 + TryOptimizeHuffmanForRle :525-560 + 3 header bits :588 */
  size_t llc[ZO_NUM_LL], dc[ZO_NUM_D], llc2[ZO_NUM_LL], dc2[ZO_NUM_D];
  unsigned ll[ZO_NUM_LL], d[ZO_NUM_D], ll2[ZO_NUM_LL], d2[ZO_NUM_D];
  double treesize, datasize, treesize2, datasize2, result;
  memcpy(llc, ll_in, sizeof(llc));
  memcpy(dc, d_in, sizeof(dc));
  llc[256] = 1;
  zo_length_limited_code_lengths(llc, ZO_NUM_LL, 15, ll);
  zo_length_limited_code_lengths(dc, ZO_NUM_D, 15, d);
  patch_distance_codes(d);
  treesize = (double)tree_size(ll, d);
  datasize = (double)symbol_size(llc, dc, ll, d);
  memcpy(llc2, llc, sizeof(llc));
  memcpy(dc2, dc, sizeof(dc));
  zo_optimize_huffman_for_rle(ZO_NUM_LL, llc2);
  zo_optimize_huffman_for_rle(ZO_NUM_D, dc2);
  zo_length_limited_code_lengths(llc2, ZO_NUM_LL, 15, ll2);
  zo_length_limited_code_lengths(dc2, ZO_NUM_D, 15, d2);
  patch_distance_codes(d2);
  treesize2 = (double)tree_size(ll2, d2);
  datasize2 = (double)symbol_size(llc, dc, ll2, d2);
  if (treesize2 + datasize2 < treesize + datasize) {
    memcpy(ll, ll2, sizeof(ll));
    memcpy(d, d2, sizeof(d));
    result = treesize2 + datasize2;
  } else {
    result = treesize + datasize;
  }
  if (ll_out) memcpy(ll_out, ll, sizeof(ll));
  if (d_out) memcpy(d_out, d, sizeof(d));
  return 3 + result;
}

/* ------------------------------------------------------------------ squeeze.c */

typedef struct {
  size_t litlens[ZO_NUM_LL];
  size_t dists[ZO_NUM_D];
  double ll_symbols[ZO_NUM_LL];
  double d_symbols[ZO_NUM_D];
} ZoStats;

static void calc_statistics(ZoStats* st) { /* squeeze.c:392-395 */
  zo_calculate_entropy(st->litlens, ZO_NUM_LL, st->ll_symbols);
  zo_calculate_entropy(st->dists, ZO_NUM_D, st->d_symbols);
}
static void get_statistics(const ZoStore* store, ZoStats* st) { /* squeeze.c:398-411 */
  size_t i;
  for (i = 0; i < store->size; i++) {
    if (store->dists[i] == 0) st->litlens[store->litlens[i]]++;
    else {
      st->litlens[length_symbol(store->litlens[i])]++;
      st->dists[dist_symbol(store->dists[i])]++;
    }
  }
  st->litlens[256] = 1;
  calc_statistics(st);
}

/* GetCostStat squeeze.c:146-157 -- association (lbits + dbits) + ll + d, all in double */
static double cost_stat(unsigned litlen, unsigned dist, const ZoStats* st) {
  if (dist == 0) return st->ll_symbols[litlen];
  {
    int lsym = length_symbol((int)litlen), lbits = length_extra_bits((int)litlen);
    int dsym = dist_symbol((int)dist), dbits = dist_extra_bits((int)dist);
    return lbits + dbits + st->ll_symbols[lsym] + st->d_symbols[dsym];
  }
}

static double model_min_cost(const ZoStats* st) { /* squeeze.c:163-198 */
  static const int dsymbols[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257,
    385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
  double mincost = ZO_LARGE;
  int bestlength = 0, bestdist = 0, i;
  for (i = 3; i < 259; i++) {
    double c = cost_stat((unsigned)i, 1, st);
    if (c < mincost) { bestlength = i; mincost = c; }
  }
  mincost = ZO_LARGE;
  for (i = 0; i < 30; i++) {
    double c = cost_stat(3, (unsigned)dsymbols[i], st);
    if (c < mincost) { bestdist = dsymbols[i]; mincost = c; }
  }
  return cost_stat((unsigned)bestlength, (unsigned)bestdist, st);
}

/* Per-block match table: the pure-function replacement of the longest-match cache. */
typedef struct {
  uint16_t* length;   /* [nb] */
  uint32_t* runoff;   /* [nb+1] offsets into runs */
  uint32_t* runs;     /* (len_end << 16) | dist, ascending len_end */
  uint8_t* skipped;   /* [nb] long-run shortcut mask, squeeze.c:251-271 */
} ZoTable;

static void table_build(const ZoSegment* seg, ZoTable* t) {
  size_t nb = seg->inend - seg->instart, j, cap = nb * 2 + 16, nr = 0;
  uint16_t sub[259];
  t->length = (uint16_t*)malloc((nb + 1) * sizeof(uint16_t));
  t->runoff = (uint32_t*)malloc((nb + 2) * sizeof(uint32_t));
  t->runs = (uint32_t*)malloc(cap * sizeof(uint32_t));
  t->skipped = (uint8_t*)calloc(nb + 1, 1);
  for (j = 0; j < nb; j++) {
    uint16_t leng, dist;
    unsigned k;
    zo_find_longest_match(seg, seg->instart + j, ZO_MAX_MATCH, sub, &dist, &leng);
    if (leng < ZO_MIN_MATCH) leng = 0; /* lz77.c:399-400 */
    t->length[j] = leng;
    t->runoff[j] = (uint32_t)nr;
    if (nr + 260 > cap) { cap *= 2; t->runs = (uint32_t*)realloc(t->runs, cap * sizeof(uint32_t)); }
    for (k = 3; k <= leng; k++)
      if (k == leng || sub[k] != sub[k + 1]) t->runs[nr++] = ((uint32_t)k << 16) | sub[k];
  }
  t->runoff[nb] = (uint32_t)nr;
  /* Long-run shortcut as a mask over source positions (SURVEY App. A.4): depends only on
   * same[] and the block range. */
  {
    size_t i = seg->instart;
    while (i < seg->inend) {
      if (zo_segment_same(seg, i) > ZO_MAX_MATCH * 2 && i > seg->instart + ZO_MAX_MATCH + 1 &&
          i + ZO_MAX_MATCH * 2 + 1 < seg->inend &&
          zo_segment_same(seg, i - ZO_MAX_MATCH) > ZO_MAX_MATCH) {
        for (j = 0; j < ZO_MAX_MATCH; j++) t->skipped[i - seg->instart + j] = 1;
        i += ZO_MAX_MATCH; /* position i (after the run of 258) is processed normally */
      }
      i++;
    }
  }
}
static void table_free(ZoTable* t) { free(t->length); free(t->runoff); free(t->runs); free(t->skipped); }

static unsigned table_dist(const ZoTable* t, size_t j, unsigned len) {
  uint32_t r;
  for (r = t->runoff[j]; r < t->runoff[j + 1]; r++)
    if ((t->runs[r] >> 16) >= len) return t->runs[r] & 0xffff;
  assert(0);
  return 0;
}

/* Optional observer of every DP pass (oracle/dp_int_model.c checks the kernels' integer restatement
 * of the cost arithmetic against the result computed below).  NULL in the oracle library proper. */
typedef void (*ZoDpObserver)(const ZoSegment* seg, const ZoTable* t, const ZoStats* st,
                             const uint16_t* length_array, const float* costs);
static ZoDpObserver zo_dp_observer = NULL;
static void best_lengths_ref(const ZoSegment* seg, const ZoTable* t, const ZoStats* st,
                             uint16_t* length_array, float* costs);
static void best_lengths(const ZoSegment* seg, const ZoTable* t, const ZoStats* st,
                         uint16_t* length_array, float* costs) {
  best_lengths_ref(seg, t, st, length_array, costs);
  if (zo_dp_observer) zo_dp_observer(seg, t, st, length_array, costs);
}

/* GetBestLengths squeeze.c:217-309 */
static void best_lengths_ref(const ZoSegment* seg, const ZoTable* t, const ZoStats* st,
                             uint16_t* length_array, float* costs) {
  const uint8_t* in = seg->in;
  size_t nb = seg->inend - seg->instart, j, k;
  double mincost = model_min_cost(st);
  double cost258 = cost_stat(ZO_MAX_MATCH, 1, st);
  for (j = 1; j < nb + 1; j++) costs[j] = (float)ZO_LARGE;
  costs[0] = 0;
  length_array[0] = 0;
  for (j = 0; j < nb; j++) {
    size_t i = seg->instart + j, kend;
    unsigned leng;
    uint32_t r;
    double mc;
    if (t->skipped[j]) { /* squeeze.c:258-267 */
      costs[j + ZO_MAX_MATCH] = (float)(costs[j] + cost258);
      length_array[j + ZO_MAX_MATCH] = ZO_MAX_MATCH;
      continue;
    }
    { /* literal squeeze.c:277-284 */
      double nc = cost_stat(in[i], 0, st) + costs[j];
      if (nc < costs[j + 1]) { costs[j + 1] = (float)nc; length_array[j + 1] = 1; }
    }
    leng = t->length[j];
    kend = leng < nb - j ? leng : nb - j;
    mc = mincost + costs[j];
    r = t->runoff[j];
    for (k = 3; k <= kend; k++) { /* squeeze.c:286-302 */
      double nc;
      while ((t->runs[r] >> 16) < k) r++;
      if (costs[j + k] <= mc) continue;
      nc = cost_stat((unsigned)k, t->runs[r] & 0xffff, st) + costs[j];
      if (nc < costs[j + k]) { costs[j + k] = (float)nc; length_array[j + k] = (uint16_t)k; }
    }
  }
}

/* TraceBackwards squeeze.c:317-336 + FollowPath squeeze.c:338-389 (distance = table lookup,
 * SURVEY App. A.3) */
static void trace_and_follow(const ZoSegment* seg, const ZoTable* t, const uint16_t* length_array,
                             ZoStore* store) {
  size_t nb = seg->inend - seg->instart, idx = nb, np = 0, i, pos;
  uint16_t* path;
  if (nb == 0) return;
  path = (uint16_t*)malloc((nb + 1) * sizeof(uint16_t));
  for (;;) {
    path[np++] = length_array[idx];
    assert(length_array[idx] != 0 && length_array[idx] <= idx);
    idx -= length_array[idx];
    if (idx == 0) break;
  }
  pos = 0;
  for (i = np; i-- > 0;) {
    unsigned len = path[i];
    if (len >= ZO_MIN_MATCH) {
      store_push(store, len, table_dist(t, pos, len), seg->instart + pos);
    } else {
      len = 1;
      store_push(store, seg->in[seg->instart + pos], 0, seg->instart + pos);
    }
    pos += len;
  }
  free(path);
}

static void store_histogram(const ZoStore* s, size_t* llc, size_t* dc) {
  size_t i;
  memset(llc, 0, ZO_NUM_LL * sizeof(size_t));
  memset(dc, 0, ZO_NUM_D * sizeof(size_t));
  for (i = 0; i < s->size; i++) {
    if (s->dists[i] == 0) llc[s->litlens[i]]++;
    else { llc[length_symbol(s->litlens[i])]++; dc[dist_symbol(s->dists[i])]++; }
  }
}

typedef struct { unsigned m_w, m_z; } ZoRan;
static unsigned ran(ZoRan* s) { /* squeeze.c:90-94 */
  s->m_z = 36969 * (s->m_z & 65535) + (s->m_z >> 16);
  s->m_w = 18000 * (s->m_w & 65535) + (s->m_w >> 16);
  return (s->m_z << 16) + s->m_w;
}
static void randomize_freqs(ZoRan* s, size_t* freqs, int n) { /* squeeze.c:96-101 */
  int i;
  for (i = 0; i < n; i++)
    if ((ran(s) >> 4) % 3 == 0) freqs[i] = freqs[ran(s) % (unsigned)n];
}

/* the largest sum of either statistics array, and the largest single count, that calc_statistics takes: how far
 * the log table of an implementation that looks up log(n) must reach (the blend and RandomizeFreqs can take the
 * sum past twice the block's symbols) */
static void note_stats(const ZoStats* st, size_t* max_sum, size_t* max_count) {
  size_t sl = 0, sd = 0;
  int k;
  if (!max_sum) return;
  for (k = 0; k < ZO_NUM_LL; k++) {
    sl += st->litlens[k];
    if (st->litlens[k] > *max_count) *max_count = st->litlens[k];
  }
  for (k = 0; k < ZO_NUM_D; k++) {
    sd += st->dists[k];
    if (st->dists[k] > *max_count) *max_count = st->dists[k];
  }
  if (sl > *max_sum) *max_sum = sl;
  if (sd > *max_sum) *max_sum = sd;
}

void zo_lz77_optimal(const uint8_t* in, size_t instart, size_t inend, int numiterations,
                     ZoStore* out) {
  zo_lz77_optimal_stats(in, instart, inend, numiterations, out, NULL, NULL);
}

void zo_lz77_optimal_stats(const uint8_t* in, size_t instart, size_t inend, int numiterations,
                           ZoStore* out, size_t* max_sum, size_t* max_count) {
  size_t nb = inend - instart;
  ZoSegment* seg;
  ZoTable tab;
  ZoStore current;
  ZoStats stats, beststats, laststats;
  uint16_t* length_array;
  float* costs;
  double cost, bestcost = ZO_LARGE, lastcost = 0;
  ZoRan rs = {1, 2}; /* squeeze.c:85-88 */
  int lastrandomstep = -1, i;
  out->size = 0;
  if (max_sum) *max_sum = *max_count = 0;
  if (nb == 0) return;
  seg = zo_segment_new(in, instart, inend);
  table_build(seg, &tab);
  length_array = (uint16_t*)malloc((nb + 1) * sizeof(uint16_t));
  costs = (float*)malloc((nb + 1) * sizeof(float));
  zo_store_init(&current);
  memset(&stats, 0, sizeof(stats));
  memset(&beststats, 0, sizeof(beststats));
  greedy_segment(seg, &current); /* squeeze.c:481 */
  get_statistics(&current, &stats);
  note_stats(&stats, max_sum, max_count);
  for (i = 0; i < numiterations; i++) { /* squeeze.c:486-519 */
    size_t llc[ZO_NUM_LL], dc[ZO_NUM_D];
    int k;
    current.size = 0;
    best_lengths(seg, &tab, &stats, length_array, costs);
    trace_and_follow(seg, &tab, length_array, &current);
    store_histogram(&current, llc, dc);
    cost = zo_dynamic_block_size(llc, dc, NULL, NULL); /* squeeze.c:492 */
    if (cost < bestcost) {
      store_copy(&current, out);
      beststats = stats;
      bestcost = cost;
    }
    laststats = stats;
    memset(stats.litlens, 0, sizeof(stats.litlens));
    memset(stats.dists, 0, sizeof(stats.dists));
    get_statistics(&current, &stats);
    note_stats(&stats, max_sum, max_count);
    if (lastrandomstep != -1) { /* squeeze.c:505-511, AddWeighedStatFreqs :65-78 */
      for (k = 0; k < ZO_NUM_LL; k++)
        stats.litlens[k] = (size_t)(stats.litlens[k] * 1.0 + laststats.litlens[k] * 0.5);
      for (k = 0; k < ZO_NUM_D; k++)
        stats.dists[k] = (size_t)(stats.dists[k] * 1.0 + laststats.dists[k] * 0.5);
      stats.litlens[256] = 1;
      calc_statistics(&stats);
      note_stats(&stats, max_sum, max_count);
    }
    if (i > 5 && cost == lastcost) { /* squeeze.c:512-517 */
      stats = beststats;
      randomize_freqs(&rs, stats.litlens, ZO_NUM_LL);
      randomize_freqs(&rs, stats.dists, ZO_NUM_D);
      stats.litlens[256] = 1;
      calc_statistics(&stats);
      note_stats(&stats, max_sum, max_count);
      lastrandomstep = i;
    }
    lastcost = cost;
  }
  free(length_array);
  free(costs);
  zo_store_free(&current);
  table_free(&tab);
  zo_segment_free(seg);
}

void zo_lz77_optimal_fixed(const uint8_t* in, size_t instart, size_t inend, ZoStore* out) {
  /* squeeze.c:528-560 with GetCostFixed (:125-140) expressed as a stat model whose symbol
   * costs are the fixed-tree code lengths: (lbits+dbits) + {7|8} + 5 are exact small integers
   * in double, so the sum is identical whatever the association. */
  size_t nb = inend - instart;
  ZoSegment* seg;
  ZoTable tab;
  ZoStats st;
  uint16_t* length_array;
  float* costs;
  int i;
  out->size = 0;
  if (nb == 0) return;
  memset(&st, 0, sizeof(st));
  for (i = 0; i < 144; i++) st.ll_symbols[i] = 8;
  for (i = 144; i < 256; i++) st.ll_symbols[i] = 9;
  for (i = 256; i < 280; i++) st.ll_symbols[i] = 7;
  for (i = 280; i < 288; i++) st.ll_symbols[i] = 8;
  for (i = 0; i < 32; i++) st.d_symbols[i] = 5;
  seg = zo_segment_new(in, instart, inend);
  table_build(seg, &tab);
  length_array = (uint16_t*)malloc((nb + 1) * sizeof(uint16_t));
  costs = (float*)malloc((nb + 1) * sizeof(float));
  best_lengths(seg, &tab, &st, length_array, costs);
  trace_and_follow(seg, &tab, length_array, out);
  free(length_array);
  free(costs);
  table_free(&tab);
  zo_segment_free(seg);
}

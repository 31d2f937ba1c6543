// sm_90a kernels of the zopfli hot path (SURVEY.md section 8(a) rows a1-a13).
//
// Pipeline per batch of parse ranges ("segments": a master block for the splitter's greedy
// pass, or one deflate block for the optimal parse; both carry their own `inend`, which clips
// matches, `same` and therefore the second hash, exactly like the reference's per-call hash):
//
//   k_same_*      run lengths of equal bytes for the whole input            hash.c:116-126
//   k_keys        hv / hv2 per (segment, position) + bucket histograms      hash.c:96-135
//   k_bucket_scan exclusive scan of the 32768 bucket counts
//   k_scatter     stable counting sort = both hash chains laid out as       hash.c:110-114,131-135
//                 position-sorted buckets (the chains become coalesced lists)
//   k_match       one warp per position: walk the bucket slices 32 candidates  lz77.c:407-542
//                 at a time, replay the sequential best/sublen/switch/hop-cap
//                 semantics with warp scans; emits (len,dist) and the run list
//   k_greedy      lazy-matching greedy parse over the (len,dist) table      lz77.c:544-630
//   k_iterate     persistent CTA per block (DP warp + feeder warp): forward DP, trace-back, follow-path, histogram,
//                 exact dynamic-block size, statistics / entropy / randomisation -- the whole
//                 ZopfliLZ77Optimal loop with no host round trip            squeeze.c:217-526
//
// No tensor-core work exists on this path (no dense contraction); the kernels are integer /
// byte kernels plus a scalar fp64 dependency chain in the DP.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "deflate_size.hpp"
#include "symbols.hpp"

namespace zb {

constexpr uint16_t kShortcutFlag = 0x8000;
constexpr uint32_t kNoEdge = 30;       // dsx value for "no match of this length" (row 30 of the cost table is +inf)
constexpr int kRunSlots = 8;           // table slots per position (cache.c:30-33 keeps 8 too)
constexpr uint32_t kOverflowBit = 0x80000000u;
constexpr int kSameTile = 1024;        // tile of the run-length pre-pass
constexpr uint32_t kNoBreak = 0xffffffffu;

// run-list entry: len_end (9 bits) | dist << 9 (15 bits) | dsym << 24 (5 bits)
__host__ __device__ inline uint32_t run_pack(uint32_t len_end, uint32_t dist) {
  return len_end | (dist << 9) | ((uint32_t)dist_symbol((int)dist) << 24);
}
__host__ __device__ inline uint32_t run_len(uint32_t e) { return e & 511u; }
__host__ __device__ inline uint32_t run_dist(uint32_t e) { return (e >> 9) & 32767u; }
__host__ __device__ inline uint32_t run_dsym(uint32_t e) { return (e >> 24) & 31u; }

// The run list of a parse position, as k_match writes it: entries in increasing len_end (and distance), entry r
// covering the lengths above entry r-1's len_end, in eight slots a = slots 0-3, c = slots 4-7; unused slots are 0.
// A position with more than eight entries keeps the first seven in slots 0-6 and kOverflowBit | off in slot 7,
// and the overflow arena holds ovf[off] = count, then entries 7.. at ovf[off + 1 ..].
// Returns the shortest-distance entry with len_end >= k (what FollowPath's limited search finds, squeeze.c:367).
__device__ __forceinline__ uint32_t run_for_len(uint4 a, uint4 c, uint32_t k, const uint32_t* ovf) {
  uint32_t e = c.w;
  if (c.w & kOverflowBit) {
    e = 0;
    if (k > run_len(c.z)) {
      const uint32_t off = c.w & ~kOverflowBit, cnt = ovf[off];
      for (uint32_t i = 0; i < cnt; i++) { const uint32_t x = ovf[off + 1 + i]; if (run_len(x) >= k) { e = x; break; } }
    }
  }
  if (k <= run_len(c.z)) e = c.z;
  if (k <= run_len(c.y)) e = c.y;
  if (k <= run_len(c.x)) e = c.x;
  if (k <= run_len(a.w)) e = a.w;
  if (k <= run_len(a.z)) e = a.z;
  if (k <= run_len(a.y)) e = a.y;
  if (k <= run_len(a.x)) e = a.x;
  return e;
}

struct SegDesc {
  uint64_t instart, inend, winstart;  // absolute byte positions
  uint64_t key_off;   // element offset of this segment in hv/hv2/idx/rank arrays
  uint64_t pos_off;   // element offset of this segment in per-parse-position arrays
  uint32_t nkeys;     // inend - winstart
  uint32_t npos;      // inend - instart
  int32_t mode;       // 0 greedy only, 1 optimal (iterate), 2 optimal with fixed-tree costs
  int32_t numiterations;
};

struct JobState {   // per segment, written by k_greedy / k_iterate
  uint32_t greedy_size;
  uint32_t best_size;
  uint32_t best_buf;     // which of the 3 store buffers holds the best parse
  uint32_t out_off;      // offset of the packed result (k_pack)
  uint32_t flags;        // bit0: log table overflow (needs host assistance)
  uint32_t iters_done;
  uint32_t int_groups;   // groups of 32 DP steps that ran in the integer window (all iterations)
  uint32_t log_miss;     // with flags bit 0: the value whose log fell outside the table (the host grows it past it)
  uint64_t best_cost;
  uint64_t cyc[6];       // SM cycles spent in: model, DP, trace, follow, block cost, statistics
  uint64_t dpc[5];       // DP cycles by kind of group: integer window, fp64 fast (magic / plain / ring-joining), general
  uint32_t dpn[6];       // groups of each kind; [5] = positions that went through the per-step general loop
};

struct Counters {                // per batch, zeroed before its launches
  unsigned long long ovf_used;   // overflow-arena entries k_match asked for, including those that did not fit (64 bits:
                                 // a batch may ask for more than 2^32, and a wrapped count would hand out used offsets)
  uint32_t out_used;             // symbols of the packed results (k_pack)
  uint32_t pad_;
};

struct Batch {
  const uint8_t* in;        // whole input (device), padded by >= 16 readable bytes
  uint64_t insize;
  const uint16_t* same_g;   // per input byte: min(65535, following equal bytes)
  const SegDesc* segs;
  int nsegs;
  // hash chains as sorted buckets
  uint16_t* hv;
  uint16_t* hv2;
  uint32_t* idx1;
  uint32_t* idx2;
  uint32_t* rank1;
  uint32_t* rank2;
  uint32_t* bkt1;   // [nsegs][32769] counts -> starts
  uint32_t* bkt2;
  // match table
  uint32_t* ld;     // [npos] (len << 16) | dist of the longest match (raw, len may be 0/1/2)
  uint16_t* mlen;   // [npos] longest length or 0 (optimal segments only); bit 15 = long-run
                    // shortcut candidate (squeeze.c:251-257 condition, a pure function of position)
  uint32_t* runs;   // [npos][kRunSlots]
  uint8_t* dsx;     // [npos][32] (row j rotated left by j+3) distance symbol of the shortest-distance match of length 3+l, or
                    // kNoEdge if 3+l exceeds the longest match / the block end (the DP's 32-wide
                    // register window works on these)
  uint32_t* ovf;    // overflow arena: [count, entries...]
  unsigned long long* ovf_used;  // Counters::ovf_used
  uint32_t ovf_cap;              // <= 2^31: slot 7 of a run list holds kOverflowBit | offset
  // parse state
  uint16_t* la;     // [npos + nsegs] length_array, nb+1 per segment (offset pos_off + seg)
  uint64_t* path;   // [npos + nsegs] traced symbols (start position << 9 | length), filled from the end; 64 bits
                    // because a block may hold more than 2^23 positions (build_layout accepts up to 0x7fff0000)
  uint16_t* st_ll[3];
  uint16_t* st_d[3];
  JobState* jobs;
  const double* logtab;      // L[n] = log(n) * 1.4426950408889 (host libm), n in [0, logtab_n)
  uint32_t logtab_n;
  // packed results
  uint16_t* out_ll;
  uint16_t* out_d;
  uint32_t* out_used;       // Counters::out_used
  // verbose: cost of every iteration of every block (squeeze.c:492-495), [nsegs][iter_stride]; null otherwise
  uint64_t* iter_cost;
  uint32_t iter_stride;
  uint32_t dp_flags;   // bit 0: integer window of the forward DP enabled (ZOPFLI_B200_INTDP, default on)
};


// ---------------------------------------------------------------------------------------------
// helpers

__device__ __forceinline__ uint32_t ld_u32_unaligned(const uint8_t* p) {
  const uintptr_t a = (uintptr_t)p;
  const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
  uint32_t lo = __ldg(w), hi = __ldg(w + 1);
  return __funnelshift_r(lo, hi, (uint32_t)(a & 3) * 8);
}

__device__ __forceinline__ uint64_t ld_u64_unaligned(const uint8_t* p) {
  return (uint64_t)ld_u32_unaligned(p) | ((uint64_t)ld_u32_unaligned(p + 4) << 32);
}

// common prefix of in[a..] and in[b..], capped at limit; starts comparing at offset `from`
// (bytes before `from` are known equal or irrelevant to the caller).
__device__ __forceinline__ uint32_t match_len(const uint8_t* a, const uint8_t* b, uint32_t from,
                                              uint32_t limit) {
  uint32_t m = from;
  while (m < limit) {
    uint32_t x = ld_u32_unaligned(a + m) ^ ld_u32_unaligned(b + m);
    if (x) { m += (uint32_t)(__ffs((int)x) - 1) >> 3; break; }
    m += 4;
  }
  return m < limit ? m : limit;
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ---- mbarrier / bulk-copy (TMA 1-D) primitives ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
  } while (!done);
}


// ---------------------------------------------------------------------------------------------
// k_same_*: same_g[p] = min(65535, #{t>=1: in[p+t]==in[p] contiguous}) over the whole input.
// A "break" at e means in[e] != in[e+1] (or e is the last byte).  same_g[p] = nextbreak(p) - p.

__global__ void k_same_tiles(const uint8_t* __restrict__ in, uint64_t n, uint32_t* __restrict__ tile_first) {
  // first break position inside each tile (relative), or kNoBreak
  __shared__ uint32_t first;
  uint64_t tile = blockIdx.x;
  uint64_t base = tile * kSameTile;
  if (threadIdx.x == 0) first = kNoBreak;
  __syncthreads();
  for (uint32_t t = threadIdx.x; t < kSameTile; t += blockDim.x) {
    uint64_t p = base + t;
    if (p < n) {
      bool brk = (p + 1 >= n) || in[p] != in[p + 1];
      if (brk) atomicMin(&first, t);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) tile_first[tile] = first;
}

// next_tile[t] = smallest tile index >= t that contains a break (always exists: last byte breaks).
__global__ void k_same_next_tile(const uint32_t* __restrict__ tile_first, uint32_t ntiles,
                                 uint32_t* __restrict__ next_tile) {
  // single CTA, backward sweep in chunks; ntiles <= insize/1024 so this is tiny
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = ntiles;  // sentinel
  __syncthreads();
  for (int64_t hi = ntiles; hi > 0; hi -= blockDim.x) {
    int64_t t = hi - 1 - threadIdx.x;
    // each thread: nearest tile >= t with a break, searched within this chunk first
    uint32_t mine = kNoBreak;
    if (t >= 0 && tile_first[t] != kNoBreak) mine = (uint32_t)t;
    // suffix-min within the chunk via shared memory (chunk is reversed: thread 0 is highest t)
    __shared__ uint32_t buf[1024];
    buf[threadIdx.x] = mine;
    __syncthreads();
    // thread i needs min over threads j <= i (higher tiles have smaller thread idx) of tiles >= t
    // i.e. the smallest tile index >= t: scan from own index towards lower thread idx is wrong
    // direction (those are higher tiles); we want the closest one, i.e. the largest j <= i
    // with buf[j] != kNoBreak has the smallest tile >= t.
    uint32_t res = kNoBreak;
    for (int j = threadIdx.x; j >= 0; j--) {
      if (buf[j] != kNoBreak) { res = buf[j]; break; }
    }
    if (res == kNoBreak) res = carry;
    if (t >= 0) next_tile[t] = res;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1 || t == 0) {
      // lowest tile of this chunk becomes the carry for the next (lower) chunk
      if (t >= 0) carry = res;
    }
    __syncthreads();
  }
}

__global__ void k_same_fill(const uint8_t* __restrict__ in, uint64_t n,
                            const uint32_t* __restrict__ tile_first,
                            const uint32_t* __restrict__ next_tile, uint32_t ntiles,
                            uint16_t* __restrict__ same_g) {
  __shared__ uint32_t brk[kSameTile];  // per position: 1 if break
  __shared__ uint32_t nb[kSameTile];   // next break position (relative) at or after t, or kNoBreak
  uint64_t tile = blockIdx.x, base = tile * kSameTile;
  for (uint32_t t = threadIdx.x; t < kSameTile; t += blockDim.x) {
    uint64_t p = base + t;
    brk[t] = (p < n) && ((p + 1 >= n) || in[p] != in[p + 1]);
  }
  __syncthreads();
  // backward sweep by warp 0 in 32-wide steps using ballots
  if (threadIdx.x < 32) {
    uint32_t carry = kNoBreak;
    for (int w = kSameTile / 32 - 1; w >= 0; w--) {
      uint32_t t = (uint32_t)w * 32 + threadIdx.x;
      uint32_t mask = __ballot_sync(0xffffffffu, brk[t] != 0);
      uint32_t up = mask & (0xffffffffu << threadIdx.x);  // breaks at lanes >= mine
      uint32_t r = up ? (uint32_t)w * 32 + (uint32_t)(__ffs((int)up) - 1) : carry;
      nb[t] = r;
      if (mask) carry = (uint32_t)w * 32 + (uint32_t)(__ffs((int)mask) - 1);
    }
  }
  __syncthreads();
  for (uint32_t t = threadIdx.x; t < kSameTile; t += blockDim.x) {
    uint64_t p = base + t;
    if (p >= n) continue;
    uint64_t e;
    if (nb[t] != kNoBreak) {
      e = base + nb[t];
    } else {
      uint32_t nt = (tile + 1 < ntiles) ? next_tile[tile + 1] : ntiles;
      e = (nt < ntiles) ? (uint64_t)nt * kSameTile + tile_first[nt] : n - 1;
    }
    uint64_t s = e - p;
    same_g[p] = (uint16_t)(s > 65535 ? 65535 : s);
  }
}

// ---------------------------------------------------------------------------------------------
// k_keys: hv/hv2 per (segment, key position) and bucket histograms.
// work item = (segment, first key) covering kKeyChunk keys.

constexpr int kKeyChunk = 2048;
struct KeyWork { uint32_t seg, first; };

__global__ void k_keys(Batch b, const KeyWork* __restrict__ work) {
  KeyWork w = work[blockIdx.x];
  const SegDesc sd = b.segs[w.seg];
  uint32_t* c1 = b.bkt1 + (uint64_t)w.seg * 32769;
  uint32_t* c2 = b.bkt2 + (uint64_t)w.seg * 32769;
  for (uint32_t t = threadIdx.x; t < kKeyChunk; t += blockDim.x) {
    uint32_t i = w.first + t;
    if (i >= sd.nkeys) break;
    uint64_t p = sd.winstart + i;
    // hash.c:96-98,107-108 (bytes at or past `end` count as 0)
    uint32_t b0 = b.in[p];
    uint32_t b1 = p + 1 < sd.inend ? b.in[p + 1] : 0;
    uint32_t b2 = p + 2 < sd.inend ? b.in[p + 2] : 0;
    uint32_t hv = ((b0 << 10) ^ (b1 << 5) ^ b2) & 32767u;
    // hash.c:116-126 with `end` = this segment's inend
    uint64_t clip = sd.inend - 1 - p;
    uint32_t same = b.same_g[p];
    if ((uint64_t)same > clip) same = (uint32_t)clip;
    uint32_t hv2 = (((int)same - kMinMatch) & 255) ^ hv;  // hash.c:129
    b.hv[sd.key_off + i] = (uint16_t)hv;
    b.hv2[sd.key_off + i] = (uint16_t)hv2;
    atomicAdd(&c1[hv], 1u);
    atomicAdd(&c2[hv2], 1u);
  }
}

// exclusive scan of 32768 counts per (segment, chain); entry 32768 receives the total
__global__ void k_bucket_scan(Batch b) {
  uint32_t seg = blockIdx.x >> 1;
  uint32_t* c = ((blockIdx.x & 1) ? b.bkt2 : b.bkt1) + (uint64_t)seg * 32769;
  __shared__ uint32_t part[1024];
  const int per = 32;  // 1024 threads x 32 bins
  uint32_t base = threadIdx.x * per, sum = 0;
  uint32_t v[per];
#pragma unroll
  for (int i = 0; i < per; i++) { v[i] = c[base + i]; sum += v[i]; }
  part[threadIdx.x] = sum;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    uint32_t t = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
    __syncthreads();
    part[threadIdx.x] += t;
    __syncthreads();
  }
  uint32_t run = part[threadIdx.x] - sum;
#pragma unroll
  for (int i = 0; i < per; i++) { c[base + i] = run; run += v[i]; }
  if (threadIdx.x == 1023) c[32768] = run;
}

// Stable scatter.  kScatterParts warps per (segment, chain): warp r owns the buckets whose top bits are r
// (a contiguous 1/kScatterParts of the 32768), walks ALL keys of the segment in position order and places
// the ones that fall into its range -- every bucket is filled by exactly one warp in position order, so
// the sort stays stable, and the serial walk that was one warp's 8 ms per master block is shared by
// kScatterParts warps.  The running bucket cursors of a warp's range live in shared memory.
// idx[dest] = position, rank[position] = dest.
constexpr uint32_t kPackedIdxLimit = 1u << 24;  // chain-1 entries of smaller segments: position | s8 << 24
constexpr int kScatterParts = 8;
constexpr int kScatterBuckets = 32768 / kScatterParts;
__global__ void __launch_bounds__(32) k_scatter(Batch b) {
  __shared__ uint32_t cursor[kScatterBuckets];
  const uint32_t part = blockIdx.x % kScatterParts;
  const uint32_t sc = blockIdx.x / kScatterParts;
  uint32_t seg = sc >> 1;
  bool second = sc & 1;
  const SegDesc sd = b.segs[seg];
  const uint32_t* bs = (second ? b.bkt2 : b.bkt1) + (uint64_t)seg * 32769 + part * kScatterBuckets;
  const uint16_t* key = (second ? b.hv2 : b.hv) + sd.key_off;
  uint32_t* idx = (second ? b.idx2 : b.idx1) + sd.key_off;
  uint32_t* rank = (second ? b.rank2 : b.rank1) + sd.key_off;
  const uint32_t lane = threadIdx.x;
  const uint16_t* other = b.hv2 + sd.key_off;
  const bool pack = !second && sd.nkeys < kPackedIdxLimit;
  for (uint32_t i = lane; i < (uint32_t)kScatterBuckets; i += 32) cursor[i] = bs[i];
  __syncwarp();
  // keys of 8 rounds are fetched up front so that the global-load latency is paid once per 256
  // positions instead of once per round
  for (uint32_t base0 = 0; base0 < sd.nkeys; base0 += 256) {
    uint32_t kreg[8], sreg[8];
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const uint32_t i = base0 + u * 32 + lane;
      kreg[u] = i < sd.nkeys ? key[i] : 0xffffffffu;
      sreg[u] = (pack && i < sd.nkeys) ? (uint32_t)other[i] : 0u;
    }
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const uint32_t i = base0 + u * 32 + lane;
      const uint32_t kk = kreg[u];
      const bool act = kk != 0xffffffffu && (kk / (uint32_t)kScatterBuckets) == part;
      if (!__any_sync(0xffffffffu, act)) continue;
      const uint32_t k = act ? kk - part * kScatterBuckets : 0x80000000u + lane;  // inactive lanes get a key no other lane has
      const uint32_t peers = __match_any_sync(0xffffffffu, k);
      const uint32_t before = __popc(peers & ((1u << lane) - 1));
      const uint32_t cur = act ? cursor[k] : 0;
      __syncwarp();
      if (act && before == 0) cursor[k] = cur + __popc(peers);
      __syncwarp();
      if (act) {
        const uint32_t d = cur + before;
        // chain 1 entries carry (hashval2 ^ hashval) & 255 = (same - 3) & 255 of their position in the top byte:
        // inside one hashval bucket that byte decides hashval2 equality (hash.c:129), so k_match's
        // chain-switch test (lz77.c:509-519) needs no second random read
        idx[d] = pack ? (i | (((sreg[u] ^ kk) & 255u) << 24)) : i;
        rank[i] = d;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// k_match: ZopfliFindLongestMatch for every parse position, cache-free (lz77.c:407-542).

// One CTA takes kMatchPosPerCta consecutive positions.  Everything a position's walk compares -- its own
// bytes and every candidate within the 32 KiB window (lz77.c:464) -- lies in one contiguous stretch of
// the input: [first position - 32767, last position + 258].  That stretch (~34 KB) is staged into shared
// memory with ONE TMA bulk copy (cp.async.bulk + mbarrier) per CTA, so the byte compares of the walk
// (the src[best] == cand[best] pre-check that most candidates fail, and the common-prefix loop) hit shared
// memory instead of a random 32-byte sector of L2 each.  The chain lists themselves (bucket slices of idx)
// are read coalesced from global memory, 32 candidates per round; the chain-switch test reads the
// candidate's (same-3)&255 from the top byte of its bucket entry (k_scatter) instead of hashval2[candidate].
constexpr int kMatchWarps = 8;
constexpr int kMatchPosPerCta = 512;
constexpr int kMatchWinBytes = 32768 + kMatchPosPerCta + kMaxMatch + 78;  // window + tile + longest match + alignment slack (multiple of 16)
static_assert(kMatchWinBytes % 16 == 0, "TMA bulk copies move multiples of 16 bytes");
constexpr int kMatchSmemBytes = kMatchWinBytes + kMatchWarps * 256 * 4;
struct PosWork { uint32_t seg, first; };

__device__ __forceinline__ uint32_t lds32_unaligned(const uint8_t* p) {  // p points into shared memory
  const uint32_t a = smem_u32(p);
  uint32_t lo, hi;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(lo) : "r"(a & ~3u));
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(hi) : "r"((a & ~3u) + 4u));
  return __funnelshift_r(lo, hi, (a & 3u) * 8u);
}
__device__ __forceinline__ uint32_t match_len_smem(const uint8_t* a, const uint8_t* b, uint32_t limit) {
  uint32_t m = 0;
  while (m < limit) {
    const uint32_t x = lds32_unaligned(a + m) ^ lds32_unaligned(b + m);
    if (x) { m += (uint32_t)(__ffs((int)x) - 1) >> 3; break; }
    m += 4;
  }
  return m < limit ? m : limit;
}

__global__ void __launch_bounds__(kMatchWarps * 32) k_match(Batch b, const PosWork* __restrict__ work) {
  extern __shared__ __align__(16) uint8_t win[];           // kMatchWinBytes, then the run-list staging
  uint32_t (*stage)[256] = (uint32_t (*)[256])(win + kMatchWinBytes);
  __shared__ __align__(8) uint64_t win_bar;
  const PosWork w = work[blockIdx.x];
  const SegDesc sd = b.segs[w.seg];
  const uint32_t lane = lane_id(), warp = threadIdx.x >> 5;
  const uint16_t* hv = b.hv + sd.key_off;
  const uint16_t* hv2 = b.hv2 + sd.key_off;
  const uint32_t* bs1 = b.bkt1 + (uint64_t)w.seg * 32769;
  const uint32_t* bs2 = b.bkt2 + (uint64_t)w.seg * 32769;
  const uint32_t woff = (uint32_t)(sd.instart - sd.winstart);  // key index of parse position 0
  const bool packed = sd.nkeys < kPackedIdxLimit;
  uint32_t* myruns = stage[warp];

  // ---- stage the window: key indices [wlo, whi) of the segment, wlo 16-byte aligned in the input ----
  const uint32_t ip0 = woff + w.first;                        // key index of the tile's first position
  const uint64_t g0 = sd.winstart + (ip0 > 32767u ? ip0 - 32767u : 0u);  // absolute input byte of the oldest candidate
  const uint64_t gal = g0 & ~(uint64_t)15;                    // the input buffer itself is 16-byte aligned
  const int64_t wlo = (int64_t)gal - (int64_t)sd.winstart;    // key index of window byte 0 (>= -15: winstart need not be aligned)
  uint64_t gend = sd.winstart + (uint64_t)ip0 + kMatchPosPerCta + kMaxMatch + 8;
  const uint64_t gmax = (b.insize + 16) & ~(uint64_t)15;      // the engine keeps >= 16 readable bytes behind the input
  if (gend > gmax) gend = gmax;
  const uint32_t nbytes = (uint32_t)(((gend - gal) + 15) & ~(uint64_t)15) <= (uint32_t)kMatchWinBytes
                              ? (uint32_t)(((gend - gal) + 15) & ~(uint64_t)15) : (uint32_t)kMatchWinBytes;
  if (threadIdx.x == 0) {
    mbar_init(&win_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_expect_tx(&win_bar, nbytes);
    bulk_g2s(win, b.in + gal, nbytes, &win_bar);
  }
  __syncthreads();
  mbar_wait(&win_bar, 0);
  const uint8_t* wsm = win - wlo;                             // wsm[key index] = input byte of that key position

  for (uint32_t t = warp; t < (uint32_t)kMatchPosPerCta; t += kMatchWarps) {
    const uint32_t j = w.first + t;  // parse position within the segment
    if (j >= sd.npos) break;
    const uint32_t ip = woff + j;    // key index of pos
    const uint32_t remain = sd.npos - j;  // inend - pos
    uint32_t best = 1, bestdist = 0, nruns = 0;
    if (remain >= (uint32_t)kMinMatch) {  // lz77.c:440-446
      const uint32_t limit = remain < (uint32_t)kMaxMatch ? remain : (uint32_t)kMaxMatch;  // :448-450
      uint32_t same0 = b.same_g[sd.winstart + ip];
      { uint64_t clip = sd.inend - 1 - (sd.winstart + ip); if (same0 > clip) same0 = (uint32_t)clip; }
      const uint32_t v2 = hv2[ip];
      const uint32_t s8p = (v2 ^ hv[ip]) & 255u;
      int hops = kMaxChainHits;
      bool chain2 = false;
      const uint32_t* idx = b.idx1 + sd.key_off;
      uint32_t lo = bs1[hv[ip]];
      uint32_t cur = b.rank1[sd.key_off + ip];  // next candidate is idx[cur-1]
      const uint8_t* src = wsm + ip;
      for (;;) {
        uint32_t avail = cur - lo;
        uint32_t take = avail < 32u ? avail : 32u;
        if ((uint32_t)hops < take) take = (uint32_t)hops;
        if (take == 0) break;  // bucket exhausted == self link lz77.c:523
        uint32_t iq = 0, dist = 0, m = 0;
        bool valid = lane < take;
        bool h2eq = false;
        if (valid) {
          const uint32_t e = idx[cur - 1 - lane];
          iq = (!chain2 && packed) ? (e & 0xffffffu) : e;
          dist = ip - iq;
          valid = dist < (uint32_t)kWindow;  // lz77.c:464
          if (valid) {
            const uint8_t* cand = wsm + iq;
            // lz77.c:478-479: a candidate that differs at offset `best` cannot beat it
            if (src[best] == cand[best]) m = match_len_smem(src, cand, limit);
            if (!chain2) h2eq = packed ? ((e >> 24) == s8p) : (hv2[iq] == v2);
          }
        }
        const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
        const uint32_t nv = __popc(vmask);  // valid lanes form a prefix (distances increase)
        if (nv == 0) break;
        // inclusive prefix max of m, seeded with best
        uint32_t pm = m;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          uint32_t o = __shfl_up_sync(0xffffffffu, pm, d);
          if (lane >= (uint32_t)d && o > pm) pm = o;
        }
        uint32_t pm_prev = __shfl_up_sync(0xffffffffu, pm, 1);
        const uint32_t pm_excl = (lane == 0) ? best : (pm_prev > best ? pm_prev : best);
        const uint32_t pm_incl = pm > best ? pm : best;
        const bool improved = valid && m > pm_excl;
        const uint32_t exitmask = __ballot_sync(0xffffffffu, valid && m >= limit);
        const uint32_t swmask = __ballot_sync(0xffffffffu, valid && h2eq && pm_incl >= same0);
        uint32_t c = nv - 1;
        bool do_exit = false, do_switch = false;
        uint32_t e = exitmask ? (uint32_t)(__ffs((int)exitmask) - 1) : 32u;
        uint32_t s = swmask ? (uint32_t)(__ffs((int)swmask) - 1) : 32u;
        if (e <= c && e <= s) { c = e; do_exit = true; }       // break before the switch test
        else if (s <= c) { c = s; do_switch = true; }
        const uint32_t keep = (c == 31) ? 0xffffffffu : ((1u << (c + 1)) - 1);
        const uint32_t impmask = __ballot_sync(0xffffffffu, improved) & keep;
        // a candidate that only reaches length 2 moves `best` but owns no usable length
        const bool rec = improved && m >= (uint32_t)kMinMatch;
        const uint32_t recmask = __ballot_sync(0xffffffffu, rec) & keep;
        if (rec && lane <= c) {
          uint32_t slot = nruns + __popc(recmask & ((1u << lane) - 1));
          myruns[slot] = run_pack(m, dist);  // lengths (pm_excl, m] first reached at `dist`
        }
        nruns += __popc(recmask);
        if (impmask) {
          int last = 31 - __clz((int)impmask);
          bestdist = __shfl_sync(0xffffffffu, dist, last);
        }
        best = __shfl_sync(0xffffffffu, pm_incl, c);
        hops -= (int)(c + 1);
        if (do_exit) break;
        if (do_switch) {  // lz77.c:509-519: continue from this candidate along chain 2
          uint32_t iqs = __shfl_sync(0xffffffffu, iq, s);
          chain2 = true;
          idx = b.idx2 + sd.key_off;
          lo = bs2[v2];
          cur = b.rank2[sd.key_off + iqs];
        } else {
          if (nv < 32u) break;  // window limit / bucket end / hop cap inside this round
          cur -= 32u;
        }
        if (hops <= 0) break;  // lz77.c:527-530
      }
    } else {
      best = 0;
    }
    __syncwarp();
    // outputs
    const uint64_t o = sd.pos_off + j;
    if (lane == 0) b.ld[o] = (best << 16) | bestdist;
    if (sd.mode != 0) {
      if (best < (uint32_t)kMinMatch) nruns = 0;
      if (lane == 0) {
        uint16_t ml = (uint16_t)(best >= (uint32_t)kMinMatch ? best : 0);
        // squeeze.c:251-257: same[i] > 516 && i > instart+259 && i+517 < inend && same[i-258] > 258
        if (j > (uint32_t)kMaxMatch + 1 && j + kMaxMatch * 2 + 1 < sd.npos) {
          const uint64_t p = sd.instart + j;
          uint64_t s0 = b.same_g[p], c0 = sd.inend - 1 - p;
          uint64_t s1 = b.same_g[p - kMaxMatch], c1 = sd.inend - 1 - (p - kMaxMatch);
          if ((s0 > c0 ? c0 : s0) > (uint64_t)kMaxMatch * 2 && (s1 > c1 ? c1 : s1) > (uint64_t)kMaxMatch) ml |= kShortcutFlag;
        }
        b.mlen[o] = ml;
      }
      {  // first-round distance symbols: lane l serves length 3+l
        const uint32_t k = 3 + lane;
        uint32_t v = kNoEdge;
        if (nruns && k <= best) {  // best <= inend - pos, so edges never leave the block
          for (uint32_t r = 0; r < nruns; r++) { uint32_t e = myruns[r]; if (run_len(e) >= k) { v = run_dsym(e); break; } }
        }
        b.dsx[o * 32 + ((lane + j + 3u) & 31u)] = (uint8_t)v;  // rotated: k_iterate's lane t reads byte t of row j
      }
      uint32_t* dst = b.runs + o * kRunSlots;
      if (nruns <= (uint32_t)kRunSlots) {
        if (lane < (uint32_t)kRunSlots) dst[lane] = lane < nruns ? myruns[lane] : 0u;
      } else {
        uint32_t off = 0;
        uint32_t extra = nruns - (kRunSlots - 1);
        // an offset past the end of the arena is clamped to it: these entries do not fit, and ovf_used > ovf_cap
        // makes the host grow the arena and redo the batch
        if (lane == 0) off = (uint32_t)min(atomicAdd(b.ovf_used, (unsigned long long)(extra + 1)), (unsigned long long)b.ovf_cap);
        off = __shfl_sync(0xffffffffu, off, 0);
        if (off + extra + 1 <= b.ovf_cap) {
          if (lane == 0) b.ovf[off] = extra;
          for (uint32_t r = lane; r < extra; r += 32) b.ovf[off + 1 + r] = myruns[kRunSlots - 1 + r];
          if (lane < (uint32_t)kRunSlots - 1) dst[lane] = myruns[lane];
          if (lane == (uint32_t)kRunSlots - 1) dst[lane] = kOverflowBit | off;
        } else {
          // arena exhausted: flagged through ovf_used > ovf_cap, host re-runs with a larger arena
          if (lane < (uint32_t)kRunSlots) dst[lane] = 0;
        }
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// k_greedy: ZopfliLZ77Greedy (lz77.c:544-630) over the (len,dist) table; one CTA of four warps per segment.
//
// The reference's lazy-matching loop is a state machine with two kinds of state per position:
// B(i) "at i, nothing pending" and H(j) "at j, the match found at j-1 is pending".  Everything
// that happens between one B state and the next is a pure function of the table entries just
// ahead (the H chain needs the score to grow by at least 2 per step, so it is at most 128 long).
// Per window of positions the warp therefore
//   1. evaluates that function for EVERY position as if it were a B state (32 wide): how far the
//      next B state is and how many symbols are emitted on the way;
//   2. lets lane 0 hop from B state to B state through that table (one shared-memory load per hop);
//   3. re-walks the visited B states 32 wide to emit their symbols at the offsets found in 2.
// Only step 2 is serial, and it costs one load per hop instead of the whole lazy-matching logic.

constexpr int kGreedyWin = 2048;    // B states evaluated per window
constexpr int kGreedyLook = 192;    // table entries loaded past the window (H chain <= 128 steps)

// walks from B(r) to the next B state.  T = (len << 16 | dist) entries, relative indexing.
// Emit(sym_index, litlen, dist) is called for each symbol in order.  Returns the next B position.
template <typename Emit>
__device__ __forceinline__ uint32_t greedy_walk(const uint32_t* T, const uint8_t* by, uint32_t r, uint32_t& cnt,
                                                Emit emit) {
  auto score = [](uint32_t e) { return (int)(e >> 16) - ((e & 0xffffu) > 1024u ? 1 : 0); };  // lz77.c:265-271
  auto holdable = [&](uint32_t e) { return score(e) >= kMinMatch && (e >> 16) < (uint32_t)kMaxMatch; };
  cnt = 0;
  uint32_t e = T[r];
  if (!holdable(e)) {  // lz77.c:619-629
    if (score(e) >= kMinMatch) { emit(cnt++, e >> 16, e & 0xffffu); return r + (e >> 16); }
    emit(cnt++, (uint32_t)by[r], 0u);
    return r + 1;
  }
  uint32_t j = r + 1;
  for (;;) {  // H(j): the match at j-1 is pending (lz77.c:584-609)
    const uint32_t ej = T[j];
    if (score(ej) > score(e) + 1) {
      emit(cnt++, (uint32_t)by[j - 1], 0u);         // the pending match loses: its position becomes a literal
      if (holdable(ej)) { e = ej; j++; continue; }
      emit(cnt++, ej >> 16, ej & 0xffffu);          // cannot be held (length 258): emitted at once
      return j + (ej >> 16);
    }
    emit(cnt++, e >> 16, e & 0xffffu);              // the pending match wins
    return j - 1 + (e >> 16);
  }
}

constexpr int kGreedyThreads = 128;

__global__ void __launch_bounds__(kGreedyThreads) k_greedy(Batch b, int buf) {
  __shared__ uint32_t wld[kGreedyWin + kGreedyLook];
  __shared__ uint8_t wby[kGreedyWin + kGreedyLook];
  __shared__ uint32_t wf[kGreedyWin];      // distance to the next B state (16) | symbols emitted (16)
  __shared__ uint32_t bl[kGreedyWin];      // visited B states: relative position (16) | output offset (16)
  __shared__ uint16_t oll[kGreedyWin + 512], od[kGreedyWin + 512];
  __shared__ uint32_t hop_r, hop_k, hop_off;
  const uint32_t seg = blockIdx.x, tid = threadIdx.x;
  const SegDesc sd = b.segs[seg];
  if (sd.mode == 2) {  // fixed-tree parse needs no greedy seed
    if (tid == 0) b.jobs[seg].greedy_size = 0;
    return;
  }
  const uint32_t* ld = b.ld + sd.pos_off;
  const uint8_t* in = b.in + sd.instart;
  uint16_t* out_ll = b.st_ll[buf] + sd.pos_off;
  uint16_t* out_d = b.st_d[buf] + sd.pos_off;
  const uint32_t n = sd.npos;
  uint32_t i = 0, nout = 0;
  while (i < n) {
    const uint32_t wb = i;
    const uint32_t wn = (n - wb) < (uint32_t)(kGreedyWin + kGreedyLook) ? (n - wb) : (uint32_t)(kGreedyWin + kGreedyLook);
    const uint32_t nchain = wn < (uint32_t)kGreedyWin ? wn : (uint32_t)kGreedyWin;
    for (uint32_t tb = 0; tb < wn; tb += kGreedyThreads * 4) {  // several loads in flight per thread: the refill is pure latency
      uint32_t v[4], c[4];
#pragma unroll
      for (int u = 0; u < 4; u++) { const uint32_t t = tb + u * kGreedyThreads + tid; v[u] = t < wn ? ld[wb + t] : 0u; c[u] = t < wn ? (uint32_t)in[wb + t] : 0u; }
#pragma unroll
      for (int u = 0; u < 4; u++) { const uint32_t t = tb + u * kGreedyThreads + tid; if (t < wn) { wld[t] = v[u]; wby[t] = (uint8_t)c[u]; } }
    }
    __syncthreads();
    for (uint32_t r = tid; r < nchain; r += kGreedyThreads) {  // 1: every position as a B state
      uint32_t cnt;
      const uint32_t nx = greedy_walk(wld, wby, r, cnt, [](uint32_t, uint32_t, uint32_t) {});
      wf[r] = (nx - r) | (cnt << 16);
    }
    __syncthreads();
    if (tid == 0) {  // 2: hop through the B states that are actually reached
      uint32_t r = 0, k = 0, off = 0;
      while (r < nchain) {
        const uint32_t e = wf[r];
        bl[k++] = r | (off << 16);
        off += e >> 16;
        r += e & 0xffffu;
      }
      hop_r = r;
      hop_k = k;
      hop_off = off;
    }
    __syncthreads();
    const uint32_t r = hop_r, k = hop_k, off = hop_off;
    for (uint32_t q = tid; q < k; q += kGreedyThreads) {  // 3: emit
      const uint32_t e = bl[q], o = e >> 16;
      uint32_t cnt;
      greedy_walk(wld, wby, e & 0xffffu, cnt, [&](uint32_t t, uint32_t l, uint32_t d) {
        oll[o + t] = (uint16_t)l;
        od[o + t] = (uint16_t)d;
      });
    }
    __syncthreads();
    for (uint32_t t = tid; t < off; t += kGreedyThreads) { out_ll[nout + t] = oll[t]; out_d[nout + t] = od[t]; }
    nout += off;
    i = wb + r;
    __syncthreads();
  }
  if (tid == 0) b.jobs[seg].greedy_size = nout;
}

}  // namespace zb

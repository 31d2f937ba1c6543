// k_iterate: the whole ZopfliLZ77Optimal loop for one deflate block in one persistent CTA of two
// warps -- warp 0 runs the algorithm, warp 1 feeds the forward DP
// (/root/reference/src/zopfli/squeeze.c:446-526; fixed-tree variant :528-560).  The wide form (eight
// warps, for launches that take whole SMs) runs trace-back and follow-path on all of them.
//
//   per iteration:  cost model constants (GetCostModelMinCost squeeze.c:163-198)
//                   forward DP          (GetBestLengths squeeze.c:217-309)   push form, pending costs
//                                        of the next 32 targets in a register window, longer edges
//                                        in a 512-entry shared-memory ring; the reference's fp64 add /
//                                        fp32 store arithmetic, carried out in integers while a group's
//                                        costs stay inside one float binade ("integer window" below)
//                   trace-back          (TraceBackwards squeeze.c:317-336)   speculative multi-start
//                                        chase in shared-memory windows
//                   follow + histogram  (FollowPath squeeze.c:338-389)       table lookups, 32 wide
//                   exact block size    (ZopfliCalculateBlockSize deflate.c:584-608)
//                   statistics          (squeeze.c:496-518, tree.c:71-94, RNG squeeze.c:80-107)
//
// fp discipline: every cost is (double)(lbits+dbits) + ll + d, then + (double)costs[j], compared
// in double against (double)float, stored rounded to float -- the reference's exact sequence.
// The file is compiled with -fmad=false; there is no multiply on the path anyway.
// log() is not evaluated on the device: entropies come from a table L[n] = log(n)*1.4426950408889
// filled by the host's libm, so they are bit-identical to what the reference computes on this box.
#pragma once
#include "kernels.cuh"

namespace zb {

struct XchEnt { double c; uint32_t code; uint32_t pad; };   // hand-off slot of the fp64 window: cost (float-representable) + length code
struct RingEnt { uint32_t fb; uint32_t code; };             // pending cost of a far target as FLOAT BITS (what the reference's costs[] holds)
                                                             // + length code of the best edge; the same for the fp64 and the integer paths
constexpr uint32_t kInfBits = 0x7149f2cau;                  // (float)1e30, ZOPFLI_LARGE_FLOAT squeeze.c:243
// length codes (decoded by decode_len): the window records only WHICH step produced the best edge
constexpr uint32_t kCodeLit = 0x800u;    // literal
constexpr uint32_t kCodeLong = 0x400u;   // | length, for edges longer than 34 (shared-memory ring)
                                         // otherwise: (source step & 31) + 3 (length = target - source, 3..34)
__host__ __device__ __forceinline__ uint32_t decode_len(uint32_t code, uint32_t target) {
  if (code & kCodeLit) return 1u;
  if (code & kCodeLong) return code & 0x3ffu;
  return ((target - code) & 31u) + 3u;
}
// ---- integer window (round 2, v10) ----
// While every cost a group of 32 positions can touch stays inside one float binade [2^e, 2^(e+1)) -- the
// same condition the magic-constant rounding needs -- the reference's arithmetic collapses to integers:
//   fl64(x + c) = x + c' with c' = c on the binade's double grid, (float) of that = x + k1 ulp with
//   k1 = round(c' / ulp) independent of x (x is a multiple of ulp) unless c'/ulp is an exact tie, and
//   the strict compare newCost < costs[t] (squeeze.c:278,296) is  x + k1 < costs[t], or equal and the
//   float rounding went up.
// A cost becomes (float bits - bits(2^e)); an edge is "+ k1"; and the sequential rule "first strict
// improvement wins" becomes ONE unsigned minimum over packed words (value << 7 | tiebreak) with
// tiebreak = up ? 63 - o : 64 + o, o = order of the edge's source among the sources of its target
// (0: length >= 35 via the ring, 1..32: lengths 34..3, 33: the literal).  A DP step is then two
// VIADDMNMX and one LOP3 on the chain instead of six DADDs, two DSETPs and eight selects.  Tables
// (k1, up) are rebuilt per binade; a binade whose table holds an exact tie (or that is too narrow
// for the safety margins) runs on the fp64 paths.  oracle/dp_int_model.c is the sequential model of
// this formulation, checked against the reference DP on every pass (tests/test_oracle.py).
constexpr uint32_t kIntInf = 0xffffffffu;   // no edge yet
constexpr uint32_t kIntNoEdge = 1u << 30;   // table entry "no such length here"; any word >= this is infinite
constexpr uint32_t kCodeInt = 0x1000u;      // length code taken from an integer word: | tiebreak bits
struct IterDyn {                       // dynamic shared memory of k_iterate (engine.cu pads the launch to at least this)
  uint32_t ti[31 * 64];                // integer edge table of the current binade, indexed like IterSmem::t0
  uint32_t liti[2][256];               // integer literal edges, double-buffered by generation parity (DP warp -> feeder)
  uint32_t gli[4 * 32 + 4];            // literal edge of each staged position; [128..129] mirror [0..1]   (feeder warp)
  uint32_t tag[4];                     // generation of liti a stage was filled from                        (feeder warp)
  uint32_t tl[29 * 32];                // long edges (length >= 35): (k1 << 1 | up) per (length symbol - 257, distance symbol)
  uint32_t xchi[4];                    // hand-off slots of the integer window
  uint32_t gen;                        // published generation of liti
};
struct DpStage {                       // forward-DP working set; 4 stages of 32 positions each
  RingEnt ring[512];                   // pending costs of targets >= j+35 (long edges only); slot (t-3) & 511
  uint32_t runs[4][32 * kRunSlots];    // TMA-staged run lists
  uint8_t dsx[4 * 32 * 32 + 128];      // TMA-staged first-round distance symbols, rows pre-rotated by k_match;
                                       // the last 128 bytes mirror rows 0-3 of stage 0 (reads run 3 rows ahead)
  double gl[4 * 32 + 2];               // literal cost of the byte at each position; [128..129] mirror [0..1] (feeder warp)
  uint16_t mk[4][32];                  // mlen16 of each position                             (feeder warp)
  uint16_t lac[4][32];                 // length codes of length_array[32g + l]              (DP warp -> feeder)
  uint32_t flag[4];                    // ballot: position needs the general path            (feeder warp)
  uint32_t flagS[4];                   // ballot: long-run shortcut candidate (fp64 general path only)   (feeder warp)
  XchEnt xch[4];                       // pending(j+3) handed from its owner lane to all lanes: written at step j,
                                       // loaded at step j+1, used at step j+2.  Shared memory rather than shuffles
                                       // because the order of memory operations is the one thing the assembler keeps:
                                       // a shuffle is sunk to just before its use and its latency lands on the chain.
};
// length code -> length_array entry; integer words that won through a long edge find its length in the ring slot
__device__ __forceinline__ uint32_t decode_code(uint32_t code, uint32_t target, const RingEnt* ring) {
  if (code & kCodeInt) {
    const uint32_t tb = code & 127u, o = tb < 64u ? 63u - tb : tb - 64u;
    if (o == 33u) return 1u;
    if (o == 0u) return ring[(target - 3u) & 511u].code & 0x3ffu;
    return 35u - o;
  }
  return decode_len(code, target);
}
struct WarpPm {                        // warp-wide package-merge working set (warp_length_limited)
  uint32_t key[kNumLL];                // active symbols sorted by (weight << 9 | symbol)
  uint32_t pk[kNumLL];                 // package weights of the level being built
  uint32_t row[2][2 * kNumLL];         // item weights of the previous / current level
  uint32_t mask[15][(2 * kNumLL + 31) / 32];  // bit = item is a leaf
};
struct CostStage {                     // block-size working set
  uint32_t cnt2[320];                  // RLE-smoothed copies (ll: [0,288), d: [288,320))
  uint8_t len[2][320];                 // code lengths: set 0 plain, set 1 smoothed
  WarpPm pm;
};
struct IterSmem {
  double llcost[kNumLL];   // ll_symbols
  double dcost[kNumD];     // d_symbols
  double lencost[260];     // llcost[length_symbol(k)]
  double t0[31 * 64];      // first-round edge costs, each row twice: t0[dsym*64 + c] = cost(3 + ((c - 1) & 31), dist
                           // of dsym) so that a lane's column (cm + 33 - step) needs no wrap; row 30 = +inf
  union __align__(16) {
    DpStage dp;
    CostStage cs;
    struct { uint16_t la[4096]; uint16_t mark[4096]; } tr;  // trace-back window: length_array slice + visit marks
  } u;
  __align__(8) uint64_t full[4];   // stage filled (TMA bytes + feeder scalars)
  __align__(8) uint64_t empty[4];  // stage consumed by the DP warp
  uint32_t go;                     // DP warp -> feeder warp: another iteration follows
  unsigned long long dpc[5];       // DP cycles / groups by kind (see JobState)
  uint32_t dpn[6];
  uint32_t hist[320];
  uint32_t stats[320], last[320], bests[320];
};

// ---- mbarrier / bulk-copy (TMA 1-D) primitives: smem_u32, mbar_init, mbar_expect_tx, bulk_g2s, mbar_wait live in kernels.cuh ----
__device__ __forceinline__ double lds_f64(uint32_t a) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
// predicated 16-byte store of a ring entry {cost, len}
__device__ __forceinline__ void sts_ring_if(uint32_t a, double c, uint32_t len, bool p) {
  asm volatile("{ .reg .pred q; setp.ne.u32 q, %3, 0; @q st.shared.v2.b64 [%0], {%1, %2}; }" ::"r"(a),
               "l"(__double_as_longlong(c)), "l"((long long)len), "r"((uint32_t)p)
               : "memory");
}
// (double)(float)x for 0 <= x < 3e38 outside the float-denormal range: round-to-nearest-even on
// the 29 low mantissa bits, in integer arithmetic (keeps the conversion pipe off the cost chain)
__device__ __forceinline__ double round_to_f32(double x) {
  long long b = __double_as_longlong(x);
  b += 0x0FFFFFFFLL + ((b >> 29) & 1);
  b &= ~0x1FFFFFFFLL;
  return __longlong_as_double(b);
}
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar_a) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar_a) : "memory");
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar_a, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done)
                 : "r"(bar_a), "r"(parity)
                 : "memory");
  } while (!done);
}
__device__ __forceinline__ void cta_sync64() { asm volatile("bar.sync 1, 64;" ::: "memory"); }
// every warp of the wide form (trace-back and follow-path); cta_sync64 counts only warp 0 and the feeder
template <int NW>
__device__ __forceinline__ void cta_sync_all() { asm volatile("bar.sync 2, %0;" ::"n"(NW * 32) : "memory"); }
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts_u16_if(uint32_t a, uint32_t v, bool p) {
  asm volatile("{ .reg .pred q; setp.ne.u32 q, %2, 0; @q st.shared.u16 [%0], %1; }" ::"r"(a), "h"((unsigned short)v), "r"((uint32_t)p) : "memory");
}
__device__ __forceinline__ void sts_u32_if(uint32_t a, uint32_t v, bool p) {
  asm volatile("{ .reg .pred q; setp.ne.u32 q, %2, 0; @q st.shared.u32 [%0], %1; }" ::"r"(a), "r"(v), "r"((uint32_t)p) : "memory");
}
// ring entry {cost, code}
__device__ __forceinline__ void lds_ring(uint32_t a, double& c, uint32_t& code) {
  unsigned long long x, y;
  asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(x), "=l"(y) : "r"(a) : "memory");
  c = __longlong_as_double((long long)x);
  code = (uint32_t)y;
}
// ring entry {float bits, code}
__device__ __forceinline__ void lds_ring8(uint32_t a, uint32_t& fb, uint32_t& code) {
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(fb), "=r"(code) : "r"(a) : "memory");
}
__device__ __forceinline__ void sts_ring8_if(uint32_t a, uint32_t fb, uint32_t code, bool p) {
  asm volatile("{ .reg .pred q; setp.ne.u32 q, %3, 0; @q st.shared.v2.u32 [%0], {%1, %2}; }" ::"r"(a), "r"(fb), "r"(code), "r"((uint32_t)p)
               : "memory");
}
__device__ __forceinline__ double warp_min_first(double v, int& idx) {
  // minimum with the smallest index among equals (sequential strict-< scan order)
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    double ov = __shfl_xor_sync(0xffffffffu, v, d);
    int oi = __shfl_xor_sync(0xffffffffu, idx, d);
    if (ov < v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  return v;
}

// ZopfliCalculateEntropy tree.c:71-94 over n counts (n = 288 or 32). Returns false if a count or
// the sum falls outside the host-provided log table.
__device__ bool warp_entropy(const uint32_t* cnt, int n, double* out, const Batch& b, uint32_t lane) {
  uint32_t sum = 0;
  for (int i = lane; i < n; i += 32) sum += cnt[i];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
  uint32_t si = sum == 0 ? (uint32_t)n : sum;
  bool ok = si < b.logtab_n;
  double log2sum = ok ? b.logtab[si] : 0.0;
  for (int i = lane; i < n; i += 32) {
    uint32_t c = cnt[i];
    double v = log2sum;
    if (c) {
      if (c < b.logtab_n) v = log2sum - b.logtab[c];
      else ok = false;
    }
    if (v < 0 && v > -1e-5) v = 0;  // tree.c:91
    out[i] = v;
  }
  return __all_sync(0xffffffffu, ok);
}

// ---- ZopfliLengthLimitedCodeLengths (katajainen.c:172-262) by the whole warp ----
// Same level-by-level package-merge as length_limited() in deflate_size.hpp (and the same tie rule:
// a package precedes a leaf of equal weight), but every level is built as a parallel MERGE BY RANK:
// leaf i lands at i + #{packages <= w_i}, package p at p + #{leaves < sum_p}; both counts are
// branch-free binary searches over sorted shared-memory arrays.  The serial version walks
// 15 x 574 items through one lane; this one needs ~15 x 9 search rounds per lane.
template <int ITEMS>
__device__ __forceinline__ void warp_bitonic_sort(uint32_t* keys, int ns, uint32_t lane) {
  const uint32_t full = 0xffffffffu;
  uint32_t v[ITEMS];
#pragma unroll
  for (int r = 0; r < ITEMS; r++) {
    const int e = (int)lane * ITEMS + r;
    v[r] = e < ns ? keys[e] : 0xffffffffu;
  }
  constexpr int N = 32 * ITEMS;
#pragma unroll
  for (int k = 2; k <= N; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j >= ITEMS) {
        const int lj = j / ITEMS;
        const bool lower = (lane & lj) == 0;
#pragma unroll
        for (int r = 0; r < ITEMS; r++) {
          const uint32_t o = __shfl_xor_sync(full, v[r], lj);
          const bool asc = ((((int)lane * ITEMS + r) & k) == 0);
          v[r] = (lower == asc) ? min(v[r], o) : max(v[r], o);
        }
      } else {
#pragma unroll
        for (int r = 0; r < ITEMS; r++) {
          if ((r & j) == 0) {
            const bool asc = ((((int)lane * ITEMS + r) & k) == 0);
            const uint32_t a = v[r], c = v[r | j];
            const uint32_t lo = min(a, c), hi = max(a, c);
            v[r] = asc ? lo : hi;
            v[r | j] = asc ? hi : lo;
          }
        }
      }
    }
  }
  __syncwarp();
#pragma unroll
  for (int r = 0; r < ITEMS; r++) {
    const int e = (int)lane * ITEMS + r;
    if (e < ns) keys[e] = v[r];
  }
  __syncwarp();
}

// freq: n counts in shared memory (n <= 288, counts < 2^22); out: n code lengths, maxbits 15
__device__ __noinline__ void warp_length_limited(const uint32_t* freq, int n, uint8_t* out, WarpPm& pm, uint32_t lane) {
  const uint32_t full = 0xffffffffu;
  int ns = 0;
  for (int base = 0; base < n; base += 32) {
    const int i = base + (int)lane;
    const uint32_t f = i < n ? freq[i] : 0u;
    if (i < n) out[i] = 0;
    const uint32_t bal = __ballot_sync(full, f != 0);
    if (f) pm.key[ns + __popc(bal & ((1u << lane) - 1u))] = (f << 9) | (uint32_t)i;
    ns += __popc(bal);
  }
  __syncwarp();
  if (ns == 0) return;                                                       // katajainen.c:208-211
  if (ns <= 2) { if ((int)lane < ns) out[pm.key[lane] & 511] = 1; __syncwarp(); return; }  // :212-222
  if (ns > 256) warp_bitonic_sort<16>(pm.key, ns, lane);                     // :224-235
  else if (ns > 128) warp_bitonic_sort<8>(pm.key, ns, lane);
  else if (ns > 32) warp_bitonic_sort<4>(pm.key, ns, lane);
  else warp_bitonic_sort<1>(pm.key, ns, lane);
  const int maxbits = ns - 1 < 15 ? ns - 1 : 15;                             // :238-240
  const int maxitems = 2 * ns - 2;
  for (int i = lane; i < ns; i += 32) pm.row[0][i] = pm.key[i] >> 9;
  __syncwarp();
  int prevlen = ns, cur = 1;
  for (int lev = 1; lev < maxbits; lev++, cur ^= 1) {
    const uint32_t* prev = pm.row[cur ^ 1];
    uint32_t* row = pm.row[cur];
    const int npk = prevlen >> 1;
    if (lane < (2 * kNumLL + 31) / 32) pm.mask[lev][lane] = 0;
    for (int p = lane; p < npk; p += 32) {
      const uint2 pr = *(const uint2*)&prev[2 * p];
      pm.pk[p] = pr.x + pr.y;
    }
    __syncwarp();
    const int tmax = ((ns > npk ? ns : npk) + 31) >> 5;
    for (int t = 0; t < tmax; t++) {
      const int i = (int)lane + 32 * t;
      const bool hl = i < ns, hp = i < npk;
      const uint32_t wl = hl ? pm.key[i] >> 9 : 0u, wp = hp ? pm.pk[i] : 0u;
      int ub = 0, lb = 0;
#pragma unroll
      for (int step = 256; step; step >>= 1) {
        const int a = ub + step, c = lb + step;
        const uint32_t va = pm.pk[(a < npk ? a : npk) - 1];
        const uint32_t vc = pm.key[(c < ns ? c : ns) - 1] >> 9;
        if (a <= npk && va <= wl) ub = a;   // packages that precede leaf i: sum <= w_i
        if (c <= ns && vc < wp) lb = c;     // leaves that precede package i: w < sum_i
      }
      if (hl) {
        const int pos = i + ub;
        if (pos < maxitems) { row[pos] = wl; atomicOr(&pm.mask[lev][pos >> 5], 1u << (pos & 31)); }
      }
      if (hp) {
        const int pos = i + lb;
        if (pos < maxitems) row[pos] = wp;
      }
    }
    __syncwarp();
    prevlen = ns + npk < maxitems ? ns + npk : maxitems;
  }
  // selection (ExtractBitLengths katajainen.c:145-163): rank r gets one bit per level whose
  // selected-leaf count exceeds r
  uint32_t cnt[9];
#pragma unroll
  for (int t = 0; t < 9; t++) cnt[t] = 0;
  int need = maxitems;
  for (int lev = maxbits - 1; lev >= 0; lev--) {
    int c;
    if (lev == 0) {
      c = need < ns ? need : ns;
    } else {
      const uint32_t word = lane < (2 * kNumLL + 31) / 32 ? pm.mask[lev][lane] : 0u;
      int bits = need - 32 * (int)lane;
      bits = bits < 0 ? 0 : (bits > 32 ? 32 : bits);
      const uint32_t m = bits >= 32 ? 0xffffffffu : ((1u << bits) - 1u);
      c = __popc(word & m);
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(full, c, d);
    }
#pragma unroll
    for (int t = 0; t < 9; t++) cnt[t] += (c > (int)lane + 32 * t) ? 1u : 0u;
    need = 2 * (need - c);
  }
#pragma unroll
  for (int t = 0; t < 9; t++) {
    const int i = (int)lane + 32 * t;
    if (i < ns) out[pm.key[i] & 511] = (uint8_t)cnt[t];
  }
  __syncwarp();
}

// exact dynamic block size from s.hist (hist[256] already 1): deflate.c:569-608.  With `choice` the
// code-length set (cs.len[choice->set]) and the tree flags that realise the size are reported too
// (what AddDynamicTree / GetDynamicLengths would pick: first minimum of the 8 flag combinations).
struct DynChoice { uint32_t set, flags, tree_bits; };

// Tree-header bits of both code-length sets (cs.len[0], cs.len[1]) under all 8 flag combinations
// (EncodeTree size_only, deflate.c:105-249): lane l < 16 returns the size for set l >> 3, flags l & 7.
// The token counts are summed per maximal run of equal lengths (run_token_counts), with the runs of
// each set spread over the warp, instead of 16 lanes walking the sequence one length at a time down
// eight diverging paths.  The counts, and so the sizes, are those encode_tree_size computes.
__device__ __noinline__ uint32_t warp_tree_sizes(CostStage& cs, uint32_t lane) {
  uint32_t* cl = cs.cnt2;            // [set][flags][19] counts; the smoothed counts are spent by now
  uint32_t* starts = cs.pm.mask[0];  // run starts of one set, a bit per position
  for (int i = lane; i < 2 * 8 * 19; i += 32) cl[i] = 0;
  for (int set = 0; set < 2; set++) {
    const uint8_t* ll = cs.len[set];
    const uint8_t* dl = ll + 288;
    const TreeShape sh = tree_shape(ll, dl);
    const unsigned nll = sh.hlit + 257, nwords = (sh.total + 31) >> 5;
    auto at = [&](unsigned i) -> unsigned { return i < nll ? ll[i] : dl[i - nll]; };
    __syncwarp();
    for (unsigned w = 0; w < nwords; w++) {
      const unsigned i = w * 32 + lane;
      const bool st = i < sh.total && (i == 0 || at(i) != at(i - 1));
      const uint32_t m = __ballot_sync(0xffffffffu, st);
      if (lane == 0) starts[w] = m;
    }
    __syncwarp();
    for (unsigned i = lane; i < sh.total; i += 32) {
      const unsigned b = i & 31;
      unsigned w = i >> 5;
      if (!((starts[w] >> b) & 1u)) continue;
      unsigned end = sh.total;   // the run ends at the next run start
      uint32_t m = b == 31 ? 0u : starts[w] & ~((2u << b) - 1u);
      while (!m && ++w < nwords) m = starts[w];
      if (m) end = w * 32 + (unsigned)(__ffs(m) - 1);
      const unsigned v = at(i), c = end - i;
      for (unsigned f = 0; f < 8; f++) {
        uint32_t* dst = cl + (set * 8 + f) * 19;
        run_token_counts(v, c, f, [&](unsigned sym, unsigned n) { atomicAdd(&dst[sym], n); });
      }
    }
  }
  __syncwarp();
  // the code-length code's cost from a Huffman tree in registers; the lanes where that tree is deeper than
  // 7 bits take the package-merge, each on its own scratch in the package-merge working set (free by now).
  // tree_header_bits_huffman is the CPU model.
  static_assert(16 * sizeof(PmScratch<19, 7>) + 16 * 19 <= sizeof(WarpPm), "cl-code scratch");
  uint32_t r = 0xffffffffu, bits = 0;
  const bool fits = lane < 16 && clcode_bits_unlimited(cl + lane * 19, &bits);
  if (fits) r = tree_header_bits_from(cl + lane * 19, bits);
  if (lane < 16 && !fits) {
    PmScratch<19, 7>* pms = reinterpret_cast<PmScratch<19, 7>*>(cs.pm.key);
    uint8_t* clcl = reinterpret_cast<uint8_t*>(pms + 16) + lane * 19;
    length_limited<19, 7>(cl + lane * 19, 19, 7, clcl, pms[lane]);
    bits = 0;
    for (int i = 0; i < 19; i++) bits += clcl[i] * cl[lane * 19 + i];
    r = tree_header_bits_from(cl + lane * 19, bits);
  }
  __syncwarp();
  return r;
}

// first marked position after i in the bit words[0 .. nw) (a bit per position), or `none`
__device__ __forceinline__ int next_mark(const uint32_t* words, int nw, int i, int none) {
  const uint32_t b = i & 31;
  int w = i >> 5;
  uint32_t m = b == 31 ? 0u : words[w] & ~((2u << b) - 1u);
  while (!m && ++w < nw) m = words[w];
  return m ? w * 32 + (__ffs(m) - 1) : none;
}

// OptimizeHuffmanForRle (optimize_for_rle, deflate.c:434-518) by the whole warp, in place on n <= 288
// counts in shared memory; the package-merge working set is its scratch.  Pass 1: the last non-zero count
// by ballot.  Pass 2: run starts by ballot; each lane measures the runs that start on its positions and
// pins the long ones, a bit per position.  Pass 3 (rle_segment_end in deflate_size.hpp): from each segment
// start reached, the warp tests the next 32 positions against the start's limit with one ballot, so the
// serial part is one hop per segment; then the lanes the segment starts fall on flatten them.
// optimize_for_rle_by_segments is the CPU model of this order.
__device__ __noinline__ void warp_optimize_for_rle(uint32_t* counts, int n, WarpPm& pm, uint32_t lane) {
  const uint32_t full = 0xffffffffu;
  uint32_t* ends = pm.row[0];    // end of the segment that would start at each position (0: not measured)
  uint32_t* runs = pm.mask[0];   // run starts
  uint32_t* pin = pm.mask[1];    // pinned positions (good_for_rle)
  uint32_t* seg = pm.mask[2];    // segment starts
  int length = 0;
  for (int base = 0; base < n; base += 32) {
    const int i = base + (int)lane;
    const uint32_t m = __ballot_sync(full, i < n && counts[i] != 0);
    if (m) length = base + 32 - __clz(m);
  }
  if (length == 0) return;
  const int nw = (length + 31) >> 5;
  for (int w = 0; w < nw; w++) {
    const int i = w * 32 + (int)lane;
    const uint32_t m = __ballot_sync(full, i < length && (i == 0 || counts[i] != counts[i - 1]));
    if (lane == 0) runs[w] = m;
    if ((int)lane == w) pin[w] = 0;
  }
  __syncwarp();
  for (int i = lane; i < length; i += 32) {
    if (!((runs[i >> 5] >> (i & 31)) & 1u)) continue;
    const int end = next_mark(runs, nw, i, length);
    if (end - i < (counts[i] == 0 ? 5 : 7)) continue;
    for (int w = i >> 5; w <= (end - 1) >> 5; w++) {
      const int lo = (i > w * 32 ? i : w * 32) - w * 32, hi = (end < w * 32 + 32 ? end : w * 32 + 32) - w * 32;
      atomicOr(&pin[w], (hi - lo == 32 ? full : (1u << (hi - lo)) - 1u) << lo);
    }
  }
  __syncwarp();
  const bool good0 = pin[0] & 1u;
  auto stops = [&](int p, uint32_t lim) {   // position p ends the segment (rle_segment_end's loop test)
    return p >= length || ((pin[p >> 5] >> (p & 31)) & 1u) || !rle_extends(counts[p], lim);
  };
  // every position's segment end, as far as 32 counts ahead, by the lane that owns it
  for (int a = lane; a < length; a += 32) {
    const uint32_t lim = rle_segment_limit(counts, length, good0, a);
    int b = a + 1;
    while (b <= a + 32 && !stops(b, lim)) b++;
    ends[a] = b <= a + 32 ? (uint32_t)b : 0u;
  }
  __syncwarp();
  // hop through the reached starts: one shared-memory load per segment; a segment longer than 32 is
  // followed by the whole warp, 32 positions per ballot
  uint32_t segw = 0;   // lane w: the segment starts among positions [32w, 32w + 32)
  for (int a = 0; a < length;) {
    if ((int)lane == (a >> 5)) segw |= 1u << (a & 31);
    int b = (int)ends[a];
    if (b == 0) {
      const uint32_t lim = rle_segment_limit(counts, length, good0, a);
      for (int base = a + 33;; base += 32) {
        const uint32_t m = __ballot_sync(full, stops(base + (int)lane, lim));
        if (m) { b = base + __ffs(m) - 1; break; }
      }
    }
    a = b;
  }
  if ((int)lane < nw) seg[lane] = segw;
  __syncwarp();
  for (int a = lane; a < length; a += 32) {
    if (!((seg[a >> 5] >> (a & 31)) & 1u)) continue;
    const int end = next_mark(seg, nw, a, length);
    uint64_t sum = 0;
    for (int k = a; k < end; k++) sum += counts[k];
    uint32_t mean;
    if (rle_flatten(sum, end - a, &mean))
      for (int k = a; k < end; k++) counts[k] = mean;
  }
  __syncwarp();
}

__device__ uint64_t warp_dynamic_bits(const uint32_t* hist, CostStage& cs, uint32_t lane, DynChoice* choice = nullptr) {
  // RLE-smoothed copies of both histograms (TryOptimizeHuffmanForRle deflate.c:525-567), then four
  // warp-wide code constructions
  for (int i = lane; i < 320; i += 32) cs.cnt2[i] = hist[i];
  __syncwarp();
  warp_optimize_for_rle(cs.cnt2, kNumLL, cs.pm, lane);
  warp_optimize_for_rle(cs.cnt2 + 288, kNumD, cs.pm, lane);
  warp_length_limited(hist, kNumLL, cs.len[0], cs.pm, lane);
  warp_length_limited(hist + 288, kNumD, cs.len[0] + 288, cs.pm, lane);
  warp_length_limited(cs.cnt2, kNumLL, cs.len[1], cs.pm, lane);
  warp_length_limited(cs.cnt2 + 288, kNumD, cs.len[1] + 288, cs.pm, lane);
  if (lane < 2) patch_distance_codes(cs.len[lane] + 288);
  __syncwarp();
  uint32_t tsz = warp_tree_sizes(cs, lane);
  if (lane < 16) tsz = (tsz << 3) | (lane & 7u);  // ties go to the lowest flag index (deflate.c:259-267 keeps the first minimum)
  // min over lanes 0..7 and 8..15 (deflate.c:277-290)
#pragma unroll
  for (int d = 4; d > 0; d >>= 1) {
    uint32_t o = __shfl_xor_sync(0xffffffffu, tsz, d);
    tsz = o < tsz ? o : tsz;
  }
  const uint32_t key0 = __shfl_sync(0xffffffffu, tsz, 0), key1 = __shfl_sync(0xffffffffu, tsz, 8);
  const uint32_t tree0 = key0 >> 3, tree1 = key1 >> 3;
  // symbol bits of both length sets (deflate.c:379-401), all lanes
  uint64_t sb0 = 0, sb1 = 0;
  for (int i = lane; i < 320; i += 32) {
    uint32_t c = hist[i];
    int extra;
    bool use;
    if (i < 288) { use = i < 256 || (i >= 257 && i < 286); extra = i >= 257 ? length_symbol_extra_bits(i) : 0; }
    else { use = (i - 288) < 30; extra = dist_symbol_extra_bits(i - 288); }
    if (use) {
      sb0 += (uint64_t)(cs.len[0][i] + extra) * c;
      sb1 += (uint64_t)(cs.len[1][i] + extra) * c;
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    sb0 += __shfl_xor_sync(0xffffffffu, sb0, d);
    sb1 += __shfl_xor_sync(0xffffffffu, sb1, d);
  }
  const uint64_t size0 = tree0 + sb0 + cs.len[0][256];
  const uint64_t size1 = tree1 + sb1 + cs.len[1][256];
  if (choice) {
    const bool second = size1 < size0;  // deflate.c:553-559
    choice->set = second ? 1u : 0u;
    choice->flags = (second ? key1 : key0) & 7u;
    choice->tree_bits = second ? tree1 : tree0;
  }
  return 3 + (size1 < size0 ? size1 : size0);  // deflate.c:553-559
}

// FollowPath (squeeze.c:338-389) of the traced symbols psym[cursor + t], t in [t0, t1), by one warp: store
// entries t of cl / cd, histogram into `hist`.  128 symbols in flight per trip, fetched one trip ahead.
// The two-warp form runs it over [0, nsym), the wide form over one slice per warp.
__device__ __forceinline__ void follow_path(const Batch& b, const SegDesc& sd, const uint8_t* in, const uint64_t* psym,
                                            uint32_t cursor, uint32_t t0, uint32_t t1, uint16_t* cl, uint16_t* cd,
                                            uint32_t* hist, uint32_t lane) {
  uint64_t en[4];  // symbols of the next trip, fetched one trip ahead
#pragma unroll
  for (int u = 0; u < 4; u++) {
    const uint32_t t = t0 + u * 32 + lane;
    en[u] = t < t1 ? psym[cursor + t] : 1u;  // dummy literal at position 0 for the tail
  }
  for (uint32_t base = t0; base < t1; base += 128) {
    uint64_t e[4];
    uint4 ra[4], rc[4];
    uint32_t by[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      e[u] = en[u];
      const uint32_t t = base + 128 + u * 32 + lane;
      en[u] = t < t1 ? psym[cursor + t] : 1u;
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const uint32_t len = (uint32_t)e[u] & 511u, pj = (uint32_t)(e[u] >> 9);
      const uint4* r4 = (const uint4*)(b.runs + (sd.pos_off + pj) * kRunSlots);
      if (len >= (uint32_t)kMinMatch) { ra[u] = r4[0]; rc[u] = r4[1]; by[u] = 0; }
      else { ra[u] = make_uint4(0, 0, 0, 0); rc[u] = ra[u]; by[u] = in[pj]; }
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const uint32_t t = base + u * 32 + lane;
      if (t >= t1) continue;
      const uint32_t len = (uint32_t)e[u] & 511u;
      if (len >= (uint32_t)kMinMatch) {
        const uint32_t x = run_for_len(ra[u], rc[u], len, b.ovf);
        cl[t] = (uint16_t)len; cd[t] = (uint16_t)run_dist(x);
        atomicAdd(&hist[length_symbol((int)len)], 1u);
        atomicAdd(&hist[288 + run_dsym(x)], 1u);
      } else {
        cl[t] = (uint16_t)by[u]; cd[t] = 0;
        atomicAdd(&hist[by[u]], 1u);
      }
    }
  }
}

// ---- wide form of k_iterate (NW = 8 warps; launches whose CTAs take a whole SM) ----
// The DP runs on warp 0 and the feeder exactly as in the two-warp form while warps 2.. wait at
// cta_sync_all; trace-back and follow-path then run on every warp.  Their working set lies in the dynamic
// shared memory the launch pads anyway, after IterDyn.
constexpr int kWideWarps = 8;
constexpr uint32_t kTrSegLen = 128;   // positions per speculative chain of the trace-back
template <int NW>
struct WideSmem {
  static constexpr uint32_t kSeg = NW * 32, kWin = kSeg * kTrSegLen;   // one segment per thread
  uint16_t la[kWin];                  // trace-back window: length_array slice
  uint16_t mark[kWin];                // visit number of a node on its segment's speculative chain (0: not visited)
  uint32_t cnt[kSeg], exit[kSeg];     // length and exit node of each segment's speculative chain
  uint32_t in[kSeg], out[kSeg];       // the true path in each segment: entry node, exit node,
  uint32_t ns[kSeg], off[kSeg];       //   symbols, and symbols of the segments above it in the window
  uint32_t hist[NW][320];             // follow-path histogram of each warp
  uint32_t idx, cursor, nact, curbuf; // next window's top node, psym cursor, live segments; warp 0's curbuf
};
constexpr size_t kWideOff = (sizeof(IterDyn) + 15) & ~(size_t)15;   // offset of WideSmem in the dynamic shared memory
template <int NW>
constexpr size_t wide_dyn_bytes() { return kWideOff + sizeof(WideSmem<NW>); }

// one hop of the trace-back from node i: length_array[i] clamped to [1, i] so a corrupted chain cannot hang
__device__ __forceinline__ uint32_t tr_hop(uint32_t la_a, uint32_t wlo, uint32_t i) {
  uint32_t l;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(l) : "r"(la_a + (i - wlo) * 2));
  return min(max(l, 1u), i);
}
struct TrSeg { uint32_t hi, floor_; bool live; };   // segment sg of a window: positions (floor_, hi]
__device__ __forceinline__ TrSeg tr_seg(uint32_t idx, uint32_t wlo, uint32_t sg) {
  const uint32_t hi = idx >= sg * kTrSegLen ? idx - sg * kTrSegLen : 0u;
  const uint32_t lo = hi >= kTrSegLen ? hi - kTrSegLen : 0u;
  return {hi, lo > wlo ? lo : (wlo > 0 ? wlo - 1 : 0u), hi > 0 && hi >= wlo};   // stop below the window as well
}
// the path entering a segment at node i: hop until it meets the segment's speculative chain at its node
// number m (then it follows the chain's cnt - m + 1 remaining hops to ex) or leaves the segment.  Returns the
// exit node; n = the symbols on the way.
__device__ __forceinline__ uint32_t tr_walk(uint32_t la_a, uint32_t mk_a, uint32_t wlo, uint32_t i, uint32_t floor_,
                                            uint32_t cnt, uint32_t ex, uint32_t& n) {
  uint32_t h = 0;
  while (i > floor_) {
    uint32_t mk;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(mk) : "r"(mk_a + (i - wlo) * 2));
    if (mk) { n = h + cnt - mk + 1; return ex; }
    i -= tr_hop(la_a, wlo, i);
    h++;
  }
  n = h;
  return i;
}

// TraceBackwards (squeeze.c:317-336) on every thread of the CTA.  Same speculative scheme as the two-warp
// form, with one 128-position segment per thread and windows of kWin positions:
//   pass 1  every thread chases the chain from the top of its segment and numbers the nodes it visits;
//   pass 2  every segment assumes the path enters it where the chain of the segment above leaves, and walks
//           to where it meets its own chain (tr_walk); warp 0 then checks the assumptions 32 segments at a
//           time (entry == exit of the segment above) and re-walks only the segments where one failed;
//   pass 3  every segment writes its symbols at their offset in psym.
// psym[cursor .. nb] comes out as (start position << 9 | length) of the path, in order.  Returns cursor.
template <int NW>
__device__ __noinline__ uint32_t wide_trace(WideSmem<NW>& W, const uint16_t* la, uint64_t* psym, uint32_t nb) {
  constexpr uint32_t kSeg = WideSmem<NW>::kSeg, kWin = WideSmem<NW>::kWin, NT = NW * 32;
  const uint32_t s = threadIdx.x, lane = s & 31u, full = 0xffffffffu;
  const uint32_t la_a = smem_u32(&W.la[0]), mk_a = smem_u32(&W.mark[0]);
  const bool la_odd = (((uintptr_t)la) >> 1) & 1;  // make 4-byte loads aligned
  uint32_t idx = nb, cursor = nb + 1;
  while (idx > 0) {
    // window covers la[wlo .. idx], wlo chosen so that &la[wlo] is 4-byte aligned
    uint32_t wlo = idx >= kWin - 8 ? idx - (kWin - 9) : 0u;
    if (((wlo & 1u) != 0) != la_odd) wlo = wlo > 0 ? wlo - 1 : 0;
    const uint32_t cnt = idx - wlo + 1;
    if ((((uintptr_t)(la + wlo)) & 3) == 0) {
      const uint32_t* src = (const uint32_t*)(la + wlo);
      uint32_t* dst = (uint32_t*)&W.la[0];
      const uint32_t nw = (cnt + 1) / 2;
      for (uint32_t tb = 0; tb < nw; tb += NT * 8) {  // 8 loads in flight per thread
        uint32_t v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) { const uint32_t t = tb + u * NT + s; v[u] = t < nw ? src[t] : 0u; }
#pragma unroll
        for (int u = 0; u < 8; u++) { const uint32_t t = tb + u * NT + s; if (t < nw) dst[t] = v[u]; }
      }
    } else {
      for (uint32_t t = s; t < cnt; t += NT) W.la[t] = la[wlo + t];
    }
    for (uint32_t t = s; t < (cnt + 7) / 8; t += NT) ((uint4*)&W.mark[0])[t] = make_uint4(0, 0, 0, 0);
    cta_sync_all<NW>();
    // ---- pass 1: the speculative chain of this thread's segment ----
    const TrSeg g = tr_seg(idx, wlo, s);
    uint32_t exit_s = g.hi, cnt_s = 0;
    if (g.live) {
      uint32_t i = g.hi;
      while (i > g.floor_) {
        cnt_s++;
        asm volatile("st.shared.u16 [%0], %1;" ::"r"(mk_a + (i - wlo) * 2), "h"((unsigned short)cnt_s) : "memory");
        i -= tr_hop(la_a, wlo, i);
      }
      exit_s = i;
    }
    W.cnt[s] = cnt_s;
    W.exit[s] = exit_s;
    cta_sync_all<NW>();
    // ---- pass 2: walk from the assumed entry ----
    if (g.live) {
      const uint32_t e = s == 0 ? idx : W.exit[s - 1];
      uint32_t n;
      W.in[s] = e;
      W.out[s] = tr_walk(la_a, mk_a, wlo, e, g.floor_, cnt_s, exit_s, n);
      W.ns[s] = n;
    }
    cta_sync_all<NW>();
    // ---- pass 2, warp 0: accept every segment whose entry is the exit of the one above (one ballot per 32 of
    // them), re-walk the first one that is not from its true entry, go on behind it; stop where the path leaves
    // the window or ends ----
    if (s < 32) {
      uint32_t e = idx, tot = 0, nact = kSeg;
      for (uint32_t s0 = 0; s0 < kSeg; s0 += 32) {
        const uint32_t sg = s0 + lane;
        const bool dead = !tr_seg(idx, wlo, sg).live;
        uint32_t gin = W.in[sg], gout = W.out[sg], gn = W.ns[sg];
        uint32_t start = 0, stop = 32;  // lanes below start are settled; the path stops at lane `stop`
        while (start < 32) {
          const uint32_t up = __shfl_up_sync(full, gout, 1);
          const uint32_t ent = lane == start ? e : up;   // true entry, if the lanes in between are right
          const bool halt = dead || ent == 0 || ent < wlo;
          const uint32_t bad = __ballot_sync(full, lane >= start && (halt || gin != ent));
          if (bad == 0) { e = __shfl_sync(full, gout, 31); break; }
          const uint32_t f = __ffs(bad) - 1;
          e = __shfl_sync(full, ent, f);
          if (__shfl_sync(full, halt ? 1u : 0u, f)) { stop = f; break; }
          const TrSeg gf = tr_seg(idx, wlo, s0 + f);
          uint32_t n;
          const uint32_t o = tr_walk(la_a, mk_a, wlo, e, gf.floor_, W.cnt[s0 + f], W.exit[s0 + f], n);
          if (lane == f) { gin = e; gout = o; gn = n; }
          e = o;
          start = f + 1;
        }
        const uint32_t v = lane < stop ? gn : 0u;
        uint32_t incl = v;
#pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(full, incl, d); if (lane >= d) incl += o; }
        if (lane < stop) { W.in[sg] = gin; W.ns[sg] = gn; W.off[sg] = tot + incl - v; }
        tot += __shfl_sync(full, incl, 31);
        if (stop < 32) { nact = s0 + stop; break; }
      }
      if (lane == 0) { W.nact = nact; W.idx = e; W.cursor = cursor - tot; }
    }
    cta_sync_all<NW>();
    // ---- pass 3: write the symbols ----
    const uint32_t nact = W.nact, nidx = W.idx, ncur = W.cursor;
    if (s < nact) {
      uint32_t i = W.in[s];
      const uint32_t n = W.ns[s], top = cursor - W.off[s];
      for (uint32_t k = 0; k < n; k++) {
        const uint32_t l = tr_hop(la_a, wlo, i);
        i -= l;
        psym[top - 1 - k] = ((uint64_t)i << 9) | l;
      }
    }
    idx = nidx;
    cursor = ncur;
    cta_sync_all<NW>();  // the next window reuses la, mark and the segment tables
  }
  return cursor;
}

// follow-path + histogram on every warp: warp w takes a contiguous slice of the nsym symbols and counts into a
// histogram of its own; warp 0 adds them up into s.hist (integer sums: exact in any order)
template <int NW>
__device__ __noinline__ void wide_follow(WideSmem<NW>& W, uint32_t* hist_out, const Batch& b, const SegDesc& sd,
                                         const uint8_t* in, const uint64_t* psym, uint32_t cursor, uint32_t nsym) {
  const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const int cb = (int)W.curbuf;
  uint32_t* h = W.hist[wid];
  for (int i = lane; i < 320; i += 32) h[i] = 0;
  __syncwarp();
  const uint32_t per = ((nsym + NW - 1) / NW + 31) & ~31u;
  const uint32_t t0 = min(nsym, wid * per), t1 = min(nsym, t0 + per);
  follow_path(b, sd, in, psym, cursor, t0, t1, b.st_ll[cb] + sd.pos_off, b.st_d[cb] + sd.pos_off, h, lane);
  cta_sync_all<NW>();
  if (wid == 0) {
    for (int i = lane; i < 320; i += 32) {
      uint32_t c = 0;
#pragma unroll
      for (int w = 0; w < NW; w++) c += W.hist[w][i];
      hist_out[i] = c;
    }
    __syncwarp();
  }
}

// Two warps per block.  Warp 0 runs the whole algorithm; warp 1 is the FEEDER of the forward DP: it
// issues the TMA copies of the match-table rows, stages the per-position scalars (literal cost,
// match length, general-path flags) and writes the finished length_array entries back to global
// memory, three groups of 32 positions ahead of / behind the DP warp (full[] / empty[] mbarriers).
// Outside the DP phase it is parked at a named barrier.
// NW = 2: that pair alone, four CTAs per SM.  NW = 8 (wide form, launches that take whole SMs): warps 2..7
// wait at cta_sync_all during the DP; trace-back and follow-path run on all eight warps (wide_trace,
// wide_follow), the feeder included.
template <int NW>
__global__ void __launch_bounds__(NW * 32, NW == 2 ? 4 : 1) k_iterate(Batch b, const uint32_t* __restrict__ order) {
  static_assert(NW == 2 || NW == 8, "k_iterate: two warps, or the wide form");
  __shared__ IterSmem s;
  extern __shared__ __align__(16) unsigned char zb_iter_dyn[];
  IterDyn& dyn = *reinterpret_cast<IterDyn*>(zb_iter_dyn);
  WideSmem<NW>& W = *reinterpret_cast<WideSmem<NW>*>(zb_iter_dyn + kWideOff);   // wide form only
  const uint32_t seg = order[blockIdx.x], lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const SegDesc sd = b.segs[seg];
  if (sd.mode == 0) return;
  JobState* js = &b.jobs[seg];
  const uint32_t nb = sd.npos;
  if (nb == 0) {
    if (threadIdx.x == 0) { js->best_size = 0; js->best_buf = 0; js->best_cost = 0; js->iters_done = 0; }
    return;
  }
  uint16_t* la = b.la + sd.pos_off + seg;
  uint64_t* psym = b.path + sd.pos_off + seg;  // traced symbols: (start position << 9) | length
  const uint8_t* in = b.in + sd.instart;
  const uint16_t* mlen = b.mlen + sd.pos_off;
  const uint32_t* runs_g = b.runs + sd.pos_off * kRunSlots;
  const uint8_t* dsx_g = b.dsx + sd.pos_off * 32;
  const bool fixed = sd.mode == 2;
  int curbuf = 0, bestbuf = 1;
  uint32_t flags = 0;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; i++) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 1); dyn.tag[i] = 0; dyn.xchi[i] = kIntInf; }
    dyn.gen = 0;
    for (int i = 0; i < 5; i++) s.dpc[i] = 0;
    for (int i = 0; i < 6; i++) s.dpn[i] = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // the staged distance symbols index the cost table: keep every byte of the staging area <= 30
  for (uint32_t t = threadIdx.x; t < sizeof(s.u.dp.dsx) / 4; t += NW * 32) ((uint32_t*)&s.u.dp.dsx[0])[t] = 0;
  __syncthreads();
  uint32_t seq_base = 0;  // running group sequence number: stage = seq & 3, parity = (seq >> 2) & 1
  uint32_t igroups = 0;   // groups that ran in the integer window
  const bool int_on = (b.dp_flags & 1u) != 0;
  uint32_t i_gen = 0;     // generation of the integer tables (DP warp); a stage is usable only if its tag equals it
  const uint32_t ngroups = (nb + 31) >> 5;

  if constexpr (NW > 2) {
    if (wid >= 2) {
      // ================================================================== helper warps (wide form)
      for (;;) {
        cta_sync_all<NW>();  // (C) the DP is over and length_array complete, or warp 0 has finished
        if (*(volatile uint32_t*)&s.go == 0) break;
        const uint32_t cursor = wide_trace<NW>(W, la, psym, nb);
        wide_follow<NW>(W, s.hist, b, sd, in, psym, cursor, nb + 1 - cursor);
      }
      return;
    }
  }
  if (wid == 1) {
    // ================================================================== feeder warp
    for (;;) {
      cta_sync64();  // (A) the DP warp has published go and this iteration's literal costs
      if (*(volatile uint32_t*)&s.go == 0) break;
      const uint32_t end = seq_base + ngroups;
      uint32_t fed = seq_base, fl = seq_base;
      uint32_t pf_m16 = 0, pf_byte = 0;
      { const uint32_t p = lane; if (p < nb) { pf_m16 = mlen[p]; pf_byte = in[p]; } }
      while (fl < end) {
        if (fed < end && fed < fl + 4) {
          // ---- fill stage fed & 3 with group g ----
          const uint32_t g = fed - seq_base, st = fed & 3u;
          const uint32_t m16 = pf_m16;
          const double lc = s.llcost[pf_byte];
          s.u.dp.gl[st * 32 + lane] = lc;
          if (st == 0 && lane < 2) s.u.dp.gl[128 + lane] = lc;
          s.u.dp.mk[st][lane] = (uint16_t)m16;
          {  // integer literal edge from the tables of the generation published right now; the DP warp
             // uses it only if the stage's tag still equals its own generation when it gets there
            const uint32_t gn = *(volatile uint32_t*)&dyn.gen;
            const uint32_t li = dyn.liti[gn & 1u][pf_byte];
            dyn.gli[st * 32 + lane] = li;
            if (st == 0 && lane < 2) dyn.gli[128 + lane] = li;
            if (lane == 0) dyn.tag[st] = gn;
          }
          const uint32_t fw = __ballot_sync(0xffffffffu, (m16 & kShortcutFlag) != 0 || (m16 & 0x7fffu) > 34u);
          const uint32_t fs = __ballot_sync(0xffffffffu, (m16 & kShortcutFlag) != 0);
          if (lane == 0) { s.u.dp.flag[st] = fw; s.u.dp.flagS[st] = fs; }
          { const uint32_t p = (g + 1) * 32 + lane; pf_m16 = 0; pf_byte = 0; if (p < nb) { pf_m16 = mlen[p]; pf_byte = in[p]; } }
          __syncwarp();
          if (lane == 0) {
            const uint32_t cnt = nb - g * 32 < 32u ? nb - g * 32 : 32u, bytes = cnt * 32;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            const uint32_t mirror = st == 0 ? (bytes < 128u ? bytes : 128u) : 0u;
            mbar_expect_tx(&s.full[st], bytes * 2 + mirror);
            bulk_g2s(&s.u.dp.dsx[st * 1024], dsx_g + (size_t)g * 1024, bytes, &s.full[st]);
            if (mirror) bulk_g2s(&s.u.dp.dsx[4096], dsx_g + (size_t)g * 1024, mirror, &s.full[st]);
            bulk_g2s(s.u.dp.runs[st], runs_g + (size_t)g * 256, bytes, &s.full[st]);
          }
          fed++;
        } else {
          // ---- group fl is done: write its length_array entries, which frees its stage ----
          const uint32_t st = fl & 3u;
          mbar_wait(&s.empty[st], (fl >> 2) & 1u);
          const uint32_t p = (fl - seq_base) * 32 + lane;
          if (p < nb) la[p] = (uint16_t)decode_code(s.u.dp.lac[st][lane], p, s.u.dp.ring);
          __syncwarp();
          fl++;
        }
      }
      seq_base = end;
      cta_sync64();  // (B) length_array complete
      if constexpr (NW > 2) {
        cta_sync_all<NW>();  // (C)
        const uint32_t cursor = wide_trace<NW>(W, la, psym, nb);
        wide_follow<NW>(W, s.hist, b, sd, in, psym, cursor, nb + 1 - cursor);
      }
    }
    if constexpr (NW > 2) cta_sync_all<NW>();  // (C) at warp 0's exit: releases the helper warps
    return;
  }
  // ====================================================================== DP warp (warp 0)

  // ---- initial statistics: greedy parse (squeeze.c:481-482) or the fixed tree (:125-140) ----
  if (!fixed) {
    for (int i = lane; i < 320; i += 32) s.stats[i] = 0;
    __syncwarp();
    const uint32_t gs = js->greedy_size;
    const uint16_t* gl = b.st_ll[0] + sd.pos_off;
    const uint16_t* gd = b.st_d[0] + sd.pos_off;
    for (uint32_t tb = 0; tb < gs; tb += 32 * 8) {  // loads batched: the loop is latency-bound otherwise
      uint32_t lv[8], dv[8];
#pragma unroll
      for (int u = 0; u < 8; u++) { const uint32_t t = tb + u * 32 + lane; lv[u] = t < gs ? gl[t] : 0u; dv[u] = t < gs ? gd[t] : 0u; }
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const uint32_t t = tb + u * 32 + lane;
        if (t >= gs) continue;
        const uint32_t l = lv[u], d = dv[u];
        if (d == 0) atomicAdd(&s.stats[l], 1u);
        else { atomicAdd(&s.stats[length_symbol((int)l)], 1u); atomicAdd(&s.stats[288 + dist_symbol((int)d)], 1u); }
      }
    }
    __syncwarp();
    if (lane == 0) s.stats[256] = 1;  // squeeze.c:409
    __syncwarp();
    bool ok = warp_entropy(s.stats, kNumLL, s.llcost, b, lane);
    ok &= warp_entropy(s.stats + 288, kNumD, s.dcost, b, lane);
    if (!ok) flags |= 1;
  } else {
    for (int i = lane; i < kNumLL; i += 32) s.llcost[i] = (double)fixed_ll_length(i);
    if (lane < kNumD) s.dcost[lane] = 5.0;
  }
  __syncwarp();

  uint64_t bestcost = ~(uint64_t)0, lastcost = 0;
  uint32_t ran_w = 1, ran_z = 2;  // squeeze.c:85-88
  int lastrandomstep = -1;
  uint32_t best_size = 0;
  const int niter = fixed ? 1 : sd.numiterations;
  int it = 0;
  long long cyc[6] = {0, 0, 0, 0, 0, 0};
  long long tk = clock64();
#define ZB_TICK(i) do { long long t_ = clock64(); cyc[i] += t_ - tk; tk = t_; } while (0)

  for (; it < niter && !(flags & 1); it++) {
    // ------------------------------------------------------------------ model constants
    for (int k = lane; k < 260; k += 32) s.lencost[k] = k >= 3 && k <= 258 ? s.llcost[length_symbol(k)] : 0.0;
    __syncwarp();
    for (int i = lane; i < 31 * 64; i += 32) {  // GetCostStat squeeze.c:146-157 for lengths 3..34
      const int ds = i >> 6, k = 3 + ((i + 31) & 31);
      s.t0[i] = ds < 30 ? (double)(length_extra_bits(k) + dist_symbol_extra_bits(ds)) + s.lencost[k] + s.dcost[ds] : 1e300;
    }
    __syncwarp();
    double mincost;
    {
      double bv = 1e30; int bi = 0x7fffffff;
      for (int k = 3 + (int)lane; k < 259; k += 32) {  // squeeze.c:181-187, dist 1
        double c = (double)(length_extra_bits(k) + 0) + s.lencost[k] + s.dcost[0];
        if (c < bv) { bv = c; bi = k; }
      }
      if (!(bv < 1e30)) bi = 0x7fffffff;
      warp_min_first(bv, bi);
      bi = __shfl_sync(0xffffffffu, bi, 0);
      const int bestlength = bi == 0x7fffffff ? 0 : bi;
      double dv = 1e30; int di = 0x7fffffff;
      if (lane < 30) {  // squeeze.c:190-196, length 3
        double c = (double)(0 + dist_symbol_extra_bits((int)lane)) + s.lencost[3] + s.dcost[lane];
        if (c < dv) { dv = c; di = (int)lane; }
      }
      warp_min_first(dv, di);
      di = __shfl_sync(0xffffffffu, di, 0);
      // squeeze.c:198 costmodel(bestlength, bestdist); bestlength/bestdist stay 0 if nothing
      // was below 1e30 (not reachable with finite entropies)
      const int bl = bestlength, dsym = di == 0x7fffffff ? 0 : di;
      mincost = (double)(length_extra_bits(bl) + dist_symbol_extra_bits(dsym)) + s.lencost[bl < 3 ? 3 : bl] + s.dcost[dsym];
    }
    // squeeze.c:293 skips an edge when costs[j+k] <= mincost + costs[j].  That is a pure
    // optimisation exactly when mincost <= every edge cost the model can produce (then
    // cost + c_j >= mincost + c_j by monotonicity of rounding and the edge could not win anyway).
    // Check it for all 256 x 30 (length, distance symbol) pairs; if it ever fails, the fast path
    // is disabled for this iteration and every edge goes through the explicit test.
    bool skip_noop;
    double margin_dn, margin_up;  // how far the cost can move below / above its value at a group start (see "magic" below)
    {
      double mn = 1e300, mx = 0.0, ml = 0.0;
      for (int k = 3 + (int)lane; k < 259; k += 32) {
        const int lb = length_extra_bits(k);
        const double lc = s.lencost[k];
        for (int ds = 0; ds < 30; ds++) {
          const double c = (double)(lb + dist_symbol_extra_bits(ds)) + lc + s.dcost[ds];
          mn = c < mn ? c : mn;
          mx = c > mx ? c : mx;
        }
      }
      for (int i = lane; i < 256; i += 32) ml = s.llcost[i] > ml ? s.llcost[i] : ml;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        const double o = __shfl_xor_sync(0xffffffffu, mn, d); mn = o < mn ? o : mn;
        const double p = __shfl_xor_sync(0xffffffffu, mx, d); mx = p > mx ? p : mx;
        const double q = __shfl_xor_sync(0xffffffffu, ml, d); ml = q > ml ? q : ml;
      }
      skip_noop = mincost <= mn;
      margin_dn = 258.0 * ml + 1.0;
      margin_up = 36.0 * ml + mx + 1.0;
    }
    const double cost258 = (double)(0 + 0) + s.lencost[258] + s.dcost[0];  // costmodel(258, 1)
    ZB_TICK(0);

    // ------------------------------------------------------------------ forward DP
    // Push form with a REGISTER WINDOW.  Lane l owns the targets t == l (mod 32): at step j it
    // holds pending(t) for the one such t in [j+3, j+34], complete for sources < j, and relaxes it
    // with length k = t - j.  The lane whose target is j+3 hands its completed value to the chain
    // (it meets the literal edge two steps later) and takes on target j+35.  The short edges never
    // touch memory; only edges longer than 34 (rare outside byte runs) go through a shared-memory
    // ring whose entry joins the window when its target comes within reach.  Costs are doubles that
    // are exactly float-representable: the reference stores floats and widens them on every use
    // (squeeze.c:222,278-300); rounding is done in integer arithmetic.  Relaxation order per target
    // is source order, as in the reference, so ties resolve identically.  The window keeps a
    // length CODE (which step produced the edge), decoded when length_array is written.
    const double kInfD = (double)(float)1e30;  // ZOPFLI_LARGE_FLOAT stored to float, squeeze.c:243
    for (int t = lane; t < 512; t += 32) { s.u.dp.ring[t].fb = kInfBits; s.u.dp.ring[t].code = 0; }
    if (lane < 4) { s.u.dp.xch[lane].c = kInfD; s.u.dp.xch[lane].code = 0; }
    i_gen++;  // new cost model: stages tagged with an older generation (or this one, which has no tables) are fp64-only
    if (lane == 0) { s.go = 1; *(volatile uint32_t*)&dyn.gen = i_gen; }
    __syncwarp();
    cta_sync64();  // (A) start the feeder
    {
      // shared-memory base addresses, kept opaque so they stay in registers
      // this lane's cost-table column at step jl' of a group is t0_l - 8 jl' for jl' in [2, 33] (32, 33: steps 0, 1 of the next group)
      uint32_t t0_l = smem_u32(&s.t0[0]) + (((lane - 3u) & 31u) + 33u) * 8u;
      uint32_t dsx_r = smem_u32(&s.u.dp.dsx[0]) + lane, gl_r = smem_u32(&s.u.dp.gl[0]);
      uint32_t ring_r = smem_u32(&s.u.dp.ring[0]), lac_r = smem_u32(&s.u.dp.lac[0][0]), mk_r = smem_u32(&s.u.dp.mk[0][0]);
      asm volatile("" : "+r"(t0_l), "+r"(dsx_r), "+r"(gl_r), "+r"(ring_r), "+r"(lac_r), "+r"(mk_r));
      const bool is_l0 = lane == 0;
      double w = kInfD; uint32_t wl = 0;
      double e2c = kInfD; uint32_t e2l = 0;  // pending(j+1)
      uint32_t xch_r = smem_u32(&s.u.dp.xch[0]), full_r = smem_u32(&s.full[0]), empty_r = smem_u32(&s.empty[0]);
      uint32_t flag_r = smem_u32(&s.u.dp.flag[0]);
      asm volatile("" : "+r"(xch_r), "+r"(full_r), "+r"(empty_r), "+r"(flag_r));
      // magic-rounding state: the constant and the cost interval it is valid for (see below)
      double Cm = 0.0, mg_lo = 1.0, mg_hi = 0.0;
      double cj = 0.0;
      uint32_t lfin_prev = 0;           // code of length_array[j], stored one step late
      uint32_t dirty_until = 0;         // largest target that has a ring entry
      uint32_t skip_left = 0, guard_until = 0;
      bool just_finished = false;
      // operand pipeline, two steps deep so that no shared-memory latency meets the cost chain:
      // tv / tv1 = edge costs for steps j, j+1; ds2 = distance symbol for step j+2; llb / llb1 = literal costs
      mbar_wait_a(full_r + (seq_base & 3u) * 8, (seq_base >> 2) & 1u);
      double tv, tv1, llb, llb1;
      uint32_t ds2;
      {
        const uint32_t d0 = dsx_r + (seq_base & 3u) * 1024, g0 = gl_r + (seq_base & 3u) * 256;
        tv = lds_f64(t0_l + lds_u8(d0) * 512 - 32 * 8);
        tv1 = lds_f64(t0_l + lds_u8(d0 + 32) * 512 - 33 * 8);
        ds2 = lds_u8(d0 + 64);
        llb = lds_f64(g0);
        llb1 = lds_f64(g0 + 8);
      }

      // one step of the common case: no shortcut, no length > 34 at this position, the squeeze.c:293
      // test proven redundant.  Straight-line code in blocks of eight steps (the loop body has to
      // stay inside the ~6 KB L0 instruction cache: a single warp cannot hide instruction fetches);
      // U, the step within the block, is a literal, so every shared-memory address is a register
      // plus an immediate.  RING: join/clear ring entries.
#define ZB_DP_FAST_STEP(U, RING, MAGIC)                                                                          \
      {                                                                                                     \
        const double tv2_ = lds_f64(t0_s + ds2 * 512 - (((U) + 2) * 8));                                    \
        const uint32_t ds3_ = lds_u8(dsx_s + (((U) + 3) * 32));                                             \
        const double llb2_ = lds_f64(gl_s + (((U) + 2) * 8));                                               \
        double en_c_; uint32_t en_l_;                                                                       \
        lds_ring(xch_r + ((((U) + 3) & 3) * 16), en_c_, en_l_);   /* pending(j+2), made at step j-1 */       \
        double inc_ = kInfD; uint32_t inl_ = 0;                                                             \
        if (RING) { uint32_t fb_; lds_ring8(ring_s + (U) * 8, fb_, inl_); inc_ = (double)__uint_as_float(fb_);    \
                    sts_u32_if(ring_s + (U) * 8, kInfBits, is_l0); }                                         \
        sts_u16_if(lac_s + (U) * 2, lfin_prev, is_l0);                                                      \
        const double lit_ = llb + cj;                                                                       \
        double rl_ = (MAGIC) ? (lit_ + Cm) - Cm : round_to_f32(lit_);   /* unconditional: runs beside the compare */ \
        asm volatile("" : "+d"(rl_));                                                                       \
        const bool take_ = lit_ < e2c;                                                                      \
        const double cnext_ = take_ ? rl_ : e2c;                                                            \
        lfin_prev = take_ ? kCodeLit : e2l;                                                                 \
        const double nc_ = tv + cj;                                                                         \
        double rn_ = (MAGIC) ? (nc_ + Cm) - Cm : round_to_f32(nc_);                                         \
        asm volatile("" : "+d"(rn_));                                                                       \
        const bool ok_ = nc_ < w;                                                                           \
        w = ok_ ? rn_ : w;                                                                                  \
        wl = ok_ ? sidx : wl;                                                                               \
        const bool mine_ = lane_rot == (uint32_t)(U);   /* this lane's target is j+3: complete now */       \
        sts_ring_if(xch_r + (((U) & 3) * 16), w, wl, mine_);                                                \
        if (mine_) { w = inc_; wl = inl_; }                                                                 \
        sidx++;                                                                                             \
        e2c = en_c_; e2l = en_l_;                                                                           \
        cj = cnext_;                                                                                        \
        tv = tv1; tv1 = tv2_; ds2 = ds3_; llb = llb1; llb1 = llb2_;                                         \
      }
#define ZB_DP_FAST_4A(R, M) ZB_DP_FAST_STEP(0, R, M) ZB_DP_FAST_STEP(1, R, M) ZB_DP_FAST_STEP(2, R, M) ZB_DP_FAST_STEP(3, R, M)
#define ZB_DP_FAST_4B(R, M) ZB_DP_FAST_STEP(4, R, M) ZB_DP_FAST_STEP(5, R, M) ZB_DP_FAST_STEP(6, R, M) ZB_DP_FAST_STEP(7, R, M)
#define ZB_DP_FAST_8(R, M) ZB_DP_FAST_4A(R, M) ZB_DP_FAST_4B(R, M)
#define ZB_DP_FAST_GROUP(R, M)                                                                               \
      {                                                                                                     \
        uint32_t t0_s = t0_l, dsx_s = dsx_c, gl_s = gl_c, lac_s = lac_c, ring_s = ring_c;                   \
        uint32_t lane_rot = (lane - 3u) & 31u, sidx = 3u;   /* sidx = (step & 31) + 3: shuffle source and length code */ \
        _Pragma("unroll 1")                                                                                 \
        for (int sb_ = 0; sb_ < 4; sb_++) {                                                                 \
          ZB_DP_FAST_8(R, M)                                                                                \
          t0_s -= 64; dsx_s += 256; gl_s += 64; lac_s += 16; ring_s += 64;                                  \
          lane_rot = (lane_rot - 8u) & 31u;                                                                 \
        }                                                                                                   \
      }

      // ---- integer window: one step = two VIADDMNMX (literal edge against pending(j+1); this lane's length
      // edge against its pending target) and one LOP3 (strip the tiebreak bits) on the chain ----
#define ZB_DPI_STEP(U, RING)                                                                                \
      {                                                                                                     \
        const uint32_t tv2_ = lds_u32(ti_s + ds2 * 256 - (((U) + 2) * 4));                                  \
        const uint32_t ds3_ = lds_u8(dsx_s + (((U) + 3) * 32));                                             \
        const uint32_t llb2_ = lds_u32(gli_s + (((U) + 2) * 4));                                            \
        const uint32_t en_ = lds_u32(xchi_r + ((((U) + 3) & 3) * 4));   /* pending(j+2), made at step j-1 */ \
        uint32_t inc_ = kIntInf;                                                                            \
        if (RING) {   /* the ring entry of target j+35 joins the window (float bits -> packed word, order 0) */ \
          uint32_t fb_, cd_;                                                                                \
          lds_ring8(ring_s + (U) * 8, fb_, cd_); (void)cd_;                                                 \
          inc_ = fb_ == kInfBits ? kIntInf : (((fb_ - i_base) << 7) | 64u);                                 \
          sts_u32_if(ring_s + (U) * 8, kInfBits, is_l0);                                                    \
        }                                                                                                   \
        sts_u16_if(lac_s + (U) * 2, lfin_prev, is_l0);                                                      \
        const uint32_t x_ = __viaddmin_u32(CJ, llbI, e2I);   /* literal edge against pending(j+1) */        \
        lfin_prev = (x_ & 127u) | kCodeInt;                                                                 \
        wI = __viaddmin_u32(CJ, tvI, wI);                   /* this lane's length edge */                  \
        const bool mine_ = lane_rot == (uint32_t)(U);   /* this lane's target is j+3: complete now */       \
        sts_u32_if(xchi_r + (((U) & 3) * 4), wI, mine_);                                                    \
        wI = mine_ ? inc_ : wI;                                                                             \
        e2I = en_; CJ = x_ & ~127u;                                                                         \
        tvI = tv1I; tv1I = tv2_; ds2 = ds3_; llbI = llb1I; llb1I = llb2_;                                   \
      }
#define ZB_DPI_4A(R) ZB_DPI_STEP(0, R) ZB_DPI_STEP(1, R) ZB_DPI_STEP(2, R) ZB_DPI_STEP(3, R)
#define ZB_DPI_4B(R) ZB_DPI_STEP(4, R) ZB_DPI_STEP(5, R) ZB_DPI_STEP(6, R) ZB_DPI_STEP(7, R)
#define ZB_DPI_GROUP(ST)                                                                                    \
      {                                                                                                     \
        uint32_t ti_s = ti_l, dsx_s = dsx_r + (ST) * 1024, gli_s = gli_r + (ST) * 128, lac_s = lac_r + (ST) * 64; \
        uint32_t lane_rot = (lane - 3u) & 31u;                                                              \
        const uint32_t ring_s = 0; (void)ring_s;                                                            \
        _Pragma("unroll 1")                                                                                 \
        for (int sb_ = 0; sb_ < 2; sb_++) {                                                                 \
          ZB_DPI_4A(false) ZB_DPI_4B(false)                                                                 \
          ZB_DPI_STEP(8, false) ZB_DPI_STEP(9, false) ZB_DPI_STEP(10, false) ZB_DPI_STEP(11, false)         \
          ZB_DPI_STEP(12, false) ZB_DPI_STEP(13, false) ZB_DPI_STEP(14, false) ZB_DPI_STEP(15, false)       \
          ti_s -= 64; dsx_s += 512; gli_s += 64; lac_s += 32;                                               \
          lane_rot = (lane_rot - 16u) & 31u;                                                                \
        }                                                                                                   \
      }
      uint32_t ti_l = smem_u32(&dyn.ti[0]) + (((lane - 3u) & 31u) + 33u) * 4u;   // this lane's column, as t0_l
      uint32_t gli_r = smem_u32(&dyn.gli[0]), xchi_r = smem_u32(&dyn.xchi[0]), tag_r = smem_u32(&dyn.tag[0]);
      uint32_t tl_r = smem_u32(&dyn.tl[0]), flagS_r = smem_u32(&s.u.dp.flagS[0]);
      asm volatile("" : "+r"(ti_l), "+r"(gli_r), "+r"(xchi_r), "+r"(tag_r), "+r"(tl_r), "+r"(flagS_r));
      bool imode = false, i_ok = false;   // window currently held as integers; tables of i_lowb usable
      long long i_lowb = -1;              // exponent bits of the binade the tables were (or could not be) built for
      uint32_t i_base = 0, i_hi = 0;      // float bits of 2^e; upper end of the interval of CJ the mode is valid in
      double i_lo_d = 1.0, i_hi_d = 0.0, i_top = 0.0;
      uint32_t wI = kIntInf, e2I = kIntInf, CJ = 0, tvI = 0, tv1I = 0, llbI = 0, llb1I = 0;
      // fp64 value + length code <-> packed word (entries carried over lose their `up` bit, which only matters
      // against EARLIER sources: 64 + o loses to every later source that rounds up and beats every later one that does not)
      auto d2i = [&](double c, uint32_t code, uint32_t target) -> uint32_t {
        if (!(c < i_top)) return kIntInf;   // beyond the binade: cannot be the minimum of a target finished in this group
        const uint32_t o = (code & kCodeLong) ? 0u : 35u - decode_len(code, target);
        return ((__float_as_uint(__double2float_rn(c)) - i_base) << 7) | (64u + o);
      };
      auto i2d = [&](uint32_t pw, uint32_t target, double& c, uint32_t& code) {
        if (pw >= kIntNoEdge) { c = kInfD; code = 0; return; }
        c = (double)__uint_as_float((pw >> 7) + i_base);
        const uint32_t tb = pw & 127u, o = tb < 64u ? 63u - tb : tb - 64u;
        code = o == 0u ? s.u.dp.ring[(target - 3u) & 511u].code : ((target - (35u - o)) & 31u) + 3u;
      };

      uint32_t flag_pref = lds_u32(flag_r + (seq_base & 3u) * 4);  // flags of a group are fetched one group ahead
      long long tg = clock64();
      uint32_t nslow = 0;
#ifdef ZB_DP_KINDS   /* developer build: DP cycles by kind of group (tools/one_block.py prints them) */
#define ZB_KIND_TICK(K) if (lane == 0) { const long long t_ = clock64(); s.dpc[K] += (unsigned long long)(t_ - tg); s.dpn[K]++; tg = t_; }
#else
#define ZB_KIND_TICK(K)
#endif
      for (uint32_t g = 0; g < ngroups;) {
        uint32_t kind = 4;
        const uint32_t j0 = g * 32, q = seq_base + g, st = q & 3u, stn = (q + 1) & 3u;
        if (g + 1 < ngroups) mbar_wait_a(full_r + stn * 8, ((q + 1) >> 2) & 1u);  // the operand pipeline runs into the next group
        const uint32_t flag_cur = flag_pref;
        if (g + 1 < ngroups) flag_pref = lds_u32(flag_r + stn * 4);
        const uint32_t dsx_c = dsx_r + st * 1024, gl_c = gl_r + st * 256;
        const uint32_t lac_c = lac_r + st * 64;
        const uint32_t ring_c = ring_r + ((j0 + 32) & 511u) * 8;   // slot of target j0 + 35
        const bool fast = skip_noop && flag_cur == 0 && skip_left == 0 && !just_finished && j0 + 32 <= nb;
        const uint32_t gli_c = gli_r + st * 128;
        // ---- integer window: stay / enter / leave ----
        // The integer window takes every group without long-run shortcut activity: plain ones, and ones with
        // matches longer than 34 / ring entries to join (long edges are priced from dyn.tl, straight into the ring).
        bool want_int = false;
        const bool calm = skip_noop && int_on && skip_left == 0 && !just_finished && j0 + 32 <= nb && j0 >= guard_until &&
                          lds_u32(flagS_r + st * 4) == 0;
        if (calm) {
          if (imode) {
            want_int = CJ < i_hi;   // words only grow by positive edges: nothing falls below the binade once inside
          } else {
            const long long lowb = __double_as_longlong(cj) & 0x7ff0000000000000LL;
            if (lowb != i_lowb) {  // a binade not looked at yet: build its tables (k1, up per edge), or rule it out
              i_lowb = lowb; i_ok = false;
              const double B = __longlong_as_double(lowb);
              i_top = B + B; i_lo_d = B; i_hi_d = i_top - margin_up;
              if (lowb > 0 && i_lo_d < i_hi_d) {
                const uint32_t base = __float_as_uint(__double2float_rn(B));
                const double half_ulp = __longlong_as_double(lowb - (24LL << 52));
                bool tie = false;
                i_gen++;
                uint32_t* lt = dyn.liti[i_gen & 1u];
                for (int i = lane; i < 31 * 64; i += 32) {
                  const uint32_t o = 35u - (3u + (((uint32_t)i + 31u) & 31u));   // order of this length among a target's sources
                  uint32_t E = kIntNoEdge | (64u + o);
                  if (i < 30 * 64) {
                    const double s0 = B + s.t0[i];          // the edge cost on the binade's double grid
                    const float f = __double2float_rn(s0);
                    const double df = (double)f;
                    tie |= fabs(df - s0) == half_ulp;
                    E = ((__float_as_uint(f) - base) << 7) | (df > s0 ? 63u - o : 64u + o);
                  }
                  dyn.ti[i] = E;
                }
                for (int i = lane; i < 256; i += 32) {
                  const double s0 = B + s.llcost[i];
                  const float f = __double2float_rn(s0);
                  const double df = (double)f;
                  tie |= fabs(df - s0) == half_ulp;
                  lt[i] = ((__float_as_uint(f) - base) << 7) | (df > s0 ? 63u - 33u : 64u + 33u);
                }
                for (int i = lane; i < 29 * 32; i += 32) {   // the cost of a length depends on it only through its symbol
                  const int ls = 257 + (i >> 5), ds = i & 31;
                  uint32_t E = 0;
                  if (ds < 30) {
                    const double s0 = B + ((double)(length_symbol_extra_bits(ls) + dist_symbol_extra_bits(ds)) + s.llcost[ls] + s.dcost[ds]);
                    const float f = __double2float_rn(s0);
                    const double df = (double)f;
                    tie |= fabs(df - s0) == half_ulp;
                    E = ((__float_as_uint(f) - base) << 1) | (df > s0 ? 1u : 0u);
                  }
                  dyn.tl[i] = E;
                }
                tie = __any_sync(0xffffffffu, tie);
                __syncwarp();
                __threadfence_block();
                if (lane == 0) *(volatile uint32_t*)&dyn.gen = i_gen;
                i_base = base; i_ok = !tie;
                i_hi = (__float_as_uint(__double2float_rd(i_hi_d)) - base) << 7;
              }
            }
            want_int = i_ok && cj >= i_lo_d && cj < i_hi_d;
          }
          if (want_int) {  // the staged literal edges must come from the current tables (this stage and the one the pipeline runs into)
            const uint32_t tag0 = lds_u32(tag_r + st * 4), tag1 = g + 1 < ngroups ? lds_u32(tag_r + stn * 4) : i_gen;
            want_int = tag0 == i_gen && tag1 == i_gen;
          }
          if (want_int && !imode) {  // every pending value the window holds must lie in the binade (or be infinite) to be carried over
            double xc; uint32_t xl;
            lds_ring(xch_r + ((j0 + 3u) & 3u) * 16, xc, xl);
            (void)xl;
            want_int = __all_sync(0xffffffffu, !(w < i_lo_d) && !(e2c < i_lo_d) && !(xc < i_lo_d));
            if (want_int && j0 + 35 <= dirty_until) {  // so must every finite ring entry: it joins as an integer
              bool okr = true;
              for (int t = lane; t < 512; t += 32) { const uint32_t fb = s.u.dp.ring[t].fb; okr &= fb == kInfBits || (fb - i_base) < (1u << 23); }
              want_int = __all_sync(0xffffffffu, okr);
            }
          }
        }
        if (imode != want_int) {
          const uint32_t t_l = j0 + 3u + ((lane - 3u) & 31u), xs = (j0 + 3u) & 3u;   // this lane's target; slot of pending(j0+2)
          if (want_int) {
            wI = d2i(w, wl, t_l);
            e2I = d2i(e2c, e2l, j0 + 1u);
            { double xc; uint32_t xl; lds_ring(xch_r + xs * 16, xc, xl); const uint32_t xp = d2i(xc, xl, j0 + 2u); if (is_l0) dyn.xchi[xs] = xp; }
            CJ = (__float_as_uint(__double2float_rn(cj)) - i_base) << 7;
            __syncwarp();
            tvI = lds_u32(ti_l + lds_u8(dsx_c) * 256 - 32 * 4);
            tv1I = lds_u32(ti_l + lds_u8(dsx_c + 32) * 256 - 33 * 4);
            llbI = lds_u32(gli_c);
            llb1I = lds_u32(gli_c + 4);
          } else {
            i2d(wI, t_l, w, wl);
            i2d(e2I, j0 + 1u, e2c, e2l);
            { double xc; uint32_t xl; i2d(lds_u32(xchi_r + xs * 4), j0 + 2u, xc, xl); sts_ring_if(xch_r + xs * 16, xc, xl, is_l0); }
            cj = (double)__uint_as_float((CJ >> 7) + i_base);
            __syncwarp();
            tv = lds_f64(t0_l + lds_u8(dsx_c) * 512 - 32 * 8);
            tv1 = lds_f64(t0_l + lds_u8(dsx_c + 32) * 512 - 33 * 8);
            llb = lds_f64(gl_c);
            llb1 = lds_f64(gl_c + 8);
          }
          imode = want_int;
        }
        if (imode && (flag_cur != 0 || j0 + 35 <= dirty_until)) {
          // ---- integer general group, in halves of four steps like the fp64 one: halves without a long match run
          // the straight-line step (ring-joining variant), the others go step by step and push their long edges ----
          for (uint32_t hb = 0; hb < 8; hb++) {
            const uint32_t sb = hb >> 1, jb = j0 + hb * 4;
            if (((flag_cur >> (hb * 4)) & 0xfu) == 0) {
              uint32_t ti_s = ti_l - sb * 32, dsx_s = dsx_c + sb * 256, gli_s = gli_c + sb * 32, lac_s = lac_c + sb * 16;
              uint32_t ring_s = ring_c + sb * 64, lane_rot = (lane - 3u - sb * 8u) & 31u;
              if (hb & 1) { ZB_DPI_4B(true) } else { ZB_DPI_4A(true) }
              continue;
            }
            nslow += 4;
            for (uint32_t j = jb; j < jb + 4; j++) {
              const uint32_t jl = j & 31u;
              const uint32_t tv2_ = lds_u32(ti_l + ds2 * 256 - (jl + 2) * 4);
              const uint32_t ds3_ = lds_u8(dsx_c + (jl + 3) * 32);
              const uint32_t llb2_ = lds_u32(gli_c + (jl + 2) * 4);
              const uint32_t en_ = lds_u32(xchi_r + ((j + 3) & 3) * 4);
              sts_u16_if(lac_c + jl * 2, lfin_prev, is_l0);
              const bool lng = ((flag_cur >> jl) & 1u) != 0;   // no shortcut candidates in this group: the flag means length > 34
              const uint32_t x_ = __viaddmin_u32(CJ, llbI, e2I);
              lfin_prev = (x_ & 127u) | kCodeInt;
              wI = __viaddmin_u32(CJ, tvI, wI);
              if (lng) {  // lengths 35..: first strict improvement wins, on float bits (squeeze.c:286-302)
                const uint32_t ml = lds_u16(mk_r + st * 64 + jl * 2) & 0x7fffu;
                const uint32_t room = nb - j;
                const uint32_t kend = ml < room ? ml : room;
                const uint4* st4 = (const uint4*)&s.u.dp.runs[st][jl * kRunSlots];
                const uint4 ea = st4[0], eb = st4[1];
                const uint32_t cjb = i_base + (CJ >> 7);
                for (uint32_t k = 35 + lane; k <= kend; k += 32) {
                  const uint32_t tga = ring_r + ((j + k - 3) & 511) * 8;
                  const uint32_t pendb = lds_u32(tga);
                  const uint32_t dsym = run_dsym(run_for_len(ea, eb, k, b.ovf));
                  const uint32_t E = lds_u32(tl_r + (((uint32_t)length_symbol((int)k) - 257u) * 32u + dsym) * 4u);
                  const uint32_t rl = cjb + (E >> 1);
                  sts_ring8_if(tga, rl, kCodeLong | k, rl < pendb || (rl == pendb && (E & 1u) != 0));
                }
                if (j + kend > dirty_until) dirty_until = j + kend;
              }
              const uint32_t src = (j + 3) & 31;
              sts_u32_if(xchi_r + (j & 3) * 4, wI, lane == src);
              uint32_t inc = kIntInf;
              if (lng) __syncwarp();   // this step's own length-35 edge lands in the slot that joins now
              if (j + 35 <= dirty_until) {
                const uint32_t ra = ring_r + ((j + 32) & 511) * 8;
                uint32_t fbj, cdj;
                lds_ring8(ra, fbj, cdj);
                (void)cdj;
                inc = fbj == kInfBits ? kIntInf : (((fbj - i_base) << 7) | 64u);
                sts_u32_if(ra, kInfBits, lane == 0);   // free the slot for target j+35+512 (first written 254 steps from now)
              }
              if (lane == src) wI = inc;
              e2I = en_; CJ = x_ & ~127u;
              tvI = tv1I; tv1I = tv2_; ds2 = ds3_; llbI = llb1I; llb1I = llb2_;
            }
          }
          igroups++;
          kind = 3;
        } else if (imode) {
          // Integer groups run back to back in a loop of their own: the conditions that can change from one
          // group to the next (flags of the next group, the interval, the block end, the tag of the stage the
          // pipeline runs into) cost a dozen instructions; everything else (ring clean, no shortcut zone nearby)
          // cannot change while no long edge is pushed.  Anything else goes back to the top of the outer loop.
          uint32_t stc = st;
          for (;;) {
            ZB_DPI_GROUP(stc)
            igroups++;
            __syncwarp();
            if (lane == 0) mbar_arrive_a(empty_r + stc * 8);
            ZB_KIND_TICK(0)
            g++;
            if (g + 1 >= ngroups) break;
            const uint32_t qn = seq_base + g + 1u, st2 = qn & 3u;
            mbar_wait_a(full_r + st2 * 8, (qn >> 2) & 1u);
            const uint32_t fl2 = lds_u32(flag_r + st2 * 4), tg2 = lds_u32(tag_r + st2 * 4);
            if (flag_pref != 0 || !(CJ < i_hi) || (g + 1u) * 32u > nb || tg2 != i_gen) break;
            flag_pref = fl2;
            stc = (seq_base + g) & 3u;
          }
          continue;
        } else if (fast) {
          // "magic" rounding: while every cost of the group provably stays inside one binade
          // [2^k, 2^(k+1)), round-to-float is (x + C) - C with C = 1.5 * 2^(k+29) (the double grid at
          // C is the float grid of the binade, ties to even alike) -- two DADDs instead of five
          // dependent integer operations on the cost chain.  Costs are shortest-path distances with
          // a literal edge at every position, so within the group they stay above
          // c - 258 maxlit and below c + 32 maxlit (+ the largest edge for relaxed values);
          // positions after a long-run shortcut (no literal edges there) are excluded.
          bool magic = false;
          if (j0 + 35 > dirty_until && j0 >= guard_until) {
            if (!(cj >= mg_lo && cj < mg_hi)) {  // left the interval the constant was made for: look at the binade again
              const long long lowb = __double_as_longlong(cj) & 0x7ff0000000000000LL;
              mg_lo = __longlong_as_double(lowb) + margin_dn;
              mg_hi = __longlong_as_double(lowb + 0x0010000000000000LL) - margin_up;
              Cm = __longlong_as_double(lowb + (29LL << 52) + (1LL << 51));
              if (lowb <= 0) { mg_lo = 1.0; mg_hi = 0.0; }
            }
            magic = cj >= mg_lo && cj < mg_hi;
          }
          if (magic) { kind = 1; ZB_DP_FAST_GROUP(false, true) }
          else if (j0 + 35 > dirty_until) { kind = 2; ZB_DP_FAST_GROUP(false, false) }
          else { kind = 3; ZB_DP_FAST_GROUP(true, false) }
        } else {
          // ---- general group, in half-blocks of four steps: a half without a flagged position still
          // runs the straight-line code (ring-joining variant); only the others check per step.  (Halves
          // rather than whole eight-step blocks: a flagged position drags three neighbours through the
          // slow loop instead of seven.) ----
          for (uint32_t hb = 0; hb < 8; hb++) {
          const uint32_t sb = hb >> 1, jb = j0 + hb * 4;
          if (jb >= nb) break;
          if (skip_noop && ((flag_cur >> (hb * 4)) & 0xfu) == 0 && skip_left == 0 && !just_finished && jb + 4 <= nb) {
            uint32_t t0_s = t0_l - sb * 64, dsx_s = dsx_c + sb * 256, gl_s = gl_c + sb * 64, lac_s = lac_c + sb * 16;
            uint32_t ring_s = ring_c + sb * 64, lane_rot = (lane - 3u - sb * 8u) & 31u, sidx = 3u + hb * 4u;
            if (hb & 1) { ZB_DP_FAST_4B(true, false) } else { ZB_DP_FAST_4A(true, false) }
            (void)lane_rot;
            continue;
          }
          const uint32_t jend = jb + 4 < nb ? jb + 4 : nb;
          nslow += jend - jb;
          for (uint32_t j = jb; j < jend; j++) {
            const uint32_t jl = j & 31u;
            const double tv2 = lds_f64(t0_l + ds2 * 512 - (jl + 2) * 8);
            const uint32_t ds3 = lds_u8(dsx_c + (jl + 3) * 32);   // rows 32.. are the next stage (or its mirror)
            const double llb2 = lds_f64(gl_c + (jl + 2) * 8);
            double en_c; uint32_t en_l;
            lds_ring(xch_r + ((j + 3) & 3) * 16, en_c, en_l);  // pending(j+2), made at step j-1
            sts_u16_if(lac_c + jl * 2, lfin_prev, is_l0);
            const uint32_t m16 = lds_u16(mk_r + st * 64 + jl * 2);
            const uint32_t ml = m16 & 0x7fffu;
            double cnext;
            bool relax = true;
            // long-run shortcut squeeze.c:251-271 (candidate flag precomputed by k_match)
            if ((m16 & kShortcutFlag) && skip_left == 0 && !just_finished) skip_left = kMaxMatch;
            if (skip_left > 0) {
              // costs[j+258] = costs[j] + cost(258,1), unconditionally; no literal, no other edge
              sts_ring8_if(ring_r + ((j + kMaxMatch - 3) & 511) * 8, __float_as_uint(__double2float_rn(cj + cost258)), kCodeLong | (uint32_t)kMaxMatch, lane == 0);
              if (j + kMaxMatch > dirty_until) dirty_until = j + kMaxMatch;
              skip_left--;
              guard_until = j + 600;
              just_finished = skip_left == 0;
              relax = false;
            } else {
              just_finished = false;
            }
            if (relax) {
              // literal squeeze.c:277-284 (every lane computes the same values)
              const double lit = llb + cj;
              const bool take = lit < e2c;
              cnext = take ? round_to_f32(lit) : e2c;
              lfin_prev = take ? kCodeLit : e2l;
              // lengths 3..34 squeeze.c:286-302: this lane's length is target - j
              const double nc = tv + cj;
              const double mc = mincost + cj;
              const bool ok = !(w <= mc) & (nc < w);
              w = ok ? round_to_f32(nc) : w;
              wl = ok ? jl + 3u : wl;
              if (ml > 34u) {  // longer lengths: run-list lookup, pushed into the ring
                const uint32_t room = nb - j;
                const uint32_t kend = ml < room ? ml : room;
                const uint4* st4 = (const uint4*)&s.u.dp.runs[st][jl * kRunSlots];
                const uint4 ea = st4[0], eb = st4[1];
                for (uint32_t k = 35 + lane; k <= kend; k += 32) {
                  const uint32_t e = run_for_len(ea, eb, k, b.ovf);
                  const uint32_t tga = ring_r + ((j + k - 3) & 511) * 8;
                  const double pend = (double)__uint_as_float(lds_u32(tga));
                  if (pend <= mc) continue;  // squeeze.c:293
                  const int dsym = (int)run_dsym(e);
                  double nc2 = (double)(length_extra_bits((int)k) + dist_symbol_extra_bits(dsym)) + s.lencost[k] + s.dcost[dsym];
                  nc2 = nc2 + cj;
                  sts_ring8_if(tga, __float_as_uint(__double2float_rn(nc2)), kCodeLong | k, nc2 < pend);
                }
                if (j + kend > dirty_until) dirty_until = j + kend;
              }
            } else {
              cnext = e2c;  // a skipped source contributes no literal edge
              lfin_prev = e2l;
            }
            // target j+3 is complete for every length edge: hand it to the chain; its lane takes
            // on target j+35, whose ring entry (edges longer than 34) is complete as well
            const uint32_t src = (j + 3) & 31;
            sts_ring_if(xch_r + (j & 3) * 16, w, wl, lane == src);
            double inc = kInfD; uint32_t inl = 0;
            __syncwarp();
            if (j + 35 <= dirty_until) {
              const uint32_t ra = ring_r + ((j + 32) & 511) * 8;
              uint32_t fbj;
              lds_ring8(ra, fbj, inl);
              inc = (double)__uint_as_float(fbj);
              sts_u32_if(ra, kInfBits, lane == 0);  // free the slot for target j+35+512
              __syncwarp();
            }
            if (lane == src) { w = inc; wl = inl; }
            e2c = en_c; e2l = en_l;
            cj = cnext;
            tv = tv1; tv1 = tv2; ds2 = ds3; llb = llb1; llb1 = llb2;
          }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive_a(empty_r + st * 8);  // the feeder may write back lac[st] and refill the stage
        ZB_KIND_TICK(kind)
        (void)kind;
        g++;
      }
      if (lane == 0) s.dpn[5] += nslow;
#undef ZB_KIND_TICK
#undef ZB_DPI_GROUP
#undef ZB_DPI_4A
#undef ZB_DPI_4B
#undef ZB_DPI_STEP
#undef ZB_DP_FAST_GROUP
#undef ZB_DP_FAST_8
#undef ZB_DP_FAST_4A
#undef ZB_DP_FAST_4B
#undef ZB_DP_FAST_STEP
      if (lane == 0) la[nb] = (uint16_t)decode_code(lfin_prev, nb, s.u.dp.ring);
      seq_base += ngroups;
    }
    cta_sync64();  // (B) the feeder has written length_array[0 .. nb)

    ZB_TICK(1);
    // ------------------------------------------------------------------ trace back
    // TraceBackwards (squeeze.c:317-336) is a pointer chase i -> i - length_array[i].  Per window of
    // 4096 positions (in shared memory) it is run SPECULATIVELY from 32 starting points at once:
    // lane s chases from the top of its 128-position segment and numbers the nodes it visits.  The
    // true path enters a segment within 258 positions of its top; chains from nearby starts merge
    // after a few hops, so lane 0 then only stitches: follow the true path inside a segment until it
    // hits a numbered node (or leaves the segment), adopt the speculative chain from there on.  A
    // third pass re-walks the chains 32 wide and writes the adopted nodes.  Each symbol is emitted
    // as (start position << 9 | length); psym[cursor .. nb+1) holds the symbols in order.
    uint32_t cursor = nb + 1;
    if constexpr (NW > 2) {
      if (lane == 0) W.curbuf = (uint32_t)curbuf;
      cta_sync_all<NW>();  // (C) every warp joins for trace-back and follow-path
      cursor = wide_trace<NW>(W, la, psym, nb);
    } else {
      uint32_t idx = nb;  // current true path node
      const uint32_t la_a = smem_u32(&s.u.tr.la[0]), mk_a = smem_u32(&s.u.tr.mark[0]);
      const bool la_odd = (((uintptr_t)la) >> 1) & 1;  // make 4-byte loads aligned
      while (idx > 0) {
        // window covers la[wlo .. idx], wlo chosen so that &la[wlo] is 4-byte aligned
        uint32_t wlo = idx >= 4088u ? idx - 4087u : 0u;
        if (((wlo & 1u) != 0) != la_odd) wlo = wlo > 0 ? wlo - 1 : 0;  // align (or start at 0)
        const uint32_t cnt = idx - wlo + 1;
        if ((((uintptr_t)(la + wlo)) & 3) == 0) {
          const uint32_t* src = (const uint32_t*)(la + wlo);
          uint32_t* dst = (uint32_t*)&s.u.tr.la[0];
          const uint32_t nw = (cnt + 1) / 2;
          for (uint32_t tb = 0; tb < nw; tb += 32 * 16) {  // 16 loads in flight per lane
            uint32_t v[16];
#pragma unroll
            for (int u = 0; u < 16; u++) { const uint32_t t = tb + u * 32 + lane; v[u] = t < nw ? src[t] : 0u; }
#pragma unroll
            for (int u = 0; u < 16; u++) { const uint32_t t = tb + u * 32 + lane; if (t < nw) dst[t] = v[u]; }
          }
        } else {
          for (uint32_t t = lane; t < cnt; t += 32) s.u.tr.la[t] = la[wlo + t];
        }
        for (uint32_t t = lane; t < 2048; t += 32) ((uint32_t*)&s.u.tr.mark[0])[t] = 0;
        __syncwarp();
        // ---- pass 1: speculative chains.  Lane s takes segment s = positions (lo, hi], hi = idx - 128 s ----
        const TrSeg g = tr_seg(idx, wlo, lane);
        uint32_t exit_s = g.hi, cnt_s = 0;
        if (g.live) {
          uint32_t i = g.hi;
          while (i > g.floor_) {
            cnt_s++;
            asm volatile("st.shared.u16 [%0], %1;" ::"r"(mk_a + (i - wlo) * 2), "h"((unsigned short)cnt_s) : "memory");
            i -= tr_hop(la_a, wlo, i);
          }
          exit_s = i;
        }
        __syncwarp();
        // ---- pass 2: stitch (segment by segment; the few sequential hops run on every lane alike) ----
        uint32_t e = idx;         // true node entering the current segment
        uint32_t my_from = 0xffffffffu, my_base = 0;  // this lane's chain is adopted from node number my_from on
        for (uint32_t sg = 0; sg < 32; sg++) {
          const TrSeg gs = tr_seg(idx, wlo, sg);
          if (!gs.live || e == 0 || e < wlo) break;
          const uint32_t s_exit = __shfl_sync(0xffffffffu, exit_s, sg), s_cnt = __shfl_sync(0xffffffffu, cnt_s, sg);
          if (e <= gs.floor_) continue;  // the path jumps over this segment
          uint32_t i = e, from = 0;
          while (i > gs.floor_) {
            uint32_t mk;
            asm volatile("ld.shared.u16 %0, [%1];" : "=r"(mk) : "r"(mk_a + (i - wlo) * 2));
            if (mk) { from = mk; break; }
            const uint32_t l = tr_hop(la_a, wlo, i);
            i -= l;
            --cursor;
            if (lane == 0) psym[cursor] = ((uint64_t)i << 9) | l;
          }
          if (from) {  // merged: nodes from..s_cnt of lane sg's chain are on the path
            if (lane == sg) { my_from = from; my_base = cursor; }
            cursor -= s_cnt - from + 1;
            e = s_exit;
          } else {
            e = i;
          }
        }
        // ---- pass 3: emit the adopted part of every chain ----
        if (my_from != 0xffffffffu) {
          uint32_t i = g.hi, k = 0;
          while (i > g.floor_) {
            k++;
            const uint32_t l = tr_hop(la_a, wlo, i);
            i -= l;
            if (k >= my_from) psym[my_base - 1 - (k - my_from)] = ((uint64_t)i << 9) | l;
          }
        }
        idx = e;
        __syncwarp();
      }
    }
    const uint32_t nsym = nb + 1 - cursor;
    ZB_TICK(2);

    // ------------------------------------------------------------------ follow path + histogram
    if constexpr (NW > 2) {
      wide_follow<NW>(W, s.hist, b, sd, in, psym, cursor, nsym);
    } else {
      for (int i = lane; i < 320; i += 32) s.hist[i] = 0;
      __syncwarp();
      follow_path(b, sd, in, psym, cursor, 0, nsym, b.st_ll[curbuf] + sd.pos_off, b.st_d[curbuf] + sd.pos_off, s.hist, lane);
      __syncwarp();
    }
    ZB_TICK(3);
    if (fixed) { bestbuf = curbuf; best_size = nsym; bestcost = 0; it++; break; }
    if (lane == 0) s.hist[256] = 1;  // deflate.c:575 and squeeze.c:409
    __syncwarp();

    // ------------------------------------------------------------------ block size, best, statistics
    const uint64_t cost = warp_dynamic_bits(s.hist, s.u.cs, lane);  // squeeze.c:492
    if (b.iter_cost && lane == 0 && (uint32_t)it < b.iter_stride) b.iter_cost[(uint64_t)seg * b.iter_stride + it] = cost;
    ZB_TICK(4);
    if (cost < bestcost) {  // squeeze.c:496-501
      int t = curbuf; curbuf = bestbuf; bestbuf = t;
      best_size = nsym;
      for (int i = lane; i < 320; i += 32) s.bests[i] = s.stats[i];
      bestcost = cost;
    }
    for (int i = lane; i < 320; i += 32) { s.last[i] = s.stats[i]; s.stats[i] = s.hist[i]; }  // :502-504
    __syncwarp();
    bool need_entropy = true;
    if (lastrandomstep != -1) {  // :505-511; (size_t)(a*1.0 + b*0.5) == a + (b >> 1)
      for (int i = lane; i < 320; i += 32) s.stats[i] = s.stats[i] + (s.last[i] >> 1);
      __syncwarp();
      if (lane == 0) s.stats[256] = 1;
      __syncwarp();
    }
    if (it > 5 && cost == lastcost) {  // :512-517
      for (int i = lane; i < 320; i += 32) s.stats[i] = s.bests[i];
      __syncwarp();
      if (lane == 0) {  // RandomizeFreqs squeeze.c:96-101 (sequential, in place)
        for (int part = 0; part < 2; part++) {
          uint32_t* f = s.stats + (part ? 288 : 0);
          const uint32_t n = part ? kNumD : kNumLL;
          for (uint32_t i = 0; i < n; i++) {
            ran_z = 36969u * (ran_z & 65535u) + (ran_z >> 16);
            ran_w = 18000u * (ran_w & 65535u) + (ran_w >> 16);
            uint32_t r = (ran_z << 16) + ran_w;
            if ((r >> 4) % 3 == 0) {
              ran_z = 36969u * (ran_z & 65535u) + (ran_z >> 16);
              ran_w = 18000u * (ran_w & 65535u) + (ran_w >> 16);
              uint32_t r2 = (ran_z << 16) + ran_w;
              f[i] = f[r2 % n];
            }
          }
        }
        s.stats[256] = 1;
      }
      ran_z = __shfl_sync(0xffffffffu, ran_z, 0);
      ran_w = __shfl_sync(0xffffffffu, ran_w, 0);
      __syncwarp();
      lastrandomstep = it;
    }
    if (need_entropy) {
      bool ok = warp_entropy(s.stats, kNumLL, s.llcost, b, lane);
      ok &= warp_entropy(s.stats + 288, kNumD, s.dcost, b, lane);
      if (!ok) flags |= 1;
      __syncwarp();
    }
    lastcost = cost;
    ZB_TICK(5);
  }

  if (lane == 0) s.go = 0;
  __syncwarp();
  cta_sync64();  // (A) releases the feeder warp for good
  if constexpr (NW > 2) cta_sync_all<NW>();  // (C) with go == 0: releases the helper warps; the feeder joins after (A)
  if (lane == 0) {
    for (int i = 0; i < 6; i++) js->cyc[i] = (uint64_t)cyc[i];
    js->best_size = best_size;
    js->best_buf = (uint32_t)bestbuf;
    js->best_cost = bestcost;
    js->flags = flags;
    js->iters_done = (uint32_t)it;
    js->int_groups = igroups;
    for (int i = 0; i < 5; i++) js->dpc[i] = s.dpc[i];
    for (int i = 0; i < 6; i++) js->dpn[i] = s.dpn[i];
  }
}

// copies every segment's best parse into one packed buffer (offsets via atomic allocation)
__global__ void k_pack(Batch b, int greedy) {
  __shared__ uint32_t off;
  const uint32_t seg = blockIdx.x;
  const SegDesc sd = b.segs[seg];
  JobState* js = &b.jobs[seg];
  const uint32_t n = greedy ? js->greedy_size : js->best_size;
  const int buf = greedy ? 0 : (int)js->best_buf;
  if (threadIdx.x == 0) { off = atomicAdd(b.out_used, n); js->out_off = off; }
  __syncthreads();
  const uint16_t* sl = b.st_ll[buf] + sd.pos_off;
  const uint16_t* sdp = b.st_d[buf] + sd.pos_off;
  for (uint32_t t = threadIdx.x; t < n; t += blockDim.x) {
    b.out_ll[off + t] = sl[t];
    b.out_d[off + t] = sdp[t];
  }
}

}  // namespace zb

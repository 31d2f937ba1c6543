// Device-resident finish of a deflate call (SURVEY 8(f)#2): the LZ77 stores never leave the GPU.
//
//   k_keep         best parse of every block -> byte-indexed slot of a store buffer
//   k_sym_copy     block stores -> contiguous master-block stores      ZopfliAppendLZ77Store lz77.c:151-158
//   k_block_plan   per block: histogram, stored / fixed / dynamic sizes, the dynamic code lengths and
//                  tree flags that realise the size                    deflate.c:569-621, 251-290
//   k_emit         per block: header, tree, symbols, end code written at the block's FINAL bit
//                  position of the output stream; stored blocks likewise deflate.c:625-745, tree.c:30-69
//
// The host only sees three bit counts per block, decides (block types, second split: deflate.c:747-800,
// 872-893), runs a prefix sum over the chosen sizes and launches k_emit once per call.  Sizes are exact
// (ZopfliCalculateBlockSize is), so every block knows where it starts before a single bit is written;
// k_emit verifies each block against its predicted size.
#pragma once
#include "emit_bits.hpp"
#include "iterate.cuh"

namespace zb {

// ---- k_keep: segment i's best parse -> dst[instart_i + t] (a block never has more symbols than bytes) ----
__global__ void k_keep(Batch b, uint16_t* __restrict__ dst_ll, uint16_t* __restrict__ dst_d) {
  const uint32_t seg = blockIdx.x;
  const SegDesc sd = b.segs[seg];
  const JobState* js = &b.jobs[seg];
  const uint32_t n = js->best_size;
  const int buf = (int)js->best_buf;
  const uint16_t* sl = b.st_ll[buf] + sd.pos_off;
  const uint16_t* sdp = b.st_d[buf] + sd.pos_off;
  for (uint32_t t = threadIdx.x; t < n; t += blockDim.x) {
    dst_ll[sd.instart + t] = sl[t];
    dst_d[sd.instart + t] = sdp[t];
  }
}

struct SymCopyDev { uint64_t src_off, dst_off; uint32_t n, pad; };
__global__ void k_sym_copy(const SymCopyDev* __restrict__ req, const uint16_t* __restrict__ src_ll,
                           const uint16_t* __restrict__ src_d, uint16_t* __restrict__ dst_ll,
                           uint16_t* __restrict__ dst_d) {
  const SymCopyDev r = req[blockIdx.x];
  for (uint32_t t = threadIdx.x; t < r.n; t += blockDim.x) {
    dst_ll[r.dst_off + t] = src_ll[r.src_off + t];
    dst_d[r.dst_off + t] = src_d[r.src_off + t];
  }
}

// ---- k_block_plan ----
struct PlanReqDev { const uint16_t* ll; const uint16_t* d; BlockPlan* out; uint32_t n, pad; };

struct PlanSmem {
  uint32_t hist[320];
  CostStage cs;
  unsigned long long nbytes;
};

constexpr int kPlanThreads = 256;

__global__ void __launch_bounds__(kPlanThreads) k_block_plan(const PlanReqDev* __restrict__ reqs) {
  __shared__ PlanSmem s;
  const PlanReqDev r = reqs[blockIdx.x];
  const uint32_t tid = threadIdx.x, lane = tid & 31u;
  for (uint32_t i = tid; i < 320; i += kPlanThreads) s.hist[i] = 0;
  if (tid == 0) s.nbytes = 0;
  __syncthreads();
  // histogram (ZopfliLZ77GetHistogram lz77.c:189-217) and byte range
  unsigned long long nb = 0;
  for (uint32_t i = tid; i < r.n; i += kPlanThreads) {
    const uint32_t l = r.ll[i], dd = r.d[i];
    if (dd == 0) {
      atomicAdd(&s.hist[l], 1u);
      nb += 1;
    } else {
      atomicAdd(&s.hist[length_symbol((int)l)], 1u);
      atomicAdd(&s.hist[288 + dist_symbol((int)dd)], 1u);
      nb += l;
    }
  }
#pragma unroll
  for (int dlt = 16; dlt > 0; dlt >>= 1) nb += __shfl_xor_sync(0xffffffffu, nb, dlt);
  if (lane == 0 && nb) atomicAdd(&s.nbytes, nb);
  __syncthreads();
  if (tid >= 32) return;
  // fixed-tree size (deflate.c:599-601): 3 header bits + symbols + the 7-bit end code
  uint64_t f = 0;
  for (int i = lane; i < 320; i += 32) {
    const uint32_t c = s.hist[i];
    if (i < 288) {
      if (i < 256) f += (uint64_t)fixed_ll_length(i) * c;
      else if (i >= 257 && i < 286) f += (uint64_t)(fixed_ll_length(i) + length_symbol_extra_bits(i)) * c;
    } else if (i - 288 < 30) {
      f += (uint64_t)(5 + dist_symbol_extra_bits(i - 288)) * c;
    }
  }
#pragma unroll
  for (int dlt = 16; dlt > 0; dlt >>= 1) f += __shfl_xor_sync(0xffffffffu, f, dlt);
  if (lane == 0) s.hist[256] = 1;  // deflate.c:575
  __syncwarp();
  DynChoice ch;
  const uint64_t dyn = warp_dynamic_bits(s.hist, s.cs, lane, &ch);
  BlockPlan* o = r.out;
  for (int i = lane; i < kNumLL; i += 32) o->ll_len[i] = s.cs.len[ch.set][i];
  o->d_len[lane] = s.cs.len[ch.set][288 + lane];
  if (lane == 0) {
    o->tree_flags = ch.flags;
    o->tree_bits = ch.tree_bits;
    o->dyn_bits = dyn;
    o->fixed_bits = 3 + f + 7;
    o->unc_bits = stored_bits(s.nbytes);
    o->nbytes = s.nbytes;
  }
}

// ---- k_emit ----
struct EmitDesc {
  uint64_t bit_start;       // absolute bit position in the output buffer
  uint64_t nbits;           // predicted size (compressed blocks)
  const uint16_t* ll;       // symbols (compressed blocks)
  const uint16_t* d;
  const BlockPlan* plan;    // dynamic blocks
  uint64_t in_start;        // stored blocks: bytes [in_start, in_start + in_len) of the device input
  uint64_t in_len;
  uint32_t n;               // symbols
  uint32_t type_final;      // btype (0 stored, 1 fixed, 2 dynamic) | final << 8
};

struct WordSink {  // LSB-first bit writer for one thread: every word it touches may be shared
  uint32_t* words;
  uint64_t pos;
  __device__ void put(uint32_t v, int n) {
    if (n == 0) return;
    const uint64_t val = (uint64_t)v << (pos & 31);
    if ((uint32_t)val) atomicOr(&words[pos >> 5], (uint32_t)val);
    if ((uint32_t)(val >> 32)) atomicOr(&words[(pos >> 5) + 1], (uint32_t)(val >> 32));
    pos += (uint64_t)n;
  }
};

constexpr int kEmitThreads = 256;
constexpr int kEmitItems = 4;   // symbols per thread per round

// AddNonCompressedBlock deflate.c:625-663, the one writer of stored blocks on the device: bytes [ip, ip + len) of
// `in` as sub-blocks of at most 65,535 bytes from bit q of a zeroed stream, BFINAL on the last one when `final`.
// The header's byte may be shared with the block before (its bit is ORed in); every later byte belongs to this
// block alone and gets a plain store.  Called by all kThreads threads of the CTA.
template <int kThreads>
__device__ __forceinline__ void write_stored(uint32_t* __restrict__ out, uint64_t q, const uint8_t* __restrict__ in,
                                             uint64_t ip, uint64_t len, uint32_t final, uint32_t tid) {
  uint8_t* out8 = (uint8_t*)out;
  uint64_t left = len;
  do {
    const uint64_t bs = left > 65535 ? 65535 : left;
    const bool last = left == bs;
    const uint64_t lenpos = (q + 3 + 7) >> 3;  // LEN starts at the next byte boundary after the 3 header bits
    if (tid == 0) {
      if (final && last) atomicOr(&out[q >> 5], 1u << (q & 31));  // BFINAL; BTYPE 00 and the padding are zero bits
      const uint32_t nlen = (~(uint32_t)bs) & 0xffffu;
      out8[lenpos] = (uint8_t)(bs & 255);
      out8[lenpos + 1] = (uint8_t)(bs >> 8);
      out8[lenpos + 2] = (uint8_t)(nlen & 255);
      out8[lenpos + 3] = (uint8_t)(nlen >> 8);
    }
    for (uint64_t i = tid; i < bs; i += kThreads) out8[lenpos + 4 + i] = in[ip + i];
    q = (lenpos + 4 + bs) * 8;
    ip += bs;
    left -= bs;
  } while (left);
}

__global__ void __launch_bounds__(kEmitThreads) k_emit(const EmitDesc* __restrict__ pieces, const uint8_t* __restrict__ in,
                                                       uint32_t* __restrict__ out, uint32_t* __restrict__ err) {
  __shared__ uint8_t ll_len[kNumLL], d_len[kNumD];
  __shared__ uint16_t ll_code[kNumLL], d_code[kNumD];
  __shared__ unsigned long long sym_start_s;
  __shared__ uint32_t warp_tot[kEmitThreads / 32];
  const EmitDesc p = pieces[blockIdx.x];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
  const uint32_t type = p.type_final & 255u, final = p.type_final >> 8;

  if (type == 0) {
    write_stored<kEmitThreads>(out, p.bit_start, in, p.in_start, p.in_len, final, tid);
    return;
  }

  if (type == 2) {
    for (uint32_t i = tid; i < kNumLL; i += kEmitThreads) ll_len[i] = p.plan->ll_len[i];
    if (tid < kNumD) d_len[tid] = p.plan->d_len[tid];
  } else {  // GetFixedTree deflate.c:335-342
    for (uint32_t i = tid; i < kNumLL; i += kEmitThreads) ll_len[i] = (uint8_t)fixed_ll_length((int)i);
    if (tid < kNumD) d_len[tid] = 5;
  }
  __syncthreads();
  if (tid == 0) canonical_codes(ll_len, kNumLL, ll_code);
  if (tid == 32) canonical_codes(d_len, kNumD, d_code);
  if (tid == 64) {  // block header + tree (AddLZ77Block deflate.c:697-716, AddDynamicTree :251-272)
    WordSink sink{out, p.bit_start};
    sink.put(final | (type == 1 ? 2u : 4u), 3);
    if (type == 2) {
      const uint32_t tb = write_tree_header(ll_len, d_len, p.plan->tree_flags, sink);
      if (tb != p.plan->tree_bits) atomicExch(err, 0x40000000u | blockIdx.x);
    }
    sym_start_s = sink.pos;
  }
  __syncthreads();
  // AddLZ77Data deflate.c:297-333: bit length of every symbol -> exclusive scan -> shifted writes
  uint64_t run = sym_start_s;
  for (uint32_t base = 0; base < p.n; base += kEmitThreads * kEmitItems) {
    SymBits sb[kEmitItems];
    uint32_t tot = 0;
#pragma unroll
    for (int k = 0; k < kEmitItems; k++) {
      const uint32_t i = base + tid * kEmitItems + k;
      if (i < p.n) sb[k] = symbol_bits_of(p.ll[i], p.d[i], ll_len, ll_code, d_len, d_code);
      else { sb[k].v0 = sb[k].v1 = 0; sb[k].n0 = sb[k].n1 = 0; }
      tot += sb[k].n0 + sb[k].n1;
    }
    uint32_t incl = tot;
#pragma unroll
    for (int dlt = 1; dlt < 32; dlt <<= 1) {
      const uint32_t o = __shfl_up_sync(0xffffffffu, incl, dlt);
      if (lane >= (uint32_t)dlt) incl += o;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    uint32_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kEmitThreads / 32; w++) {
      const uint32_t t = warp_tot[w];
      if ((uint32_t)w < wid) before += t;
      all += t;
    }
    if (tot) {
      const uint64_t pos = run + before + (incl - tot);
      uint32_t* w = out + (pos >> 5);
      uint64_t acc = 0;
      int nacc = (int)(pos & 31);
      bool first = true;  // the first and the last word of this thread's bit range are shared with neighbours
#pragma unroll
      for (int k = 0; k < kEmitItems; k++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const uint32_t v = h ? sb[k].v1 : sb[k].v0;
          const int n = h ? sb[k].n1 : sb[k].n0;
          acc |= (uint64_t)v << nacc;
          nacc += n;
          if (nacc >= 32) {
            if (first) { atomicOr(w, (uint32_t)acc); first = false; }
            else *w = (uint32_t)acc;  // a word strictly inside the range belongs to this thread alone
            w++;
            acc >>= 32;
            nacc -= 32;
          }
        }
      }
      if (nacc > 0 && (uint32_t)acc) atomicOr(w, (uint32_t)acc);
    }
    run += all;
    __syncthreads();
  }
  if (tid == 0) {
    WordSink sink{out, run};
    sink.put(ll_code[256], ll_len[256]);  // end code (deflate.c:718-719)
    if (sink.pos - p.bit_start != p.nbits) atomicExch(err, 0x80000000u | blockIdx.x);
  }
}

// ---- k_splice: span records at absolute bit positions of a stream (a device compressor's pending bytes) ----
// The destination is zero from its first bit on, as k_emit's is.  A bit record is a tile of at most
// kSpliceTileBits bits that start at bit 0 of src (4-byte aligned, readable to the end of the tile's last word);
// the host cuts longer records into tiles.  A stored record is one sub-block of at most 65,535 bytes (the host
// cuts longer ones at the same boundaries write_stored does), written by write_stored.
struct SpliceDesc {
  uint64_t bit_start;       // absolute bit position in the destination
  uint64_t nbits;           // bit records: bits of the tile
  const uint8_t* src;       // bit records: the tile's bits; stored records: the payload
  uint64_t len;             // stored records: payload bytes
  uint32_t stored_final;    // 1 for a stored record | BFINAL << 8
  uint32_t pad;
};

constexpr int kSpliceThreads = 256;
constexpr uint64_t kSpliceTileBits = 32ull * kSpliceThreads * 8;  // 8 words per thread

__global__ void __launch_bounds__(kSpliceThreads) k_splice(const SpliceDesc* __restrict__ recs, uint32_t* __restrict__ out) {
  const SpliceDesc r = recs[blockIdx.x];
  const uint32_t tid = threadIdx.x;
  if (r.stored_final & 1u) {
    write_stored<kSpliceThreads>(out, r.bit_start, r.src, 0, r.len, r.stored_final >> 8, tid);
    return;
  }
  if (r.nbits == 0) return;
  const uint32_t* s = (const uint32_t*)r.src;
  const uint64_t nw = (r.nbits + 31) >> 5;  // source words
  const uint32_t tail = (uint32_t)(r.nbits & 31);
  const uint32_t sh = (uint32_t)(r.bit_start & 31);
  const uint64_t w0 = r.bit_start >> 5, w1 = (r.bit_start + r.nbits - 1) >> 5;
  auto word = [&](uint64_t k) -> uint32_t {  // source word k, zero past the record's last bit
    if (k >= nw) return 0u;
    const uint32_t v = s[k];
    return (k + 1 == nw && tail) ? (v & ((1u << tail) - 1u)) : v;
  };
  // destination word w0 + k holds source bits [32k - sh, 32k - sh + 32)
  for (uint64_t k = tid; w0 + k <= w1; k += kSpliceThreads) {
    uint32_t v = word(k) << sh;
    if (sh && k) v |= word(k - 1) >> (32 - sh);
    if (k == 0 || w0 + k == w1) {  // the first and the last word may be shared with neighbours
      if (v) atomicOr(out + w0 + k, v);
    } else {
      out[w0 + k] = v;  // a word strictly inside the record belongs to it alone
    }
  }
}

}  // namespace zb

// Multi-GPU ZopfliDeflate inside the library (SURVEY 8(e)): one input, one RFC1951 stream, the master
// blocks (the reference's independent unit, /root/reference/src/zopfli/deflate.c:908-931) sharded over
// the GPUs of one box.  NCCL carries exactly two things over NVLink:
//   scatter  rank 0 stages the input on its GPU and ncclSends every other rank its shard plus the
//            32 KiB dictionary in front of it (squeeze.c:229-230)
//   gather   after a ncclAllGather of the per-rank stream lengths every rank knows its absolute bit
//            offset, emits its blocks at that bit phase (finish.cuh) and ncclSends the bytes straight to
//            their final place in rank 0's output buffer -- a distributed splice: no span is ever shifted
//            or copied on the host; the one byte two ranks can share travels separately and is ORed in.
// Two ways in: one process per GPU (ZopfliB200DistInit + ZopfliB200DistCompress, e.g. under torchrun),
// or one process driving several GPUs (ZopfliCompress with ZOPFLI_B200_GPUS=N: ncclCommInitAll, one
// host thread per GPU).  Both run the same rank body below.
//
// NCCL is loaded with dlopen at first use, so single-GPU users do not need it installed.
#include "dist.hpp"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <thread>
#include <utility>
#include <vector>

#include "../../include/zopfli_b200.h"
#include "dist_layout.hpp"
#include "driver.hpp"
#include "engine.hpp"
#include "symbols.hpp"

namespace zb {
namespace {

#define DCK(call)                                                                                           \
  do {                                                                                                      \
    cudaError_t e_ = (call);                                                                                \
    if (e_ != cudaSuccess) {                                                                                \
      fprintf(stderr, "zopfli-b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      abort();                                                                                              \
    }                                                                                                       \
  } while (0)

struct NcclApi {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool load() {
    if (h) return true;
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (h) break;
    }
    if (!h) { fprintf(stderr, "zopfli-b200: multi-GPU mode needs NCCL (libnccl.so.2): %s\n", dlerror()); return false; }
#define ZB_SYM(field, sym) *(void**)(&field) = dlsym(h, sym); if (!field) { fprintf(stderr, "zopfli-b200: %s missing in libnccl\n", sym); return false; }
    ZB_SYM(GetUniqueId, "ncclGetUniqueId") ZB_SYM(CommInitRank, "ncclCommInitRank") ZB_SYM(CommInitAll, "ncclCommInitAll")
    ZB_SYM(CommDestroy, "ncclCommDestroy") ZB_SYM(Send, "ncclSend") ZB_SYM(Recv, "ncclRecv") ZB_SYM(AllGather, "ncclAllGather")
    ZB_SYM(GroupStart, "ncclGroupStart") ZB_SYM(GroupEnd, "ncclGroupEnd") ZB_SYM(GetErrorString, "ncclGetErrorString")
#undef ZB_SYM
    return true;
  }
};
NcclApi g_nccl;
std::mutex g_dist_mu;

#define NCK(call)                                                                                              \
  do {                                                                                                         \
    ncclResult_t r_ = (call);                                                                                  \
    if (r_ != ncclSuccess) {                                                                                   \
      fprintf(stderr, "zopfli-b200: NCCL error %s at %s:%d\n", g_nccl.GetErrorString(r_), __FILE__, __LINE__); \
      abort();                                                                                                 \
    }                                                                                                          \
  } while (0)

struct Scratch {  // grow-only device / pinned scratch of one rank
  void* p = nullptr;
  size_t cap = 0;
  void* ensure(size_t n) {
    if (n > cap) {
      if (p) DCK(cudaFree(p));
      cap = n + n / 8 + 256;
      DCK(cudaMalloc(&p, cap));
    }
    return p;
  }
};

struct Rank {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1, dev = 0;
  Scratch input;     // rank 0: the whole input; others: shard + dictionary
  size_t staged_insize = (size_t)-1;  // input size of the last scatter (ZOPFLI_B200_DIST_STAGED reuses it)
  Scratch meta;      // allgather buffers + first-byte slots
  uint64_t* host_meta = nullptr;  // pinned
};

constexpr int kMetaPerRank = 9;  // stream length for each of the 8 start phases + (rank 0) the caller's bit phase


// One rank of a distributed ZopfliDeflate(btype 2).  `in`, `bp`, `out`, `outsize` are used on rank 0 only.
void rank_deflate(Rank& rk, const ZopfliOptions* opt, int final, const unsigned char* in, size_t insize, unsigned char* bp,
                  unsigned char** out, size_t* outsize, std::vector<uint64_t>* unit_bits, bool staged = false) {
  const int r = rk.rank, W = rk.world;
  DCK(cudaSetDevice(rk.dev));
  Engine::Lease eng(rk.dev);
  cudaStream_t st = (cudaStream_t)eng->stream();
  const size_t nm = dist_num_master_blocks(insize);
  auto shard = [&](int q, size_t& a, size_t& b, size_t& base) { dist_shard(insize, W, q, &a, &b, &base); };
  size_t a, b, base;
  shard(r, a, b, base);
  const size_t lo = (size_t)r * nm / W, hi = (size_t)(r + 1) * nm / W;

  // ---- scatter ----
  const uint8_t* d_in = nullptr;
  size_t d_len = 0;
  if (staged && rk.staged_insize == insize) {  // the shards of this very input are still on the devices
    d_in = (const uint8_t*)rk.input.p;
    d_len = r == 0 ? b : b - base;
    if (r == 0) base = 0;
  } else if (r == 0) {
    uint8_t* d = (uint8_t*)rk.input.ensure(insize + 64);
    DCK(cudaMemsetAsync(d + insize, 0, 64, st));
    eng->upload(d, in, insize);  // threaded pinned staging; synchronous
    NCK(g_nccl.GroupStart());
    for (int q = 1; q < W; q++) {
      size_t qa, qb, qbase;
      shard(q, qa, qb, qbase);
      if (qb > qbase) NCK(g_nccl.Send(d + qbase, qb - qbase, ncclUint8, q, rk.comm, st));
    }
    NCK(g_nccl.GroupEnd());
    d_in = d;
    d_len = b;  // rank 0 parses a prefix of the staged input in place
    base = 0;
  } else {
    d_len = b - base;
    uint8_t* d = (uint8_t*)rk.input.ensure(d_len + 64);
    DCK(cudaMemsetAsync(d + d_len, 0, 64, st));
    if (d_len) {
      NCK(g_nccl.GroupStart());
      NCK(g_nccl.Recv(d, d_len, ncclUint8, 0, rk.comm, st));
      NCK(g_nccl.GroupEnd());
    }
    d_in = d;
  }
  rk.staged_insize = insize;
  eng->set_input_device(d_in, d_len);  // same stream: ordered behind the copy / receive

  // ---- this rank's master blocks ----
  std::vector<Piece> pieces;
  if (lo < hi) deflate_units(*eng, opt, 2, final != 0 && hi == nm, master_blocks(a, b), base, pieces);

  // ---- every rank learns every rank's stream length (for each of the 8 possible start phases: the
  // padding of stored blocks depends on it, deflate.c:643-649) ----
  uint64_t* hm = rk.host_meta;
  std::vector<Engine::EmitPiece> ep;
  for (int p = 0; p < 8; p++) hm[p] = pieces.empty() ? 0 : layout_pieces(pieces, base, (uint64_t)p, ep, nullptr) - (uint64_t)p;
  hm[8] = (r == 0 && *outsize > 0) ? (uint64_t)(*bp & 7) : 0;
  uint64_t* d_meta = (uint64_t*)rk.meta.ensure((size_t)(kMetaPerRank * (W + 1)) * 8 + 64 + (size_t)W * 8);
  uint64_t* d_all = d_meta + kMetaPerRank;
  uint8_t* d_first = (uint8_t*)(d_all + (size_t)kMetaPerRank * W);  // rank 0: first byte of every rank's stream
  DCK(cudaMemcpyAsync(d_meta, hm, kMetaPerRank * 8, cudaMemcpyHostToDevice, st));
  NCK(g_nccl.AllGather(d_meta, d_all, kMetaPerRank, ncclUint64, rk.comm, st));
  uint64_t* hall = hm + kMetaPerRank;
  DCK(cudaMemcpyAsync(hall, d_all, (size_t)kMetaPerRank * W * 8, cudaMemcpyDeviceToHost, st));
  DCK(cudaStreamSynchronize(st));
  std::vector<uint64_t> start(W + 1);
  dist_placement(hall, kMetaPerRank, W, (unsigned)hall[8], start.data());
  const uint64_t total_bits = start[W];
  const size_t total_bytes = (size_t)((total_bits + 7) / 8);

  // ---- emit at the final bit phase; move the bytes to rank 0 ----
  const uint64_t bit0 = start[r] & 7;
  const uint64_t local_end = pieces.empty() ? bit0 : layout_pieces(pieces, base, bit0, ep, unit_bits);
  const size_t local_bytes = pieces.empty() ? 0 : (size_t)((local_end + 7) / 8);
  if (pieces.empty()) ep.clear();
  uint8_t* d_out = (uint8_t*)eng->emit_device(ep, pieces.empty() ? 0 : local_end, r == 0 ? total_bytes + 64 : 0);
  auto bytes_of = [&](int q) -> size_t { return dist_bytes_touched(start.data(), q); };
  if (r == 0) {
    DCK(cudaMemsetAsync(d_first, 0, (size_t)W, st));
    if (total_bytes > local_bytes) DCK(cudaMemsetAsync(d_out + local_bytes, 0, total_bytes - local_bytes, st));
    NCK(g_nccl.GroupStart());
    for (int q = 1; q < W; q++) {
      const size_t nb = bytes_of(q);
      if (nb == 0) continue;
      NCK(g_nccl.Recv(d_first + q, 1, ncclUint8, q, rk.comm, st));
      if (nb > 1) NCK(g_nccl.Recv(d_out + (size_t)(start[q] >> 3) + 1, nb - 1, ncclUint8, q, rk.comm, st));
    }
    NCK(g_nccl.GroupEnd());
    uint8_t* hfirst = (uint8_t*)(hall + (size_t)kMetaPerRank * W);
    DCK(cudaMemcpyAsync(hfirst, d_first, (size_t)W, cudaMemcpyDeviceToHost, st));
    DCK(cudaStreamSynchronize(st));
    // append to the caller's buffer; the byte at every rank boundary is shared by two ranks
    if (total_bytes)
      append_stream(total_bytes, (unsigned)(start[0] & 7), out, outsize, [&](unsigned char* dst) {
        eng->download(d_out, dst, total_bytes);
        for (int q = 1; q < W; q++)
          if (bytes_of(q)) dst[start[q] >> 3] |= hfirst[q];
      });
    *bp = (unsigned char)(total_bits & 7);
  } else if (local_bytes) {
    NCK(g_nccl.GroupStart());
    NCK(g_nccl.Send(d_out, 1, ncclUint8, 0, rk.comm, st));
    if (local_bytes > 1) NCK(g_nccl.Send(d_out + 1, local_bytes - 1, ncclUint8, 0, rk.comm, st));
    NCK(g_nccl.GroupEnd());
    DCK(cudaStreamSynchronize(st));
  }
}

void rank_init_buffers(Rank& rk) {
  DCK(cudaSetDevice(rk.dev));
  if (!rk.host_meta) DCK(cudaMallocHost((void**)&rk.host_meta, (size_t)(kMetaPerRank * (rk.world + 1)) * 8 + 64 + (size_t)rk.world * 8));
}

// ---- process-per-GPU mode ----
Rank g_self;
bool g_self_ready = false;

// ---- one process, several GPUs ----
std::vector<Rank> g_local;
int g_local_n = 0;

bool local_init(int n) {
  std::lock_guard<std::mutex> g(g_dist_mu);
  if (g_local_n == n) return true;
  if (g_local_n != 0) return false;  // one topology per process
  if (!g_nccl.load()) return false;
  if (Engine::device_count() < n) { fprintf(stderr, "zopfli-b200: ZOPFLI_B200_GPUS=%d but only %d devices are visible\n", n, Engine::device_count()); return false; }
  std::vector<int> devs(n);
  for (int i = 0; i < n; i++) devs[i] = i;
  std::vector<ncclComm_t> comms(n);
  NCK(g_nccl.CommInitAll(comms.data(), n, devs.data()));
  g_local.resize(n);
  for (int i = 0; i < n; i++) {
    g_local[i].comm = comms[i];
    g_local[i].rank = i;
    g_local[i].world = n;
    g_local[i].dev = devs[i];
    rank_init_buffers(g_local[i]);
  }
  g_local_n = n;
  return true;
}

}  // namespace

int dist_local_gpus() {
  static int n = [] {
    const char* e = getenv("ZOPFLI_B200_GPUS");
    int v = e ? atoi(e) : 1;
    return v < 1 ? 1 : v;
  }();
  return n;
}

bool dist_local_deflate(int ngpus, const ZopfliOptions* opt, int final, const unsigned char* in, size_t insize, unsigned char* bp,
                        unsigned char** out, size_t* outsize) {
  if (!local_init(ngpus)) return false;
  std::lock_guard<std::mutex> g(g_dist_mu);  // one collective at a time on the process's communicators
  std::vector<std::thread> th;
  for (int i = 1; i < ngpus; i++)
    th.emplace_back([&, i] { rank_deflate(g_local[i], opt, final, nullptr, insize, nullptr, nullptr, nullptr, nullptr); });
  rank_deflate(g_local[0], opt, final, in, insize, bp, out, outsize, nullptr);
  for (auto& t : th) t.join();
  return true;
}

bool dist_rank_ready() { return g_self_ready; }
int dist_rank() { return g_self.rank; }

void dist_rank_deflate(const ZopfliOptions* opt, int final, const unsigned char* in, size_t insize, unsigned char* bp,
                       unsigned char** out, size_t* outsize, bool staged) {
  std::lock_guard<std::mutex> g(g_dist_mu);
  rank_deflate(g_self, opt, final, in, insize, bp, out, outsize, nullptr, staged);
}

}  // namespace zb

using namespace zb;

extern "C" {

int ZopfliB200DistUniqueId(unsigned char* id128) {
  if (!g_nccl.load()) return 1;
  static_assert(sizeof(ncclUniqueId) == ZOPFLI_B200_UNIQUE_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  if (g_nccl.GetUniqueId(&id) != ncclSuccess) return 1;
  memcpy(id128, &id, sizeof(id));
  return 0;
}

int ZopfliB200DistInit(int rank, int world, const unsigned char* id128) {
  std::lock_guard<std::mutex> g(g_dist_mu);
  if (g_self_ready) return (g_self.rank == rank && g_self.world == world) ? 0 : 1;
  if (world < 1 || rank < 0 || rank >= world || !g_nccl.load()) return 1;
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  g_self.rank = rank;
  g_self.world = world;
  g_self.dev = Engine::default_device();
  DCK(cudaSetDevice(g_self.dev));
  NCK(g_nccl.CommInitRank(&g_self.comm, world, id, rank));
  rank_init_buffers(g_self);
  g_self_ready = true;
  return 0;
}

void ZopfliB200DistFinalize(void) {
  std::lock_guard<std::mutex> g(g_dist_mu);
  if (g_self_ready) { g_nccl.CommDestroy(g_self.comm); g_self_ready = false; }
}

}  // extern "C"

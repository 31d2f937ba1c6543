// CUDA engine: device memory, launch sequencing and result transfer for the zopfli hot path.
// Built for sm_90a only.  There is NO CPU fallback: any CUDA failure aborts with a message
// (the reference's own error model is exit(), squeeze.c:469-470).
#include "engine.hpp"

#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <condition_variable>
#include <mutex>
#include <thread>

#include "checksum.cuh"
#include "iterate.cuh"
#include "kernels.cuh"
#include "split.cuh"
#include "finish.cuh"

namespace zb {

#define CK(call)                                                                              \
  do {                                                                                        \
    cudaError_t e_ = (call);                                                                  \
    if (e_ != cudaSuccess) {                                                                  \
      fprintf(stderr, "zopfli-b200: CUDA error %s at %s:%d: %s\n", cudaGetErrorName(e_),      \
              __FILE__, __LINE__, cudaGetErrorString(e_));                                    \
      abort();                                                                                \
    }                                                                                         \
  } while (0)

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaStream_t st = nullptr;  // owning lane's stream: allocations are stream-ordered (cudaMallocAsync),
                              // so growing one lane's arena never synchronises the whole device
  void ensure(size_t bytes) {
    if (bytes <= cap) return;
    if (p) CK(cudaFreeAsync(p, st));
    size_t want = bytes + bytes / 8 + 256;
    CK(cudaMallocAsync(&p, want, st));
    cap = want;
  }
  template <typename T>
  T* as() { return (T*)p; }
};

__global__ void k_test_block_bits(Batch b, const uint32_t* hist, uint64_t* out) {
  __shared__ IterSmem s;
  const uint32_t lane = threadIdx.x;
  for (int i = lane; i < 320; i += 32) s.hist[i] = hist[i];
  __syncwarp();
  if (lane == 0) s.hist[256] = 1;
  __syncwarp();
  uint64_t r = warp_dynamic_bits(s.hist, s.u.cs, lane);
  if (lane == 0) *out = r;
}

// the pieces of warp_dynamic_bits for one histogram per CTA (ZopfliB200DeviceProbeParts)
__global__ void k_test_probe_parts(const uint32_t* hists, uint32_t* smoothed, uint8_t* lengths, uint32_t* tree_bits,
                                   uint64_t* dyn) {
  __shared__ SplitSmem s;
  const uint32_t lane = threadIdx.x, h = blockIdx.x;
  CostStage& cs = s.cs;
  for (int i = lane; i < 320; i += 32) s.hist[i] = hists[h * 320 + i];
  __syncwarp();
  if (lane == 0) s.hist[256] = 1;
  __syncwarp();
  for (int i = lane; i < 320; i += 32) cs.cnt2[i] = s.hist[i];
  __syncwarp();
  warp_optimize_for_rle(cs.cnt2, kNumLL, cs.pm, lane);
  warp_optimize_for_rle(cs.cnt2 + 288, kNumD, cs.pm, lane);
  warp_length_limited(s.hist, kNumLL, cs.len[0], cs.pm, lane);
  warp_length_limited(s.hist + 288, kNumD, cs.len[0] + 288, cs.pm, lane);
  warp_length_limited(cs.cnt2, kNumLL, cs.len[1], cs.pm, lane);
  warp_length_limited(cs.cnt2 + 288, kNumD, cs.len[1] + 288, cs.pm, lane);
  if (lane < 2) patch_distance_codes(cs.len[lane] + 288);
  __syncwarp();
  for (int i = lane; i < 320; i += 32) {
    smoothed[h * 320 + i] = cs.cnt2[i];
    lengths[h * 640 + i] = cs.len[0][i];
    lengths[h * 640 + 320 + i] = cs.len[1][i];
  }
  __syncwarp();
  const uint32_t t = warp_tree_sizes(cs, lane);   // overwrites cs.cnt2
  if (lane < 16) tree_bits[h * 16 + lane] = t;
  __syncwarp();
  const uint64_t r = warp_dynamic_bits(s.hist, cs, lane);
  if (lane == 0) dyn[h] = r;
}

struct Timer {
  cudaEvent_t a, b;
  Timer() { CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b)); }
};

constexpr uint32_t kLogTabN = 1u << 21;

// L[n] = log(n) * kInvLog2 with the HOST libm, exactly the two operations of tree.c:79,85.  Filled once
// per process by a background thread, uploaded once per device; read-only afterwards, shared by all
// engine contexts.
struct LogService {
  std::mutex mu;
  std::thread filler;
  std::vector<double> host;
  bool started = false, joined = false;
  double* dev[64] = {nullptr};
  uint32_t dev_n[64] = {0};
  static void fill(std::vector<double>& t, uint32_t from, uint32_t to) {
    static const double kInvLog2 = 1.4426950408889;
    for (uint32_t i = from; i < to; i++) {
      volatile double l = i ? log((double)i) : 0.0;
      t[i] = i ? l * kInvLog2 : 0.0;
    }
  }
  void start() {
    std::lock_guard<std::mutex> g(mu);
    if (started) return;
    started = true;
    filler = std::thread([this]() {
      host.resize(kLogTabN);
      fill(host, 0, kLogTabN);
    });
  }
  // A process whose engines never parse (emission, checksums, block sizes only) never joins the filler in
  // get(); a joinable std::thread destroyed at exit would call std::terminate.
  ~LogService() {
    if (filler.joinable()) filler.join();
  }
  // table with at least need_n entries on `device`.  No fixed size covers every statistics sum: the blend
  // (squeeze.c:505-511) adds half the previous statistics, and RandomizeFreqs copies counts between entries, so
  // the sum the entropy takes can exceed twice the block's symbols (2.2x has been seen on random data).  The
  // default 2^21 entries and parse_common's 2 x positions pre-size cover the usual case; a batch that still
  // meets a sum past the table grows it here and is redone.  An outgrown device copy is left allocated: other
  // contexts may still be reading it.
  const double* get(int device, cudaStream_t st, uint32_t need_n, uint32_t* have_n) {
    std::lock_guard<std::mutex> g(mu);
    if (!joined) { filler.join(); joined = true; }
    if (need_n < kLogTabN) need_n = kLogTabN;
    if (host.size() < need_n) {
      const uint32_t old = (uint32_t)host.size();
      host.resize(need_n);
      fill(host, old, need_n);
    }
    double*& d = dev[device & 63];
    if (!d || dev_n[device & 63] < need_n) {
      CK(cudaMalloc(&d, (size_t)need_n * sizeof(double)));
      CK(cudaMemcpyAsync(d, host.data(), (size_t)need_n * sizeof(double), cudaMemcpyHostToDevice, st));
      CK(cudaStreamSynchronize(st));
      dev_n[device & 63] = need_n;
    }
    *have_n = dev_n[device & 63];
    return d;
  }
};
LogService g_log;

}  // namespace

struct PinBuf {  // grow-only page-locked host staging: round trips through it skip the driver's own staging copy
  void* p = nullptr;
  size_t cap = 0;
  void* ensure(size_t bytes) {
    if (bytes > cap) {
      if (p) CK(cudaFreeHost(p));
      cap = bytes + bytes / 4 + 4096;
      CK(cudaMallocHost(&p, cap));
    }
    return p;
  }
};

// Pageable host memory <-> device through page-locked staging, several host threads deep: a pageable
// cudaMemcpy is one thread's memcpy into the driver's staging buffer (~10 GB/s); here kThreads threads
// each shuttle 4 MB chunks through their own pinned double buffer and stream, so the copy runs at
// whatever the link sustains.  Buffers that are already page-locked go straight to the DMA engine.
struct Stager {
  static constexpr int kThreads = 12;
  static constexpr size_t kChunk = 4u << 20;
  int dev = 0;
  bool ready = false;
  std::mutex mu;
  cudaStream_t st[kThreads];
  cudaEvent_t ev[kThreads][2];
  uint8_t* pin[kThreads][2];
  void init(int device) {
    if (ready) return;
    dev = device;
    for (int t = 0; t < kThreads; t++) {
      CK(cudaStreamCreateWithFlags(&st[t], cudaStreamNonBlocking));
      for (int k = 0; k < 2; k++) {
        CK(cudaEventCreateWithFlags(&ev[t][k], cudaEventDisableTiming));
        CK(cudaMallocHost((void**)&pin[t][k], kChunk));
      }
    }
    ready = true;
  }
  static bool page_locked(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
  }
  // synchronous: returns when all n bytes have arrived
  void copy(uint8_t* dst, const uint8_t* src, size_t n, bool to_device, int device) {
    if (n == 0) return;
    std::lock_guard<std::mutex> g(mu);
    CK(cudaSetDevice(device));
    init(device);
    if (n < 2 * kChunk || page_locked(to_device ? (const void*)src : (const void*)dst)) {
      CK(cudaMemcpyAsync(dst, src, n, to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost, st[0]));
      CK(cudaStreamSynchronize(st[0]));
      return;
    }
    const size_t nchunks = (n + kChunk - 1) / kChunk;
    const int nt = (int)std::min<size_t>(kThreads, nchunks);
    auto work = [&](int t) {
      CK(cudaSetDevice(device));
      int slot = 0;
      size_t pend_off[2] = {0, 0}, pend_len[2] = {0, 0};  // device->host: chunks whose DMA is in flight
      for (size_t c = (size_t)t; c < nchunks; c += (size_t)nt, slot ^= 1) {
        const size_t off = c * kChunk, len = std::min(kChunk, n - off);
        CK(cudaEventSynchronize(ev[t][slot]));  // the slot's previous transfer is done
        if (to_device) {
          memcpy(pin[t][slot], src + off, len);
          CK(cudaMemcpyAsync(dst + off, pin[t][slot], len, cudaMemcpyHostToDevice, st[t]));
        } else {
          if (pend_len[slot]) memcpy(dst + pend_off[slot], pin[t][slot], pend_len[slot]);
          CK(cudaMemcpyAsync(pin[t][slot], src + off, len, cudaMemcpyDeviceToHost, st[t]));
          pend_off[slot] = off;
          pend_len[slot] = len;
        }
        CK(cudaEventRecord(ev[t][slot], st[t]));
      }
      CK(cudaStreamSynchronize(st[t]));
      if (!to_device)
        for (int k = 0; k < 2; k++)
          if (pend_len[k]) memcpy(dst + pend_off[k], pin[t][k], pend_len[k]);
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nt; t++) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
  }
};

struct Lane {  // an independent stream + arena set; chunk pipelines use a pair each (giant blocks beside the rest)
  std::mutex mu;
  cudaStream_t stream = nullptr;
  // kernel timing without host synchronisation: event pairs are recorded into a small pool and read
  // back at the next point where the lane's stream is synchronised anyway (flush_timers)
  static constexpr int kTimerPairs = 48;
  cudaEvent_t ev[kTimerPairs][2];
  double* ev_acc[kTimerPairs];
  int ev_used = 0;
  DevBuf segs, keywork, poswork, order, hv, hv2, idx1, idx2, rank1, rank2, bkt1, bkt2, ld, mlen, runs, dsx,
      ovf, la, path, st[4], jobs, out_ll, out_d, counters, misc, iterc;
  // split service
  DevBuf sp_ll, sp_d, sp_llsym, sp_dsym, sp_pos, sp_snaps, sp_stores, sp_work, sp_evals, sp_out;
  PinBuf pin_req, pin_out;
  std::vector<SplitStoreDesc> sp_desc;
  SplitBatch sp_batch;
  uint32_t ovf_cap = 1u << 22;
  EngineStats acc;

  void init(bool high_priority) {
    memset(&acc, 0, sizeof(acc));
    // even lanes carry the longest DP chains (driver.cpp stage C): their few CTAs must not queue
    // behind the thousands of CTAs of another lane's match kernels
    int lo = 0, hi = 0;
    CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    CK(cudaStreamCreateWithPriority(&stream, cudaStreamNonBlocking, high_priority ? hi : lo));
    for (int k = 0; k < kTimerPairs; k++) { CK(cudaEventCreate(&ev[k][0])); CK(cudaEventCreate(&ev[k][1])); }
    DevBuf* all[] = {&segs, &keywork, &poswork, &order, &hv, &hv2, &idx1, &idx2, &rank1, &rank2, &bkt1, &bkt2, &ld,
                     &mlen, &runs, &dsx, &ovf, &la, &path, &st[0], &st[1], &st[2], &st[3], &jobs, &out_ll,
                     &out_d, &counters, &misc, &iterc, &sp_ll, &sp_d, &sp_llsym, &sp_dsym, &sp_pos, &sp_snaps, &sp_stores,
                     &sp_work, &sp_evals, &sp_out};
    for (DevBuf* d : all) d->st = stream;
  }
  void tic() {
    if (ev_used == kTimerPairs) { CK(cudaStreamSynchronize(stream)); flush_timers(); }
    CK(cudaEventRecord(ev[ev_used][0], stream));
  }
  void toc(double& a) {
    CK(cudaEventRecord(ev[ev_used][1], stream));
    ev_acc[ev_used++] = &a;
    // A host synchronisation behind every timed kernel keeps each lane's queue one kernel deep.  Measured
    // on the 100 MB bench (tools/gpu_timeline.sh): 999 ms per call with it, 1757 ms without -- with whole
    // kernel chains queued per lane the chunk pipelines run one after the other instead of side by side.
    // ZOPFLI_B200_SYNC_TOC=0 switches to deferred timing (events read at the next natural sync point).
    static const bool eager = [] { const char* e = getenv("ZOPFLI_B200_SYNC_TOC"); return !e || atoi(e); }();
    if (eager) sync();
  }
  void flush_timers() {  // the stream must be idle (caller has synchronised it)
    for (int k = 0; k < ev_used; k++) {
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, ev[k][0], ev[k][1]));
      *ev_acc[k] += ms;
    }
    ev_used = 0;
  }
  void sync() {
    CK(cudaStreamSynchronize(stream));
    flush_timers();
  }
  template <typename T>
  void upload(DevBuf& d, const std::vector<T>& v) {
    d.ensure(v.size() * sizeof(T) + 16);
    if (!v.empty()) CK(cudaMemcpyAsync(d.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, stream));
  }
};

struct Engine::Impl {
  std::mutex mu;  // input / log table / statistics
  int dev = 0;
  Lane lane[Engine::kLanes];
  // input (shared, read-only while parses run)
  DevBuf in_buf, same_buf, tile_first, next_tile;
  const double* logtab = nullptr;  // shared per-device table (LogService)
  uint32_t logtab_n = 0;
  const uint8_t* d_in = nullptr;
  uint64_t insize = 0;
  EngineStats st_acc;  // input-side counters; lane counters are merged in stats()
  // device-resident finish: symbol buffers (Engine::StoreBuf), plan slabs, output stream
  std::mutex fin_mu;
  DevBuf sym_ll[3], sym_d[3];
  struct Slab { BlockPlan* p; size_t cap; };
  std::vector<Slab> slabs;
  size_t slab_idx = 0, slab_used = 0;
  DevBuf outbuf, emit_desc, err_flag;
  Stager stager;
  // device-resident calls: the caller's stream is ordered against lane 0 through events; the checksum of
  // the input runs on a low-priority stream of its own, beside the parse
  cudaStream_t ck_stream = nullptr;
  cudaEvent_t ev_user, ev_lane0, ev_ck;
  DevBuf ck_acc;
  int sm_count = 0;

  void begin_call() {  // a new input: plans of the previous call are dead
    std::lock_guard<std::mutex> g(fin_mu);
    slab_idx = 0;
    slab_used = 0;
  }
  // symbol buffer `buf`, sized like the input; allocated on lane 0's stream, which is drained before any
  // other lane may touch the memory
  void ensure_sym(int buf) {
    std::lock_guard<std::mutex> g(fin_mu);
    const size_t need = (insize + 64) * 2;
    if (sym_ll[buf].cap >= need && sym_d[buf].cap >= need) return;
    sym_ll[buf].ensure(need);
    sym_d[buf].ensure(need);
    CK(cudaStreamSynchronize(lane[0].stream));
  }
  BlockPlan* plan_alloc(size_t n) {  // n contiguous plans; slabs are kept for the context's lifetime
    std::lock_guard<std::mutex> g(fin_mu);
    for (;;) {
      if (slab_idx < slabs.size() && slabs[slab_idx].cap - slab_used >= n) {
        BlockPlan* r = slabs[slab_idx].p + slab_used;
        slab_used += n;
        return r;
      }
      if (slab_idx < slabs.size()) { slab_idx++; slab_used = 0; continue; }
      Slab sl;
      sl.cap = std::max<size_t>(n, 8192);
      CK(cudaMalloc((void**)&sl.p, sl.cap * sizeof(BlockPlan)));
      slabs.push_back(sl);
      slab_used = 0;
    }
  }

  explicit Impl(int want_dev) {
    memset(&st_acc, 0, sizeof(st_acc));
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
      fprintf(stderr, "zopfli-b200: no CUDA device available (%s). This library has no CPU path.\n",
              e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
      abort();
    }
    dev = want_dev;
    if (dev < 0 || dev >= n) { fprintf(stderr, "zopfli-b200: CUDA device %d does not exist (%d visible)\n", dev, n); abort(); }
    CK(cudaSetDevice(dev));
    cudaMemPool_t pool;
    CK(cudaDeviceGetDefaultMemPool(&pool, dev));
    uint64_t keep = ~0ull;  // keep freed arena memory cached in the pool
    CK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    for (int k = 0; k < Engine::kLanes; k++) lane[k].init((k & 1) == 0);
    DevBuf* shared[] = {&in_buf, &same_buf, &tile_first, &next_tile, &sym_ll[0], &sym_ll[1], &sym_ll[2], &sym_d[0],
                        &sym_d[1], &sym_d[2], &outbuf, &emit_desc, &err_flag};
    for (DevBuf* d : shared) d->st = lane[0].stream;
    int lo = 0, hi = 0;
    CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    CK(cudaStreamCreateWithPriority(&ck_stream, cudaStreamNonBlocking, lo));
    for (cudaEvent_t* e : {&ev_user, &ev_lane0, &ev_ck}) CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    ck_acc.st = ck_stream;
    CK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    CK(cudaFuncSetAttribute(k_match, cudaFuncAttributeMaxDynamicSharedMemorySize, kMatchSmemBytes));
    for (const void* k : {(const void*)k_iterate<2>, (const void*)k_iterate<kWideWarps>}) {
      cudaFuncAttributes fa;
      CK(cudaFuncGetAttributes(&fa, k));
      CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - (int)fa.sharedSizeBytes));
    }
    g_log.start();
  }

  uint32_t log_need = 0;  // entries the current batch asks for (0: the default size)
  void ensure_log() {  // caller holds mu
    if (!logtab || logtab_n < log_need) logtab = g_log.get(dev, lane[0].stream, log_need, &logtab_n);
  }

  void compute_same() {  // caller holds mu; runs on lane 0's stream and completes before returning
    if (insize == 0) return;
    Lane& l = lane[0];
    uint32_t ntiles = (uint32_t)((insize + kSameTile - 1) / kSameTile);
    same_buf.ensure(insize * sizeof(uint16_t) + 64);
    tile_first.ensure(ntiles * sizeof(uint32_t));
    next_tile.ensure(ntiles * sizeof(uint32_t));
    l.tic();
    k_same_tiles<<<ntiles, 256, 0, l.stream>>>(d_in, insize, tile_first.as<uint32_t>());
    k_same_next_tile<<<1, 1024, 0, l.stream>>>(tile_first.as<uint32_t>(), ntiles, next_tile.as<uint32_t>());
    k_same_fill<<<ntiles, 256, 0, l.stream>>>(d_in, insize, tile_first.as<uint32_t>(), next_tile.as<uint32_t>(),
                                              ntiles, same_buf.as<uint16_t>());
    CK(cudaGetLastError());
    l.toc(st_acc.ms_same);
    st_acc.launches += 3;
  }

  // zeroes the accumulator and queues the checksum (ChecksumKind) of d[0, n) on ck_stream; caller holds mu
  void launch_checksum(const uint8_t* d, uint64_t n, int kind) {
    ck_acc.ensure(sizeof(ChecksumAcc));
    CK(cudaMemsetAsync(ck_acc.p, 0, sizeof(ChecksumAcc), ck_stream));
    if (n == 0) return;
    const void* k = kind == kCkCrc32 ? (const void*)k_crc32 : (const void*)k_adler32;
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kCkThreads, 0));
    const uint64_t warps_wanted = n / kCkTile + 1;
    const unsigned grid = (unsigned)std::min<uint64_t>((warps_wanted + kCkThreads / 32 - 1) / (kCkThreads / 32),
                                                       (uint64_t)sm_count * std::max(per_sm, 1));
    CkArgs a{d, n, ck_acc.as<ChecksumAcc>(), crc_tab()};
    if (kind == kCkCrc32) k_crc32<<<grid, kCkThreads, 0, ck_stream>>>(a);
    else k_adler32<<<grid, kCkThreads, 0, ck_stream>>>(a);
    CK(cudaGetLastError());
    st_acc.launches++;
  }
  static const CrcShiftTable& crc_tab() {
    static const CrcShiftTable t = crc_shift_table();
    return t;
  }

  struct Layout {
    std::vector<SegDesc> segs;
    std::vector<KeyWork> kw;
    std::vector<PosWork> pw;
    std::vector<uint32_t> order;
    uint64_t nkeys = 0, npos = 0;
    bool any_parse = false;
    bool any_optimal = false;  // a segment runs the iterated optimal parse (not only fixed-tree parses)
  };

  void build_layout(const std::vector<ParseRange>& r, Layout& L) {
    L.segs.resize(r.size());
    for (size_t i = 0; i < r.size(); i++) {
      SegDesc& s = L.segs[i];
      // a range of at most 0x7fff0000 bytes keeps npos and nkeys (range + 32 KiB) in the 32-bit counts of SegDesc,
      // and every position and key index below 2^31 for the kernels' 32-bit index arithmetic (traced-path entries,
      // position << 9 | length, are 64-bit for that reason)
      if (r[i].inend < r[i].instart || r[i].inend > insize || r[i].inend - r[i].instart > 0x7fff0000ull) {
        fprintf(stderr, "zopfli-b200: bad parse range [%llu,%llu) for input of %llu bytes\n",
                (unsigned long long)r[i].instart, (unsigned long long)r[i].inend, (unsigned long long)insize);
        abort();
      }
      s.instart = r[i].instart;
      s.inend = r[i].inend;
      s.winstart = s.instart > (uint64_t)kWindow ? s.instart - kWindow : 0;  // squeeze.c:229-230
      s.key_off = L.nkeys;
      s.pos_off = L.npos;
      s.nkeys = (uint32_t)(s.inend - s.winstart);
      s.npos = (uint32_t)(s.inend - s.instart);
      s.mode = r[i].mode;
      s.numiterations = r[i].numiterations;
      if (s.npos == 0) s.nkeys = 0;
      L.nkeys += s.nkeys;
      L.npos += s.npos;
      if (s.mode != 0) L.any_parse = true;
      if (s.mode == 1) L.any_optimal = true;
      for (uint32_t f = 0; f < s.nkeys; f += kKeyChunk) L.kw.push_back({(uint32_t)i, f});
      for (uint32_t f = 0; f < s.npos; f += kMatchPosPerCta) L.pw.push_back({(uint32_t)i, f});
    }
    L.order.resize(r.size());
    for (size_t i = 0; i < r.size(); i++) L.order[i] = (uint32_t)i;
    std::stable_sort(L.order.begin(), L.order.end(), [&](uint32_t a, uint32_t b) {
      uint64_t wa = (uint64_t)L.segs[a].npos * (L.segs[a].mode == 1 ? L.segs[a].numiterations : 1);
      uint64_t wb = (uint64_t)L.segs[b].npos * (L.segs[b].mode == 1 ? L.segs[b].numiterations : 1);
      return wa > wb;
    });
  }

  // capacity of the run-list overflow arena after a launch asked for `used` entries.  Slot 7 of a run list holds
  // kOverflowBit | offset, so the arena stays within 2^31 entries.  The range guard of build_layout does not bound
  // it (a position may ask for up to ~250 entries), so a batch that needs more is refused here rather than handed
  // offsets that read the wrong entries.
  static uint32_t grown_ovf_cap(uint64_t used) {
    if (used >= kOverflowBit) {
      fprintf(stderr, "zopfli-b200: the run lists of one batch need %llu overflow entries, more than 2^31\n",
              (unsigned long long)used);
      abort();
    }
    return (uint32_t)std::min<uint64_t>(used + used / 4 + 1024, kOverflowBit);
  }

  // runs everything up to and including the match table on lane l; returns the Batch
  Batch prepare(const Layout& L, Lane& l) {
    const size_t ns = L.segs.size();
    l.upload(l.segs, L.segs);
    l.upload(l.keywork, L.kw);
    l.upload(l.poswork, L.pw);
    l.upload(l.order, L.order);
    l.hv.ensure(L.nkeys * 2 + 64);
    l.hv2.ensure(L.nkeys * 2 + 64);
    l.idx1.ensure(L.nkeys * 4 + 64);
    l.idx2.ensure(L.nkeys * 4 + 64);
    l.rank1.ensure(L.nkeys * 4 + 64);
    l.rank2.ensure(L.nkeys * 4 + 64);
    l.bkt1.ensure(ns * 32769 * 4 + 64);
    l.bkt2.ensure(ns * 32769 * 4 + 64);
    l.ld.ensure(L.npos * 4 + 64);
    for (int i = 0; i < 4; i++) l.st[i].ensure(L.npos * 2 + 64);
    l.jobs.ensure(ns * sizeof(JobState) + 64);
    l.out_ll.ensure(L.npos * 2 + 64);
    l.out_d.ensure(L.npos * 2 + 64);
    l.counters.ensure(256);
    if (L.any_parse) {
      l.mlen.ensure(L.npos * 2 + 64);
      l.runs.ensure(L.npos * kRunSlots * 4 + 64);
      l.dsx.ensure(L.npos * 32 + 64);
      l.ovf.ensure((size_t)l.ovf_cap * 4);
      l.la.ensure((L.npos + ns) * 2 + 64);
      l.path.ensure((L.npos + ns) * 8 + 64);
      { std::lock_guard<std::mutex> g(mu); ensure_log(); }
    }
    Batch b;
    memset(&b, 0, sizeof(b));
    b.in = d_in;
    b.insize = insize;
    b.same_g = same_buf.as<uint16_t>();
    b.segs = l.segs.as<SegDesc>();
    b.nsegs = (int)ns;
    b.hv = l.hv.as<uint16_t>();
    b.hv2 = l.hv2.as<uint16_t>();
    b.idx1 = l.idx1.as<uint32_t>();
    b.idx2 = l.idx2.as<uint32_t>();
    b.rank1 = l.rank1.as<uint32_t>();
    b.rank2 = l.rank2.as<uint32_t>();
    b.bkt1 = l.bkt1.as<uint32_t>();
    b.bkt2 = l.bkt2.as<uint32_t>();
    b.ld = l.ld.as<uint32_t>();
    b.mlen = l.mlen.as<uint16_t>();
    b.runs = l.runs.as<uint32_t>();
    b.dsx = l.dsx.as<uint8_t>();
    b.ovf = l.ovf.as<uint32_t>();
    b.ovf_used = &l.counters.as<Counters>()->ovf_used;
    b.ovf_cap = l.ovf_cap;
    b.la = l.la.as<uint16_t>();
    b.path = l.path.as<uint64_t>();
    b.st_ll[0] = l.st[0].as<uint16_t>();
    b.st_d[0] = l.st[1].as<uint16_t>();
    b.st_ll[1] = l.st[2].as<uint16_t>();
    b.st_d[1] = l.st[3].as<uint16_t>();
    b.st_ll[2] = nullptr;
    b.st_d[2] = nullptr;
    b.jobs = l.jobs.as<JobState>();
    b.logtab = logtab;
    b.logtab_n = logtab_n;
    b.out_ll = l.out_ll.as<uint16_t>();
    b.out_d = l.out_d.as<uint16_t>();
    b.out_used = &l.counters.as<Counters>()->out_used;
    static const uint32_t dp_flags = [] { const char* e = getenv("ZOPFLI_B200_INTDP"); return (e && atoi(e) == 0) ? 0u : 1u; }();
    b.dp_flags = dp_flags;

    CK(cudaMemsetAsync(l.bkt1.p, 0, ns * 32769 * 4, l.stream));
    CK(cudaMemsetAsync(l.bkt2.p, 0, ns * 32769 * 4, l.stream));
    CK(cudaMemsetAsync(l.counters.p, 0, 256, l.stream));
    CK(cudaMemsetAsync(l.jobs.p, 0, ns * sizeof(JobState), l.stream));
    if (L.nkeys) {
      l.tic();
      k_keys<<<(unsigned)L.kw.size(), 256, 0, l.stream>>>(b, l.keywork.as<KeyWork>());
      CK(cudaGetLastError());
      l.toc(l.acc.ms_keys);
      l.tic();
      k_bucket_scan<<<(unsigned)(2 * ns), 1024, 0, l.stream>>>(b);
      CK(cudaGetLastError());
      l.toc(l.acc.ms_scan);
      l.tic();
      k_scatter<<<(unsigned)(2 * ns * kScatterParts), 32, 0, l.stream>>>(b);
      CK(cudaGetLastError());
      l.toc(l.acc.ms_scatter);
      l.tic();
      k_match<<<(unsigned)L.pw.size(), kMatchWarps * 32, kMatchSmemBytes, l.stream>>>(b, l.poswork.as<PosWork>());
      CK(cudaGetLastError());
      l.toc(l.acc.ms_match);
      l.acc.launches += 4;
      l.acc.match_positions += L.npos;
    }
    return b;
  }
};

Engine::Engine(int dev) : p_(new Impl(dev)) {}

// ---- context pool: every API call leases one engine context (input buffers + lanes) for its whole
// duration, so concurrent callers never share mutable device state (the reference is re-entrant,
// zopfli.h:82-88).  Contexts are created on demand up to ZOPFLI_B200_CONTEXTS (default 4) and are
// intentionally leaked at exit: CUDA teardown order is undefined.
namespace {
std::mutex g_pool_mu;
std::condition_variable g_pool_cv;
std::vector<Engine*> g_all, g_free;   // contexts of every device; a context never changes device
size_t max_contexts() {
  static size_t n = [] { const char* e = getenv("ZOPFLI_B200_CONTEXTS"); int v = e ? atoi(e) : 4; return (size_t)(v < 1 ? 1 : (v > 16 ? 16 : v)); }();
  return n;
}
}  // namespace

int Engine::default_device() {  // ZOPFLI_B200_DEVICE, else the torchrun local rank, else device 0
  static int d = [] {
    if (const char* dv = getenv("ZOPFLI_B200_DEVICE")) return atoi(dv);
    if (const char* lr = getenv("LOCAL_RANK")) {
      int n = 0;
      if (cudaGetDeviceCount(&n) == cudaSuccess && n > 0) return atoi(lr) % n;
    }
    return 0;
  }();
  return d;
}

int Engine::device_count() {
  int n = 0;
  return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0;
}

Engine* Engine::acquire(int dev) {
  if (dev < 0) dev = default_device();
  std::unique_lock<std::mutex> lk(g_pool_mu);
  for (;;) {
    // the free context created first: its arenas are already grown, so a process that makes one call at a time
    // keeps using one context, and only calls that overlap grow others
    for (Engine* e : g_all) {
      if (e->device() != dev) continue;
      auto f = std::find(g_free.begin(), g_free.end(), e);
      if (f != g_free.end()) { g_free.erase(f); return e; }
    }
    size_t have = 0;
    for (Engine* e : g_all) have += e->device() == dev;
    if (have < max_contexts()) {
      Engine* e = new Engine(dev);
      g_all.push_back(e);
      return e;
    }
    g_pool_cv.wait(lk);
  }
}
void Engine::release(Engine* e) {
  { std::lock_guard<std::mutex> g(g_pool_mu); g_free.push_back(e); }
  g_pool_cv.notify_all();
}

int Engine::device() const { return p_->dev; }

void Engine::set_stream(void* s) {
  std::lock_guard<std::mutex> g(p_->mu);
  CK(cudaSetDevice(p_->dev));
  if (s) {  // lane 0 adopts the caller's stream (bench timing with events on that stream)
    Lane& l = p_->lane[0];
    std::lock_guard<std::mutex> g2(l.mu);
    l.stream = (cudaStream_t)s;
    DevBuf* all[] = {&l.segs, &l.keywork, &l.poswork, &l.order, &l.hv, &l.hv2, &l.idx1, &l.idx2, &l.rank1, &l.rank2,
                     &l.bkt1, &l.bkt2, &l.ld, &l.mlen, &l.runs, &l.dsx, &l.ovf, &l.la, &l.path, &l.st[0], &l.st[1],
                     &l.st[2], &l.st[3], &l.jobs, &l.out_ll, &l.out_d, &l.counters, &l.misc, &l.iterc, &l.sp_ll,
                     &l.sp_d, &l.sp_llsym, &l.sp_dsym, &l.sp_pos, &l.sp_snaps, &l.sp_stores, &l.sp_work, &l.sp_evals,
                     &l.sp_out, &p_->in_buf, &p_->same_buf, &p_->tile_first, &p_->next_tile, &p_->sym_ll[0], &p_->sym_ll[1],
                     &p_->sym_ll[2], &p_->sym_d[0], &p_->sym_d[1], &p_->sym_d[2], &p_->outbuf, &p_->emit_desc, &p_->err_flag};
    for (DevBuf* d : all) d->st = l.stream;
  }
}

EngineStats Engine::stats_all() {
  std::vector<Engine*> all;
  { std::lock_guard<std::mutex> g(g_pool_mu); all = g_all; }
  EngineStats r;
  memset(&r, 0, sizeof(r));
  for (Engine* e : all) {
    const EngineStats a = e->stats();
    r.ms_same += a.ms_same; r.ms_h2d += a.ms_h2d;
    r.ms_keys += a.ms_keys; r.ms_scan += a.ms_scan; r.ms_scatter += a.ms_scatter; r.ms_match += a.ms_match;
    r.ms_greedy += a.ms_greedy; r.ms_iterate += a.ms_iterate; r.ms_pack += a.ms_pack; r.ms_d2h += a.ms_d2h;
    r.ms_split += a.ms_split; r.split_evals += a.split_evals; r.split_rounds += a.split_rounds;
    r.iterate_launches += a.iterate_launches;
    r.launches += a.launches; r.match_positions += a.match_positions; r.iterate_positions += a.iterate_positions;
    r.iterate_steps += a.iterate_steps; r.h2d_bytes += a.h2d_bytes; r.d2h_bytes += a.d2h_bytes; r.int_steps += a.int_steps;
    r.ovf_regrows += a.ovf_regrows; r.log_regrows += a.log_regrows;
    uint64_t ta = 0, tr = 0;
    for (int i = 0; i < 6; i++) { r.cyc_sum[i] += a.cyc_sum[i]; ta += a.cyc_max[i]; tr += r.cyc_max[i]; }
    for (int i = 0; i < 5; i++) r.dp_cyc_sum[i] += a.dp_cyc_sum[i];
    for (int i = 0; i < 6; i++) r.dp_cnt_sum[i] += a.dp_cnt_sum[i];
    if (ta > tr) {
      for (int i = 0; i < 6; i++) r.cyc_max[i] = a.cyc_max[i];
      r.max_block_positions = a.max_block_positions;
      for (int i = 0; i < 5; i++) r.dp_cyc_max[i] = a.dp_cyc_max[i];
      for (int i = 0; i < 6; i++) r.dp_cnt_max[i] = a.dp_cnt_max[i];
    }
  }
  return r;
}
void Engine::reset_stats_all() {
  std::vector<Engine*> all;
  { std::lock_guard<std::mutex> g(g_pool_mu); all = g_all; }
  for (Engine* e : all) e->reset_stats();
}

EngineStats Engine::stats() {
  std::lock_guard<std::mutex> g(p_->mu);
  EngineStats r = p_->st_acc;
  for (int k = 0; k < Engine::kLanes; k++) {
    const EngineStats& a = p_->lane[k].acc;
    r.ms_keys += a.ms_keys; r.ms_scan += a.ms_scan; r.ms_scatter += a.ms_scatter; r.ms_match += a.ms_match;
    r.ms_greedy += a.ms_greedy; r.ms_iterate += a.ms_iterate; r.ms_pack += a.ms_pack; r.ms_d2h += a.ms_d2h;
    r.ms_split += a.ms_split; r.split_evals += a.split_evals; r.split_rounds += a.split_rounds;
    r.iterate_launches += a.iterate_launches;
    r.launches += a.launches; r.match_positions += a.match_positions; r.iterate_positions += a.iterate_positions;
    r.iterate_steps += a.iterate_steps; r.h2d_bytes += a.h2d_bytes; r.d2h_bytes += a.d2h_bytes; r.int_steps += a.int_steps;
    r.ovf_regrows += a.ovf_regrows; r.log_regrows += a.log_regrows;
    uint64_t ta = 0, tr = 0;
    for (int i = 0; i < 6; i++) { r.cyc_sum[i] += a.cyc_sum[i]; ta += a.cyc_max[i]; tr += r.cyc_max[i]; }
    for (int i = 0; i < 5; i++) r.dp_cyc_sum[i] += a.dp_cyc_sum[i];
    for (int i = 0; i < 6; i++) r.dp_cnt_sum[i] += a.dp_cnt_sum[i];
    if (ta > tr) {
      for (int i = 0; i < 6; i++) r.cyc_max[i] = a.cyc_max[i];
      r.max_block_positions = a.max_block_positions;
      for (int i = 0; i < 5; i++) r.dp_cyc_max[i] = a.dp_cyc_max[i];
      for (int i = 0; i < 6; i++) r.dp_cnt_max[i] = a.dp_cnt_max[i];
    }
  }
  return r;
}
void Engine::reset_stats() {
  std::lock_guard<std::mutex> g(p_->mu);
  memset(&p_->st_acc, 0, sizeof(p_->st_acc));
  for (int k = 0; k < Engine::kLanes; k++) memset(&p_->lane[k].acc, 0, sizeof(EngineStats));
}

void Engine::set_input_host(const uint8_t* in, size_t insize) {
  std::lock_guard<std::mutex> g(p_->mu);
  Impl& m = *p_;
  Lane& l = m.lane[0];
  CK(cudaSetDevice(m.dev));
  m.in_buf.ensure(insize + 64);
  l.tic();
  CK(cudaMemsetAsync((uint8_t*)m.in_buf.p + insize, 0, 64, l.stream));
  l.toc(m.st_acc.ms_h2d);
  l.sync();  // the buffer exists (stream-ordered allocation) before other streams write into it
  m.stager.copy((uint8_t*)m.in_buf.p, in, insize, true, m.dev);
  m.st_acc.h2d_bytes += insize;
  m.d_in = m.in_buf.as<uint8_t>();
  m.insize = insize;
  m.compute_same();
  l.sync();  // the other lanes read the input and `same` from their own streams
  m.begin_call();
}

void Engine::set_input_device(const uint8_t* dev_in, size_t insize) {
  std::lock_guard<std::mutex> g(p_->mu);
  Impl& m = *p_;
  CK(cudaSetDevice(m.dev));
  if (((uintptr_t)dev_in & 15) != 0) {
    fprintf(stderr, "zopfli-b200: device input must be 16-byte aligned\n");
    abort();
  }
  m.d_in = dev_in;
  m.insize = insize;
  m.compute_same();
  m.lane[0].sync();
  m.begin_call();
}

void Engine::set_input_device_copy(const uint8_t* dev_src, size_t insize, void* user_stream, int checksum) {
  std::lock_guard<std::mutex> g(p_->mu);
  Impl& m = *p_;
  Lane& l = m.lane[0];
  CK(cudaSetDevice(m.dev));
  m.in_buf.ensure(insize + 64);
  // the lanes are non-blocking streams: they order against the caller's stream only through an event
  CK(cudaEventRecord(m.ev_user, (cudaStream_t)user_stream));
  CK(cudaStreamWaitEvent(l.stream, m.ev_user, 0));
  if (insize) CK(cudaMemcpyAsync(m.in_buf.p, dev_src, insize, cudaMemcpyDeviceToDevice, l.stream));
  CK(cudaMemsetAsync((uint8_t*)m.in_buf.p + insize, 0, 64, l.stream));
  m.d_in = m.in_buf.as<uint8_t>();
  m.insize = insize;
  if (checksum != kCkNone) {
    CK(cudaEventRecord(m.ev_lane0, l.stream));
    CK(cudaStreamWaitEvent(m.ck_stream, m.ev_lane0, 0));
    m.launch_checksum(m.d_in, insize, checksum);
    CK(cudaEventRecord(m.ev_ck, m.ck_stream));
  }
  m.compute_same();
  l.sync();
  m.begin_call();
}

uint32_t Engine::checksum_device(const uint8_t* dev_in, size_t n, void* user_stream, int checksum) {
  std::lock_guard<std::mutex> g(p_->mu);
  Impl& m = *p_;
  CK(cudaSetDevice(m.dev));
  CK(cudaEventRecord(m.ev_user, (cudaStream_t)user_stream));
  CK(cudaStreamWaitEvent(m.ck_stream, m.ev_user, 0));
  m.launch_checksum(dev_in, n, checksum);
  ChecksumAcc h;
  CK(cudaMemcpyAsync(&h, m.ck_acc.p, sizeof(h), cudaMemcpyDeviceToHost, m.ck_stream));
  CK(cudaStreamSynchronize(m.ck_stream));
  return checksum == kCkCrc32 ? crc_finish(h.crc0, n, Impl::crc_tab()) : adler_finish(h.a, h.b, n);
}

int Engine::pointer_device(const void* p) {
  cudaPointerAttributes a;
  if (!p || cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return -1; }
  return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.device : -1;
}

int Engine::current_device() {
  int d = 0;
  CK(cudaGetDevice(&d));
  return d;
}

void Engine::free_device(void* p, void* user_stream) {
  if (!p) return;
  int prev = 0;
  CK(cudaGetDevice(&prev));
  const int d = pointer_device(p);
  if (d >= 0) CK(cudaSetDevice(d));  // a NULL stream is the legacy stream of the device that owns p
  CK(cudaFreeAsync(p, (cudaStream_t)user_stream));
  CK(cudaSetDevice(prev));
}

void Engine::parse(const std::vector<ParseRange>& ranges, ParseResult& out, int lane_id) {
  parse_common(ranges, out, -1, lane_id);
}

void Engine::parse_keep(const std::vector<ParseRange>& ranges, int dest, std::vector<uint32_t>& sizes,
                        std::vector<uint64_t>& costs, int lane_id, std::vector<uint64_t>* iter_costs) {
  for (const ParseRange& r : ranges)
    if (r.mode == 0) { fprintf(stderr, "zopfli-b200: parse_keep takes optimal-parse ranges only\n"); abort(); }
  ParseResult res;
  parse_common(ranges, res, dest, lane_id, iter_costs);
  sizes.swap(res.size);
  costs.swap(res.cost);
}

uint64_t Engine::input_size() const { return p_->insize; }

uint64_t Engine::device_memory_total() const {
  size_t fr = 0, tot = 0;
  CK(cudaSetDevice(p_->dev));
  CK(cudaMemGetInfo(&fr, &tot));
  return tot;
}

// dest < 0: the symbols come back to the host (test seams); otherwise they stay in symbol buffer `dest`
void Engine::parse_common(const std::vector<ParseRange>& ranges, ParseResult& out, int dest, int lane_id,
                          std::vector<uint64_t>* iter_costs) {
  Impl& m = *p_;
  Lane& l = m.lane[(unsigned)lane_id % Engine::kLanes];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  const size_t ns = ranges.size();
  out.off.assign(ns, 0);
  out.size.assign(ns, 0);
  out.cost.assign(ns, 0);
  out.ll.clear();
  out.d.clear();
  if (ns == 0) return;
  Impl::Layout L;
  m.build_layout(ranges, L);
  std::vector<JobState> js(ns);
  Counters counters{};
  {  // statistics sums usually stay below 2 x symbols; a blended or randomized sum past that is met below: the log
     // table is grown to it and the batch redone
    uint64_t need = 0;
    for (const SegDesc& sg : L.segs)
      if (sg.mode == 1) need = std::max<uint64_t>(need, 2ull * sg.npos + 16);
    if (need > kLogTabN) {
      std::lock_guard<std::mutex> g(m.mu);
      if (need > m.log_need) m.log_need = (uint32_t)std::min<uint64_t>(need, 0xfffffff0ull);
    }
  }
  uint32_t it_stride = 0;
  if (iter_costs)
    for (const ParseRange& r : ranges) it_stride = std::max<uint32_t>(it_stride, r.mode == 1 ? (uint32_t)std::max(r.numiterations, 0) : 0u);
  for (int attempt = 0;; attempt++) {
    Batch b = m.prepare(L, l);
    if (it_stride) {
      l.iterc.ensure((size_t)ns * it_stride * 8 + 64);
      CK(cudaMemsetAsync(l.iterc.p, 0xff, (size_t)ns * it_stride * 8, l.stream));
      b.iter_cost = l.iterc.as<uint64_t>();
      b.iter_stride = it_stride;
    }
    l.tic();
    k_greedy<<<(unsigned)ns, kGreedyThreads, 0, l.stream>>>(b, 0);
    CK(cudaGetLastError());
    l.toc(l.acc.ms_greedy);
    l.acc.launches++;
    if (L.any_parse) {
      l.tic();
      // one-warp CTAs: pad shared memory so that at most four fit on an SM and every DP chain
      // has a scheduler partition of its own (a partition mate costs the chain ~20% of its speed)
      // A batch of only a few blocks (the giants of stage C) takes whole SMs: with 188 KB of padding
      // no kernel that uses shared memory can move in beside the chain.
      // Those whole-SM launches of optimal parses run the wide form of k_iterate: its other six warps take part
      // in trace-back and follow-path.  ZOPFLI_B200_WIDE=0 / 1 forces the two-warp / wide form for every launch.
      static const unsigned static_smem = [] { cudaFuncAttributes fa; CK(cudaFuncGetAttributes(&fa, k_iterate<2>)); return (unsigned)fa.sharedSizeBytes; }();
      static const unsigned pad_many = [] { const char* e = getenv("ZOPFLI_B200_ITER_PAD"); return e ? (unsigned)atoi(e) : 56u * 1024u - static_smem; }();
      static const unsigned pad_few = [] { const char* e = getenv("ZOPFLI_B200_ITER_PAD_FEW"); return e ? (unsigned)atoi(e) : 222u * 1024u - static_smem; }();
      static const int wide_env = [] { const char* e = getenv("ZOPFLI_B200_WIDE"); return e ? atoi(e) : -1; }();
      const bool few = ns <= 64;
      const bool wide = wide_env < 0 ? few && L.any_optimal : wide_env != 0;
      unsigned pad = few ? pad_few : pad_many;
      if (pad < sizeof(IterDyn)) pad = (unsigned)sizeof(IterDyn);  // the integer window's tables live in the dynamic part
      if (wide) {
        if (pad < wide_dyn_bytes<kWideWarps>()) pad = (unsigned)wide_dyn_bytes<kWideWarps>();
        k_iterate<kWideWarps><<<(unsigned)ns, kWideWarps * 32, pad, l.stream>>>(b, l.order.as<uint32_t>());
      } else {
        k_iterate<2><<<(unsigned)ns, 64, pad, l.stream>>>(b, l.order.as<uint32_t>());
      }
      CK(cudaGetLastError());
      l.toc(l.acc.ms_iterate);
      l.acc.launches++;
      l.acc.iterate_launches++;
    }
    l.tic();
    if (dest < 0) {
      k_pack<<<(unsigned)ns, 256, 0, l.stream>>>(b, L.any_parse ? 0 : 1);
    } else {
      m.ensure_sym(dest);
      k_keep<<<(unsigned)ns, 256, 0, l.stream>>>(b, m.sym_ll[dest].as<uint16_t>(), m.sym_d[dest].as<uint16_t>());
    }
    CK(cudaGetLastError());
    l.toc(l.acc.ms_pack);
    l.acc.launches++;
    l.tic();
    CK(cudaMemcpyAsync(js.data(), l.jobs.p, ns * sizeof(JobState), cudaMemcpyDeviceToHost, l.stream));
    CK(cudaMemcpyAsync(&counters, l.counters.p, sizeof(counters), cudaMemcpyDeviceToHost, l.stream));
    if (it_stride) {
      iter_costs->assign((size_t)ns * it_stride, ~0ull);
      CK(cudaMemcpyAsync(iter_costs->data(), l.iterc.p, (size_t)ns * it_stride * 8, cudaMemcpyDeviceToHost, l.stream));
    }
    l.toc(l.acc.ms_d2h);
    l.sync();
    if (L.any_parse && counters.ovf_used > l.ovf_cap) {  // run-list overflow arena too small: grow, redo
      l.ovf_cap = Impl::grown_ovf_cap(counters.ovf_used);
      l.acc.ovf_regrows++;
      if (attempt > 2) { fprintf(stderr, "zopfli-b200: overflow arena did not converge\n"); abort(); }
      continue;
    }
    uint32_t log_miss = 0;  // the largest statistics count or sum whose log fell outside the table
    for (size_t i = 0; i < ns; i++)
      if (js[i].flags & 1) log_miss = std::max(log_miss, js[i].log_miss);
    if (log_miss) {  // a statistics sum outgrew the log table: grow it past that sum with room to spare, redo
      if (log_miss >= 0xfffffff0u) {
        fprintf(stderr, "zopfli-b200: symbol count %u beyond the largest log table\n", log_miss);
        abort();
      }
      {
        std::lock_guard<std::mutex> g(m.mu);
        m.log_need = std::max<uint32_t>(m.log_need, (uint32_t)std::min<uint64_t>(log_miss + (uint64_t)log_miss / 4 + 1024, 0xfffffff0ull));
      }
      l.acc.log_regrows++;
      if (attempt > 2) { fprintf(stderr, "zopfli-b200: log table did not converge\n"); abort(); }
      continue;
    }
    const uint32_t total = dest < 0 ? counters.out_used : 0u;
    out.ll.resize(total);
    out.d.resize(total);
    if (total) {
      l.tic();
      CK(cudaMemcpyAsync(out.ll.data(), l.out_ll.p, (size_t)total * 2, cudaMemcpyDeviceToHost, l.stream));
      CK(cudaMemcpyAsync(out.d.data(), l.out_d.p, (size_t)total * 2, cudaMemcpyDeviceToHost, l.stream));
      l.toc(l.acc.ms_d2h);
      l.sync();
    }
    l.acc.d2h_bytes += (uint64_t)total * 4 + ns * sizeof(JobState);
    break;
  }
  for (size_t i = 0; i < ns; i++) {
    const bool greedy_only = !L.any_parse;
    out.off[i] = js[i].out_off;
    out.size[i] = greedy_only ? js[i].greedy_size : js[i].best_size;
    out.cost[i] = js[i].best_cost;
    if (!greedy_only && ranges[i].mode == 0) {
      fprintf(stderr, "zopfli-b200: greedy and optimal ranges cannot share a batch\n");
      abort();
    }
    if (js[i].flags & 2) { fprintf(stderr, "zopfli-b200: corrupted length chain in block %zu\n", i); abort(); }
    if (ranges[i].mode == 1) {
      uint64_t tot = 0, cur = 0;
      for (int k = 0; k < 6; k++) { l.acc.cyc_sum[k] += js[i].cyc[k]; tot += js[i].cyc[k]; cur += l.acc.cyc_max[k]; }
      for (int k = 0; k < 5; k++) l.acc.dp_cyc_sum[k] += js[i].dpc[k];
      for (int k = 0; k < 6; k++) l.acc.dp_cnt_sum[k] += js[i].dpn[k];
      if (tot > cur) {
        for (int k = 0; k < 6; k++) l.acc.cyc_max[k] = js[i].cyc[k];
        l.acc.max_block_positions = L.segs[i].npos;
        for (int k = 0; k < 5; k++) l.acc.dp_cyc_max[k] = js[i].dpc[k];
        for (int k = 0; k < 6; k++) l.acc.dp_cnt_max[k] = js[i].dpn[k];
      }
      l.acc.iterate_positions += L.segs[i].npos;
      l.acc.iterate_steps += (uint64_t)L.segs[i].npos * ranges[i].numiterations;
      l.acc.int_steps += (uint64_t)js[i].int_groups * 32u;
    }
  }
}

void Engine::match_table(uint64_t instart, uint64_t inend, std::vector<uint16_t>& len,
                         std::vector<uint16_t>& dist, std::vector<uint16_t>& sublen,
                         std::vector<uint16_t>& same, std::vector<uint16_t>& hvv, std::vector<uint16_t>& hv2v) {
  Impl& m = *p_;
  Lane& l = m.lane[0];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  std::vector<ParseRange> r{{instart, inend, 1, 1}};
  Impl::Layout L;
  m.build_layout(r, L);
  std::vector<uint32_t> h_ld, h_runs, h_ovf;
  std::vector<uint16_t> h_mlen, h_hv, h_hv2, h_same;
  const size_t n = (size_t)(inend - instart);
  for (int attempt = 0;; attempt++) {
    m.prepare(L, l);
    Counters c{};
    CK(cudaMemcpyAsync(&c, l.counters.p, sizeof(c), cudaMemcpyDeviceToHost, l.stream));
    l.sync();
    const size_t used = c.ovf_used;
    if (used > l.ovf_cap) {
      l.ovf_cap = Impl::grown_ovf_cap(used);
      l.acc.ovf_regrows++;
      if (attempt > 2) abort();
      continue;
    }
    h_ld.resize(n); h_runs.resize(n * kRunSlots); h_mlen.resize(n); h_ovf.resize(used + 1);
    h_hv.resize(L.nkeys); h_hv2.resize(L.nkeys); h_same.resize(n);
    if (n) {
      CK(cudaMemcpy(h_ld.data(), l.ld.p, n * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h_runs.data(), l.runs.p, n * kRunSlots * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h_mlen.data(), l.mlen.p, n * 2, cudaMemcpyDeviceToHost));
      if (used) CK(cudaMemcpy(h_ovf.data(), l.ovf.p, (size_t)used * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h_hv.data(), l.hv.p, L.nkeys * 2, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h_hv2.data(), l.hv2.p, L.nkeys * 2, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h_same.data(), m.same_buf.as<uint16_t>() + instart, n * 2, cudaMemcpyDeviceToHost));
    }
    break;
  }
  len.assign(n, 0); dist.assign(n, 0); sublen.assign(n * 259, 0); same.assign(n, 0); hvv.assign(n, 0); hv2v.assign(n, 0);
  const size_t woff = (size_t)(instart - L.segs[0].winstart);
  for (size_t j = 0; j < n; j++) {
    len[j] = (uint16_t)(h_ld[j] >> 16);
    dist[j] = (uint16_t)(h_ld[j] & 0xffff);
    uint64_t clip = inend - 1 - (instart + j);
    same[j] = (uint16_t)std::min<uint64_t>(h_same[j], clip);
    hvv[j] = h_hv[woff + j];
    hv2v[j] = h_hv2[woff + j];
    uint32_t prev = 2;
    auto put = [&](uint32_t e) {
      for (uint32_t k = std::max<uint32_t>(prev + 1, 3); k <= run_len(e); k++) sublen[j * 259 + k] = (uint16_t)run_dist(e);
      prev = run_len(e);
    };
    if ((h_mlen[j] & 0x7fff) >= 3) {
      for (int r2 = 0; r2 < kRunSlots; r2++) {
        uint32_t e = h_runs[j * kRunSlots + r2];
        if (r2 == kRunSlots - 1 && (e & kOverflowBit)) {
          uint32_t off = e & ~kOverflowBit, cnt = h_ovf[off];
          for (uint32_t t = 0; t < cnt; t++) put(h_ovf[off + 1 + t]);
        } else if (run_len(e)) put(e);
      }
    }
  }
}

// builds the split service of lane `l` over stores that already sit on the device
static void split_setup(Lane& l, const uint16_t* dev_ll, const uint16_t* dev_d, const std::vector<uint64_t>& off,
                        const std::vector<uint32_t>& size) {
  const size_t ns = off.size();
  uint64_t total = 0, nsnap_total = 0, pos_total = 0;
  for (size_t i = 0; i < ns; i++) total = std::max<uint64_t>(total, off[i] + size[i]);
  l.sp_desc.resize(ns);
  std::vector<SnapWork> work;
  for (size_t i = 0; i < ns; i++) {
    SplitStoreDesc& sd = l.sp_desc[i];
    sd.sym_off = off[i];
    sd.n = size[i];
    sd.nsnap = size[i] / kSnap + 1;
    sd.snap_off = nsnap_total;
    nsnap_total += sd.nsnap;
    sd.pos_off = pos_total;  // independent of sym_off: stores may sit in any order in the flat arrays
    pos_total += (uint64_t)size[i] + 1;
    for (uint32_t c = 0; c * kSnap < size[i]; c++) work.push_back({(uint32_t)i, c});
  }
  l.sp_llsym.ensure(total * 2 + 64);
  l.sp_dsym.ensure(total + 64);
  l.sp_snaps.ensure(nsnap_total * 320 * 4 + 64);
  l.sp_pos.ensure(pos_total * 4 + 64);
  l.upload(l.sp_stores, l.sp_desc);
  l.upload(l.sp_work, work);
  SplitBatch& b = l.sp_batch;
  b.ll = dev_ll;
  b.d = dev_d;
  b.llsym = l.sp_llsym.as<uint16_t>();
  b.dsym = l.sp_dsym.as<uint8_t>();
  b.pos = l.sp_pos.as<uint32_t>();
  b.snaps = l.sp_snaps.as<uint32_t>();
  b.stores = l.sp_stores.as<SplitStoreDesc>();
  for (size_t i = 0; i < ns; i++)
    if (size[i]) k_split_prep_sym<<<(size[i] + 255) / 256, 256, 0, l.stream>>>(b, (uint32_t)i);
  if (ns) k_split_prep_pos<<<(unsigned)ns, 1024, 0, l.stream>>>(b);
  if (!work.empty())
    k_split_prep_snap<<<(unsigned)((work.size() + 7) / 8), 256, 0, l.stream>>>(b, l.sp_work.as<SnapWork>(), (uint32_t)work.size());
  if (ns) k_split_prep_prefix<<<(unsigned)ns, 320, 0, l.stream>>>(b);
  CK(cudaGetLastError());
  l.acc.launches += ns + 3;
}

void Engine::split_begin(const uint16_t* ll, const uint16_t* d, const std::vector<uint64_t>& off,
                         const std::vector<uint32_t>& size, int lane_id) {
  Impl& m = *p_;
  Lane& l = m.lane[(unsigned)lane_id % Engine::kLanes];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  uint64_t total = 0;
  for (size_t i = 0; i < off.size(); i++) total = std::max<uint64_t>(total, off[i] + size[i]);
  l.sp_ll.ensure(total * 2 + 64);
  l.sp_d.ensure(total * 2 + 64);
  l.tic();
  if (total) {
    CK(cudaMemcpyAsync(l.sp_ll.p, ll, total * 2, cudaMemcpyHostToDevice, l.stream));
    CK(cudaMemcpyAsync(l.sp_d.p, d, total * 2, cudaMemcpyHostToDevice, l.stream));
  }
  split_setup(l, l.sp_ll.as<uint16_t>(), l.sp_d.as<uint16_t>(), off, size);
  l.toc(l.acc.ms_split);
  l.sync();
  l.acc.h2d_bytes += total * 4;
}

void Engine::greedy_to_split(const std::vector<ParseRange>& ranges, std::vector<uint32_t>& sizes, int lane_id) {
  Impl& m = *p_;
  Lane& l = m.lane[(unsigned)lane_id % Engine::kLanes];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  const size_t ns = ranges.size();
  sizes.assign(ns, 0);
  if (ns == 0) return;
  for (const ParseRange& r : ranges)
    if (r.mode != 0) { fprintf(stderr, "zopfli-b200: greedy_to_split takes greedy ranges only\n"); abort(); }
  Impl::Layout L;
  m.build_layout(ranges, L);
  Batch b = m.prepare(L, l);
  l.tic();
  k_greedy<<<(unsigned)ns, kGreedyThreads, 0, l.stream>>>(b, 0);
  CK(cudaGetLastError());
  l.toc(l.acc.ms_greedy);
  l.acc.launches++;
  std::vector<JobState> js(ns);
  l.tic();
  CK(cudaMemcpyAsync(js.data(), l.jobs.p, ns * sizeof(JobState), cudaMemcpyDeviceToHost, l.stream));
  l.toc(l.acc.ms_d2h);
  l.sync();
  l.acc.d2h_bytes += ns * sizeof(JobState);
  std::vector<uint64_t> off(ns);
  for (size_t i = 0; i < ns; i++) { sizes[i] = js[i].greedy_size; off[i] = L.segs[i].pos_off; }
  l.tic();
  split_setup(l, b.st_ll[0], b.st_d[0], off, sizes);  // k_greedy wrote range i's store at its pos_off
  l.toc(l.acc.ms_split);
  l.sync();
}

__global__ void k_split_gather_pos(SplitBatch b, const Engine::SplitPos* __restrict__ q, uint32_t n, uint32_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = b.pos[b.stores[q[i].store].pos_off + q[i].idx];
}

void Engine::split_positions(const std::vector<SplitPos>& q, std::vector<uint32_t>& bytepos, int lane_id) {
  Impl& m = *p_;
  Lane& l = m.lane[(unsigned)lane_id % Engine::kLanes];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  bytepos.assign(q.size(), 0);
  if (q.empty()) return;
  l.sp_evals.ensure(q.size() * sizeof(SplitPos) + 64);
  l.sp_out.ensure(q.size() * 4 + 64);
  CK(cudaMemcpyAsync(l.sp_evals.p, q.data(), q.size() * sizeof(SplitPos), cudaMemcpyHostToDevice, l.stream));
  k_split_gather_pos<<<(unsigned)((q.size() + 255) / 256), 256, 0, l.stream>>>(l.sp_batch, l.sp_evals.as<SplitPos>(), (uint32_t)q.size(),
                                                                              l.sp_out.as<uint32_t>());
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(bytepos.data(), l.sp_out.p, q.size() * 4, cudaMemcpyDeviceToHost, l.stream));
  l.sync();
  l.acc.launches++;
}

void Engine::split_eval(const SplitReq* reqs, size_t n, uint64_t* costs, int lane_id) {
  Impl& m = *p_;
  Lane& l = m.lane[(unsigned)lane_id % Engine::kLanes];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  if (n == 0) return;
  const size_t kChunk = 32768;  // scratch is per evaluation: bound it
  l.sp_evals.ensure(n * sizeof(SplitEval) + 64);
  l.sp_out.ensure(n * 8 + 64);
  // one round of the split search = one latency-bound round trip: requests and answers go through
  // page-locked staging so that neither copy waits for the driver's pageable path
  SplitEval* ev = (SplitEval*)l.pin_req.ensure(n * sizeof(SplitEval));
  uint64_t* res = (uint64_t*)l.pin_out.ensure(n * 8);
  for (size_t i = 0; i < n; i++) ev[i] = {reqs[i].store, reqs[i].lstart, reqs[i].lend, 0};
  l.tic();
  CK(cudaMemcpyAsync(l.sp_evals.p, ev, n * sizeof(SplitEval), cudaMemcpyHostToDevice, l.stream));
  SplitBatch b = l.sp_batch;
  for (size_t o = 0; o < n; o += kChunk) {
    const size_t c = std::min(kChunk, n - o);
    k_split_eval<<<(unsigned)((c + kEvalWarps - 1) / kEvalWarps), kEvalWarps * 32, 0, l.stream>>>(
        b, l.sp_evals.as<SplitEval>() + o, (uint32_t)c, l.sp_out.as<uint64_t>() + o);
    l.acc.launches++;
  }
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(res, l.sp_out.p, n * 8, cudaMemcpyDeviceToHost, l.stream));
  l.toc(l.acc.ms_split);
  l.sync();
  memcpy(costs, res, n * 8);
  l.acc.split_evals += n;
  l.acc.split_rounds++;
}

void Engine::concat_stores(const std::vector<SymCopy>& copies, const std::vector<uint64_t>& store_off,
                           const std::vector<uint32_t>& store_size, int lane_id) {
  Impl& m = *p_;
  Lane& l = m.lane[(unsigned)lane_id % Engine::kLanes];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  m.ensure_sym(kPack);
  m.ensure_sym(kFin);
  static_assert(sizeof(SymCopy) == sizeof(SymCopyDev), "layout");
  l.tic();
  if (!copies.empty()) {
    l.misc.ensure(copies.size() * sizeof(SymCopyDev) + 64);
    CK(cudaMemcpyAsync(l.misc.p, copies.data(), copies.size() * sizeof(SymCopyDev), cudaMemcpyHostToDevice, l.stream));
    k_sym_copy<<<(unsigned)copies.size(), 256, 0, l.stream>>>(l.misc.as<SymCopyDev>(), m.sym_ll[kPack].as<uint16_t>(),
                                                            m.sym_d[kPack].as<uint16_t>(), m.sym_ll[kFin].as<uint16_t>(),
                                                            m.sym_d[kFin].as<uint16_t>());
    CK(cudaGetLastError());
    l.acc.launches++;
  }
  if (!store_off.empty()) split_setup(l, m.sym_ll[kFin].as<uint16_t>(), m.sym_d[kFin].as<uint16_t>(), store_off, store_size);
  l.toc(l.acc.ms_split);
  l.sync();
}

void Engine::plan_blocks(const std::vector<PlanReq>& reqs, std::vector<PlanCost>& costs, std::vector<uint64_t>& handles,
                         int lane_id) {
  Impl& m = *p_;
  Lane& l = m.lane[(unsigned)lane_id % Engine::kLanes];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  const size_t n = reqs.size();
  costs.assign(n, PlanCost{0, 0, 0, 0});
  handles.assign(n, 0);
  if (n == 0) return;
  BlockPlan* plans = m.plan_alloc(n);
  std::vector<PlanReqDev> rd(n);
  for (size_t i = 0; i < n; i++) {
    m.ensure_sym((int)reqs[i].buf);
    rd[i].ll = m.sym_ll[reqs[i].buf].as<uint16_t>() + reqs[i].off;
    rd[i].d = m.sym_d[reqs[i].buf].as<uint16_t>() + reqs[i].off;
    rd[i].out = plans + i;
    rd[i].n = reqs[i].n;
    rd[i].pad = 0;
    handles[i] = (uint64_t)(uintptr_t)(plans + i);
  }
  l.sp_evals.ensure(n * sizeof(PlanReqDev) + 64);
  std::vector<BlockPlan> hp(n);
  l.tic();
  CK(cudaMemcpyAsync(l.sp_evals.p, rd.data(), n * sizeof(PlanReqDev), cudaMemcpyHostToDevice, l.stream));
  k_block_plan<<<(unsigned)n, kPlanThreads, 0, l.stream>>>(l.sp_evals.as<PlanReqDev>());
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(hp.data(), plans, n * sizeof(BlockPlan), cudaMemcpyDeviceToHost, l.stream));
  l.toc(l.acc.ms_split);
  l.sync();
  l.acc.launches++;
  l.acc.d2h_bytes += n * sizeof(BlockPlan);
  for (size_t i = 0; i < n; i++) costs[i] = PlanCost{hp[i].unc_bits, hp[i].fixed_bits, hp[i].dyn_bits, hp[i].tree_bits};
}

void* Engine::stream() { return (void*)p_->lane[0].stream; }

void* Engine::emit_device(const std::vector<EmitPiece>& pieces, uint64_t total_bits, size_t reserve_bytes) {
  Impl& m = *p_;
  Lane& l = m.lane[0];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  const size_t nbytes = (size_t)((total_bits + 7) / 8);
  const size_t cap = std::max(nbytes, reserve_bytes);
  const size_t np = pieces.size();
  std::vector<EmitDesc> ed(np);
  for (size_t i = 0; i < np; i++) {
    const EmitPiece& p = pieces[i];
    EmitDesc& e = ed[i];
    memset(&e, 0, sizeof(e));
    e.bit_start = p.bit_start;
    e.nbits = p.nbits;
    if (p.type != 0) {
      m.ensure_sym(p.buf);
      e.ll = m.sym_ll[p.buf].as<uint16_t>() + p.off;
      e.d = m.sym_d[p.buf].as<uint16_t>() + p.off;
      e.plan = (const BlockPlan*)(uintptr_t)p.plan;
      e.n = p.n;
    } else {
      if (p.in_start + p.in_len > m.insize) { fprintf(stderr, "zopfli-b200: stored piece outside the input\n"); abort(); }
      e.in_start = p.in_start;
      e.in_len = p.in_len;
    }
    e.type_final = (uint32_t)p.type | ((uint32_t)(p.final ? 1 : 0) << 8);
  }
  m.outbuf.ensure(cap + 64);
  m.emit_desc.ensure(np * sizeof(EmitDesc) + 64);
  m.err_flag.ensure(64);
  l.tic();
  CK(cudaMemsetAsync(m.outbuf.p, 0, nbytes + 64, l.stream));
  CK(cudaMemsetAsync(m.err_flag.p, 0, 64, l.stream));
  uint32_t err = 0;
  if (np) {
    CK(cudaMemcpyAsync(m.emit_desc.p, ed.data(), np * sizeof(EmitDesc), cudaMemcpyHostToDevice, l.stream));
    k_emit<<<(unsigned)np, kEmitThreads, 0, l.stream>>>(m.emit_desc.as<EmitDesc>(), m.d_in, m.outbuf.as<uint32_t>(),
                                                      m.err_flag.as<uint32_t>());
    CK(cudaGetLastError());
    l.acc.launches++;
  }
  CK(cudaMemcpyAsync(&err, m.err_flag.p, 4, cudaMemcpyDeviceToHost, l.stream));
  l.toc(l.acc.ms_pack);
  l.sync();
  if (err) {
    fprintf(stderr, "zopfli-b200: emitted block %u does not match its predicted size (%s)\n", err & 0x3fffffffu,
            (err & 0x80000000u) ? "block" : "tree header");
    abort();
  }
  return m.outbuf.p;
}

void Engine::download(const void* dev_src, uint8_t* host_dst, size_t nbytes) {
  Impl& m = *p_;
  Lane& l = m.lane[0];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  if (nbytes == 0) return;
  m.stager.copy(host_dst, (const uint8_t*)dev_src, nbytes, false, m.dev);
  l.acc.d2h_bytes += nbytes;
}

void Engine::upload(void* dev_dst, const uint8_t* host_src, size_t nbytes) {
  Impl& m = *p_;
  m.stager.copy((uint8_t*)dev_dst, host_src, nbytes, true, m.dev);
  std::lock_guard<std::mutex> g(m.mu);
  m.st_acc.h2d_bytes += nbytes;
}

void Engine::load_symbols(int buf, const uint16_t* ll, const uint16_t* d, size_t n) {
  Impl& m = *p_;
  CK(cudaSetDevice(m.dev));
  if (n > m.insize) { fprintf(stderr, "zopfli-b200: more symbols than input bytes\n"); abort(); }
  m.ensure_sym(buf);
  upload(m.sym_ll[buf].p, (const uint8_t*)ll, n * 2);
  upload(m.sym_d[buf].p, (const uint8_t*)d, n * 2);
}

void Engine::emit(const std::vector<EmitPiece>& pieces, uint64_t total_bits, uint8_t* host_dst) {
  const size_t nbytes = (size_t)((total_bits + 7) / 8);
  if (nbytes == 0) return;
  const void* d = emit_device(pieces, total_bits, 0);
  download(d, host_dst, nbytes);
}

uint8_t* Engine::emit_to_device(const std::vector<EmitPiece>& pieces, uint64_t total_bits, const uint8_t* hdr,
                                int hdr_len, int checksum, void* user_stream, size_t* outsize) {
  const void* body = emit_device(pieces, total_bits, 0);
  Impl& m = *p_;
  Lane& l = m.lane[0];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  const cudaStream_t us = (cudaStream_t)user_stream;
  const size_t nbytes = (size_t)((total_bits + 7) / 8);
  const size_t trailer = checksum == kCkCrc32 ? 8 : (checksum == kCkAdler32 ? 4 : 0);
  const size_t total = (size_t)hdr_len + nbytes + trailer;
  uint8_t* out = nullptr;
  CK(cudaMallocAsync((void**)&out, total, us));
  CK(cudaEventRecord(m.ev_user, us));  // the allocation exists before lane 0 writes into it
  CK(cudaStreamWaitEvent(l.stream, m.ev_user, 0));
  if (nbytes) CK(cudaMemcpyAsync(out + hdr_len, body, nbytes, cudaMemcpyDeviceToDevice, l.stream));
  if (hdr_len || trailer) {
    if (checksum != kCkNone) CK(cudaStreamWaitEvent(l.stream, m.ev_ck, 0));
    ContainerArgs a;
    memset(&a, 0, sizeof(a));
    a.out = out;
    a.body_bytes = nbytes;
    a.isize = m.insize;
    a.acc = m.ck_acc.as<ChecksumAcc>();
    a.tab = Impl::crc_tab();
    memcpy(a.hdr, hdr, (size_t)hdr_len);
    a.hdr_len = (uint32_t)hdr_len;
    a.kind = checksum;
    k_container<<<1, 32, 0, l.stream>>>(a);
    CK(cudaGetLastError());
    l.acc.launches++;
  }
  CK(cudaEventRecord(m.ev_lane0, l.stream));
  CK(cudaStreamWaitEvent(us, m.ev_lane0, 0));
  l.sync();
  *outsize = total;
  return out;
}

uint64_t Engine::device_block_bits(const uint32_t* hist320) {
  Impl& m = *p_;
  Lane& l = m.lane[0];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  l.misc.ensure(320 * 4 + 64);
  Batch b;
  memset(&b, 0, sizeof(b));
  CK(cudaMemcpyAsync(l.misc.p, hist320, 320 * 4, cudaMemcpyHostToDevice, l.stream));
  uint64_t* dout = (uint64_t*)((uint8_t*)l.misc.p + 320 * 4 + 16);
  k_test_block_bits<<<1, 32, 0, l.stream>>>(b, l.misc.as<uint32_t>(), dout);
  CK(cudaGetLastError());
  uint64_t r = 0;
  CK(cudaMemcpyAsync(&r, dout, 8, cudaMemcpyDeviceToHost, l.stream));
  l.sync();
  return r;
}

void Engine::device_probe_parts(const uint32_t* hists, size_t n, uint32_t* smoothed, uint8_t* lengths,
                                uint32_t* tree_bits, uint64_t* dyn) {
  if (n == 0) return;
  Impl& m = *p_;
  Lane& l = m.lane[0];
  std::lock_guard<std::mutex> g(l.mu);
  CK(cudaSetDevice(m.dev));
  const size_t in_b = n * 320 * 4, sm_b = n * 320 * 4, len_b = n * 640, tb_b = n * 16 * 4, dyn_b = n * 8;
  l.misc.ensure(dyn_b + in_b + sm_b + tb_b + len_b);
  uint8_t* base = (uint8_t*)l.misc.p;   // 8-byte fields first, bytes last
  uint64_t* d_dyn = (uint64_t*)base;
  uint32_t* d_in = (uint32_t*)(base + dyn_b);
  uint32_t* d_sm = (uint32_t*)(base + dyn_b + in_b);
  uint32_t* d_tb = (uint32_t*)(base + dyn_b + in_b + sm_b);
  uint8_t* d_len = base + dyn_b + in_b + sm_b + tb_b;
  CK(cudaMemcpyAsync(d_in, hists, in_b, cudaMemcpyHostToDevice, l.stream));
  k_test_probe_parts<<<(unsigned)n, 32, 0, l.stream>>>(d_in, d_sm, d_len, d_tb, d_dyn);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(smoothed, d_sm, sm_b, cudaMemcpyDeviceToHost, l.stream));
  CK(cudaMemcpyAsync(lengths, d_len, len_b, cudaMemcpyDeviceToHost, l.stream));
  CK(cudaMemcpyAsync(tree_bits, d_tb, tb_b, cudaMemcpyDeviceToHost, l.stream));
  CK(cudaMemcpyAsync(dyn, d_dyn, dyn_b, cudaMemcpyDeviceToHost, l.stream));
  l.sync();
}

namespace {
struct OnDevice {  // makes dev current for a scope, then restores the caller's device
  int prev = 0;
  explicit OnDevice(int dev) { CK(cudaGetDevice(&prev)); CK(cudaSetDevice(dev)); }
  ~OnDevice() { cudaSetDevice(prev); }
};
}  // namespace

DeviceStaging::DeviceStaging(int dev) : dev_(dev), stream_(nullptr), ev_(nullptr) {
  OnDevice on(dev);
  cudaStream_t s;
  cudaEvent_t e;
  CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  stream_ = s;
  ev_ = e;
}

DeviceStaging::~DeviceStaging() {
  OnDevice on(dev_);
  CK(cudaStreamSynchronize((cudaStream_t)stream_));
  CK(cudaEventDestroy((cudaEvent_t)ev_));
  CK(cudaStreamDestroy((cudaStream_t)stream_));
}

void* DeviceStaging::alloc(size_t bytes) {
  OnDevice on(dev_);
  void* p = nullptr;
  CK(cudaMallocAsync(&p, bytes, (cudaStream_t)stream_));
  return p;
}

void DeviceStaging::release(void* p) {
  if (!p) return;
  OnDevice on(dev_);
  CK(cudaFreeAsync(p, (cudaStream_t)stream_));
}

void DeviceStaging::copy(void* dst, const void* src, size_t n, void* user_stream) {
  OnDevice on(dev_);
  cudaStream_t s = (cudaStream_t)stream_;
  if (user_stream != stream_) {  // the stream is non-blocking: it orders against the caller's only through an event
    CK(cudaEventRecord((cudaEvent_t)ev_, (cudaStream_t)user_stream));
    CK(cudaStreamWaitEvent(s, (cudaEvent_t)ev_, 0));
  }
  if (n) CK(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, s));
  CK(cudaStreamSynchronize(s));
}

void DeviceStaging::zero(void* dst, size_t n) {
  OnDevice on(dev_);
  CK(cudaMemsetAsync(dst, 0, n, (cudaStream_t)stream_));
  CK(cudaStreamSynchronize((cudaStream_t)stream_));
}

}  // namespace zb

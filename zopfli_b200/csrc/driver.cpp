// Host driver behind ZopfliDeflate / ZopfliDeflatePart (drop-in boundary, SURVEY 8(b)).
//
// The reference (deflate.c:811-931) runs one master block at a time, one block at a time.  Here every
// stage is batched over many master blocks so the GPU sees every independent unit at once (SURVEY 7.2 #5,
// 8(e)).  The master blocks of a call are cut into up to four chunk pipelines, each on its own host thread
// and its own pair of engine lanes, running (DESIGN.md §1):
//
//   stage A  GPU       greedy parse of every master block; the stores stay on the device and become the
//                      stores of the split service                            (blocksplitter.c:288-296)
//   stage B  GPU+host  split search: costs priced on the device, the decisions replayed on the host
//                      (batched_split.hpp)                          (blocksplitter.c:43-128, 195-273)
//   stage C  GPU       optimal parse of every block; giant blocks on the even lane, the rest on the odd
//                                                                                (deflate.c:854-869)
//   stage D  GPU+host  block stores concatenated and priced, second split attempt, block-type choice
//                                                                      (deflate.c:872-893, 747-800)
//   stage E  GPU       fixed-tree re-parses requested by stage D                  (deflate.c:771-781)
//
// then once per call (assemble): prefix sum over the exact block sizes, one emission launch, one copy.
#include "driver.hpp"

#include <sched.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <mutex>
#include <thread>

#include "batched_split.hpp"
#include "emit_bits.hpp"
#include "engine.hpp"

namespace zb {

HostTimes g_host_times;

double now_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

bool debug_on() {
  static int v = [] { const char* e = getenv("ZOPFLI_B200_DEBUG"); return e && atoi(e) ? 1 : 0; }();
  return v != 0;
}

namespace {

std::mutex g_time_mu;
void add_time(double& acc, double ms) {
  std::lock_guard<std::mutex> g(g_time_mu);
  acc += ms;
}

double g_debug_t0 = 0;
void debug_mark(int chunk, const char* what) {
  if (debug_on()) fprintf(stderr, "[zb] %8.1f ms  chunk %d  %s\n", now_ms() - g_debug_t0, chunk, what);
}

// CPUs this process may actually use: affinity mask, capped by the cgroup CPU quota (v2 cpu.max or
// v1 cfs_quota_us / cfs_period_us) -- a container on a 128-thread host is often limited to a few cores
int usable_cpus() {
  int n = (int)std::thread::hardware_concurrency();
  cpu_set_t set;
  if (sched_getaffinity(0, sizeof(set), &set) == 0) n = std::min(n > 0 ? n : 1 << 20, CPU_COUNT(&set));
  double quota = -1, period = -1;
  if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
    char q[64];
    if (fscanf(f, "%63s %lf", q, &period) == 2 && strcmp(q, "max") != 0) quota = atof(q);
    fclose(f);
  } else {
    if (FILE* g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) { if (fscanf(g, "%lf", &quota) != 1) quota = -1; fclose(g); }
    if (FILE* g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) { if (fscanf(g, "%lf", &period) != 1) period = -1; fclose(g); }
  }
  if (quota > 0 && period > 0) n = std::min(n, (int)(quota / period + 0.999));
  return n < 1 ? 1 : n;
}

}  // namespace

int host_threads() {
  static int n = [] {
    if (const char* e = getenv("ZOPFLI_B200_THREADS")) { int v = atoi(e); return v < 1 ? 1 : (v > 256 ? 256 : v); }
    int v = std::min(usable_cpus(), 32);
    // one process per GPU (torchrun): the ranks of a box share its cores
    if (const char* w = getenv("LOCAL_WORLD_SIZE")) { int k = atoi(w); if (k > 1) v = std::max(2, v / k); }
    return v < 1 ? 1 : v;
  }();
  return n;
}

namespace {

// What the stages learn of one master block: A-B its cuts, C the size of every block's parse, D-E its pieces.
struct Master {
  size_t ms, me;                       // byte range
  size_t floor;                        // the unit's floor: no parse of the master block sees a byte before it
  std::vector<size_t> cuts;            // block boundaries in bytes (ms, ..., me): the first split, or the second if it wins
  std::vector<uint32_t> bsize;         // symbols of every first-split block's optimal parse
  std::vector<Piece> pieces;
};
using BlockRef = std::pair<size_t, size_t>;  // (master block, block index)

// A master block in stage D: its blocks' stores concatenated in kFin
struct Joined {
  uint64_t off = 0, total = 0;         // first symbol in kFin (= byte offset of the master block) and symbol count
  std::vector<size_t> points;          // block boundaries in symbols: the first split, or the second if it wins
  std::vector<Engine::PlanCost> cost;  // sizes of every block
  std::vector<uint64_t> plan;          // Engine::plan_blocks handle of every block
  uint64_t bits = 0;                   // AutoType size of the first split's blocks, summed
  bool split2 = false;                 // the second split is attempted (deflate.c:872)
};

// A block of the final split, as AddLZ77BlockAutoType (deflate.c:747-800) weighs it
struct FinalBlock {
  size_t a, b;               // byte range (absolute input positions)
  uint64_t off;              // first symbol in kFin
  uint32_t n;                // symbols
  Engine::PlanCost c;
  uint64_t plan;
  int fixed_req = -1;        // index into the fixed re-parse batch
};
// the fixed-tree re-parse of a block (deflate.c:771-781): its symbols in kFix and their size
struct FixedParse { uint64_t off; uint32_t n; uint64_t bits; };

// PrintBlockSplitPoints (blocksplitter.c:148-180): byte offsets of the split points from the start of the
// store that was split (the master block), decimal then hex
void print_split_points(const std::vector<size_t>& cuts, size_t origin) {
  std::lock_guard<std::mutex> g(g_time_mu);  // chunk pipelines print concurrently: keep lines whole
  fprintf(stderr, "block split points: ");
  for (size_t c = 1; c + 1 < cuts.size(); c++) fprintf(stderr, "%d ", (int)(cuts[c] - origin));
  fprintf(stderr, "(hex:");
  for (size_t c = 1; c + 1 < cuts.size(); c++) fprintf(stderr, " %x", (int)(cuts[c] - origin));
  fprintf(stderr, ")\n");
}

// ZopfliCalculateBlockSizeAutoType (deflate.c:610-621) from the three sizes; `store_size` is the symbol
// count of the store the range belongs to (the reference tests lz77->size, SURVEY App. A.9)
uint64_t auto_type(const Engine::PlanCost& c, size_t store_size) {
  const uint64_t fixed = store_size > 1000 ? c.unc : c.fixed;
  return (c.unc < fixed && c.unc < c.dyn) ? c.unc : (fixed < c.dyn ? fixed : c.dyn);
}

// AddLZ77BlockAutoType (deflate.c:747-800): the cheapest of stored, fixed and dynamic.  `fx` is the
// block's fixed-tree re-parse, or null where none was asked for.
Piece choose_block_type(const FinalBlock& fb, const FixedParse* fx) {
  Piece p;
  p.instart = fb.a;
  p.inend = fb.b;
  if (fb.n == 0) {  // deflate.c:763-768: the smallest empty block is a fixed one
    p.type = 1;
    p.nbits = 10;
    return p;
  }
  const uint64_t fixedcost = fx ? fx->bits : fb.c.fixed;  // deflate.c:779
  if (fb.c.unc < fixedcost && fb.c.unc < fb.c.dyn) {  // deflate.c:783-785
    p.type = 0;
  } else if (fixedcost < fb.c.dyn) {
    p.type = 1;
    p.nbits = fixedcost;
    p.buf = fx ? Engine::kFix : Engine::kFin;
    p.off = fx ? fx->off : fb.off;
    p.n = fx ? fx->n : fb.n;
  } else {
    p.type = 2;
    p.nbits = fb.c.dyn;
    p.tree_bits = (uint32_t)fb.c.tree;
    p.buf = Engine::kFin;
    p.off = fb.off;
    p.n = fb.n;
    p.plan = fb.plan;
  }
  return p;
}

// The engine's parse range of input bytes [a, b) whose unit has floor `floor` (absolute positions; the engine
// holds the bytes from in_base on, so a floor below in_base is no floor for it)
ParseRange parse_range(size_t a, size_t b, size_t in_base, size_t floor, int mode, int numiterations) {
  return {a - in_base, b - in_base, mode, numiterations, floor > in_base ? floor - in_base : 0};
}

// btype 0 (deflate.c:826-828): every unit one stored piece
void deflate_stored(const std::vector<Unit>& units, bool final_last, std::vector<Piece>& pieces) {
  for (size_t m = 0; m < units.size(); m++) {
    Piece p;
    p.type = 0;
    p.instart = units[m].a;
    p.inend = units[m].b;
    p.final = final_last && m + 1 == units.size();
    p.unit = (uint32_t)m;
    pieces.push_back(p);
  }
}

// btype 1 (deflate.c:829-841): one fixed-tree optimal parse per unit
void deflate_fixed(Engine& eng, const std::vector<Unit>& units, size_t in_base, bool final_last,
                   std::vector<Piece>& pieces) {
  const size_t nm = units.size();
  std::vector<ParseRange> pr;
  for (const Unit& u : units) pr.push_back(parse_range(u.a, u.b, in_base, u.floor, 2, 0));
  std::vector<uint32_t> sizes;
  std::vector<uint64_t> costs;
  eng.parse_keep(pr, Engine::kFix, sizes, costs, 0);
  std::vector<Engine::PlanReq> rq;
  for (size_t m = 0; m < nm; m++) rq.push_back({pr[m].instart, sizes[m], (uint32_t)Engine::kFix});
  std::vector<Engine::PlanCost> pc;
  std::vector<uint64_t> ph;
  eng.plan_blocks(rq, pc, ph, 0);
  for (size_t m = 0; m < nm; m++) {
    Piece p;
    p.type = 1;
    p.buf = Engine::kFix;
    p.off = pr[m].instart;
    p.n = sizes[m];
    p.nbits = pc[m].fixed;
    p.instart = units[m].a;
    p.inend = units[m].b;
    p.final = final_last && m + 1 == nm;
    p.unit = (uint32_t)m;
    pieces.push_back(p);
  }
}

// How a call's master blocks run: as `nchunks` chunk pipelines, each taking its master blocks in batches
// of at most `batch`, with the blocks of `giant` bytes or more parsed on their own lane.
struct Schedule { size_t nchunks, batch; uint64_t giant; };
Schedule schedule(size_t nm, uint64_t device_memory) {
  Schedule s;
  s.nchunks = 4;
  if (const char* e = getenv("ZOPFLI_B200_CHUNKS")) s.nchunks = (size_t)atoi(e);
  s.nchunks = std::max<size_t>(1, std::min<size_t>(std::min<size_t>(s.nchunks, Engine::kLanes / 2), nm / 4));
  if (nm < 8) s.nchunks = 1;
  if (const char* e = getenv("ZOPFLI_B200_FORCE_CHUNKS")) s.nchunks = std::min<size_t>((size_t)atoi(e), std::min<size_t>(nm, Engine::kLanes / 2));  // tests
  if (s.nchunks < 1) s.nchunks = 1;
  // A pipeline takes its master blocks in batches because the lane arenas cost ~140 MB per master
  // block in flight (~100 B per parse position + ~22 B per key position, two lanes).  The batch is as
  // large as a quarter of the device memory allows (180 GB: ~80 master blocks per pipeline), so the
  // 100 MB bench and a 134 MB shard of the 1 GiB config run as ONE wave per pipeline -- every extra
  // wave costs a whole A + B + longest-chain latency -- and the batches of a longer input are balanced.
  s.batch = std::max<size_t>(8, (size_t)(device_memory / 4 / ((uint64_t)s.nchunks * 140000000ull)));
  if (const char* e = getenv("ZOPFLI_B200_BATCH")) s.batch = std::max<size_t>(1, (size_t)atoi(e));
  s.giant = 250000;
  if (const char* e = getenv("ZOPFLI_B200_GIANT")) s.giant = strtoull(e, nullptr, 10);  // tests: force the two-lane path
  return s;
}

}  // namespace

// A call with master blocks for every pipeline runs nchunks x batch of them at once: one wave of a call on a
// device with this much memory.
size_t wave_master_blocks(uint64_t device_memory) {
  const Schedule s = schedule(SIZE_MAX, device_memory);
  return s.nchunks * s.batch;
}

namespace {

// One deflate_units call with btype 2: the engine, its options, and the master blocks.  Every stage
// below names the fields of Master it fills; the chunk pipelines work on disjoint master blocks.
struct Call {
  Engine& eng;
  const ZopfliOptions* opt;
  size_t in_base;   // absolute position of engine byte 0
  bool final_last;
  uint64_t giant;
  std::vector<Master> M;

  // Stages A and B for the master blocks cm, on `lane`: their first-split cuts (M[m].cuts)
  void first_split(const std::vector<size_t>& cm, int lane, int cid) {
    if (!opt->blocksplitting) {
      for (size_t m : cm) M[m].cuts = {M[m].ms, M[m].me};
      return;
    }
    const double t0 = now_ms();
    // ---- stage A: greedy parse of every master block (blocksplitter.c:288-296).  The greedy stores
    // never leave the device: they become the stores of the split service, and only the byte positions
    // of the chosen split points come back (blocksplitter.c:303-313)
    std::vector<ParseRange> pr;
    for (size_t m : cm) pr.push_back(parse_range(M[m].ms, M[m].me, in_base, M[m].floor, 0, 0));
    std::vector<uint32_t> gsize;
    eng.greedy_to_split(pr, gsize, lane);
    const double t1 = now_ms();
    debug_mark(cid, "A greedy done");
    add_time(g_host_times.other, t1 - t0);
    // ---- stage B: split search (costs on the device, decisions on the host) ----
    std::vector<size_t> sizes(gsize.begin(), gsize.end());
    std::vector<std::vector<size_t>> lps =
        batched_block_split(sizes, (size_t)opt->blocksplittingmax, [&](const std::vector<EvalReq>& r, std::vector<uint64_t>& c) {
          eng.split_eval(reinterpret_cast<const Engine::SplitReq*>(r.data()), r.size(), c.data(), lane);
        });
    std::vector<Engine::SplitPos> want;
    for (size_t q = 0; q < cm.size(); q++)
      for (size_t p : lps[q]) want.push_back({(uint32_t)q, (uint32_t)p});
    std::vector<uint32_t> bytepos;
    eng.split_positions(want, bytepos, lane);
    size_t w = 0;
    for (size_t q = 0; q < cm.size(); q++) {
      Master& mb = M[cm[q]];
      mb.cuts.push_back(mb.ms);
      for (size_t k = 0; k < lps[q].size(); k++) mb.cuts.push_back(mb.ms + bytepos[w++]);
      mb.cuts.push_back(mb.me);
      if (opt->verbose) print_split_points(mb.cuts, mb.ms);
    }
    debug_mark(cid, "B split done");
    add_time(g_host_times.split, now_ms() - t1);
  }

  // Stage C (deflate.c:854-869) on `lane`: the optimal parse of the given blocks, kept on the device
  // (kPack); the symbol count of each goes to M[m].bsize
  void parse_blocks(const std::vector<BlockRef>& blocks, int lane) {
    std::vector<ParseRange> pr;
    for (const BlockRef& k : blocks) {
      const std::vector<size_t>& cuts = M[k.first].cuts;
      pr.push_back(parse_range(cuts[k.second], cuts[k.second + 1], in_base, M[k.first].floor, 1, opt->numiterations));
    }
    const bool want_iters = opt->verbose || opt->verbose_more;
    std::vector<uint32_t> sizes;
    std::vector<uint64_t> costs, itc;
    eng.parse_keep(pr, Engine::kPack, sizes, costs, lane, want_iters ? &itc : nullptr);
    for (size_t q = 0; q < blocks.size(); q++) M[blocks[q].first].bsize[blocks[q].second] = sizes[q];
    if (want_iters && !itc.empty()) {  // squeeze.c:493-495, block after block
      std::lock_guard<std::mutex> g(g_time_mu);
      const size_t stride = itc.size() / blocks.size();
      for (size_t q = 0; q < blocks.size(); q++) {
        uint64_t best = ~(uint64_t)0;
        for (size_t i = 0; i < stride && i < (size_t)opt->numiterations; i++) {
          const uint64_t c = itc[q * stride + i];
          if (c == ~(uint64_t)0) break;
          if (opt->verbose_more || c < best) fprintf(stderr, "Iteration %d: %d bit\n", (int)i, (int)c);
          if (c < best) best = c;
        }
      }
    }
  }

  // Stage D, first part, on `lane`: the block stores of every master block of ms concatenated in kFin
  // (ZopfliAppendLZ77Store, deflate.c:863) and the sizes of the first split's blocks (deflate.c:862:
  // AutoType over each block's own store)
  std::vector<Joined> join_blocks(const std::vector<size_t>& ms, int lane) {
    std::vector<Joined> J(ms.size());
    std::vector<Engine::SymCopy> copies;
    std::vector<Engine::PlanReq> rq;
    std::vector<uint64_t> soff;
    std::vector<uint32_t> ssize;
    for (size_t q = 0; q < ms.size(); q++) {
      const Master& mb = M[ms[q]];
      Joined& j = J[q];
      j.off = mb.ms - in_base;
      for (size_t i = 0; i < mb.bsize.size(); i++) {
        copies.push_back({mb.cuts[i] - in_base, j.off + j.total, mb.bsize[i], 0});
        rq.push_back({j.off + j.total, mb.bsize[i], (uint32_t)Engine::kFin});
        j.total += mb.bsize[i];
        if (i + 1 < mb.bsize.size()) j.points.push_back((size_t)j.total);
      }
      j.split2 = opt->blocksplitting && j.points.size() > 1;
      if (j.split2) { soff.push_back(j.off); ssize.push_back((uint32_t)j.total); }
    }
    eng.concat_stores(copies, soff, ssize, lane);
    std::vector<Engine::PlanCost> c;
    std::vector<uint64_t> h;
    eng.plan_blocks(rq, c, h, lane);
    for (size_t q = 0, k = 0; q < ms.size(); q++)
      for (size_t i = 0; i < M[ms[q]].bsize.size(); i++, k++) {
        J[q].cost.push_back(c[k]);
        J[q].plan.push_back(h[k]);
        J[q].bits += auto_type(c[k], M[ms[q]].bsize[i]);
      }
    return J;
  }

  // Stage D, second part (deflate.c:872-893): the second split attempt on the concatenated stores.  Where
  // it wins, J[q] takes its points and sizes and M[ms[q]].cuts its byte boundaries.
  void second_split(const std::vector<size_t>& ms, std::vector<Joined>& J, int lane) {
    std::vector<size_t> who, sizes;
    for (size_t q = 0; q < ms.size(); q++)
      if (J[q].split2) { who.push_back(q); sizes.push_back((size_t)J[q].total); }
    if (who.empty()) return;
    std::vector<std::vector<size_t>> r =
        batched_block_split(sizes, (size_t)opt->blocksplittingmax, [&](const std::vector<EvalReq>& rr, std::vector<uint64_t>& c) {
          eng.split_eval(reinterpret_cast<const Engine::SplitReq*>(rr.data()), rr.size(), c.data(), lane);
        });
    std::vector<Engine::PlanReq> rq;
    std::vector<size_t> rq_base(who.size());
    for (size_t k = 0; k < who.size(); k++) {
      const Joined& j = J[who[k]];
      rq_base[k] = rq.size();
      for (size_t i = 0; i <= r[k].size(); i++) {
        const size_t a = i == 0 ? 0 : r[k][i - 1], b = i == r[k].size() ? (size_t)j.total : r[k][i];
        rq.push_back({j.off + a, (uint32_t)(b - a), (uint32_t)Engine::kFin});
      }
    }
    std::vector<Engine::PlanCost> c;
    std::vector<uint64_t> h;
    eng.plan_blocks(rq, c, h, lane);
    std::vector<Engine::SplitPos> want;
    std::vector<size_t> want_base(who.size());
    std::vector<char> use(who.size());
    for (size_t k = 0; k < who.size(); k++) {
      uint64_t bits = 0;
      for (size_t i = 0; i <= r[k].size(); i++) bits += auto_type(c[rq_base[k] + i], (size_t)J[who[k]].total);
      use[k] = bits < J[who[k]].bits;
      want_base[k] = want.size();
      if (use[k] || opt->verbose)
        for (size_t p : r[k]) want.push_back({(uint32_t)k, (uint32_t)p});
    }
    // byte positions of the adopted second-pass split points (lz77->pos, deflate.c:769)
    std::vector<uint32_t> bytepos;
    eng.split_positions(want, bytepos, lane);
    for (size_t k = 0; k < who.size(); k++) {
      if (!use[k] && !opt->verbose) continue;
      Master& mb = M[ms[who[k]]];
      std::vector<size_t> cuts2(1, mb.ms);
      for (size_t i = 0; i < r[k].size(); i++) cuts2.push_back(mb.ms + bytepos[want_base[k] + i]);
      cuts2.push_back(mb.me);
      if (opt->verbose) print_split_points(cuts2, mb.ms);  // ZopfliBlockSplitLZ77 reports its points whether or not they win
      if (!use[k]) continue;
      Joined& j = J[who[k]];
      mb.cuts.swap(cuts2);
      j.points = r[k];
      j.cost.assign(c.begin() + rq_base[k], c.begin() + rq_base[k] + r[k].size() + 1);
      j.plan.assign(h.begin() + rq_base[k], h.begin() + rq_base[k] + r[k].size() + 1);
    }
  }

  // Stage D, third part, and stage E: the final blocks of every master block of ms, the fixed-tree
  // re-parses they ask for (deflate.c:760, 771-781) and their types (M[m].pieces)
  void choose_blocks(const std::vector<size_t>& ms, const std::vector<Joined>& J, int lane) {
    std::vector<std::vector<FinalBlock>> finals(ms.size());
    std::vector<ParseRange> prf;
    for (size_t q = 0; q < ms.size(); q++) {
      const Joined& j = J[q];
      for (size_t i = 0; i <= j.points.size(); i++) {
        const size_t ls = i == 0 ? 0 : j.points[i - 1], le = i == j.points.size() ? (size_t)j.total : j.points[i];
        FinalBlock fb{M[ms[q]].cuts[i], M[ms[q]].cuts[i + 1], j.off + ls, (uint32_t)(le - ls), j.cost[i], j.plan[i]};
        if (le > ls && (j.total < 1000 || (double)fb.c.fixed <= (double)fb.c.dyn * 1.1)) {  // deflate.c:760
          fb.fixed_req = (int)prf.size();
          prf.push_back(parse_range(fb.a, fb.b, in_base, M[ms[q]].floor, 2, 0));
        }
        finals[q].push_back(fb);
      }
    }
    std::vector<FixedParse> fixed;
    if (!prf.empty()) {
      std::vector<uint32_t> fsize;
      std::vector<uint64_t> fcost, h;
      eng.parse_keep(prf, Engine::kFix, fsize, fcost, lane);
      std::vector<Engine::PlanReq> rq;
      for (size_t g = 0; g < prf.size(); g++) rq.push_back({prf[g].instart, fsize[g], (uint32_t)Engine::kFix});
      std::vector<Engine::PlanCost> c;
      eng.plan_blocks(rq, c, h, lane);
      for (size_t g = 0; g < prf.size(); g++) fixed.push_back({prf[g].instart, fsize[g], c[g].fixed});
    }
    for (size_t q = 0; q < ms.size(); q++)
      for (size_t i = 0; i < finals[q].size(); i++) {
        const FinalBlock& fb = finals[q][i];
        Piece p = choose_block_type(fb, fb.fixed_req >= 0 ? &fixed[fb.fixed_req] : nullptr);
        p.final = final_last && ms[q] + 1 == M.size() && i + 1 == finals[q].size();
        p.unit = (uint32_t)ms[q];
        M[ms[q]].pieces.push_back(p);
      }
  }

  // Stages D-E on `lane` for master blocks whose blocks are all parsed.  Works on sizes only; every
  // store stays on the device.
  void finish(const std::vector<size_t>& ms, int lane) {
    if (ms.empty()) return;
    const double t0 = now_ms();
    std::vector<Joined> J = join_blocks(ms, lane);
    second_split(ms, J, lane);
    const double t1 = now_ms();
    add_time(g_host_times.split, t1 - t0);
    choose_blocks(ms, J, lane);
    add_time(g_host_times.other, now_ms() - t1);
  }

  // D-E of the master blocks with a giant block, once the giants' parse (thread `giants`) is done
  void finish_dirty(std::thread& giants, const std::vector<size_t>& dirty, int lane, int cid) {
    const double tw = now_ms();
    giants.join();
    debug_mark(cid, "C giants parsed");
    add_time(g_host_times.other, now_ms() - tw);
    finish(dirty, lane);  // the giants' lane is idle now and has stream priority
    debug_mark(cid, "D-E dirty done");
  }

  // Stages A-E of one batch of a chunk pipeline.  A, B and the giants' parse run on lane_g, the even lane,
  // which has stream priority: they sit on the critical path.
  void run_chunk(const std::vector<size_t>& cm, int lane_g, int lane_r) {
    const int cid = lane_g / 2;
    debug_mark(cid, "start");
    first_split(cm, lane_g, cid);
    const double t0 = now_ms();
    // The critical path of stage C is the DP chain of the largest blocks.  Giant blocks go to the even
    // lane on their own (their tables are ready within milliseconds, so their iterate kernel starts at
    // once); everything else is prepared and parsed on the odd lane meanwhile.
    std::vector<BlockRef> giants, rest;
    for (size_t m : cm) {
      const std::vector<size_t>& cuts = M[m].cuts;
      M[m].bsize.assign(cuts.size() - 1, 0);
      for (size_t i = 0; i + 1 < cuts.size(); i++) (cuts[i + 1] - cuts[i] >= giant ? giants : rest).push_back({m, i});
    }
    if (giants.empty() || rest.empty()) {
      parse_blocks(giants.empty() ? rest : giants, lane_g);
      add_time(g_host_times.other, now_ms() - t0);
      finish(cm, lane_r);
      return;
    }
    std::vector<char> has_giant(M.size(), 0);
    for (const BlockRef& k : giants) has_giant[k.first] = 1;
    std::vector<size_t> clean, dirty;
    for (size_t m : cm) (has_giant[m] ? dirty : clean).push_back(m);
    std::thread tg([&] { parse_blocks(giants, lane_g); });
    parse_blocks(rest, lane_r);
    debug_mark(cid, "C rest parsed");
    add_time(g_host_times.other, now_ms() - t0);
    // A master block with a giant also has blocks on lane_r, so its D-E waits for both lanes.  The
    // clean and the dirty D-E then run side by side, each on its own lane: their second split searches
    // are chains of short, latency-bound rounds that leave most of the GPU idle, and when the giants end
    // before the rest the dirty D-E no longer queues behind the clean one.  With verbose output the two
    // run in turn, so the split-point reports keep their order (clean master blocks first).
    const bool in_turn = opt->verbose || opt->verbose_more;
    std::thread td;
    if (!in_turn) td = std::thread([&] { finish_dirty(tg, dirty, lane_g, cid); });
    finish(clean, lane_r);  // overlaps the giants' DP chains still running on lane_g
    debug_mark(cid, "D-E clean done");
    if (in_turn) finish_dirty(tg, dirty, lane_g, cid);
    else td.join();
  }

  // Chunk pipeline c: its master blocks in balanced batches of at most `batch`, on lanes 2c and 2c + 1
  void run_pipeline(const std::vector<size_t>& all, size_t batch, int c) {
    const size_t nbatches = (all.size() + batch - 1) / batch;
    const size_t per = nbatches ? (all.size() + nbatches - 1) / nbatches : 0;
    for (size_t a = 0; a < all.size(); a += per) {
      std::vector<size_t> part(all.begin() + a, all.begin() + std::min(all.size(), a + per));
      run_chunk(part, 2 * c, 2 * c + 1);
    }
  }
};

}  // namespace

void deflate_units(Engine& eng, const ZopfliOptions* opt, int btype, bool final_last, const std::vector<Unit>& units,
                   size_t in_base, std::vector<Piece>& pieces) {
  if (btype == 0) {
    deflate_stored(units, final_last, pieces);
    return;
  }
  if (btype == 1) {
    deflate_fixed(eng, units, in_base, final_last, pieces);
    return;
  }
  // The master blocks are processed as a few independent chunk pipelines (stages A-E each), one
  // host thread and one pair of engine lanes per chunk: while one chunk's split search waits on
  // round trips or its longest DP chain is still running, the others keep the GPU busy.
  g_debug_t0 = now_ms();
  const size_t nm = units.size();
  const Schedule s = schedule(nm, eng.device_memory_total());
  Call call{eng, opt, in_base, final_last, s.giant, std::vector<Master>(nm)};
  for (size_t m = 0; m < nm; m++) {
    call.M[m].ms = units[m].a;
    call.M[m].me = units[m].b;
    call.M[m].floor = units[m].floor;
  }
  std::vector<std::vector<size_t>> chunks(s.nchunks);
  for (size_t m = 0; m < nm; m++) chunks[m * s.nchunks / nm].push_back(m);
  std::vector<std::thread> th;
  for (size_t c = 1; c < s.nchunks; c++) th.emplace_back([&, c] { call.run_pipeline(chunks[c], s.batch, (int)c); });
  call.run_pipeline(chunks[0], s.batch, 0);
  for (auto& t : th) t.join();
  for (const Master& mb : call.M) pieces.insert(pieces.end(), mb.pieces.begin(), mb.pieces.end());
}

// ---------------------------------------------------------------------------------------------
// assemble: prefix sum over the exact piece sizes -> one emission launch -> the stream lands in the
// caller's zopfli-style buffer (util.h:134-155 capacity rule)

namespace {
size_t pow2_ceil(size_t v) {
  size_t p = 1;
  while (p < v) p <<= 1;
  return p;
}
}  // namespace

uint64_t layout_pieces(const std::vector<Piece>& pieces, size_t in_base, uint64_t bit0, std::vector<Engine::EmitPiece>& ep,
                       std::vector<uint64_t>* unit_bits) {
  uint64_t pos = bit0;
  ep.resize(pieces.size());
  if (unit_bits) unit_bits->clear();
  for (size_t i = 0; i < pieces.size(); i++) {
    const Piece& p = pieces[i];
    Engine::EmitPiece& e = ep[i];
    memset(&e, 0, sizeof(e));
    if (unit_bits && (i == 0 || p.unit != pieces[i - 1].unit)) unit_bits->push_back(pos - bit0);
    e.bit_start = pos;
    e.type = p.type;
    e.final = p.final ? 1 : 0;
    if (p.type == 0) {
      e.in_start = p.instart - in_base;
      e.in_len = p.inend - p.instart;
      pos = stored_end(pos, e.in_len);
    } else {
      e.nbits = p.nbits;
      e.off = p.off;
      e.n = p.n;
      e.buf = p.buf;
      e.plan = p.plan;
      pos += p.nbits;
    }
  }
  if (unit_bits) unit_bits->push_back(pos - bit0);
  return pos;
}

uint64_t place_pieces(const std::vector<Piece>& pieces, size_t in_base, unsigned phase, std::vector<Engine::EmitPiece>& ep,
                      std::vector<uint64_t>* unit_bits, bool verbose) {
  const uint64_t total = layout_pieces(pieces, in_base, phase, ep, unit_bits);
  if (verbose) {  // AddLZ77Block's reports (deflate.c:718-744): growth of *outsize (= bytes touched so far) per part
    for (size_t i = 0; i < pieces.size(); i++) {
      const Piece& p = pieces[i];
      if (p.type == 0 || p.n == 0) continue;  // stored blocks return before the report (deflate.c:696-702); empty blocks never get there
      const uint64_t h = ep[i].bit_start + 3, t = h + p.tree_bits, e = ep[i].bit_start + ep[i].nbits;
      if (p.type == 2) fprintf(stderr, "treesize: %d\n", (int)((t + 7) / 8 - (h + 7) / 8));
      const size_t grown = (size_t)((e + 7) / 8 - (t + 7) / 8);
      fprintf(stderr, "compressed block size: %d (%dk) (unc: %d)\n", (int)grown, (int)(grown / 1024), (int)(p.inend - p.instart));
    }
  }
  return total;
}

void assemble(Engine& eng, const std::vector<Piece>& pieces, size_t in_base, unsigned char* bp, unsigned char** out,
              size_t* outsize, std::vector<uint64_t>* unit_bits, bool verbose) {
  const unsigned phase = (*outsize > 0) ? (*bp & 7u) : 0u;  // bits in use in the last byte (deflate.h:50-53)
  std::vector<Engine::EmitPiece> ep;
  const uint64_t total = place_pieces(pieces, in_base, phase, ep, unit_bits, verbose);
  const size_t nbytes = (size_t)((total + 7) / 8);
  if (nbytes == 0) return;
  append_stream(nbytes, phase, out, outsize, [&](unsigned char* dst) { eng.emit(ep, total, dst); });
  *bp = (unsigned char)(total & 7);
}

// ---------------------------------------------------------------------------------------------
// splice: append position-independent span records (ZopfliB200AppendSpan) to a zopfli-style buffer

unsigned char* append_reserve(size_t n, unsigned char** out, size_t* outsize) {
  size_t s = *outsize, ns = s + n;
  if (n == 0) return *out ? *out + s : nullptr;
  size_t cap = s == 0 ? 0 : pow2_ceil(s), ncap = pow2_ceil(ns);
  if (s == 0) *out = (unsigned char*)malloc(ncap);
  else if (ncap != cap) *out = (unsigned char*)realloc(*out, ncap);
  if (!*out) { fprintf(stderr, "zopfli-b200: out of memory\n"); exit(EXIT_FAILURE); }
  *outsize = ns;
  return *out + s;
}

void append_bytes(const unsigned char* src, size_t n, unsigned char** out, size_t* outsize) {
  if (n) memcpy(append_reserve(n, out, outsize), src, n);
}

// Every piece's bit offset follows from a prefix sum over the piece sizes, so the pieces are copied
// (shifted by their bit phase) in parallel straight into the output buffer; only the bytes shared
// between neighbouring pieces are merged serially.
uint64_t span_positions(std::vector<Engine::SpanRecord>& recs, uint64_t bit0) {
  uint64_t pos = bit0;
  for (Engine::SpanRecord& r : recs) {
    r.bit_start = pos;
    pos = r.stored ? stored_end(pos, r.n) : pos + r.n;
  }
  return pos;
}

void splice_pieces(std::vector<Engine::SpanRecord>& recs, unsigned char* bp, unsigned char** out, size_t* outsize) {
  const size_t np = recs.size();
  uint64_t bit0 = (uint64_t)*outsize * 8;
  if (*bp != 0 && *outsize > 0) bit0 = (uint64_t)(*outsize - 1) * 8 + *bp;
  const uint64_t pos = span_positions(recs, bit0);
  auto end_of = [&](size_t i) { return i + 1 < np ? recs[i + 1].bit_start : pos; };
  const size_t oldsize = *outsize, newsize = (size_t)((pos + 7) / 8);
  append_reserve(newsize - oldsize, out, outsize);  // one append of everything
  unsigned char* o = *out;
  // bytes that two pieces may share: cleared first, OR-merged after the parallel copy
  struct Edge { size_t byte; unsigned char v; };
  std::vector<Edge> edges(np * 2 + 2, Edge{(size_t)-1, 0});
  for (size_t i = 0; i < np; i++) {
    const size_t fb = (size_t)(recs[i].bit_start / 8), lb = (size_t)(end_of(i) / 8);
    if (fb >= oldsize && fb < newsize) o[fb] = 0;
    if (lb >= oldsize && lb < newsize) o[lb] = 0;
  }
  parallel_for(np, [&](size_t i) {
    const Engine::SpanRecord& p = recs[i];
    const uint64_t sb = p.bit_start, eb = end_of(i);
    if (sb == eb) return;
    Edge& e0 = edges[2 * i];
    Edge& e1 = edges[2 * i + 1];
    if (!p.stored) {
      const unsigned char* src = p.src;
      const uint64_t nb = p.n;
      const int sh = (int)(sb & 7);
      const size_t fb = (size_t)(sb / 8);
      // destination byte fb + k holds source bits [8k - sh, 8k - sh + 8)
      auto src_byte = [&](size_t k) -> unsigned {  // source byte k, zero outside the piece's bits
        if ((uint64_t)k * 8 >= nb) return 0;
        unsigned v = src[k];
        const uint64_t left = nb - (uint64_t)k * 8;
        if (left < 8) v &= (1u << left) - 1;
        return v;
      };
      const size_t first_full = sh ? 1 : 0;                 // first destination byte owned entirely
      const size_t end_full = (size_t)(eb / 8) - fb;         // one past the last entirely owned byte
      if (sh) { e0.byte = fb; e0.v = (unsigned char)(src_byte(0) << sh); }
      if (sh == 0) {
        if (end_full > 0) memcpy(o + fb, src, end_full);
      } else {
        size_t k = first_full;
        for (; k + 8 <= end_full && (uint64_t)(k + 8) * 8 <= nb; k += 8) {  // src[k-1 .. k+7] all inside
          uint64_t lo;
          memcpy(&lo, src + k - 1, 8);
          const uint64_t v = (lo >> (8 - sh)) | ((uint64_t)src[k + 7] << (56 + sh));
          memcpy(o + fb + k, &v, 8);
        }
        for (; k < end_full; k++) o[fb + k] = (unsigned char)((src_byte(k - 1) >> (8 - sh)) | (src_byte(k) << sh));
      }
      if (eb & 7) {  // trailing partial byte
        const size_t k = end_full;
        unsigned v = sh ? ((k ? src_byte(k - 1) >> (8 - sh) : 0u) | (src_byte(k) << sh)) : src_byte(k);
        if (!(sh && k == 0)) { e1.byte = fb + k; e1.v = (unsigned char)v; }  // k == 0 with sh: already in e0
      }
    } else {
      uint64_t q = sb;
      size_t ip = 0;
      bool first = true;
      for (;;) {
        size_t bs = 65535;
        if (ip + bs > p.n) bs = (size_t)p.n - ip;
        const bool cur_final = ip + bs >= p.n;
        const unsigned hdr = (p.final && cur_final) ? 1u : 0u;  // BFINAL, BTYPE 00
        if (first) {
          // header bits land in the (possibly shared) byte q/8 -- and the byte after it when the
          // three bits straddle a byte boundary, which then belongs to this piece alone
          const unsigned v = hdr << (q & 7);
          e0.byte = (size_t)(q / 8); e0.v = (unsigned char)v;
          if ((q & 7) > 5) o[q / 8 + 1] = (unsigned char)(v >> 8);
          first = false;
        } else {
          o[q / 8] = (unsigned char)hdr;  // byte aligned here
        }
        q += 3;
        q = (q + 7) & ~(uint64_t)7;
        unsigned char* d = o + q / 8;
        const unsigned nlen = (~(unsigned)bs) & 0xffff;
        d[0] = (unsigned char)(bs % 256);
        d[1] = (unsigned char)((bs / 256) % 256);
        d[2] = (unsigned char)(nlen % 256);
        d[3] = (unsigned char)((nlen / 256) % 256);
        if (bs) memcpy(d + 4, p.src + ip, bs);
        q += 32 + (uint64_t)bs * 8;
        if (cur_final) break;
        ip += bs;
      }
    }
  });
  for (const Edge& e : edges)
    if (e.byte != (size_t)-1) o[e.byte] |= e.v;
  *bp = (unsigned char)(pos & 7);
}

}  // namespace zb

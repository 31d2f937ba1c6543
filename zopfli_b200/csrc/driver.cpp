// Host driver behind ZopfliDeflate / ZopfliDeflatePart (drop-in boundary, SURVEY 8(b)).
//
// Reference control flow (/root/reference/src/zopfli/deflate.c:811-931) is one master block at a
// time, one block at a time.  Here every stage is batched over ALL master blocks of the call so
// the GPU sees every independent unit at once (SURVEY 7.2 #5, 8(e)):
//
//   stage A  GPU   greedy parse of every master block              (blocksplitter.c:288-296)
//   stage B  host  split-point search per master block, threaded   (blocksplitter.c:215-273)
//   stage C  GPU   optimal parse of every block of every master block (deflate.c:854-869)
//   stage D  host  second split attempt + block-type choice        (deflate.c:872-893, 747-800)
//   stage E  GPU   fixed-tree re-parses requested by stage D        (deflate.c:771-781)
//   stage F  host  bit emission per block (threaded) + bit-offset splice
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

namespace {

double now_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

std::mutex g_time_mu;
void add_time(double& acc, double ms) {
  std::lock_guard<std::mutex> g(g_time_mu);
  acc += ms;
}

bool debug_on() {
  static int v = [] { const char* e = getenv("ZOPFLI_B200_DEBUG"); return e && atoi(e) ? 1 : 0; }();
  return v != 0;
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

template <typename F>
void parallel_for(size_t n, F fn) {
  int nt = (int)std::min<size_t>(n, (size_t)host_threads());
  if (nt <= 1) {
    for (size_t i = 0; i < n; i++) fn(i);
    return;
  }
  std::atomic<size_t> next(0);
  std::vector<std::thread> th;
  for (int t = 0; t < nt; t++)
    th.emplace_back([&] {
      for (;;) {
        size_t i = next.fetch_add(1);
        if (i >= n) break;
        fn(i);
      }
    });
  for (auto& t : th) t.join();
}

struct FinalBlock {
  size_t lstart, lend;       // symbol range in the master block's store
  size_t a, b;               // byte range (absolute input positions)
  Engine::PlanCost c;
  uint64_t plan;
  bool expensive = false;
  int fixed_req = -1;        // index into the fixed re-parse batch
};

struct Master {
  size_t ms, me;                       // byte range
  std::vector<size_t> cuts;            // first-split block boundaries in bytes (ms, ..., me)
  std::vector<uint32_t> bsize;         // symbols of every first-split block's optimal parse
  std::vector<Piece> pieces;
};

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

}  // namespace

// in_base: absolute position of device/engine byte 0 (the engine holds bytes [in_base, ...)).
void deflate_units(Engine& eng, const ZopfliOptions* opt, int btype, bool final_last, const unsigned char* in,
                   const std::vector<std::pair<size_t, size_t>>& units, size_t in_base,
                   std::vector<Piece>& pieces) {
  const size_t nm = units.size();
  std::vector<Master> M(nm);
  for (size_t m = 0; m < nm; m++) { M[m].ms = units[m].first; M[m].me = units[m].second; }
  (void)in;

  if (btype == 0) {  // deflate.c:826-828
    for (size_t m = 0; m < nm; m++) {
      Piece p;
      p.type = 0;
      p.instart = M[m].ms;
      p.inend = M[m].me;
      p.final = final_last && m + 1 == nm;
      p.unit = (uint32_t)m;
      pieces.push_back(p);
    }
    return;
  }
  if (btype == 1) {  // deflate.c:829-841: one fixed-tree optimal parse per unit
    std::vector<ParseRange> pr;
    for (auto& mb : M) pr.push_back({mb.ms - in_base, mb.me - in_base, 2, 0});
    std::vector<uint32_t> sizes;
    std::vector<uint64_t> costs;
    eng.parse_keep(pr, Engine::kFix, sizes, costs, 0);
    std::vector<Engine::PlanReq> rq;
    for (size_t m = 0; m < nm; m++) rq.push_back({M[m].ms - in_base, sizes[m], (uint32_t)Engine::kFix});
    std::vector<Engine::PlanCost> pc;
    std::vector<uint64_t> ph;
    eng.plan_blocks(rq, pc, ph, 0);
    for (size_t m = 0; m < nm; m++) {
      Piece p;
      p.type = 1;
      p.buf = Engine::kFix;
      p.off = M[m].ms - in_base;
      p.n = sizes[m];
      p.nbits = pc[m].fixed;
      p.instart = M[m].ms;
      p.inend = M[m].me;
      p.final = final_last && m + 1 == nm;
      p.unit = (uint32_t)m;
      pieces.push_back(p);
    }
    return;
  }

  // The master blocks are processed as a few independent chunk pipelines (stages A-E each), one
  // host thread and one pair of engine lanes per chunk: while one chunk's split search waits on
  // round trips or its longest DP chain is still running, the others keep the GPU busy.
  auto run_chunk = [&](const std::vector<size_t>& cm, int lane_g, int lane_r) {
  const size_t nc = cm.size();
  const int cid = lane_g / 2;
  double t0 = now_ms();
  debug_mark(cid, "start");
  const size_t maxblocks = (size_t)opt->blocksplittingmax;
  if (opt->blocksplitting) {
    // ---- stage A: greedy parse of every master block (blocksplitter.c:288-296).  The greedy stores
    // never leave the device: they become the stores of the split service, and only the byte positions
    // of the chosen split points come back (blocksplitter.c:303-313)
    std::vector<ParseRange> pr;
    for (size_t m : cm) pr.push_back({M[m].ms - in_base, M[m].me - in_base, 0, 0});
    std::vector<uint32_t> gsize;
    eng.greedy_to_split(pr, gsize, lane_g);  // stages A and B sit on the critical path: high-priority lane
    double t1 = now_ms();
    debug_mark(cid, "A greedy done");
    add_time(g_host_times.other, t1 - t0);
    // ---- stage B: split search (costs on the device, decisions on the host) ----
    std::vector<size_t> sizes(gsize.begin(), gsize.end());
    std::vector<std::vector<size_t>> lps =
        batched_block_split(sizes, maxblocks, [&](const std::vector<EvalReq>& r, std::vector<uint64_t>& c) {
          eng.split_eval(reinterpret_cast<const Engine::SplitReq*>(r.data()), r.size(), c.data(), lane_g);
        });
    std::vector<Engine::SplitPos> want;
    for (size_t q = 0; q < nc; q++)
      for (size_t p : lps[q]) want.push_back({(uint32_t)q, (uint32_t)p});
    std::vector<uint32_t> bytepos;
    eng.split_positions(want, bytepos, lane_g);
    size_t w = 0;
    for (size_t q = 0; q < nc; q++) {
      Master& mb = M[cm[q]];
      mb.cuts.push_back(mb.ms);
      for (size_t k = 0; k < lps[q].size(); k++) mb.cuts.push_back(mb.ms + bytepos[w++]);
      mb.cuts.push_back(mb.me);
      if (opt->verbose) print_split_points(mb.cuts, mb.ms);
    }
    double t2 = now_ms();
    debug_mark(cid, "B split done");
    add_time(g_host_times.split, t2 - t1);
    t0 = t2;
  } else {
    for (size_t m : cm) { M[m].cuts.push_back(M[m].ms); M[m].cuts.push_back(M[m].me); }
  }

  // ---- stage C: optimal parse of every block (deflate.c:854-869); the stores stay on the device ----
  {
    std::vector<ParseRange> pr;
    std::vector<std::pair<size_t, size_t>> owner;
    for (size_t m : cm)
      for (size_t i = 0; i + 1 < M[m].cuts.size(); i++) {
        pr.push_back({M[m].cuts[i] - in_base, M[m].cuts[i + 1] - in_base, 1, opt->numiterations});
        owner.push_back({m, i});
      }
    // The critical path of this stage is the DP chain of the largest blocks.  Giant blocks go to
    // the even engine lane on their own (their tables are ready within milliseconds, so their iterate
    // kernel starts at once); everything else is prepared and parsed on the odd lane meanwhile.
    uint64_t kGiant = 250000;
    if (const char* e = getenv("ZOPFLI_B200_GIANT")) kGiant = strtoull(e, nullptr, 10);  // tests: force the two-lane path
    std::vector<ParseRange> prs[2];
    std::vector<size_t> idx[2];
    for (size_t k = 0; k < pr.size(); k++) {
      const int lane = (pr[k].inend - pr[k].instart >= kGiant) ? 0 : 1;
      prs[lane].push_back(pr[k]);
      idx[lane].push_back(k);
    }
    for (size_t m : cm) M[m].bsize.assign(M[m].cuts.size() - 1, 0);
    const bool want_iters = opt->verbose || opt->verbose_more;
    auto parse_lane = [&](int which, int lane) {
      std::vector<uint32_t> sizes;
      std::vector<uint64_t> costs, itc;
      eng.parse_keep(prs[which], Engine::kPack, sizes, costs, lane, want_iters ? &itc : nullptr);
      for (size_t q = 0; q < idx[which].size(); q++) {
        const size_t k = idx[which][q];
        M[owner[k].first].bsize[owner[k].second] = sizes[q];
      }
      if (want_iters && !itc.empty()) {  // squeeze.c:493-495, block after block
        std::lock_guard<std::mutex> g(g_time_mu);
        const size_t stride = itc.size() / idx[which].size();
        for (size_t q = 0; q < idx[which].size(); q++) {
          uint64_t best = ~(uint64_t)0;
          for (size_t i = 0; i < stride && i < (size_t)opt->numiterations; i++) {
            const uint64_t c = itc[q * stride + i];
            if (c == ~(uint64_t)0) break;
            if (opt->verbose_more || c < best) fprintf(stderr, "Iteration %d: %d bit\n", (int)i, (int)c);
            if (c < best) best = c;
          }
        }
      }
    };

    // ---- stages D-E for a set of master blocks whose blocks are all parsed: second split attempt,
    // block types (deflate.c:872-893, 747-800).  Works on sizes only; every store stays on the device.
    auto finish = [&](const std::vector<size_t>& ms, int lane) {
      const size_t nq = ms.size();
      if (nq == 0) return;
      double td0 = now_ms();
      // D1: concatenate the block stores of every master block (ZopfliAppendLZ77Store, deflate.c:863)
      std::vector<Engine::SymCopy> copies;
      std::vector<std::vector<size_t>> first_points(nq);
      std::vector<uint64_t> moff(nq), total(nq, 0);
      std::vector<char> want2(nq, 0);
      std::vector<uint64_t> soff;
      std::vector<uint32_t> ssize;
      std::vector<size_t> who;
      for (size_t q = 0; q < nq; q++) {
        const Master& mb = M[ms[q]];
        moff[q] = mb.ms - in_base;
        for (size_t i = 0; i < mb.bsize.size(); i++) {
          copies.push_back({mb.cuts[i] - in_base, moff[q] + total[q], mb.bsize[i], 0});
          total[q] += mb.bsize[i];
          if (i + 1 < mb.bsize.size()) first_points[q].push_back((size_t)total[q]);
        }
        want2[q] = opt->blocksplitting && first_points[q].size() > 1;  // deflate.c:872
        if (want2[q]) { who.push_back(q); soff.push_back(moff[q]); ssize.push_back((uint32_t)total[q]); }
      }
      eng.concat_stores(copies, soff, ssize, lane);
      // sizes of the first split's blocks (deflate.c:862: AutoType over each block's own store)
      std::vector<Engine::PlanReq> rq;
      std::vector<size_t> rq_base(nq);
      for (size_t q = 0; q < nq; q++) {
        const Master& mb = M[ms[q]];
        rq_base[q] = rq.size();
        uint64_t so = 0;
        for (size_t i = 0; i < mb.bsize.size(); i++) { rq.push_back({moff[q] + so, mb.bsize[i], (uint32_t)Engine::kFin}); so += mb.bsize[i]; }
      }
      std::vector<Engine::PlanCost> c1;
      std::vector<uint64_t> h1;
      eng.plan_blocks(rq, c1, h1, lane);
      std::vector<uint64_t> totalcost(nq, 0);
      for (size_t q = 0; q < nq; q++)
        for (size_t i = 0; i < M[ms[q]].bsize.size(); i++) totalcost[q] += auto_type(c1[rq_base[q] + i], M[ms[q]].bsize[i]);
      // D2: second split attempt on the concatenated stores (deflate.c:872-893)
      std::vector<std::vector<size_t>> second(nq);
      std::vector<Engine::PlanCost> c2;
      std::vector<uint64_t> h2;
      std::vector<size_t> rq2_base(nq, 0);
      std::vector<char> use2(nq, 0);
      if (!who.empty()) {
        std::vector<size_t> sizes(ssize.begin(), ssize.end());
        std::vector<std::vector<size_t>> r =
            batched_block_split(sizes, maxblocks, [&](const std::vector<EvalReq>& rr, std::vector<uint64_t>& c) {
              eng.split_eval(reinterpret_cast<const Engine::SplitReq*>(rr.data()), rr.size(), c.data(), lane);
            });
        std::vector<Engine::PlanReq> rq2;
        for (size_t k = 0; k < who.size(); k++) {
          const size_t q = who[k];
          second[q] = r[k];
          rq2_base[q] = rq2.size();
          for (size_t i = 0; i <= r[k].size(); i++) {
            const size_t a = i == 0 ? 0 : r[k][i - 1], b = i == r[k].size() ? (size_t)total[q] : r[k][i];
            rq2.push_back({moff[q] + a, (uint32_t)(b - a), (uint32_t)Engine::kFin});
          }
        }
        eng.plan_blocks(rq2, c2, h2, lane);
        std::vector<Engine::SplitPos> want;
        std::vector<size_t> want_base(who.size(), 0);
        for (size_t k = 0; k < who.size(); k++) {
          const size_t q = who[k];
          uint64_t totalcost2 = 0;
          for (size_t i = 0; i <= second[q].size(); i++) totalcost2 += auto_type(c2[rq2_base[q] + i], (size_t)total[q]);
          use2[q] = totalcost2 < totalcost[q];
          want_base[k] = want.size();
          if (use2[q] || opt->verbose)
            for (size_t p : second[q]) want.push_back({(uint32_t)k, (uint32_t)p});
        }
        // byte positions of the adopted second-pass split points (lz77->pos, deflate.c:769)
        std::vector<uint32_t> bytepos;
        eng.split_positions(want, bytepos, lane);
        for (size_t k = 0; k < who.size(); k++) {
          const size_t q = who[k];
          if (!use2[q] && !opt->verbose) continue;
          Master& mb = M[ms[q]];
          std::vector<size_t> cuts2(1, mb.ms);
          for (size_t i = 0; i < second[q].size(); i++) cuts2.push_back(mb.ms + bytepos[want_base[k] + i]);
          cuts2.push_back(mb.me);
          if (opt->verbose) print_split_points(cuts2, mb.ms);  // ZopfliBlockSplitLZ77 reports its points whether or not they win
          if (use2[q]) mb.cuts.swap(cuts2);
        }
      }
      // final blocks and the fixed-tree re-parses they ask for (AddLZ77BlockAutoType deflate.c:747-800)
      std::vector<std::vector<FinalBlock>> finals(nq);
      std::vector<ParseRange> prf;
      for (size_t q = 0; q < nq; q++) {
        const Master& mb = M[ms[q]];
        const std::vector<size_t>& points = use2[q] ? second[q] : first_points[q];
        const std::vector<Engine::PlanCost>& cc = use2[q] ? c2 : c1;
        const std::vector<uint64_t>& hh = use2[q] ? h2 : h1;
        const size_t base = use2[q] ? rq2_base[q] : rq_base[q];
        for (size_t i = 0; i <= points.size(); i++) {
          FinalBlock fb;
          fb.lstart = i == 0 ? 0 : points[i - 1];
          fb.lend = i == points.size() ? (size_t)total[q] : points[i];
          fb.a = mb.cuts[i];
          fb.b = mb.cuts[i + 1];
          fb.c = cc[base + i];
          fb.plan = hh[base + i];
          fb.expensive = ((size_t)total[q] < 1000) || ((double)fb.c.fixed <= (double)fb.c.dyn * 1.1);  // :760
          if (fb.lstart == fb.lend) fb.expensive = false;
          if (fb.expensive) {
            fb.fixed_req = (int)prf.size();
            prf.push_back({fb.a - in_base, fb.b - in_base, 2, 0});
          }
          finals[q].push_back(fb);
        }
      }
      double td1 = now_ms();
      add_time(g_host_times.split, td1 - td0);
      // stage E: fixed-tree re-parses (deflate.c:771-781) and their sizes
      std::vector<uint32_t> fsize;
      std::vector<Engine::PlanCost> c3;
      if (!prf.empty()) {
        std::vector<uint64_t> fcost, h3;
        eng.parse_keep(prf, Engine::kFix, fsize, fcost, lane);
        std::vector<Engine::PlanReq> rq3;
        for (size_t g = 0; g < prf.size(); g++) rq3.push_back({prf[g].instart, fsize[g], (uint32_t)Engine::kFix});
        eng.plan_blocks(rq3, c3, h3, lane);
      }
      for (size_t q = 0; q < nq; q++) {
        Master& mb = M[ms[q]];
        for (size_t i = 0; i < finals[q].size(); i++) {
          const FinalBlock& fb = finals[q][i];
          Piece p;
          p.final = final_last && ms[q] + 1 == nm && i + 1 == finals[q].size();
          p.unit = (uint32_t)ms[q];
          p.instart = fb.a;
          p.inend = fb.b;
          if (fb.lstart == fb.lend) {  // deflate.c:763-768: the smallest empty block is a fixed one
            p.type = 1;
            p.n = 0;
            p.nbits = 10;
            mb.pieces.push_back(p);
            continue;
          }
          const uint64_t fixedcost = fb.expensive ? c3[fb.fixed_req].fixed : fb.c.fixed;  // deflate.c:779
          if (fb.c.unc < fixedcost && fb.c.unc < fb.c.dyn) {  // deflate.c:783-785
            p.type = 0;
            p.instart = fb.a;
            p.inend = fb.b;
          } else if (fixedcost < fb.c.dyn) {
            p.type = 1;
            p.nbits = fixedcost;
            if (fb.expensive) { p.buf = Engine::kFix; p.off = fb.a - in_base; p.n = fsize[fb.fixed_req]; }
            else { p.buf = Engine::kFin; p.off = moff[q] + fb.lstart; p.n = (uint32_t)(fb.lend - fb.lstart); }
          } else {
            p.type = 2;
            p.nbits = fb.c.dyn;
            p.tree_bits = (uint32_t)fb.c.tree;
            p.buf = Engine::kFin;
            p.off = moff[q] + fb.lstart;
            p.n = (uint32_t)(fb.lend - fb.lstart);
            p.plan = fb.plan;
          }
          mb.pieces.push_back(p);
        }
      }
      add_time(g_host_times.other, now_ms() - td1);
    };

    if (prs[0].empty() || prs[1].empty()) {
      const int only = prs[0].empty() ? 1 : 0;
      parse_lane(only, lane_g);
      add_time(g_host_times.other, now_ms() - t0);
      finish(cm, lane_r);
    } else {
      std::vector<char> has_giant(nm, 0);
      for (size_t k : idx[0]) has_giant[owner[k].first] = 1;
      std::vector<size_t> clean, dirty;
      for (size_t m : cm) (has_giant[m] ? dirty : clean).push_back(m);
      std::thread tg([&] { parse_lane(0, lane_g); });
      parse_lane(1, lane_r);
      debug_mark(cid, "C rest parsed");
      add_time(g_host_times.other, now_ms() - t0);
      // A master block with a giant also has blocks on lane_r, so its D-E waits for both lanes.  The
      // clean and the dirty D-E then run side by side, each on its own lane: their second split searches
      // are chains of short, latency-bound rounds that leave most of the GPU idle, and when the giants end
      // before the rest the dirty D-E no longer queues behind the clean one.  With verbose output the two
      // run in turn, so the split-point reports keep their order (clean master blocks first).
      auto dirty_tail = [&] {
        double tw = now_ms();
        tg.join();
        debug_mark(cid, "C giants parsed");
        add_time(g_host_times.other, now_ms() - tw);
        finish(dirty, lane_g);  // the giants' lane is idle now and has stream priority
        debug_mark(cid, "D-E dirty done");
      };
      const bool in_turn = opt->verbose || opt->verbose_more;
      std::thread td;
      if (!in_turn) td = std::thread(dirty_tail);
      finish(clean, lane_r);   // overlaps the giants' DP chains still running on lane_g
      debug_mark(cid, "D-E clean done");
      if (in_turn) dirty_tail();
      else td.join();
    }
  }
  };  // run_chunk

  {
    g_debug_t0 = now_ms();
    size_t nchunks = 4;
    if (const char* e = getenv("ZOPFLI_B200_CHUNKS")) nchunks = (size_t)atoi(e);
    nchunks = std::max<size_t>(1, std::min<size_t>(std::min<size_t>(nchunks, Engine::kLanes / 2), nm / 4));
    if (nm < 8) nchunks = 1;
    if (const char* e = getenv("ZOPFLI_B200_FORCE_CHUNKS")) nchunks = std::min<size_t>((size_t)atoi(e), std::min<size_t>(nm, Engine::kLanes / 2));  // tests
    if (nchunks < 1) nchunks = 1;
    std::vector<std::vector<size_t>> chunks(nchunks);
    for (size_t m = 0; m < nm; m++) chunks[m * nchunks / nm].push_back(m);
    // A pipeline takes its master blocks in batches because the lane arenas cost ~140 MB per master
    // block in flight (~100 B per parse position + ~22 B per key position, two lanes).  The batch is as
    // large as a quarter of the device memory allows (180 GB: ~80 master blocks per pipeline), so the
    // 100 MB bench and a 134 MB shard of the 1 GiB config run as ONE wave per pipeline -- every extra
    // wave costs a whole A + B + longest-chain latency -- and the batches of a longer input are balanced.
    size_t batch = std::max<size_t>(8, (size_t)(eng.device_memory_total() / 4 / ((uint64_t)nchunks * 140000000ull)));
    if (const char* e = getenv("ZOPFLI_B200_BATCH")) batch = std::max<size_t>(1, (size_t)atoi(e));
    auto run_pipeline = [&](size_t c) {
      const std::vector<size_t>& all = chunks[c];
      const size_t nbatches = (all.size() + batch - 1) / batch;
      const size_t per = nbatches ? (all.size() + nbatches - 1) / nbatches : 0;
      for (size_t a = 0; a < all.size(); a += per) {
        std::vector<size_t> part(all.begin() + a, all.begin() + std::min(all.size(), a + per));
        run_chunk(part, (int)(2 * c), (int)(2 * c + 1));
      }
    };
    std::vector<std::thread> th;
    for (size_t c = 1; c < nchunks; c++) th.emplace_back([&, c] { run_pipeline(c); });
    run_pipeline(0);
    for (auto& t : th) t.join();
  }
  for (size_t m = 0; m < nm; m++)
    for (auto& p : M[m].pieces) pieces.push_back(p);
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
  unsigned char keep = 0;
  unsigned char* dst;
  if (phase) {  // the stream's first byte is the caller's last, partially filled one
    keep = (*out)[*outsize - 1];
    append_reserve(nbytes - 1, out, outsize);
    dst = *out + *outsize - nbytes;
  } else {
    dst = append_reserve(nbytes, out, outsize);
  }
  eng.emit(ep, total, dst);
  dst[0] |= keep;
  *bp = (unsigned char)(total & 7);
}

// ---------------------------------------------------------------------------------------------
// splice: append position-independent span records (ZopfliB200AppendSpan) to a zopfli-style buffer

// grows the buffer by n bytes under the same capacity rule and returns where they go
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
  if (n == 0) return;
  size_t s = *outsize, ns = s + n;
  size_t cap = s == 0 ? 0 : pow2_ceil(s), ncap = pow2_ceil(ns);
  if (s == 0) {
    *out = (unsigned char*)malloc(ncap);  // util.h:150: first append mallocs
  } else if (ncap != cap) {
    *out = (unsigned char*)realloc(*out, ncap);
  }
  if (!*out) { fprintf(stderr, "zopfli-b200: out of memory\n"); exit(EXIT_FAILURE); }
  memcpy(*out + s, src, n);
  *outsize = ns;
}

// Every piece's bit offset follows from a prefix sum over the piece sizes, so the pieces are copied
// (shifted by their bit phase) in parallel straight into the output buffer; only the bytes shared
// between neighbouring pieces are merged serially.
void splice_pieces(const std::vector<SpanPiece>& pieces, const unsigned char* in, unsigned char* bp,
                   unsigned char** out, size_t* outsize) {
  const size_t np = pieces.size();
  uint64_t bit0 = (uint64_t)*outsize * 8;
  if (*bp != 0 && *outsize > 0) bit0 = (uint64_t)(*outsize - 1) * 8 + *bp;
  std::vector<uint64_t> start(np + 1);
  uint64_t pos = bit0;
  for (size_t i = 0; i < np; i++) {
    const SpanPiece& p = pieces[i];
    start[i] = pos;
    if (!p.stored) {
      pos += p.bits.nbits;
    } else {  // AddNonCompressedBlock deflate.c:625-663: 3 header bits, byte align, LEN/NLEN, bytes
      size_t q = p.instart;
      for (;;) {
        size_t bs = 65535;
        if (q + bs > p.inend) bs = p.inend - q;
        pos += 3;
        pos = (pos + 7) & ~(uint64_t)7;
        pos += 32 + (uint64_t)bs * 8;
        if (q + bs >= p.inend) break;
        q += bs;
      }
    }
  }
  start[np] = pos;
  const size_t oldsize = *outsize, newsize = (size_t)((pos + 7) / 8);
  if (newsize > oldsize) {  // one append of everything (util.h:134-155 capacity rule)
    size_t cap = oldsize == 0 ? 0 : pow2_ceil(oldsize), ncap = pow2_ceil(newsize);
    if (oldsize == 0) *out = (unsigned char*)malloc(ncap);
    else if (ncap != cap) *out = (unsigned char*)realloc(*out, ncap);
    if (!*out) { fprintf(stderr, "zopfli-b200: out of memory\n"); exit(EXIT_FAILURE); }
  }
  unsigned char* o = *out;
  // bytes that two pieces may share: cleared first, OR-merged after the parallel copy
  struct Edge { size_t byte; unsigned char v; };
  std::vector<Edge> edges(np * 2 + 2, Edge{(size_t)-1, 0});
  for (size_t i = 0; i < np; i++) {
    const size_t fb = (size_t)(start[i] / 8), lb = (size_t)(start[i + 1] / 8);
    if (fb >= oldsize && fb < newsize) o[fb] = 0;
    if (lb >= oldsize && lb < newsize) o[lb] = 0;
  }
  parallel_for(np, [&](size_t i) {
    const SpanPiece& p = pieces[i];
    const uint64_t sb = start[i], eb = start[i + 1];
    if (sb == eb) return;
    Edge& e0 = edges[2 * i];
    Edge& e1 = edges[2 * i + 1];
    if (!p.stored) {
      const unsigned char* src = p.bits.bytes.data();
      const uint64_t nb = p.bits.nbits;
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
      size_t ip = p.instart;
      bool first = true;
      for (;;) {
        size_t bs = 65535;
        if (ip + bs > p.inend) bs = p.inend - ip;
        const bool cur_final = ip + bs >= p.inend;
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
        memcpy(d + 4, in + ip, bs);
        q += 32 + (uint64_t)bs * 8;
        if (cur_final) break;
        ip += bs;
      }
    }
  });
  for (const Edge& e : edges)
    if (e.byte != (size_t)-1) o[e.byte] |= e.v;
  *outsize = newsize > oldsize ? newsize : oldsize;
  *bp = (unsigned char)(pos & 7);
}

}  // namespace zb

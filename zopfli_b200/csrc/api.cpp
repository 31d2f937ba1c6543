// C-ABI of libzopfli.so.1 (zopfli-b200): the reference's public entry points
// (/root/reference/src/zopfli/zopfli.h, deflate.h, gzip_container.h, zlib_container.h) plus the
// seams declared in include/zopfli_b200.h.  The calls whose input and result live in device memory are
// in device_api.cpp.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <deque>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/zopfli_b200.h"
#include "api.hpp"
#include "batched_split.hpp"
#include "checksum.hpp"
#include "dist.hpp"
#include "dist_layout.hpp"
#include "driver.hpp"
#include "engine.hpp"
#include "host_emit.hpp"
#include "lz77_store.hpp"

using namespace zb;

namespace {

std::mutex g_api_mu;   // guards g_total_ms and g_last_layout
double g_total_ms = 0;
std::vector<uint64_t> g_last_layout;  // bit offset of every unit (master block) of the most recent deflate call

}  // namespace

namespace zb {

void api_call_done(std::vector<uint64_t>& layout, double t0) {
  std::lock_guard<std::mutex> g(g_api_mu);
  g_last_layout.swap(layout);
  g_total_ms += now_ms() - t0;
}

int trailer_kind(ZopfliFormat fmt) {
  if (fmt != ZOPFLI_FORMAT_GZIP && fmt != ZOPFLI_FORMAT_ZLIB && fmt != ZOPFLI_FORMAT_DEFLATE) return -1;
  return fmt == ZOPFLI_FORMAT_GZIP ? kCkCrc32 : (fmt == ZOPFLI_FORMAT_ZLIB ? kCkAdler32 : kCkNone);
}

// header bytes of the gzip (gzip_container.c:95-104) or zlib (zlib_container.c:58-64) container; 0 for raw deflate
int container_header(ZopfliFormat fmt, unsigned char* hdr, const uint32_t* dictid) {
  if (fmt == ZOPFLI_FORMAT_GZIP) {
    static const unsigned char gz[10] = {31, 139, 8, 0, 0, 0, 0, 0, 2, 3};
    memcpy(hdr, gz, 10);
    return 10;
  }
  if (fmt == ZOPFLI_FORMAT_ZLIB) {
    unsigned cmfflg = 256 * 120 + 3 * 64 + (dictid ? 32 : 0);  // FDICT: 78 F9, as zlib's deflateSetDictionary
    cmfflg += 31 - cmfflg % 31;
    hdr[0] = (unsigned char)(cmfflg / 256);
    hdr[1] = (unsigned char)(cmfflg % 256);
    if (!dictid) return 2;
    for (int i = 0; i < 4; i++) hdr[2 + i] = (unsigned char)(*dictid >> (24 - 8 * i));
    return 6;
  }
  return 0;
}

// the verbose report after the deflate body (fmt DEFLATE, outsize = its bytes) or after the gzip / zlib
// container (outsize = the whole output buffer)
static void report_size(ZopfliFormat fmt, size_t insize, size_t outsize) {
  const double removed = 100.0 * (double)(insize - outsize) / (double)insize;
  if (fmt == ZOPFLI_FORMAT_DEFLATE)  // deflate.c:925-928
    fprintf(stderr, "Original Size: %lu, Deflate: %lu, Compression: %f%% Removed\n", (unsigned long)insize,
            (unsigned long)outsize, removed);
  else  // gzip_container.c:118-122, zlib_container.c:73-77
    fprintf(stderr, "Original Size: %d, %s: %d, Compression: %f%% Removed\n", (int)insize,
            fmt == ZOPFLI_FORMAT_GZIP ? "Gzip" : "Zlib", (int)outsize, removed);
}

void report_sizes(ZopfliFormat fmt, size_t insize, size_t deflate_bytes, size_t outsize) {
  report_size(ZOPFLI_FORMAT_DEFLATE, insize, deflate_bytes);
  if (fmt != ZOPFLI_FORMAT_DEFLATE) report_size(fmt, insize, outsize);
}

bool seam_pieces(size_t insize, const unsigned short* ll, const unsigned short* d, size_t n, size_t npieces,
                 const size_t* lstart, const size_t* lend, const int* btype, const int* final, unsigned bp0,
                 std::vector<Piece>& pieces) {
  if (bp0 > 7) return false;
  std::vector<uint64_t> pos(n + 1, 0);
  for (size_t i = 0; i < n; i++) {
    if (d[i] == 0 ? ll[i] > 255 : (ll[i] < 3 || ll[i] > 258 || d[i] > 32768)) return false;
    pos[i + 1] = pos[i] + (d[i] == 0 ? 1 : ll[i]);
  }
  if (pos[n] > insize) return false;
  pieces.assign(npieces, Piece());
  for (size_t i = 0; i < npieces; i++) {
    if (lstart[i] > lend[i] || lend[i] > n || btype[i] < 0 || btype[i] > 2) return false;
    Piece& p = pieces[i];
    p.type = (uint8_t)btype[i];
    p.final = final[i] != 0;
    p.buf = Engine::kFin;
    p.off = lstart[i];
    p.n = (uint32_t)(lend[i] - lstart[i]);
    p.instart = (size_t)pos[lstart[i]];
    p.inend = (size_t)pos[lend[i]];
  }
  return true;
}

void seam_plan_out(const BlockPlan& b, Piece& p, unsigned char* len320, uint64_t* val6) {
  memcpy(len320, b.ll_len, kNumLL);
  memcpy(len320 + kNumLL, b.d_len, kNumD);
  const uint64_t v[6] = {b.tree_flags, b.tree_bits, b.dyn_bits, b.fixed_bits, b.unc_bits, b.nbytes};
  memcpy(val6, v, sizeof(v));
  p.nbits = p.type == 1 ? b.fixed_bits : b.dyn_bits;
  p.tree_bits = b.tree_bits;
}

void deflate_span_records(Engine& eng, const ZopfliOptions* opt, size_t base, const std::vector<Unit>& units,
                          bool final, SpanRecords& out) {
  std::vector<Piece> unit_pieces;
  deflate_units(eng, opt, 2, final, units, base, unit_pieces);
  // The marker after every unit that ends at a restart point: an empty stored piece (ZopfliDeflatePart with
  // btype 0 over an empty range).  It keeps the unit index of the piece before it, so that layout_pieces counts
  // no unit start for it: markers belong to no unit.
  std::vector<Piece>& pieces = out.pieces;
  pieces.clear();
  out.recs.clear();
  out.markers.clear();
  for (size_t i = 0; i < unit_pieces.size(); i++) {
    pieces.push_back(unit_pieces[i]);
    const Unit& u = units[unit_pieces[i].unit];
    if (u.restart && (i + 1 == unit_pieces.size() || unit_pieces[i + 1].unit != unit_pieces[i].unit)) {
      Piece m;
      m.type = 0;
      m.unit = unit_pieces[i].unit;
      m.instart = m.inend = u.b;
      out.markers.push_back(pieces.size());
      pieces.push_back(m);
    }
  }
  // Records: maximal runs of compressed pieces, each emitted on the device from bit offset 0 of a
  // byte-aligned slot of one buffer, and stored pieces as their payload in the input.
  out.ep.clear();
  out.at.clear();
  uint64_t pos = 0;
  for (size_t i = 0; i < pieces.size();) {
    Engine::SpanRecord r;
    if (pieces[i].type == 0) {
      r.stored = true;
      r.final = pieces[i].final;
      r.n = pieces[i].inend - pieces[i].instart;
      out.recs.push_back(r);
      out.at.push_back(pieces[i].instart);
      i++;
      continue;
    }
    size_t j = i;
    while (j < pieces.size() && pieces[j].type != 0) j++;
    std::vector<Piece> run(pieces.begin() + i, pieces.begin() + j);
    std::vector<Engine::EmitPiece> ep;
    const uint64_t e = layout_pieces(run, base, pos, ep, nullptr);
    r.final = pieces[j - 1].final;
    r.n = e - pos;
    out.recs.push_back(r);
    out.at.push_back(pos);
    out.ep.insert(out.ep.end(), ep.begin(), ep.end());
    pos = (e + 63) & ~(uint64_t)63;  // the next run starts on a fresh word: no shared bytes between records
    i = j;
  }
  out.run_bits = pos;
}

void point_records(SpanRecords& sr, const unsigned char* runs, const unsigned char* in, size_t base) {
  for (size_t i = 0; i < sr.recs.size(); i++) {
    Engine::SpanRecord& r = sr.recs[i];
    if (!r.stored) r.src = runs + sr.at[i] / 8;
    else r.src = r.n ? in + (sr.at[i] - base) : nullptr;  // an empty one (a marker) reads nothing
  }
}

bool parse_span(const unsigned char* span, size_t spansize, std::vector<Engine::SpanRecord>& recs) {
  size_t o = 0;
  // validate the whole span before touching the output: spans arrive over a transport
  while (o < spansize) {
    if (spansize - o < 10 || span[o] > 1 || span[o + 1] > 1) return false;
    uint64_t v;
    memcpy(&v, span + o + 2, 8);
    const uint64_t nbytes = span[o] == 1 ? v : (v + 7) / 8;
    if (nbytes > spansize - o - 10) return false;
    o += 10 + (size_t)nbytes;
  }
  for (o = 0; o < spansize;) {
    Engine::SpanRecord r;
    r.stored = span[o] == 1;
    r.final = span[o + 1] != 0;
    r.src = span + o + 10;
    memcpy(&r.n, span + o + 2, 8);
    recs.push_back(r);
    o += 10 + (size_t)(r.stored ? r.n : (r.n + 7) / 8);
  }
  return true;
}

}  // namespace zb

namespace {

// ---- CRC-32 (gzip_container.c:27-81) and Adler-32 (zlib_container.c:29-48) of host bytes ----
// The input is cut into slices of `slice` bytes (0: one slice per host thread from 4 MiB on, else a single
// slice).  The slices are reduced side by side and combined with the slice algebra of checksum.hpp, as the
// device kernels combine theirs.
uint32_t host_checksum(const unsigned char* d, size_t n, int kind, size_t slice) {
  static const struct CrcTables {
    uint32_t t[8][256];
    CrcTables() {
      for (int k = 0; k < 8; k++)
        for (uint32_t i = 0; i < 256; i++) t[k][i] = crc_table_entry(k, i);
    }
  } T;
  static const CrcShiftTable sh = crc_shift_table();
  if (slice == 0) {
    const size_t nt = n >= (4u << 20) ? (size_t)host_threads() : 1;
    slice = std::max<size_t>((n + nt - 1) / nt, 1);
  }
  std::vector<ChecksumAcc> part((n + slice - 1) / slice);
  parallel_for(part.size(), [&](size_t s) {
    const unsigned char* p = d + s * slice;
    const size_t len = std::min(slice, n - s * slice), after = n - s * slice - len;
    if (kind == kCkCrc32) {  // slicing-by-8 from register 0, then past the bytes after the slice
      uint32_t c = 0;
      size_t k = 0;
      for (; k < len && ((uintptr_t)(p + k) & 7); k++) c = T.t[0][(c ^ p[k]) & 255] ^ (c >> 8);
      for (; k + 8 <= len; k += 8) {
        uint64_t v;
        memcpy(&v, p + k, 8);
        c = crc_slice8(c, (uint32_t)v, (uint32_t)(v >> 32), T.t);
      }
      for (; k < len; k++) c = T.t[0][(c ^ p[k]) & 255] ^ (c >> 8);
      part[s].crc0 = crc_shift(c, after, sh);
    } else {
      const AdlerPart q = adler_chunk(p, len);
      part[s].a = q.s1;
      part[s].b = (q.s2 + (after % kAdlerMod) * q.s1) % kAdlerMod;
    }
  });
  ChecksumAcc acc = {0, 0, 0, 0};
  for (const ChecksumAcc& q : part) {
    acc.crc0 ^= q.crc0;
    acc.a += q.a;
    acc.b += q.b;
  }
  return kind == kCkCrc32 ? crc_finish(acc.crc0, n, sh) : adler_finish(acc.a, acc.b, n);
}

void deflate_impl(const ZopfliOptions* options, int btype, int final, const unsigned char* in,
                  size_t insize, const unsigned char* dev_in, unsigned char* bp, unsigned char** out,
                  size_t* outsize) {
  double t0 = now_ms();
  size_t offset = *outsize;
  // several GPUs in this process (ZOPFLI_B200_GPUS): master blocks sharded over them, NCCL scatter / gather
  if (btype == 2 && !dev_in && dist_local_gpus() > 1 && insize > (size_t)kMasterBlock &&
      dist_local_deflate(dist_local_gpus(), options, final, in, insize, bp, out, outsize)) {
    std::lock_guard<std::mutex> g(g_api_mu);
    g_total_ms += now_ms() - t0;
    return;
  }
  std::vector<Piece> pieces;
  Engine::Lease eng;  // this call's private engine context
  if (dev_in) eng->set_input_device(dev_in, insize);
  else eng->set_input_host(in, insize);
  const double t1 = now_ms();
  deflate_units(*eng, options, btype, final != 0, master_blocks(0, insize), 0, pieces);
  const double t2 = now_ms();
  std::vector<uint64_t> layout;
  assemble(*eng, pieces, 0, bp, out, outsize, &layout, options->verbose != 0);
  { std::lock_guard<std::mutex> g(g_api_mu); g_last_layout.swap(layout); }
  if (debug_on())
    fprintf(stderr, "[zb] api: set_input %.1f ms, deflate_units %.1f ms, emit %.1f ms\n", t1 - t0, t2 - t1, now_ms() - t2);
  if (options->verbose) report_size(ZOPFLI_FORMAT_DEFLATE, insize, *outsize - offset);
  { std::lock_guard<std::mutex> g(g_api_mu); g_total_ms += now_ms() - t0; }
}

// the containers (gzip_container.c:84-124, zlib_container.c:50-79) around a deflate body produced by `body`
template <typename Body>
void container_impl(const ZopfliOptions* options, ZopfliFormat fmt, const unsigned char* in, size_t insize,
                    unsigned char** out, size_t* outsize, Body body) {
  const int kind = trailer_kind(fmt);
  if (kind < 0) {
    fprintf(stderr, "zopfli-b200: unknown output format %d\n", (int)fmt);  // zopfli_lib.c:40 assert(0)
    abort();
  }
  unsigned char bp = 0;
  if (kind == kCkNone) {
    body(&bp);
    return;
  }
  uint32_t sum = 0;
  std::thread sum_thread([&] { sum = host_checksum(in, insize, kind, 0); });  // overlaps the GPU work
  unsigned char hdr[10], tr[8];
  append_bytes(hdr, container_header(fmt, hdr), out, outsize);
  body(&bp);
  const double tj = now_ms();
  sum_thread.join();
  if (debug_on()) fprintf(stderr, "[zb] api: %s join waited %.1f ms\n", kind == kCkCrc32 ? "crc" : "adler", now_ms() - tj);
  append_bytes(tr, container_trailer(kind, sum, insize, tr), out, outsize);
  if (options->verbose) report_size(fmt, insize, *outsize);
}

void compress_impl(const ZopfliOptions* options, ZopfliFormat fmt, const unsigned char* in, size_t insize,
                   const unsigned char* dev_in, unsigned char** out, size_t* outsize) {
  container_impl(options, fmt, in, insize, out, outsize, [&](unsigned char* bp) {
    deflate_impl(options, 2, 1, in, insize, dev_in, bp, out, outsize);
  });
}

void make_store(const unsigned short* ll, const unsigned short* dd, size_t n, Lz77Store& st) {
  st.append(ll, dd, n, 0);
  st.finalize();
}

// A compressor's waves in host memory: one buffer per slot, reserved up to the bytes of one staged wave; the
// stream is spliced on the host (splice_pieces) into a zopfli-style buffer
struct HostStaging : WaveStaging {
  std::vector<unsigned char> slot[kSlots];
  unsigned char* pend = nullptr;
  size_t pendsize = 0;
  unsigned char bp = 0;
  ~HostStaging() override { free(pend); }
  int device() const override { return -1; }
  bool accepts(const void* p, size_t n) const override {
    return n == 0 || (p && !(g_pointer_device && g_pointer_device(p) >= 0));
  }
  void put(int s, size_t off, const unsigned char* chunk, size_t n) override {
    std::vector<unsigned char>& b = slot[s];
    if (b.capacity() < off + n) b.reserve(std::max(off + n, std::min(2 * b.capacity(), slot_bytes)));
    b.resize(off);
    b.insert(b.end(), chunk, chunk + n);
  }
  void carry(int from, size_t off, int to, size_t n) override { put(to, 0, slot[from].data() + off, n); }
  const unsigned char* at(int s, size_t off) {
    static const unsigned char none[16] = {0};
    return slot[s].empty() ? none : slot[s].data() + off;
  }
  void stage(Engine& eng, int s, size_t len) override { eng.set_input_host(at(s, 0), len); }
  uint32_t checksum(Engine&, int s, size_t off, size_t n, int kind) override {
    return host_checksum(at(s, off), n, kind, 0);
  }
  // The records point into sr.runs and slot s until the wave is spliced: only the filling slot is written or
  // regrown (put, carry), and slot s is not filling again before its wave is retired.
  void take_records(Engine& eng, int s, size_t base, SpanRecords& sr) override {
    sr.runs = (unsigned char*)calloc((size_t)(sr.run_bits / 8) + 8, 1);
    if (!sr.runs) { fprintf(stderr, "zopfli-b200: out of memory\n"); exit(EXIT_FAILURE); }
    if (sr.run_bits) eng.emit(sr.ep, sr.run_bits, sr.runs);
    point_records(sr, sr.runs, slot[s].data(), base);
  }
  void drop_records(SpanRecords& sr) override {
    free(sr.runs);
    sr.runs = nullptr;
  }
  uint32_t checksum_of(const unsigned char* p, size_t n, int kind) override { return host_checksum(p, n, kind, 0); }

  unsigned phase() const override { return pendsize ? (bp & 7u) : 0u; }
  void put_bytes(const unsigned char* p, size_t n) override { append_bytes(p, n, &pend, &pendsize); }
  void splice(SpanRecords& sr) override { splice_pieces(sr.recs, &bp, &pend, &pendsize); }
  // What stays behind is at most the partly filled last byte, in a fresh one-byte buffer: zopfli's capacity rule
  // derives a buffer's capacity from its size, so a larger buffer must not be kept under a smaller size.
  size_t hand_out(bool all, bool, unsigned char** out, size_t* outsize) override {
    const size_t keep = (!all && bp != 0 && pendsize > 0) ? 1 : 0;
    const unsigned char last = keep ? pend[pendsize - 1] : 0;
    const size_t n = pendsize - keep;
    append_bytes(pend, n, out, outsize);
    free(pend);
    pend = nullptr;
    pendsize = 0;
    if (keep) append_bytes(&last, 1, &pend, &pendsize);
    return n;
  }
};

}  // namespace

namespace zb {
WaveStaging* (*g_device_staging)(int, void*) = nullptr;
int (*g_pointer_device)(const void*) = nullptr;
}  // namespace zb

// ---- input in pieces (include/zopfli_b200.h) ----
// Bytes are put into the filling slot of the staging; once a byte past a whole wave has arrived (next_wave),
// the wave runs on a worker thread of its own, which leases an engine context for just that wave and turns it
// into span records plus the checksum of its bytes.  The next wave's slot takes over the last 32 KiB as its
// dictionary.  Waves are spliced onto the stream in order, at its bit phase, by the calling thread; only the
// complete bytes go back to the caller.
// Positions are counted in X = preset dictionary || data.  A flush ends a segment: what is left becomes one
// wave however short, the sync marker follows it, and the next segment's master blocks count from there.  A
// full flush also raises the floor, the first position a later parse may see: the next slot starts there.
// Restart points (an interval N) end segments inside the waves instead: each unit carries its floor, and the
// full-flush marker after a unit that ends at a restart point is one more record of its wave.
struct ZopfliB200Compressor {
  struct Run {
    Wave w;
    size_t base;        // position of the slot's byte 0
    int slot;
    SpanRecords sr;
    uint32_t sum = 0;   // checksum of the wave's bytes [w.a, w.b)
    std::atomic<bool> done{false};
    std::thread worker;
  };

  ZopfliOptions opt;
  ZopfliFormat fmt;
  int kind;
  std::unique_ptr<WaveStaging> staging;
  size_t wave_blocks = 0;            // master blocks per wave, set when the first byte arrives
  size_t received = 0, handed = 0;   // positions: end of the bytes written; end of the bytes in waves
  size_t dict_len = 0;               // position of the first data byte
  size_t floor = 0;                  // position of the last full flush at or before `handed`
  size_t interval = 0;               // restart interval (0: none): automatic full flushes at dict_len + k * interval
  bool started = false;              // a Write or Flush was accepted: no dictionary any more
  bool has_dict = false;
  uint32_t dictid = 0;               // Adler-32 of the whole dictionary
  bool finished = false;
  int fill = -1;                     // slot taking the next bytes (-1: none yet)
  size_t fill_base = 0;              // position of its byte 0
  std::vector<int> free_slots;
  std::deque<std::unique_ptr<Run>> inflight;
  bool header_done = false;
  size_t header_bytes = 0;           // bytes of the container header
  uint64_t deflate_bits = 0;         // bits of the deflate stream spliced so far
  size_t produced = 0;               // bytes returned so far
  uint32_t sum;                      // checksum of the bytes of the spliced waves
  std::vector<uint64_t> layout;      // bit offset of every master block spliced so far
  // (data_off, stream_off) of every full-flush marker spliced so far: data position of the flush, and stream
  // offset of the first byte after the marker
  std::vector<std::pair<uint64_t, uint64_t>> index;
  double busy_ms = 0;                // time spent in Write and Finish

  ZopfliB200Compressor(const ZopfliOptions* o, ZopfliFormat f, WaveStaging* st)
      : opt(*o), fmt(f), kind(trailer_kind(f)), staging(st), sum(kind == kCkAdler32 ? 1u : 0u) {
    for (int s = WaveStaging::kSlots - 1; s >= 0; s--) free_slots.push_back(s);
  }
  ~ZopfliB200Compressor() {  // abandons unfinished work: waits for the waves in flight, drops their output
    for (auto& r : inflight) {
      r->worker.join();
      staging->drop_records(r->sr);
    }
  }

  // With verbose reports a wave starts once the one before it is spliced, so reports do not interleave.
  size_t max_inflight() const { return (opt.verbose || opt.verbose_more) ? 1 : 2; }

  void set_wave_blocks() {
    if (wave_blocks) return;
    Engine::Lease eng(staging->device());
    wave_blocks = wave_master_blocks(eng->device_memory_total() / 2);  // two waves in flight: one call's budget
    staging->slot_bytes = wave_blocks * kMasterBlock + kWindow + 16;
  }

  // the caller's bytes up to stream position `upto` into the filling slot; chunk starts at position `at`
  void fill_to(size_t upto, const unsigned char* chunk, size_t at) {
    if (upto == received) return;
    if (fill < 0) take_slot(floor);
    staging->put(fill, received - fill_base, chunk + (received - at), upto - received);
    received = upto;
  }

  void take_slot(size_t base) {
    fill = free_slots.back();
    free_slots.pop_back();
    fill_base = base;
  }

  // runs on the wave's worker thread
  void compress(Run& r) {
    Engine::Lease eng(staging->device());
    staging->stage(*eng, r.slot, r.w.b - r.base);
    const size_t off = r.w.a - r.base, n = r.w.b - r.w.a;
    std::thread ck;
    if (kind != kCkNone) {
      if (staging->device() < 0) ck = std::thread([&] { r.sum = staging->checksum(*eng, r.slot, off, n, kind); });  // overlaps the GPU work
      else r.sum = staging->checksum(*eng, r.slot, off, n, kind);
    }
    deflate_span_records(*eng, &opt, r.base, r.w.units, r.w.final, r.sr);
    staging->take_records(*eng, r.slot, r.base, r.sr);
    if (ck.joinable()) ck.join();
    r.done = true;
  }

  // starts wave w on the filling slot; a wave that is not the last hands its last 32 KiB above the floor at its
  // end (w.floor_end) to a fresh slot
  void launch(const Wave& w) {
    while (inflight.size() >= max_inflight()) retire_oldest();
    if (fill < 0) take_slot(floor);  // an empty stream
    std::unique_ptr<Run> r(new Run);
    r->w = w;
    r->base = fill_base;
    r->slot = fill;
    Run* p = r.get();
    p->worker = std::thread([this, p] { compress(*p); });
    inflight.push_back(std::move(r));
    handed = w.b;
    floor = w.floor_end;
    fill = -1;
    if (w.final) return;
    const size_t base = wave_base(w.b, floor);
    take_slot(base);
    staging->carry(p->slot, base - p->base, fill, w.b - base);
  }

  void put_header() {
    if (header_done) return;
    unsigned char hdr[10];
    header_bytes = (size_t)container_header(fmt, hdr, has_dict ? &dictid : nullptr);
    staging->put_bytes(hdr, header_bytes);
    header_done = true;
  }

  // the oldest wave in flight, once done, spliced onto the stream (with the block reports of verbose)
  void retire_oldest() {
    std::unique_ptr<Run> r = std::move(inflight.front());
    inflight.pop_front();
    r->worker.join();
    put_header();
    const unsigned phase = staging->phase();
    std::vector<Engine::EmitPiece> ep;
    std::vector<uint64_t> ub;
    const uint64_t end = place_pieces(r->sr.pieces, r->base, phase, ep, &ub, opt.verbose != 0);
    for (size_t i = 0; i + 1 < ub.size(); i++) layout.push_back(deflate_bits + ub[i]);
    // deflate_bits - phase is the body bit of the wave's bit 0, a byte boundary; after a marker the stream is
    // byte-aligned
    for (size_t m : r->sr.markers)
      index.push_back({r->sr.pieces[m].instart - dict_len,
                       header_bytes + (deflate_bits - phase + stored_end(ep[m].bit_start, 0)) / 8});
    deflate_bits += end - phase;
    staging->splice(r->sr);
    staging->drop_records(r->sr);
    const uint64_t n = r->w.b - r->w.a;
    if (kind == kCkCrc32) sum = crc32_combine(sum, r->sum, n);
    else if (kind == kCkAdler32) sum = adler32_combine(sum, r->sum, n);
    free_slots.push_back(r->slot);
  }

  // the complete bytes (all of them with `all`) to the caller: appended to a host buffer, or with to_device a
  // fresh device allocation
  void hand_out(unsigned char** out, size_t* outsize, bool all, bool to_device) {
    produced += staging->hand_out(all, to_device, out, outsize);
  }

  // what every output call refuses: no place for the output, a finished compressor, device output of a host one
  bool refuses(unsigned char** out, size_t* outsize, bool to_device) const {
    return !out || !outsize || finished || (to_device && staging->device() < 0);
  }

  int set_dictionary(const unsigned char* dict, size_t n) {
    if (fmt == ZOPFLI_FORMAT_GZIP || started || has_dict || (!dict && n) || !staging->accepts(dict, n)) return 1;
    const double t0 = now_ms();
    has_dict = true;
    dictid = n ? staging->checksum_of(dict, n, kCkAdler32) : 1u;
    if (n) {  // only the last 32 KiB can be matched: they go in front of the first wave
      set_wave_blocks();
      take_slot(wave_base(n));
      staging->put(fill, 0, dict + fill_base, n - fill_base);
    }
    received = handed = dict_len = n;
    busy_ms += now_ms() - t0;
    return 0;
  }

  // the sync marker behind everything spliced so far; a full one (mode 3) raises the floor to the bytes
  // received and enters the index.  The stream is then byte-aligned.
  void put_marker(bool full) {
    while (!inflight.empty()) retire_oldest();
    put_header();
    SpanRecords marker;
    marker.recs.resize(1);
    marker.recs[0].stored = true;
    staging->splice(marker);
    deflate_bits = stored_end(deflate_bits, 0);
    if (!full) return;
    floor = received;
    if (fill >= 0) fill_base = floor;  // the filling slot holds nothing past the floor: drop what it carried
    index.push_back({received - dict_len, header_bytes + deflate_bits / 8});
  }

  int set_restart_interval(size_t n) {
    if (n == 0 || interval != 0 || started || finished) return 1;
    interval = n;
    return 0;
  }

  // entries of the index whose marker's bytes have been returned
  size_t restart_points(uint64_t* data_off, uint64_t* stream_off, size_t cap) const {
    size_t k = 0;
    while (k < index.size() && index[k].second <= produced) k++;
    for (size_t i = 0; i < k && i < cap; i++) {
      if (data_off) data_off[i] = index[i].first;
      if (stream_off) stream_off[i] = index[i].second;
    }
    return k;
  }

  int write(const unsigned char* chunk, size_t n, unsigned char** out, size_t* outsize, bool to_device) {
    if (refuses(out, outsize, to_device) || !staging->accepts(chunk, n)) return 1;
    const double t0 = now_ms();
    started = true;
    if (n) {
      set_wave_blocks();
      // A flush that ended exactly at a restart point: its automatic full flush comes now that a byte past the
      // point arrives.  (A wave ends at a restart point only with a byte past it, and then carries the marker.)
      if (handed == received && received > dict_len && interval && (received - dict_len) % interval == 0)
        put_marker(true);
      const size_t at = received, total = received + n;
      Wave w;
      while (next_wave(total, kWaveWrite, handed, floor, dict_len, interval, wave_blocks, &w)) {
        fill_to(w.b, chunk, at);
        launch(w);
      }
      fill_to(total, chunk, at);
    }
    while (!inflight.empty() && inflight.front()->done) retire_oldest();
    hand_out(out, outsize, false, to_device);
    busy_ms += now_ms() - t0;
    return 0;
  }

  // mode 2 (sync) or 3 (full): what is left becomes one wave, then the marker, a stored block of BFINAL 0 and
  // LEN 0 (ZopfliDeflatePart with btype 0 over an empty range, deflate.c:625-663); the stream is byte-aligned
  int flush(int mode, unsigned char** out, size_t* outsize, bool to_device) {
    if (refuses(out, outsize, to_device) || (mode != 2 && mode != 3)) return 1;
    const double t0 = now_ms();
    started = true;
    Wave w;
    if (next_wave(received, kWaveFlush, handed, floor, dict_len, interval, wave_blocks, &w)) {
      if (mode == 3) w.floor_end = w.b;  // the next slot starts at the floor, with nothing carried
      launch(w);
    }
    put_marker(mode == 3);
    hand_out(out, outsize, true, to_device);
    busy_ms += now_ms() - t0;
    return 0;
  }

  int finish(unsigned char** out, size_t* outsize, bool to_device) {
    if (refuses(out, outsize, to_device)) return 1;
    const double t0 = now_ms();
    finished = true;
    Wave w;
    next_wave(received, kWaveFinish, handed, floor, dict_len, interval, wave_blocks, &w);
    launch(w);
    while (!inflight.empty()) retire_oldest();
    const size_t insize = received - dict_len;
    unsigned char tr[8];
    staging->put_bytes(tr, container_trailer(kind, sum, insize, tr));
    hand_out(out, outsize, true, to_device);
    if (opt.verbose) report_sizes(fmt, insize, (size_t)((deflate_bits + 7) / 8), produced);
    layout.push_back(deflate_bits);
    busy_ms += now_ms() - t0;
    api_call_done(layout, now_ms() - busy_ms);
    return 0;
  }
};

extern "C" {

void ZopfliInitOptions(ZopfliOptions* options) {  // util.c:28-35
  options->verbose = 0;
  options->verbose_more = 0;
  options->numiterations = 15;
  options->blocksplitting = 1;
  options->blocksplittinglast = 0;
  options->blocksplittingmax = 15;
}

void ZopfliCompress(const ZopfliOptions* options, ZopfliFormat output_type, const unsigned char* in,
                    size_t insize, unsigned char** out, size_t* outsize) {
  compress_impl(options, output_type, in, insize, nullptr, out, outsize);
}

void ZopfliB200CompressDevice(const ZopfliOptions* options, ZopfliFormat output_type, const unsigned char* in,
                              size_t insize, const unsigned char* dev_in, unsigned char** out, size_t* outsize) {
  compress_impl(options, output_type, in, insize, dev_in, out, outsize);
}

void ZopfliGzipCompress(const ZopfliOptions* options, const unsigned char* in, size_t insize,
                        unsigned char** out, size_t* outsize) {
  compress_impl(options, ZOPFLI_FORMAT_GZIP, in, insize, nullptr, out, outsize);
}

void ZopfliZlibCompress(const ZopfliOptions* options, const unsigned char* in, size_t insize,
                        unsigned char** out, size_t* outsize) {
  compress_impl(options, ZOPFLI_FORMAT_ZLIB, in, insize, nullptr, out, outsize);
}

void ZopfliDeflate(const ZopfliOptions* options, int btype, int final, const unsigned char* in, size_t insize,
                   unsigned char* bp, unsigned char** out, size_t* outsize) {
  deflate_impl(options, btype, final, in, insize, nullptr, bp, out, outsize);
}

void ZopfliDeflatePart(const ZopfliOptions* options, int btype, int final, const unsigned char* in,
                       size_t instart, size_t inend, unsigned char* bp, unsigned char** out,
                       size_t* outsize) {
  // only in[max(0, instart-32768), inend) can influence the result (squeeze.c:229-241)
  size_t base = instart > (size_t)kWindow ? instart - kWindow : 0;
  base &= ~(size_t)15;
  std::vector<Piece> pieces;
  Engine::Lease eng;
  eng->set_input_host(in + base, inend - base);
  deflate_units(*eng, options, btype, final != 0, {Unit{instart, inend}}, base, pieces);
  assemble(*eng, pieces, base, bp, out, outsize, nullptr, options->verbose != 0);
}

int ZopfliB200DistCompress(const ZopfliOptions* options, ZopfliFormat output_type, const unsigned char* in, size_t insize,
                           int flags, unsigned char** out, size_t* outsize) {
  if (!dist_rank_ready()) return 1;
  const bool staged = (flags & ZOPFLI_B200_DIST_STAGED) != 0;
  if (dist_rank() != 0) {  // workers take part in the deflate body only
    dist_rank_deflate(options, 1, nullptr, insize, nullptr, nullptr, nullptr, staged);
    return 0;
  }
  container_impl(options, output_type, in, insize, out, outsize, [&](unsigned char* bp) {
    dist_rank_deflate(options, 1, in, insize, bp, out, outsize, staged);
  });
  return 0;
}

int ZopfliB200DeflateSpan(const ZopfliOptions* options, const unsigned char* in, size_t insize,
                          const unsigned char* dev_in, size_t start, size_t end, int final,
                          unsigned char** span, size_t* spansize) {
  if (end > insize || start > end) return 1;
  if (start == end && insize > 0) return 0;  // an empty span of an empty input is one empty master block
  size_t base = 0;
  Engine::Lease eng;
  if (dev_in) {
    eng->set_input_device(dev_in, insize);
  } else {
    base = wave_base(start);
    eng->set_input_host(in + base, end - base);
  }
  SpanRecords sr;
  deflate_span_records(*eng, options, base, master_blocks(start, end), final != 0, sr);
  std::vector<unsigned char> runs((size_t)(sr.run_bits / 8) + 8, 0);
  if (sr.run_bits) eng->emit(sr.ep, sr.run_bits, runs.data());
  point_records(sr, runs.data(), in, 0);
  size_t total = 0;
  for (const Engine::SpanRecord& r : sr.recs) total += 10 + (size_t)(r.stored ? r.n : (r.n + 7) / 8);
  unsigned char* d = append_reserve(total, span, spansize);
  for (const Engine::SpanRecord& r : sr.recs) {
    d[0] = r.stored ? 1 : 0;
    d[1] = r.final ? 1 : 0;
    memcpy(d + 2, &r.n, 8);
    const size_t nb = (size_t)(r.stored ? r.n : (r.n + 7) / 8);
    if (nb) memcpy(d + 10, r.src, nb);
    d += 10 + nb;
  }
  return 0;
}

uint32_t ZopfliB200Crc32(const unsigned char* data, size_t size) { return host_checksum(data, size, kCkCrc32, 0); }
uint32_t ZopfliB200Crc32Combine(uint32_t crc1, uint32_t crc2, uint64_t len2) { return crc32_combine(crc1, crc2, len2); }
uint32_t ZopfliB200Adler32Combine(uint32_t adler1, uint32_t adler2, uint64_t len2) { return adler32_combine(adler1, adler2, len2); }
uint32_t ZopfliB200Adler32(const unsigned char* data, size_t size) { return host_checksum(data, size, kCkAdler32, 0); }
uint32_t ZopfliB200HostChecksumSliced(const unsigned char* data, size_t size, size_t slice_bytes, int kind) {
  return host_checksum(data, size, kind, slice_bytes ? slice_bytes : 1);
}

int ZopfliB200AppendSpan(const unsigned char* span, size_t spansize, unsigned char* bp, unsigned char** out,
                         size_t* outsize) {
  std::vector<Engine::SpanRecord> recs;
  if (!parse_span(span, spansize, recs)) return 1;
  splice_pieces(recs, bp, out, outsize);
  return 0;
}

int ZopfliB200CompressorNew(const ZopfliOptions* options, ZopfliFormat output_type, int device, void* cuda_stream,
                            ZopfliB200Compressor** c) {
  if (!options || !c) return 1;
  if (trailer_kind(output_type) < 0) return 1;
  WaveStaging* st = nullptr;
  if (device < 0) st = new HostStaging;
  else if (!g_device_staging || !(st = g_device_staging(device, cuda_stream))) return 1;
  *c = new ZopfliB200Compressor(options, output_type, st);
  return 0;
}

int ZopfliB200CompressorWrite(ZopfliB200Compressor* c, const unsigned char* chunk, size_t n, unsigned char** out,
                              size_t* outsize) {
  return c ? c->write(chunk, n, out, outsize, false) : 1;
}

int ZopfliB200CompressorFinish(ZopfliB200Compressor* c, unsigned char** out, size_t* outsize) {
  return c ? c->finish(out, outsize, false) : 1;
}

int ZopfliB200CompressorFlush(ZopfliB200Compressor* c, int mode, unsigned char** out, size_t* outsize) {
  return c ? c->flush(mode, out, outsize, false) : 1;
}

int ZopfliB200CompressorWriteToDevice(ZopfliB200Compressor* c, const unsigned char* chunk, size_t n,
                                      unsigned char** dev_out, size_t* outsize) {
  return c ? c->write(chunk, n, dev_out, outsize, true) : 1;
}

int ZopfliB200CompressorFlushToDevice(ZopfliB200Compressor* c, int mode, unsigned char** dev_out, size_t* outsize) {
  return c ? c->flush(mode, dev_out, outsize, true) : 1;
}

int ZopfliB200CompressorFinishToDevice(ZopfliB200Compressor* c, unsigned char** dev_out, size_t* outsize) {
  return c ? c->finish(dev_out, outsize, true) : 1;
}

int ZopfliB200CompressorSetDictionary(ZopfliB200Compressor* c, const unsigned char* dict, size_t n) {
  return c ? c->set_dictionary(dict, n) : 1;
}

int ZopfliB200CompressorSetRestartInterval(ZopfliB200Compressor* c, size_t interval) {
  return c ? c->set_restart_interval(interval) : 1;
}

size_t ZopfliB200CompressorRestartPoints(ZopfliB200Compressor* c, uint64_t* data_off, uint64_t* stream_off, size_t cap) {
  return c ? c->restart_points(data_off, stream_off, cap) : 0;
}

void ZopfliB200CompressorFree(ZopfliB200Compressor* c) { delete c; }

int ZopfliB200CompressorWave(size_t received, int finished, size_t handed, size_t wave_blocks, size_t* a, size_t* b,
                             int* final) {
  Wave w;
  const int call = finished == kWaveFlush ? (int)kWaveFlush : (finished != 0 ? (int)kWaveFinish : (int)kWaveWrite);
  if (!next_wave(received, call, handed, 0, 0, 0, wave_blocks, &w)) return 0;
  *a = w.a;
  *b = w.b;
  *final = w.final ? 1 : 0;
  return 1;
}

size_t ZopfliB200CompressorWaveUnits(size_t received, int finished, size_t handed, size_t floor, size_t dict_len,
                                     size_t interval, size_t wave_blocks, size_t* a, size_t* b, size_t* floors,
                                     int* restart, size_t cap, int* final) {
  Wave w;
  const int call = finished == kWaveFlush ? (int)kWaveFlush : (finished != 0 ? (int)kWaveFinish : (int)kWaveWrite);
  if (!next_wave(received, call, handed, floor, dict_len, interval, wave_blocks, &w)) return 0;
  for (size_t i = 0; i < w.units.size() && i < cap; i++) {
    if (a) a[i] = w.units[i].a;
    if (b) b[i] = w.units[i].b;
    if (floors) floors[i] = w.units[i].floor;
    if (restart) restart[i] = w.units[i].restart ? 1 : 0;
  }
  if (final) *final = w.final ? 1 : 0;
  return w.units.size();
}

size_t ZopfliB200LastMasterBitOffsets(uint64_t* offsets, size_t cap) {
  std::lock_guard<std::mutex> g(g_api_mu);
  for (size_t i = 0; i < g_last_layout.size() && i < cap; i++) offsets[i] = g_last_layout[i];
  return g_last_layout.size();
}

int ZopfliB200LZ77Batch(const unsigned char* in, size_t insize, size_t n, const size_t* instart,
                        const size_t* inend, int mode, int numiterations, unsigned short* litlens,
                        unsigned short* dists, size_t cap, size_t* off, size_t* cnt, uint64_t* cost) {
  Engine::Lease lease;
  Engine& e = *lease;
  e.set_input_host(in, insize);
  std::vector<ParseRange> pr(n);
  for (size_t i = 0; i < n; i++) pr[i] = {instart[i], inend[i], mode == 0 ? 1 : (mode == 1 ? 2 : 0), numiterations};
  ParseResult res;
  e.parse(pr, res);
  size_t total = 0;
  for (size_t i = 0; i < n; i++) {
    off[i] = total;
    cnt[i] = res.size[i];
    if (total + res.size[i] <= cap) {
      memcpy(litlens + total, res.ll.data() + res.off[i], res.size[i] * 2);
      memcpy(dists + total, res.d.data() + res.off[i], res.size[i] * 2);
    }
    total += res.size[i];
    if (cost) cost[i] = res.cost[i];
  }
  return total <= cap ? 0 : 1;
}

int ZopfliB200LZ77(const unsigned char* in, size_t insize, size_t instart, size_t inend, int mode,
                   int numiterations, unsigned short* litlens, unsigned short* dists, size_t cap, size_t* size) {
  size_t off = 0, cnt = 0;
  int r = ZopfliB200LZ77Batch(in, insize, 1, &instart, &inend, mode, numiterations, litlens, dists, cap, &off, &cnt, nullptr);
  *size = cnt;
  return r;
}

int ZopfliB200MatchTable(const unsigned char* in, size_t insize, size_t instart, size_t inend,
                         unsigned short* length, unsigned short* distance, unsigned short* sublen,
                         unsigned short* same, unsigned short* hashval, unsigned short* hashval2) {
  Engine::Lease lease;
  Engine& e = *lease;
  e.set_input_host(in, insize);
  std::vector<uint16_t> l, d, s, sm, h1, h2;
  e.match_table(instart, inend, l, d, s, sm, h1, h2);
  size_t n = inend - instart;
  if (length) memcpy(length, l.data(), n * 2);
  if (distance) memcpy(distance, d.data(), n * 2);
  if (sublen) memcpy(sublen, s.data(), n * 259 * 2);
  if (same) memcpy(same, sm.data(), n * 2);
  if (hashval) memcpy(hashval, h1.data(), n * 2);
  if (hashval2) memcpy(hashval2, h2.data(), n * 2);
  return 0;
}

uint64_t ZopfliB200DynamicBlockBits(const uint32_t* hist320, int where) {
  if (where == 1) { Engine::Lease e; return e->device_block_bits(hist320); }
  DynScratch s;
  return dynamic_block_bits(hist320, nullptr, nullptr, s);
}

int ZopfliB200DeviceAutoTypeBits(const unsigned short* litlens, const unsigned short* dists, size_t n, size_t nreq,
                                 const size_t* lstart, const size_t* lend, uint64_t* out) {
  Engine::Lease lease;
  Engine& e = *lease;
  std::vector<uint64_t> off{0};
  std::vector<uint32_t> size{(uint32_t)n};
  e.split_begin(litlens, dists, off, size);
  std::vector<Engine::SplitReq> r(nreq);
  for (size_t i = 0; i < nreq; i++) r[i] = {0u, (uint32_t)lstart[i], (uint32_t)lend[i]};
  e.split_eval(r.data(), nreq, out);
  return 0;
}

size_t ZopfliB200HostBlockSplitLZ77(const unsigned char* in, const unsigned short* litlens,
                                    const unsigned short* dists, size_t n, size_t maxblocks, size_t* points,
                                    size_t cap) {
  (void)in;
  Lz77Store st;
  make_store(litlens, dists, n, st);
  // the product's own search (batched_split.hpp) with one store and a serial round: every probe is
  // priced as the reference would, by the host estimators
  std::vector<size_t> p = batched_block_split({st.size()}, maxblocks, [&](const std::vector<EvalReq>& q, std::vector<uint64_t>& c) {
    DynScratch sc;
    for (size_t i = 0; i < q.size(); i++) c[i] = auto_type_bits(st, q[i].lstart, q[i].lend, sc);
  }, 0)[0];
  for (size_t i = 0; i < p.size() && i < cap; i++) points[i] = p[i];
  return p.size();
}

void ZopfliB200HostBatchedSplit(const unsigned short* litlens, const unsigned short* dists, size_t nstores,
                                const size_t* off, const size_t* size, size_t maxblocks, size_t budget,
                                size_t* points, size_t cap, size_t* npoints) {
  std::vector<Lz77Store> st(nstores);
  std::vector<size_t> sizes(nstores);
  for (size_t s = 0; s < nstores; s++) { make_store(litlens + off[s], dists + off[s], size[s], st[s]); sizes[s] = size[s]; }
  std::vector<std::vector<size_t>> r = batched_block_split(sizes, maxblocks, [&](const std::vector<EvalReq>& q, std::vector<uint64_t>& c) {
    DynScratch sc;
    for (size_t i = 0; i < q.size(); i++) c[i] = auto_type_bits(st[q[i].store], q[i].lstart, q[i].lend, sc);
  }, budget);
  for (size_t s = 0; s < nstores; s++) {
    npoints[s] = r[s].size();
    for (size_t i = 0; i < r[s].size() && i < cap; i++) points[s * cap + i] = r[s][i];
  }
}

double ZopfliB200HostBlockSize(const unsigned char* in, const unsigned short* litlens,
                               const unsigned short* dists, size_t n, size_t lstart, size_t lend, int btype) {
  (void)in;
  Lz77Store st;
  make_store(litlens, dists, n, st);
  DynScratch s;
  if (btype < 0) return (double)auto_type_bits(st, lstart, lend, s);
  uint32_t h[320];
  st.range_hist(lstart, lend, h);
  if (btype == 0) return (double)stored_bits(st.byte_range(lstart, lend));
  if (btype == 1) return (double)fixed_block_bits(h);
  return (double)dynamic_block_bits(h, nullptr, nullptr, s);
}

double ZopfliCalculateBlockSize(const ZopfliLZ77Store* lz77, size_t lstart, size_t lend, int btype) {
  return ZopfliB200HostBlockSize(lz77->data, lz77->litlens, lz77->dists, lz77->size, lstart, lend, btype);
}

double ZopfliCalculateBlockSizeAutoType(const ZopfliLZ77Store* lz77, size_t lstart, size_t lend) {
  return ZopfliB200HostBlockSize(lz77->data, lz77->litlens, lz77->dists, lz77->size, lstart, lend, -1);
}

uint64_t ZopfliB200HostEmitBlock(const unsigned char* in, const unsigned short* litlens,
                                 const unsigned short* dists, size_t n, size_t lstart, size_t lend, int btype,
                                 int final, unsigned char* out, size_t cap) {
  (void)in;
  if (lstart > lend || lend > n || (btype != 1 && btype != 2)) return 0;
  BlockPlan plan;
  host_block_plan(litlens + lstart, dists + lstart, lend - lstart, plan);
  const uint64_t want = btype == 2 ? plan.dyn_bits : plan.fixed_bits;
  std::vector<uint8_t> buf((size_t)(want / 8) + 16, 0);
  HostBitSink sink{buf.data(), 0};
  const uint64_t nbits = host_emit_block(btype, final != 0, litlens + lstart, dists + lstart, lend - lstart, &plan, sink);
  if (nbits != want) { fprintf(stderr, "zopfli-b200: emitted %llu bits, predicted %llu\n", (unsigned long long)nbits, (unsigned long long)want); abort(); }
  if ((nbits + 7) / 8 <= cap) memcpy(out, buf.data(), (size_t)((nbits + 7) / 8));
  return nbits;
}

int ZopfliB200HostEmitBlocks(const unsigned char* in, size_t insize, const unsigned short* litlens,
                             const unsigned short* dists, size_t n, size_t npieces, const size_t* lstart,
                             const size_t* lend, const int* btype, const int* final, unsigned bp0,
                             unsigned char* out, size_t cap, uint64_t* nbits, unsigned char* plan_len,
                             uint64_t* plan_val) {
  std::vector<Piece> pieces;
  if (!seam_pieces(insize, litlens, dists, n, npieces, lstart, lend, btype, final, bp0, pieces)) return 1;
  std::vector<BlockPlan> plans(npieces);
  for (size_t i = 0; i < npieces; i++) {
    host_block_plan(litlens + pieces[i].off, dists + pieces[i].off, pieces[i].n, plans[i]);
    seam_plan_out(plans[i], pieces[i], plan_len + i * 320, plan_val + i * 6);
  }
  std::vector<Engine::EmitPiece> ep;
  *nbits = layout_pieces(pieces, 0, bp0, ep, nullptr);
  const size_t nbytes = (size_t)((*nbits + 7) / 8);
  if (nbytes > cap) return 1;
  std::vector<uint8_t> buf(nbytes + 16, 0);
  for (size_t i = 0; i < npieces; i++) {
    const Engine::EmitPiece& e = ep[i];
    HostBitSink sink{buf.data(), e.bit_start};
    if (e.type == 0) {
      host_emit_stored(e.final != 0, in + e.in_start, e.in_len, sink);
      continue;
    }
    const uint64_t nb = host_emit_block(e.type, e.final != 0, litlens + e.off, dists + e.off, e.n, &plans[i], sink);
    if (nb != e.nbits) { fprintf(stderr, "zopfli-b200: emitted %llu bits, predicted %llu\n", (unsigned long long)nb, (unsigned long long)e.nbits); abort(); }
  }
  memcpy(out, buf.data(), nbytes);
  return 0;
}

int ZopfliB200HostLengthLimited(const uint32_t* freq, int n, int maxbits, unsigned* bitlengths) {
  if (n > kNumLL || maxbits > 15) return 1;
  static thread_local PmScratch<kNumLL, 15> s;
  std::vector<uint8_t> out(n);
  length_limited<kNumLL, 15>(freq, n, maxbits, out.data(), s);
  for (int i = 0; i < n; i++) bitlengths[i] = out[i];
  return 0;
}

void ZopfliB200DistShard(size_t insize, int world, int rank, size_t* a, size_t* b, size_t* base) {
  dist_shard(insize, world, rank, a, b, base);
}

void ZopfliB200DistPlacement(const uint64_t* len8, int world, unsigned phase0, uint64_t* start) {
  dist_placement(len8, 8, world, phase0, start);
}

void ZopfliB200HostOptimizeRle(uint32_t* counts, int n) {
  if (n < 0 || n > kNumLL) return;
  uint8_t good[kNumLL];
  optimize_for_rle(n, counts, good);
}

void ZopfliB200HostOptimizeRleBatch(uint32_t* counts, int n, size_t nhist, int by_segments) {
  if (n < 0 || n > kNumLL) return;
  uint8_t good[kNumLL];
  for (size_t h = 0; h < nhist; h++) {
    if (by_segments) optimize_for_rle_by_segments(n, counts + h * n, good);
    else optimize_for_rle(n, counts + h * n, good);
  }
}

void ZopfliB200HostTreeHeaderBits(const uint32_t* clcounts, size_t nvec, int by_huffman, uint32_t* out) {
  for (size_t v = 0; v < nvec; v++)
    out[v] = by_huffman ? tree_header_bits_huffman(clcounts + v * 19) : tree_header_bits(clcounts + v * 19);
}

int ZopfliB200HostProbeParts(const uint32_t* hists, size_t nhist, uint32_t* smoothed, unsigned char* lengths,
                             uint32_t* tree_bits, uint64_t* dyn_bits) {
  static thread_local PmScratch<kNumLL, 15> pm;
  static thread_local DynScratch ds;
  uint8_t good[kNumLL];
  for (size_t h = 0; h < nhist; h++) {
    uint32_t* sm = smoothed + h * 320;
    unsigned char* len = lengths + h * 640;
    uint32_t hist[320];
    memcpy(hist, hists + h * 320, sizeof(hist));
    hist[256] = 1;  // deflate.c:575
    memcpy(sm, hist, sizeof(hist));
    optimize_for_rle(kNumLL, sm, good);
    optimize_for_rle(kNumD, sm + 288, good);
    for (int set = 0; set < 2; set++) {
      const uint32_t* c = set ? sm : hist;
      unsigned char* l = len + set * 320;
      length_limited<kNumLL, 15>(c, kNumLL, 15, l, pm);
      length_limited<kNumLL, 15>(c + 288, kNumD, 15, l + 288, pm);
      patch_distance_codes(l + 288);
      for (int f = 0; f < 8; f++)
        tree_bits[h * 16 + set * 8 + f] = encode_tree_size(l, l + 288, (f & 1) != 0, (f & 2) != 0, (f & 4) != 0);
    }
    dyn_bits[h] = dynamic_block_bits(hist, nullptr, nullptr, ds);
  }
  return 0;
}

void ZopfliB200GetStats(ZopfliB200Stats* o) {
  EngineStats e = Engine::stats_all();
  o->ms_same = e.ms_same; o->ms_keys = e.ms_keys; o->ms_scan = e.ms_scan; o->ms_scatter = e.ms_scatter;
  o->ms_match = e.ms_match; o->ms_greedy = e.ms_greedy; o->ms_iterate = e.ms_iterate; o->ms_pack = e.ms_pack;
  o->ms_h2d = e.ms_h2d; o->ms_d2h = e.ms_d2h;
  o->ms_host_split = g_host_times.split; o->ms_host_emit = g_host_times.emit; o->ms_host_other = g_host_times.other;
  { std::lock_guard<std::mutex> g(g_api_mu); o->ms_total = g_total_ms; }
  o->launches = e.launches; o->match_positions = e.match_positions; o->iterate_positions = e.iterate_positions;
  o->iterate_steps = e.iterate_steps; o->h2d_bytes = e.h2d_bytes; o->d2h_bytes = e.d2h_bytes;
  for (int k = 0; k < 6; k++) { o->cyc_sum[k] = e.cyc_sum[k]; o->cyc_max[k] = e.cyc_max[k]; }
  o->max_block_positions = e.max_block_positions;
  o->ovf_regrows = e.ovf_regrows;
  o->log_regrows = e.log_regrows;
  o->ms_split = e.ms_split; o->split_evals = e.split_evals; o->split_rounds = e.split_rounds;
  o->iterate_launches = e.iterate_launches;
  o->int_steps = e.int_steps;
  for (int k = 0; k < 5; k++) { o->dp_cyc_sum[k] = e.dp_cyc_sum[k]; o->dp_cyc_max[k] = e.dp_cyc_max[k]; }
  for (int k = 0; k < 6; k++) { o->dp_cnt_sum[k] = e.dp_cnt_sum[k]; o->dp_cnt_max[k] = e.dp_cnt_max[k]; }
}

void ZopfliB200ResetStats(void) {
  Engine::reset_stats_all();
  g_host_times = HostTimes();
  { std::lock_guard<std::mutex> g(g_api_mu); g_total_ms = 0; }
}

void ZopfliB200SetStream(void* s) { Engine::Lease e; e->set_stream(s); }
int ZopfliB200Device(void) { Engine::Lease e; return e->device(); }
const char* ZopfliB200Version(void) { return "zopfli-b200 0.1 (ABI libzopfli.so.1, reference 1.0.3)"; }

}  // extern "C"

// Internal interface between the C-ABI layer (api.cpp) and the batched deflate driver.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <atomic>
#include <thread>
#include <utility>
#include <vector>

#include "../../include/zopfli.h"
#include "dist_layout.hpp"
#include "engine.hpp"

namespace zb {

// One deflate block of the output stream.  Compressed blocks live on the device as (store buffer,
// symbol range, plan); their exact bit size is known, so the host can place every block before a bit
// is written.  Stored blocks name input bytes; their size depends on the bit offset (deflate.c:643-649).
struct Piece {
  uint8_t type = 2;          // 0 stored, 1 fixed, 2 dynamic
  bool final = false;
  uint8_t buf = 0;           // Engine::StoreBuf
  uint32_t unit = 0;         // index of the unit (master block) the piece belongs to
  uint32_t n = 0;            // symbols
  uint64_t off = 0;          // first symbol in `buf`
  uint64_t plan = 0;         // Engine::plan_blocks handle (dynamic blocks)
  uint64_t nbits = 0;        // exact size (compressed blocks)
  uint32_t tree_bits = 0;    // dynamic blocks: size of the tree header inside nbits (verbose report only)
  size_t instart = 0, inend = 0;  // stored blocks: absolute input positions
};

// ZopfliB200DeflateSpan's records of a range of units: the driver's pieces, and the records made of them
// (maximal runs of compressed pieces as bits, stored pieces as their payload).  `markers` indexes the pieces
// that are full-flush markers after units that end at a restart point.  The runs are emitted together (ep,
// run_bits bits) into one buffer; until point_records (api.hpp) points the records at their bytes, at[i] says
// where record i's bytes are: a bit record's first bit in that buffer, a stored record's input position.
// `runs` is that buffer when a compressor's staging made it (WaveStaging::take_records; drop_records frees it).
struct SpanRecords {
  std::vector<Piece> pieces;
  std::vector<Engine::SpanRecord> recs;
  std::vector<uint64_t> at;
  std::vector<size_t> markers;
  std::vector<Engine::EmitPiece> ep;
  uint64_t run_bits = 0;
  unsigned char* runs = nullptr;
};

struct HostTimes { double split = 0, emit = 0, other = 0; };
extern HostTimes g_host_times;

// steady clock in milliseconds, for the stats and the ZOPFLI_B200_DEBUG timeline
double now_ms();
// ZOPFLI_B200_DEBUG=1: timeline of the chunk pipelines and the API calls on stderr
bool debug_on();

// Host threads the library's CPU work may use: ZOPFLI_B200_THREADS, else the CPUs of the affinity mask and
// the cgroup CPU quota (at most 32), shared among the LOCAL_WORLD_SIZE ranks of a box.
int host_threads();

// fn(0) ... fn(n - 1) on up to host_threads() threads, each taking the next index as it becomes free
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

// Compresses the given units of the input (dist_layout.hpp Unit: master blocks, or the single range of a
// ZopfliDeflatePart call, each with its floor); the engine must already hold its bytes [in_base ...).  Every
// parse of a unit sees no byte before the unit's floor.
void deflate_units(Engine& eng, const ZopfliOptions* opt, int btype, bool final_last, const std::vector<Unit>& units,
                   size_t in_base, std::vector<Piece>& pieces);

// Master blocks that deflate_units runs at once on a device with this much memory (chunk pipelines x batch,
// both from its schedule): the wave of a long ZopfliCompress call.  ZopfliB200Compressor asks for half the
// device, so that its two waves in flight fit the budget of one call.
size_t wave_master_blocks(uint64_t device_memory);

// Places the pieces behind the caller's stream (bit phase *bp), emits them on the device and appends
// the bytes to *out.  unit_bits (optional) receives the bit offset of every unit's first piece relative
// to the first bit written, plus the end offset as last entry.
void assemble(Engine& eng, const std::vector<Piece>& pieces, size_t in_base, unsigned char* bp, unsigned char** out,
              size_t* outsize, std::vector<uint64_t>* unit_bits = nullptr, bool verbose = false);

// assemble() up to the emission: layout_pieces from bit `phase`, plus the per-block verbose report
uint64_t place_pieces(const std::vector<Piece>& pieces, size_t in_base, unsigned phase, std::vector<Engine::EmitPiece>& ep,
                      std::vector<uint64_t>* unit_bits, bool verbose);

// bit position of every piece when the first one starts at bit0; returns the end position
uint64_t layout_pieces(const std::vector<Piece>& pieces, size_t in_base, uint64_t bit0, std::vector<Engine::EmitPiece>& ep,
                       std::vector<uint64_t>* unit_bits);

// Where span records go when the first starts at bit0: fills in every record's bit_start and returns the end.
// The one placement of records, for the host splice below and the device splice (k_splice).
uint64_t span_positions(std::vector<Engine::SpanRecord>& recs, uint64_t bit0);

// Appends the records, their src in host memory, to a zopfli-style buffer at its bit phase *bp.
void splice_pieces(std::vector<Engine::SpanRecord>& recs, unsigned char* bp, unsigned char** out, size_t* outsize);

// Grows a zopfli-style buffer by n bytes under its capacity rule (util.h:134-155) and returns where they go.
unsigned char* append_reserve(size_t n, unsigned char** out, size_t* outsize);
void append_bytes(const unsigned char* src, size_t n, unsigned char** out, size_t* outsize);

// Appends nbytes of stream whose first bit sits at bit `phase` of the caller's last byte (0: a fresh byte).
// write(dst) fills all nbytes at dst; with a phase dst[0] is the caller's partly filled last byte, whose
// bits are ORed back in afterwards.
template <typename Write>
void append_stream(size_t nbytes, unsigned phase, unsigned char** out, size_t* outsize, Write write) {
  const unsigned char keep = phase ? (*out)[*outsize - 1] : 0;
  append_reserve(phase ? nbytes - 1 : nbytes, out, outsize);
  unsigned char* dst = *out + *outsize - nbytes;
  write(dst);
  dst[0] |= keep;
}

}  // namespace zb

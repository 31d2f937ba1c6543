// What the C-ABI sources share: api.cpp (every call with host-side results) and device_api.cpp (input
// and result in device memory).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "../../include/zopfli.h"
#include "engine.hpp"

namespace zb {

struct BlockPlan;
struct Piece;
struct SpanRecords;
struct Unit;

// ZopfliB200DeflateSpan's body: the units of the input (master blocks, each with its floor), whose bytes from
// position `base` on the engine already holds, as span records; after every unit marked `restart` comes a sync
// marker (an empty stored block of BFINAL 0).  The runs of compressed blocks are laid out, not yet emitted.
void deflate_span_records(Engine& eng, const ZopfliOptions* opt, size_t base, const std::vector<Unit>& units,
                          bool final, SpanRecords& out);
// Points the records at their bytes once the runs are emitted: bit records into `runs`, the emission of sr.ep,
// stored records at their payload in `in`, the input bytes from position `base` on.
void point_records(SpanRecords& sr, const unsigned char* runs, const unsigned char* in, size_t base);

// A span of ZopfliB200AppendSpan's format as records that point into it; false, with nothing parsed, when it
// is malformed.
bool parse_span(const unsigned char* span, size_t spansize, std::vector<Engine::SpanRecord>& recs);

// Where a compressor (ZopfliB200Compressor) keeps the bytes of its waves and of the stream it has not returned
// yet: host memory here, device memory in device_api.cpp.  Slot s holds stream bytes from the slot's base on;
// it grows as bytes are put into it.
struct WaveStaging {
  static constexpr int kSlots = 3;  // two waves in flight and one filling
  size_t slot_bytes = 0;            // the most a slot holds: one wave and its dictionary (set by the compressor)
  virtual ~WaveStaging() {}
  virtual int device() const = 0;  // -1: host memory
  // whether a chunk of n bytes at p is memory of the kind this staging takes
  virtual bool accepts(const void* p, size_t n) const = 0;
  // slot s, offset off <- chunk[0, n) (the caller may reuse the chunk when put returns)
  virtual void put(int s, size_t off, const unsigned char* chunk, size_t n) = 0;
  // slot to, offset 0 <- slot from, bytes [off, off + n): the dictionary a wave takes over from the one before
  virtual void carry(int from, size_t off, int to, size_t n) = 0;
  // on a wave's worker, holding eng: slot s's bytes [0, len) become the engine's input
  virtual void stage(Engine& eng, int s, size_t len) = 0;
  // CRC-32 / Adler-32 (ChecksumKind) of slot s's bytes [off, off + n), with the engine set up by stage()
  virtual uint32_t checksum(Engine& eng, int s, size_t off, size_t n, int kind) = 0;
  // on a wave's worker, holding eng: emits the runs of slot s's records (base: position of the slot's byte 0)
  // into a buffer of sr.runs, in memory of the staging's kind, and points the records there, stored ones at
  // their payload in the slot.
  virtual void take_records(Engine& eng, int s, size_t base, SpanRecords& sr) = 0;
  // frees what take_records allocated
  virtual void drop_records(SpanRecords& sr) = 0;
  // CRC-32 / Adler-32 of n bytes at p, memory of the kind this staging takes (a preset dictionary)
  virtual uint32_t checksum_of(const unsigned char* p, size_t n, int kind) = 0;

  // ---- the stream not yet returned: at most the partly filled last byte between calls ----
  // bits in use in the stream's last byte (0: none, or it is full)
  virtual unsigned phase() const = 0;
  // n whole bytes behind the stream's last byte (the container header and trailer)
  virtual void put_bytes(const unsigned char* p, size_t n) = 0;
  // records at the stream's bit phase, from the bytes take_records pointed them at
  virtual void splice(SpanRecords& sr) = 0;
  // Returns the complete bytes (all of them with `all`) and their count: appended zopfli-style to *out, or with
  // to_device (device staging only) as a fresh allocation *out of exactly *outsize bytes, NULL when there are none.
  virtual size_t hand_out(bool all, bool to_device, unsigned char** out, size_t* outsize) = 0;
};
// The device side of ZopfliB200CompressorNew, registered by device_api.cpp (null in a host-only build): a
// staging on device dev, ordered after cuda_stream, or null when dev is not a usable device.
extern WaveStaging* (*g_device_staging)(int dev, void* cuda_stream);
// device that owns p, else -1 (always -1 in a host-only build)
extern int (*g_pointer_device)(const void* p);

// a compression call that started at t0 (now_ms) is done: `layout` becomes what
// ZopfliB200LastMasterBitOffsets returns, and the call's time is added to ZopfliB200Stats::ms_total
void api_call_done(std::vector<uint64_t>& layout, double t0);
// the ChecksumKind of the trailer an output format carries (kCkNone for raw deflate), or -1 for a value
// that is not a ZopfliFormat
int trailer_kind(ZopfliFormat fmt);
// header bytes of the gzip or zlib container (at most 10); 0 for raw deflate.  With dictid, the zlib header
// of a stream with a preset dictionary: FDICT set and the dictionary's Adler-32 (RFC 1950, 2.2).
int container_header(ZopfliFormat fmt, unsigned char* hdr, const uint32_t* dictid = nullptr);
// the verbose reports of a whole compression in the reference's formats: the deflate body's
// (deflate_bytes), then with a gzip / zlib container the container's (outsize = the whole output)
void report_sizes(ZopfliFormat fmt, size_t insize, size_t deflate_bytes, size_t outsize);
// The pieces of ZopfliB200{Device,Host}EmitBlocks as the driver describes blocks (kFin symbols, input bytes
// for stored pieces); plan and nbits are filled in by the caller.  False if bp0 > 7, a symbol is not a valid
// literal / (length, distance), a range lies outside the store, or the store covers more than insize bytes.
bool seam_pieces(size_t insize, const unsigned short* ll, const unsigned short* d, size_t n, size_t npieces,
                 const size_t* lstart, const size_t* lend, const int* btype, const int* final, unsigned bp0,
                 std::vector<Piece>& pieces);
// one BlockPlan as the seams' flat arrays (288 + 32 code lengths; tree flags, tree bits, dynamic, fixed and
// stored bits, bytes), and the size of piece p under its block type
void seam_plan_out(const BlockPlan& b, Piece& p, unsigned char* len320, uint64_t* val6);

}  // namespace zb

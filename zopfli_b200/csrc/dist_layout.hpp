// Pure arithmetic of cutting an input into master blocks and of the multi-GPU path (dist.cpp), kept apart
// so it can be tested without GPUs or NCCL (tests/test_sharding_gloo.py drives it over gloo): which bytes
// a rank owns, and where every rank's bits land in the one output stream.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <utility>
#include <vector>

#include "symbols.hpp"

namespace zb {

inline size_t dist_num_master_blocks(size_t insize) {  // deflate.c:912-924 do/while
  return insize == 0 ? 1 : (insize + kMasterBlock - 1) / kMasterBlock;
}

// A unit of the driver (deflate_units): a master block, or the single range of a ZopfliDeflatePart call.  Its
// bytes [a, b) are parsed seeing no byte before `floor` (squeeze.c:229-230 on the input from floor on).  In a
// compressor's wave, `restart` marks a unit that ends at a restart point: the full-flush marker follows it.
struct Unit {
  size_t a, b;
  size_t floor = 0;
  bool restart = false;
};

// The master blocks of bytes [a, b) (deflate.c:912-924): kMasterBlock bytes each from a, the last one
// shorter.  The do/while makes an empty range one empty master block.
inline std::vector<Unit> master_blocks(size_t a, size_t b) {
  std::vector<Unit> u;
  do {
    u.push_back({a, b - a > (size_t)kMasterBlock ? a + kMasterBlock : b});
    a = u.back().b;
  } while (a < b);
  return u;
}

// The first restart point past position p of a compressor with restart interval `interval` (0: none) whose
// data starts at position d: the points are d + k * interval, k >= 1.  SIZE_MAX when there is none.
inline size_t next_restart(size_t p, size_t d, size_t interval) {
  if (interval == 0) return SIZE_MAX;
  const size_t k = p < d ? 1 : (p - d) / interval + 1;
  size_t r;
  if (__builtin_mul_overflow(k, interval, &r) || __builtin_add_overflow(r, d, &r)) return SIZE_MAX;
  return r;
}

// The next wave of a compressor fed in pieces (ZopfliB200Compressor): `received` bytes have arrived,
// `handed` of them already belong to waves, no byte before `floor` may be seen at `handed`, and restart points
// lie at d + k * interval (next_restart).  Segments are cut at flush points (every wave ends at one) and at
// restart points; units are the master blocks of segments, counted from the segment's start, so from `handed`
// and from every restart point inside the wave.  A unit that ends at a restart point before `received` carries
// `restart`: the automatic full flush there is due once a byte past it has arrived.  The units after it have
// that point as their floor, and floor_end is the floor at b.
// While writing (kWaveWrite) a wave is the next wave_blocks whole units, released only once a byte past them
// has arrived, because the last unit's BFINAL depends on whether more input follows.  At Finish (kWaveFinish)
// everything left is one final wave (an empty stream or segment: one empty unit).  At a flush (kWaveFlush)
// everything left is one wave that is not final, or none when nothing is left.  Returns false when no wave is
// ready.  After a final wave there is none.
struct Wave {
  size_t a, b;
  bool final;
  size_t floor_end;
  std::vector<Unit> units;
};
enum WaveCall { kWaveWrite = 0, kWaveFinish = 1, kWaveFlush = 2 };
inline bool next_wave(size_t received, int call, size_t handed, size_t floor, size_t d, size_t interval,
                      size_t wave_blocks, Wave* w) {
  if (call == kWaveFlush && received <= handed) return false;
  const size_t nb = wave_blocks < 1 ? 1 : wave_blocks;
  std::vector<Unit> u;
  size_t p = handed;
  do {
    const size_t r = next_restart(p, d, interval);
    size_t e = std::min(p + (size_t)kMasterBlock, r);
    if (call == kWaveWrite && e >= received) return false;
    e = std::min(e, received);
    const bool restart = e == r && r < received;
    u.push_back({p, e, floor, restart});
    if (restart) floor = e;
    p = e;
  } while (call == kWaveWrite ? u.size() < nb : p < received);
  w->a = handed;
  w->b = p;
  w->final = call == kWaveFinish;
  w->floor_end = floor;
  w->units.swap(u);
  return true;
}

// Where a wave's staged bytes start: the 32 KiB dictionary in front of byte a (squeeze.c:229-230), rounded
// down to 16 bytes for the kernels' vector loads, as ZopfliB200DeflateSpan and dist_shard stage it.  With a
// floor (a compressor's last full flush) no byte before it is staged: the parse then sees none of them.
inline size_t wave_base(size_t a, size_t floor = 0) {
  const size_t b = a > (size_t)kWindow ? (a - kWindow) & ~(size_t)15 : 0;
  return b > floor ? b : floor;
}

// Rank `rank` of `world` owns the master blocks [rank*nm/world, (rank+1)*nm/world): bytes [a, b).  Its
// device copy starts at `base` <= a: the 32 KiB dictionary in front of the shard (squeeze.c:229-230),
// rounded down to 16 bytes for the vector loads of the kernels.  Ranks without a master block get a == b.
inline void dist_shard(size_t insize, int world, int rank, size_t* a, size_t* b, size_t* base) {
  const size_t nm = dist_num_master_blocks(insize);
  const size_t lo = (size_t)rank * nm / (size_t)world, hi = (size_t)(rank + 1) * nm / (size_t)world;
  *a = lo * (size_t)kMasterBlock < insize ? lo * (size_t)kMasterBlock : insize;
  *b = hi * (size_t)kMasterBlock < insize ? hi * (size_t)kMasterBlock : insize;
  *base = *a > (size_t)kWindow ? (*a - kWindow) & ~(size_t)15 : 0;
  if (lo == hi) *base = *a = *b;
}

// len8[r*stride + p] = bits rank r's blocks occupy when its first bit sits at bit phase p (stored blocks pad
// to a byte boundary, deflate.c:643-649, so the length depends on the phase).  start[0] = phase0 and
// start[r+1] = start[r] + len8[r][start[r] & 7]: absolute bit offsets counted from bit 0 of the byte that
// holds the caller's phase0 bits.
inline void dist_placement(const uint64_t* len8, size_t stride, int world, unsigned phase0, uint64_t* start) {
  start[0] = phase0 & 7u;
  for (int r = 0; r < world; r++) start[r + 1] = start[r] + len8[(size_t)r * stride + (start[r] & 7)];
}

// bytes of the stream rank r's bits touch, counted from the byte of its first bit
inline size_t dist_bytes_touched(const uint64_t* start, int r) {
  if (start[r + 1] == start[r]) return 0;
  return (size_t)(((start[r] & 7) + (start[r + 1] - start[r]) + 7) / 8);
}

}  // namespace zb

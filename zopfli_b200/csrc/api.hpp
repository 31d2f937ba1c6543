// What the C-ABI sources share: api.cpp (every call with host-side results) and device_api.cpp (input
// and result in device memory).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <utility>
#include <vector>

#include "../../include/zopfli.h"

namespace zb {

struct BlockPlan;
struct Piece;

double api_now_ms();
// the master blocks (deflate.c:908-931) of an insize-byte input, as ZopfliCompress cuts it
std::vector<std::pair<size_t, size_t>> api_master_units(size_t insize);
// a compression call that started at t0 (api_now_ms) is done: `layout` becomes what
// ZopfliB200LastMasterBitOffsets returns, and the call's time is added to ZopfliB200Stats::ms_total
void api_call_done(std::vector<uint64_t>& layout, double t0);
// header bytes of the gzip or zlib container (at most 10); 0 for raw deflate
int container_header(ZopfliFormat fmt, unsigned char* hdr);
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

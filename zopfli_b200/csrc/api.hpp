// What the C-ABI sources share: api.cpp (every call with host-side results) and device_api.cpp (input
// and result in device memory).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <utility>
#include <vector>

#include "../../include/zopfli.h"

namespace zb {

double api_now_ms();
// the master blocks (deflate.c:908-931) of an insize-byte input, as ZopfliCompress cuts it
std::vector<std::pair<size_t, size_t>> api_master_units(size_t insize);
// a compression call that started at t0 (api_now_ms) is done: `layout` becomes what
// ZopfliB200LastMasterBitOffsets returns, and the call's time is added to ZopfliB200Stats::ms_total
void api_call_done(std::vector<uint64_t>& layout, double t0);
// header bytes of the gzip or zlib container (at most 10); 0 for raw deflate
int container_header(ZopfliFormat fmt, unsigned char* hdr);

}  // namespace zb

// C-ABI of libzopfli.so.1 (zopfli-b200): the reference's public entry points
// (/root/reference/src/zopfli/zopfli.h, deflate.h, gzip_container.h, zlib_container.h) plus the
// seams declared in include/zopfli_b200.h.  The calls whose input and result live in device memory are
// in device_api.cpp.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
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

double now_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}
std::mutex g_api_mu;   // guards g_total_ms and g_last_layout
double g_total_ms = 0;
std::vector<uint64_t> g_last_layout;  // bit offset of every unit (master block) of the most recent deflate call

}  // namespace

namespace zb {

double api_now_ms() { return now_ms(); }

void api_call_done(std::vector<uint64_t>& layout, double t0) {
  std::lock_guard<std::mutex> g(g_api_mu);
  g_last_layout.swap(layout);
  g_total_ms += now_ms() - t0;
}

// header bytes of the gzip (gzip_container.c:95-104) or zlib (zlib_container.c:58-64) container; 0 for raw deflate
int container_header(ZopfliFormat fmt, unsigned char* hdr) {
  if (fmt == ZOPFLI_FORMAT_GZIP) {
    static const unsigned char gz[10] = {31, 139, 8, 0, 0, 0, 0, 0, 2, 3};
    memcpy(hdr, gz, 10);
    return 10;
  }
  if (fmt == ZOPFLI_FORMAT_ZLIB) {
    unsigned cmfflg = 256 * 120 + 3 * 64;
    cmfflg += 31 - cmfflg % 31;
    hdr[0] = (unsigned char)(cmfflg / 256);
    hdr[1] = (unsigned char)(cmfflg % 256);
    return 2;
  }
  return 0;
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

}  // namespace zb

namespace {

// ---- CRC-32 (gzip_container.c:27-81 computes the same polynomial bytewise): slicing-by-8 ----
uint32_t g_crc_tab[8][256];
std::once_flag g_crc_once;
void crc_fill() {
  for (uint32_t i = 0; i < 256; i++) g_crc_tab[0][i] = crc_table_entry(0, i);
  for (uint32_t i = 0; i < 256; i++)
    for (int t = 1; t < 8; t++) g_crc_tab[t][i] = (g_crc_tab[t - 1][i] >> 8) ^ g_crc_tab[0][g_crc_tab[t - 1][i] & 255];
}
void crc_init() { std::call_once(g_crc_once, crc_fill); }
uint32_t crc32_range(const unsigned char* p, size_t n, uint32_t crc) {  // crc is the running (inverted) state
  while (n && ((uintptr_t)p & 7)) { crc = g_crc_tab[0][(crc ^ *p++) & 255] ^ (crc >> 8); n--; }
  while (n >= 8) {
    uint64_t v;
    memcpy(&v, p, 8);
    uint32_t lo = (uint32_t)v ^ crc, hi = (uint32_t)(v >> 32);
    crc = g_crc_tab[7][lo & 255] ^ g_crc_tab[6][(lo >> 8) & 255] ^ g_crc_tab[5][(lo >> 16) & 255] ^
          g_crc_tab[4][lo >> 24] ^ g_crc_tab[3][hi & 255] ^ g_crc_tab[2][(hi >> 8) & 255] ^
          g_crc_tab[1][(hi >> 16) & 255] ^ g_crc_tab[0][hi >> 24];
    p += 8;
    n -= 8;
  }
  while (n--) crc = g_crc_tab[0][(crc ^ *p++) & 255] ^ (crc >> 8);
  return crc;
}
uint32_t crc32_parallel(const unsigned char* p, size_t n) {
  crc_init();
  unsigned nt = std::thread::hardware_concurrency();
  if (nt < 1) nt = 1;
  if (nt > 16) nt = 16;
  if (n < (4u << 20) || nt == 1) return crc32_range(p, n, 0xffffffffu) ^ 0xffffffffu;
  std::vector<uint32_t> part(nt);
  std::vector<std::thread> th;
  size_t chunk = (n + nt - 1) / nt;
  for (unsigned t = 0; t < nt; t++)
    th.emplace_back([&, t] {
      size_t a = t * chunk, b = a + chunk > n ? n : a + chunk;
      part[t] = a < b ? (crc32_range(p + a, b - a, 0xffffffffu) ^ 0xffffffffu) : 0;
    });
  for (auto& t : th) t.join();
  uint32_t crc = part[0];
  for (unsigned t = 1; t < nt; t++) {
    size_t a = t * chunk, b = a + chunk > n ? n : a + chunk;
    if (a < b) crc = crc32_combine(crc, part[t], b - a);
  }
  return crc;
}

// ---- Adler-32 (zlib_container.c:29-48 computes it serially) ----
// s1 = 1 + sum(d_i), s2 = sum over i of s1 after byte i (both mod 65521).  Sums of byte values and of
// position-weighted byte values are associative, so chunks (adler_chunk, checksum.hpp) are summed by
// threads and combined below.
uint32_t adler32(const unsigned char* data, size_t size) {
  unsigned nt = std::thread::hardware_concurrency();
  if (nt < 1) nt = 1;
  if (nt > 16) nt = 16;
  if (size < (4u << 20)) nt = 1;
  std::vector<AdlerPart> part(nt);
  const size_t chunk = (size + nt - 1) / nt;
  std::vector<std::thread> th;
  for (unsigned t = 1; t < nt; t++)
    th.emplace_back([&, t] {
      const size_t a = std::min(size, t * chunk), b = std::min(size, a + chunk);
      part[t] = adler_chunk(data + a, b - a);
    });
  part[0] = adler_chunk(data, std::min(size, chunk));
  for (auto& t : th) t.join();
  // with a = sum of bytes and b = sum of prefix sums (both without the initial 1):
  //   a(A|B) = a(A) + a(B),  b(A|B) = b(A) + len(B) * a(A) + b(B);  the initial s1 = 1 adds `size` to s2
  uint64_t a = 0, b = 0;
  for (unsigned t = 0; t < nt; t++) {
    b = (b + (part[t].len % 65521) * a + part[t].s2) % 65521;
    a = (a + part[t].s1) % 65521;
  }
  const uint64_t s1 = (1 + a) % 65521, s2 = (b + size % 65521) % 65521;
  return (uint32_t)((s2 << 16) | s1);
}

std::vector<std::pair<size_t, size_t>> master_units(size_t insize, size_t mb_begin, size_t mb_end) {
  std::vector<std::pair<size_t, size_t>> u;
  for (size_t m = mb_begin; m < mb_end; m++) {
    size_t a = m * (size_t)kMasterBlock, b = a + kMasterBlock;
    if (b > insize) b = insize;
    u.push_back({a, b});
  }
  return u;
}
size_t num_master_blocks(size_t insize) {  // deflate.c:912-924 do/while
  return insize == 0 ? 1 : (insize + kMasterBlock - 1) / kMasterBlock;
}

}  // namespace

std::vector<std::pair<size_t, size_t>> zb::api_master_units(size_t insize) {
  return master_units(insize, 0, num_master_blocks(insize));
}

namespace {

bool api_debug() {
  static int v = [] { const char* e = getenv("ZOPFLI_B200_DEBUG"); return e && atoi(e) ? 1 : 0; }();
  return v != 0;
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
  deflate_units(*eng, options, btype, final != 0, in, master_units(insize, 0, num_master_blocks(insize)), 0, pieces);
  const double t2 = now_ms();
  std::vector<uint64_t> layout;
  assemble(*eng, pieces, 0, bp, out, outsize, &layout, options->verbose != 0);
  { std::lock_guard<std::mutex> g(g_api_mu); g_last_layout.swap(layout); }
  if (api_debug())
    fprintf(stderr, "[zb] api: set_input %.1f ms, deflate_units %.1f ms, emit %.1f ms\n", t1 - t0, t2 - t1, now_ms() - t2);
  if (options->verbose) {
    fprintf(stderr, "Original Size: %lu, Deflate: %lu, Compression: %f%% Removed\n", (unsigned long)insize,
            (unsigned long)(*outsize - offset), 100.0 * (double)(insize - (*outsize - offset)) / (double)insize);
  }
  { std::lock_guard<std::mutex> g(g_api_mu); g_total_ms += now_ms() - t0; }
}

// the containers (gzip_container.c:84-124, zlib_container.c:50-79) around a deflate body produced by `body`
template <typename Body>
void container_impl(const ZopfliOptions* options, ZopfliFormat fmt, const unsigned char* in, size_t insize,
                    unsigned char** out, size_t* outsize, Body deflate_impl_fn);

void compress_impl(const ZopfliOptions* options, ZopfliFormat fmt, const unsigned char* in, size_t insize,
                   const unsigned char* dev_in, unsigned char** out, size_t* outsize) {
  container_impl(options, fmt, in, insize, out, outsize, [&](unsigned char* bp) {
    deflate_impl(options, 2, 1, in, insize, dev_in, bp, out, outsize);
  });
}

template <typename Body>
void container_impl(const ZopfliOptions* options, ZopfliFormat fmt, const unsigned char* in, size_t insize,
                    unsigned char** out, size_t* outsize, Body body) {
  unsigned char bp = 0;
  unsigned char hdr[10];
  if (fmt == ZOPFLI_FORMAT_GZIP) {  // gzip_container.c:84-124
    uint32_t crc = 0;
    std::thread crc_thread([&] { crc = crc32_parallel(in, insize); });  // overlaps the GPU work
    append_bytes(hdr, container_header(fmt, hdr), out, outsize);
    body(&bp);
    const double tj = now_ms();
    crc_thread.join();
    if (api_debug()) fprintf(stderr, "[zb] api: crc join waited %.1f ms\n", now_ms() - tj);
    unsigned char tr[8] = {(unsigned char)(crc & 255), (unsigned char)((crc >> 8) & 255),
                           (unsigned char)((crc >> 16) & 255), (unsigned char)((crc >> 24) & 255),
                           (unsigned char)(insize & 255), (unsigned char)((insize >> 8) & 255),
                           (unsigned char)((insize >> 16) & 255), (unsigned char)((insize >> 24) & 255)};
    append_bytes(tr, 8, out, outsize);
    if (options->verbose)
      fprintf(stderr, "Original Size: %d, Gzip: %d, Compression: %f%% Removed\n", (int)insize, (int)*outsize,
              100.0 * (double)(insize - *outsize) / (double)insize);
  } else if (fmt == ZOPFLI_FORMAT_ZLIB) {  // zlib_container.c:50-79
    uint32_t checksum = 0;
    std::thread adler_thread([&] { checksum = adler32(in, insize); });  // overlaps the GPU work
    append_bytes(hdr, container_header(fmt, hdr), out, outsize);
    body(&bp);
    adler_thread.join();
    unsigned char tr[4] = {(unsigned char)((checksum >> 24) & 255), (unsigned char)((checksum >> 16) & 255),
                           (unsigned char)((checksum >> 8) & 255), (unsigned char)(checksum & 255)};
    append_bytes(tr, 4, out, outsize);
    if (options->verbose)
      fprintf(stderr, "Original Size: %d, Zlib: %d, Compression: %f%% Removed\n", (int)insize, (int)*outsize,
              100.0 * (double)(insize - *outsize) / (double)insize);
  } else if (fmt == ZOPFLI_FORMAT_DEFLATE) {
    body(&bp);
  } else {
    fprintf(stderr, "zopfli-b200: unknown output format %d\n", (int)fmt);  // zopfli_lib.c:40 assert(0)
    abort();
  }
}

void make_store(const unsigned short* ll, const unsigned short* dd, size_t n, Lz77Store& st) {
  st.append(ll, dd, n, 0);
  st.finalize();
}

}  // namespace

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
  deflate_units(*eng, options, btype, final != 0, in, {{instart, inend}}, base, pieces);
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
  std::vector<Piece> pieces;
  std::vector<std::pair<size_t, size_t>> units;
  if (end > insize || start > end) return 1;
  for (size_t a = start; a < end; a += kMasterBlock) units.push_back({a, a + kMasterBlock < end ? a + kMasterBlock : end});
  if (units.empty() && insize == 0) units.push_back({0, 0});
  if (units.empty()) return 0;
  size_t base = 0;
  Engine::Lease eng;
  if (dev_in) {
    eng->set_input_device(dev_in, insize);
  } else {
    base = start > (size_t)kWindow ? start - kWindow : 0;
    base &= ~(size_t)15;
    eng->set_input_host(in + base, end - base);
  }
  deflate_units(*eng, options, 2, final != 0, in, units, base, pieces);
  // Records: maximal runs of compressed pieces, each emitted on the device from bit offset 0 of a
  // byte-aligned slot of one download buffer, and stored pieces as raw bytes.
  struct Rec { bool stored; bool final; size_t first, count; uint64_t bit0, nbits; };
  std::vector<Rec> recs;
  std::vector<Engine::EmitPiece> ep_all;
  uint64_t pos = 0;
  for (size_t i = 0; i < pieces.size();) {
    if (pieces[i].type == 0) { recs.push_back({true, pieces[i].final, i, 1, 0, 0}); i++; continue; }
    size_t j = i;
    while (j < pieces.size() && pieces[j].type != 0) j++;
    std::vector<Piece> run(pieces.begin() + i, pieces.begin() + j);
    std::vector<Engine::EmitPiece> ep;
    const uint64_t end = layout_pieces(run, base, pos, ep, nullptr);
    recs.push_back({false, pieces[j - 1].final, i, j - i, pos, end - pos});
    ep_all.insert(ep_all.end(), ep.begin(), ep.end());
    pos = (end + 63) & ~(uint64_t)63;  // the next run starts on a fresh word: no shared bytes between records
    i = j;
  }
  std::vector<unsigned char> bits((size_t)(pos / 8) + 8, 0);
  if (pos) eng->emit(ep_all, pos, bits.data());
  size_t total = 0;
  for (const Rec& r : recs) total += 10 + (r.stored ? pieces[r.first].inend - pieces[r.first].instart : (size_t)((r.nbits + 7) / 8));
  unsigned char* d = append_reserve(total, span, spansize);
  for (const Rec& r : recs) {
    d[0] = r.stored ? 1 : 0;
    d[1] = r.final ? 1 : 0;
    const uint64_t v = r.stored ? (uint64_t)(pieces[r.first].inend - pieces[r.first].instart) : r.nbits;
    memcpy(d + 2, &v, 8);
    const size_t nb = r.stored ? (size_t)v : (size_t)((v + 7) / 8);
    if (r.stored) memcpy(d + 10, in + pieces[r.first].instart, nb);
    else memcpy(d + 10, bits.data() + r.bit0 / 8, nb);
    d += 10 + nb;
  }
  return 0;
}

uint32_t ZopfliB200Crc32(const unsigned char* data, size_t size) { return crc32_parallel(data, size); }
uint32_t ZopfliB200Crc32Combine(uint32_t crc1, uint32_t crc2, uint64_t len2) { return crc32_combine(crc1, crc2, len2); }
uint32_t ZopfliB200Adler32(const unsigned char* data, size_t size) { return adler32(data, size); }
uint32_t ZopfliB200HostChecksumSliced(const unsigned char* data, size_t size, size_t slice_bytes, int kind) {
  return checksum_sliced(data, size, slice_bytes, kind);
}

int ZopfliB200AppendSpan(const unsigned char* span, size_t spansize, unsigned char* bp, unsigned char** out,
                         size_t* outsize) {
  std::vector<SpanPiece> pieces;
  std::vector<unsigned char> rawbytes;  // stored payloads, addressed through instart/inend
  size_t o = 0;
  // validate the whole span before touching the output: spans arrive over a transport
  while (o < spansize) {
    if (spansize - o < 10 || span[o] > 1 || span[o + 1] > 1) return 1;
    uint64_t v;
    memcpy(&v, span + o + 2, 8);
    const uint64_t nbytes = span[o] == 1 ? v : (v + 7) / 8;
    if (nbytes > spansize - o - 10) return 1;
    o += 10 + (size_t)nbytes;
  }
  o = 0;
  // first pass: collect stored payloads contiguously so Piece offsets can index one buffer
  while (o + 10 <= spansize) {
    uint64_t v;
    memcpy(&v, span + o + 2, 8);
    bool stored = span[o] == 1;
    size_t nbytes = stored ? (size_t)v : (size_t)((v + 7) / 8);
    SpanPiece p;
    p.stored = stored;
    p.final = span[o + 1] != 0;
    if (stored) {
      p.instart = rawbytes.size();
      rawbytes.insert(rawbytes.end(), span + o + 10, span + o + 10 + nbytes);
      p.inend = rawbytes.size();
    } else {
      p.bits.bytes.assign(span + o + 10, span + o + 10 + nbytes);
      p.bits.nbits = v;
    }
    pieces.push_back(std::move(p));
    o += 10 + nbytes;
  }
  splice_pieces(pieces, rawbytes.data(), bp, out, outsize);
  return 0;
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

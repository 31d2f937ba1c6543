/*
 * zopfli_b200.h -- additional C-ABI entry points of libzopfli.so.1 (zopfli-b200 build).
 *
 * These expose the hot-path seams the reference keeps internal, for parity tests, the bench
 * harness and multi-GPU sharding.  Plain pointers and sizes only.  Each cites the reference
 * function whose result it returns (paths relative to /root/reference/src/zopfli/).
 * All functions return 0 on success; CUDA failures abort (no CPU fallback exists).
 */
#ifndef ZOPFLI_B200_EXTRA_H_
#define ZOPFLI_B200_EXTRA_H_

#include <stddef.h>
#include <stdint.h>

#include "zopfli.h"

#ifdef __cplusplus
extern "C" {
#endif

/* LZ77 parse of in[instart, inend) with in[max(0,instart-32768), instart) as dictionary.
 * mode 0: ZopfliLZ77Optimal (squeeze.h:41-44) with `numiterations`;
 * mode 1: ZopfliLZ77OptimalFixed (squeeze.h:56-59);
 * mode 2: ZopfliLZ77Greedy (lz77.h:136-138).
 * Writes up to cap symbols (dists[i]==0 => literal litlens[i]) and the symbol count. */
int ZopfliB200LZ77(const unsigned char* in, size_t insize, size_t instart, size_t inend, int mode,
                   int numiterations, unsigned short* litlens, unsigned short* dists, size_t cap,
                   size_t* size);

/* Batched form: n ranges of one input parsed in one device pass.  off[i]/cnt[i] locate the
 * symbols of range i inside litlens/dists (total capacity cap); cost[i] (may be NULL) receives
 * the exact dynamic-block bit size of the returned parse (ZopfliCalculateBlockSize btype 2,
 * deflate.h:79-80) for mode 0. */
int ZopfliB200LZ77Batch(const unsigned char* in, size_t insize, size_t n, const size_t* instart,
                        const size_t* inend, int mode, int numiterations, unsigned short* litlens,
                        unsigned short* dists, size_t cap, size_t* off, size_t* cnt,
                        uint64_t* cost);

/* ZopfliFindLongestMatch (lz77.h:112-115) for every position of [instart, inend), limit 258,
 * cache disabled: length[j], distance[j], sublen[j*259 + k] for k in 3..length[j] (0 elsewhere),
 * plus the per-position hash state same / hashval / hashval2 (hash.h:29-47). Any output may be NULL. */
int ZopfliB200MatchTable(const unsigned char* in, size_t insize, size_t instart, size_t inend,
                         unsigned short* length, unsigned short* distance, unsigned short* sublen,
                         unsigned short* same, unsigned short* hashval, unsigned short* hashval2);

/* ZopfliCalculateBlockSize(btype 2) as a function of the 288+32 symbol histogram
 * (deflate.c:569-608), evaluated on the device (where=1) or by the host code (where=0). */
uint64_t ZopfliB200DynamicBlockBits(const uint32_t* hist320, int where);

/* ZopfliCalculateBlockSizeAutoType (deflate.h:85-86) of nreq symbol ranges of one LZ77 store,
 * evaluated on the device (k_split_eval) -- the splitter's cost oracle. */
int ZopfliB200DeviceAutoTypeBits(const unsigned short* litlens, const unsigned short* dists, size_t n,
                                 size_t nreq, const size_t* lstart, const size_t* lend, uint64_t* out);

/* Host logic seams (no GPU needed): ZopfliBlockSplitLZ77 (blocksplitter.h:42-45) and
 * ZopfliCalculateBlockSize[AutoType] (deflate.h:79-86) over an explicit symbol list whose first
 * symbol starts at byte 0 of `in`. */
size_t ZopfliB200HostBlockSplitLZ77(const unsigned char* in, const unsigned short* litlens,
                                    const unsigned short* dists, size_t n, size_t maxblocks,
                                    size_t* points, size_t cap);
/* The same search as the product runs it (batched_split.hpp: every FindMinimum of every current
 * block in lockstep rounds, `budget` probes per round bound the speculation depth), costs from the
 * host estimators, for several stores at once: store s = symbols [off[s], off[s]+size[s]).
 * points[s*cap ..] receives store s's split points, npoints[s] their number. */
void ZopfliB200HostBatchedSplit(const unsigned short* litlens, const unsigned short* dists, size_t nstores,
                                const size_t* off, const size_t* size, size_t maxblocks, size_t budget,
                                size_t* points, size_t cap, size_t* npoints);
double ZopfliB200HostBlockSize(const unsigned char* in, const unsigned short* litlens,
                               const unsigned short* dists, size_t n, size_t lstart, size_t lend,
                               int btype /* 0,1,2 or -1 for AutoType */);
/* AddLZ77Block (deflate.c:682-745) for btype 1/2 at bit offset 0: emits one block into out
 * (capacity cap bytes), returns the number of bits. */
uint64_t ZopfliB200HostEmitBlock(const unsigned char* in, const unsigned short* litlens,
                                 const unsigned short* dists, size_t n, size_t lstart, size_t lend,
                                 int btype, int final, unsigned char* out, size_t cap);
/* AddLZ77Block (deflate.c:682-745) for a list of pieces of one LZ77 store, placed one after the other as
 * the driver places blocks.  Piece i is symbols [lstart[i], lend[i]) of (litlens, dists), block type
 * btype[i] (0 stored, 1 fixed, 2 dynamic) with BFINAL final[i].  The store's first symbol covers in[0]
 * and the store covers at most insize bytes (stored pieces copy them).  The stream starts at bit bp0
 * (0..7) of out[0], the bits before it zero; *nbits receives its end bit position, out (cap bytes) the
 * bytes [0, ceil(*nbits / 8)).  Every piece gets a plan, the block plan the emission uses:
 * plan_len[i*320 ..] its 288 + 32 dynamic code lengths, plan_val[i*6 ..] its tree flags (use_16 | use_17
 * << 1 | use_18 << 2), tree-header bits, dynamic / fixed / stored block bits and input bytes.
 * Device: the plan from k_block_plan, the stream from k_emit (product library only, like the device-memory
 * calls below).  Host: their host twins (host_emit.hpp).
 * Return 1 on invalid symbols or ranges or when the stream does not fit in cap (*nbits is set then). */
int ZopfliB200DeviceEmitBlocks(const unsigned char* in, size_t insize, const unsigned short* litlens,
                               const unsigned short* dists, size_t n, size_t npieces, const size_t* lstart,
                               const size_t* lend, const int* btype, const int* final, unsigned bp0,
                               unsigned char* out, size_t cap, uint64_t* nbits, unsigned char* plan_len,
                               uint64_t* plan_val);
int ZopfliB200HostEmitBlocks(const unsigned char* in, size_t insize, const unsigned short* litlens,
                             const unsigned short* dists, size_t n, size_t npieces, const size_t* lstart,
                             const size_t* lend, const int* btype, const int* final, unsigned bp0,
                             unsigned char* out, size_t cap, uint64_t* nbits, unsigned char* plan_len,
                             uint64_t* plan_val);
/* OptimizeHuffmanForRle (deflate.c:434-518) as restated for host and device, in place, n <= 288. */
void ZopfliB200HostOptimizeRle(uint32_t* counts, int n);
/* The same on nhist histograms of n counts each, in place: by_segments=0 as above, 1 in the device's order
 * (optimize_for_rle_by_segments: segment ends as a function of the segment start, reached by hops). */
void ZopfliB200HostOptimizeRleBatch(uint32_t* counts, int n, size_t nhist, int by_segments);
/* ZopfliLengthLimitedCodeLengths (katajainen.h:35-36) as restated for host and device. */
int ZopfliB200HostLengthLimited(const uint32_t* freq, int n, int maxbits, unsigned* bitlengths);
/* Tree-header bits (EncodeTree deflate.c:205-241) of nvec code-length-code count vectors clcounts[v*19 ..]:
 * by_huffman=0 from the 7-limited package-merge, 1 from an unlimited Huffman code where it is no deeper than 7
 * (the device's way). */
void ZopfliB200HostTreeHeaderBits(const uint32_t* clcounts, size_t nvec, int by_huffman, uint32_t* out);
/* The pieces of the exact dynamic block size of nhist histograms hists[h*320 ..] (taken with the end symbol's
 * count 1, deflate.c:575): smoothed[h*320 ..] the RLE-smoothed counts (ll, then d), lengths[h*640 ..] the
 * code lengths of the plain then the smoothed counts (320 each, distance codes patched), tree_bits[h*16 + 8*set
 * + flags] the tree-header bits of each set under each flag combination, dyn_bits[h] the block size.  Device:
 * the warp functions of k_split_eval / k_iterate / k_block_plan (product library only).  Host: their twins. */
int ZopfliB200DeviceProbeParts(const uint32_t* hists, size_t nhist, uint32_t* smoothed, unsigned char* lengths,
                               uint32_t* tree_bits, uint64_t* dyn_bits);
int ZopfliB200HostProbeParts(const uint32_t* hists, size_t nhist, uint32_t* smoothed, unsigned char* lengths,
                             uint32_t* tree_bits, uint64_t* dyn_bits);

/* Sharding (SURVEY 8(e)): compress in[start, end) -- cut into master blocks of 1,000,000 bytes
 * counted from `start` (util.h:60; deflate.c:912-924), bytes before `start` being the LZ77
 * dictionary (the 32 KiB halo of a shard) -- into a position-independent SPAN: a sequence of
 *   u8 kind (0 bits, 1 stored) | u8 final | u64 nbits-or-nbytes | payload bytes
 * Compressed blocks are encoded at bit offset 0; stored blocks carry their raw bytes because
 * their padding depends on the final bit offset (deflate.c:643-649).  `final` marks the last
 * block of the range.  If dev_in is non-NULL it is a device pointer holding the same bytes as
 * `in` (16-byte aligned, readable 16 bytes past insize) and no host-to-device copy is made. */
int ZopfliB200DeflateSpan(const ZopfliOptions* options, const unsigned char* in, size_t insize,
                          const unsigned char* dev_in, size_t start, size_t end, int final,
                          unsigned char** span, size_t* spansize);
/* Splices a span onto a stream whose last byte has *bp bits in use (bit-offset scan).  The span is
 * validated first (record sizes against spansize); returns 1 and leaves the output untouched if
 * it is truncated or malformed. */
int ZopfliB200AppendSpan(const unsigned char* span, size_t spansize, unsigned char* bp,
                         unsigned char** out, size_t* outsize);
/* Bit offset, relative to the first bit the call wrote, at which each master block (deflate.c:
 * 908-931) of the most recent ZopfliDeflate / ZopfliCompress call starts, plus the end offset as last
 * entry.  Returns the number of entries (master blocks + 1).  Lets a checker compare sampled master
 * blocks of one big stream with the reference's ZopfliDeflatePart of the same range. */
size_t ZopfliB200LastMasterBitOffsets(uint64_t* offsets, size_t cap);
/* ZopfliCompress with the input already resident on the device (bench `value` leg). */
void ZopfliB200CompressDevice(const ZopfliOptions* options, ZopfliFormat output_type,
                              const unsigned char* in, size_t insize, const unsigned char* dev_in,
                              unsigned char** out, size_t* outsize);

/* ---- input and output in device memory ----
 * ZopfliCompress (zopfli.h:86-88) of the insize bytes at device address dev_in, result in device memory.
 * The bytes of *dev_out equal what ZopfliCompress(options, output_type, <same bytes>) returns.
 * dev_in: any alignment, nothing past insize is read; work is ordered after what is queued on cuda_stream
 * (a cudaStream_t of dev_in's device, NULL = legacy default stream), and cuda_stream is made to wait for the
 * result.  Runs on the device that owns dev_in (one GPU: ZOPFLI_B200_GPUS does not apply); the call blocks
 * until the result is complete.  The CRC-32 / Adler-32 of the trailer is computed on the device, so no byte of
 * the input or of the stream crosses PCIe.  *dev_out: exactly *outsize bytes from cudaMallocAsync on
 * cuda_stream; the caller owns it (cudaFreeAsync / cudaFree / ZopfliB200FreeDevice).  Unlike ZopfliCompress
 * nothing is appended: *dev_out and *outsize are outputs only.  With insize == 0, dev_in may be NULL and the
 * call runs on the current device.  Updates ZopfliB200LastMasterBitOffsets and prints the verbose reports
 * as ZopfliCompress does.  Returns 0, or nonzero with the outputs untouched when dev_in is not device memory,
 * an output pointer is NULL or the format is unknown. */
int ZopfliB200CompressDeviceToDevice(const ZopfliOptions* options, ZopfliFormat output_type,
                                     const unsigned char* dev_in, size_t insize, void* cuda_stream,
                                     unsigned char** dev_out, size_t* outsize);
void ZopfliB200FreeDevice(void* dev_ptr, void* cuda_stream); /* cudaFreeAsync on the device that owns dev_ptr */
/* zlib-compatible CRC-32 / Adler-32 of device bytes (any alignment, size 0 with NULL allowed), computed on
 * the device; blocking, ordered after cuda_stream.  Return nonzero when dev_in is not device memory. */
int ZopfliB200Crc32Device(const unsigned char* dev_in, size_t size, void* cuda_stream, uint32_t* crc);
int ZopfliB200Adler32Device(const unsigned char* dev_in, size_t size, void* cuda_stream, uint32_t* adler);

/* ---- input in pieces ----
 * A compressor takes its input in pieces (chunks) and returns the bytes ZopfliCompress returns for all of them
 * concatenated, in bounded memory, like zlib's deflate stream.  Master block i (deflate.c:908-931) depends only
 * on its bytes, the 32 KiB before it and whether it is the last one, so the compressor runs the input as waves
 * of whole master blocks (half as many as ZopfliCompress runs at once on the device, so that the two waves in
 * flight fit the device memory of one call: about 72 on an 80 GB card by the driver's schedule; ZOPFLI_B200_BATCH and ZOPFLI_B200_CHUNKS shrink them) while more bytes arrive.
 *  - Identical bytes: without a flush, a dictionary or restart points (below), every Write output followed by the Finish
 *    output, concatenated, equals ZopfliCompress(options, output_type, <all chunks concatenated>), for every
 *    chunking (zero-length writes included) and all three formats.  A compressor finished at once gives
 *    ZopfliCompress of an empty input.
 *  - Ownership: *out / *outsize follow ZopfliCompress's rule (bytes are appended under zopfli's capacity rule,
 *    the caller frees).  Only complete bytes are returned; the compressor keeps the partly filled last byte.
 *    The gzip / zlib header comes out with the first Write that returns bytes, or with Finish.
 *  - Chunks: device < 0: chunks are host memory.  device >= 0: chunks are memory of that device, and each
 *    Write is ordered after the work queued on cuda_stream (a stream of that device, NULL = legacy default
 *    stream).  A chunk may be reused or freed as soon as Write returns; for device chunks Write waits for its
 *    own device-to-device copy, not for the compression.  A full master block is compressed once a byte past
 *    it has arrived, so a Write may return no bytes.
 *  - Errors: Write and Finish return nonzero and leave every output untouched for a NULL c, out or outsize,
 *    device memory given to a host compressor, host memory or another device's memory given to a device
 *    compressor (n > 0), and any call after Finish.  New returns nonzero, *c untouched, for NULL options or
 *    c, an unknown format, or a device that does not exist.
 *  - Threads: one compressor is used by one thread at a time; different compressors may run at the same time
 *    from any threads.  One compressor runs on one GPU: ZOPFLI_B200_GPUS does not apply.
 *  - Reports: Finish updates ZopfliB200LastMasterBitOffsets to the whole stream's offsets (those ZopfliCompress
 *    leaves for the same input).  With verbose, each wave prints its reports as ZopfliCompress does, waves
 *    running one at a time, and Finish prints the size reports: a one-wave input prints what ZopfliCompress
 *    prints.
 *  - Memory: at most two waves are in flight and one fills; a Write that completes a third wave waits for the
 *    oldest.  The staging a compressor holds (host memory, or device memory for device chunks) is at most
 *    three slots of one wave plus its dictionary each: 3 x (wave bytes + 32 KiB + 16), whatever the total
 *    length.  Output not yet returned is at most one byte between calls. */
typedef struct ZopfliB200Compressor ZopfliB200Compressor;
int ZopfliB200CompressorNew(const ZopfliOptions* options, ZopfliFormat output_type, int device, void* cuda_stream,
                            ZopfliB200Compressor** c);
/* Appends to (*out, *outsize), zopfli-style, whatever output bytes are complete.  May return none. */
int ZopfliB200CompressorWrite(ZopfliB200Compressor* c, const unsigned char* chunk, size_t n, unsigned char** out,
                              size_t* outsize);
/* Compresses the rest and appends it together with the trailer. */
int ZopfliB200CompressorFinish(ZopfliB200Compressor* c, unsigned char** out, size_t* outsize);
/* Also valid before Finish: abandons the work (waits for the waves in flight, drops their output). */
void ZopfliB200CompressorFree(ZopfliB200Compressor* c);
/* Flush points and a preset dictionary, zlib's Z_SYNC_FLUSH / Z_FULL_FLUSH and deflateSetDictionary.
 * Byte contract.  Let X = dictionary || data (the dictionary empty if none was set), positions in X, d = its
 * length.  Flush calls cut the data into segments [s, e): the first starts at d, each Flush ends one and Finish
 * ends the last.  The floor of a segment is the position of the most recent full flush at or before s, else 0.
 * The deflate body is this chain of the reference's calls, each continuing at the bp and output buffer the one
 * before left:
 *  1. Data of a segment, if e > s or it is the last one: master blocks [s + i*1e6, min(s + (i+1)*1e6, e)), cut
 *     as ZopfliDeflate cuts them (an empty last segment is one empty master block), each
 *     ZopfliDeflatePart(options, 2, final, X + floor, mb_start - floor, mb_end - floor, ...) over X[floor, e);
 *     final is 1 only on the last master block of the last segment.
 *  2. End of a flushed segment: ZopfliDeflatePart(options, 0, 0, X, e, e, ...), the sync marker (a stored block
 *     of BFINAL 0 and LEN 0, deflate.c:625-663).  Every Flush call emits exactly one marker; a flushed segment
 *     with no bytes contributes only the marker.
 * So only the last 32 KiB of the dictionary can influence the output, and after a full flush neither the
 * dictionary nor earlier data can.  With no dictionary and no flush this is ZopfliDeflate of the data: the
 * identical-bytes rule above.  Containers: gzip as always, and a dictionary is refused (the format has no field
 * for one; zlib refuses it the same way).  zlib without a dictionary as always (78 DA); with one, 78 F9 (FDICT)
 * and DICTID, the big-endian Adler-32 of the whole dictionary, as deflateSetDictionary writes it (1 for 0 bytes).
 * In every format the trailer's checksum and ISIZE cover the data only.
 * Flush compresses everything written so far as one wave, however short (later waves count master blocks from
 * the flush point), waits for every wave in flight and appends all remaining output: the header if it has not
 * gone out, the segment's blocks and the marker.  The stream is then byte-aligned: nothing stays behind.  It
 * returns nonzero, every output untouched, for a NULL c, out or outsize, a mode other than 2 or 3, and after
 * Finish.  The staging bound stays 3 x (wave bytes + 32 KiB + 16).
 * SetDictionary is accepted once, before the first Write or Flush call of any length.  dict is memory of the
 * kind the compressor takes for chunks: host memory for a host compressor, or that device's memory for a device
 * compressor, ordered after cuda_stream; the DICTID of a device dictionary is computed on the device
 * (k_adler32), so the dictionary does not cross PCIe.  Its last 32 KiB are staged in front of the first wave.
 * It returns nonzero, nothing changed, for gzip, a NULL c, a NULL dict with n > 0, the wrong kind of memory, a
 * second call, and a call after the first Write or Flush.
 * Reports: after Finish, ZopfliB200LastMasterBitOffsets gives the bit offset of every master block of every
 * segment in stream order (the bit positions before each data call above), then the end offset.  With
 * verbose, each flush wave prints its reports as a wave does. */
#define ZOPFLI_B200_SYNC_FLUSH 2 /* zlib's Z_SYNC_FLUSH */
#define ZOPFLI_B200_FULL_FLUSH 3 /* zlib's Z_FULL_FLUSH */
int ZopfliB200CompressorFlush(ZopfliB200Compressor* c, int mode, unsigned char** out, size_t* outsize);
int ZopfliB200CompressorSetDictionary(ZopfliB200Compressor* c, const unsigned char* dict, size_t n);
/* The compressor's wave policy as a pure function (csrc/dist_layout.hpp next_wave; no GPU needed): with
 * `received` bytes written, `handed` bytes already in waves and waves of wave_blocks master blocks, returns 1 and
 * the next wave [*a, *b) with its BFINAL flag, or 0 when no wave is ready.  finished: 0 while writing (a wave is
 * whole master blocks from `handed` with a byte past it), 1 at Finish (all that is left, final), 2 at a flush
 * (all that is left, not final; 0 when handed == received). */
int ZopfliB200CompressorWave(size_t received, int finished, size_t handed, size_t wave_blocks, size_t* a, size_t* b,
                             int* final);
/* Restart points: a full flush every `interval` bytes of data, made inside the waves.
 * Byte contract.  An interval N >= 1 means a full flush at every data position k*N (k >= 1) that has at least one
 * data byte after it: X position d + k*N with a dictionary of d bytes.  The automatic flush at k*N happens once
 * byte k*N + 1 has arrived, and never at the end of the data, where Finish comes instead.  The stream is exactly
 * the one the contract above defines for the caller's flushes plus (k*N, FULL) for every such k, merged by
 * position; at equal positions the caller's flush comes first (it was called before the byte past it arrived),
 * so a Flush(FULL) at k*N yields two markers.  Without an interval nothing changes.
 * Segments cut at restart points share waves: a wave is still wave_blocks units, a unit being a master block of
 * a segment (counted from the segment's start), and every unit's parse sees no byte before the last full flush
 * at or before it.  So an interval below 1e6 makes waves shorter in bytes, not fewer in units; the staging bound
 * and the two waves in flight stay as they are.
 * SetRestartInterval is accepted once, before the first Write or Flush call of any length, and combines with
 * SetDictionary and with explicit flushes.  It returns nonzero, nothing changed, for a NULL c, interval 0, a
 * second call, a call after the first Write or Flush, and a call after Finish.
 * RestartPoints lists one entry per full flush, automatic or explicit, in stream order: data_off is the data
 * position of the flush, stream_off the offset of the first byte after its marker, counted from the first byte
 * the compressor returned (header included).  Raw inflate of the stream from stream_off on (zlib wbits -15)
 * yields data[data_off:], in all three formats.  An entry is listed once its marker's bytes have been returned;
 * after Finish the list is complete.  The start of the stream is not an entry: a reader whose target lies before
 * the first entry decodes from the start, with the dictionary if there is one.  Returns the number of entries and
 * writes min(count, cap) of them; either array may be NULL.  Returns 0 for a NULL c.
 * After Finish, ZopfliB200LastMasterBitOffsets gives every master block of every segment, then the end; markers
 * are not entries. */
int ZopfliB200CompressorSetRestartInterval(ZopfliB200Compressor* c, size_t interval);
size_t ZopfliB200CompressorRestartPoints(ZopfliB200Compressor* c, uint64_t* data_off, uint64_t* stream_off, size_t cap);
/* The compressor's schedule with restart points as a pure function (csrc/dist_layout.hpp next_wave; no GPU
 * needed): as ZopfliB200CompressorWave, with `floor` the last full flush at or before `handed` and restart points at
 * dict_len + k*interval (interval 0: none).  Returns the number of units of the next wave (0: no wave is ready)
 * and writes min(count, cap) of them: unit i is bytes [a[i], b[i]) parsed seeing no byte before floors[i], and
 * restart[i] is 1 where the automatic full flush's marker follows it.  *final is the wave's BFINAL.  Any of the
 * arrays and final may be NULL. */
size_t ZopfliB200CompressorWaveUnits(size_t received, int finished, size_t handed, size_t floor, size_t dict_len,
                                     size_t interval, size_t wave_blocks, size_t* a, size_t* b, size_t* floors,
                                     int* restart, size_t cap, int* final);
/* Output in device memory: a device compressor (device >= 0) keeps its stream on the device.  Each wave's runs of
 * compressed blocks are emitted on the device into an allocation of the wave's own, and k_splice places them and
 * the wave's stored blocks (read from its staging slot) at the stream's bit position in a pending buffer on the
 * device; the header, the markers and the trailer are written by the same kernel.  So no compressed byte is
 * downloaded except those a caller asks for on the host.
 * WriteToDevice, FlushToDevice and FinishToDevice are Write, Flush and Finish with the output in device memory:
 * the same bytes are complete after each call, so the byte counts per call match, and the calls of both kinds
 * may be mixed on one compressor (the stream is the concatenation in call order).  *dev_out is exactly *outsize
 * bytes from cudaMallocAsync on cuda_stream, as ZopfliB200CompressDeviceToDevice's result: outputs only, nothing
 * appended, the caller frees it (ZopfliB200FreeDevice / cudaFreeAsync); NULL and 0 when the call completes no
 * byte.  The call returns once the bytes are in place, and cuda_stream waits for them.  They return nonzero,
 * every output untouched, for everything Write, Flush and Finish refuse and for a host compressor (device < 0).
 * Write, Flush and Finish on a device compressor download exactly the bytes they return, once.
 * Device memory of a device compressor: the staging above; plus, for each wave in flight, its runs of compressed
 * blocks, at most the wave's bytes plus 5 bytes per started 65,535 bytes of each block (no compressed block is
 * larger than its stored form) plus 8 bytes per run; plus the pending stream of one call, a buffer that grows
 * by doubling and is kept: at most twice the most bytes one call has returned, plus 4. */
int ZopfliB200CompressorWriteToDevice(ZopfliB200Compressor* c, const unsigned char* chunk, size_t n,
                                      unsigned char** dev_out, size_t* outsize);
int ZopfliB200CompressorFlushToDevice(ZopfliB200Compressor* c, int mode, unsigned char** dev_out, size_t* outsize);
int ZopfliB200CompressorFinishToDevice(ZopfliB200Compressor* c, unsigned char** dev_out, size_t* outsize);
/* seam: ZopfliB200AppendSpan with the splice done by k_splice on the current device (product library only): the
 * span is validated as AppendSpan validates it, uploaded with the partly filled last byte, spliced on the device
 * and the new bytes downloaded.  Returns 1, output untouched, for what AppendSpan refuses and for *bp > 7. */
int ZopfliB200DeviceAppendSpan(const unsigned char* span, size_t spansize, unsigned char* bp,
                               unsigned char** out, size_t* outsize);

/* ---- several GPUs, one stream (SURVEY 8(e)) ----
 * The master blocks of one input (the reference's independent unit, deflate.c:908-931) are sharded
 * over the GPUs of one box; NCCL scatters the byte ranges (+ 32 KiB dictionary) from rank 0's GPU and
 * gathers the compressed bits straight into their final bit positions on rank 0.
 *  - one process, N GPUs: set ZOPFLI_B200_GPUS=N; ZopfliCompress / ZopfliDeflate(btype 2) use it
 *    transparently (ncclCommInitAll, one host thread per GPU);
 *  - one process per GPU (e.g. torchrun): rank 0 calls ZopfliB200DistUniqueId, the id is given to every
 *    rank out of band, every rank calls ZopfliB200DistInit once (device = ZOPFLI_B200_DEVICE / LOCAL_RANK)
 *    and then ZopfliB200DistCompress COLLECTIVELY with the same options, format and insize.  `in` is read
 *    and *out / *outsize are written on rank 0 only (same ownership rule as ZopfliCompress).
 * All return 0 on success. */
#define ZOPFLI_B200_UNIQUE_ID_BYTES 128
int ZopfliB200DistUniqueId(unsigned char* id128);
int ZopfliB200DistInit(int rank, int world, const unsigned char* id128);
#define ZOPFLI_B200_DIST_STAGED 1 /* flags: the shards of this very input are still on the GPUs from the
                                    previous ZopfliB200DistCompress call -- skip the H2D copy and the scatter
                                    (the bench's "input resident in HBM" leg); `in` is still read for the checksum */
int ZopfliB200DistCompress(const ZopfliOptions* options, ZopfliFormat output_type, const unsigned char* in,
                           size_t insize, int flags, unsigned char** out, size_t* outsize);
void ZopfliB200DistFinalize(void);
/* The placement arithmetic of the multi-GPU path as pure functions (csrc/dist_layout.hpp; no GPU needed):
 * the byte range [a, b) rank `rank` owns and the start `base` of its device copy (shard + dictionary);
 * and, from len8[world][8] (bits of every rank's blocks for each start phase), the absolute bit offsets
 * start[0..world] of the ranks in the one stream. */
void ZopfliB200DistShard(size_t insize, int world, int rank, size_t* a, size_t* b, size_t* base);
void ZopfliB200DistPlacement(const uint64_t* len8, int world, unsigned phase0, uint64_t* start);

/* CRC-32 of the gzip trailer (gzip_container.c:27-81) and its combination across shards. */
uint32_t ZopfliB200Crc32(const unsigned char* data, size_t size);
uint32_t ZopfliB200Crc32Combine(uint32_t crc1, uint32_t crc2, uint64_t len2);
/* Adler-32 of the zlib trailer (zlib_container.c:29-48), computed as ZopfliB200Crc32 is (from 4 MiB on, one
 * slice per host thread, the slices combined exactly), and the combination of consecutive slices (adler32
 * of A|B from those of A and B and |B|). */
uint32_t ZopfliB200Adler32(const unsigned char* data, size_t size);
uint32_t ZopfliB200Adler32Combine(uint32_t adler1, uint32_t adler2, uint64_t len2);
/* The host checksum behind ZopfliB200Crc32, ZopfliB200Adler32 and the gzip / zlib trailers, run at a chosen
 * slice size: the input cut into slices of slice_bytes (0 counts as 1), reduced side by side and combined
 * with the slice algebra of the device checksums (csrc/checksum.hpp).  kind 0: CRC-32, 1: Adler-32. */
uint32_t ZopfliB200HostChecksumSliced(const unsigned char* data, size_t size, size_t slice_bytes, int kind);

/* Engine control / introspection. */
typedef struct ZopfliB200Stats {
  double ms_same, ms_keys, ms_scan, ms_scatter, ms_match, ms_greedy, ms_iterate, ms_pack, ms_h2d, ms_d2h;
  double ms_host_split, ms_host_emit, ms_host_other, ms_total;
  uint64_t launches, match_positions, iterate_positions, iterate_steps, h2d_bytes, d2h_bytes;
  uint64_t cyc_sum[6], cyc_max[6], max_block_positions; /* k_iterate phase cycles, see engine.hpp */
  double ms_split; uint64_t split_evals, split_rounds;  /* device split-cost service */
  uint64_t iterate_launches;                             /* k_iterate launches (ms_iterate is the sum of their durations) */
  uint64_t int_steps;                                    /* forward-DP steps that ran in the integer window (see iterate.cuh) */
  uint64_t dp_cyc_sum[5], dp_cnt_sum[6];                 /* DP cycles / groups of 32 steps by kind: integer window, fp64 magic, fp64 plain, */
  uint64_t dp_cyc_max[5], dp_cnt_max[6];                 /* fp64 ring-joining, general; cnt[5] = positions in the per-step loop; sum over blocks / critical block */
  uint64_t ovf_regrows;                                  /* batches redone because their run lists outgrew the overflow arena */
  uint64_t log_regrows;                                  /* batches redone because a statistics sum outgrew the log table */
} ZopfliB200Stats;
void ZopfliB200GetStats(ZopfliB200Stats* out);
void ZopfliB200ResetStats(void);
void ZopfliB200SetStream(void* cuda_stream);
int ZopfliB200Device(void);
const char* ZopfliB200Version(void);

#ifdef __cplusplus
}
#endif
#endif

// Host-visible interface of the CUDA engine (no CUDA types leak out of engine.cu).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

namespace zb {

struct ParseRange {
  uint64_t instart, inend;
  int mode;           // 0 greedy parse only (ZopfliLZ77Greedy), 1 optimal parse (ZopfliLZ77Optimal),
                      // 2 optimal parse with fixed-tree costs (ZopfliLZ77OptimalFixed)
  int numiterations;  // mode 1 only
};

struct ParseResult {        // symbols of range i: [off[i], off[i]+size[i]) in ll / d
  std::vector<uint32_t> off, size;
  std::vector<uint16_t> ll, d;
  std::vector<uint64_t> cost;  // mode 1: exact dynamic-block bit cost of the returned parse
};

struct EngineStats {  // accumulated since the last reset; times from CUDA events on the engine stream
  double ms_same, ms_keys, ms_scan, ms_scatter, ms_match, ms_greedy, ms_iterate, ms_pack, ms_h2d, ms_d2h, ms_split;
  uint64_t split_evals, split_rounds, iterate_launches;
  uint64_t launches;
  uint64_t match_positions, iterate_positions, iterate_steps;  // steps = positions x iterations
  uint64_t h2d_bytes, d2h_bytes;
  uint64_t cyc_sum[6];   // k_iterate phase cycles summed over blocks (model, DP, trace, follow, cost, stats)
  uint64_t cyc_max[6];   // same for the block with the largest total (the critical path)
  uint64_t max_block_positions;
  uint64_t int_steps;    // DP steps that ran in the integer window
  uint64_t dp_cyc_sum[5], dp_cnt_sum[6];   // DP cycles / groups by kind of group (JobState::dpc, dpn), summed over blocks
  uint64_t dp_cyc_max[5], dp_cnt_max[6];   // same for the critical-path block
  uint64_t ovf_regrows;  // batches redone because their run lists outgrew the overflow arena
  uint64_t log_regrows;  // batches redone because a statistics sum outgrew the log table
};

class Engine {
 public:
  // Engine contexts are leased for the duration of one API call (Engine::Lease): a context owns its
  // input buffers, lanes and arenas, so concurrent calls never share mutable device state.
  // dev < 0: the process's default device (ZOPFLI_B200_DEVICE, else LOCAL_RANK, else 0)
  static Engine* acquire(int dev = -1);
  static void release(Engine* e);
  static int default_device();
  static int device_count();
  struct Lease {
    Engine* e;
    explicit Lease(int dev = -1) : e(Engine::acquire(dev)) {}
    ~Lease() { Engine::release(e); }
    Lease(const Lease&) = delete;
    Lease& operator=(const Lease&) = delete;
    Engine& operator*() { return *e; }
    Engine* operator->() { return e; }
  };
  static EngineStats stats_all();   // summed over every context of the process
  static void reset_stats_all();

  // Input residency. set_input_host copies to the device (inside the caller's timed region);
  // set_input_device adopts an existing device buffer that must stay valid and be readable
  // 16 bytes past insize (e.g. a padded torch tensor).
  void set_input_host(const uint8_t* in, size_t insize);
  void set_input_device(const uint8_t* dev_in, size_t insize);
  // Device bytes of any alignment (nothing past insize is read), copied device to device after the work
  // queued on user_stream (cudaStream_t of this context's device, NULL = legacy default stream).
  // checksum (checksum.hpp ChecksumKind: 0 CRC-32, 1 Adler-32, 2 none) starts on a stream of its own
  // beside the parse; its result stays on the device for emit_to_device.
  void set_input_device_copy(const uint8_t* dev_src, size_t insize, void* user_stream, int checksum);
  // CRC-32 / Adler-32 (ChecksumKind) of dev_in[0, n) computed on the device, after the work queued on
  // user_stream; blocks until the result is known.
  uint32_t checksum_device(const uint8_t* dev_in, size_t n, void* user_stream, int checksum);
  // device that owns p (device or managed memory), else -1
  static int pointer_device(const void* p);
  static int current_device();
  // cudaFreeAsync of an allocation made by emit_to_device
  static void free_device(void* p, void* user_stream);

  // `lane` selects one of kLanes independent stream + arena sets; calls on different lanes may run
  // concurrently from different host threads (chunk pipelines; giant blocks beside the rest).
  static constexpr int kLanes = 8;
  void parse(const std::vector<ParseRange>& ranges, ParseResult& out, int lane = 0);

  // test seam: raw match table of one range (length, dist, expanded sublen[259] per position)
  void match_table(uint64_t instart, uint64_t inend, std::vector<uint16_t>& len,
                   std::vector<uint16_t>& dist, std::vector<uint16_t>& sublen,
                   std::vector<uint16_t>& same, std::vector<uint16_t>& hv, std::vector<uint16_t>& hv2);
  // test seam: device-side exact dynamic block size of a 320-bin histogram
  uint64_t device_block_bits(const uint32_t* hist320);
  // test seam: the pieces of that size for n histograms (ZopfliB200DeviceProbeParts)
  void device_probe_parts(const uint32_t* hists, size_t n, uint32_t* smoothed, uint8_t* lengths, uint32_t* tree_bits,
                          uint64_t* dyn);

  // Split-cost service (ZopfliCalculateBlockSizeAutoType over symbol ranges, deflate.c:610-621):
  // split_begin uploads n stores given as flat symbol arrays with per-store offset/size,
  // split_eval prices a batch of (store, lstart, lend) ranges on the device.
  void split_begin(const uint16_t* ll, const uint16_t* d, const std::vector<uint64_t>& off,
                   const std::vector<uint32_t>& size, int lane = 1);
  // Stage A + B without a symbol round trip: greedy parse of `ranges` whose stores stay on the device
  // and become the stores of the split service of the same lane.  sizes[i] = symbols of range i.
  void greedy_to_split(const std::vector<ParseRange>& ranges, std::vector<uint32_t>& sizes, int lane = 1);
  // byte offset (from the start of its range) of symbol idx of store `store`, for many (store, idx)
  struct SplitPos { uint32_t store, idx; };
  void split_positions(const std::vector<SplitPos>& q, std::vector<uint32_t>& bytepos, int lane = 1);
  struct SplitReq { uint32_t store, lstart, lend; };
  void split_eval(const SplitReq* reqs, size_t n, uint64_t* costs, int lane = 1);

  // ---- device-resident finish (SURVEY 8(f)#2, finish.cuh): stores, plans and the output stay on the GPU ----
  // Three symbol buffers, all indexed like the input (a block never has more symbols than bytes):
  //   kPack  best parse of every first-split block at [block start ...)
  //   kFin   the master block's concatenated store at [master start ...)
  //   kFix   fixed-tree re-parse of a final block at [block start ...)
  enum StoreBuf { kPack = 0, kFin = 1, kFix = 2 };
  // parse() whose results stay on the device in buffer `dest`; sizes / costs as in ParseResult
  // iter_costs (optional, for the verbose report of squeeze.c:493-495): cost of iteration i of range r at
  // [r * numiterations_max + i], ~0 where an iteration did not run
  void parse_keep(const std::vector<ParseRange>& ranges, int dest, std::vector<uint32_t>& sizes,
                  std::vector<uint64_t>& costs, int lane = 0, std::vector<uint64_t>* iter_costs = nullptr);
  // kPack -> kFin copies (ZopfliAppendLZ77Store), then the split service of `lane` over the kFin stores
  // [store_off[i], store_off[i] + store_size[i]) (skipped when store_off is empty)
  struct SymCopy { uint64_t src_off, dst_off; uint32_t n, pad; };
  void concat_stores(const std::vector<SymCopy>& copies, const std::vector<uint64_t>& store_off,
                     const std::vector<uint32_t>& store_size, int lane = 1);
  // stored / fixed / dynamic sizes of symbol ranges + the emission plan of each (kept on the device);
  // handles[i] identifies range i's plan in emit()
  struct PlanReq { uint64_t off; uint32_t n; uint32_t buf; };
  struct PlanCost { uint64_t unc, fixed, dyn, tree; };  // tree: bits of the dynamic block's tree header (part of dyn)
  void plan_blocks(const std::vector<PlanReq>& reqs, std::vector<PlanCost>& costs, std::vector<uint64_t>& handles,
                   int lane = 1);
  // Writes every piece at its final bit position and copies bytes [0, ceil(total_bits / 8)) of the
  // stream to host_dst.  Positions are absolute within the stream of this call (the first piece starts
  // at the caller's bit phase 0..7); stored pieces name bytes of the engine's input.
  struct EmitPiece {
    uint64_t bit_start, nbits;   // nbits: predicted size of a compressed piece (checked by the kernel)
    uint64_t off;                // symbols [off, off + n) of buffer `buf`
    uint64_t plan;               // handle from plan_blocks (dynamic pieces)
    uint64_t in_start, in_len;   // stored pieces: engine-relative input bytes
    uint32_t n;
    uint8_t buf, type, final, pad;   // type: 0 stored, 1 fixed, 2 dynamic
  };
  void emit(const std::vector<EmitPiece>& pieces, uint64_t total_bits, uint8_t* host_dst);
  // The two halves of emit(), for callers that move the stream between GPUs first (dist.cpp): the
  // emission leaves the stream in this context's output buffer (capacity >= reserve_bytes, zeroed up to
  // the emitted size) and returns its device address; download() copies device bytes to the host.
  void* emit_device(const std::vector<EmitPiece>& pieces, uint64_t total_bits, size_t reserve_bytes);
  void download(const void* dev_src, uint8_t* host_dst, size_t nbytes);
  // emit() into device memory: a fresh cudaMallocAsync allocation on user_stream of *outsize bytes holding
  // hdr[0, hdr_len), the stream (bit phase 0) and the trailer of `checksum` (the one started by
  // set_input_device_copy) with ISIZE = the input size.  user_stream waits for the result; the caller owns it.
  uint8_t* emit_to_device(const std::vector<EmitPiece>& pieces, uint64_t total_bits, const uint8_t* hdr, int hdr_len,
                          int checksum, void* user_stream, size_t* outsize);
  // host -> device through the context's threaded pinned staging (synchronous)
  void upload(void* dev_dst, const uint8_t* host_src, size_t nbytes);
  // test seam: symbols [0, n) of buffer `buf` (StoreBuf) from host arrays; n <= input size
  void load_symbols(int buf, const uint16_t* ll, const uint16_t* d, size_t n);
  void* stream();   // cudaStream_t of lane 0, the stream emit / download / set_input run on
  uint64_t input_size() const;
  uint64_t device_memory_total() const;   // bytes of device memory (sizes the master-block batches of a pipeline)

  void set_stream(void* cuda_stream);  // optional: run on the caller's stream
  EngineStats stats();
  void reset_stats();
  int device() const;

 private:
  void parse_common(const std::vector<ParseRange>& ranges, ParseResult& out, int dest, int lane,
                    std::vector<uint64_t>* iter_costs = nullptr);
  explicit Engine(int dev);
  struct Impl;
  Impl* p_;
};

// Stream-ordered device memory of a caller that holds no engine context between its calls (the device
// staging of ZopfliB200Compressor): allocations on a non-blocking stream of one device, and device-to-device
// copies on it.  Every call leaves the calling thread's current device as it found it.
class DeviceStaging {
 public:
  explicit DeviceStaging(int dev);
  ~DeviceStaging();               // waits for the stream's work
  void* alloc(size_t bytes);      // cudaMallocAsync on the stream
  void release(void* p);          // cudaFreeAsync on the stream
  // dst[0, n) <- src[0, n), ordered after the work queued on user_stream (a stream of this device, NULL = the
  // legacy default stream; ignored when user_stream is this staging's own stream); blocks until the copy is done
  void copy(void* dst, const void* src, size_t n, void* user_stream);
  void zero(void* dst, size_t n);  // blocks until done
  void* stream() const { return stream_; }
  int device() const { return dev_; }

 private:
  int dev_;
  void* stream_;
  void* ev_;
};

}  // namespace zb

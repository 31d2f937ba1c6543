// Micro-benchmark (developer tool): where the cycles of one exact dynamic block size (warp_dynamic_bits,
// the work of one split-cost probe in k_split_eval and of the per-iteration cost in k_iterate) go, on one
// warp with the SM to itself, for a text-like histogram; then the probe throughput per SM as the number of
// warps per SM grows.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false block_size.cu -o block_size && ./block_size
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../zopfli_b200/csrc/split.cuh"
using namespace zb;

__global__ void k_phases(const uint32_t* hin, unsigned long long* out, uint64_t* res) {
  __shared__ SplitSmem s;
  __shared__ uint32_t serial[320];  // optimize_for_rle's result, for the comparison
  __shared__ uint8_t good[320];
  const uint32_t lane = threadIdx.x;
  for (int i = lane; i < 320; i += 32) s.hist[i] = hin[i];
  __syncwarp();
  CostStage& cs = s.cs;
  unsigned long long t[7];
  t[0] = clock64();
  for (int i = lane; i < 320; i += 32) serial[i] = s.hist[i];
  __syncwarp();
  if (lane < 2) optimize_for_rle(lane ? kNumD : kNumLL, serial + (lane ? 288 : 0), good + (lane ? 288 : 0));
  __syncwarp();
  t[1] = clock64();
  for (int i = lane; i < 320; i += 32) cs.cnt2[i] = s.hist[i];
  __syncwarp();
  warp_optimize_for_rle(cs.cnt2, kNumLL, cs.pm, lane);
  warp_optimize_for_rle(cs.cnt2 + 288, kNumD, cs.pm, lane);
  t[2] = clock64();
  bool rle_differ = false;
  for (int i = lane; i < 320; i += 32) rle_differ |= serial[i] != cs.cnt2[i];
  const uint32_t rle_bad = __ballot_sync(0xffffffffu, rle_differ);
  const unsigned long long t2b = clock64();   // the comparison stays out of the timed phases
  warp_length_limited(s.hist, kNumLL, cs.len[0], cs.pm, lane);
  warp_length_limited(s.hist + 288, kNumD, cs.len[0] + 288, cs.pm, lane);
  warp_length_limited(cs.cnt2, kNumLL, cs.len[1], cs.pm, lane);
  warp_length_limited(cs.cnt2 + 288, kNumD, cs.len[1] + 288, cs.pm, lane);
  if (lane < 2) patch_distance_codes(cs.len[lane] + 288);
  __syncwarp();
  t[3] = clock64();
  uint32_t walk = 0xffffffffu;  // one length at a time, one lane per (set, flags), package-merge per lane
  if (lane < 16) {
    const uint8_t* l = cs.len[lane >> 3];
    walk = encode_tree_size(l, l + 288, (lane & 1) != 0, (lane & 2) != 0, (lane & 4) != 0);
  }
  __syncwarp();
  t[4] = clock64();
  const uint32_t runs = warp_tree_sizes(cs, lane);
  __syncwarp();
  t[5] = clock64();
  const uint64_t r = warp_dynamic_bits(s.hist, s.cs, lane);
  t[6] = clock64();
  const uint32_t differ = __ballot_sync(0xffffffffu, lane < 16 && walk != runs);
  if (lane == 0) {
    for (int i = 0; i < 6; i++) out[i] = t[i + 1] - (i == 2 ? t2b : t[i]);
    out[6] = differ;
    out[7] = rle_bad;
    res[0] = r;
  }
}

__global__ void k_many(const uint32_t* hin, int reps, uint64_t* res) {
  extern __shared__ SplitSmem sm[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  SplitSmem& s = sm[warp];
  uint64_t acc = 0;
  for (int r = 0; r < reps; r++) {
    for (int i = lane; i < 320; i += 32) s.hist[i] = hin[i] + (r & 1);
    __syncwarp();
    acc += warp_dynamic_bits(s.hist, s.cs, lane);
    __syncwarp();
  }
  if (lane == 0) res[blockIdx.x * 32 + warp] = acc;
}

int main() {
  std::vector<uint32_t> h(320, 0);
  srand(1);
  for (int i = 0; i < 256; i++) h[i] = (i >= 32 && i < 127) ? 200 + rand() % 20000 : (rand() % 4 == 0 ? rand() % 50 : 0);
  for (int i = 257; i < 286; i++) h[i] = 100 + rand() % 8000;
  for (int i = 0; i < 30; i++) h[288 + i] = 50 + rand() % 9000;
  h[256] = 1;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  uint32_t* dh;
  unsigned long long* dout;
  uint64_t* dres;
  cudaMalloc(&dh, 320 * 4);
  cudaMalloc(&dout, 128);
  cudaMalloc(&dres, 1 << 20);
  cudaMemcpy(dh, h.data(), 320 * 4, cudaMemcpyHostToDevice);
  for (int k = 0; k < 3; k++) {
    k_phases<<<1, 32>>>(dh, dout, dres);
    unsigned long long o[8];
    cudaMemcpy(o, dout, sizeof(o), cudaMemcpyDeviceToHost);
    printf("cycles: RLE smoothing serial %llu, by the warp %llu (%s); 4 package merges %llu; tree sizes walked %llu, "
           "by runs %llu (%s); warp_dynamic_bits %llu\n", o[0], o[1], o[7] ? "DIFFER" : "equal", o[2], o[3], o[4],
           o[6] ? "DIFFER" : "equal", o[5]);
  }
  cudaFuncSetAttribute(k_many, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  for (int wps : {1, 4, 8, 16}) {  // warps per SM, in CTAs of up to four warps as k_split_eval launches them
    const int w = wps < 4 ? wps : 4, cps = wps / w, reps = 8, grid = sms * cps;
    const size_t smem = (size_t)w * sizeof(SplitSmem);
    k_many<<<grid, 32 * w, smem>>>(dh, 1, dres);
    cudaEventRecord(a);
    k_many<<<grid, 32 * w, smem>>>(dh, reps, dres);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    printf("%2d warps per SM: %.1f us per block size per warp, %.2f us per block size per SM (%s)\n", w * cps,
           ms * 1e3 / reps, ms * 1e3 * sms / ((double)grid * w * reps), cudaGetErrorString(cudaGetLastError()));
  }
  return 0;
}

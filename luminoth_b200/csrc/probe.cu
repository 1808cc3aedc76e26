// Measurement hook (not on the product path): whether the lanes of one warp see different answers from a single
// mbarrier.try_wait instruction.
#include "../../include/luminoth_b200.h"
#include "common.cuh"

#include <algorithm>
#include <string>
#include <vector>

namespace lumi {

// ---------------------------------------------------------------------------------------------------------------
// Probe: can the 32 lanes of ONE warp instruction `mbarrier.try_wait` see different answers?  Warp 0 spins on a
// barrier with all lanes (a whole-warp barrier-polling role), counting its attempts per lane; warp 1 arrives
// after a pseudo-random pause.  Lanes that run in lockstep make the same number of attempts unless the instruction
// answered them differently.  Reports the number of rounds in which the per-lane attempt counts differed.
__global__ void __launch_bounds__(64, 1) trywait_probe_kernel(int rounds, unsigned* out) {
  __shared__ __align__(8) uint64_t bar, ack;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) { mbar_init(&bar, 1); mbar_init(&ack, 1); fence_mbar_init(); }
  __syncthreads();
  unsigned diverged = 0, max_spread = 0;
  unsigned long long total_attempts = 0;
  for (int r = 0; r < rounds; ++r) {
    const uint32_t ph = (uint32_t)r & 1u;
    if (warp == 0) {
      unsigned attempts = 1;
      while (!mbar_try_wait(&bar, ph)) ++attempts;
      __syncwarp();
      unsigned lo = attempts, hi = attempts;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
      }
      if (hi != lo) { ++diverged; max_spread = max(max_spread, hi - lo); }
      total_attempts += hi;
      if (lane == 0) mbar_arrive(&ack);
      __syncwarp();
    } else {
      if (lane == 0) {
        const long long t = clock64();
        const long long pause = 200 + ((r * 2654435761u) >> 22) % 3000;      // 200 .. 3200 clk
        while (clock64() - t < pause) {}
        mbar_arrive(&bar);
        mbar_wait(&ack, ph);
      }
      __syncwarp();
    }
  }
  if (threadIdx.x == 0) {
    out[blockIdx.x * 4 + 0] = diverged;
    out[blockIdx.x * 4 + 1] = max_spread;
    out[blockIdx.x * 4 + 2] = (unsigned)(total_attempts / (unsigned long long)rounds);
  }
}

}  // namespace lumi

extern "C" int lumi_op_trywait_probe(int rounds, unsigned* diverged_rounds, unsigned* max_spread, unsigned* mean_attempts) {
  using namespace lumi;
  try {
    LUMI_REQUIRE(rounds > 0, "trywait_probe: bad arguments");
    int dev = 0, sms = 0;
    LUMI_CUDA_CHECK(cudaGetDevice(&dev));
    LUMI_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    unsigned* d = nullptr;
    LUMI_CUDA_CHECK(cudaMalloc(&d, (size_t)sms * 4 * sizeof(unsigned)));
    LUMI_CUDA_CHECK(cudaMemset(d, 0, (size_t)sms * 4 * sizeof(unsigned)));
    trywait_probe_kernel<<<sms, 64>>>(rounds, d);
    cudaError_t e = cudaDeviceSynchronize();
    std::vector<unsigned> h((size_t)sms * 4);
    if (e == cudaSuccess) e = cudaMemcpy(h.data(), d, h.size() * sizeof(unsigned), cudaMemcpyDeviceToHost);
    cudaFree(d);
    LUMI_CUDA_CHECK(e);
    unsigned dv = 0, sp = 0;
    unsigned long long at = 0;
    for (int i = 0; i < sms; ++i) { dv += h[i * 4]; sp = std::max(sp, h[i * 4 + 1]); at += h[i * 4 + 2]; }
    if (diverged_rounds) *diverged_rounds = dv;          // summed over the CTAs (one per SM)
    if (max_spread) *max_spread = sp;
    if (mean_attempts) *mean_attempts = (unsigned)(at / (unsigned long long)sms);
    return LUMI_OK;
  } catch (const std::exception& ex) {
    return LUMI_EINVAL;
  }
}

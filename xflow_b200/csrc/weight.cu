// Importance weighting of a training step (include/xflow_b200.h, xf_trainer_set_negative_sampling and the _weighted
// steps): one pass over the batch's rows before the step kernel, run only when the step has caller weights or a
// negative-sampling policy.  A warp per row computes the row's effective weight
//   e_r = c_r x s_r   (__fmul_rn; c_r = the caller's weight or 1; s_r = 1 for a positive row or without a policy,
//                      inv = (float)(1 / rate) for a kept negative, 0 for a dropped one)
// where a negative is kept iff top24(splitmix64(seed ^ F_r)) < p24, F_r = sum over the row's tokens of
// splitmix64(key) mod 2^64.  The sum ignores token order, so the lanes reduce it in any order, and the decision
// depends on the row alone: not on the block cut, the slice or the entry point.  The pass also adds, with one atomic
// per warp:
//   *W       += ceil(e_r) x len_r over the rows it trains (e_r > 0), the bound of every key's |residual sum| in the
//               lazy step's fixed-point field (ceil(e_r) is capped at 2^31 so that the sum of at most 2^32 tokens
//               cannot wrap; such weights are far beyond the field anyway);
//   *skipped += the number of rows with e_r = 0.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "table.cuh"

__global__ void __launch_bounds__(256)
xf_k_row_weights(const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
                 const uint8_t* __restrict__ labels, const float* __restrict__ caller_w, int B, int sample,
                 uint32_t p24, float inv, uint64_t seed, float* __restrict__ e_out, unsigned long long* W,
                 unsigned long long* skipped) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * warps_per_block;
  unsigned long long w_acc = 0ull, skip_acc = 0ull;  // lane 0's
  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    float s = 1.f;
    if (sample && __ldg(labels + row) == 0) {
      uint64_t f = 0ull;
      for (uint32_t j = beg + (uint32_t)lane; j < end; j += 32u) f += xf_splitmix64(__ldcs(keys + j));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) f += __shfl_xor_sync(0xffffffffu, f, o);
      s = (uint32_t)(xf_splitmix64(seed ^ f) >> 40) < p24 ? inv : 0.f;
    }
    const float e = __fmul_rn(caller_w ? __ldg(caller_w + row) : 1.f, s);
    if (lane == 0) {
      e_out[row] = e;
      if (e > 0.f) {
        const float c = ceilf(e);
        const unsigned long long m = c >= 2147483648.f ? 2147483648ull : (unsigned long long)c;
        w_acc += m * (unsigned long long)(end - beg);
      } else {
        ++skip_acc;
      }
    }
  }
  if (lane == 0) {
    if (w_acc) atomicAdd(W, w_acc);
    if (skip_acc) atomicAdd(skipped, skip_acc);
  }
}

void xf_launch_row_weights(const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* labels, const float* caller_w,
                           int B, bool sample, uint32_t p24, float inv, uint64_t seed, float* e_out,
                           unsigned long long* W, unsigned long long* skipped, cudaStream_t st) {
  if (B <= 0) return;
  const int grid = xf_grid_for((uint64_t)B * 32, 256, 8);
  xf_k_row_weights<<<grid, 256, 0, st>>>(row_ptr, keys, labels, caller_w, B, sample ? 1 : 0, p24, inv, seed, e_out, W,
                                         skipped);
}

// The forward passes' arithmetic shared by the serving kernels (serve.cu) and the deterministic training step
// (step_det.cu): the canonical FM's per-lane sums in xf_k_step_fmc's order, the multi-view machine's same-field adds in
// token order and its product over the present fields, and the launchers' map from K to the lane count C.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "kernels.h"

// The canonical forward's arithmetic, op for op as xf_k_step_fmc's machine code does it.  step_fmc.cu writes it with
// plain operators and nvcc contracts them into FMAs; which products it fuses is read off its SASS (cuobjdump -sass:
// the FMUL / FFMA / FADD after the latent load) and spelled out here with explicit rounding, so that a kernel using
// it computes the same bits whatever its own instantiation would contract:
//   a_k = x v_k;  S_k += a_k;  Q += fma(a3, a3, fma(a2, a2, fma(a1, a1, a0 a0)));  wx = fma(w, x, wx)  (lane c == 0)
//   s2 = fma(S3, S3, fma(S2, S2, fma(S0, S0, S1 S1)))  then the shuffle sums;  arg = fma(0.5, s2 - Q, wx)
__device__ __forceinline__ void xf_fmc_add(const float4& v, float x, float w, bool lead, float (&S)[4], float& Q, float& wx) {
  const float a0 = __fmul_rn(v.x, x), a1 = __fmul_rn(v.y, x), a2 = __fmul_rn(v.z, x), a3 = __fmul_rn(v.w, x);
  S[0] = __fadd_rn(S[0], a0); S[1] = __fadd_rn(S[1], a1); S[2] = __fadd_rn(S[2], a2); S[3] = __fadd_rn(S[3], a3);
  Q = __fadd_rn(Q, __fmaf_rn(a3, a3, __fmaf_rn(a2, a2, __fmaf_rn(a1, a1, __fmul_rn(a0, a0)))));
  if (lead) wx = __fmaf_rn(w, x, wx);
}
// S_k over the tokens (lanes with the same c), sum_k S_k^2 over the c's, Q and wx over the warp, in xf_k_step_fmc's
// order; the argument of the sigmoid
template <int C>
__device__ __forceinline__ float xf_fmc_arg(float (&S)[4], float Q, float wx) {
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int o = C; o < 32; o <<= 1) S[e] = __fadd_rn(S[e], __shfl_xor_sync(0xffffffffu, S[e], o));
  float s2 = __fmaf_rn(S[3], S[3], __fmaf_rn(S[2], S[2], __fmaf_rn(S[0], S[0], __fmul_rn(S[1], S[1]))));
#pragma unroll
  for (int o = 1; o < C; o <<= 1) s2 = __fadd_rn(s2, __shfl_xor_sync(0xffffffffu, s2, o));
  Q = xf_warp_sum(Q);
  wx = xf_warp_sum(wx);
  return __fmaf_rn(0.5f, __fsub_rn(s2, Q), wx);
}

// One pass's tokens into the warp's sums S[f][k]: lane (token, c) adds v[4c .. 4c+3] x into S[f][4c .. 4c+3] with one
// float4 read-modify-write.  The pass's tokens of one field are ranked in token order (lanes with the same (f, c), lower
// lanes holding earlier tokens) and added a rank per round, __syncwarp between rounds, so each S[f][k] takes its terms
// in token order and no two lanes touch one entry in a round.  A pass without two tokens of one field is one round.
template <int K>
__device__ __forceinline__ void xf_mvm_add(float (*S)[K], bool live, uint32_t f, int c, float4 v, float x) {
  const unsigned lane = threadIdx.x & 31u;
  const unsigned peers = __match_any_sync(0xffffffffu, live ? (f << 5 | (unsigned)c) : 0xFFFFFFFFu);
  const unsigned rank = __popc(peers & ((1u << lane) - 1u));
  const unsigned rounds = __reduce_max_sync(0xffffffffu, live ? rank + 1u : 0u);
  const float4 a = make_float4(__fmul_rn(v.x, x), __fmul_rn(v.y, x), __fmul_rn(v.z, x), __fmul_rn(v.w, x));
  float4* s = reinterpret_cast<float4*>(&S[f][4 * c]);
  for (unsigned r = 0; r < rounds; ++r) {
    if (live && rank == r) {
      float4 t = *s;
      t.x = __fadd_rn(t.x, a.x); t.y = __fadd_rn(t.y, a.y); t.z = __fadd_rn(t.z, a.z); t.w = __fadd_rn(t.w, a.w);
      *s = t;
    }
    __syncwarp();
  }
}

// Lane k < K's P_k = the product of S[f][k] over the present fields in ascending order; 0 on the other lanes and when
// no field is present.  The warp sum of the P_k is the machine's y.
template <int K>
__device__ __forceinline__ float xf_mvm_product(float (*S)[K], unsigned present) {
  const int lane = threadIdx.x & 31;
  float P = 0.f;
  if (lane < K && present) {
    P = 1.f;
    for (unsigned q = present; q; q &= q - 1) P = __fmul_rn(P, S[__ffs(q) - 1][lane]);
  }
  return P;
}

// f(std::integral_constant<int, C>()) for the lane count C = K/4 of latent dimension K, C <= MAX_C; a K that is not
// 4C for such a C takes C = MAX_C (the multi-view machine's kernels stop at 8: their shared memory grows with K)
template <int MAX_C, int C = 1, typename F>
inline void xf_with_lanes(int K, F&& f) {
  if constexpr (C < MAX_C) {
    if (K != 4 * C) return xf_with_lanes<MAX_C, 2 * C>(K, static_cast<F&&>(f));
  }
  f(std::integral_constant<int, C>());
}


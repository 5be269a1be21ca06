// The forward passes' arithmetic, stated once for every kernel that runs it: the canonical FM's per-lane sums and
// finishing step (xf_k_step_fmc, the deterministic step in step_det.cu, the canonical serving kernels), the multi-view
// machine's same-field adds in token order and its product over the present fields (step_det.cu, serve.cu), the
// field-aware FM's pass and pair sum (xf_k_step_ffm, the field-aware serving kernels), and the launchers' map from K to
// the lane count C.  Training and serving predict the same bits because they call the same functions here.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "kernels.h"
#include "table.cuh"

// Every float operation below names its rounding (__fmul_rn, __fadd_rn, __fmaf_rn), so no kernel's contraction of
// plain operators can change a result, and a kernel that inlines these functions computes the bits of every other.
// The FMAs are the ones nvcc chose when the training steps wrote the forward with plain operators, kept so that
// training's bits did not change when the steps came here.
//
// The canonical FM, C = K/4 lanes per token, lane c holding coordinates 4c .. 4c+3:
//   a_k = x v_k;  S_k += a_k;  Q += fma(a3, a3, fma(a2, a2, fma(a1, a1, a0 a0)));  wx = fma(w, x, wx)  (lane c == 0)
//   s2 = fma(S3, S3, fma(S2, S2, fma(S0, S0, S1 S1)))  then the shuffle sums;  arg = fma(0.5, s2 - Q, wx)
__device__ __forceinline__ void xf_fmc_add(const float4& v, float x, float w, bool lead, float (&S)[4], float& Q, float& wx) {
  const float a0 = __fmul_rn(v.x, x), a1 = __fmul_rn(v.y, x), a2 = __fmul_rn(v.z, x), a3 = __fmul_rn(v.w, x);
  S[0] = __fadd_rn(S[0], a0); S[1] = __fadd_rn(S[1], a1); S[2] = __fadd_rn(S[2], a2); S[3] = __fadd_rn(S[3], a3);
  Q = __fadd_rn(Q, __fmaf_rn(a3, a3, __fmaf_rn(a2, a2, __fmaf_rn(a1, a1, __fmul_rn(a0, a0)))));
  if (lead) wx = __fmaf_rn(w, x, wx);
}
// S_k over the tokens (lanes with the same c), sum_k S_k^2 over the c's, Q and wx over the warp; the argument of the
// sigmoid.  C is a run-time value so that xf_k_step_fmc, one kernel for every K, calls it too; a caller whose C is a
// constant gets the shuffle loops unrolled.
__device__ __forceinline__ float xf_fmc_arg(int C, float (&S)[4], float Q, float wx) {
#pragma unroll
  for (int e = 0; e < 4; ++e)
    for (int o = C; o < 32; o <<= 1) S[e] = __fadd_rn(S[e], __shfl_xor_sync(0xffffffffu, S[e], o));
  float s2 = __fmaf_rn(S[3], S[3], __fmaf_rn(S[2], S[2], __fmaf_rn(S[0], S[0], __fmul_rn(S[1], S[1]))));
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

// The field-aware FM, C = F = L/4 lanes per token, lane c holding the token's piece c (its vector for field c); the
// warp's field sums T[a][b] are F x F float4 in shared memory (T[a * C + b]), Σwx and Q are warp-uniform:
//   a_k = x v_k;  q = fma(a3, a3, fma(a2, a2, fma(a1, a1, a0 a0)))  (lane c == f);  wxt = w x  (lane c == 0)
//   Σwx = Σwx + wxt, Q = Q + q and T[f][c]_k = T[f][c]_k + a_k, each in token order
//   P = P + fma(u3, s3, fma(u2, s2, fma(u0, s0, u1 s1)))   u = T[a][b], s = T[b][a], a over the present fields ascending
//   arg = fma(0.5, (xor 16 .. 1 warp sum of P) - Q, Σwx)
// One pass's tokens into the warp's state: lane (token g, c) holds the token's field f, piece c of v, w and x; `on`: the
// token adds its terms.  Σwx and Q take the pass's first `groups` token groups in turn, a group that is not on adding
// +0; a field's tokens are ranked with __match_any_sync and added to T[f][*] a rank per round, lowest position first.
// ON_GROUPS: the groups are the ones whose lanes are on (which must be the pass's first ones), counted with a ballot.
template <int C, bool ON_GROUPS = false>
__device__ __forceinline__ void xf_ffm_add(float4* T, bool on, int groups, uint32_t f, float4 v, float w, float x,
                                           float& wx, float& Q) {
  constexpr int TP = 32 / C;
  const int lane = threadIdx.x & 31;
  const int c = lane & (C - 1);
  const int lead = lane & ~(C - 1);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  float q = 0.f, wxt = 0.f;
  if (on) {
    a = make_float4(__fmul_rn(v.x, x), __fmul_rn(v.y, x), __fmul_rn(v.z, x), __fmul_rn(v.w, x));
    if (c == (int)f) q = __fmaf_rn(a.w, a.w, __fmaf_rn(a.z, a.z, __fmaf_rn(a.y, a.y, __fmul_rn(a.x, a.x))));
    if (c == 0) wxt = __fmul_rn(w, x);
  }
  const float qt = __shfl_sync(0xffffffffu, q, lead + (int)f);  // the self term, from lane f of the token's group
  const int n = ON_GROUPS ? __popc(__ballot_sync(0xffffffffu, on)) / C : groups;
  for (int g = 0; g < n; ++g) {
    wx = __fadd_rn(wx, __shfl_sync(0xffffffffu, wxt, g * C));
    Q = __fadd_rn(Q, __shfl_sync(0xffffffffu, qt, g * C));
  }
  int rank = 0, last = 0;
  if (TP > 1) {
    const unsigned peers = __match_any_sync(0xffffffffu, on ? f : 0xFFu);
    rank = __popc(peers & ((1u << lead) - 1u)) / C;
    last = (int)__reduce_max_sync(0xffffffffu, on ? (unsigned)rank : 0u);
  }
  for (int r = 0; r <= last; ++r) {
    if (on && rank == r) {
      float4 s = T[f * C + c];
      s.x = __fadd_rn(s.x, a.x); s.y = __fadd_rn(s.y, a.y); s.z = __fadd_rn(s.z, a.z); s.w = __fadd_rn(s.w, a.w);
      T[f * C + c] = s;
    }
    __syncwarp();
  }
}

// the pair sum over the present fields and the sigmoid's argument (every lane returns it)
template <int C>
__device__ __forceinline__ float xf_ffm_arg(const float4* T, unsigned present, float wx, float Q) {
  const int lane = threadIdx.x & 31;
  float P = 0.f;
  if (lane < C && ((present >> lane) & 1u))
    for (unsigned q = present; q; q &= q - 1) {
      const int fa = __ffs(q) - 1;
      const float4 u = T[fa * C + lane], s = T[lane * C + fa];
      P = __fadd_rn(P, __fmaf_rn(u.w, s.w, __fmaf_rn(u.z, s.z, __fmaf_rn(u.x, s.x, __fmul_rn(u.y, s.y)))));
    }
  return __fmaf_rn(0.5f, __fsub_rn(xf_warp_sum(P), Q), wx);
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


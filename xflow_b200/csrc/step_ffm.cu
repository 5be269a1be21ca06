// The field-aware factorisation machine (Juan, Zhuang, Chin, Lin, RecSys 2016; libffm's model) on canonical tables.
// A key's latent row v[L] holds F = L / 4 pieces of 4 coordinates (libffm's default k = 4): piece b (coordinates
// 4b .. 4b+3) is v_{i,b}, the key's vector for interacting with field b.  Row r has tokens i (key, field f_i < F,
// value x_i, 1 without a value array):
//     y = sum_i w_i x_i + sum_{i<j} <v_{i,f_j}, v_{j,f_i}> x_i x_j            (pairs of token positions)
// through field sums T[a][b] = sum_{i: f_i = a} x_i v_{i,b} and Q = sum_i x_i^2 |v_{i,f_i}|^2:
//     y = sum_i w_i x_i + 1/2 ( sum_{a,b present} <T[a][b], T[b][a]> - Q )
//     dL/dw_i = r x_i ,  dL/dv_{i,b} = r x_i ( T[b][f_i] - [b = f_i] x_i v_{i,f_i} )      r = sigmoid(y) - label
// Per key the batch adds G = sum r x into g (with its first-touch marker, as step_fmc.cu) and the whole latent
// gradient into the L float accumulators A (one float4 RED per lane); the L accumulator stays 0, so xf_k_update
// takes gv = A / rows and applies FTRL / SGD per coordinate.  The canonical FM's A - v L2 factorisation does not
// carry over: the self term touches only the piece of the token's own field, and one key may occur under several.
//
// One warp per row, C = L/4 lanes per token (lane c holds the token's piece c, its vector for field c), 32/C
// tokens per pass.  T lives in shared memory, F x F float4 per warp (L^2 bytes).  Every part of the forward has a
// fixed order, so a row's pctr depends only on its tokens and on the table:
//   - T: each (a, b) is a left fold from +0 over the row's tokens of field a in ascending position (within a pass,
//     the token groups that share a field add in turn, lowest position first);
//   - sum w x and Q: left folds from +0 in ascending position;
//   - lane b adds <T[a][b], T[b][a]> over the present a ascending from +0, then the xor 16 .. 1 warp tree.
// T starts zeroed; after a row only the rows T[a][*] of its present fields are cleared again.  The forward's arithmetic
// is forward.cuh's (xf_ffm_add, xf_ffm_arg), which the serving kernels run too.
// Parity: a float64 numpy model (tests/ffm_model.py, tests/test_gpu_ffm.py).
#include <cuda_runtime.h>
#include <stdint.h>

#include "forward.cuh"

#define XF_NO_SLOT 0xFFFFFFFFu

template <int C>
__global__ void __launch_bounds__(256)
xf_k_step_ffm(XfTableView t, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
              const uint8_t* __restrict__ fields, const float* __restrict__ vals, const uint8_t* __restrict__ labels,
              int B, int mode, uint32_t* __restrict__ touched, float* __restrict__ loss_out,
              float* __restrict__ pctr_out, float* __restrict__ abs_loss_sum) {
  constexpr int F = C;        // fields = pieces per latent row
  constexpr int TP = 32 / C;  // tokens per pass
  extern __shared__ float4 s_T[];
  __shared__ float s_abs[8];
  float abs_acc = 0.f;
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const int gwarp = blockIdx.x * wpb + wib;
  const int nwarps = gridDim.x * wpb;
  const int c = lane & (C - 1);  // which piece
  const int tg = lane / C;       // which token of the pass
  const int lead = lane & ~(C - 1);
  float4* T = s_T + (size_t)wib * (F * F);  // T[a * F + b]
  for (int i = lane; i < F * F; i += 32) T[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncwarp();

  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row), end = __ldg(row_ptr + row + 1);
    unsigned present = 0u;
    float wx = 0.f, Q = 0.f;  // warp-uniform
    // ---------------- pass 1: pull, field sums, sum w x and Q in token order
    for (uint32_t j0 = beg; j0 < end; j0 += (uint32_t)TP) {
      const uint32_t j = j0 + (uint32_t)tg;
      const bool live = j < end;
      uint32_t slot = XF_NO_SLOT, flags = 0, f = 0;
      uint64_t key = 0;
      float w = 0.f;
      if (live && c == 0) {
        key = __ldcs(keys + j);
        f = (uint32_t)__ldg(fields + j) & (F - 1);
        XfHead h;
        const int64_t r = xf_probe<true>(t, key, &h);
        if (r >= 0) { slot = (uint32_t)r; flags = h.flags; w = h.w; }
        touched[j] = slot;  // remembered for pass 2 (overwritten there with the first-touch marker)
      }
      slot = __shfl_sync(0xffffffffu, slot, lead);
      flags = __shfl_sync(0xffffffffu, flags, lead);
      f = __shfl_sync(0xffffffffu, f, lead);
      key = __shfl_sync(0xffffffffu, (unsigned long long)key, lead);
      const bool ok = live && slot != XF_NO_SLOT;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      float x = 0.f;
      if (ok) {
        x = vals ? __ldg(vals + j) : 1.0f;
        if (flags & XF_FLAG_V_READY) v = __ldcg(reinterpret_cast<const float4*>(xf_row(t, slot) + 32) + c);
        else v = xf_v_init_piece(t, key, c);
      }
      // a live token without a row adds nothing to T and +0 to Σwx and Q
      xf_ffm_add<C>(T, ok, (int)min((uint32_t)TP, end - j0), f, v, w, x, wx, Q);
      if (ok) present |= 1u << f;
    }
    present = __reduce_or_sync(0xffffffffu, present);
    const float pctr = xf_sigmoid(xf_ffm_arg<C>(T, present, wx, Q));
    if (lane == 0 && pctr_out) pctr_out[row] = pctr;  // training: only for progressive validation
    if (mode == 0) {
      const float loss = pctr - (float)labels[row];
      if (lane == 0 && loss_out) loss_out[row] = loss;
      abs_acc += fabsf(loss);
      // ---------------- pass 2: per-key gradient sums
      for (uint32_t j0 = beg; j0 < end; j0 += (uint32_t)TP) {
        const uint32_t j = j0 + (uint32_t)tg;
        const bool live = j < end;
        uint32_t slot = XF_NO_SLOT, f = 0;
        if (live && c == 0) {
          slot = touched[j];
          f = (uint32_t)__ldg(fields + j) & (F - 1);
        }
        slot = __shfl_sync(0xffffffffu, slot, lead);
        f = __shfl_sync(0xffffffffu, f, lead);
        if (!live || slot == XF_NO_SLOT) continue;
        const float x = vals ? __ldg(vals + j) : 1.0f;
        uint8_t* rowp = xf_row(t, slot);
        float4 d = T[c * F + f];  // T[b][f_i], b = c
        if (c == (int)f) {
          // the self term, with the v pass 1 read (the step changes no v or flags)
          const uint32_t flags = __ldcg(reinterpret_cast<const unsigned int*>(rowp + XF_OFF_FLAGS));
          float4 v;
          if (flags & XF_FLAG_V_READY) v = __ldcg(reinterpret_cast<const float4*>(rowp + 32) + c);
          else {
            const uint64_t key = __ldcs(keys + j);
            v = xf_v_init_piece(t, key, c);
          }
          d.x -= v.x * x; d.y -= v.y * x; d.z -= v.z * x; d.w -= v.w * x;
        }
        const float rx = loss * x;
        atomicAdd(reinterpret_cast<float4*>(xf_row_ca(t, rowp)) + c, make_float4(rx * d.x, rx * d.y, rx * d.z, rx * d.w));
        if (c == 0) {
          const double old = atomicAdd(xf_row_g(rowp), (double)loss * (double)x);
          touched[j] = ((unsigned long long)__double_as_longlong(old) == XF_NEG_ZERO_BITS64) ? slot : XF_NO_SLOT;
        }
      }
    }
    // clear the rows of T this row used, for the warp's next row
    __syncwarp();
    if (lane < F)
      for (unsigned m = present; m; m &= m - 1) T[(__ffs(m) - 1) * F + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncwarp();
  }
  if (abs_loss_sum != nullptr && mode == 0) {
    if (lane == 0) s_abs[wib] = abs_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int w = 0; w < wpb; ++w) tot += s_abs[w];
      atomicAdd(abs_loss_sum, tot);
    }
  }
}

void xf_launch_step_ffm(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* fields,
                        const float* vals, const uint8_t* labels, int B, int mode, uint32_t* touched, float* loss_out,
                        float* pctr_out, float* abs_loss_sum, cudaStream_t st) {
  if (B <= 0) return;
  xf_with_lanes<32>(t.K, [&](auto C) {
    // C = 32 (L = 128) holds 16 KB of field sums per warp: 4 warps per CTA (64 KB, opt-in), 3 CTAs per SM
    constexpr int block = C == 32 ? 128 : 256;
    constexpr size_t smem = (size_t)(block / 32) * C * C * sizeof(float4);
    xf_k_step_ffm<C><<<xf_grid_smem((const void*)xf_k_step_ffm<C>, (uint64_t)B * 32, block, smem), block, smem, st>>>(
        t, row_ptr, keys, fields, vals, labels, B, mode, touched, loss_out, pctr_out, abs_loss_sum);
  });
}

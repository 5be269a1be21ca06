// A DEFINED multi-view machine behind the table API (SURVEY.md section 8f-4).  The reference's MVMWorker
// (src/model/mvm/mvm_worker.cc) sizes its per-row field sums by the row's LARGEST field id and then indexes them
// with that id (one past the end, :43,57,75,262) and multiplies in the zero sums of fields the row does not have
// (:86-92): its output depends on heap contents, so there is nothing to be bit-compatible with.  This is the
// model its code is reaching for, with every term defined:
//     s[f][k] = sum over the row's tokens of field f of v_ik x_i          (x = 1 without a value array)
//     y       = sum_k  prod over the fields f PRESENT in the row of s[f][k]          (a row without tokens: y = 0)
//     dL/dv_ik = r x_i prod_{f' present, f' != field(i)} s[f'][k]                     r = sigmoid(y) - label
// like mvm_worker.cc:60-92 (pull v only, per-k products over the field sums, sigmoid of their sum) and
// :255-300 (gradient = residual x product of the OTHER fields' sums); there is no linear term: the w of a row
// stays what it is (the optimizer step sees a zero gradient).  Per key the batch needs A_k = sum of the token
// gradients: the K float accumulators of canonical tables (table.cuh xf_row_ca); xf_k_update then takes
// gv_k = A_k / rows (the L accumulator stays 0) and applies FTRL / SGD per coordinate as for FM.
//
// One warp per row, C = K/4 lanes per token (one 16-byte piece of the latent row each), the per-(field, k) sums of
// the row in shared memory (XF_MVM_FIELDS x K floats per warp).  Field ids must be < XF_MVM_FIELDS (checked by
// the host entry point).  Parity: a float64 numpy model of the definition above (tests/test_gpu_parity.py).
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "table.cuh"

#define XF_NO_SLOT 0xFFFFFFFFu
#define XF_MVM_K_MAX 32

__global__ void __launch_bounds__(256)
xf_k_step_mvm(XfTableView t, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
              const uint8_t* __restrict__ fields, const float* __restrict__ vals, const uint8_t* __restrict__ labels,
              int B, int mode, uint32_t* __restrict__ touched, float* __restrict__ loss_out,
              float* __restrict__ pctr_out, float* __restrict__ abs_loss_sum) {
  __shared__ float s_sum[8][XF_MVM_FIELDS][XF_MVM_K_MAX];  // 32 KB
  __shared__ float s_abs[8];
  float abs_acc = 0.f;
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const int gwarp = blockIdx.x * wpb + wib;
  const int nwarps = gridDim.x * wpb;
  const int K = t.K;
  const int C = K >> 2;          // lanes per token (power of two, <= 8)
  const int T = 32 / C;          // tokens per pass
  const int c = lane & (C - 1);  // which 4 coordinates
  const int tg = lane / C;       // which token of the pass
  const int lead = lane & ~(C - 1);
  float (*S)[XF_MVM_K_MAX] = s_sum[wib];

  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row), end = __ldg(row_ptr + row + 1);
    for (int f = 0; f < XF_MVM_FIELDS; ++f) S[f][lane] = 0.f;
    __syncwarp();
    unsigned present = 0u;
    // ---------------- pass 1: pull, per-(field, k) sums
    for (uint32_t j0 = beg; j0 < end; j0 += (uint32_t)T) {
      const uint32_t j = j0 + (uint32_t)tg;
      const bool live = j < end;
      uint32_t slot = XF_NO_SLOT, flags = 0, f = 0;
      uint64_t key = 0;
      if (live && c == 0) {
        key = __ldcs(keys + j);
        f = (uint32_t)__ldg(fields + j) & (XF_MVM_FIELDS - 1);
        XfHead h;
        const int64_t r = xf_probe<true>(t, key, &h);
        if (r >= 0) { slot = (uint32_t)r; flags = h.flags; }
        touched[j] = slot;  // remembered for pass 2 (overwritten there with the first-touch marker)
      }
      slot = __shfl_sync(0xffffffffu, slot, lead);
      flags = __shfl_sync(0xffffffffu, flags, lead);
      f = __shfl_sync(0xffffffffu, f, lead);
      key = __shfl_sync(0xffffffffu, (unsigned long long)key, lead);
      if (!live || slot == XF_NO_SLOT) continue;
      const float x = vals ? __ldg(vals + j) : 1.0f;
      float4 v;
      if (flags & XF_FLAG_V_READY) v = __ldcg(reinterpret_cast<const float4*>(xf_row(t, slot) + 32) + c);
      else v = xf_v_init_piece(t, key, c);
      atomicAdd(&S[f][4 * c + 0], v.x * x);
      atomicAdd(&S[f][4 * c + 1], v.y * x);
      atomicAdd(&S[f][4 * c + 2], v.z * x);
      atomicAdd(&S[f][4 * c + 3], v.w * x);
      present |= 1u << f;
    }
    present = __reduce_or_sync(0xffffffffu, present);
    __syncwarp();
    // y = sum_k prod_f s[f][k]: lane k takes coordinate k
    float P = 0.f;
    if (lane < K && present) {
      P = 1.f;
      for (unsigned m = present; m; m &= m - 1) P *= S[__ffs(m) - 1][lane];
    }
    const float pctr = xf_sigmoid(xf_warp_sum(P));
    if (lane == 0 && pctr_out) pctr_out[row] = pctr;  // training: only for progressive validation
    if (mode == 1) {
      __syncwarp();
      continue;
    }
    const float loss = pctr - (float)labels[row];
    if (lane == 0 && loss_out) loss_out[row] = loss;
    abs_acc += fabsf(loss);
    // ---------------- pass 2: per-key gradient sums
    for (uint32_t j0 = beg; j0 < end; j0 += (uint32_t)T) {
      const uint32_t j = j0 + (uint32_t)tg;
      const bool live = j < end;
      uint32_t slot = XF_NO_SLOT, f = 0;
      if (live && c == 0) {
        slot = touched[j];
        f = (uint32_t)__ldg(fields + j) & (XF_MVM_FIELDS - 1);
      }
      slot = __shfl_sync(0xffffffffu, slot, lead);
      f = __shfl_sync(0xffffffffu, f, lead);
      if (!live || slot == XF_NO_SLOT) continue;
      const float x = vals ? __ldg(vals + j) : 1.0f;
      float o0 = 1.f, o1 = 1.f, o2 = 1.f, o3 = 1.f;  // products over the OTHER fields of the row
      for (unsigned m = present & ~(1u << f); m; m &= m - 1) {
        const float* sf = S[__ffs(m) - 1] + 4 * c;
        o0 *= sf[0]; o1 *= sf[1]; o2 *= sf[2]; o3 *= sf[3];
      }
      uint8_t* rowp = xf_row(t, slot);
      const float rx = loss * x;
      atomicAdd(reinterpret_cast<float4*>(xf_row_ca(t, rowp)) + c, make_float4(rx * o0, rx * o1, rx * o2, rx * o3));
      if (c == 0) {
        // first touch of the row in this batch (g: -0.0 = untouched; the w-gradient itself stays zero)
        const double old = atomicAdd(xf_row_g(rowp), 0.0);
        touched[j] = ((unsigned long long)__double_as_longlong(old) == XF_NEG_ZERO_BITS64) ? slot : XF_NO_SLOT;
      }
    }
    __syncwarp();  // the sums are zeroed again for the warp's next row
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

void xf_launch_step_mvm(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* fields,
                        const float* vals, const uint8_t* labels, int B, int mode, uint32_t* touched, float* loss_out,
                        float* pctr_out, float* abs_loss_sum, cudaStream_t st) {
  if (B <= 0) return;
  xf_k_step_mvm<<<xf_grid_for((uint64_t)B * 32, 256, 8), 256, 0, st>>>(t, row_ptr, keys, fields, vals, labels, B, mode,
                                                                        touched, loss_out, pctr_out, abs_loss_sum);
}

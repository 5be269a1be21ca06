// LR with "update on next touch" (lazy tables, K == 0): ONE kernel per batch, no optimizer kernel.
//
// The optimizer step of batch p for a key is not applied when batch p ends; the residual sum stays in
// the row (g, tagged p) and is folded in by the first token of a later batch b that touches the row
// ("opening" the row for b).  Every other reader applies it on the fly (xf_apply_pending, table.cuh), so
// the observable table is the reference's at every batch boundary.
//
// Why: on a multi-GB table every row-touching instruction costs about the same (load, store or atomic, hit or
// miss — tools/membench.cu), so the kernel's time is (row-touching instructions per token) x a fixed cost x
// tokens.  The eager pair (step + update) needs 4.3 per token, round 1's lazy protocol (load, CAS on the tag,
// full-sector store, RED) also 4.3 in one launch; this one 2.3:
//   phase A  load the row (1.3 with the collision probes) and compute, in registers, the weight the batch
//            pulls: the row's state with the pending step applied (pure function of what was loaded)
//   phase B  after the row reduction, ONE 128-bit CAS per distinct key of the token group deposits the
//            residual, publishes the new state and stamps the row for this batch (xf_lazy_deposit, table.cuh);
//            a key that another token of the batch has opened already gets a 64-bit integer add instead.
// No row is written before its residual is known, nobody waits, and because the residual sums are integers
// the result does not depend on the order in which the atomics land (bit-reproducible).
// Inside a warp, tokens with the same slot elect one lane (__match_any_sync): one deposit of
// count x residual per distinct key of a 32-token group.
//
// Tried on the 1e8-id table: bucketised probing (collision probes inside one 128-byte line: faster, kept), L2
// prefetch by dedicated warps running ahead (slower: the prefetches are requests too, removed), claim + publish
// in one CAS.128 with a separate RED (3.3 instructions per token: between round 1's protocol and this one).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "kernels.h"
#include "table.cuh"

#define XF_NO_SLOT 0xFFFFFFFFu
#define XF_LAZY_CACHED 2  // 64-token chunks whose group leaders keep their look at the row for phase B

__global__ void __launch_bounds__(256, 3)
xf_k_step_lr_lazy(XfTableView t, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
                  const uint8_t* __restrict__ labels, int B, int mode, uint32_t seq, uint32_t* rows_by_seq,
                  float* __restrict__ loss_out, float* __restrict__ pctr_out, float* __restrict__ abs_loss_sum,
                  unsigned long long* __restrict__ unique_total) {
  __shared__ float s_abs[8];
  __shared__ unsigned int s_open;
  if (threadIdx.x == 0) s_open = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0 && mode == 0) rows_by_seq[seq] = (uint32_t)B;  // read by later batches only
  __syncthreads();
  float abs_acc = 0.f;
  unsigned int open_acc = 0;
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * warps_per_block;

  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    const int chunks = (int)((end - beg + 63u) >> 6);
    float wsum = 0.f;
    // first XF_LAZY_CACHED chunks (rows <= 128 tokens), per half: if this lane leads its group of equal slots,
    // the slot, the group size, and the row's second half as it looked (old) and as it will be published (new)
    uint32_t lead_s[2 * XF_LAZY_CACHED];
    uint32_t cnt_c[XF_LAZY_CACHED];  // 8 bits per half
    uint64_t q2_c[2 * XF_LAZY_CACHED], q3_c[2 * XF_LAZY_CACHED], q2n_c[2 * XF_LAZY_CACHED];
#pragma unroll
    for (int c = 0; c < XF_LAZY_CACHED; ++c) {
      lead_s[2 * c] = lead_s[2 * c + 1] = XF_NO_SLOT;
      q2_c[2 * c] = q2_c[2 * c + 1] = q3_c[2 * c] = q3_c[2 * c + 1] = q2n_c[2 * c] = q2n_c[2 * c + 1] = 0ull;
      cnt_c[c] = 0;
    }

    // ---------------- phase A: pull every token's row; nothing is written
    for (int ch = 0; ch < chunks; ++ch) {
      const uint32_t j0 = beg + (uint32_t)ch * 64u + (uint32_t)lane;
      const uint32_t j1 = j0 + 32u;
      const bool v0 = j0 < end, v1 = j1 < end;
      const uint64_t k0 = v0 ? __ldcs(keys + j0) : 0ull;
      const uint64_t k1 = v1 ? __ldcs(keys + j1) : 0ull;
      const uint64_t p0 = xf_home_slot(t, k0), p1 = xf_home_slot(t, k1);
      XfHead h0, h1;
      h0.key = h1.key = XF_EMPTY_KEY;
      h0.flags = h1.flags = 0u;
      h0.w = h0.n = h0.z = h1.w = h1.n = h1.z = 0.f;
      h0.g = h1.g = 0.0;
      if (v0) h0 = xf_load_head(xf_row(t, p0));
      if (v1) h1 = xf_load_head(xf_row(t, p1));
      uint32_t s0 = XF_NO_SLOT, s1 = XF_NO_SLOT;
      if (v0) { const int64_t r = xf_probe_from<true>(t, k0, p0, h0); if (r >= 0) s0 = (uint32_t)r; }
      if (v1) { const int64_t r = xf_probe_from<true>(t, k1, p1, h1); if (r >= 0) s1 = (uint32_t)r; }
      // the weight this batch pulls = the row with its pending step applied (computed, not stored)
      const uint64_t a2 = xf_raw_q2(h0), a3 = xf_raw_q3(h0), b2 = xf_raw_q2(h1), b3 = xf_raw_q3(h1);
      uint64_t a2n = a2, b2n = b2;
      float w0 = 0.f, w1 = 0.f;
      if (s0 != XF_NO_SLOT) w0 = xf_lazy_fold(t, xf_raw_q1(h0), a2, a3, mode == 1 ? 0xFFFFFFFFu : seq, a2n);
      if (s1 != XF_NO_SLOT) w1 = xf_lazy_fold(t, xf_raw_q1(h1), b2, b3, mode == 1 ? 0xFFFFFFFFu : seq, b2n);
      wsum += w0;
      wsum += w1;
      if (mode == 1) continue;
      // lanes with the same slot elect their lowest lane; invalid lanes get unique dummy values
      const unsigned grp0 = __match_any_sync(0xffffffffu, (s0 != XF_NO_SLOT) ? s0 : (0xFFFFFF00u | (uint32_t)lane));
      const unsigned grp1 = __match_any_sync(0xffffffffu, (s1 != XF_NO_SLOT) ? s1 : (0xFFFFFF00u | (uint32_t)lane));
      const bool L0 = s0 != XF_NO_SLOT && lane == __ffs(grp0) - 1, L1 = s1 != XF_NO_SLOT && lane == __ffs(grp1) - 1;
      if (ch >= XF_LAZY_CACHED) {
        // long rows (> 128 tokens): nothing is remembered for phase B; open the row now with an empty deposit
        if (L0 && xf_lazy_deposit(t, xf_row(t, s0), a2, a3, a2n, seq, 0ll)) ++open_acc;
        if (L1 && xf_lazy_deposit(t, xf_row(t, s1), b2, b3, b2n, seq, 0ll)) ++open_acc;
      }
#pragma unroll
      for (int c = 0; c < XF_LAZY_CACHED; ++c)
        if (ch == c) {
          lead_s[2 * c] = L0 ? s0 : XF_NO_SLOT;
          lead_s[2 * c + 1] = L1 ? s1 : XF_NO_SLOT;
          q2_c[2 * c] = a2; q3_c[2 * c] = a3; q2n_c[2 * c] = a2n;
          q2_c[2 * c + 1] = b2; q3_c[2 * c + 1] = b3; q2n_c[2 * c + 1] = b2n;
          cnt_c[c] = (L0 ? (uint32_t)__popc(grp0) : 0u) | ((L1 ? (uint32_t)__popc(grp1) : 0u) << 8);
        }
    }

    const float wx = xf_warp_sum(wsum);
    const float pctr = xf_sigmoid(wx);
    if (mode == 1) {
      if (lane == 0 && pctr_out) pctr_out[row] = pctr;
      continue;
    }
    const float loss = __fsub_rn(pctr, (float)labels[row]);  // lr_worker.cc:141
    if (lane == 0 && loss_out) loss_out[row] = loss;
    abs_acc += fabsf(loss);
    // ---------------- phase B: one deposit per distinct key of a token group: count x residual, integer, exact
    const long long lf = xf_fix_of(loss);
#pragma unroll
    for (int c = 0; c < XF_LAZY_CACHED; ++c) {
      if (lead_s[2 * c] != XF_NO_SLOT &&
          xf_lazy_deposit(t, xf_row(t, lead_s[2 * c]), q2_c[2 * c], q3_c[2 * c], q2n_c[2 * c], seq, lf * (long long)(cnt_c[c] & 0xFFu)))
        ++open_acc;
      if (lead_s[2 * c + 1] != XF_NO_SLOT &&
          xf_lazy_deposit(t, xf_row(t, lead_s[2 * c + 1]), q2_c[2 * c + 1], q3_c[2 * c + 1], q2n_c[2 * c + 1], seq,
                          lf * (long long)(cnt_c[c] >> 8)))
        ++open_acc;
    }
    for (int ch = XF_LAZY_CACHED; ch < chunks; ++ch) {
      // long rows (> 128 tokens): the rows were opened in phase A
      const uint32_t j0 = beg + (uint32_t)ch * 64u + (uint32_t)lane;
      const uint32_t j1 = j0 + 32u;
      XfHead h;
      if (j0 < end) { const int64_t r = xf_probe<false>(t, __ldg(keys + j0), &h); if (r >= 0) xf_lazy_add(xf_row(t, (uint64_t)r), lf); }
      if (j1 < end) { const int64_t r = xf_probe<false>(t, __ldg(keys + j1), &h); if (r >= 0) xf_lazy_add(xf_row(t, (uint64_t)r), lf); }
    }
  }
  if (mode == 0) {
    if (lane == 0) s_abs[threadIdx.x >> 5] = abs_acc;
    if (open_acc) atomicAdd(&s_open, open_acc);
    __syncthreads();
    if (threadIdx.x == 0) {
      if (abs_loss_sum != nullptr) {
        float tot = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += s_abs[w];
        atomicAdd(abs_loss_sum, tot);
      }
      if (unique_total != nullptr && s_open) atomicAdd(unique_total, (unsigned long long)s_open);
    }
  }
}

void xf_launch_step_lr_lazy(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys,
                            const uint8_t* labels, int B, int mode, uint32_t seq, uint32_t* rows_by_seq,
                            float* loss_out, float* pctr_out, float* abs_loss_sum, unsigned long long* unique_total,
                            cudaStream_t st) {
  if (B <= 0) return;
  const int grid = xf_grid_for((uint64_t)B * 32, 256, 8);
  xf_k_step_lr_lazy<<<grid, 256, 0, st>>>(t, row_ptr, keys, labels, B, mode, seq, rows_by_seq, loss_out, pctr_out,
                                           abs_loss_sum, unique_total);
}

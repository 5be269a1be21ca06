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
//            pulls: the row's state with the pending step applied (pure function of what was loaded).
//            sm_90 has no 256-bit load: a 32-byte row read by one lane is two 128-bit loads, i.e. two requests,
//            so the probe runs convergent across the warp, one look per round for every unresolved token, and
//            every look is a lane-pair load (xf_ld32_pair, table.cuh) that costs one request per row.
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
// On the H100 the rule above holds only in part: a lane-pair row look runs at 1.4x the rate of a one-lane one,
// not 2x, and an atomic costs about 2.5 paired looks (tools/membench.cu), so phase B's CAS.128 sets most of the
// kernel's time.
// What a CAS.128 costs depends on whether it finds the line its row's look brought into L2: 49 ps per row right after
// the look, 82 ps once the GPU has looked at about 25 MB of other lines in between (tools/membench.cu, "look, then
// CAS.128 after D MB").  So a row should close (deposit) soon after it is first looked at.  Its phase-B CASes are all
// sent before any answer is acted on (xf_lazy_deposit_issue / _resolve), where one at a time they used to add up to
// three CAS round trips to every row; its label and second chunk's keys are loaded when the row starts.  The grid is
// the CTAs that fit on the GPU at once, 2 per SM.  Measured and slower (DESIGN.md section 6): fewer rows open (1 CTA
// per SM, or 128-thread CTAs), and all 128 tokens' first looks issued together in one probe chain (more looks in
// flight per warp; with the row loads of the next row prefetched, slower still).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "kernels.h"
#include "table.cuh"

#define XF_NO_SLOT 0xFFFFFFFFu
#define XF_LAZY_CACHED 2  // 64-token chunks whose group leaders keep their look at the row for phase B

// One step of xf_probe_from<true> for a token of `key` whose probe number i is at slot s and whose look at that
// row is (q0..q3).  Returns true when the token is resolved: found (slot = s), inserted (q0..q3 = what xf_k_fill
// left in the row with the key claimed, *created = true), or out of probes (slot stays XF_NO_SLOT, *t.error = 1).
// Otherwise s and i move on to the next probe slot, which the caller loads.
// ADMIT: an absent key asks the admission policy before its CAS; a key it does not admit resolves with slot =
// XF_NO_SLOT (it pulls w = 0 and takes no part in phase B) and *rejected = true (predict: false, nothing counted).
// STAMP (feature eviction): a key this look inserts is stamped with sv.now.
template <bool ADMIT, bool STAMP>
__device__ __forceinline__ bool xf_lazy_look(const XfTableView& t, uint64_t key, uint64_t& s, uint32_t& i, uint64_t& q0,
                                             uint64_t& q1, uint64_t& q2, uint64_t& q3, uint32_t& slot, bool& created,
                                             const XfAdmitView& adm, bool& rejected, const XfStampView& sv) {
  if (q0 == key) { slot = (uint32_t)s; return true; }
  if (q0 == XF_EMPTY_KEY) {
    if (ADMIT && !xf_admit(adm, key)) {
      rejected = adm.mode != XF_ADM_NEVER;
      return true;
    }
    const unsigned long long old =
        atomicCAS(reinterpret_cast<unsigned long long*>(xf_row(t, s)), (unsigned long long)XF_EMPTY_KEY, (unsigned long long)key);
    if (old == XF_EMPTY_KEY) {
      if (STAMP) sv.stamp[s] = sv.now;
      created = true;
      q0 = key; q1 = q2 = q3 = 0ull;  // lazy rows: g is the integer 0, no state, no tag
      slot = (uint32_t)s;
      return true;
    }
    if (old == key) {  // raced with another inserter of the same key: the other fields are still what was loaded
      q0 = key;
      slot = (uint32_t)s;
      return true;
    }
    // a different key took the slot: on to the next one
  }
  if (++i == XF_MAX_PROBE) { *t.error = 1; return true; }
  s = xf_probe_slot(t, key, i);
  return false;
}

// ADMIT = false is the kernel without an admission policy (every absent key is inserted); ADMIT = true asks `adm`.
// STAMP = true (feature eviction) stores stamp[slot] = sv.now where a key is inserted and where a training
// batch opens a row (the deposit that returns true: once per key and batch); STAMP = false is the kernel without it.
// WEIGHT = true (importance weighting, weight.cu; training only): a row with wv.e[row] = 0 is skipped before phase A
// (no probe, no insert, no admission, no stamp, no deposit; loss_out 0); every other row deposits the weighted
// residual e x (pctr - label), and the fixed-point unit comes from the device bound *wv.W instead of fix_shift.
template <bool ADMIT, bool STAMP, bool WEIGHT>
__global__ void __launch_bounds__(256, 2)
xf_k_step_lr_lazy(XfTableView t, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
                  const uint8_t* __restrict__ labels, int B, int mode, uint32_t seq, uint64_t* rows_by_seq, int fix_shift,
                  float* __restrict__ loss_out, float* __restrict__ pctr_out, float* __restrict__ abs_loss_sum,
                  unsigned long long* __restrict__ unique_total, XfAdmitView adm, XfStampView sv, XfWeightView wv) {
  __shared__ float s_abs[8];
  __shared__ unsigned int s_open;
  if (WEIGHT) fix_shift = xf_fix_shift(*wv.W);  // the host does not know W of a device batch
  // the group leaders' looks at their rows, from phase A to phase B.  In registers (24 more) they would take the
  // kernel past the 128 registers that 2 CTAs of 256 threads per SM leave it.
  __shared__ uint64_t s_q2[2 * XF_LAZY_CACHED][256], s_q3[2 * XF_LAZY_CACHED][256], s_q2n[2 * XF_LAZY_CACHED][256];
  if (threadIdx.x == 0) s_open = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0 && mode == 0)  // read by later batches only
    rows_by_seq[seq] = (uint64_t)(uint32_t)B | ((uint64_t)fix_shift << 32);
  __syncthreads();
  float abs_acc = 0.f;
  unsigned int open_acc = 0;
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * warps_per_block;

  for (int row = gwarp; row < B; row += nwarps) {
    if (WEIGHT && __ldg(wv.e + row) == 0.f) {
      if (lane == 0 && loss_out) loss_out[row] = 0.f;
      continue;
    }
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    const int chunks = (int)((end - beg + 63u) >> 6);
    // loaded now, used once the row is summed: the label, and the keys of the second chunk, needed after the first
    // chunk's probe; neither load then stands between the row's first look and its deposits
    const uint8_t label = mode == 0 ? labels[row] : 0;
    uint64_t k1_0 = 0ull, k1_1 = 0ull;
    if (beg + 64u + (uint32_t)lane < end) k1_0 = __ldcs(keys + beg + 64u + lane);
    if (beg + 96u + (uint32_t)lane < end) k1_1 = __ldcs(keys + beg + 96u + lane);
    float wsum = 0.f;
    // first XF_LAZY_CACHED chunks (rows <= 128 tokens), per half: if this lane leads its group of equal slots,
    // the slot, the group size, and the row's second half as it looked (old) and as it will be published (new)
    // (the old and new second halves live in shared memory: s_q2 / s_q3 / s_q2n, indexed like lead_s)
    uint32_t lead_s[2 * XF_LAZY_CACHED];
    uint32_t cnt_c[XF_LAZY_CACHED];  // 8 bits per half
#pragma unroll
    for (int c = 0; c < XF_LAZY_CACHED; ++c) {
      lead_s[2 * c] = lead_s[2 * c + 1] = XF_NO_SLOT;
      cnt_c[c] = 0;
    }

    // ---------------- phase A: pull every token's row; nothing is written
    for (int ch = 0; ch < chunks; ++ch) {
      const uint32_t j0 = beg + (uint32_t)ch * 64u + (uint32_t)lane;
      const uint32_t j1 = j0 + 32u;
      const bool v0 = j0 < end, v1 = j1 < end;
      uint64_t k0 = k1_0, k1 = k1_1;
      if (ch != 1) {
        k0 = v0 ? __ldcs(keys + j0) : 0ull;
        k1 = v1 ? __ldcs(keys + j1) : 0ull;
      }
      uint64_t p0 = xf_home_slot(t, k0), p1 = xf_home_slot(t, k1);
      // the probe (xf_probe_from<true>), one look per round for every token of the warp that is still unresolved,
      // so that every look is a lane-pair load
      uint64_t a0, a1, a2, a3, b0, b1, b2, b3;
      xf_ld32_pair(v0 ? xf_row(t, p0) : nullptr, a0, a1, a2, a3);
      xf_ld32_pair(v1 ? xf_row(t, p1) : nullptr, b0, b1, b2, b3);
      uint32_t s0 = XF_NO_SLOT, s1 = XF_NO_SLOT, i0 = 0, i1 = 0;
      bool u0 = v0, u1 = v1, r0 = false, r1 = false;
      for (;;) {
        bool c0 = false, c1 = false;
        if (u0) u0 = !xf_lazy_look<ADMIT, STAMP>(t, k0, p0, i0, a0, a1, a2, a3, s0, c0, adm, r0, sv);
        if (u1) u1 = !xf_lazy_look<ADMIT, STAMP>(t, k1, p1, i1, b0, b1, b2, b3, s1, c1, adm, r1, sv);
        const unsigned created = __popc(__ballot_sync(0xffffffffu, c0)) + __popc(__ballot_sync(0xffffffffu, c1));
        if (created && lane == 0) {
          atomicAdd(t.size, (unsigned long long)created);
          if (ADMIT) atomicAdd(adm.admitted, (unsigned long long)created);
        }
        if (!__any_sync(0xffffffffu, u0 || u1)) break;
        uint64_t x0, x1, x2, x3;
        xf_ld32_pair(u0 ? xf_row(t, p0) : nullptr, x0, x1, x2, x3);
        if (u0) { a0 = x0; a1 = x1; a2 = x2; a3 = x3; }
        xf_ld32_pair(u1 ? xf_row(t, p1) : nullptr, x0, x1, x2, x3);
        if (u1) { b0 = x0; b1 = x1; b2 = x2; b3 = x3; }
      }
      if (ADMIT) xf_admit_append(adm, r0, k0, r1, k1);
      // the weight this batch pulls = the row with its pending step applied (computed, not stored)
      uint64_t a2n = a2, b2n = b2;
      float w0 = 0.f, w1 = 0.f;
      if (s0 != XF_NO_SLOT) w0 = xf_lazy_fold(t, a1, a2, a3, mode == 1 ? 0xFFFFFFFFu : seq, a2n);
      if (s1 != XF_NO_SLOT) w1 = xf_lazy_fold(t, b1, b2, b3, mode == 1 ? 0xFFFFFFFFu : seq, b2n);
      wsum += w0;
      wsum += w1;
      if (mode == 1) continue;
      // lanes with the same slot elect their lowest lane; invalid lanes get unique dummy values
      const unsigned grp0 = __match_any_sync(0xffffffffu, (s0 != XF_NO_SLOT) ? s0 : (0xFFFFFF00u | (uint32_t)lane));
      const unsigned grp1 = __match_any_sync(0xffffffffu, (s1 != XF_NO_SLOT) ? s1 : (0xFFFFFF00u | (uint32_t)lane));
      const bool L0 = s0 != XF_NO_SLOT && lane == __ffs(grp0) - 1, L1 = s1 != XF_NO_SLOT && lane == __ffs(grp1) - 1;
      if (ch >= XF_LAZY_CACHED) {
        // long rows (> 128 tokens): nothing is remembered for phase B; open the row now with an empty deposit
        if (L0 && xf_lazy_deposit(t, xf_row(t, s0), a2, a3, a2n, seq, 0ll)) {
          ++open_acc;
          if (STAMP) sv.stamp[s0] = sv.now;
        }
        if (L1 && xf_lazy_deposit(t, xf_row(t, s1), b2, b3, b2n, seq, 0ll)) {
          ++open_acc;
          if (STAMP) sv.stamp[s1] = sv.now;
        }
      }
#pragma unroll
      for (int c = 0; c < XF_LAZY_CACHED; ++c)
        if (ch == c) {
          lead_s[2 * c] = L0 ? s0 : XF_NO_SLOT;
          lead_s[2 * c + 1] = L1 ? s1 : XF_NO_SLOT;
          cnt_c[c] = (L0 ? (uint32_t)__popc(grp0) : 0u) | ((L1 ? (uint32_t)__popc(grp1) : 0u) << 8);
        }
      if (ch < XF_LAZY_CACHED) {
        if (L0) { s_q2[2 * ch][threadIdx.x] = a2; s_q3[2 * ch][threadIdx.x] = a3; s_q2n[2 * ch][threadIdx.x] = a2n; }
        if (L1) { s_q2[2 * ch + 1][threadIdx.x] = b2; s_q3[2 * ch + 1][threadIdx.x] = b3; s_q2n[2 * ch + 1][threadIdx.x] = b2n; }
      }
    }

    const float wx = xf_warp_sum(wsum);
    const float pctr = xf_sigmoid(wx);
    if (mode == 1) {
      if (lane == 0 && pctr_out) pctr_out[row] = pctr;
      continue;
    }
    float loss = __fsub_rn(pctr, (float)label);  // lr_worker.cc:141
    if (lane == 0 && loss_out) loss_out[row] = loss;
    if (WEIGHT) loss = __fmul_rn(__ldg(wv.e + row), loss);  // read again: not kept live through phase A
    abs_acc += fabsf(loss);
    // ---------------- phase B: one deposit per distinct key of a token group: count x residual, integer, exact
    const long long lf = xf_fix_of(loss, fix_shift);
    // every deposit of the row is sent before any answer is looked at, so that the row's CASes are in flight together
    uint64_t o2[2 * XF_LAZY_CACHED], o3[2 * XF_LAZY_CACHED];
    bool issued[2 * XF_LAZY_CACHED];
#pragma unroll
    for (int g = 0; g < 2 * XF_LAZY_CACHED; ++g) {
      const int x = threadIdx.x;
      issued[g] = lead_s[g] != XF_NO_SLOT &&
                  xf_lazy_deposit_issue(xf_row(t, lead_s[g]), s_q2[g][x], s_q3[g][x], s_q2n[g][x], seq,
                                        lf * (long long)((cnt_c[g >> 1] >> (8 * (g & 1))) & 0xFFu), o2[g], o3[g]);
    }
#pragma unroll
    for (int g = 0; g < 2 * XF_LAZY_CACHED; ++g) {
      const int x = threadIdx.x;
      bool stale = false;
      if (issued[g] && xf_lazy_deposit_resolve(xf_row(t, lead_s[g]), true, s_q2[g][x], s_q3[g][x], o2[g], o3[g], seq,
                                               lf * (long long)((cnt_c[g >> 1] >> (8 * (g & 1))) & 0xFFu), &stale)) {
        ++open_acc;
        if (STAMP) sv.stamp[lead_s[g]] = sv.now;
      }
      if (stale) *t.error = 2;  // inside a batch a row only ever goes from "pending" to "open for seq"
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

// CTAs of the kernel that fit on one SM at once
template <bool A, bool S, bool W>
static int xf_lazy_ctas_per_sm() {
  static const int n = [] {
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, xf_k_step_lr_lazy<A, S, W>, 256, 0) != cudaSuccess || v < 1) {
      cudaGetLastError();
      v = 1;
    }
    return v;
  }();
  return n;
}

void xf_launch_step_lr_lazy(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys,
                            const uint8_t* labels, int B, uint64_t nnz, int mode, uint32_t seq, uint64_t* rows_by_seq,
                            float* loss_out, float* pctr_out, float* abs_loss_sum, unsigned long long* unique_total,
                            const XfAdmitView* adm, const XfStampView& sv, const XfWeightView& wv, cudaStream_t st) {
  if (B <= 0) return;
  const int fs = xf_fix_shift(nnz);  // nnz bounds every key's residual sum in this batch (weighted: *wv.W, in-kernel)
  const XfAdmitView a = adm ? *adm : XfAdmitView{};
#define XF_LAZY_ARGS t, row_ptr, keys, labels, B, mode, seq, rows_by_seq, fs, loss_out, pctr_out, abs_loss_sum, unique_total, a, sv, wv
  // a grid of the CTAs that fit on the GPU at once (or fewer, for a small batch): each warp strides over the rows
#define XF_LAZY_LAUNCH(A, S, W)                                                                                      \
  xf_k_step_lr_lazy<A, S, W><<<xf_grid_for((uint64_t)B * 32, 256, xf_lazy_ctas_per_sm<A, S, W>()), 256, 0, st>>>( \
      XF_LAZY_ARGS)
#define XF_LAZY_LAUNCH_W(A, S)            \
  do {                                    \
    if (wv.e) XF_LAZY_LAUNCH(A, S, true); \
    else XF_LAZY_LAUNCH(A, S, false);     \
  } while (0)
  const bool stamp = sv.stamp != nullptr;
  if (adm && stamp) XF_LAZY_LAUNCH_W(true, true);
  else if (adm) XF_LAZY_LAUNCH_W(true, false);
  else if (stamp) XF_LAZY_LAUNCH_W(false, true);
  else XF_LAZY_LAUNCH_W(false, false);
#undef XF_LAZY_LAUNCH_W
#undef XF_LAZY_LAUNCH
#undef XF_LAZY_ARGS
}

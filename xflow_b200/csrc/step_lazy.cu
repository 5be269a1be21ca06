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
// CAS.128 after D MB").  So a row should close (deposit) soon after it is first looked at.  A row belongs to a group of
// 128 threads (64 when the batch's rows average at most 64 tokens), one token per thread, so all of a row's first
// looks go out in one round; a warp that owned a row with two tokens per lane looked at a 100-token row in two 64-token
// chunks, one after the other, and kept the row open for at least two look latencies.  The group's first warp sums
// the row in that warp's order (bit-identical pctr) and hands the residual to the group through shared memory; each
// group leader then sends its CAS at once and acts on the answer after (xf_lazy_deposit_issue / _resolve).  At 62-64
// registers the kernel runs 4 CTAs of 256 per SM: 1 024 tokens per SM in flight, as before with 512 threads of two
// tokens.  The grid is the CTAs that fit on the GPU at once.  Measured and slower (DESIGN.md section 6): fewer rows
// open (1 CTA per SM, 128-thread CTAs, or this mapping at 2 CTAs per SM), and all 128 tokens' first looks issued
// together in one probe chain per warp (more looks in flight per warp; with the row loads of the next row
// prefetched, slower still).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "kernels.h"
#include "table.cuh"

#define XF_NO_SLOT 0xFFFFFFFFu

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

// The named barrier of row group `grp` of the CTA (barrier 1 + grp: 0 is __syncthreads'); n = the group's threads.
// The ids are immediates: with an id in a register ptxas reserves all 16 barriers for the CTA.
__device__ __forceinline__ void xf_group_sync(int grp, int n) {
  switch (grp) {
    case 0: asm volatile("bar.sync 1, %0;" ::"r"(n) : "memory"); break;
    case 1: asm volatile("bar.sync 2, %0;" ::"r"(n) : "memory"); break;
    case 2: asm volatile("bar.sync 3, %0;" ::"r"(n) : "memory"); break;
    default: asm volatile("bar.sync 4, %0;" ::"r"(n) : "memory"); break;
  }
}

// A group of G = 2^gshift threads (64 or 128, xf_launch_step_lr_lazy) per row, one token per thread: token beg + G r + x
// of round r to thread x of the group, so warp w of a round holds the row's tokens 32 w .. 32 w + 31 of that round.
// ADMIT = false is the kernel without an admission policy (every absent key is inserted); ADMIT = true asks `adm`.
// STAMP = true (feature eviction) stores stamp[slot] = sv.now where a key is inserted and where a training
// batch opens a row (the deposit that returns true: once per key and batch); STAMP = false is the kernel without it.
// WEIGHT = true (importance weighting, weight.cu; training only): a row with wv.e[row] = 0 is skipped before phase A
// (no probe, no insert, no admission, no stamp, no deposit; loss_out 0); every other row deposits the weighted
// residual e x (pctr - label), and the fixed-point unit comes from the device bound *wv.W instead of fix_shift.
// ADAGRAD = true for AdaGrad tables, false for FTRL and SGD ones (xf_lazy_fold_t).
template <bool ADMIT, bool STAMP, bool WEIGHT, bool ADAGRAD>
__global__ void __launch_bounds__(256, 4)
xf_k_step_lr_lazy(XfTableView t, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
                  const uint8_t* __restrict__ labels, int B, int mode, uint32_t seq, uint64_t* rows_by_seq, int fix_shift,
                  int gshift, float* __restrict__ loss_out, float* __restrict__ pctr_out, float* __restrict__ abs_loss_sum,
                  unsigned long long* __restrict__ unique_total, XfAdmitView adm, XfStampView sv, XfWeightView wv) {
  __shared__ float s_w[256];        // the weight each thread's token pulls, for its group's warp 0 to sum
  __shared__ long long s_lf[4];     // each group's row residual in fixed point, from its warp 0 to the group
  __shared__ float s_abs[8];
  __shared__ unsigned int s_open;
  if (WEIGHT) fix_shift = xf_fix_shift(*wv.W);  // the host does not know W of a device batch
  if (threadIdx.x == 0) s_open = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0 && mode == 0)  // read by later batches only
    rows_by_seq[seq] = (uint64_t)(uint32_t)B | ((uint64_t)fix_shift << 32);
  __syncthreads();
  float abs_acc = 0.f;
  unsigned int open_acc = 0;
  const int G = 1 << gshift;
  const int lane = threadIdx.x & 31;
  const int x = threadIdx.x & (G - 1);  // this thread's token in each round of the row
  const int grp = threadIdx.x >> gshift;
  const int gbase = grp << gshift;      // the group's slice of s_w
  const bool summer = x < 32;           // warp 0 of the group sums the row
  const int groups_per_block = blockDim.x >> gshift;

  for (int row = blockIdx.x * groups_per_block + grp; row < B; row += gridDim.x * groups_per_block) {
    if (WEIGHT && __ldg(wv.e + row) == 0.f) {
      if (x == 0 && loss_out) loss_out[row] = 0.f;
      continue;
    }
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    const int rounds = (int)((end - beg + (uint32_t)G - 1u) >> gshift);
    // loaded now, used once the row is summed: the load does not stand between the row's first look and its deposits
    const uint8_t label = (mode == 0 && summer) ? labels[row] : 0;
    float wsum = 0.f;
    // round 0 (rows <= G tokens): if this thread leads its warp's group of equal slots, the slot, the group size, and
    // the row's second half as it looked (q2, q3) and as it will be published (q2n)
    uint32_t lead_s = XF_NO_SLOT, cnt = 0;
    uint64_t lq2 = 0ull, lq3 = 0ull, lq2n = 0ull;
    bool lmark = false;  // the row carries an imported weight and has not been opened since (xf_lazy_mark_open)

    // ---------------- phase A: pull every token's row; nothing is written
    for (int rd = 0; rd < rounds; ++rd) {
      const uint32_t j = beg + ((uint32_t)rd << gshift) + (uint32_t)x;
      const bool v = j < end;
      const uint64_t k = v ? __ldcs(keys + j) : 0ull;
      uint64_t p = xf_home_slot(t, k);
      // the probe (xf_probe_from<true>), one look per round for every token of the warp that is still unresolved,
      // so that every look is a lane-pair load
      uint64_t a0, a1, a2, a3;
      xf_ld32_pair(v ? xf_row(t, p) : nullptr, a0, a1, a2, a3);
      uint32_t s = XF_NO_SLOT, i = 0;
      bool u = v, r = false;
      for (;;) {
        bool c = false;
        if (u) u = !xf_lazy_look<ADMIT, STAMP>(t, k, p, i, a0, a1, a2, a3, s, c, adm, r, sv);
        const unsigned created = __popc(__ballot_sync(0xffffffffu, c));
        if (created && lane == 0) {
          atomicAdd(t.size, (unsigned long long)created);
          if (ADMIT) atomicAdd(adm.admitted, (unsigned long long)created);
        }
        if (!__any_sync(0xffffffffu, u)) break;
        uint64_t x0, x1, x2, x3;
        xf_ld32_pair(u ? xf_row(t, p) : nullptr, x0, x1, x2, x3);
        if (u) { a0 = x0; a1 = x1; a2 = x2; a3 = x3; }
      }
      if (ADMIT) xf_admit_append(adm, r, k);
      // the weight this batch pulls = the row with its pending step applied (computed, not stored)
      uint64_t a2n = a2;
      float w = 0.f;
      if (s != XF_NO_SLOT) w = xf_lazy_fold_t<ADAGRAD>(t, a1, a2, a3, mode == 1 ? 0xFFFFFFFFu : seq, a2n);
      s_w[threadIdx.x] = w;
      if (mode == 0) {
        // lanes with the same slot elect their lowest lane; invalid lanes get unique dummy values
        const unsigned gm = __match_any_sync(0xffffffffu, (s != XF_NO_SLOT) ? s : (0xFFFFFF00u | (uint32_t)lane));
        const bool L = s != XF_NO_SLOT && lane == __ffs(gm) - 1;
        if (rd == 0) {
          if (L) {
            lead_s = s; cnt = (uint32_t)__popc(gm); lq2 = a2; lq3 = a3; lq2n = a2n;
            lmark = (a3 & XF_TAG_MASK) == 0ull && (uint32_t)(a1 >> 32) == xf_lazy_check(a2);
          }
        } else if (L && xf_lazy_deposit(t, xf_row(t, s), a2, a3, a2n, seq, 0ll)) {
          // long rows (> G tokens): nothing is remembered for phase B; open the row now with an empty deposit
          xf_lazy_mark_open(xf_row(t, s), a1, a2, a3, seq);
          ++open_acc;
          if (STAMP) sv.stamp[s] = sv.now;
        }
      }
      // lane l of warp 0 adds the weights of tokens l, l + 32, ... of each round in turn: the order in which a warp
      // holding two tokens per lane per 64-token chunk added them, so pctr is the same float whatever G is
      xf_group_sync(grp, G);
      if (summer)
        for (int o = 0; o < G; o += 32) wsum += s_w[gbase + o + lane];
      if (rd + 1 < rounds) xf_group_sync(grp, G);  // s_w is read before the next round writes it
    }

    if (summer) {
      const float wx = xf_warp_sum(wsum);
      const float pctr = xf_sigmoid(wx);
      if (lane == 0 && pctr_out) pctr_out[row] = pctr;  // training: only for progressive validation
      if (mode == 0) {
        float loss = __fsub_rn(pctr, (float)label);  // lr_worker.cc:141
        if (lane == 0 && loss_out) loss_out[row] = loss;
        if (WEIGHT) loss = __fmul_rn(__ldg(wv.e + row), loss);  // read again: not kept live through phase A
        abs_acc += fabsf(loss);
        // s_lf is written only by a row with tokens, i.e. after that row's first group barrier, which no thread of the
        // group reaches before it has read s_lf for the previous row.  An empty row (no round, no barrier before this
        // point) deposits nothing, so it neither writes s_lf nor reads it.
        if (lane == 0 && rounds > 0) s_lf[grp] = xf_fix_of(loss, fix_shift);
      }
    }
    xf_group_sync(grp, G);  // s_lf is written and s_w read before the group goes on
    if (mode == 1 || rounds == 0) continue;
    // ---------------- phase B: one deposit per distinct key of a token group: count x residual, integer, exact
    const long long lf = s_lf[grp];
    // the CAS is sent before its answer is looked at, so that the row's CASes are in flight together
    if (lead_s != XF_NO_SLOT) {
      uint8_t* rowp = xf_row(t, lead_s);
      const long long fix = lf * (long long)cnt;
      uint64_t o2, o3;
      bool stale = false;
      const bool issued = xf_lazy_deposit_issue(rowp, lq2, lq3, lq2n, seq, fix, o2, o3);
      if (issued && xf_lazy_deposit_resolve(rowp, true, lq2, lq3, o2, o3, seq, fix, &stale)) {
        if (lmark) *reinterpret_cast<uint32_t*>(rowp + 12) = xf_lazy_open_check(lq2, seq);  // xf_lazy_mark_open
        ++open_acc;
        if (STAMP) sv.stamp[lead_s] = sv.now;
      }
      if (stale) *t.error = 2;  // inside a batch a row only ever goes from "pending" to "open for seq"
    }
    for (int rd = 1; rd < rounds; ++rd) {
      // long rows (> G tokens): the rows were opened in phase A
      const uint32_t j = beg + ((uint32_t)rd << gshift) + (uint32_t)x;
      XfHead h;
      if (j < end) { const int64_t r = xf_probe<false>(t, __ldg(keys + j), &h); if (r >= 0) xf_lazy_add(xf_row(t, (uint64_t)r), lf); }
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
template <bool A, bool S, bool W, bool G>
static int xf_lazy_ctas_per_sm() {
  static const int n = [] {
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, xf_k_step_lr_lazy<A, S, W, G>, 256, 0) != cudaSuccess || v < 1) {
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
  // a group of 128 threads per row, or of 64 when the rows average at most 64 tokens, so that most threads have a token.
  // Tokens past the group's size take the long-row path (an empty deposit in phase A, then a second look and an integer
  // add per token in phase B): the same table, more requests.  So in a batch of 64-thread groups, tokens 64..127 of its
  // longer rows cost those requests where 128-thread groups would deposit them with their row's first round.
  const int gshift = nnz <= 64ull * (uint64_t)B ? 6 : 7;
#define XF_LAZY_ARGS t, row_ptr, keys, labels, B, mode, seq, rows_by_seq, fs, gshift, loss_out, pctr_out, abs_loss_sum, unique_total, a, sv, wv
  // a grid of the CTAs that fit on the GPU at once (or fewer, for a small batch): each group strides over the rows
#define XF_LAZY_LAUNCH(A, S, W, G)                                                                                   \
  xf_k_step_lr_lazy<A, S, W, G>                                                                                       \
      <<<xf_grid_for((uint64_t)B << gshift, 256, xf_lazy_ctas_per_sm<A, S, W, G>()), 256, 0, st>>>(XF_LAZY_ARGS)
  // AdaGrad tables run instances of their own (xf_lazy_fold_t)
#define XF_LAZY_LAUNCH_W(A, S)                        \
  do {                                                \
    if (t.opt == XF_OPT_ADAGRAD) {                    \
      if (wv.e) XF_LAZY_LAUNCH(A, S, true, true);     \
      else XF_LAZY_LAUNCH(A, S, false, true);         \
    } else {                                          \
      if (wv.e) XF_LAZY_LAUNCH(A, S, true, false);    \
      else XF_LAZY_LAUNCH(A, S, false, false);        \
    }                                                 \
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

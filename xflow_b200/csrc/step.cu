// The fused worker step (sm_90a): what LRWorker::update / FMWorker::update do between reading a
// slice and returning from the last Push (src/model/lr/lr_worker.cc:121-177, fm/fm_worker.cc:126-245)
// WITHOUT the reference's sort / unique / merge-join: the table row is the per-key accumulator.
//
//   CSR slice -> probe/insert every token's key (Pull semantics: missing keys are created; with a feature-admission
//                policy only the keys it admits, admit.cu)
//             -> w (and for FM the latent row reduced to sum_k v, sum_k v^2) from the row just found
//             -> per-row warp-segmented sums -> clamped sigmoid -> residual  (calculate_loss)
//             -> every token adds its contribution to its key's gradient accumulators with L2
//                atomics on the 32-byte sector it has just loaded                (calculate_gradient)
//             -> the token that finds the "untouched" marker (-0.0) in g records the slot at its own
//                position of the per-token `touched` array (no shared counter: a single contended
//                append counter was measured to serialise the whole kernel); the optimizer kernel
//                (kernels.cu) walks that array                                                (Push)
//
// One warp per row, one lane per token, two tokens per lane in flight: keys for a 64-token chunk are
// loaded first, then the two first-probe sectors (xf_load_head), then resolved; the two
// returning atomics of phase B are likewise issued back to back.  HBM / L2-latency bound integer and
// float work on random sectors: no shared-memory tile, no tensor core — see DESIGN.md.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "kernels.h"
#include "table.cuh"

#define XF_NO_SLOT 0xFFFFFFFFu
#define XF_CACHED_CHUNKS 2  // 64-token chunks whose slots stay in registers (rows <= 128 tokens)

// Hot-key cache (FM only): with skewed ids a handful of keys take a large share of all tokens (Zipf
// 1.05 over 1e8 ids: the top key is ~8 % of the tokens of every batch) and their L2 atomics serialise
// the whole kernel (17 contended atomics per token on a cfg5-shaped batch).  Each CTA
// therefore keeps NC direct-mapped accumulator rows in shared memory, claimed first-come with a CAS on
// the tag; a token whose key owns (or obtains) an entry accumulates there with shared-memory atomics,
// everything else goes to HBM as before.  The entries are flushed once, when the CTA has finished all
// its rows: 3 global atomics per entry and CTA instead of one set per token.  Sums are unchanged (same
// terms, different association).  touched[] gets gridDim.x * NC extra positions for the flush.
// Per (group of) token(s) the step adds three doubles to the key: G (the w-gradient), L = loss and
// Aq = loss * S (the factorised latent gradient, table.cuh); loss * S is exact in double.
//   mode: 0 = train, 1 = predict (forward only; the Pull still inserts missing keys, lr_worker.cc:47)
// ADMIT: absent keys are inserted only if the admission policy `adm` admits them (xf_probe_from); a rejected token
// adds nothing to its row's sums and never reaches the hot-key cache or touched[] (its slot stays XF_NO_SLOT).
// STAMP (feature eviction): a key this kernel inserts is stamped with sv.now; the training step's other keys
// are stamped by the optimizer pass over touched[] (xf_k_update).
// WEIGHT (importance weighting, weight.cu; training only): a row with wv.e[row] = 0 is skipped before phase A (no probe,
// no insert, no admission; its touched[] positions get XF_NO_SLOT, loss_out 0); every other row accumulates the weighted
// residual e x (pctr - label) in G, L and Aq.  xf_k_update still divides by the batch's row count.
template <bool FM, int VEC, bool ADMIT, bool STAMP, bool WEIGHT>
__global__ void __launch_bounds__(256)
xf_k_step(XfTableView t, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
          const uint8_t* __restrict__ labels, int B, int mode, uint32_t* __restrict__ touched,
          float* __restrict__ loss_out, float* __restrict__ pctr_out, float* __restrict__ abs_loss_sum,
          int log2nc, uint32_t touched_base, XfAdmitView adm, XfStampView sv, XfWeightView wv) {
  __shared__ float s_abs[8];
  extern __shared__ __align__(16) unsigned char xf_smem[];
  float abs_acc = 0.f;
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * warps_per_block;
  const int K = t.K;
  // hot-key cache layout: double acc[NC][3] = {G, L, Aq} | uint32 tag[NC]
  const int NC = (FM && log2nc >= 0) ? (1 << log2nc) : 0;
  double* c_acc = reinterpret_cast<double*>(xf_smem);
  uint32_t* c_tag = reinterpret_cast<uint32_t*>(xf_smem + (size_t)NC * 24);
  if (NC) {
    for (int e = threadIdx.x; e < NC; e += blockDim.x) c_tag[e] = XF_NO_SLOT;
    for (int e = threadIdx.x; e < NC * 3; e += blockDim.x) c_acc[e] = 0.0;
    __syncthreads();
  }

  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    if (WEIGHT && __ldg(wv.e + row) == 0.f) {
      if (lane == 0 && loss_out) loss_out[row] = 0.f;
      for (uint32_t j = beg + (uint32_t)lane; j < end; j += 32u) __stcs(touched + j, XF_NO_SLOT);
      continue;
    }
    const int chunks = (int)((end - beg + 63u) >> 6);

    float wsum = 0.f, ssum = 0.f, qsum = 0.f;
    uint32_t slot_c[2 * XF_CACHED_CHUNKS];
#pragma unroll
    for (int c = 0; c < 2 * XF_CACHED_CHUNKS; ++c) slot_c[c] = XF_NO_SLOT;

    // ---------------- phase A: pull + per-token terms
    for (int ch = 0; ch < chunks; ++ch) {
      const uint32_t j0 = beg + (uint32_t)ch * 64u + (uint32_t)lane;
      const uint32_t j1 = j0 + 32u;
      const bool v0 = j0 < end, v1 = j1 < end;
      const uint64_t k0 = v0 ? __ldcs(keys + j0) : 0ull;  // streaming: do not displace table sectors in L2
      const uint64_t k1 = v1 ? __ldcs(keys + j1) : 0ull;
      const uint64_t p0 = xf_home_slot(t, k0), p1 = xf_home_slot(t, k1);
      XfHead h0, h1;
      h0.key = h1.key = XF_EMPTY_KEY;
      if (v0) h0 = FM ? xf_load_head_l1(xf_row(t, p0)) : xf_load_head(xf_row(t, p0));
      if (v1) h1 = FM ? xf_load_head_l1(xf_row(t, p1)) : xf_load_head(xf_row(t, p1));
      uint32_t s0 = XF_NO_SLOT, s1 = XF_NO_SLOT;
      bool r0 = false, r1 = false;
      if (v0) {
        const int64_t r = xf_probe_from<true, ADMIT, STAMP>(t, k0, p0, h0, &adm, &r0, &sv);
        if (r >= 0) { s0 = (uint32_t)r; wsum += h0.w; }
      }
      if (v1) {
        const int64_t r = xf_probe_from<true, ADMIT, STAMP>(t, k1, p1, h1, &adm, &r1, &sv);
        if (r >= 0) { s1 = (uint32_t)r; wsum += h1.w; }
      }
      if (ADMIT) xf_admit_append(adm, r0, k0, r1, k1);
      if (FM) {
        float st, qt;
        if (s0 != XF_NO_SLOT) { xf_fm_token<VEC>(t, s0, h0.flags, k0, st, qt); ssum += st; qsum += qt; }
        if (s1 != XF_NO_SLOT) { xf_fm_token<VEC>(t, s1, h1.flags, k1, st, qt); ssum += st; qsum += qt; }
      }
#pragma unroll
      for (int c = 0; c < XF_CACHED_CHUNKS; ++c)
        if (ch == c) { slot_c[2 * c] = s0; slot_c[2 * c + 1] = s1; }
    }

    // ---------------- per-row reduction, sigmoid, residual
    const float wx = xf_warp_sum(wsum);
    float S = 0.f, arg = wx;
    if (FM) {
      S = xf_warp_sum(ssum);
      const float Q = xf_warp_sum(qsum);
      const float v_y = __fsub_rn(__fmul_rn(S, S), Q);  // fm_worker.cc:193-196: no 1/2, collapsed over k
      arg = __fadd_rn(wx, v_y);
    }
    const float pctr = xf_sigmoid(arg);
    if (lane == 0 && pctr_out) pctr_out[row] = pctr;  // training: only for progressive validation
    if (mode == 1) continue;
    float loss = __fsub_rn(pctr, (float)labels[row]);  // lr_worker.cc:141 ; fm_worker.cc:200
    if (lane == 0 && loss_out) loss_out[row] = loss;
    if (WEIGHT) loss = __fmul_rn(__ldg(wv.e + row), loss);
    abs_acc += fabsf(loss);

    // ---------------- phase B: per-key gradient accumulation (the Push payload)
    float gw_c = loss;
    if (FM) {
      // fm_worker.cc:140 accumulates the w-gradient inside the k loop: K sequential float adds
      gw_c = 0.f;
      for (int k = 0; k < K; ++k) gw_c += loss;
    }
    const double gw_d = (double)gw_c;
    for (int ch = 0; ch < chunks; ++ch) {
      const uint32_t j0 = beg + (uint32_t)ch * 64u + (uint32_t)lane;
      const uint32_t j1 = j0 + 32u;
      uint32_t s0 = XF_NO_SLOT, s1 = XF_NO_SLOT;
      if (ch < XF_CACHED_CHUNKS) {
#pragma unroll
        for (int c = 0; c < XF_CACHED_CHUNKS; ++c)
          if (ch == c) { s0 = slot_c[2 * c]; s1 = slot_c[2 * c + 1]; }
      } else {
        XfHead h;
        if (j0 < end) { const int64_t r = xf_probe<false>(t, __ldg(keys + j0), &h); if (r >= 0) s0 = (uint32_t)r; }
        if (j1 < end) { const int64_t r = xf_probe<false>(t, __ldg(keys + j1), &h); if (r >= 0) s1 = (uint32_t)r; }
      }
      // Tokens of this row that hit the same key contribute identical terms (same residual, same S,
      // same v): the lowest lane of each group adds count x term, the others add nothing.  Cuts the
      // atomics on hot keys (Zipf ids: the top key is ~8 % of all tokens) without changing the sums.
      const unsigned g0 = __match_any_sync(0xffffffffu, (s0 != XF_NO_SLOT) ? s0 : (0xFFFFFF00u | (uint32_t)lane));
      const unsigned g1 = __match_any_sync(0xffffffffu, (s1 != XF_NO_SLOT) ? s1 : (0xFFFFFF00u | (uint32_t)lane));
      const bool lead0 = s0 != XF_NO_SLOT && lane == __ffs(g0) - 1;
      const bool lead1 = s1 != XF_NO_SLOT && lane == __ffs(g1) - 1;
      const double c0 = (double)__popc(g0), c1 = (double)__popc(g1);
      const double ld = (double)loss, ad = (double)loss * (double)S;  // exact products
      double old0 = 0.0, old1 = 0.0;
      bool cached0 = false, cached1 = false;
      if (NC) {
        // try the CTA's hot-key cache first (claim an empty entry or find our own)
        if (lead0) {
          const uint32_t e = (s0 * 2654435761u) >> (32 - log2nc);
          const uint32_t prev = atomicCAS(c_tag + e, XF_NO_SLOT, s0);
          if (prev == XF_NO_SLOT || prev == s0) {
            cached0 = true;
            atomicAdd(c_acc + 3 * e, gw_d * c0);
            atomicAdd(c_acc + 3 * e + 1, ld * c0);
            atomicAdd(c_acc + 3 * e + 2, ad * c0);
          }
        }
        if (lead1) {
          const uint32_t e = (s1 * 2654435761u) >> (32 - log2nc);
          const uint32_t prev = atomicCAS(c_tag + e, XF_NO_SLOT, s1);
          if (prev == XF_NO_SLOT || prev == s1) {
            cached1 = true;
            atomicAdd(c_acc + 3 * e, gw_d * c1);
            atomicAdd(c_acc + 3 * e + 1, ld * c1);
            atomicAdd(c_acc + 3 * e + 2, ad * c1);
          }
        }
      }
      if (lead0 && !cached0) old0 = atomicAdd(xf_row_g(xf_row(t, s0)), gw_d * c0);
      if (lead1 && !cached1) old1 = atomicAdd(xf_row_g(xf_row(t, s1)), gw_d * c1);
      if (FM) {
        if (lead0 && !cached0) { double* a = xf_row_acc(xf_row(t, s0), K); atomicAdd(a, ld * c0); atomicAdd(a + 1, ad * c0); }
        if (lead1 && !cached1) { double* a = xf_row_acc(xf_row(t, s1), K); atomicAdd(a, ld * c1); atomicAdd(a + 1, ad * c1); }
      }
      const bool f0 = lead0 && !cached0 && (unsigned long long)__double_as_longlong(old0) == XF_NEG_ZERO_BITS64;
      const bool f1 = lead1 && !cached1 && (unsigned long long)__double_as_longlong(old1) == XF_NEG_ZERO_BITS64;
      if (j0 < end) __stcs(touched + j0, f0 ? s0 : XF_NO_SLOT);
      if (j1 < end) __stcs(touched + j1, f1 ? s1 : XF_NO_SLOT);
    }
  }
  if (NC && mode == 0) {
    // flush the hot-key cache: one set of global atomics per entry; the flush that finds the untouched
    // marker records the slot in this CTA's extra touched[] positions
    __syncthreads();
    for (int e = threadIdx.x; e < NC; e += blockDim.x) {
      const uint32_t s = c_tag[e];
      uint32_t rec = XF_NO_SLOT;
      if (s != XF_NO_SLOT) {
        uint8_t* rowp = xf_row(t, s);
        const double old = atomicAdd(xf_row_g(rowp), c_acc[3 * e]);
        if ((unsigned long long)__double_as_longlong(old) == XF_NEG_ZERO_BITS64) rec = s;
        double* a = xf_row_acc(rowp, K);
        atomicAdd(a, c_acc[3 * e + 1]);
        atomicAdd(a + 1, c_acc[3 * e + 2]);
      }
      touched[touched_base + (uint32_t)blockIdx.x * (uint32_t)NC + (uint32_t)e] = rec;
    }
  }
  // monitoring scalar: sum over rows of |pctr - label| (one atomic per block)
  if (abs_loss_sum != nullptr && mode == 0) {
    if (lane == 0) s_abs[threadIdx.x >> 5] = abs_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += s_abs[w];
      atomicAdd(abs_loss_sum, tot);
    }
  }
}

int xf_sms();
int xf_grid_for(uint64_t work_items, int block, int blocks_per_sm);

// shared-memory hot-key cache sizing for the FM step: NC entries of 3 doubles + a tag (28 bytes)
#define XF_STEP_CACHE_LOG2 9
int xf_step_cache_log2(int K) {
  if (K <= 0) return -1;
  static const int lg = [] {
    const char* e = getenv("XFLOW_FM_CACHE_LOG2");  // tuning knob; 0..10
    const int v = (e && *e) ? atoi(e) : XF_STEP_CACHE_LOG2;
    return v < 0 ? 0 : (v > 10 ? 10 : v);
  }();
  return lg;
}
// extra touched[] positions the FM step needs beyond nnz (grid x NC)
uint32_t xf_step_touched_extra(int K, int B) {
  const int lg = xf_step_cache_log2(K);
  if (lg < 0) return 0;
  return (uint32_t)xf_grid_for((uint64_t)B * 32, 256, 8) << lg;
}

void xf_launch_step(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* labels,
                    int B, int mode, uint32_t* touched, uint32_t nnz, float* loss_out, float* pctr_out,
                    float* abs_loss_sum, const XfAdmitView* adm, const XfStampView& sv, const XfWeightView& wv,
                    cudaStream_t st) {
  if (B <= 0) return;
  const int block = 256;
  const int grid = xf_grid_for((uint64_t)B * 32, block, 8);
  const int lg = xf_step_cache_log2(t.K);
  const size_t smem = lg >= 0 ? ((size_t)1 << lg) * 28 : 0;
#define XF_STEP_ARGS t, row_ptr, keys, labels, B, mode, touched, loss_out, pctr_out, abs_loss_sum, lg, nnz, a, sv, wv
#define XF_STEP_LAUNCH_W(A, S, W)                                                             \
  if (t.K == 0) {                                                                             \
    xf_k_step<false, 1, A, S, W><<<grid, block, 0, st>>>(XF_STEP_ARGS);                       \
  } else {                                                                                    \
    switch (xf_vec_for(t.K)) {                                                                \
      case 4: xf_k_step<true, 4, A, S, W><<<grid, block, smem, st>>>(XF_STEP_ARGS); break;    \
      case 2: xf_k_step<true, 2, A, S, W><<<grid, block, smem, st>>>(XF_STEP_ARGS); break;    \
      default: xf_k_step<true, 1, A, S, W><<<grid, block, smem, st>>>(XF_STEP_ARGS); break;   \
    }                                                                                         \
  }
#define XF_STEP_LAUNCH(A, S)        \
  if (wv.e) {                       \
    XF_STEP_LAUNCH_W(A, S, true)    \
  } else {                          \
    XF_STEP_LAUNCH_W(A, S, false)   \
  }
  const XfAdmitView a = adm ? *adm : XfAdmitView{};
  const bool stamp = sv.stamp != nullptr;
  if (adm && stamp) {
    XF_STEP_LAUNCH(true, true)
  } else if (adm) {
    XF_STEP_LAUNCH(true, false)
  } else if (stamp) {
    XF_STEP_LAUNCH(false, true)
  } else {
    XF_STEP_LAUNCH(false, false)
  }
#undef XF_STEP_LAUNCH
#undef XF_STEP_LAUNCH_W
#undef XF_STEP_ARGS
}

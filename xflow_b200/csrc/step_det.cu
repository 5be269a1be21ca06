// Deterministic training steps for the canonical FM (step_fmc.cu) and the multi-view machine (step_mvm.cu), the
// kernels of xf_trainer_set_deterministic (include/xflow_b200.h, section 3).  The default steps add every token's
// gradient terms into its key's accumulators with float / f64 atomics, so a key with several tokens in a batch ends up
// with bits that depend on the order the atomics land in (and the machine's forward adds a row's same-field terms with
// shared-memory atomics).  Here each key's terms are summed in one fixed association instead:
//   1. the step kernel runs the forward pass (canonical FM: xf_k_step_fmc's arithmetic, forward.cuh; the machine: its
//      field sums in token order, as the frozen model's predict) and stores, per token, its slot (the sort key), its
//      position and what the reduction needs: the row id (FM; the row's S[K] is stored once per row) or the token's K
//      latent terms (MVM); per row the residual;
//   2. a stable radix sort (CUB, bits [0, log2cap + 1)) orders the (slot, position) pairs: a key's tokens become one
//      segment in token order, the tokens without a slot (probe overflow, 0xFFFFFFFF) sort last and are skipped;
//   3. xf_k_det_reduce walks the sorted array: a segment of one token is added by its own lane, a segment of 2 .. 32
//      tokens by a warp (one run: the xor butterfly of the header's contract, lanes holding -0.0 past the run), and a
//      longer segment is queued; xf_k_det_runs sums the queued segments' runs of 32, one warp per run, and
//      xf_k_det_fold adds each queued segment's run sums in order onto the row.  One writer per key: plain stores.
//      touched[] gets the slot at each segment's head and 0xFFFFFFFF elsewhere;
//   4. the optimizer pass xf_k_update (kernels.cu) then runs unchanged.
// xf_k_det_abs sums the rows' |residual| in an order fixed by the row count (the step's mean_abs_loss).
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/cub.cuh>

#include "forward.cuh"
#include "internal.h"

#define XF_NO_SLOT 0xFFFFFFFFu

// the scratch of one deterministic step on the device (XfDetBufs, internal.h)
struct XfDetView {
  uint32_t* keys_in;        // [nnz] slot of token j (sort key)
  uint32_t* toks_in;        // [nnz] j (sort value)
  const uint32_t* keys;     // [nnz] sorted slots
  const uint32_t* toks;     // [nnz] token positions in sorted order
  uint32_t* tok_row;        // FM: [nnz] the token's row
  float* row_s;             // FM: [rows][K] the row's S_k
  float* res;               // [rows] residual pctr - label
  float* terms;             // MVM: [nnz][K] the token's terms r x o_k
  float* run_a;             // queued segments: [runs][K] run sums of A
  double* run_d;            // queued segments: [runs][2] run sums of G and L2
  uint4* longs;             // queued segments: {first position, end position, first run, 0}
  uint32_t* rdesc;          // [runs] the queued segment of each run
  unsigned* cnt;            // {queued segments, runs}
  const float* vals;        // [nnz] feature values, or NULL (all 1)
};

// ---------------------------------------------------------------------------------------------------------------
// 1. step kernels
// ---------------------------------------------------------------------------------------------------------------
// The canonical FM: xf_k_step_fmc's mapping and forward arithmetic (one warp per row, C = K/4 lanes per token), then
// S[K] and the residual of the row and (slot, j, row) of each token.  Training only: predict runs xf_k_step_fmc.
template <int C>
__global__ void __launch_bounds__(256)
xf_k_det_fmc(XfTableView t, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
             const float* __restrict__ vals, const uint8_t* __restrict__ labels, int B, XfDetView d,
             float* __restrict__ loss_out, float* __restrict__ pctr_out) {
  constexpr int K = 4 * C;
  constexpr int T = 32 / C;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int gwarp = blockIdx.x * wpb + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * wpb;
  const int c = lane & (C - 1);
  const int tg = lane / C;
  const int lead = lane & ~(C - 1);
  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row), end = __ldg(row_ptr + row + 1);
    float S[4] = {0.f, 0.f, 0.f, 0.f};
    float Q = 0.f, wx = 0.f;
    for (uint32_t j0 = beg; j0 < end; j0 += (uint32_t)T) {
      const uint32_t j = j0 + (uint32_t)tg;
      const bool live = j < end;
      uint32_t slot = XF_NO_SLOT, flags = 0;
      uint64_t key = 0;
      float w = 0.f;
      if (live && c == 0) {
        key = __ldcs(keys + j);
        XfHead h;
        const int64_t r = xf_probe<true>(t, key, &h);
        if (r >= 0) { slot = (uint32_t)r; flags = h.flags; w = h.w; }
        d.keys_in[j] = slot;
        d.toks_in[j] = j;
        d.tok_row[j] = (uint32_t)row;
      }
      slot = __shfl_sync(0xffffffffu, slot, lead);
      flags = __shfl_sync(0xffffffffu, flags, lead);
      key = __shfl_sync(0xffffffffu, (unsigned long long)key, lead);
      if (!live || slot == XF_NO_SLOT) continue;
      const float x = vals ? __ldg(vals + j) : 1.0f;
      float4 v;
      if (flags & XF_FLAG_V_READY) v = __ldcg(reinterpret_cast<const float4*>(xf_row(t, slot) + 32) + c);
      else v = xf_v_init_piece(t, key, c);
      xf_fmc_add(v, x, w, c == 0, S, Q, wx);
    }
    const float pctr = xf_sigmoid(xf_fmc_arg(C, S, Q, wx));
    const float loss = __fsub_rn(pctr, (float)labels[row]);
    if (lane == 0) {
      d.res[row] = loss;
      if (pctr_out) pctr_out[row] = pctr;
      if (loss_out) loss_out[row] = loss;
    }
    if (tg == 0) reinterpret_cast<float4*>(d.row_s + (size_t)row * K)[c] = make_float4(S[0], S[1], S[2], S[3]);
  }
}

// The multi-view machine: the frozen model's forward (header section 6: field sums in token order from +0, P_k over
// the present fields ascending, y by xor 16 .. 1), on the table's rows with insert as xf_k_step_mvm; training then
// stores each token's terms r x o_k, o_k the product of the other present fields' sums in ascending order.
template <int C>
__global__ void __launch_bounds__(256)
xf_k_det_mvm(XfTableView t, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
             const uint8_t* __restrict__ fields, const float* __restrict__ vals, const uint8_t* __restrict__ labels,
             int B, int mode, XfDetView d, float* __restrict__ loss_out, float* __restrict__ pctr_out) {
  constexpr int K = 4 * C;
  constexpr int T = 32 / C;
  __shared__ __align__(16) float s_sum[8][XF_MVM_FIELDS][K];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const int gwarp = blockIdx.x * wpb + wib;
  const int nwarps = gridDim.x * wpb;
  const int c = lane & (C - 1);
  const int tg = lane / C;
  const int lead = lane & ~(C - 1);
  float (*S)[K] = s_sum[wib];
  if (lane < K)
    for (int f = 0; f < XF_MVM_FIELDS; ++f) S[f][lane] = 0.f;
  __syncwarp();
  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row), end = __ldg(row_ptr + row + 1);
    unsigned present = 0u;
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
        if (mode == 0) {
          d.keys_in[j] = slot;
          d.toks_in[j] = j;
        }
      }
      slot = __shfl_sync(0xffffffffu, slot, lead);
      flags = __shfl_sync(0xffffffffu, flags, lead);
      f = __shfl_sync(0xffffffffu, f, lead);
      key = __shfl_sync(0xffffffffu, (unsigned long long)key, lead);
      const bool on = live && slot != XF_NO_SLOT;  // as xf_k_step_mvm: a token without a row is skipped
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      float x = 1.0f;
      if (on) {
        if (vals) x = __ldg(vals + j);
        if (flags & XF_FLAG_V_READY) v = __ldcg(reinterpret_cast<const float4*>(xf_row(t, slot) + 32) + c);
        else v = xf_v_init_piece(t, key, c);
        present |= 1u << f;
      }
      xf_mvm_add<K>(S, on, f, c, v, x);
    }
    present = __reduce_or_sync(0xffffffffu, present);
    const float pctr = xf_sigmoid(xf_warp_sum(xf_mvm_product<K>(S, present)));
    if (lane == 0 && pctr_out) pctr_out[row] = pctr;
    if (mode == 0) {
      const float loss = __fsub_rn(pctr, (float)labels[row]);
      if (lane == 0) {
        d.res[row] = loss;
        if (loss_out) loss_out[row] = loss;
      }
      for (uint32_t j0 = beg; j0 < end; j0 += (uint32_t)T) {
        const uint32_t j = j0 + (uint32_t)tg;
        const bool live = j < end;
        uint32_t slot = XF_NO_SLOT, f = 0;
        if (live && c == 0) {
          slot = d.keys_in[j];
          f = (uint32_t)__ldg(fields + j) & (XF_MVM_FIELDS - 1);
        }
        slot = __shfl_sync(0xffffffffu, slot, lead);
        f = __shfl_sync(0xffffffffu, f, lead);
        if (!live || slot == XF_NO_SLOT) continue;
        const float x = vals ? __ldg(vals + j) : 1.0f;
        float o0 = 1.f, o1 = 1.f, o2 = 1.f, o3 = 1.f;  // products over the OTHER present fields, ascending
        for (unsigned m = present & ~(1u << f); m; m &= m - 1) {
          const float* sf = S[__ffs(m) - 1] + 4 * c;
          o0 = __fmul_rn(o0, sf[0]); o1 = __fmul_rn(o1, sf[1]); o2 = __fmul_rn(o2, sf[2]); o3 = __fmul_rn(o3, sf[3]);
        }
        const float rx = __fmul_rn(loss, x);
        reinterpret_cast<float4*>(d.terms + (size_t)j * K)[c] =
            make_float4(__fmul_rn(rx, o0), __fmul_rn(rx, o1), __fmul_rn(rx, o2), __fmul_rn(rx, o3));
      }
    }
    __syncwarp();  // every lane has read the sums
    if (lane < K)
      for (unsigned q = present; q; q &= q - 1) S[__ffs(q) - 1][lane] = 0.f;
    __syncwarp();  // the sums are clear before the warp's next row adds to them
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 2. the per-key sums
// ---------------------------------------------------------------------------------------------------------------
// One run: sorted positions [a, a + m), 1 <= m <= 32, summed by the xor butterfly: lane i holds term i (-0.0 for
// i >= m) and adds lane i ^ o's value to its own for o = 16, 8, 4, 2, 1; lane 0's value is the run's sum.  G and L
// (f64, lane 0) are returned; lane 0 stores A[k] into out[k] (add: out[k] + A[k]).
template <bool MVM, int K>
__device__ __forceinline__ void xf_det_run(const XfDetView& d, uint32_t a, int m, float* out, bool add, double& G,
                                           double& L) {
  const int lane = threadIdx.x & 31;
  const bool on = lane < m;
  uint32_t tok = 0, row = 0;
  float rx = 0.f;
  double g = -0.0, l = -0.0;
  if (on) {
    tok = __ldcg(d.toks + a + lane);
    if (MVM) {
      g = 0.0;  // the machine's w-gradient term
    } else {
      row = __ldcg(d.tok_row + tok);
      const float r = __ldcg(d.res + row);
      const float x = d.vals ? __ldg(d.vals + tok) : 1.0f;
      rx = __fmul_rn(r, x);
      g = __dmul_rn((double)r, (double)x);
      l = __dmul_rn(g, (double)x);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    g = __dadd_rn(g, __shfl_xor_sync(0xffffffffu, g, o));
    if (!MVM) l = __dadd_rn(l, __shfl_xor_sync(0xffffffffu, l, o));
  }
  G = g;
  L = l;
  for (int q = 0; q < K / 4; ++q) {
    float4 v = make_float4(-0.f, -0.f, -0.f, -0.f);
    if (on) {
      if (MVM) {
        v = __ldcg(reinterpret_cast<const float4*>(d.terms + (size_t)tok * K) + q);
      } else {
        const float4 sk = __ldcg(reinterpret_cast<const float4*>(d.row_s + (size_t)row * K) + q);
        v = make_float4(__fmul_rn(rx, sk.x), __fmul_rn(rx, sk.y), __fmul_rn(rx, sk.z), __fmul_rn(rx, sk.w));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      v.x = __fadd_rn(v.x, __shfl_xor_sync(0xffffffffu, v.x, o));
      v.y = __fadd_rn(v.y, __shfl_xor_sync(0xffffffffu, v.y, o));
      v.z = __fadd_rn(v.z, __shfl_xor_sync(0xffffffffu, v.z, o));
      v.w = __fadd_rn(v.w, __shfl_xor_sync(0xffffffffu, v.w, o));
    }
    if (lane == 0) {
      float4* p = reinterpret_cast<float4*>(out) + q;
      if (add) {
        const float4 c = *p;
        v = make_float4(__fadd_rn(c.x, v.x), __fadd_rn(c.y, v.y), __fadd_rn(c.z, v.z), __fadd_rn(c.w, v.w));
      }
      *p = v;
    }
  }
}

// One warp per 32 sorted positions.  touched[i] = the slot at a segment's head, else 0xFFFFFFFF.  A one-token
// segment is added by its lane (the butterfly of one term and 31 times -0.0 is the term); longer segments, one at a
// time by the warp: the end is found by a 32-ary search, a segment of at most 32 tokens is one run added onto the
// row, a longer one is queued for xf_k_det_runs / xf_k_det_fold with its runs.
template <bool MVM, int K>
__global__ void __launch_bounds__(256)
xf_k_det_reduce(XfTableView t, XfDetView d, uint32_t n, uint32_t* __restrict__ touched) {
  const int lane = threadIdx.x & 31;
  const uint64_t gwarp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t base = gwarp * 32; base < n; base += nwarps * 32) {
    const uint64_t i = base + (uint64_t)lane;
    const uint32_t s = i < n ? __ldcg(d.keys + i) : XF_NO_SLOT;
    const uint32_t prev = (i < n && i > 0) ? __ldcg(d.keys + i - 1) : XF_NO_SLOT;
    const uint32_t next = i + 1 < n ? __ldcg(d.keys + i + 1) : XF_NO_SLOT;
    const bool head = s != XF_NO_SLOT && (i == 0 || prev != s);
    if (i < n) touched[i] = head ? s : XF_NO_SLOT;
    if (head && next != s) {
      // a key with one token: its terms added to the row's accumulators as they are
      const uint32_t tok = __ldcg(d.toks + i);
      uint8_t* rowp = xf_row(t, s);
      float4* ca = reinterpret_cast<float4*>(xf_row_ca(t, rowp));
      if (MVM) {
        const float4* tp = reinterpret_cast<const float4*>(d.terms + (size_t)tok * K);
        for (int q = 0; q < K / 4; ++q) {
          const float4 a = ca[q], b = __ldcg(tp + q);
          ca[q] = make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
        }
        *xf_row_g(rowp) = __dadd_rn(*xf_row_g(rowp), 0.0);
      } else {
        const uint32_t row = __ldcg(d.tok_row + tok);
        const float r = __ldcg(d.res + row);
        const float x = d.vals ? __ldg(d.vals + tok) : 1.0f;
        const float rx = __fmul_rn(r, x);
        const float4* sp = reinterpret_cast<const float4*>(d.row_s + (size_t)row * K);
        for (int q = 0; q < K / 4; ++q) {
          const float4 a = ca[q], b = __ldcg(sp + q);
          ca[q] = make_float4(__fadd_rn(a.x, __fmul_rn(rx, b.x)), __fadd_rn(a.y, __fmul_rn(rx, b.y)),
                              __fadd_rn(a.z, __fmul_rn(rx, b.z)), __fadd_rn(a.w, __fmul_rn(rx, b.w)));
        }
        const double gt = __dmul_rn((double)r, (double)x);
        *xf_row_g(rowp) = __dadd_rn(*xf_row_g(rowp), gt);
        double* acc = xf_row_acc(rowp, K);
        *acc = __dadd_rn(*acc, __dmul_rn(gt, (double)x));
      }
    }
    unsigned multi = __ballot_sync(0xffffffffu, head && next == s);
    while (multi) {
      const int src = __ffs(multi) - 1;
      multi &= multi - 1;
      const uint32_t h = (uint32_t)(base + (uint64_t)src);
      const uint32_t sl = __shfl_sync(0xffffffffu, s, src);
      // lo: the last position known to hold sl; the end lies in (lo, lo + 32 step]
      uint32_t lo = h, step = 1;
      for (;;) {
        const uint64_t p = (uint64_t)lo + (uint64_t)(lane + 1) * step;
        const bool in = p < n && __ldcg(d.keys + p) == sl;
        const int cnt = __popc(__ballot_sync(0xffffffffu, in));
        lo += (uint32_t)cnt * step;
        if (cnt == 32) step <<= 5;
        else if (step == 1) break;
        else step >>= 5;
      }
      const uint32_t len = lo + 1 - h;
      if (len <= 32) {
        double G, L;
        uint8_t* rowp = xf_row(t, sl);
        xf_det_run<MVM, K>(d, h, (int)len, xf_row_ca(t, rowp), true, G, L);
        if (lane == 0) {
          *xf_row_g(rowp) = __dadd_rn(*xf_row_g(rowp), G);
          if (!MVM) {
            double* acc = xf_row_acc(rowp, K);
            *acc = __dadd_rn(*acc, L);
          }
        }
      } else {
        const uint32_t nr = (len + 31) / 32;
        uint32_t li = 0, rb = 0;
        if (lane == 0) {
          li = atomicAdd(d.cnt, 1u);
          rb = atomicAdd(d.cnt + 1, nr);
          d.longs[li] = make_uint4(h, h + len, rb, 0u);
        }
        li = __shfl_sync(0xffffffffu, li, 0);
        rb = __shfl_sync(0xffffffffu, rb, 0);
        for (uint32_t q = (uint32_t)lane; q < nr; q += 32) d.rdesc[rb + q] = li;
      }
    }
  }
}

// The runs of the queued segments, one warp per run: its sums into run_a / run_d
template <bool MVM, int K>
__global__ void __launch_bounds__(256) xf_k_det_runs(XfDetView d) {
  const int lane = threadIdx.x & 31;
  const uint32_t runs = d.cnt[1];
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < runs; r += nwarps) {
    const uint4 seg = d.longs[d.rdesc[r]];
    const uint32_t a = seg.x + 32u * (r - seg.z);
    const int m = (int)min(32u, seg.y - a);
    double G, L;
    xf_det_run<MVM, K>(d, a, m, d.run_a + (size_t)r * K, false, G, L);
    if (lane == 0) reinterpret_cast<double2*>(d.run_d)[r] = make_double2(G, L);
  }
}

// Each queued segment's run sums added in order onto its row, one warp per segment (lane: coordinates; lanes 0 and 1:
// G and L2)
template <bool MVM, int K>
__global__ void __launch_bounds__(256) xf_k_det_fold(XfTableView t, XfDetView d) {
  const int lane = threadIdx.x & 31;
  const uint32_t segs = d.cnt[0];
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t li = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; li < segs; li += nwarps) {
    const uint4 seg = d.longs[li];
    const uint32_t nr = (seg.y - seg.x + 31) / 32;
    uint8_t* rowp = xf_row(t, __ldcg(d.keys + seg.x));
    float* ca = xf_row_ca(t, rowp);
    for (int k = lane; k < K; k += 32) {
      float acc = ca[k];
#pragma unroll 8
      for (uint32_t q = 0; q < nr; ++q) acc = __fadd_rn(acc, __ldcg(d.run_a + (size_t)(seg.z + q) * K + k));
      ca[k] = acc;
    }
    if (lane < (MVM ? 1 : 2)) {
      double* dst = lane == 0 ? xf_row_g(rowp) : xf_row_acc(rowp, K);
      double acc = *dst;
#pragma unroll 8
      for (uint32_t q = 0; q < nr; ++q) acc = __dadd_rn(acc, __ldcg(d.run_d + 2 * (size_t)(seg.z + q) + lane));
      *dst = acc;
    }
  }
}

// sum over the rows of |residual|: thread t of 256 adds rows t, t + 256, ... in order from +0, then s[i] += s[i + o]
// for o = 128, 64, .., 1; the result is stored (the step's abs-loss word)
__global__ void __launch_bounds__(256) xf_k_det_abs(const float* __restrict__ res, int B, float* __restrict__ out) {
  __shared__ float s[256];
  float a = 0.f;
  for (int r = threadIdx.x; r < B; r += 256) a = __fadd_rn(a, fabsf(res[r]));
  s[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s[threadIdx.x] = __fadd_rn(s[threadIdx.x], s[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = s[0];
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// Kernels CUB's DeviceRadixSort::SortPairs launches on sm_90 for n pairs of 32-bit keys and values over `bits` bits
// (cub/device/dispatch/dispatch_radix_sort.cuh with Policy900): one single-tile kernel up to 256 x 19 items; else the
// onesweep path: a histogram kernel, an exclusive-sum kernel and one kernel per 8-bit pass and portion of at most
// ~2^28 items (384 x 23 per tile).
static uint64_t xf_det_sort_launches(uint64_t n, int bits) {
  if (n == 0) return 0;
  if (n <= 256u * 19u) return 1;
  const uint64_t tile = 384u * 23u;
  const uint64_t portion = ((1u << 28) - 1) / tile * tile;
  const uint64_t portions = (n + portion - 1) / portion;
  return 2 + portions * (uint64_t)((bits + 7) / 8);
}

uint64_t xf_det_extra_launches(uint32_t nnz, uint32_t log2cap, bool abs_sum) {
  return (nnz ? xf_det_sort_launches(nnz, (int)log2cap + 1) + 3 : 0) + (abs_sum ? 1 : 0);
}

static size_t xf_det_sort_bytes(uint32_t n) {
  size_t tb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)n, 0, 32);
  return tb;
}

// queued segments hold >= 33 tokens, so they have at most nnz / 33 + 1 segments and nnz / 32 + nnz / 33 + 1 runs
static uint64_t xf_det_max_segs(uint64_t nnz) { return nnz / 33 + 1; }
static uint64_t xf_det_max_runs(uint64_t nnz) { return nnz / 16 + 1; }

int XfDetBufs::alloc(bool mvm, int K, uint32_t max_rows, uint32_t max_nnz) {
  const size_t n = max_nnz, R = max_rows;
  XF_TRY(keys_in.ensure(n * 4));
  XF_TRY(keys_out.ensure(n * 4));
  XF_TRY(toks_in.ensure(n * 4));
  XF_TRY(toks_out.ensure(n * 4));
  XF_TRY(res.ensure(R * 4));
  if (mvm) {
    XF_TRY(terms.ensure(n * (size_t)K * 4));
  } else {
    XF_TRY(tok_row.ensure(n * 4));
    XF_TRY(row_s.ensure(R * (size_t)K * 4));
  }
  XF_TRY(run_a.ensure(xf_det_max_runs(n) * (size_t)K * 4));
  XF_TRY(run_d.ensure(xf_det_max_runs(n) * 16));
  XF_TRY(rdesc.ensure(xf_det_max_runs(n) * 4));
  XF_TRY(longs.ensure(xf_det_max_segs(n) * 16));
  XF_TRY(cnt.ensure(16));
  XF_TRY(tmp.ensure(std::max<size_t>(xf_det_sort_bytes(max_nnz), 16)));
  return XF_OK;
}

void XfDetBufs::release() {
  for (XfDevBuf* b : {&keys_in, &keys_out, &toks_in, &toks_out, &tok_row, &row_s, &res, &terms, &run_a, &run_d, &longs,
                      &rdesc, &cnt, &tmp})
    b->release();
}

template <bool MVM, int K>
static void xf_det_launch_reduce(const XfTableView& t, const XfDetView& d, uint32_t nnz, uint32_t* touched,
                                 cudaStream_t st) {
  xf_k_det_reduce<MVM, K><<<xf_grid_for(nnz, 256, 8), 256, 0, st>>>(t, d, nnz, touched);
  xf_k_det_runs<MVM, K><<<xf_grid_for(xf_det_max_runs(nnz) * 32, 256, 8), 256, 0, st>>>(d);
  xf_k_det_fold<MVM, K><<<xf_grid_for(xf_det_max_segs(nnz) * 32, 256, 8), 256, 0, st>>>(t, d);
}

int xf_det_step(const XfTableView& t, XfDetBufs& b, bool mvm, const uint32_t* row_ptr, const uint64_t* keys,
                const float* vals, const uint8_t* fields, const uint8_t* labels, uint32_t rows, uint32_t nnz, int mode,
                uint32_t* touched, float* loss_out, float* pctr_out, float* abs_loss_sum, cudaStream_t st) {
  XfDetView d;
  d.keys_in = b.keys_in.as<uint32_t>();
  d.toks_in = b.toks_in.as<uint32_t>();
  d.keys = b.keys_out.as<uint32_t>();
  d.toks = b.toks_out.as<uint32_t>();
  d.tok_row = b.tok_row.as<uint32_t>();
  d.row_s = b.row_s.as<float>();
  d.res = b.res.as<float>();
  d.terms = b.terms.as<float>();
  d.run_a = b.run_a.as<float>();
  d.run_d = b.run_d.as<double>();
  d.longs = b.longs.as<uint4>();
  d.rdesc = b.rdesc.as<uint32_t>();
  d.cnt = b.cnt.as<unsigned>();
  d.vals = vals;
  const int B = (int)rows;
  const int grid = xf_grid_for((uint64_t)B * 32, 256, 8);
  // positions outside the rows (a slice of an ingested block) keep no slot
  if (mode == 0 && nnz) XF_CUDA_TRY(cudaMemsetAsync(d.keys_in, 0xFF, (size_t)nnz * 4, st));
  if (mvm)
    xf_with_lanes<8>(t.K, [&](auto C) {
      xf_k_det_mvm<C><<<grid, 256, 0, st>>>(t, row_ptr, keys, fields, vals, labels, B, mode, d, loss_out, pctr_out);
    });
  else
    xf_with_lanes<32>(t.K, [&](auto C) {
      xf_k_det_fmc<C><<<grid, 256, 0, st>>>(t, row_ptr, keys, vals, labels, B, d, loss_out, pctr_out);
    });
  if (mode != 0) return XF_OK;
  if (nnz) {
    const int bits = (int)t.log2cap + 1;
    size_t tb = 0;
    XF_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, b.keys_in.as<uint32_t>(), b.keys_out.as<uint32_t>(),
                                                b.toks_in.as<uint32_t>(), b.toks_out.as<uint32_t>(), (int)nnz, 0, bits, st));
    XF_TRY(b.tmp.ensure(std::max<size_t>(tb, 16)));
    tb = b.tmp.cap;
    XF_CUDA_TRY(cub::DeviceRadixSort::SortPairs(b.tmp.p, tb, b.keys_in.as<uint32_t>(), b.keys_out.as<uint32_t>(),
                                                b.toks_in.as<uint32_t>(), b.toks_out.as<uint32_t>(), (int)nnz, 0, bits, st));
    XF_CUDA_TRY(cudaMemsetAsync(d.cnt, 0, 2 * sizeof(unsigned), st));
    if (mvm) xf_with_lanes<8>(t.K, [&](auto C) { xf_det_launch_reduce<true, 4 * C>(t, d, nnz, touched, st); });
    else xf_with_lanes<32>(t.K, [&](auto C) { xf_det_launch_reduce<false, 4 * C>(t, d, nnz, touched, st); });
  }
  if (abs_loss_sum) xf_k_det_abs<<<1, 256, 0, st>>>(d.res, B, abs_loss_sum);
  return XF_OK;
}

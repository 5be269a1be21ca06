// sm_90a kernels of the xflow hot path.  All of them are HBM / L2-latency bound integer+float work
// on 32-byte table sectors (see table.cuh); there is no dense tile anywhere on this path (the
// reference's FM term is a per-row scalar, fm_worker.cc:177-196), so no tensor-core code.
//
//   xf_k_fill               table initialisation (EMPTY keys, g = -0.0f)
//   (the fused worker step lives in step.cu / step_lazy.cu)
//   xf_k_update<VEC,SLOTG>  optimizer step over a list of rows (FTRL ftrl.h:54-79,112-146 /
//                           SGD sgd.h:46-59,90-103 / AdaGrad), gradient either from the row's accumulators
//                           (fused step; divides by the slice row count) or from a pushed array.
//   xf_k_probe              keys -> slot indices (insert or find)     } generic Pull / Push /
//   xf_k_gather             slot rows -> w / v arrays                 } import / export pieces
//   xf_k_import / xf_k_export
//   xf_k_rehash             growth and eviction sweeps
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <mutex>
#include <set>
#include <utility>

#include "kernels.h"
#include "table.cuh"

// -------------------------------------------------------------------------------------------------
// fill
// -------------------------------------------------------------------------------------------------
__global__ void xf_k_fill(uint8_t* base, uint64_t cap, uint32_t stride, int lazy) {
  // one thread per 16-byte chunk of the table
  const uint64_t chunks_per_row = stride / 16;
  const uint64_t total = cap * chunks_per_row;
  for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < total;
       c += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t r = c / chunks_per_row;
    uint32_t q = (uint32_t)(c % chunks_per_row);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (q == 0) {
      v.x = 0xFFFFFFFFu; v.y = 0xFFFFFFFFu;    // EMPTY key
      if (!lazy) v.w = XF_NEG_ZERO_BITS;       // high word of the f64 accumulator g = -0.0 ("untouched"); lazy: integer 0
    }
    *reinterpret_cast<uint4*>(base + r * stride + (uint64_t)q * 16) = v;
  }
}

// -------------------------------------------------------------------------------------------------
// vector helpers for the latent blocks
// -------------------------------------------------------------------------------------------------
template <int VEC>
__device__ __forceinline__ void xf_ldv(const float* p, float (&o)[VEC]) {
  if (VEC == 4) { float4 t = __ldcg(reinterpret_cast<const float4*>(p)); o[0] = t.x; o[1 % VEC] = t.y; o[2 % VEC] = t.z; o[3 % VEC] = t.w; }
  else if (VEC == 2) { float2 t = __ldcg(reinterpret_cast<const float2*>(p)); o[0] = t.x; o[1 % VEC] = t.y; }
  else { o[0] = __ldcg(p); }
}
template <int VEC>
__device__ __forceinline__ void xf_stv(float* p, const float (&o)[VEC]) {
  if (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(o[0], o[1 % VEC], o[2 % VEC], o[3 % VEC]);
  else if (VEC == 2) *reinterpret_cast<float2*>(p) = make_float2(o[0], o[1 % VEC]);
  else *p = o[0];
}
// -------------------------------------------------------------------------------------------------
// optimizer step over a list of rows
// -------------------------------------------------------------------------------------------------
// A warp takes 32 consecutive entries of the row list (one coalesced load), compacts the live ones with a
// ballot (the fused step's touched[] is mostly empty: one entry per TOKEN, one live entry per KEY) and
// hands them out to groups of TPS (power of two <= 32) consecutive lanes: lane q of a group handles
// latent coordinates [q*VEC, q*VEC+VEC) and lane 0 additionally the scalar w coordinate.
//   SLOTG = true : gradients are the row's own accumulators (fused step).  g <- g / rows, then the
//                  accumulators are reset (g = -0.0 marker, L = Aq = 0).
//   SLOTG = false: gradients come from gw[i] / gv[i*K+k] (Push).  part bit0: apply w, bit1: apply v.
// Sharded step (comm.cu): the list is the first *n_dev entries of `slots` plus `extra_n` entries at
// slots[extra_base ...) (the accumulation kernel's cache flushes), and the divisor is *rows_dev — both
// known only on the device (they arrive with the source rank's flag).  live_total may be peer memory.
// v0_side (sources >= 1 of a round): the latent gradient is formed with the row as the source PULLED it,
// v0_side[token * K ..], token = the entry's own position, or slots[extra_base + extra_n + j] for extra entry j
// (earlier sources of the same round may have changed v since).
// STAMP (feature eviction, the training call only): every row updated gets stamp[slot] = sv.now.
template <int VEC, bool SLOTG, bool STAMP>
__global__ void __launch_bounds__(256)
xf_k_update(XfTableView t, const uint32_t* __restrict__ slots, uint64_t n, int tps, double rows,
            const float* __restrict__ gw, const float* __restrict__ gv, int part,
            unsigned long long* __restrict__ live_total, const uint32_t* __restrict__ n_dev,
            const uint32_t* __restrict__ rows_dev, uint32_t extra_base, uint32_t extra_n,
            const float* __restrict__ v0_side, XfStampView sv) {
  __shared__ unsigned int s_live;
  if (threadIdx.x == 0) s_live = 0;
  __syncthreads();
  uint64_t n_head = n;  // entries [0, n_head) are slots[0, n_head); entries [n_head, n) are slots[extra_base, ...)
  if (n_dev != nullptr) {
    n_head = min((uint64_t)__ldg(n_dev), (uint64_t)extra_base);
    n = n_head + extra_n;
    rows = (double)__ldg(rows_dev);
  }
  unsigned int live_acc = 0;
  const int K = t.K;
  const unsigned lane = threadIdx.x & 31u;
  const uint64_t gwarp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  const int q = (int)(lane & (unsigned)(tps - 1));
  const int gi = (int)(lane / (unsigned)tps);  // which group of the warp
  const int ngroups = 32 / tps;
  const int leader = (int)(lane & ~(unsigned)(tps - 1));
  const unsigned group_mask = (tps == 32) ? 0xffffffffu : (((1u << tps) - 1u) << leader);
  const int nchunk = K / VEC;

  for (uint64_t base = gwarp * 32; base < n; base += nwarps * 32) {
    // Fused step: walk the touched array BACKWARDS.  The rows touched last by the step kernel are
    // the ones still resident (dirty) in L2; a forward walk meets them only after they have been
    // evicted (LRU thrash).
    const uint64_t e_fwd = base + lane;
    const uint64_t e_i = (SLOTG && e_fwd < n) ? (n - 1 - e_fwd) : e_fwd;
    const uint64_t e_phys = (e_i < n_head) ? e_i : (uint64_t)extra_base + (e_i - n_head);
    const uint32_t s_lane = (e_fwd < n) ? __ldcs(slots + e_phys) : 0xFFFFFFFFu;
    unsigned pend = __ballot_sync(0xffffffffu, s_lane != 0xFFFFFFFFu);
    // rows actually updated (= unique keys of the batch in the fused step)
    if (live_total != nullptr && lane == 0) live_acc += __popc(pend);

    while (pend) {
      // group gi takes the gi-th live entry of this round
      const int cnt = __popc(pend);
      const unsigned src = (gi < cnt) ? __fns(pend, 0, gi + 1) : 0u;
      const uint32_t s = __shfl_sync(0xffffffffu, s_lane, (int)src);
      const uint64_t i = __shfl_sync(0xffffffffu, (unsigned long long)e_i, (int)src);
      const uint64_t i_phys = __shfl_sync(0xffffffffu, (unsigned long long)e_phys, (int)src);
      uint8_t* rowp = (gi < cnt) ? xf_row(t, s) : nullptr;
      pend = (cnt <= ngroups) ? 0u : (pend & ~((2u << __fns(pend, 0, ngroups)) - 1u));

      // Every load of the row is issued before anything is consumed: slot -> {head, accumulators, v, nv,
      // zv} is then two DRAM latencies deep instead of a dependent chain head -> v -> nv/zv.
      // The latent loads are speculative: a row whose latent block is not materialised ignores them.
      const bool lat = K > 0 && (part & 2) && rowp != nullptr;
      float* vp = lat ? xf_row_v(rowp) : nullptr;
      float* nvp = lat ? xf_row_nv(rowp, K) : nullptr;
      float* zvp = lat ? xf_row_zv(rowp, K) : nullptr;
      float v0[VEC], n0[VEC], z0[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) { v0[e] = 0.f; n0[e] = 0.f; z0[e] = 0.f; }
      const bool has0 = lat && q < nchunk;
      if (has0) {
        xf_ldv<VEC>(vp + q * VEC, v0);
        if (t.opt == XF_OPT_FTRL) { xf_ldv<VEC>(nvp + q * VEC, n0); xf_ldv<VEC>(zvp + q * VEC, z0); }
        else if (t.opt == XF_OPT_ADAGRAD) xf_ldv<VEC>(nvp + q * VEC, n0);
      }
      // sharded step, sources >= 1: the latent row as pulled (issued with the other loads)
      float p0[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) p0[e] = 0.f;
      if (SLOTG && v0_side != nullptr && has0) {
        const uint64_t tok = (i_phys < (uint64_t)extra_base) ? i_phys : (uint64_t)__ldg(slots + i_phys + extra_n);
        xf_ldv<VEC>(v0_side + tok * (uint64_t)K + q * VEC, p0);
      }
      // canonical FM tables (step_fmc.cu): gv[k] = A[k] - v[k] * L2, A a float per coordinate behind the state
      float ca0[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) ca0[e] = 0.f;
      if (SLOTG && t.canon && has0) xf_ldv<VEC>(xf_row_ca(t, rowp) + q * VEC, ca0);
      // fused step: gv[k] = Aq - v[k] * L (table.cuh); every lane of the group reads the same 16 bytes
      double accL = 0.0, accA = 0.0;
      if (SLOTG && has0) {
        const double2 a = __ldcg(reinterpret_cast<const double2*>(xf_row_acc(rowp, K)));
        accL = a.x;
        accA = a.y;
      }
      // the group leader reads the head sector once and shares key / flags
      XfHead h;
      h.key = 0; h.flags = 0; h.w = h.n = h.z = 0.f; h.g = 0.0;
      if (q == 0 && rowp != nullptr) h = xf_load_head(rowp);
      const uint64_t key = __shfl_sync(group_mask, (unsigned long long)h.key, leader);
      const uint32_t flags = __shfl_sync(group_mask, h.flags, leader);
      if (rowp == nullptr) continue;  // whole group (pend is warp-uniform, so the loop stays converged)

      if (q == 0) {
        if (!SLOTG) xf_apply_pending(t, h);  // lazy tables: fold the pending batch step in first
        if (part & 1) {
          // the accumulated sum is rounded to float once (push_gradient is a float vector), then / rows
          const float g = SLOTG ? xf_div_rows((float)h.g, rows) : gw[i];
          xf_opt_coord(t, g, h.w, h.n, h.z);
        }
        if (SLOTG) h.g = -0.0;  // "untouched" marker for the next batch
        if (K > 0 && (part & 2)) h.flags |= XF_FLAG_V_READY;
        xf_store_head_t(t, rowp, h);  // one full-sector store (lazy tables: in their own encoding)
        if (STAMP) sv.stamp[s] = sv.now;
      }
      if (lat) {
        const bool ready = (flags & XF_FLAG_V_READY) != 0;
        for (int c = q; c < nchunk; c += tps) {
          const int k = c * VEC;
          float v[VEC], g[VEC], nn[VEC], zz[VEC];
#pragma unroll
          for (int e = 0; e < VEC; ++e) { v[e] = v0[e]; nn[e] = n0[e]; zz[e] = z0[e]; }
          if (c != q && ready) {  // K / VEC > 32 only
            xf_ldv<VEC>(vp + k, v);
            if (t.opt == XF_OPT_FTRL) { xf_ldv<VEC>(nvp + k, nn); xf_ldv<VEC>(zvp + k, zz); }
            else if (t.opt == XF_OPT_ADAGRAD) xf_ldv<VEC>(nvp + k, nn);
          }
          if (!ready) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) { v[e] = xf_v_init(t, key, (uint32_t)(k + e)); nn[e] = 0.f; zz[e] = 0.f; }
          }
          if (SLOTG) {
            float vp0[VEC];  // v the gradient is defined on: the pulled one if given, else the row's
#pragma unroll
            for (int e = 0; e < VEC; ++e) vp0[e] = v[e];
            if (v0_side != nullptr) {
              if (c == q) {
#pragma unroll
                for (int e = 0; e < VEC; ++e) vp0[e] = p0[e];
              } else {
                const uint64_t tok = (i_phys < (uint64_t)extra_base) ? i_phys : (uint64_t)__ldg(slots + i_phys + extra_n);
                xf_ldv<VEC>(v0_side + tok * (uint64_t)K + k, vp0);
              }
            }
            if (t.canon) {
              float ca[VEC];
#pragma unroll
              for (int e = 0; e < VEC; ++e) ca[e] = ca0[e];
              if (c != q) xf_ldv<VEC>(xf_row_ca(t, rowp) + k, ca);
#pragma unroll
              for (int e = 0; e < VEC; ++e) g[e] = xf_div_rows((float)((double)ca[e] - (double)vp0[e] * accL), rows);
              const float zero[VEC] = {};
              xf_stv<VEC>(xf_row_ca(t, rowp) + k, zero);
            } else {
#pragma unroll
              for (int e = 0; e < VEC; ++e) g[e] = xf_div_rows((float)(accA - (double)vp0[e] * accL), rows);
            }
          } else {
#pragma unroll
            for (int e = 0; e < VEC; ++e) g[e] = gv[i * (uint64_t)K + k + e];
          }
          if (t.opt == XF_OPT_FTRL) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) xf_ftrl_coord(t, g[e], v[e], nn[e], zz[e]);
            xf_stv<VEC>(nvp + k, nn);
            xf_stv<VEC>(zvp + k, zz);
          } else if (t.opt == XF_OPT_ADAGRAD) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) xf_adagrad_coord(t, g[e], v[e], nn[e]);
            xf_stv<VEC>(nvp + k, nn);
          } else {
#pragma unroll
            for (int e = 0; e < VEC; ++e) xf_sgd_coord(t, g[e], v[e]);
          }
          xf_stv<VEC>(vp + k, v);
        }
        if (SLOTG) {
          // every lane that needs the accumulators has consumed them by now
          __syncwarp(group_mask);
          if (q == 0) *reinterpret_cast<double2*>(xf_row_acc(rowp, K)) = make_double2(0.0, 0.0);
        }
      }
    }
  }
  if (live_total != nullptr) {
    if (lane == 0 && live_acc) atomicAdd(&s_live, live_acc);
    __syncthreads();
    if (threadIdx.x == 0 && s_live) atomicAdd_system(live_total, (unsigned long long)s_live);
  }
}

// -------------------------------------------------------------------------------------------------
// generic pieces: Pull / Push / import / export / growth
// -------------------------------------------------------------------------------------------------
// keys -> slots (0xFFFFFFFF = absent / overflow).  Optionally emits w (app-0 Pull, ftrl.h:75-77).  A key it inserts
// is stamped with the current batch number when the table tracks stamps; an existing key's stamp is left alone.
template <bool INSERT>
__global__ void xf_k_probe(XfTableView t, const uint64_t* __restrict__ keys, uint64_t n,
                           uint32_t* __restrict__ slots, float* __restrict__ w_out, XfStampView sv) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (uint64_t)gridDim.x * blockDim.x) {
    XfHead h;
    h.w = 0.f;
    int64_t s = xf_probe<INSERT, true>(t, keys[i], &h, &sv);
    slots[i] = s >= 0 ? (uint32_t)s : 0xFFFFFFFFu;
    if (w_out) {
      if (s >= 0) xf_apply_pending(t, h);  // lazy tables: the value the reference's server would hold
      w_out[i] = s >= 0 ? h.w : 0.f;
    }
  }
}

// latent rows of `slots` -> v_out[n*K] (app-1 Pull, ftrl.h:142-144); one thread per coordinate
__global__ void xf_k_gather_v(XfTableView t, const uint32_t* __restrict__ slots, const uint64_t* __restrict__ keys,
                              uint64_t n, float* __restrict__ v_out) {
  const int K = t.K;
  const uint64_t total = n * (uint64_t)K;
  for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total;
       x += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = x / K;
    const int k = (int)(x % K);
    const uint32_t s = slots[i];
    float v = 0.f;
    if (s != 0xFFFFFFFFu) {
      const uint8_t* rowp = xf_row(t, s);
      const uint32_t flags = __ldcg(reinterpret_cast<const uint32_t*>(rowp + XF_OFF_FLAGS));
      v = (flags & XF_FLAG_V_READY) ? __ldcg(reinterpret_cast<const float*>(rowp + 32) + k)
                                    : xf_v_init(t, keys[i], (uint32_t)k);
    }
    v_out[x] = v;
  }
}

// overwrite rows (replay of an exported table).  Keys must be unique; slots from xf_k_probe<true>.
__global__ void xf_k_import(XfTableView t, const uint32_t* __restrict__ slots, uint64_t n,
                            const float* w, const float* nw, const float* zw, const float* v,
                            const float* nv, const float* zv) {
  const int K = t.K;
  const uint64_t per = (uint64_t)K + 1;
  const uint64_t total = n * per;
  for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total;
       x += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = x / per;
    const int c = (int)(x % per);
    const uint32_t s = slots[i];
    if (s == 0xFFFFFFFFu) continue;
    uint8_t* rowp = xf_row(t, s);
    if (c == 0) {
      if (w) {
        if (t.lazy) {
          // lazy rows store (n, z) and derive the weight (FTRL), or store the weight (SGD) or (w, n) (AdaGrad): table.cuh
          XfHead h;
          h.key = *reinterpret_cast<const uint64_t*>(rowp);
          h.w = w[i]; h.n = nw ? nw[i] : 0.f; h.z = zw ? zw[i] : 0.f; h.flags = 0u; h.g = 0.0;
          xf_lazy_store(t, rowp, h, true);  // an imported weight need not be f(z, n): kept beside the state
        } else {
          *reinterpret_cast<float2*>(rowp + XF_OFF_STATE) = make_float2(w[i], nw ? nw[i] : 0.f);
          *reinterpret_cast<float*>(rowp + XF_OFF_STATE + 8) = (zw && t.opt != XF_OPT_ADAGRAD) ? zw[i] : 0.f;  // AdaGrad: z = 0
          *reinterpret_cast<unsigned long long*>(rowp + 8) = XF_NEG_ZERO_BITS64;
        }
      }
      if (v && K > 0) *reinterpret_cast<uint32_t*>(rowp + XF_OFF_FLAGS) = XF_FLAG_V_READY;
    } else if (v) {
      const int k = c - 1;
      xf_row_v(rowp)[k] = v[i * K + k];
      if (k == 0) *reinterpret_cast<double2*>(xf_row_acc(rowp, K)) = make_double2(0.0, 0.0);
      if (t.opt == XF_OPT_FTRL) {
        xf_row_nv(rowp, K)[k] = nv ? nv[i * K + k] : 0.f;
        xf_row_zv(rowp, K)[k] = zv ? zv[i * K + k] : 0.f;
      } else if (t.opt == XF_OPT_ADAGRAD) {
        xf_row_nv(rowp, K)[k] = nv ? nv[i * K + k] : 0.f;  // AdaGrad keeps no zv: zv[] is ignored
      }
    }
  }
}

// read rows without inserting; slots from xf_k_probe<false>
__global__ void xf_k_export(XfTableView t, const uint32_t* __restrict__ slots, const uint64_t* __restrict__ keys,
                            uint64_t n, float* w, float* nw, float* zw, float* v, float* nv, float* zv,
                            uint8_t* present) {
  const int K = t.K;
  const uint64_t per = (uint64_t)K + 1;
  const uint64_t total = n * per;
  for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total;
       x += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = x / per;
    const int c = (int)(x % per);
    const uint32_t s = slots[i];
    const bool have = s != 0xFFFFFFFFu;
    const uint8_t* rowp = have ? xf_row(t, s) : nullptr;
    if (c == 0) {
      XfHead h;
      h.w = h.n = h.z = 0.f;
      if (have) {
        h = xf_load_head(rowp);
        xf_apply_pending(t, h);
      }
      if (present) present[i] = have ? 1 : 0;
      if (w) w[i] = h.w;
      if (nw) nw[i] = h.n;
      if (zw) zw[i] = h.z;
    } else if (v) {
      const int k = c - 1;
      float vv = 0.f, nn = 0.f, zz = 0.f;
      if (have) {
        const uint32_t flags = __ldcg(reinterpret_cast<const uint32_t*>(rowp + XF_OFF_FLAGS));
        if (flags & XF_FLAG_V_READY) {
          vv = __ldcg(reinterpret_cast<const float*>(rowp + 32) + k);
          if (t.opt == XF_OPT_FTRL) {
            nn = __ldcg(xf_row_nv(const_cast<uint8_t*>(rowp), K) + k);
            zz = __ldcg(xf_row_zv(const_cast<uint8_t*>(rowp), K) + k);
          } else if (t.opt == XF_OPT_ADAGRAD) {
            nn = __ldcg(xf_row_nv(const_cast<uint8_t*>(rowp), K) + k);
          }
        } else {
          vv = xf_v_init(t, keys[i], (uint32_t)k);
        }
      }
      v[i * K + k] = vv;
      if (nv) nv[i * K + k] = nn;
      if (zv) zv[i * K + k] = zz;
    }
  }
}

// growth and eviction sweeps: re-insert every live row of `src` that `keep` keeps (growth: all of them) into the
// freshly filled `dst`, exactly as it is (a lazy row's pending step included), and its stamp with it
__global__ void xf_k_rehash(XfTableView src, XfTableView dst, XfKeep keep, const uint32_t* __restrict__ src_stamp,
                            uint32_t* __restrict__ dst_stamp) {
  const uint64_t cap = src.mask + 1;
  const uint32_t chunks = src.stride / 16;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap;
       r += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* srow = xf_row(src, r);
    uint4 a = *reinterpret_cast<const uint4*>(srow);
    uint64_t key = (uint64_t)a.x | ((uint64_t)a.y << 32);
    if (key == XF_EMPTY_KEY) continue;
    const uint32_t stamp = src_stamp != nullptr ? src_stamp[r] : 0u;
    if (src_stamp != nullptr && !xf_keeps(keep, stamp, key)) continue;
    XfHead h;
    int64_t s = xf_probe<true>(dst, key, &h);
    if (s < 0) continue;
    uint8_t* drow = xf_row(dst, (uint64_t)s);
    // the key word is already in place (CAS); copy w, n and everything after
    *reinterpret_cast<uint2*>(drow + 8) = make_uint2(a.z, a.w);
    for (uint32_t c = 1; c < chunks; ++c)
      *reinterpret_cast<uint4*>(drow + 16 * c) = *reinterpret_cast<const uint4*>(srow + 16 * c);
    if (dst_stamp != nullptr) dst_stamp[s] = stamp;
  }
}

// list every live key (checkpoint / full export)
__global__ void xf_k_list_keys(XfTableView t, uint64_t* keys_out, unsigned long long* count, uint64_t max_out) {
  const uint64_t cap = t.mask + 1;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap;
       r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t key = *reinterpret_cast<const uint64_t*>(xf_row(t, r));
    if (key == XF_EMPTY_KEY) continue;
    unsigned long long idx = atomicAdd(count, 1ull);
    if (idx < max_out) keys_out[idx] = key;
  }
}

// -------------------------------------------------------------------------------------------------
// host-side launchers (plain C++ signatures, see kernels.h)
// -------------------------------------------------------------------------------------------------
static int g_sm_count = 0;
int xf_sms() {
  if (g_sm_count == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (g_sm_count <= 0) g_sm_count = 132;  // H100 SXM
  }
  return g_sm_count;
}
int xf_grid_for(uint64_t work_items, int block, int blocks_per_sm) {
  uint64_t want = (work_items + block - 1) / block;
  uint64_t cap = (uint64_t)xf_sms() * blocks_per_sm;
  if (want < 1) want = 1;
  return (int)(want < cap ? want : cap);
}
int xf_grid_smem(const void* kernel, uint64_t work_items, int block, size_t smem) {
  if (smem > 48 * 1024) {
    // the opt-in is per device and per kernel: made once each, however many host threads launch at once
    static std::mutex mu;
    static std::set<std::pair<int, const void*>> done;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(mu);
    if (done.insert({dev, kernel}).second)
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  const int per_sm = (int)(227 * 1024 / (smem + 1024));
  return xf_grid_for(work_items, block, per_sm < 8 ? per_sm : 8);
}

int xf_vec_for(int K) { return K <= 0 ? 1 : (K % 4 == 0 ? 4 : (K % 2 == 0 ? 2 : 1)); }
int xf_tps_for(int K) {
  if (K <= 0) return 1;
  int chunks = K / xf_vec_for(K);
  int tps = 1;
  while (tps < chunks && tps < 32) tps <<= 1;
  return tps;
}

void xf_launch_fill(const XfTableView& t, cudaStream_t st) {
  uint64_t cap = t.mask + 1;
  uint64_t total = cap * (t.stride / 16);
  xf_k_fill<<<xf_grid_for(total, 256, 16), 256, 0, st>>>(t.base, cap, t.stride, t.lazy);
}

template <bool SLOTG, bool STAMP = false>
static void xf_launch_update_t(const XfTableView& t, const uint32_t* slots, uint64_t n, double rows,
                               const float* gw, const float* gv, int part, unsigned long long* live_total,
                               cudaStream_t st, const uint32_t* n_dev = nullptr, const uint32_t* rows_dev = nullptr,
                               uint32_t extra_base = 0, uint32_t extra_n = 0, const float* v0_side = nullptr,
                               XfStampView sv = XfStampView{nullptr, 0u}) {
  const int tps = xf_tps_for(t.K);
  const int grid = xf_grid_for(n * (uint64_t)tps, 256, 8);
#define XF_UPD_ARGS t, slots, n, tps, rows, gw, gv, part, live_total, n_dev, rows_dev, extra_base, extra_n, v0_side, sv
  switch (xf_vec_for(t.K)) {
    case 4: xf_k_update<4, SLOTG, STAMP><<<grid, 256, 0, st>>>(XF_UPD_ARGS); break;
    case 2: xf_k_update<2, SLOTG, STAMP><<<grid, 256, 0, st>>>(XF_UPD_ARGS); break;
    default: xf_k_update<1, SLOTG, STAMP><<<grid, 256, 0, st>>>(XF_UPD_ARGS); break;
  }
#undef XF_UPD_ARGS
}

// sharded step: touched[] of one source rank, list length and divisor read on the device
void xf_launch_update_touched_dev(const XfTableView& t, const uint32_t* touched, uint64_t work_bound,
                                  const uint32_t* n_dev, const uint32_t* rows_dev, uint32_t extra_base,
                                  uint32_t extra_n, const float* v0_side, unsigned long long* unique_total,
                                  cudaStream_t st) {
  xf_launch_update_t<true>(t, touched, work_bound + extra_n, 1.0, nullptr, nullptr, 3, unique_total, st, n_dev, rows_dev,
                           extra_base, extra_n, v0_side);
}

// lazy tables: fold every pending optimizer step into its row (tags back to 0); lets the batch sequence
// numbers restart, so rows_by_seq is a fixed-size ring instead of an ever-growing array
__global__ void xf_k_flush_pending(XfTableView t) {
  const uint64_t cap = t.mask + 1;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap; r += (uint64_t)gridDim.x * blockDim.x) {
    uint8_t* rowp = xf_row(t, r);
    XfHead h = xf_load_head(rowp);
    if (h.key == XF_EMPTY_KEY || !xf_lazy_has_pending(h)) continue;
    xf_apply_pending(t, h);
    xf_lazy_store(t, rowp, h);
  }
}
void xf_launch_flush_pending(const XfTableView& t, cudaStream_t st) {
  xf_k_flush_pending<<<xf_grid_for(t.mask + 1, 256, 8), 256, 0, st>>>(t);
}

void xf_launch_update_touched(const XfTableView& t, const uint32_t* touched, uint64_t nnz, double rows,
                              unsigned long long* unique_total, const XfStampView& sv, cudaStream_t st) {
  if (nnz == 0) return;
  if (sv.stamp)
    xf_launch_update_t<true, true>(t, touched, nnz, rows, nullptr, nullptr, 3, unique_total, st, nullptr, nullptr, 0, 0,
                                   nullptr, sv);
  else
    xf_launch_update_t<true>(t, touched, nnz, rows, nullptr, nullptr, 3, unique_total, st);
}

void xf_launch_update_pushed(const XfTableView& t, const uint32_t* slots, uint64_t n, const float* gw,
                             const float* gv, cudaStream_t st) {
  if (n == 0) return;
  int part = (gw ? 1 : 0) | (gv ? 2 : 0);
  xf_launch_update_t<false>(t, slots, n, 1.0, gw, gv, part, nullptr, st);
}

void xf_launch_probe(const XfTableView& t, const uint64_t* keys, uint64_t n, bool insert, uint32_t* slots,
                     float* w_out, cudaStream_t st, const XfStampView& sv) {
  if (n == 0) return;
  const int grid = xf_grid_for(n, 256, 8);
  if (insert) xf_k_probe<true><<<grid, 256, 0, st>>>(t, keys, n, slots, w_out, sv);
  else xf_k_probe<false><<<grid, 256, 0, st>>>(t, keys, n, slots, w_out, sv);
}

void xf_launch_gather_v(const XfTableView& t, const uint32_t* slots, const uint64_t* keys, uint64_t n,
                        float* v_out, cudaStream_t st) {
  if (n == 0 || t.K == 0) return;
  xf_k_gather_v<<<xf_grid_for(n * t.K, 256, 8), 256, 0, st>>>(t, slots, keys, n, v_out);
}

void xf_launch_import(const XfTableView& t, const uint32_t* slots, uint64_t n, const float* w, const float* nw,
                      const float* zw, const float* v, const float* nv, const float* zv, cudaStream_t st) {
  if (n == 0) return;
  xf_k_import<<<xf_grid_for(n * (t.K + 1), 256, 8), 256, 0, st>>>(t, slots, n, w, nw, zw, v, nv, zv);
}

void xf_launch_export(const XfTableView& t, const uint32_t* slots, const uint64_t* keys, uint64_t n, float* w,
                      float* nw, float* zw, float* v, float* nv, float* zv, uint8_t* present, cudaStream_t st) {
  if (n == 0) return;
  xf_k_export<<<xf_grid_for(n * (t.K + 1), 256, 8), 256, 0, st>>>(t, slots, keys, n, w, nw, zw, v, nv, zv, present);
}

void xf_launch_rehash(const XfTableView& src, const XfTableView& dst, const XfKeep& keep, const uint32_t* src_stamp,
                      uint32_t* dst_stamp, cudaStream_t st) {
  xf_k_rehash<<<xf_grid_for(src.mask + 1, 256, 8), 256, 0, st>>>(src, dst, keep, src_stamp, dst_stamp);
}

void xf_launch_list_keys(const XfTableView& t, uint64_t* keys_out, unsigned long long* count, uint64_t max_out,
                         cudaStream_t st) {
  xf_k_list_keys<<<xf_grid_for(t.mask + 1, 256, 8), 256, 0, st>>>(t, keys_out, count, max_out);
}

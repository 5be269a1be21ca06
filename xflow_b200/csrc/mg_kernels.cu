// sm_90a kernels of the sharded (multi-GPU) step; layout and protocol in mg.cuh, stream schedule in
// comm.cu.  Every exchange is done by the producing kernel itself with stores into the consumer's
// memory over NVLink (cudaIpc-mapped slabs); xf_k_signal / xf_k_wait order them with step counters.
//
// Arithmetic is the single-GPU step's (step.cu / step_lazy.cu), split at the two places where the
// reference has a process boundary: Pull (lr_worker.cc:159-161, fm_worker.cc:219-226) and Push
// (lr_worker.cc:172-175, fm_worker.cc:236-243).
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "mg.cuh"
#include "table.cuh"

#define XF_NO_SLOT 0xFFFFFFFFu

// ---------------------------------------------------------------------------------------------------
// flags
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long xf_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint64_t xf_ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void xf_st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// thread q tells rank q "my data of `step` for `flag` is in your slab".  Everything this rank's earlier
// kernels (same stream) stored into peer memory is ordered before the flag by the system-scope fence.
// For XF_F_KEYS the flag carries the bucket size and the batch's row count (meta).
__global__ void xf_k_signal(XfPeers peers, XfSlabLayout L, int S, int me, int flag, uint64_t step, int parity,
                            const uint32_t* __restrict__ bucket_cnt, uint32_t rows) {
  const int q = threadIdx.x;
  if (q >= S) return;
  uint8_t* slab = peers.slab[q];
  if (bucket_cnt != nullptr) {
    volatile uint32_t* m = reinterpret_cast<uint32_t*>(slab + L.off_meta) + ((size_t)(parity * XF_MG_MAX_SHARDS + me) * 4);
    m[0] = bucket_cnt[q];
    m[1] = rows;
  }
  // the release orders everything before it in this stream (the producing kernel included) ahead of the flag;
  // a separate fence in front of it would drain the peer stores a second time
  xf_st_release_sys(reinterpret_cast<uint64_t*>(slab + L.off_flags) + (size_t)flag * XF_MG_MAX_SHARDS + me, step);
}

// thread q waits until rank q's counter for this flag has reached `step` (bounded: error 4, no hung GPU)
__global__ void xf_k_wait(const uint64_t* __restrict__ flags, int S, uint64_t step, int* error,
                          unsigned long long timeout_ns) {
  const int q = threadIdx.x;
  if (q >= S) return;
  const unsigned long long t0 = xf_globaltimer();
  while (xf_ld_acquire_sys(flags + q) < step) {
    if (xf_globaltimer() - t0 > timeout_ns) {
      *error = 4;
      break;
    }
    __nanosleep(64);
  }
}

// ---------------------------------------------------------------------------------------------------
// worker: route every token to the owner of its key
// ---------------------------------------------------------------------------------------------------
#define XF_RT_THREADS 512
#define XF_RT_TOK 4
#define XF_RT_TILE (XF_RT_THREADS * XF_RT_TOK)

__device__ __forceinline__ int xf_dev_shard_of(uint64_t key, uint64_t width, int S) {
  const uint64_t s = key / width;
  return (int)(s < (uint64_t)S ? s : (uint64_t)S - 1);
}

// last r in [lo, hi] with a[r] <= j (a ascending; a[lo] <= j is guaranteed by the caller)
__device__ __forceinline__ uint32_t xf_row_of(const uint32_t* a, uint32_t lo, uint32_t hi, uint32_t j) {
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (a[mid] <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// A CTA takes a tile of 2048 consecutive tokens, groups them by owner in shared memory (ranks from
// shared-memory atomics, one global atomic per CTA and owner reserves the tile's run inside the
// (me -> owner) segment) and writes each owner's run with coalesced stores into that owner's slab:
// key (8 B) and row number (4 B) per token.  tok_pos[j] = owner * cap + position remembers where the
// answer for token j will land in this rank's vals[] array.
__global__ void __launch_bounds__(XF_RT_THREADS)
xf_k_route(const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys, uint32_t rows, uint64_t width,
           int S, int me, uint32_t cap, XfPeers peers, uint64_t off_keys, uint64_t off_rows,
           uint32_t* __restrict__ bucket_cnt, uint32_t* __restrict__ tok_pos) {
  __shared__ uint64_t s_key[XF_RT_TILE];
  __shared__ uint32_t s_row[XF_RT_TILE];
  __shared__ uint32_t s_rp[XF_RT_TILE + 1];  // row_ptr slice of the tile (when it fits)
  __shared__ uint32_t s_cnt[XF_MG_MAX_SHARDS], s_base[XF_MG_MAX_SHARDS], s_off[XF_MG_MAX_SHARDS + 1];
  __shared__ uint32_t s_rlo, s_rhi;
  const uint32_t beg = __ldg(row_ptr), end = __ldg(row_ptr + rows);
  const uint32_t j0 = beg + blockIdx.x * XF_RT_TILE;
  if (j0 >= end) return;
  const uint32_t j1 = min(j0 + (uint32_t)XF_RT_TILE, end);  // exclusive
  if (threadIdx.x < XF_MG_MAX_SHARDS) s_cnt[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_rlo = xf_row_of(row_ptr, 0, rows - 1, j0);
  if (threadIdx.x == 32) s_rhi = xf_row_of(row_ptr, 0, rows - 1, j1 - 1);
  __syncthreads();
  const uint32_t rlo = s_rlo, rhi = s_rhi;
  const bool cached = (rhi - rlo + 1) <= (uint32_t)XF_RT_TILE;
  if (cached)
    for (uint32_t r = threadIdx.x; r <= rhi - rlo + 1; r += XF_RT_THREADS) s_rp[r] = __ldg(row_ptr + rlo + r);
  __syncthreads();

  uint64_t my_key[XF_RT_TOK];
  uint32_t my_rank[XF_RT_TOK], my_row[XF_RT_TOK];
  int my_q[XF_RT_TOK];
#pragma unroll
  for (int i = 0; i < XF_RT_TOK; ++i) {
    const uint32_t j = j0 + threadIdx.x + i * XF_RT_THREADS;
    my_q[i] = -1;
    if (j < j1) {
      my_key[i] = __ldcs(keys + j);
      my_q[i] = xf_dev_shard_of(my_key[i], width, S);
      my_rank[i] = atomicAdd(&s_cnt[my_q[i]], 1u);
      my_row[i] = cached ? (rlo + xf_row_of(s_rp, 0, rhi - rlo, j)) : xf_row_of(row_ptr, rlo, rhi, j);
    }
  }
  __syncthreads();
  if (threadIdx.x < S && s_cnt[threadIdx.x]) s_base[threadIdx.x] = atomicAdd(bucket_cnt + threadIdx.x, s_cnt[threadIdx.x]);
  if (threadIdx.x == 0) {
    uint32_t o = 0;
    for (int q = 0; q < S; ++q) { s_off[q] = o; o += s_cnt[q]; }
    s_off[S] = o;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < XF_RT_TOK; ++i) {
    if (my_q[i] < 0) continue;
    const uint32_t j = j0 + threadIdx.x + i * XF_RT_THREADS;
    const uint32_t at = s_off[my_q[i]] + my_rank[i];
    s_key[at] = my_key[i];
    s_row[at] = my_row[i];
    tok_pos[j] = (uint32_t)my_q[i] * cap + s_base[my_q[i]] + my_rank[i];
  }
  __syncthreads();
  const uint32_t n = j1 - j0;
  for (uint32_t x = threadIdx.x; x < n; x += XF_RT_THREADS) {
    int q = 0;
    while (x >= s_off[q + 1]) ++q;
    const uint64_t dst = (uint64_t)me * cap + s_base[q] + (x - s_off[q]);
    reinterpret_cast<uint64_t*>(peers.slab[q] + off_keys)[dst] = s_key[x];
    reinterpret_cast<uint32_t*>(peers.slab[q] + off_rows)[dst] = s_row[x];
  }
}

// ---------------------------------------------------------------------------------------------------
// owner: Pull handler over the routed tokens of all sources (insert-on-pull, ftrl.h:56,114-120)
// ---------------------------------------------------------------------------------------------------
// One thread per token (all sources in one launch).  The answer goes straight into the source's vals[]
// (segment `me`): LR one float w; FM float4 {w, sum_k v, sum_k v^2, -} — the forward pass needs only
// these two sums of a latent row (fm_worker.cc:178-192) and the owner forms the latent gradient itself
// from its own copy of v (table.cuh: gv = Aq - v L), so neither v nor gv ever crosses NVLink.
// The gradient of a worker is defined on the values it PULLED (fm_worker.cc:141-142): when several sources
// push the same key in one round, the pushes of sources >= 1 find v already changed by the earlier ones.
// The pulled latent row of every token of a source >= 1 is therefore kept in side_v[(s*cap+i)*K ..]
// (streaming writes, local memory) for that source's optimizer pass (xf_k_update, v0_side).
template <bool FM, int VEC>
__global__ void __launch_bounds__(256)
xf_k_pull_tokens(XfTableView t, const uint64_t* __restrict__ in_keys, const uint32_t* __restrict__ meta, int S, int me,
                 uint32_t cap, XfPeers peers, uint64_t off_vals, uint32_t* __restrict__ slots,
                 float* __restrict__ side_v, uint4* __restrict__ stash) {
  __shared__ uint32_t s_pre[XF_MG_MAX_SHARDS + 1];
  if (threadIdx.x == 0) {
    uint32_t o = 0;
    for (int s = 0; s < S; ++s) { s_pre[s] = o; o += min(meta[s * 4], cap); }
    s_pre[S] = o;
  }
  __syncthreads();
  const uint32_t total = s_pre[S];
  const int K = t.K;
  for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < total; x += gridDim.x * blockDim.x) {
    int s = 0;
    while (x >= s_pre[s + 1]) ++s;
    const uint32_t i = x - s_pre[s];
    const uint64_t key = __ldcs(in_keys + (uint64_t)s * cap + i);
    const uint64_t home = xf_home_slot(t, key);
    // FM rows do not change while this kernel runs (only inserts): hot rows may be served by L1
    XfHead h = FM ? xf_load_head_l1(xf_row(t, home)) : xf_load_head(xf_row(t, home));
    const int64_t r = xf_probe_from<true>(t, key, home, h);
    float w = 0.f, st = 0.f, qt = 0.f;
    if (!FM && stash != nullptr) {
      // LR, lazy table: the row's state words exactly as found go to the Push handler of this step (streaming,
      // 16 B per token): its open then needs no load of the row — one row-touching instruction less per token.
      // A row that carries an imported weight beside its state (bytes 8..15, rare) is marked with the tag no
      // batch ever has, and the Push takes a fresh look at it instead.
      const uint64_t q1 = xf_raw_q1(h), q2 = xf_raw_q2(h);
      uint64_t q3 = xf_raw_q3(h);
      if (xf_lazy_given(q1, q2, q3)) q3 |= XF_TAG_MASK;
      __stcs(stash + ((uint64_t)s * cap + i), make_uint4((uint32_t)q2, (uint32_t)(q2 >> 32), (uint32_t)q3, (uint32_t)(q3 >> 32)));
    }
    if (r >= 0) {
      xf_apply_pending(t, h);  // lazy LR tables: the value the reference's server would hold
      w = h.w;
      if (FM) {
        float* sv = (s > 0 && side_v != nullptr) ? side_v + ((uint64_t)s * cap + i) * (uint64_t)K : nullptr;
        if ((h.flags & XF_FLAG_V_READY) && (K & 7) == 0) {
          const float* vp = reinterpret_cast<const float*>(xf_row(t, (uint64_t)r) + 32);
          for (int k = 0; k < K; k += 8) {  // a sector at a time
            float v[8];
            xf_ld8_l1(vp + k, v);
#pragma unroll
            for (int e = 0; e < 8; ++e) { st += v[e]; qt = __fadd_rn(qt, __fmul_rn(v[e], v[e])); }
            if (sv) {
              __stcs(reinterpret_cast<float4*>(sv + k), make_float4(v[0], v[1], v[2], v[3]));
              __stcs(reinterpret_cast<float4*>(sv + k + 4), make_float4(v[4], v[5], v[6], v[7]));
            }
          }
        } else if (h.flags & XF_FLAG_V_READY) {
          const float* vp = reinterpret_cast<const float*>(xf_row(t, (uint64_t)r) + 32);
          for (int k = 0; k < K; k += VEC) {
            float v[VEC];
            if (VEC == 4) { const float4 q4 = __ldca(reinterpret_cast<const float4*>(vp + k)); v[0] = q4.x; v[1 % VEC] = q4.y; v[2 % VEC] = q4.z; v[3 % VEC] = q4.w; }
            else if (VEC == 2) { const float2 q2 = __ldca(reinterpret_cast<const float2*>(vp + k)); v[0] = q2.x; v[1 % VEC] = q2.y; }
            else { v[0] = __ldca(vp + k); }
#pragma unroll
            for (int e = 0; e < VEC; ++e) { st += v[e]; qt = __fadd_rn(qt, __fmul_rn(v[e], v[e])); }
            if (sv) {
              if (VEC == 4) __stcs(reinterpret_cast<float4*>(sv + k), make_float4(v[0], v[1 % VEC], v[2 % VEC], v[3 % VEC]));
              else if (VEC == 2) __stcs(reinterpret_cast<float2*>(sv + k), make_float2(v[0], v[1 % VEC]));
              else __stcs(sv + k, v[0]);
            }
          }
        } else {
          for (int k = 0; k < K; ++k) {
            const float v = xf_v_init(t, key, (uint32_t)k);
            st += v;
            qt = __fadd_rn(qt, __fmul_rn(v, v));
            if (sv) __stcs(sv + k, v);
          }
        }
      }
    }
    slots[(uint64_t)s * cap + i] = r >= 0 ? (uint32_t)r : XF_NO_SLOT;
    const uint64_t dst = (uint64_t)me * cap + i;
    if (FM) reinterpret_cast<float4*>(peers.slab[s] + off_vals)[dst] = make_float4(w, st, qt, 0.f);
    else reinterpret_cast<float*>(peers.slab[s] + off_vals)[dst] = w;
  }
}

// ---------------------------------------------------------------------------------------------------
// worker: per-row sums, sigmoid, residual  (calculate_loss, lr_worker.cc:121-143 / fm_worker.cc:159-202)
// ---------------------------------------------------------------------------------------------------
template <bool FM>
__global__ void __launch_bounds__(256)
xf_k_rows(const uint32_t* __restrict__ row_ptr, const uint8_t* __restrict__ labels, int B, int mode,
          const uint32_t* __restrict__ tok_pos, const void* __restrict__ vals, float* __restrict__ rowv,
          float* __restrict__ loss_out, float* __restrict__ pctr_out, float* __restrict__ abs_loss_sum) {
  __shared__ float s_abs[8];
  float abs_acc = 0.f;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int gwarp = blockIdx.x * wpb + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * wpb;
  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row), end = __ldg(row_ptr + row + 1);
    float wsum = 0.f, ssum = 0.f, qsum = 0.f;
    for (uint32_t j = beg + lane; j < end; j += 32) {
      const uint32_t pos = __ldcs(tok_pos + j);
      if (FM) {
        const float4 a = __ldcg(reinterpret_cast<const float4*>(vals) + pos);
        wsum += a.x; ssum += a.y; qsum += a.z;
      } else {
        wsum += __ldcg(reinterpret_cast<const float*>(vals) + pos);
      }
    }
    const float wx = xf_warp_sum(wsum);
    float Ssum = 0.f, arg = wx;
    if (FM) {
      Ssum = xf_warp_sum(ssum);
      const float Q = xf_warp_sum(qsum);
      arg = __fadd_rn(wx, __fsub_rn(__fmul_rn(Ssum, Ssum), Q));  // fm_worker.cc:193-196
    }
    const float pctr = xf_sigmoid(arg);
    if (mode == 1) {
      if (lane == 0 && pctr_out) pctr_out[row] = pctr;
      continue;
    }
    const float loss = __fsub_rn(pctr, (float)labels[row]);  // lr_worker.cc:141 ; fm_worker.cc:200
    if (lane == 0) {
      if (loss_out) loss_out[row] = loss;
      if (FM) reinterpret_cast<float2*>(rowv)[row] = make_float2(loss, Ssum);
      else rowv[row] = loss;
    }
    abs_acc += fabsf(loss);
  }
  if (abs_loss_sum != nullptr && mode == 0) {
    if (lane == 0) s_abs[threadIdx.x >> 5] = abs_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int w = 0; w < wpb; ++w) tot += s_abs[w];
      atomicAdd(abs_loss_sum, tot);
    }
  }
}

// the per-row residuals of this rank's batch to every owner's in_rowv[me] (blockIdx.y = owner)
__global__ void xf_k_bcast_rowv(const uint32_t* __restrict__ src, uint32_t n_words, XfPeers peers, uint64_t off_rowv,
                                uint64_t dst_word_off) {
  uint32_t* dst = reinterpret_cast<uint32_t*>(peers.slab[blockIdx.y] + off_rowv) + dst_word_off;
  for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < n_words; x += gridDim.x * blockDim.x) dst[x] = __ldcg(src + x);
}

// ---------------------------------------------------------------------------------------------------
// owner: Push handler of ONE source rank, LR on a lazy table ("update on next touch", step_lazy.cu)
// ---------------------------------------------------------------------------------------------------
// The first token of this (step, source) that reaches a row folds the pending optimizer step of the row's
// previous (step, source) in, stamps the row with `seq` and deposits its residual — one 128-bit CAS,
// xf_lazy_deposit in table.cuh; later tokens of the same key add theirs with an integer RED.  The optimizer step
// of THIS push is applied by the next touch (next opener, or on the fly by any reader) with divisor
// rows_by_seq[seq] = the source's batch size: exactly one FTRL/SGD step per (source, key), sources in rank order
// because the S launches are stream-ordered.  One token per lane; with the look at the row that this step's Pull
// stashed (16 B per token, streaming) a token costs ONE row-touching instruction; lanes of a warp that hit the
// same row elect one of them.
__global__ void __launch_bounds__(256)
xf_k_push_tokens_lr(XfTableView t, const uint32_t* __restrict__ slots, const uint32_t* __restrict__ in_rows,
                    const float* __restrict__ rowv, const uint32_t* __restrict__ meta_s, uint32_t cap, uint32_t seq,
                    uint64_t* rows_by_seq, unsigned long long* uniq_remote, const uint4* __restrict__ stash) {
  __shared__ unsigned int s_open;
  if (threadIdx.x == 0) s_open = 0;
  const uint32_t n = min(__ldg(meta_s), cap);
  // the source's tokens for this shard bound every key's residual sum of this push: they set its fixed-point unit
  const int fs = xf_fix_shift(n);
  if (blockIdx.x == 0 && threadIdx.x == 0)  // read by later launches only
    rows_by_seq[seq] = (uint64_t)__ldg(meta_s + 1) | ((uint64_t)fs << 32);
  __syncthreads();
  unsigned int open_acc = 0;
  const int lane = threadIdx.x & 31;
  const uint32_t wpb = blockDim.x >> 5;
  const uint32_t gwarp = blockIdx.x * wpb + (threadIdx.x >> 5);
  const uint32_t nwarps = gridDim.x * wpb;
  // Two groups of 32 tokens per warp and iteration: both deposits are issued before any result is looked at, and
  // the coalesced inputs of the NEXT iteration (slot, row index, stashed state words) are requested before this
  // iteration's atomics go out.  The first version (one group, nothing ahead) stalled on a chain of four dependent
  // round trips per 32 tokens.
  uint32_t s_n[2], r_n[2];
  uint4 b_n[2];
#define XF_PUSH_FETCH(base_)                                                        \
  _Pragma("unroll") for (int u = 0; u < 2; ++u) {                                    \
    const uint32_t i = (base_) + 32u * u + lane;                                     \
    s_n[u] = XF_NO_SLOT; r_n[u] = 0u; b_n[u] = make_uint4(0u, 0u, 0u, 0u);            \
    if (i < n) {                                                                     \
      s_n[u] = __ldcs(slots + i);                                                    \
      r_n[u] = __ldcs(in_rows + i);                                                  \
      b_n[u] = __ldcs(stash + (uint64_t)i);                                          \
    }                                                                                \
  }
  uint32_t base = gwarp * 64;
  if (base < n) { XF_PUSH_FETCH(base) }
  for (; base < n; base += nwarps * 64) {
    uint32_t s[2];
    float l[2];
    uint64_t q2[2], q3[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      s[u] = s_n[u];
      l[u] = 0.f;
      q2[u] = 0ull; q3[u] = (uint64_t)seq;  // invalid lanes: "open", nothing to do
      if (s[u] == XF_NO_SLOT) continue;
      l[u] = __ldcg(rowv + r_n[u]);
      // the row's state as this step's Pull found it (coalesced, streaming) instead of a load of the row
      q2[u] = (uint64_t)b_n[u].x | ((uint64_t)b_n[u].y << 32);
      q3[u] = (uint64_t)b_n[u].z | ((uint64_t)b_n[u].w << 32);
    }
    if (base + nwarps * 64 < n) { XF_PUSH_FETCH(base + nwarps * 64) }
    bool lead[2], issued[2], reload[2];
    long long fix[2];
    uint64_t q2n[2], o2[2], o3[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const bool valid = s[u] != XF_NO_SLOT;
      // tokens of this group that hit the same row: the lowest lane deposits the group's residuals
      const unsigned grp = __match_any_sync(0xffffffffu, valid ? s[u] : (0xFFFFFF00u | (uint32_t)lane));
      lead[u] = valid && lane == __ffs(grp) - 1;
      fix[u] = valid ? xf_fix_of(l[u], fs) : 0ll;
      if (__any_sync(0xffffffffu, valid && __popc(grp) > 1)) {
        long long sum = 0ll;
        for (int b = 0; b < 32; ++b) {
          const long long o = __shfl_sync(0xffffffffu, fix[u], b);
          if ((grp >> b) & 1u) sum += o;
        }
        fix[u] = sum;
      }
      issued[u] = false;
      q2n[u] = q2[u]; o2[u] = q2[u]; o3[u] = q3[u];
      reload[u] = lead[u] && (q3[u] & XF_TAG_MASK) == XF_TAG_MASK;  // the Pull saw an imported weight
      if (lead[u] && !reload[u]) {
        xf_lazy_fold(t, 0ull, q2[u], q3[u], seq, q2n[u]);  // no imported weight: bytes 8..15 play no part
        issued[u] = xf_lazy_deposit_issue(xf_row(t, s[u]), q2[u], q3[u], q2n[u], seq, fix[u], o2[u], o3[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (!lead[u]) continue;
      uint8_t* rowp = xf_row(t, s[u]);
      bool stale = false;
      if (!reload[u] &&
          xf_lazy_deposit_resolve(rowp, issued[u], q2[u], q3[u], o2[u], o3[u], seq, fix[u], &stale))
        ++open_acc;
      if (stale) {
        // An earlier source of this round changed the row since the Pull.  The failed CAS has brought the row's
        // current state words back; rows with an imported weight never come this way (marked by the Pull), so
        // bytes 8..15 play no part and no further look at the row is needed.
        uint64_t r2n;
        xf_lazy_fold(t, 0ull, o2[u], o3[u], seq, r2n);
        if (xf_lazy_deposit(t, rowp, o2[u], o3[u], r2n, seq, fix[u])) ++open_acc;
      } else if (reload[u]) {
        const XfHead h = xf_load_head(rowp);
        uint64_t r2n;
        xf_lazy_fold(t, xf_raw_q1(h), xf_raw_q2(h), xf_raw_q3(h), seq, r2n);
        if (xf_lazy_deposit(t, rowp, xf_raw_q2(h), xf_raw_q3(h), r2n, seq, fix[u])) {
          xf_lazy_mark_open(rowp, xf_raw_q1(h), xf_raw_q2(h), xf_raw_q3(h), seq);
          ++open_acc;
        }
      }
    }
  }
#undef XF_PUSH_FETCH
  if (open_acc) atomicAdd(&s_open, open_acc);
  __syncthreads();
  if (threadIdx.x == 0 && s_open && uniq_remote) atomicAdd_system(uniq_remote, (unsigned long long)s_open);
}

// ---------------------------------------------------------------------------------------------------
// owner: Push handler of ONE source rank, gradient accumulation on an eager table (FM, or LR with
// XFLOW_EAGER=1); followed by xf_k_update over touched[] (kernels.cu).  Same accumulators, hot-key cache
// and first-touch detection as phase B of xf_k_step (step.cu); the terms of a token come from the row
// record the source broadcast: residual (and S for FM).
// ---------------------------------------------------------------------------------------------------
template <bool FM>
__global__ void __launch_bounds__(256)
xf_k_acc_tokens(XfTableView t, const uint32_t* __restrict__ slots, const uint32_t* __restrict__ in_rows,
                const void* __restrict__ rowv, const uint32_t* __restrict__ meta_s, uint32_t cap,
                uint32_t* __restrict__ touched, int log2nc) {
  extern __shared__ __align__(16) unsigned char xf_smem[];
  const int K = t.K;
  const int NC = (FM && log2nc >= 0) ? (1 << log2nc) : 0;
  double* c_acc = reinterpret_cast<double*>(xf_smem);
  uint32_t* c_tag = reinterpret_cast<uint32_t*>(xf_smem + (size_t)NC * 24);
  uint32_t* c_tok = c_tag + NC;  // a token of the entry's key (its pulled latent row is in side_v)
  if (NC) {
    for (int e = threadIdx.x; e < NC; e += blockDim.x) { c_tag[e] = XF_NO_SLOT; c_tok[e] = 0; }
    for (int e = threadIdx.x; e < NC * 3; e += blockDim.x) c_acc[e] = 0.0;
    __syncthreads();
  }
  const uint32_t n = min(__ldg(meta_s), cap);
  const int lane = threadIdx.x & 31;
  const uint32_t wpb = blockDim.x >> 5;
  const uint32_t gwarp = blockIdx.x * wpb + (threadIdx.x >> 5);
  const uint32_t nwarps = gridDim.x * wpb;
  for (uint32_t base = gwarp * 32; base < n; base += nwarps * 32) {
    const uint32_t i = base + lane;
    uint32_t s = XF_NO_SLOT;
    float loss = 0.f, Srow = 0.f;
    if (i < n) {
      s = __ldcs(slots + i);
      const uint32_t row = __ldcs(in_rows + i);
      if (FM) { const float2 a = __ldcg(reinterpret_cast<const float2*>(rowv) + row); loss = a.x; Srow = a.y; }
      else loss = __ldcg(reinterpret_cast<const float*>(rowv) + row);
    }
    const bool valid = s != XF_NO_SLOT;
    float gw_c = loss;
    if (FM) {  // fm_worker.cc:140 accumulates the w-gradient inside the k loop: K sequential float adds
      gw_c = 0.f;
      for (int k = 0; k < K; ++k) gw_c += loss;
    }
    double gd = (double)gw_c, ld = (double)loss, ad = (double)loss * (double)Srow;  // exact products
    // tokens of this warp that hit the same row are merged: the group's lowest lane adds the group's sums
    const unsigned grp = __match_any_sync(0xffffffffu, valid ? s : (0xFFFFFF00u | (uint32_t)lane));
    const bool lead = valid && lane == __ffs(grp) - 1;
    if (__any_sync(0xffffffffu, valid && __popc(grp) > 1)) {
      double sg = 0.0, sl = 0.0, sa = 0.0;
      for (int b = 0; b < 32; ++b) {
        const double og = __shfl_sync(0xffffffffu, gd, b), ol = __shfl_sync(0xffffffffu, ld, b),
                     oa = __shfl_sync(0xffffffffu, ad, b);
        if ((grp >> b) & 1u) { sg += og; sl += ol; sa += oa; }
      }
      gd = sg; ld = sl; ad = sa;
    }
    bool first = false;
    if (lead) {
      bool cached = false;
      if (NC) {
        const uint32_t e = (s * 2654435761u) >> (32 - log2nc);
        const uint32_t prev = atomicCAS(c_tag + e, XF_NO_SLOT, s);
        if (prev == XF_NO_SLOT || prev == s) {
          cached = true;
          if (prev == XF_NO_SLOT) c_tok[e] = i;
          atomicAdd(c_acc + 3 * e, gd);
          atomicAdd(c_acc + 3 * e + 1, ld);
          atomicAdd(c_acc + 3 * e + 2, ad);
        }
      }
      if (!cached) {
        uint8_t* rowp = xf_row(t, s);
        const double old = atomicAdd(xf_row_g(rowp), gd);
        if (FM) { double* a = xf_row_acc(rowp, K); atomicAdd(a, ld); atomicAdd(a + 1, ad); }
        first = (unsigned long long)__double_as_longlong(old) == XF_NEG_ZERO_BITS64;
      }
    }
    if (i < n) __stcs(touched + i, first ? s : XF_NO_SLOT);
  }
  if (NC) {
    // flush the hot-key cache: one set of global atomics per entry; extras live at touched[cap ...), the
    // token that stands for each extra entry right behind them (touched[cap + gridDim.x * NC ...))
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
      touched[cap + (uint32_t)blockIdx.x * (uint32_t)NC + (uint32_t)e] = rec;
      touched[cap + (gridDim.x + (uint32_t)blockIdx.x) * (uint32_t)NC + (uint32_t)e] = c_tok[e];
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------------
int xf_step_cache_log2(int K);

void xf_launch_signal(const XfPeers& peers, const XfSlabLayout& L, int S, int me, int flag, uint64_t step, int parity,
                      const uint32_t* bucket_cnt, uint32_t rows, cudaStream_t st) {
  xf_k_signal<<<1, 32, 0, st>>>(peers, L, S, me, flag, step, parity, bucket_cnt, rows);
}
void xf_launch_wait(const uint64_t* flags, int S, uint64_t step, int* error, unsigned long long timeout_ns,
                    cudaStream_t st) {
  xf_k_wait<<<1, 32, 0, st>>>(flags, S, step, error, timeout_ns);
}
void xf_launch_route(const uint32_t* row_ptr, const uint64_t* keys, uint32_t rows, uint32_t nnz_bound, uint64_t width,
                     int S, int me, uint32_t cap, const XfPeers& peers, uint64_t off_keys, uint64_t off_rows,
                     uint32_t* bucket_cnt, uint32_t* tok_pos, cudaStream_t st) {
  if (rows == 0 || nnz_bound == 0) return;
  const uint32_t grid = (nnz_bound + XF_RT_TILE - 1) / XF_RT_TILE;
  xf_k_route<<<grid, XF_RT_THREADS, 0, st>>>(row_ptr, keys, rows, width, S, me, cap, peers, off_keys, off_rows,
                                              bucket_cnt, tok_pos);
}
void xf_launch_pull_tokens(const XfTableView& t, const uint64_t* in_keys, const uint32_t* meta, int S, int me,
                           uint32_t cap, uint64_t work_bound, const XfPeers& peers, uint64_t off_vals,
                           uint32_t* slots, float* side_v, void* stash, cudaStream_t st) {
  const int grid = xf_grid_for(work_bound ? work_bound : 1, 256, 8);
#define XF_PT_ARGS t, in_keys, meta, S, me, cap, peers, off_vals, slots, side_v, reinterpret_cast<uint4*>(stash)
  if (t.K == 0) {
    xf_k_pull_tokens<false, 1><<<grid, 256, 0, st>>>(XF_PT_ARGS);
  } else {
    switch (xf_vec_for(t.K)) {
      case 4: xf_k_pull_tokens<true, 4><<<grid, 256, 0, st>>>(XF_PT_ARGS); break;
      case 2: xf_k_pull_tokens<true, 2><<<grid, 256, 0, st>>>(XF_PT_ARGS); break;
      default: xf_k_pull_tokens<true, 1><<<grid, 256, 0, st>>>(XF_PT_ARGS); break;
    }
  }
#undef XF_PT_ARGS
}
void xf_launch_rows(bool fm, const uint32_t* row_ptr, const uint8_t* labels, int B, int mode, const uint32_t* tok_pos,
                    const void* vals, float* rowv, float* loss_out, float* pctr_out, float* abs_loss_sum,
                    cudaStream_t st) {
  if (B <= 0) return;
  const int grid = xf_grid_for((uint64_t)B * 32, 256, 8);
  if (fm) xf_k_rows<true><<<grid, 256, 0, st>>>(row_ptr, labels, B, mode, tok_pos, vals, rowv, loss_out, pctr_out, abs_loss_sum);
  else xf_k_rows<false><<<grid, 256, 0, st>>>(row_ptr, labels, B, mode, tok_pos, vals, rowv, loss_out, pctr_out, abs_loss_sum);
}
void xf_launch_bcast_rowv(const float* src, uint32_t n_words, int S, const XfPeers& peers, uint64_t off_rowv,
                          uint64_t dst_word_off, cudaStream_t st) {
  if (n_words == 0) return;
  dim3 grid((unsigned)xf_grid_for(n_words, 256, 1), (unsigned)S);
  if (grid.x > 64) grid.x = 64;
  xf_k_bcast_rowv<<<grid, 256, 0, st>>>(reinterpret_cast<const uint32_t*>(src), n_words, peers, off_rowv, dst_word_off);
}
void xf_launch_push_tokens_lr(const XfTableView& t, const uint32_t* slots, const uint32_t* in_rows, const float* rowv,
                              const uint32_t* meta_s, uint32_t cap, uint64_t work_bound, uint32_t seq,
                              uint64_t* rows_by_seq, unsigned long long* uniq_remote, const void* stash,
                              cudaStream_t st) {
  const int grid = xf_grid_for(work_bound ? work_bound : 1, 256, 8);
  xf_k_push_tokens_lr<<<grid, 256, 0, st>>>(t, slots, in_rows, rowv, meta_s, cap, seq, rows_by_seq, uniq_remote,
                                             reinterpret_cast<const uint4*>(stash));
}
// extra touched[] ENTRIES the accumulation kernel appends beyond cap (grid x NC); it needs twice that many
// positions (the entries' representative tokens follow them)
uint32_t xf_acc_touched_extra(int K, uint64_t work_bound) {
  const int lg = xf_step_cache_log2(K);
  if (lg < 0) return 0;
  return (uint32_t)xf_grid_for(work_bound ? work_bound : 1, 256, 8) << lg;
}
void xf_launch_acc_tokens(const XfTableView& t, const uint32_t* slots, const uint32_t* in_rows, const void* rowv,
                          const uint32_t* meta_s, uint32_t cap, uint64_t work_bound, uint32_t* touched,
                          cudaStream_t st) {
  const int grid = xf_grid_for(work_bound ? work_bound : 1, 256, 8);
  const int lg = xf_step_cache_log2(t.K);
  const size_t smem = lg >= 0 ? ((size_t)1 << lg) * 32 : 0;
  if (t.K > 0) xf_k_acc_tokens<true><<<grid, 256, smem, st>>>(t, slots, in_rows, rowv, meta_s, cap, touched, lg);
  else xf_k_acc_tokens<false><<<grid, 256, 0, st>>>(t, slots, in_rows, rowv, meta_s, cap, touched, -1);
}

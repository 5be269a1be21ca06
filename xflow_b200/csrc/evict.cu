// Feature eviction (semantics in include/xflow_b200.h): per-key stamps of the last training batch, and the sweep.
//
// The stamps are one uint32_t per slot (xf_table::d_stamp; kernels get XfStampView) beside the rows: one array serves every row layout
// (the 32-byte lazy LR row has no spare bytes).  The step kernels store them in their tracking instantiations
// (STAMP = true); xf_k_rehash carries them when the table grows or is swept.
//
// A sweep keeps the keys with stamp >= cutoff (the idle limit) and, if more than max_keys of them remain, the
// max_keys most recent ones in the total order (stamp descending, then key ascending).  The boundary (s*, k*) of
// that order is found by radix select over the table itself, with no sort buffer of table size:
//   pass 1  histogram of the stamps' high 16 bits (stamps >= cutoff): the survivors of the idle limit, and the bin
//           of the boundary stamp;
//   pass 2  histogram of the low 16 bits inside that bin: s*;
//   only if fewer than all keys stamped s* survive, passes 3-6 over the 16-bit digits of those keys, high digit
//   first: k*, the largest key that survives.
// Every pass is one read of the keys and stamps.  The rebuild is growth's (xf_table::rebuild), with the predicate.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "internal.h"

__global__ void xf_k_stamp_fill(uint32_t* stamp, uint64_t n, uint32_t value) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    stamp[i] = value;
}

__global__ void xf_k_gather_stamps(const uint32_t* __restrict__ stamp, const uint32_t* __restrict__ slots, uint64_t n,
                                   uint64_t* __restrict__ out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t s = slots[i];
    out[i] = s != 0xFFFFFFFFu ? (uint64_t)stamp[s] : 0xFFFFFFFFFFFFFFFFull;
  }
}

// One pass of the radix select (XfEvictPass, kernels.h).  Keys of one batch share a stamp, so the bins are few and
// hot: lanes with the same bin add once per warp (__match_any_sync).
__global__ void xf_k_evict_hist(XfTableView t, const uint32_t* __restrict__ stamp, XfEvictPass p,
                                unsigned int* __restrict__ hist) {
  const uint64_t cap = t.mask + 1;
  const unsigned lane = threadIdx.x & 31u;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  // the loop runs the same number of rounds in every lane of a warp, so that the match below is warp-wide
  const uint64_t first = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u);
  for (uint64_t base = first; base < cap; base += stride) {
    const uint64_t r = base + lane;
    uint32_t bin = 0xFFFFFFFFu;
    if (r < cap) {
      const uint64_t key = __ldcs(reinterpret_cast<const unsigned long long*>(xf_row(t, r)));
      const uint32_t s = __ldcs(stamp + r);
      if (key != XF_EMPTY_KEY && s >= p.cutoff) {
        if (p.what == 0) {
          bin = s >> 16;
        } else if (p.what == 1) {
          if ((s >> 16) == p.hi) bin = s & 0xFFFFu;
        } else if (s == p.s_star && (p.shift >= 48 || (key >> (p.shift + 16)) == p.prefix)) {
          bin = (uint32_t)(key >> p.shift) & 0xFFFFu;
        }
      }
    }
    const unsigned grp = __match_any_sync(0xffffffffu, bin);
    if (bin != 0xFFFFFFFFu && lane == (unsigned)(__ffs(grp) - 1)) atomicAdd(hist + bin, (unsigned int)__popc(grp));
  }
}

void xf_launch_stamp_fill(uint32_t* stamp, uint64_t n, uint32_t value, cudaStream_t st) {
  xf_k_stamp_fill<<<xf_grid_for(n, 256, 8), 256, 0, st>>>(stamp, n, value);
}
void xf_launch_gather_stamps(const uint32_t* stamp, const uint32_t* slots, uint64_t n, uint64_t* out, cudaStream_t st) {
  if (n == 0) return;
  xf_k_gather_stamps<<<xf_grid_for(n, 256, 8), 256, 0, st>>>(stamp, slots, n, out);
}
void xf_launch_evict_hist(const XfTableView& t, const uint32_t* stamp, const XfEvictPass& p, unsigned int* hist,
                          cudaStream_t st) {
  xf_k_evict_hist<<<xf_grid_for(t.mask + 1, 256, 8), 256, 0, st>>>(t, stamp, p, hist);
}

// -------------------------------------------------------------------------------------------------
// C ABI
// -------------------------------------------------------------------------------------------------
XF_DLL int xf_table_set_eviction(xf_table* t, const xf_eviction_config* cfg) {
  if (!t) { xf_set_error("null argument"); return XF_ERR_ARG; }
  XF_CUDA_TRY(cudaSetDevice(t->cfg.device));
  if (!cfg) {  // stop tracking
    XF_CUDA_TRY(cudaStreamSynchronize(t->stream));  // steps in flight may still store stamps
    if (t->d_stamp) cudaFree(t->d_stamp);
    t->d_stamp = nullptr;
    memset(&t->evict, 0, sizeof(t->evict));
    t->s_hist.release();
    return XF_OK;
  }
  if (t->cfg.canonical_fm) {
    xf_set_error("feature eviction does not serve canonical tables (canonical_fm = 1)");
    return XF_ERR_ARG;
  }
  if (t->cfg.num_shards > 1) {
    xf_set_error("feature eviction needs a single-shard table (this one is shard %d of %d)", t->cfg.shard_index,
                 t->cfg.num_shards);
    return XF_ERR_ARG;
  }
  if (!t->d_stamp) {
    if (t->admit_batches > 0xFFFFFFFFull) {
      xf_set_error("the table has run %llu training batches: more than 32-bit eviction stamps can number",
                   (unsigned long long)t->admit_batches);
      return XF_ERR_STATE;
    }
    const uint64_t cap = t->view.mask + 1;
    uint32_t* stamp = nullptr;
    if (cudaMalloc(&stamp, cap * sizeof(uint32_t)) != cudaSuccess) {
      cudaGetLastError();
      xf_set_error("cannot allocate the eviction stamps of %llu slots", (unsigned long long)cap);
      return XF_ERR_CUDA;
    }
    // every key present now (and whatever the stream still inserts) gets the current batch number
    xf_launch_stamp_fill(stamp, cap, t->stamps().now, t->stream);
    ++t->launches;
    if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(t->stream) != cudaSuccess) {
      cudaFree(stamp);
      xf_set_error("cannot initialise the eviction stamps");
      return XF_ERR_CUDA;
    }
    t->d_stamp = stamp;
  }
  t->evict = *cfg;
  return XF_OK;
}

// the 2^16-bin histogram of one select pass, on the host
static int xf_evict_pass(xf_table* t, const XfEvictPass& p, std::vector<unsigned int>& h) {
  unsigned int* d = t->s_hist.as<unsigned int>();
  XF_CUDA_TRY(cudaMemsetAsync(d, 0, 65536 * sizeof(unsigned int), t->stream));
  xf_launch_evict_hist(t->view, t->d_stamp, p, d, t->stream);
  ++t->launches;
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(h.data(), d, 65536 * sizeof(unsigned int), cudaMemcpyDeviceToHost, t->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(t->stream));
  return XF_OK;
}

XF_DLL int xf_table_evict(xf_table* t, uint64_t* evicted) {
  if (!t) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (evicted) *evicted = 0;
  if (!t->d_stamp) { xf_set_error("xf_table_evict needs eviction tracking (xf_table_set_eviction)"); return XF_ERR_STATE; }
  std::lock_guard<std::mutex> host_lock(t->host_mu);
  XF_CUDA_TRY(cudaSetDevice(t->cfg.device));
  XF_TRY(t->check_error());  // waits for the stream: the stamps and the size are final
  unsigned long long size = 0;
  XF_CUDA_TRY(cudaMemcpy(&size, t->d_size, sizeof(size), cudaMemcpyDeviceToHost));
  XF_TRY(t->s_hist.ensure(65536 * sizeof(unsigned int)));
  std::vector<unsigned int> h(65536);
  const uint64_t B = t->admit_batches, T = t->evict.max_idle_batches, N = t->evict.max_keys;
  XfKeep keep{0u, 0, 0u, 0ull};
  if (T > 0 && B > T) keep.cutoff = (uint32_t)(B - T);
  XfEvictPass p{};
  p.cutoff = keep.cutoff;
  // pass 1: the survivors of the idle limit, by the stamps' high 16 bits
  XF_TRY(xf_evict_pass(t, p, h));
  uint64_t survivors = 0;
  for (unsigned int c : h) survivors += c;
  if (N > 0 && survivors > N) {
    // the N-th most recent key: walk the bins from the most recent down
    uint64_t need = N;
    uint32_t hi = 0;
    for (int b = 65535; b >= 0; --b) {
      if (h[b] >= need) { hi = (uint32_t)b; break; }
      need -= h[b];
    }
    p.what = 1;
    p.hi = hi;
    XF_TRY(xf_evict_pass(t, p, h));
    uint32_t lo = 0;
    for (int b = 65535; b >= 0; --b) {
      if (h[b] >= need) { lo = (uint32_t)b; break; }
      need -= h[b];
    }
    keep.bounded = 1;
    keep.s_star = (hi << 16) | lo;
    keep.k_star = 0xFFFFFFFFFFFFFFFFull;  // every key of stamp s* survives ...
    if (need < h[lo]) {
      // ... unless only `need` of them do: the need-th smallest key of that stamp, 16 bits at a time
      p.what = 2;
      p.s_star = keep.s_star;
      uint64_t prefix = 0;
      for (int shift = 48; shift >= 0; shift -= 16) {
        p.shift = shift;
        p.prefix = prefix;
        XF_TRY(xf_evict_pass(t, p, h));
        uint32_t d = 0;
        for (uint32_t b = 0; b < 65536u; ++b) {
          if (h[b] >= need) { d = b; break; }
          need -= h[b];
        }
        prefix = (prefix << 16) | d;
      }
      keep.k_star = prefix;
    }
    survivors = N;
  }
  const uint64_t cap = t->view.mask + 1;
  uint64_t want = t->cap_floor;
  while (survivors * 2 > want) want <<= 1;
  want = std::min(want, cap);
  if (survivors == size && want == cap) return XF_OK;  // nothing to remove, nothing to shrink
  XF_TRY(t->rebuild(want, keep));
  XF_TRY(t->check_error());
  unsigned long long now = 0;
  XF_CUDA_TRY(cudaMemcpy(&now, t->d_size, sizeof(now), cudaMemcpyDeviceToHost));
  if (now != survivors) {
    xf_set_error("internal error: the eviction sweep kept %llu keys, %llu expected", now, (unsigned long long)survivors);
    return XF_ERR_STATE;
  }
  // ensure_room's bound restarts from the exact count; a size read-back still in flight predates the sweep
  t->size_bound = survivors;
  t->known_size = survivors;
  t->known_at = t->cum_incoming;
  for (int i = 0; i < 4; ++i) t->size_inflight[i] = false;
  if (evicted) *evicted = size - survivors;
  return XF_OK;
}

XF_DLL int xf_table_last_touch(xf_table* t, const uint64_t* keys, uint64_t n, uint64_t* out) {
  if (!t || ((!keys || !out) && n)) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (!t->d_stamp) { xf_set_error("xf_table_last_touch needs eviction tracking (xf_table_set_eviction)"); return XF_ERR_STATE; }
  XF_TRY(xf_check_host_keys(keys, n, "xf_table_last_touch"));
  std::lock_guard<std::mutex> host_lock(t->host_mu);
  if (n == 0) return XF_OK;
  XF_CUDA_TRY(cudaSetDevice(t->cfg.device));
  XF_TRY(t->s_keys.ensure(n * 8));
  XF_TRY(t->s_slots.ensure(n * 4));
  XF_TRY(t->s_w.ensure(n * 8));  // the stamps, as uint64_t
  XF_CUDA_TRY(cudaMemcpyAsync(t->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, t->stream));
  xf_launch_probe(t->view, t->s_keys.as<uint64_t>(), n, false, t->s_slots.as<uint32_t>(), nullptr, t->stream);
  xf_launch_gather_stamps(t->d_stamp, t->s_slots.as<uint32_t>(), n, t->s_w.as<uint64_t>(), t->stream);
  t->launches += 2;
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(out, t->s_w.p, n * 8, cudaMemcpyDeviceToHost, t->stream));
  return xf_table_sync(t);
}

// Serving model deltas: carry one frozen model to the next (layer 7 of include/xflow_b200.h, which documents the
// semantics and the XFSD file format).
//
//   fingerprint  xf_k_fingerprint        one pass over a model's slots: each row's splitmix64 chain, a warp sum, one
//                                        atomic per warp for the sum and one for the row count
//   diff         xf_k_delta_emit<DEL>    one pass over next's slots probing base (the upserts), one over base's slots
//                                        probing next (the deletes), through xf_model_find_slot; a warp-aggregated
//                                        atomic cursor; then the (key, slot) pairs are sorted by key as a model file's
//                                        are, and the upsert rows gathered from next
//   apply        the upserts inserted into a new model sized for the result; xf_k_apply_base puts every row of base
//                whose key is not deleted (a binary search over the sorted delete keys) and not upserted (the claim
//                keeps the row it finds); then the result's fingerprint and key count are checked
//   file         header, upsert rows, delete keys: the chunked sections of serve.cu (xf_chunks_save, xf_chunks_load)
// Every pass hashes, compares or copies whole rows at the model's stride, so one kernel serves every row kind.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <mutex>

#include "serve.cuh"

#define XF_SD_VERSION 1u

// The file header (little-endian, 144 bytes; the layout is documented in include/xflow_b200.h)
struct XfDeltaHeader {
  char magic[4];                // 0 "XFSD"
  uint32_t version;             // 4
  uint64_t header_bytes;        // 8
  int32_t fm;                   // 16
  int32_t latent_dim;           // 20
  int32_t optimizer;            // 24
  int32_t absent;               // 28
  int32_t v_init;               // 32 resolved
  float v_const;                // 36
  uint64_t seed;                // 40
  uint32_t row_bytes;           // 48
  uint32_t precision;           // 52 XF_PRECISION_* (reserved as 0 before F16 models)
  uint64_t base_keys;           // 56
  uint64_t base_fingerprint;    // 64
  uint64_t result_keys;         // 72
  uint64_t source_keys;         // 80
  uint64_t pruned_keys;         // 88
  uint64_t result_fingerprint;  // 96
  uint64_t upserts;             // 104
  uint64_t deletes;             // 112
  uint64_t chunk_rows;          // 120
  uint64_t chunk_keys;          // 128
  uint64_t header_checksum;     // 136 over bytes [0, 136)
};
static_assert(sizeof(XfDeltaHeader) == 144 && offsetof(XfDeltaHeader, seed) == 40 &&
                  offsetof(XfDeltaHeader, base_keys) == 56 && offsetof(XfDeltaHeader, header_checksum) == 136,
              "the documented header is 144 bytes");

struct xf_delta {
  XfDeltaHeader h{};   // everything the file's header records (magic, sizes and checksum filled in by a save)
  int device = 0;
  cudaStream_t stream = nullptr;
  XfDevBuf rows;       // the upsert rows, sorted by key, packed
  XfDevBuf dels;       // the delete keys, sorted
  std::mutex mu;       // serialises saves: the pinned staging
  XfPinBuf stage;
};

// the delta's side of the compatibility check (serve.cuh: XfCompat)
static XfCompat xf_compat_of(const XfDeltaHeader& h) {
  return XfCompat{h.fm, h.latent_dim, h.optimizer, h.absent, h.v_init, h.v_const, h.seed, (int)h.precision};
}

static uint64_t xf_sd_file_bytes(const XfDeltaHeader& h) {
  return sizeof(XfDeltaHeader) + xf_section_bytes(h.upserts, h.row_bytes, h.chunk_rows) + xf_section_bytes(h.deletes, 8u, h.chunk_keys);
}

// -------------------------------------------------------------------------------------------------
// kernels
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t xf_shfl_xor_u64(uint64_t v, int lane_mask) {
  const uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t)v, lane_mask);
  const uint32_t hi = __shfl_xor_sync(0xffffffffu, (uint32_t)(v >> 32), lane_mask);
  return (uint64_t)hi << 32 | lo;
}

// out[0] += the fingerprint of the rows of `m`, out[1] += their number.  A row's fingerprint chains its stride / 8 words
// through splitmix64 (h_0 = 0, h_{i+1} = splitmix64(h_i ^ word_i)), two words per 16-byte load.
__global__ void __launch_bounds__(256) xf_k_fingerprint(XfTableView m, unsigned long long* out) {
  const uint64_t cap = m.mask + 1;
  uint64_t sum = 0ull, rows = 0ull;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* p = xf_row(m, r);
    const ulonglong2 a = *reinterpret_cast<const ulonglong2*>(p);
    if (a.x == XF_EMPTY_KEY) continue;
    uint64_t h = xf_splitmix64(a.y ^ xf_splitmix64(a.x));
    for (uint32_t o = 16; o < m.stride; o += 16) {
      const ulonglong2 b = *reinterpret_cast<const ulonglong2*>(p + o);
      h = xf_splitmix64(xf_splitmix64(h ^ b.x) ^ b.y);
    }
    sum += h;
    ++rows;
  }
  for (int o = 16; o > 0; o >>= 1) {
    sum += xf_shfl_xor_u64(sum, o);
    rows += xf_shfl_xor_u64(rows, o);
  }
  if ((threadIdx.x & 31u) == 0u && rows) {
    atomicAdd(out, (unsigned long long)sum);  // wraps mod 2^64: the fingerprint is that sum
    atomicAdd(out + 1, (unsigned long long)rows);
  }
}

// The rows of `a` that `b` does not hold and, DEL = false, also those `b` holds with other bytes, as (key, slot of
// `a`) pairs at an atomic cursor.  diff(base, next): upserts = emit<false>(next, base), deletes = emit<true>(base, next).
// Whole rows are compared, 16 bytes per load: the padding is zero in every model (xf_model_padding_zero).
template <bool DEL>
__global__ void __launch_bounds__(256)
xf_k_delta_emit(XfTableView a, XfTableView b, uint64_t* __restrict__ keys_out, uint32_t* __restrict__ slots_out,
                unsigned long long* count) {
  const uint64_t cap = a.mask + 1;
  const uint32_t lane = threadIdx.x & 31u;
  // a warp walks 32 consecutive slots per iteration (cap and the stride are multiples of 32: the loop is warp-uniform)
  for (uint64_t r0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull; r0 < cap; r0 += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t r = r0 + lane;
    bool emit = false;
    uint64_t key = XF_EMPTY_KEY;
    if (r < cap) {
      const uint8_t* pa = xf_row(a, r);
      key = __ldg(reinterpret_cast<const unsigned long long*>(pa));
      if (key != XF_EMPTY_KEY) {
        const int64_t s = xf_model_find_slot(b, key);
        emit = s < 0;
        if (!DEL && s >= 0) {
          const uint8_t* pb = xf_row(b, (uint64_t)s);
          for (uint32_t o = 0; o < a.stride && !emit; o += 16) {
            const uint4 x = __ldg(reinterpret_cast<const uint4*>(pa + o)), y = __ldg(reinterpret_cast<const uint4*>(pb + o));
            emit = ((x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w)) != 0u;
          }
        }
      }
    }
    const uint32_t mask = __ballot_sync(0xffffffffu, emit);
    if (mask == 0u) continue;
    unsigned long long first = 0ull;
    if (lane == 0u) first = atomicAdd(count, (unsigned long long)__popc(mask));
    first = __shfl_sync(0xffffffffu, first, 0);
    if (emit) {
      const unsigned long long idx = first + (unsigned long long)__popc(mask & ((1u << lane) - 1u));
      keys_out[idx] = key;
      slots_out[idx] = (uint32_t)r;
    }
  }
}

// whether the sorted keys p[0], p[stride], ... p[(n - 1) stride] (the key word of packed rows, or a key array with
// stride 8) hold `key`
__device__ __forceinline__ bool xf_sorted_has(const uint8_t* __restrict__ p, uint64_t n, uint32_t stride, uint64_t key) {
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    const uint64_t k = __ldg(reinterpret_cast<const unsigned long long*>(p + mid * stride));
    if (k < key) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && __ldg(reinterpret_cast<const unsigned long long*>(p + lo * stride)) == key;
}

// every row of `base` whose key is not in dels[0 .. n_del) into `out`, keeping a row `out` already holds (an upsert)
__global__ void __launch_bounds__(256)
xf_k_apply_base(XfTableView base, XfTableView out, const uint64_t* __restrict__ dels, uint64_t n_del, int* error) {
  const uint64_t cap = base.mask + 1;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* src = xf_row(base, r);
    const ulonglong2 head = __ldg(reinterpret_cast<const ulonglong2*>(src));
    if (head.x == XF_EMPTY_KEY) continue;
    if (n_del && xf_sorted_has(reinterpret_cast<const uint8_t*>(dels), n_del, 8u, head.x)) continue;
    xf_model_put_row<true>(out, src, head, error);
  }
}

// *flag = 1 if a delete key is also an upsert key
__global__ void xf_k_delta_overlap(const uint8_t* __restrict__ rows, uint64_t n_up, uint32_t stride,
                                   const uint64_t* __restrict__ dels, uint64_t n_del, int* flag) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_del; i += (uint64_t)gridDim.x * blockDim.x)
    if (xf_sorted_has(rows, n_up, stride, dels[i])) *flag = 1;
}

// -------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------
// the fingerprint and row count of the rows of `v`, added into d_out[0], d_out[1] on `st`
static int xf_launch_fingerprint(const XfTableView& v, unsigned long long* d_out, cudaStream_t st) {
  xf_k_fingerprint<<<xf_grid_for(v.mask + 1, 256, 8), 256, 0, st>>>(v, d_out);
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

static void xf_delta_free(xf_delta* d) {
  if (!d) return;
  cudaSetDevice(d->device);
  if (d->stream) cudaStreamSynchronize(d->stream);
  d->rows.release();
  d->dels.release();
  d->stage.release();
  if (d->stream) cudaStreamDestroy(d->stream);
  delete d;
}

// the pairs emit<DEL>(a, b) lists, sorted by key; returns their number in *n
static int xf_delta_list(const XfTableView& a, const XfTableView& b, bool del, XfSortedSlots& s, uint64_t* n,
                         cudaStream_t st) {
  XF_CUDA_TRY(cudaMemsetAsync(s.count.p, 0, 8, st));
  const int grid = xf_grid_for(a.mask + 1, 256, 8);
  uint64_t* ko = s.keys_in.as<uint64_t>();
  uint32_t* so = s.slots_in.as<uint32_t>();
  unsigned long long* c = s.count.as<unsigned long long>();
  if (del) xf_k_delta_emit<true><<<grid, 256, 0, st>>>(a, b, ko, so, c);
  else xf_k_delta_emit<false><<<grid, 256, 0, st>>>(a, b, ko, so, c);
  XF_CUDA_TRY(cudaGetLastError());
  unsigned long long got = 0;
  XF_CUDA_TRY(cudaMemcpyAsync(&got, c, 8, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  *n = got;
  return xf_sort_slots(s, got, st);
}

static int xf_diff_into(xf_model* base, xf_model* next, xf_delta* d) {
  d->device = base->device;
  XF_CUDA_TRY(cudaSetDevice(d->device));
  XF_CUDA_TRY(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
  cudaStream_t st = d->stream;
  XfDeltaHeader& h = d->h;
  const XfCompat c = xf_compat_of(next);
  h.fm = c.fm; h.latent_dim = c.latent_dim; h.optimizer = c.optimizer; h.absent = c.absent; h.v_init = c.v_init;
  h.v_const = c.v_const; h.seed = c.seed; h.precision = (uint32_t)c.precision;
  h.row_bytes = next->view.stride;
  h.base_keys = base->keys;
  h.result_keys = next->keys;
  h.source_keys = next->source_keys;
  h.pruned_keys = next->pruned_keys;
  h.chunk_rows = XF_ST_CHUNK_BYTES / h.row_bytes;
  h.chunk_keys = XF_ST_CHUNK_BYTES / 8;
  // both models' fingerprints: {base sum, base rows, next sum, next rows}
  XfDevBuf fp;
  XfSortedSlots s;
  struct Release { XfDevBuf* f; XfSortedSlots* s; ~Release() { f->release(); s->release(); } } rel{&fp, &s};
  XF_TRY(fp.ensure(32));
  XF_CUDA_TRY(cudaMemsetAsync(fp.p, 0, 32, st));
  XF_TRY(xf_launch_fingerprint(base->view, fp.as<unsigned long long>(), st));
  XF_TRY(xf_launch_fingerprint(next->view, fp.as<unsigned long long>() + 2, st));
  XF_TRY(s.ensure(std::max(base->keys, next->keys)));
  // upserts: next's rows that base lacks or holds otherwise, gathered from next in key order
  XF_TRY(xf_delta_list(next->view, base->view, false, s, &h.upserts, st));
  XF_TRY(d->rows.ensure(std::max<uint64_t>(h.upserts * h.row_bytes, 16)));
  XF_TRY(xf_model_gather(next->view, s.slots_out.as<uint32_t>(), h.upserts, d->rows.p, st));
  // deletes: base's keys that next lacks
  XF_TRY(xf_delta_list(base->view, next->view, true, s, &h.deletes, st));
  XF_TRY(d->dels.ensure(std::max<uint64_t>(h.deletes * 8, 16)));
  if (h.deletes) XF_CUDA_TRY(cudaMemcpyAsync(d->dels.p, s.keys_out.p, h.deletes * 8, cudaMemcpyDeviceToDevice, st));
  unsigned long long f[4] = {0, 0, 0, 0};
  XF_CUDA_TRY(cudaMemcpyAsync(f, fp.p, sizeof(f), cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  if (f[1] != base->keys || f[3] != next->keys) {
    xf_set_error("xf_model_diff: a model holds %llu / %llu rows, its info says %llu / %llu", f[1], f[3],
                 (unsigned long long)base->keys, (unsigned long long)next->keys);
    return XF_ERR_STATE;
  }
  h.base_fingerprint = f[0];
  h.result_fingerprint = f[2];
  return XF_OK;
}

XF_DLL int xf_model_diff(xf_model* base, xf_model* next, xf_delta** out) {
  if (out) *out = nullptr;
  if (!base || !next || !out) { xf_set_error("null argument"); return XF_ERR_ARG; }
  XF_TRY(xf_refuse_part(base, "xf_model_diff"));
  XF_TRY(xf_refuse_part(next, "xf_model_diff"));
  if (const char* f = xf_compat_diff(xf_compat_of(base), xf_compat_of(next))) {
    xf_set_error("xf_model_diff: the models differ in %s: a delta carries contents only, not how an absent key reads", f);
    return XF_ERR_ARG;
  }
  if (base->device != next->device) {
    xf_set_error("xf_model_diff: the base is on device %d, the next model on device %d", base->device, next->device);
    return XF_ERR_ARG;
  }
  xf_delta* d = new xf_delta;
  const int rc = xf_diff_into(base, next, d);
  if (rc != XF_OK) { xf_delta_free(d); return rc; }
  *out = d;
  return XF_OK;
}

// the body of xf_model_apply_delta: on failure the caller frees `m`
static int xf_apply_into(xf_model* base, const xf_delta* d, xf_model* m) {
  const XfDeltaHeader& h = d->h;
  XF_TRY(xf_model_init(m, base->device, xf_compat_of(base)));
  cudaStream_t st = m->stream;
  m->keys = h.result_keys;
  m->source_keys = h.source_keys;
  m->pruned_keys = h.pruned_keys;
  // {base sum, base rows, result sum, result rows} and the insert's error flag
  XfDevBuf aux;
  struct Release { XfDevBuf* a; ~Release() { a->release(); } } rel{&aux};
  XF_TRY(aux.ensure(40));
  unsigned long long* fp = aux.as<unsigned long long>();
  int* d_error = reinterpret_cast<int*>(fp + 4);
  XF_CUDA_TRY(cudaMemsetAsync(aux.p, 0, 40, st));
  XF_TRY(xf_launch_fingerprint(base->view, fp, st));
  unsigned long long f[4] = {0, 0, 0, 0};
  XF_CUDA_TRY(cudaMemcpyAsync(f, fp, 16, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  if (f[0] != h.base_fingerprint || f[1] != h.base_keys) {
    xf_set_error("xf_model_apply_delta: the model is not the delta's base (fingerprint %016llx over %llu keys, the delta's "
                 "base: %016llx over %llu keys)", f[0], f[1], (unsigned long long)h.base_fingerprint,
                 (unsigned long long)h.base_keys);
    return XF_ERR_STATE;
  }
  XF_TRY(xf_model_alloc(m, xf_model_capacity(h.result_keys)));
  // 1. the upserts; 2. base's rows that are neither deleted nor upserted; 3. the result's fingerprint
  XF_TRY(xf_model_insert_rows(m->view, static_cast<const uint8_t*>(d->rows.p), h.upserts, d_error, st));
  const int grid = xf_grid_for(base->view.mask + 1, 256, 8);
  const uint64_t* dels = static_cast<const uint64_t*>(d->dels.p);
  xf_k_apply_base<<<grid, 256, 0, st>>>(base->view, m->view, dels, h.deletes, d_error);
  XF_CUDA_TRY(cudaGetLastError());
  XF_TRY(xf_launch_fingerprint(m->view, fp + 2, st));
  int e = 0;
  XF_CUDA_TRY(cudaMemcpyAsync(f, fp, sizeof(f), cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaMemcpyAsync(&e, d_error, 4, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  if (e) {
    xf_set_error("xf_model_apply_delta: a probe sequence of the result overflowed, or an upsert key came twice");
    return XF_ERR_STATE;
  }
  if (f[2] != h.result_fingerprint || f[3] != h.result_keys) {
    xf_set_error("xf_model_apply_delta: the result (fingerprint %016llx over %llu keys) is not the delta's (%016llx over "
                 "%llu keys)", f[2], f[3], (unsigned long long)h.result_fingerprint, (unsigned long long)h.result_keys);
    return XF_ERR_STATE;
  }
  return XF_OK;
}

XF_DLL int xf_model_apply_delta(xf_model* base, const xf_delta* d, xf_model** out) {
  if (out) *out = nullptr;
  if (!base || !d || !out) { xf_set_error("null argument"); return XF_ERR_ARG; }
  XF_TRY(xf_refuse_part(base, "xf_model_apply_delta"));
  if (const char* f = xf_compat_diff(xf_compat_of(base), xf_compat_of(d->h))) {
    xf_set_error("xf_model_apply_delta: the model and the delta differ in %s", f);
    return XF_ERR_ARG;
  }
  if (base->device != d->device) {
    xf_set_error("xf_model_apply_delta: the model is on device %d, the delta on device %d", base->device, d->device);
    return XF_ERR_ARG;
  }
  if (base->keys != d->h.base_keys) {
    xf_set_error("xf_model_apply_delta: the model is not the delta's base: it holds %llu keys, the delta's base %llu",
                 (unsigned long long)base->keys, (unsigned long long)d->h.base_keys);
    return XF_ERR_STATE;
  }
  xf_model* m = new xf_model;
  const int rc = xf_apply_into(base, d, m);
  if (rc != XF_OK) { xf_model_free(m); return rc; }
  *out = m;
  return XF_OK;
}

XF_DLL int xf_model_fingerprint(xf_model* m, uint64_t* out) {
  if (!m || !out) { xf_set_error("null argument"); return XF_ERR_ARG; }
  std::lock_guard<std::mutex> lock(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  XF_TRY(m->s_aux.ensure(16));
  XF_CUDA_TRY(cudaMemsetAsync(m->s_aux.p, 0, 16, m->stream));
  XF_TRY(xf_launch_fingerprint(m->view, m->s_aux.as<unsigned long long>(), m->stream));
  unsigned long long f[2] = {0, 0};
  XF_CUDA_TRY(cudaMemcpyAsync(f, m->s_aux.p, sizeof(f), cudaMemcpyDeviceToHost, m->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(m->stream));
  *out = f[0];
  return XF_OK;
}

XF_DLL int xf_delta_get_info(xf_delta* d, xf_delta_info* out) {
  if (!d || !out) return XF_ERR_ARG;
  memset(out, 0, sizeof(*out));
  const XfDeltaHeader& h = d->h;
  out->upserts = h.upserts;
  out->deletes = h.deletes;
  out->base_keys = h.base_keys;
  out->base_fingerprint = h.base_fingerprint;
  out->result_keys = h.result_keys;
  out->result_fingerprint = h.result_fingerprint;
  out->source_keys = h.source_keys;
  out->pruned_keys = h.pruned_keys;
  out->file_bytes = xf_sd_file_bytes(h);
  out->row_bytes = h.row_bytes;
  out->latent_dim = h.latent_dim;
  out->precision = (int)h.precision;
  return XF_OK;
}

XF_DLL int xf_delta_destroy(xf_delta* d) {
  xf_delta_free(d);
  return XF_OK;
}

// ---- file
static int xf_sd_save_body(xf_delta* d, FILE* f, const char* name) {
  XfDeltaHeader h = d->h;
  memcpy(h.magic, "XFSD", 4);
  h.version = XF_SD_VERSION;
  h.header_bytes = sizeof(h);
  h.header_checksum = xf_st_host_sum(&h, offsetof(XfDeltaHeader, header_checksum), 0);
  if (fwrite(&h, 1, sizeof(h), f) != sizeof(h)) { xf_set_error("write to %s failed", name); return XF_ERR_IO; }
  uint64_t chunk = 0;
  XF_TRY(xf_chunks_save(f, name, h.upserts, h.row_bytes, h.chunk_rows, &chunk, d->stage, d->stream,
                        [&](uint64_t first, uint64_t, const void** dev) {
                          *dev = d->rows.as<uint8_t>() + first * h.row_bytes;
                          return XF_OK;
                        }));
  return xf_chunks_save(f, name, h.deletes, 8u, h.chunk_keys, &chunk, d->stage, d->stream,
                        [&](uint64_t first, uint64_t, const void** dev) {
                          *dev = d->dels.as<uint64_t>() + first;
                          return XF_OK;
                        });
}

XF_DLL int xf_delta_save(xf_delta* d, const char* path) {
  if (!d || !path) { xf_set_error("null argument"); return XF_ERR_ARG; }
  std::lock_guard<std::mutex> lock(d->mu);
  XF_CUDA_TRY(cudaSetDevice(d->device));
  return xf_save_atomic(path, [&](FILE* f, const char* name) { return xf_sd_save_body(d, f, name); });
}

// the header's own consistency (after its checksum): every size derived from it is bounded before it is used
static bool xf_sd_header_sane(const XfDeltaHeader& h) {
  if (!xf_compat_sane(xf_compat_of(h), h.row_bytes)) return false;
  if (h.chunk_rows != XF_ST_CHUNK_BYTES / h.row_bytes || h.chunk_keys != XF_ST_CHUNK_BYTES / 8) return false;
  // a model holds at most 2^31 keys; a result past that is refused by apply (XF_ERR_FULL), not by the file
  if (h.base_keys > (1ull << 31) || h.result_keys > (1ull << 62) || h.source_keys < h.result_keys ||
      h.source_keys - h.result_keys != h.pruned_keys)
    return false;
  return h.upserts <= h.result_keys && h.upserts <= (1ull << 31) && h.deletes <= h.base_keys;
}

static int xf_sd_load_body(xf_delta* d, FILE* f, const char* path, const XfDeltaHeader& h) {
  XF_TRY(xf_file_size_check(f, path, "delta file", xf_sd_file_bytes(h), sizeof(XfDeltaHeader)));
  d->h = h;
  XF_CUDA_TRY(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
  XF_TRY(d->rows.ensure(std::max<uint64_t>(h.upserts * h.row_bytes, 16)));
  XF_TRY(d->dels.ensure(std::max<uint64_t>(h.deletes * 8, 16)));
  // each section into its device buffer as it is
  auto into = [&](XfDevBuf& dst, uint32_t bytes) {
    return [&dst, bytes, d](uint64_t first, uint64_t c, const void* host) {
      XF_CUDA_TRY(cudaMemcpyAsync(dst.as<uint8_t>() + first * bytes, host, c * bytes, cudaMemcpyHostToDevice, d->stream));
      return XF_OK;
    };
  };
  uint64_t chunk = 0;
  XF_TRY(xf_chunks_load(f, path, h.upserts, h.row_bytes, h.chunk_rows, &chunk,
                        XfChunkCheck{"delta file", "upsert", h.fm, h.latent_dim, (int)h.precision, 0, 0}, d->stage, d->stream,
                        into(d->rows, h.row_bytes)));
  XF_TRY(xf_chunks_load(f, path, h.deletes, 8u, h.chunk_keys, &chunk, XfChunkCheck{"delta file", "delete", -1, 0, 0, 0, 0},
                        d->stage, d->stream, into(d->dels, 8u)));
  if (h.upserts && h.deletes) {
    XfDevBuf flag;
    struct Release { XfDevBuf* b; ~Release() { b->release(); } } rel{&flag};
    XF_TRY(flag.ensure(4));
    XF_CUDA_TRY(cudaMemsetAsync(flag.p, 0, 4, d->stream));
    xf_k_delta_overlap<<<xf_grid_for(h.deletes, 256, 8), 256, 0, d->stream>>>(d->rows.as<uint8_t>(), h.upserts, h.row_bytes,
                                                                               d->dels.as<uint64_t>(), h.deletes, flag.as<int>());
    XF_CUDA_TRY(cudaGetLastError());
    int e = 0;
    XF_CUDA_TRY(cudaMemcpyAsync(&e, flag.p, 4, cudaMemcpyDeviceToHost, d->stream));
    XF_CUDA_TRY(cudaStreamSynchronize(d->stream));
    if (e) { xf_set_error("delta file %s: a key is both upserted and deleted", path); return XF_ERR_IO; }
  }
  return XF_OK;
}

XF_DLL int xf_delta_load(xf_delta** out, const char* path, int device) {
  if (out) *out = nullptr;
  if (!out || !path) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (device < 0 || device >= xf_device_count()) { xf_set_error("xf_delta_load: no CUDA device %d", device); return XF_ERR_CUDA; }
  FILE* f = fopen(path, "rb");
  if (!f) { xf_set_error("cannot open %s", path); return XF_ERR_IO; }
  XfDeltaHeader h;
  memset(&h, 0, sizeof(h));
  const size_t got = fread(&h, 1, sizeof(h), f);
  int rc = XF_OK;
  if (xf_refuse_foreign(h.magic, got, path, "XFSD") != XF_OK) {
    rc = XF_ERR_IO;
  } else if (got < 4 || memcmp(h.magic, "XFSD", 4) != 0) {
    xf_set_error("%s is not a serving model delta (no XFSD magic)", path);
    rc = XF_ERR_IO;
  } else if (got != sizeof(h) || h.header_bytes != sizeof(h) || h.version != XF_SD_VERSION) {
    xf_set_error("delta file %s: truncated header or unknown version %u", path, h.version);
    rc = XF_ERR_IO;
  } else if (h.header_checksum != xf_st_host_sum(&h, offsetof(XfDeltaHeader, header_checksum), 0) || !xf_sd_header_sane(h)) {
    xf_set_error("delta file %s: the header is damaged (checksum mismatch or inconsistent fields)", path);
    rc = XF_ERR_IO;
  }
  xf_delta* d = nullptr;
  if (rc == XF_OK) {
    d = new xf_delta;
    d->device = device;
    rc = cudaSetDevice(device) == cudaSuccess ? xf_sd_load_body(d, f, path, h) : XF_ERR_CUDA;
  }
  fclose(f);
  if (rc != XF_OK) { xf_delta_free(d); return rc; }
  *out = d;
  return XF_OK;
}

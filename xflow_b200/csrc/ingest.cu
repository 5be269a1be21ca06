// Device side of the ingest (SURVEY.md section 8, row a1 / next-row f-1): feature-id hashing on the GPU.
//
// The reference's loader turns the id token of "field:id:val" into the parameter-server key with
// std::hash<std::string> (load_data_from_disk.cc:151,173,194).  For numeric ids — what the bundled data
// and every synthetic config use — the key is the MurmurHash64A (hash.h) of the id's decimal string.
// A caller that already holds integer ids can therefore ship 4 bytes per token instead of 8-byte keys
// and let the device make the keys: halves the PCIe traffic of the end-to-end path, bit-exact by
// construction (same hash.h function, __host__ __device__).
#include <cuda_runtime.h>
#include <stdint.h>

#include "hash.h"
#include "internal.h"

__global__ void xf_k_hash_ids(const uint32_t* __restrict__ ids, uint32_t n, uint64_t* __restrict__ keys) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    uint32_t v = __ldcs(ids + i);
    char rev[12];
    int len = 0;
    do { rev[len++] = (char)('0' + v % 10u); v /= 10u; } while (v);
    char buf[12];
    for (int j = 0; j < len; ++j) buf[j] = rev[len - 1 - j];
    keys[i] = xf_murmur64a(buf, (uint64_t)len);
  }
}

int xf_launch_hash_ids(const uint32_t* d_ids, uint32_t n, uint64_t* d_keys, cudaStream_t st) {
  if (n == 0) return XF_OK;
  xf_k_hash_ids<<<xf_grid_for(n, 256, 8), 256, 0, st>>>(d_ids, n, d_keys);
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

XF_DLL int xf_hash_decimal_ids_device(const uint32_t* d_ids, uint64_t n, uint64_t* d_keys, void* cuda_stream) {
  if ((!d_ids || !d_keys) && n) return XF_ERR_ARG;
  if (n > 0xFFFFFFFFull) return XF_ERR_ARG;
  return xf_launch_hash_ids(d_ids, (uint32_t)n, d_keys, (cudaStream_t)cuda_stream);
}

// Pre-population: what a Pull of the ids [first, first + n) by any worker leaves behind — their keys
// exist in the table with default contents (store[key], ftrl.h:56 / sgd.h:48).  Sharded tables keep only
// the keys of their own range (postoffice.cc:134-143).  Ids are hashed as their decimal strings.
__global__ void xf_k_touch_ids(XfTableView t, uint64_t first, uint64_t n, uint64_t width, int S, int shard, XfStampView sv) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t v = first + i;
    char rev[20];
    int len = 0;
    do { rev[len++] = (char)('0' + v % 10u); v /= 10u; } while (v);
    char buf[20];
    for (int j = 0; j < len; ++j) buf[j] = rev[len - 1 - j];
    const uint64_t key = xf_murmur64a(buf, (uint64_t)len);
    if (S > 1) {
      const uint64_t q = key / width;
      if ((int)(q < (uint64_t)S ? q : (uint64_t)S - 1) != shard) continue;
    }
    XfHead h;
    xf_probe<true, true>(t, key, &h, &sv);  // an inserted key is stamped when the table tracks stamps
  }
}

XF_DLL int xf_table_touch_decimal_ids(xf_table* t, uint64_t first_id, uint64_t count) {
  if (!t) return XF_ERR_ARG;
  XF_CUDA_TRY(cudaSetDevice(t->cfg.device));
  const int S = t->cfg.num_shards;
  const uint64_t width = 0xFFFFFFFFFFFFFFFFull / (uint64_t)(S > 0 ? S : 1);
  const uint64_t chunk = 1ull << 24;
  for (uint64_t done = 0; done < count; done += chunk) {
    const uint64_t n = count - done < chunk ? count - done : chunk;
    XF_TRY(t->ensure_room(S > 1 ? n / (uint64_t)S + n / (8 * (uint64_t)S) + 65536 : n));
    xf_k_touch_ids<<<xf_grid_for(n, 256, 8), 256, 0, t->stream>>>(t->view, first_id + done, n, width, S, t->cfg.shard_index,
                                                                        t->stamps());
    ++t->launches;
    XF_CUDA_TRY(cudaGetLastError());
  }
  return XF_OK;
}

// -------------------------------------------------------------------------------------------------
// Text block -> CSR on the device (SURVEY.md section 8f-1): the parser half of
// LoadData::load_minibatch_hash_data_fread (load_data_from_disk.cc:126-209).  The host still forms the
// block (reads the file, cuts at the last newline, carries the tail, :108-124) and ships the raw bytes;
// everything per byte happens here, so file-to-model throughput is no longer capped by one CPU core.
//
//   row   = "<label>\t<tok> <tok> ...\n"      label = ((float)atof(text) > 1e-7)        (:131-135)
//   tok   = "<fgid>:<fid>:<val>"              key = std::hash(<fid>)                     (:146-157)
// A row is owned by the chunk that holds its first byte, a token by the chunk that holds its first
// byte.  Pass 1 counts line starts and token starts per chunk, a two-level scan turns the counts into
// offsets, pass 2 re-walks each chunk and emits row_ptr / labels / keys.  Well-formed input only (every
// token has two ':'), like the reference; a malformed token sets *error.
// -------------------------------------------------------------------------------------------------
#define XF_PARSE_CHUNK 256

__device__ __forceinline__ bool xf_is_line_start(const char* t, uint64_t p) {
  return (p == 0 || t[p - 1] == '\n') && t[p] != '\n';
}
__device__ __forceinline__ bool xf_is_tok_start(const char* t, uint64_t p) {
  if (p == 0) return false;
  const char c = t[p], b = t[p - 1];
  return (b == ' ' || b == '\t') && c != ' ' && c != '\n' && c != '\t' && c != '\r';
}

__global__ void xf_k_parse_count(const char* __restrict__ text, uint64_t len, uint32_t* __restrict__ cnt_rows,
                                 uint32_t* __restrict__ cnt_tok, uint64_t nchunks) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nchunks) return;
  const uint64_t lo = c * XF_PARSE_CHUNK, hi = min(len, lo + XF_PARSE_CHUNK);
  uint32_t r = 0, k = 0;
  for (uint64_t p = lo; p < hi; ++p) {
    r += xf_is_line_start(text, p) ? 1u : 0u;
    k += xf_is_tok_start(text, p) ? 1u : 0u;
  }
  cnt_rows[c] = r;
  cnt_tok[c] = k;
}

// exclusive scan of two arrays of n counts: level 1 (per 1024-element tile) ...
__global__ void __launch_bounds__(1024)
xf_k_scan_tiles(uint32_t* __restrict__ a, uint32_t* __restrict__ b, uint64_t n, uint32_t* __restrict__ tile_a,
                uint32_t* __restrict__ tile_b) {
  __shared__ uint32_t sa[32], sb[32];
  const uint64_t i = (uint64_t)blockIdx.x * 1024 + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t va = i < n ? a[i] : 0u, vb = i < n ? b[i] : 0u;
  uint32_t ia = va, ib = vb;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t ua = __shfl_up_sync(0xffffffffu, ia, o), ub = __shfl_up_sync(0xffffffffu, ib, o);
    if (lane >= o) { ia += ua; ib += ub; }
  }
  if (lane == 31) { sa[warp] = ia; sb[warp] = ib; }
  __syncthreads();
  if (warp == 0) {
    uint32_t wa = sa[lane], wb = sb[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t ua = __shfl_up_sync(0xffffffffu, wa, o), ub = __shfl_up_sync(0xffffffffu, wb, o);
      if (lane >= o) { wa += ua; wb += ub; }
    }
    sa[lane] = wa;
    sb[lane] = wb;
  }
  __syncthreads();
  const uint32_t base_a = warp ? sa[warp - 1] : 0u, base_b = warp ? sb[warp - 1] : 0u;
  if (i < n) { a[i] = base_a + ia - va; b[i] = base_b + ib - vb; }
  if (threadIdx.x == 1023) { tile_a[blockIdx.x] = sa[31]; tile_b[blockIdx.x] = sb[31]; }
}
// ... level 2: one thread block walks the (few) tile totals, then every element adds its tile's base
__global__ void xf_k_scan_tile_totals(uint32_t* tile_a, uint32_t* tile_b, uint32_t ntiles, uint32_t* totals) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    uint32_t ra = 0, rb = 0;
    for (uint32_t i = 0; i < ntiles; ++i) {
      const uint32_t a = tile_a[i], b = tile_b[i];
      tile_a[i] = ra;
      tile_b[i] = rb;
      ra += a;
      rb += b;
    }
    totals[0] = ra;
    totals[1] = rb;
  }
}

// minimal decimal parser for labels that are not the plain "0" / "1": [sign] digits [. digits] [e[sign]digits]
__device__ float xf_parse_label(const char* s, const char* e) {
  while (s < e && (*s == ' ' || *s == '\n' || *s == '\r')) ++s;
  double sign = 1.0;
  if (s < e && (*s == '-' || *s == '+')) { if (*s == '-') sign = -1.0; ++s; }
  double v = 0.0;
  while (s < e && *s >= '0' && *s <= '9') { v = v * 10.0 + (*s - '0'); ++s; }
  if (s < e && *s == '.') {
    ++s;
    double f = 0.1;
    while (s < e && *s >= '0' && *s <= '9') { v += (*s - '0') * f; f *= 0.1; ++s; }
  }
  if (s < e && (*s == 'e' || *s == 'E')) {
    ++s;
    int es = 1, ex = 0;
    if (s < e && (*s == '-' || *s == '+')) { if (*s == '-') es = -1; ++s; }
    while (s < e && *s >= '0' && *s <= '9') { ex = ex * 10 + (*s - '0'); ++s; }
    v *= pow(10.0, (double)(es * ex));
  }
  return (float)(sign * v);
}

__global__ void xf_k_parse_emit(const char* __restrict__ text, uint64_t len, const uint32_t* __restrict__ off_rows,
                                const uint32_t* __restrict__ off_tok, const uint32_t* __restrict__ tile_rows,
                                const uint32_t* __restrict__ tile_tok, uint64_t nchunks, uint32_t max_rows,
                                uint32_t max_tok, uint32_t* __restrict__ row_ptr, uint64_t* __restrict__ keys,
                                uint8_t* __restrict__ labels, int* __restrict__ error) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nchunks) return;
  const uint64_t lo = c * XF_PARSE_CHUNK, hi = min(len, lo + XF_PARSE_CHUNK);
  uint32_t r = off_rows[c] + tile_rows[c >> 10];
  uint32_t k = off_tok[c] + tile_tok[c >> 10];
  for (uint64_t p = lo; p < hi; ++p) {
    if (xf_is_line_start(text, p)) {
      if (r < max_rows) {
        row_ptr[r] = k;
        // label: text from p to the next '\t'
        uint64_t q = p;
        while (q < len && text[q] != '\t' && text[q] != '\n') ++q;
        uint8_t y;
        if (q - p == 1 && (text[p] == '0' || text[p] == '1')) y = (uint8_t)(text[p] - '0');
        else y = (xf_parse_label(text + p, text + q) > 0.0000001) ? 1 : 0;
        labels[r] = y;
      } else {
        *error = 3;
      }
      ++r;
    }
    if (xf_is_tok_start(text, p)) {
      // fid = text between the first and the second ':' of the token
      uint64_t q = p, c1 = 0, c2 = 0;
      int colons = 0;
      for (; q < len && text[q] != ' ' && text[q] != '\n'; ++q) {
        if (text[q] == ':') {
          ++colons;
          if (colons == 1) c1 = q;
          else if (colons == 2) { c2 = q; break; }
        }
      }
      if (colons < 2) { *error = 4; c1 = p; c2 = p + 1; }
      if (k < max_tok) keys[k] = xf_murmur64a(text + c1 + 1, c2 - c1 - 1);
      else *error = 3;
      ++k;
    }
  }
}

// text (device) -> CSR (device).  totals[0] = rows, totals[1] = tokens (device, 2 x u32); row_ptr[rows] is
// written by the caller once it knows `rows` (xf_k_parse_finish).
__global__ void xf_k_parse_finish(uint32_t* row_ptr, const uint32_t* totals, uint32_t max_rows) {
  if (threadIdx.x == 0 && blockIdx.x == 0 && totals[0] <= max_rows) row_ptr[totals[0]] = totals[1];
}

int xf_launch_parse(const char* d_text, uint64_t len, XfDevBuf& scratch, uint32_t* d_row_ptr, uint64_t* d_keys,
                    uint8_t* d_labels, uint32_t max_rows, uint32_t max_tok, uint32_t* d_totals, int* d_error,
                    cudaStream_t st) {
  const uint64_t nchunks = (len + XF_PARSE_CHUNK - 1) / XF_PARSE_CHUNK;
  const uint64_t ntiles = (nchunks + 1023) / 1024;
  XF_TRY(scratch.ensure((nchunks * 2 + ntiles * 2 + 4) * sizeof(uint32_t)));
  uint32_t* cnt_rows = scratch.as<uint32_t>();
  uint32_t* cnt_tok = cnt_rows + nchunks;
  uint32_t* tile_rows = cnt_tok + nchunks;
  uint32_t* tile_tok = tile_rows + ntiles;
  if (nchunks == 0) {
    XF_CUDA_TRY(cudaMemsetAsync(d_row_ptr, 0, 4, st));
    return XF_OK;
  }
  const int block = 256;
  const unsigned grid = (unsigned)((nchunks + block - 1) / block);
  xf_k_parse_count<<<grid, block, 0, st>>>(d_text, len, cnt_rows, cnt_tok, nchunks);
  xf_k_scan_tiles<<<(unsigned)ntiles, 1024, 0, st>>>(cnt_rows, cnt_tok, nchunks, tile_rows, tile_tok);
  xf_k_scan_tile_totals<<<1, 32, 0, st>>>(tile_rows, tile_tok, (uint32_t)ntiles, d_totals);
  xf_k_parse_emit<<<grid, block, 0, st>>>(d_text, len, cnt_rows, cnt_tok, tile_rows, tile_tok, nchunks, max_rows,
                                           max_tok, d_row_ptr, d_keys, d_labels, d_error);
  xf_k_parse_finish<<<1, 32, 0, st>>>(d_row_ptr, d_totals, max_rows);
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

// Exact training-state checkpoint of one table: xf_table_save_state / xf_table_load_state (semantics and file format in
// include/xflow_b200.h).
//
// The image is the table's own bytes: every live row as it lies in its slot, with its slot index and stamp.  Nothing
// is re-probed on either side, so the loaded table is byte-identical to the saved one, and nothing depends on where
// a key lies.  The rows are streamed through bounded staging, one chunk of `chunk_slots` slots at a time:
//   save  xf_k_state_count  live rows per tile of XF_ST_TILE slots
//         xf_k_state_pack   each tile's base = the sum of the counts before it (an exclusive scan of at most a few
//                           thousand counts, which every block recomputes); the live rows go to the device staging in
//                           slot order, read and written with 16-byte accesses, and the chunk's checksum is summed
//         while chunk i+1 is packed, chunk i is copied to one of two pinned buffers and chunk i-1 is written to the file
//   load  chunk i+1 is read from the file while chunk i is copied to the device and scattered into its slots of a
//         freshly filled table (xf_k_state_unpack), which sums the checksum of what it read
// The checksum of a section is the integer sum, mod 2^64, of splitmix64(word ^ offset) over its 8-byte words: any
// order of adds gives it, so the kernels sum it with atomics.  A load verifies every section before the table sees
// any of it: everything is built in new allocations, and the table adopts them only when all checks have passed.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "internal.h"

#define XF_ST_TILE 1024                     // slots per block of the pack kernels
#define XF_ST_VERSION 1u

// The file header (little-endian, 232 bytes; the layout is documented in include/xflow_b200.h)
struct XfStateHeader {
  char magic[4];           //   0 "XFST"
  uint32_t version;        //   4
  uint64_t header_bytes;   //   8 sizeof(XfStateHeader)
  uint64_t capacity;       //  16 slots
  uint64_t cap_floor;      //  24
  uint64_t n_keys;         //  32
  uint32_t stride;         //  40 bytes per row
  uint32_t log2cap;        //  44
  uint32_t bshift;         //  48 bucket shift of the probe sequence
  uint32_t lazy;           //  52 1: lazy LR rows
  int32_t latent_dim;      //  56
  int32_t optimizer;       //  60
  float alpha, beta, lambda1, lambda2, learning_rate;  // 64 .. 83
  int32_t v_init;          //  84 resolved: 0 constant, 1 counter-based normal, 3 zero
  uint64_t seed;           //  88
  int32_t shard_index;     //  96
  int32_t num_shards;      // 100
  int32_t canonical_fm;    // 104
  uint32_t seq;            // 108 lazy tables: the batch number of the last batch in the pending-step ring
  uint64_t batches;        // 112 training batches run
  uint64_t rejected_tokens;  // 120
  uint64_t admitted_keys;  // 128
  int32_t admit_mode;      // 136
  float admit_probability; // 140
  uint32_t admit_threshold;   // 144
  uint32_t admit_log2_cells;  // 148
  uint32_t admit_hashes;   // 152
  uint32_t tracking;       // 156 1: eviction stamps
  uint64_t admit_decay_batches;  // 160
  uint64_t admit_seed;     // 168
  uint64_t evict_max_idle_batches;  // 176
  uint64_t evict_max_keys; // 184
  uint64_t user;           // 192
  uint64_t chunk_slots;    // 200 slots per chunk of the rows section
  uint64_t filter_bytes;   // 208 Bloom filter cells (0: no filter section)
  uint64_t ring_entries;   // 216 lazy tables: seq + 1 (0: no ring section)
  uint64_t header_checksum;  // 224 over bytes [0, 224)
};
static_assert(sizeof(XfStateHeader) == 232, "the documented header is 232 bytes");
static_assert(offsetof(XfStateHeader, batches) == 112 && offsetof(XfStateHeader, user) == 192 &&
                  offsetof(XfStateHeader, header_checksum) == 224,
              "header layout");
#define XF_ST_CHUNK_HEAD 32  // {u64 first_slot, u64 live rows, u64 checksum, u64 0}

uint64_t xf_st_host_sum(const void* p, uint64_t bytes, uint64_t off0) {
  const uint8_t* b = (const uint8_t*)p;
  uint64_t s = 0;
  for (uint64_t i = 0; i + 8 <= bytes; i += 8) {
    uint64_t w;
    memcpy(&w, b + i, 8);
    s += xf_st_hash(w, off0 + i);
  }
  return s;
}

int xf_save_atomic(const char* path, const std::function<int(FILE* f, const char* name)>& body) {
  const std::string tmp = std::string(path) + ".tmp";
  FILE* f = fopen(tmp.c_str(), "wb");
  if (!f) { xf_set_error("cannot open %s for writing", tmp.c_str()); return XF_ERR_IO; }
  int rc = body(f, tmp.c_str());
  if (fclose(f) != 0 && rc == XF_OK) { xf_set_error("write to %s failed", tmp.c_str()); rc = XF_ERR_IO; }
  if (rc == XF_OK && rename(tmp.c_str(), path) != 0) { xf_set_error("cannot rename %s to %s", tmp.c_str(), path); rc = XF_ERR_IO; }
  if (rc != XF_OK) remove(tmp.c_str());
  return rc;
}

// the project's file formats: what each is, the call that writes it and the call that loads it
static const struct { char magic[5]; const char *kind, *save, *load; } xf_file_formats[] = {
    {"XFTB", "portable training checkpoint", "xf_table_save", "xf_table_load"},
    {"XFST", "training state checkpoint", "xf_table_save_state", "xf_table_load_state"},
    {"XFSM", "serving model", "xf_model_save", "xf_model_load"},
    {"XFSP", "serving model part", "xf_model_save", "xf_model_load"},
    {"XFSD", "serving model delta", "xf_delta_save", "xf_delta_load"},
};

int xf_refuse_foreign(const void* head, size_t got, const char* path, const char* own) {
  if (got < 4) return XF_OK;
  for (size_t o = 0; own[o]; o += 4)
    if (memcmp(head, own + o, 4) == 0) return XF_OK;
  const char* own_kind = "";
  for (const auto& x : xf_file_formats)
    if (memcmp(x.magic, own, 4) == 0) own_kind = x.kind;
  for (const auto& x : xf_file_formats)
    if (memcmp(head, x.magic, 4) == 0) {
      xf_set_error("%s is a %s written by %s (%s), not a %s: load it with %s", path, x.kind, x.save, x.magic, own_kind, x.load);
      return XF_ERR_IO;
    }
  return XF_OK;
}

__device__ __forceinline__ unsigned long long xf_st_warp_sum(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// live rows of tile blockIdx.x of the chunk [first, first + n_slots)
__global__ void __launch_bounds__(256) xf_k_state_count(XfTableView t, uint64_t first, uint32_t n_slots,
                                                        uint32_t* __restrict__ tile_live) {
  __shared__ uint32_t cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  uint32_t c = 0;
  for (uint32_t j = threadIdx.x; j < XF_ST_TILE; j += blockDim.x) {
    const uint32_t r = blockIdx.x * XF_ST_TILE + j;
    if (r < n_slots) c += *reinterpret_cast<const uint64_t*>(xf_row(t, first + r)) != XF_EMPTY_KEY ? 1u : 0u;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31u) == 0u) atomicAdd(&cnt, c);
  __syncthreads();
  if (threadIdx.x == 0) tile_live[blockIdx.x] = cnt;
}

// The live rows of the chunk in slot order: rows[n][stride] then meta[n] = slot | stamp << 32 at `out`;
// meta_out = {n, checksum of the payload}.  256 threads, XF_ST_TILE slots per block.
__global__ void __launch_bounds__(256) xf_k_state_pack(XfTableView t, const uint32_t* __restrict__ stamp, uint64_t first,
                                                       uint32_t n_slots, uint32_t n_tiles,
                                                       const uint32_t* __restrict__ tile_live, uint64_t tag,
                                                       uint8_t* __restrict__ out,
                                                       unsigned long long* __restrict__ meta_out) {
  __shared__ int16_t idx[XF_ST_TILE];  // a slot's position among the tile's live rows, -1: empty
  __shared__ uint32_t warp_tot[8];
  __shared__ uint32_t s_base, s_total;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_base = 0; s_total = 0; }
  __syncthreads();
  // this tile's base and the chunk's total from the tiles' counts
  uint32_t before = 0, all = 0;
  for (uint32_t b = threadIdx.x; b < n_tiles; b += blockDim.x) {
    const uint32_t v = tile_live[b];
    all += v;
    if (b < blockIdx.x) before += v;
  }
  before = __reduce_add_sync(0xffffffffu, before);
  all = __reduce_add_sync(0xffffffffu, all);
  if (lane == 0) { atomicAdd(&s_base, before); atomicAdd(&s_total, all); }
  // each thread's four consecutive slots, and their exclusive scan over the block
  const uint32_t tile0 = blockIdx.x * XF_ST_TILE;
  const uint32_t j0 = threadIdx.x * 4u;
  bool live[4];
  uint32_t c = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t r = tile0 + j0 + k;
    live[k] = r < n_slots && *reinterpret_cast<const uint64_t*>(xf_row(t, first + r)) != XF_EMPTY_KEY;
    c += live[k] ? 1u : 0u;
  }
  uint32_t incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += y;
  }
  if (lane == 31u) warp_tot[warp] = incl;
  __syncthreads();
  uint32_t woff = 0;
  for (uint32_t w = 0; w < warp; ++w) woff += warp_tot[w];
  uint32_t pos = woff + incl - c;
#pragma unroll
  for (int k = 0; k < 4; ++k) idx[j0 + k] = live[k] ? (int16_t)(pos++) : (int16_t)-1;
  __syncthreads();
  const uint64_t base = s_base, total = s_total;
  const uint32_t q = t.stride / 16u;
  unsigned long long sum = 0;
  // the rows, 16 bytes per thread and access: consecutive threads read consecutive bytes of the table
  for (uint32_t j = threadIdx.x; j < XF_ST_TILE * q; j += blockDim.x) {
    const uint32_t r = j / q, c16 = j - r * q;
    const int d = idx[r];
    if (d < 0) continue;
    const uint4 v = *reinterpret_cast<const uint4*>(xf_row(t, first + tile0 + r) + 16u * c16);
    const uint64_t off = (base + (uint64_t)d) * t.stride + 16u * c16;
    *reinterpret_cast<uint4*>(out + off) = v;
    sum += xf_st_hash((uint64_t)v.x | ((uint64_t)v.y << 32), tag | off) +
           xf_st_hash((uint64_t)v.z | ((uint64_t)v.w << 32), tag | (off + 8));
  }
  // the slots and stamps
  uint64_t* meta = reinterpret_cast<uint64_t*>(out + total * t.stride);
  for (uint32_t j = threadIdx.x; j < XF_ST_TILE; j += blockDim.x) {
    const int d = idx[j];
    if (d < 0) continue;
    const uint64_t slot = first + tile0 + j;
    const uint64_t m = slot | ((uint64_t)(stamp != nullptr ? stamp[slot] : 0u) << 32);
    meta[base + d] = m;
    sum += xf_st_hash(m, tag | (total * t.stride + (base + (uint64_t)d) * 8u));
  }
  sum = xf_st_warp_sum(sum);
  if (lane == 0) atomicAdd(meta_out + 1, sum);
  if (blockIdx.x == 0 && threadIdx.x == 0) meta_out[0] = total;
}

// Scatter the n rows of a chunk payload (rows[n][stride], meta[n]) into their slots of `t` (and their stamps), summing
// the checksum of what was read into *sum.  A slot outside the chunk [first, first + chunk_slots) sets *bad and is
// skipped: a damaged file never writes outside the table.
__global__ void __launch_bounds__(256) xf_k_state_unpack(XfTableView t, uint32_t* __restrict__ stamp,
                                                         const uint8_t* __restrict__ in, uint64_t n, uint64_t first,
                                                         uint64_t chunk_slots, uint64_t tag,
                                                         unsigned long long* __restrict__ sum_out, int* __restrict__ bad) {
  const uint32_t q = t.stride / 16u;
  const uint64_t* meta = reinterpret_cast<const uint64_t*>(in + n * t.stride);
  const uint64_t items = n * q;
  unsigned long long sum = 0;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < items; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t r = j / q;
    const uint32_t c16 = (uint32_t)(j - r * q);
    const uint64_t off = r * t.stride + 16u * c16;
    const uint4 v = *reinterpret_cast<const uint4*>(in + off);
    sum += xf_st_hash((uint64_t)v.x | ((uint64_t)v.y << 32), tag | off) +
           xf_st_hash((uint64_t)v.z | ((uint64_t)v.w << 32), tag | (off + 8));
    const uint64_t m = meta[r];
    if (c16 == 0) sum += xf_st_hash(m, tag | (n * t.stride + r * 8u));
    const uint64_t slot = (uint32_t)m;
    if (slot < first || slot >= first + chunk_slots || slot > t.mask) {
      if (c16 == 0) *bad = 1;
      continue;
    }
    *reinterpret_cast<uint4*>(xf_row(t, slot) + 16u * c16) = v;
    if (c16 == 0 && stamp != nullptr) stamp[slot] = (uint32_t)(m >> 32);
  }
  sum = xf_st_warp_sum(sum);
  if ((threadIdx.x & 31u) == 0) atomicAdd(sum_out, sum);
}

// checksum of n_words 8-byte words at p, offsets off0, off0 + 8, ... (the Bloom filter section)
__global__ void __launch_bounds__(256) xf_k_state_sum(const uint64_t* __restrict__ p, uint64_t n_words, uint64_t off0,
                                                      unsigned long long* __restrict__ sum_out) {
  unsigned long long sum = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += (uint64_t)gridDim.x * blockDim.x)
    sum += xf_st_hash(p[i], off0 + i * 8u);
  sum = xf_st_warp_sum(sum);
  if ((threadIdx.x & 31u) == 0) atomicAdd(sum_out, sum);
}

// -------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------
// slots per chunk: the largest power of two whose staging (rows + one u64 each) fits XF_ST_CHUNK_BYTES, at least one
// tile, at most the table
static uint64_t xf_st_chunk_slots(uint32_t stride, uint64_t capacity) {
  uint64_t c = XF_ST_TILE;
  while (c * 2 <= capacity && c * 2 * (stride + 8ull) <= XF_ST_CHUNK_BYTES) c *= 2;
  return std::min(c, capacity);
}

// The staging of one save or load: two device chunks, two pinned chunks, a copy stream, events and a few counters.
// Its memory is bounded by the chunk size, whatever the size of the table.
struct XfStateIo {
  uint8_t* dev[2] = {nullptr, nullptr};
  uint8_t* pin[2] = {nullptr, nullptr};
  uint32_t* d_tiles[2] = {nullptr, nullptr};
  unsigned long long* d_small = nullptr;  // {n, checksum} x 2 chunks, rows checksum, filter checksum, error flag
  unsigned long long* h_small = nullptr;
  cudaStream_t copy = nullptr;
  cudaStream_t work = nullptr;                 // the table's stream, which runs the kernels
  cudaEvent_t done[2] = {nullptr, nullptr};    // the kernel of the chunk in dev[b] has finished
  cudaEvent_t copied[2] = {nullptr, nullptr};  // the copy between dev[b] and pin[b] has finished
  size_t bytes = 0;
  ~XfStateIo() {
    if (work) cudaStreamSynchronize(work);
    if (copy) cudaStreamSynchronize(copy);
    for (int b = 0; b < 2; ++b) {
      if (done[b]) cudaEventSynchronize(done[b]);
      if (dev[b]) cudaFree(dev[b]);
      if (pin[b]) cudaFreeHost(pin[b]);
      if (d_tiles[b]) cudaFree(d_tiles[b]);
      if (done[b]) cudaEventDestroy(done[b]);
      if (copied[b]) cudaEventDestroy(copied[b]);
    }
    if (d_small) cudaFree(d_small);
    if (h_small) cudaFreeHost(h_small);
    if (copy) cudaStreamDestroy(copy);
  }
  int init(size_t chunk_bytes, uint32_t n_tiles, cudaStream_t st) {
    bytes = chunk_bytes;
    work = st;
    for (int b = 0; b < 2; ++b) {
      if (cudaMalloc(&dev[b], chunk_bytes) != cudaSuccess || cudaHostAlloc(&pin[b], chunk_bytes, cudaHostAllocDefault) != cudaSuccess ||
          cudaMalloc(&d_tiles[b], (size_t)n_tiles * 4) != cudaSuccess) {
        cudaGetLastError();
        xf_set_error("cannot allocate the checkpoint staging (2 x %zu bytes of device and of page-locked memory)", chunk_bytes);
        return XF_ERR_CUDA;
      }
    }
    if (cudaMalloc(&d_small, 8 * sizeof(unsigned long long)) != cudaSuccess ||
        cudaHostAlloc(&h_small, 8 * sizeof(unsigned long long), cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      xf_set_error("cannot allocate the checkpoint counters");
      return XF_ERR_CUDA;
    }
    XF_CUDA_TRY(cudaMemsetAsync(d_small, 0, 8 * sizeof(unsigned long long), st));
    XF_CUDA_TRY(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
    for (int b = 0; b < 2; ++b) {
      XF_CUDA_TRY(cudaEventCreateWithFlags(&done[b], cudaEventDisableTiming));
      XF_CUDA_TRY(cudaEventCreateWithFlags(&copied[b], cudaEventDisableTiming));
    }
    return XF_OK;
  }
};

static bool xf_st_write(FILE* f, const void* p, size_t n) { return n == 0 || fwrite(p, 1, n, f) == n; }
static bool xf_st_read(FILE* f, void* p, size_t n) { return n == 0 || fread(p, 1, n, f) == n; }

// everything after the header is opened: the sections of an image of `t`, whose header is `h`
static int xf_st_save_body(xf_table* t, const XfStateHeader& h, FILE* f, const char* path) {
  const uint64_t cap = h.capacity, C = h.chunk_slots, nch = cap / C;
  const uint32_t stride = h.stride, n_tiles = (uint32_t)(C / XF_ST_TILE);
  if (!xf_st_write(f, &h, sizeof(h))) { xf_set_error("write to %s failed", path); return XF_ERR_IO; }
  if (h.ring_entries) {
    std::vector<uint64_t> ring(h.ring_entries);
    XF_CUDA_TRY(cudaMemcpy(ring.data(), t->d_rows_by_seq, ring.size() * 8, cudaMemcpyDeviceToHost));
    const uint64_t s = xf_st_host_sum(ring.data(), ring.size() * 8, 0);
    if (!xf_st_write(f, ring.data(), ring.size() * 8) || !xf_st_write(f, &s, 8)) { xf_set_error("write to %s failed", path); return XF_ERR_IO; }
  }
  XfStateIo io;
  XF_TRY(io.init((size_t)C * (stride + 8ull), n_tiles, t->stream));
  cudaStream_t st = t->stream;
  uint64_t n_of[2] = {0, 0}, sum_of[2] = {0, 0}, written = 0;
  // iteration i: pack chunk i on the device, copy chunk i-1 to the host, write chunk i-2 to the file
  for (uint64_t i = 0; i < nch + 2; ++i) {
    if (i < nch) {
      const int b = (int)(i & 1);
      if (i >= 2) XF_CUDA_TRY(cudaStreamWaitEvent(st, io.copied[b], 0));  // chunk i-2 has left dev[b]
      XF_CUDA_TRY(cudaMemsetAsync(io.d_small + 2 * b, 0, 16, st));
      xf_k_state_count<<<n_tiles, 256, 0, st>>>(t->view, i * C, (uint32_t)C, io.d_tiles[b]);
      xf_k_state_pack<<<n_tiles, 256, 0, st>>>(t->view, t->d_stamp, i * C, (uint32_t)C, n_tiles, io.d_tiles[b],
                                               xf_st_tag(i), io.dev[b], io.d_small + 2 * b);
      t->launches += 2;
      XF_CUDA_TRY(cudaGetLastError());
      XF_CUDA_TRY(cudaMemcpyAsync(io.h_small + 2 * b, io.d_small + 2 * b, 16, cudaMemcpyDeviceToHost, st));
      XF_CUDA_TRY(cudaEventRecord(io.done[b], st));
    }
    if (i >= 1 && i - 1 < nch) {
      const int b = (int)((i - 1) & 1);
      XF_CUDA_TRY(cudaEventSynchronize(io.done[b]));
      n_of[b] = io.h_small[2 * b];
      sum_of[b] = io.h_small[2 * b + 1];
      if (n_of[b] > C) { xf_set_error("internal error: chunk %llu packed %llu rows", (unsigned long long)(i - 1), (unsigned long long)n_of[b]); return XF_ERR_STATE; }
      XF_CUDA_TRY(cudaMemcpyAsync(io.pin[b], io.dev[b], n_of[b] * (stride + 8ull), cudaMemcpyDeviceToHost, io.copy));
      XF_CUDA_TRY(cudaEventRecord(io.copied[b], io.copy));
    }
    if (i >= 2) {
      const int b = (int)(i & 1);
      XF_CUDA_TRY(cudaEventSynchronize(io.copied[b]));
      const uint64_t head[4] = {(i - 2) * C, n_of[b], sum_of[b], 0ull};
      if (!xf_st_write(f, head, sizeof(head)) || !xf_st_write(f, io.pin[b], n_of[b] * (stride + 8ull))) {
        xf_set_error("write to %s failed", path);
        return XF_ERR_IO;
      }
      written += n_of[b];
    }
  }
  if (written != h.n_keys) {
    xf_set_error("internal error: the image holds %llu rows, the table %llu keys", (unsigned long long)written,
                 (unsigned long long)h.n_keys);
    return XF_ERR_STATE;
  }
  if (h.filter_bytes) {
    // the filter needs no packing: it goes from the device to the pinned buffers as it is, chunk by chunk
    const uint64_t fc = std::min<uint64_t>(h.filter_bytes, (uint64_t)1 << (63 - __builtin_clzll(io.bytes)));
    const uint64_t nf = h.filter_bytes / fc;
    xf_k_state_sum<<<xf_grid_for(h.filter_bytes / 8, 256, 8), 256, 0, st>>>(
        reinterpret_cast<const uint64_t*>(t->d_filter), h.filter_bytes / 8, 0ull, io.d_small + 5);
    ++t->launches;
    XF_CUDA_TRY(cudaGetLastError());
    for (uint64_t j = 0; j < nf + 1; ++j) {
      if (j < nf) {
        const int b = (int)(j & 1);
        XF_CUDA_TRY(cudaMemcpyAsync(io.pin[b], t->d_filter + j * fc, fc, cudaMemcpyDeviceToHost, st));
        XF_CUDA_TRY(cudaEventRecord(io.copied[b], st));
      }
      if (j >= 1) {
        const int b = (int)((j - 1) & 1);
        XF_CUDA_TRY(cudaEventSynchronize(io.copied[b]));
        if (!xf_st_write(f, io.pin[b], fc)) { xf_set_error("write to %s failed", path); return XF_ERR_IO; }
      }
    }
    uint64_t s = 0;
    XF_CUDA_TRY(cudaMemcpyAsync(&s, io.d_small + 5, 8, cudaMemcpyDeviceToHost, st));
    XF_CUDA_TRY(cudaStreamSynchronize(st));
    if (!xf_st_write(f, &s, 8)) { xf_set_error("write to %s failed", path); return XF_ERR_IO; }
  }
  return XF_OK;
}

XF_DLL int xf_table_save_state(xf_table* t, const char* path, uint64_t user) {
  if (!t || !path) { xf_set_error("null argument"); return XF_ERR_ARG; }
  std::lock_guard<std::mutex> host_lock(t->host_mu);
  XF_CUDA_TRY(cudaSetDevice(t->cfg.device));
  XF_TRY(t->check_error());  // waits for everything enqueued on the table's stream; a table that overflowed is not saved
  unsigned long long size = 0, counters[2] = {0ull, 0ull};
  XF_CUDA_TRY(cudaMemcpy(&size, t->d_size, sizeof(size), cudaMemcpyDeviceToHost));
  if (t->d_admit) XF_CUDA_TRY(cudaMemcpy(counters, t->d_admit, sizeof(counters), cudaMemcpyDeviceToHost));
  XfStateHeader h;
  memset(&h, 0, sizeof(h));
  memcpy(h.magic, "XFST", 4);
  h.version = XF_ST_VERSION;
  h.header_bytes = sizeof(h);
  h.capacity = t->view.mask + 1;
  h.cap_floor = t->cap_floor;
  h.n_keys = size;
  h.stride = t->view.stride;
  h.log2cap = t->view.log2cap;
  h.bshift = t->view.bshift;
  h.lazy = (uint32_t)t->view.lazy;
  h.latent_dim = t->cfg.latent_dim;
  h.optimizer = t->cfg.optimizer;
  h.alpha = t->cfg.alpha; h.beta = t->cfg.beta; h.lambda1 = t->cfg.lambda1; h.lambda2 = t->cfg.lambda2;
  h.learning_rate = t->cfg.learning_rate;
  h.v_init = t->view.v_init;
  h.seed = t->cfg.seed;
  h.shard_index = t->cfg.shard_index;
  h.num_shards = t->cfg.num_shards;
  h.canonical_fm = t->cfg.canonical_fm;
  h.seq = t->view.lazy ? t->seq : 0u;
  h.batches = t->admit_batches;
  h.rejected_tokens = counters[0];
  h.admitted_keys = counters[1];
  h.admit_mode = t->admit.mode;
  h.admit_probability = t->admit.probability;
  h.admit_threshold = t->admit.threshold;
  h.admit_log2_cells = t->admit.log2_cells;
  h.admit_hashes = t->admit.hashes;
  h.admit_decay_batches = t->admit.decay_batches;
  h.admit_seed = t->admit.seed;
  h.tracking = t->d_stamp != nullptr ? 1u : 0u;
  h.evict_max_idle_batches = t->evict.max_idle_batches;
  h.evict_max_keys = t->evict.max_keys;
  h.user = user;
  h.chunk_slots = xf_st_chunk_slots(h.stride, h.capacity);
  h.filter_bytes = (t->admit.mode == XF_ADMIT_BLOOM && t->d_filter) ? (1ull << t->admit.log2_cells) : 0ull;
  h.ring_entries = t->view.lazy ? (uint64_t)t->seq + 1 : 0ull;
  h.header_checksum = xf_st_host_sum(&h, offsetof(XfStateHeader, header_checksum), 0);
  return xf_save_atomic(path, [&](FILE* f, const char* name) { return xf_st_save_body(t, h, f, name); });
}

// -------------------------------------------------------------------------------------------------
// load
// -------------------------------------------------------------------------------------------------
// XF_ERR_ARG naming the first field in which the image and the table `t` differ
static int xf_st_match(const xf_table* t, const XfStateHeader& h) {
  const xf_table_config& c = t->cfg;
  auto fbits = [](float x) { uint32_t u; memcpy(&u, &x, 4); return u; };
  const char* field = nullptr;
  if (h.latent_dim != c.latent_dim) field = "latent_dim";
  else if (h.optimizer != c.optimizer) field = "optimizer";
  else if (fbits(h.alpha) != fbits(c.alpha)) field = "alpha";
  else if (fbits(h.beta) != fbits(c.beta)) field = "beta";
  else if (fbits(h.lambda1) != fbits(c.lambda1)) field = "lambda1";
  else if (fbits(h.lambda2) != fbits(c.lambda2)) field = "lambda2";
  else if (fbits(h.learning_rate) != fbits(c.learning_rate)) field = "learning_rate";
  else if (h.v_init != t->view.v_init) field = "v_init";
  else if (h.seed != c.seed) field = "seed";
  else if (h.shard_index != c.shard_index) field = "shard_index";
  else if (h.num_shards != c.num_shards) field = "num_shards";
  else if (h.canonical_fm != c.canonical_fm) field = "canonical_fm";
  else if (h.stride != t->view.stride) field = "row stride";
  else if (h.lazy != (uint32_t)t->view.lazy) field = "row layout (lazy or eager)";
  else if (h.bshift != xf_bucket_shift(t->view.stride, h.log2cap)) field = "bucket shift";
  if (!field) return XF_OK;
  xf_set_error("xf_table_load_state: the image's %s differs from the table's", field);
  return XF_ERR_ARG;
}

// the header's own consistency (after its checksum): every size derived from it is bounded before it is used
static bool xf_st_header_sane(const XfStateHeader& h) {
  const bool pow2 = h.capacity >= 1024 && h.capacity <= (1ull << 31) && (h.capacity & (h.capacity - 1)) == 0;
  if (!pow2 || (1ull << h.log2cap) != h.capacity || h.n_keys > h.capacity || h.stride < 32 || h.stride % 32 != 0) return false;
  if (h.chunk_slots != xf_st_chunk_slots(h.stride, h.capacity)) return false;
  if (h.cap_floor > (1ull << 31)) return false;
  if (h.admit_mode == XF_ADMIT_BLOOM) {
    if (h.admit_log2_cells < 10 || h.admit_log2_cells > 36 || h.filter_bytes != (1ull << h.admit_log2_cells)) return false;
    if (h.admit_hashes < 1 || h.admit_hashes > XF_ADM_MAX_HASHES || h.admit_threshold < 1 || h.admit_threshold > 255) return false;
  } else if (h.filter_bytes != 0 || (h.admit_mode != XF_ADMIT_ALL && h.admit_mode != XF_ADMIT_POISSON)) {
    return false;
  }
  if (h.ring_entries != (h.lazy ? (uint64_t)h.seq + 1 : 0ull) || h.tracking > 1) return false;
  return true;
}

// what a load allocates; freed unless the table adopts it
struct XfStateNew {
  uint8_t* base = nullptr;
  uint32_t* stamp = nullptr;
  uint8_t* filter = nullptr;
  unsigned long long* admit = nullptr;
  ~XfStateNew() {
    if (base) cudaFree(base);
    if (stamp) cudaFree(stamp);
    if (filter) cudaFree(filter);
    if (admit) cudaFree(admit);
  }
};

static int xf_st_load_body(xf_table* t, FILE* f, const char* path, const XfStateHeader& h, XfStateNew& nw,
                           std::vector<uint64_t>& ring) {
  // the sizes the header announces must add up to the file's size before anything is allocated from them
  const uint64_t C = h.chunk_slots, nch = h.capacity / C, per = h.stride + 8ull;
  const uint64_t expect = sizeof(XfStateHeader) + (h.ring_entries ? h.ring_entries * 8 + 8 : 0) + nch * XF_ST_CHUNK_HEAD +
                          h.n_keys * per + (h.filter_bytes ? h.filter_bytes + 8 : 0);
  if (fseek(f, 0, SEEK_END) != 0) { xf_set_error("cannot read %s", path); return XF_ERR_IO; }
  const long fsz = ftell(f);
  if (fsz < 0 || (uint64_t)fsz != expect) {
    xf_set_error("corrupt or truncated state image %s: %ld bytes, its header announces %llu", path, fsz, (unsigned long long)expect);
    return XF_ERR_IO;
  }
  if (fseek(f, sizeof(XfStateHeader), SEEK_SET) != 0) { xf_set_error("cannot read %s", path); return XF_ERR_IO; }
  if (h.ring_entries) {
    if (h.ring_entries > t->rows_cap) {
      xf_set_error("xf_table_load_state: the image's batch-number ring position %u does not fit this table's ring of %zu "
                   "(XFLOW_SEQ_RING)", h.seq, t->rows_cap);
      return XF_ERR_ARG;
    }
    ring.resize(h.ring_entries);
    uint64_t s = 0;
    if (!xf_st_read(f, ring.data(), ring.size() * 8) || !xf_st_read(f, &s, 8)) { xf_set_error("truncated state image %s", path); return XF_ERR_IO; }
    if (s != xf_st_host_sum(ring.data(), ring.size() * 8, 0)) {
      xf_set_error("state image %s: checksum mismatch in the batch-number ring section", path);
      return XF_ERR_IO;
    }
  }
  // the new table, its stamps, filter and counters
  if (cudaMalloc(&nw.base, h.capacity * (uint64_t)h.stride) != cudaSuccess ||
      (h.tracking && cudaMalloc(&nw.stamp, h.capacity * sizeof(uint32_t)) != cudaSuccess) ||
      (h.filter_bytes && cudaMalloc(&nw.filter, h.filter_bytes) != cudaSuccess) ||
      (!t->d_admit && cudaMalloc(&nw.admit, 4 * sizeof(unsigned long long)) != cudaSuccess)) {
    cudaGetLastError();
    xf_set_error("cannot allocate a table of %llu slots for the state image %s", (unsigned long long)h.capacity, path);
    return XF_ERR_CUDA;
  }
  XfTableView v = t->view;
  v.base = nw.base;
  v.mask = h.capacity - 1;
  v.log2cap = h.log2cap;
  v.bshift = h.bshift;
  cudaStream_t st = t->stream;
  xf_launch_fill(v, st);
  ++t->launches;
  // a stamp of a slot without a key is never read; zeros keep the memory defined
  if (nw.stamp) XF_CUDA_TRY(cudaMemsetAsync(nw.stamp, 0, h.capacity * sizeof(uint32_t), st));
  XfStateIo io;
  XF_TRY(io.init((size_t)C * per, (uint32_t)(C / XF_ST_TILE), st));
  unsigned long long* d_rows_sum = io.d_small + 4;
  unsigned long long* d_filter_sum = io.d_small + 5;
  int* d_bad = reinterpret_cast<int*>(io.d_small + 6);
  uint64_t stated = 0, total = 0;
  // iteration i: read chunk i from the file while chunk i-1 is copied and scattered on the device
  for (uint64_t i = 0; i < nch; ++i) {
    const int b = (int)(i & 1);
    if (i >= 2) XF_CUDA_TRY(cudaEventSynchronize(io.copied[b]));  // chunk i-2 has left pin[b]
    uint64_t head[4];
    if (!xf_st_read(f, head, sizeof(head))) { xf_set_error("truncated state image %s", path); return XF_ERR_IO; }
    if (head[0] != i * C || head[1] > C || head[3] != 0 || total + head[1] > h.n_keys) {
      xf_set_error("state image %s: chunk %llu of the rows section is damaged", path, (unsigned long long)i);
      return XF_ERR_IO;
    }
    const uint64_t n = head[1];
    if (!xf_st_read(f, io.pin[b], n * per)) { xf_set_error("truncated state image %s", path); return XF_ERR_IO; }
    stated += head[2];
    total += n;
    if (i >= 2) XF_CUDA_TRY(cudaStreamWaitEvent(io.copy, io.done[b], 0));  // chunk i-2 has been scattered from dev[b]
    XF_CUDA_TRY(cudaMemcpyAsync(io.dev[b], io.pin[b], n * per, cudaMemcpyHostToDevice, io.copy));
    XF_CUDA_TRY(cudaEventRecord(io.copied[b], io.copy));
    XF_CUDA_TRY(cudaStreamWaitEvent(st, io.copied[b], 0));
    if (n) {
      xf_k_state_unpack<<<xf_grid_for(n * (h.stride / 16), 256, 8), 256, 0, st>>>(v, nw.stamp, io.dev[b], n, i * C, C,
                                                                                  xf_st_tag(i), d_rows_sum, d_bad);
      ++t->launches;
      XF_CUDA_TRY(cudaGetLastError());
    }
    XF_CUDA_TRY(cudaEventRecord(io.done[b], st));
  }
  if (total != h.n_keys) { xf_set_error("state image %s: the rows section holds %llu rows, its header announces %llu", path, (unsigned long long)total, (unsigned long long)h.n_keys); return XF_ERR_IO; }
  uint64_t filter_stated = 0;
  if (h.filter_bytes) {
    const uint64_t fc = std::min<uint64_t>(h.filter_bytes, (uint64_t)1 << (63 - __builtin_clzll(io.bytes)));
    const uint64_t nf = h.filter_bytes / fc;
    for (uint64_t j = 0; j < nf; ++j) {
      const int b = (int)(j & 1);
      XF_CUDA_TRY(cudaEventSynchronize(io.copied[b]));  // the copy that last read pin[b] has finished
      if (!xf_st_read(f, io.pin[b], fc)) { xf_set_error("truncated state image %s", path); return XF_ERR_IO; }
      XF_CUDA_TRY(cudaMemcpyAsync(nw.filter + j * fc, io.pin[b], fc, cudaMemcpyHostToDevice, io.copy));
      XF_CUDA_TRY(cudaEventRecord(io.copied[b], io.copy));
    }
    if (!xf_st_read(f, &filter_stated, 8)) { xf_set_error("truncated state image %s", path); return XF_ERR_IO; }
    XF_CUDA_TRY(cudaEventRecord(io.done[0], io.copy));
    XF_CUDA_TRY(cudaStreamWaitEvent(st, io.done[0], 0));
    xf_k_state_sum<<<xf_grid_for(h.filter_bytes / 8, 256, 8), 256, 0, st>>>(reinterpret_cast<const uint64_t*>(nw.filter),
                                                                            h.filter_bytes / 8, 0ull, d_filter_sum);
    ++t->launches;
    XF_CUDA_TRY(cudaGetLastError());
  }
  XF_CUDA_TRY(cudaMemcpyAsync(io.h_small + 4, io.d_small + 4, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  XF_CUDA_TRY(cudaStreamSynchronize(io.copy));
  if (io.h_small[6] != 0 || io.h_small[4] != stated) {
    xf_set_error("state image %s: checksum mismatch in the rows section", path);
    return XF_ERR_IO;
  }
  if (h.filter_bytes && io.h_small[5] != filter_stated) {
    xf_set_error("state image %s: checksum mismatch in the admission filter section", path);
    return XF_ERR_IO;
  }
  return XF_OK;
}

XF_DLL int xf_table_load_state(xf_table* t, const char* path, uint64_t* user) {
  if (!t || !path) { xf_set_error("null argument"); return XF_ERR_ARG; }
  std::lock_guard<std::mutex> host_lock(t->host_mu);
  XF_CUDA_TRY(cudaSetDevice(t->cfg.device));
  XF_TRY(t->check_error());
  unsigned long long size = 0;
  XF_CUDA_TRY(cudaMemcpy(&size, t->d_size, sizeof(size), cudaMemcpyDeviceToHost));
  if (size != 0 || t->admit_batches != 0) {
    xf_set_error("xf_table_load_state needs a table that has never held state (this one has %llu keys and has run %llu "
                 "training batches)", size, (unsigned long long)t->admit_batches);
    return XF_ERR_STATE;
  }
  FILE* f = fopen(path, "rb");
  if (!f) { xf_set_error("cannot open %s", path); return XF_ERR_IO; }
  XfStateHeader h;
  memset(&h, 0, sizeof(h));
  const size_t got = fread(&h, 1, sizeof(h), f);
  int rc = XF_OK;
  if (xf_refuse_foreign(h.magic, got, path, "XFST") != XF_OK) {
    rc = XF_ERR_IO;
  } else if (got < 4 || memcmp(h.magic, "XFST", 4) != 0) {
    xf_set_error("%s is not a state image (no XFST magic)", path);
    rc = XF_ERR_IO;
  } else if (got != sizeof(h) || h.header_bytes != sizeof(h) || h.version != XF_ST_VERSION) {
    xf_set_error("state image %s: truncated header or unknown version %u", path, h.version);
    rc = XF_ERR_IO;
  } else if (h.header_checksum != xf_st_host_sum(&h, offsetof(XfStateHeader, header_checksum), 0) || !xf_st_header_sane(h)) {
    xf_set_error("state image %s: the header is damaged (checksum mismatch)", path);
    rc = XF_ERR_IO;
  }
  if (rc == XF_OK) rc = xf_st_match(t, h);
  XfStateNew nw;
  std::vector<uint64_t> ring;
  if (rc == XF_OK) rc = xf_st_load_body(t, f, path, h, nw, ring);
  fclose(f);
  if (rc != XF_OK) {
    cudaStreamSynchronize(t->stream);  // nothing in flight may still write the allocations about to be freed
    return rc;
  }
  // every check has passed: the table adopts the image
  if (h.ring_entries) XF_CUDA_TRY(cudaMemcpy(t->d_rows_by_seq, ring.data(), ring.size() * 8, cudaMemcpyHostToDevice));
  if (nw.admit) { t->d_admit = nw.admit; nw.admit = nullptr; }
  const unsigned long long counters[4] = {h.rejected_tokens, h.admitted_keys, 0ull, 0ull};
  XF_CUDA_TRY(cudaMemcpy(t->d_admit, counters, sizeof(counters), cudaMemcpyHostToDevice));
  const unsigned long long n_keys = h.n_keys;
  XF_CUDA_TRY(cudaMemcpy(t->d_size, &n_keys, sizeof(n_keys), cudaMemcpyHostToDevice));
  cudaFree(t->view.base);
  if (t->d_stamp) cudaFree(t->d_stamp);
  if (t->d_filter) cudaFree(t->d_filter);
  t->view.base = nw.base;
  t->view.mask = h.capacity - 1;
  t->view.log2cap = h.log2cap;
  t->view.bshift = h.bshift;
  t->d_stamp = nw.stamp;
  t->d_filter = nw.filter;
  nw.base = nullptr; nw.stamp = nullptr; nw.filter = nullptr;
  xf_admission_config_default(&t->admit);
  t->admit.mode = h.admit_mode;
  t->admit.probability = h.admit_probability;
  t->admit.threshold = h.admit_threshold;
  t->admit.log2_cells = h.admit_log2_cells;
  t->admit.hashes = h.admit_hashes;
  t->admit.decay_batches = h.admit_decay_batches;
  t->admit.seed = h.admit_seed;
  t->evict.max_idle_batches = h.tracking ? h.evict_max_idle_batches : 0;
  t->evict.max_keys = h.tracking ? h.evict_max_keys : 0;
  t->admit_batches = h.batches;
  t->cap_floor = h.cap_floor;
  if (t->view.lazy) t->seq = h.seq;
  // ensure_room's bound restarts from the exact count, as after an eviction sweep
  t->size_bound = h.n_keys;
  t->known_size = h.n_keys;
  t->known_at = t->cum_incoming;
  for (int i = 0; i < 4; ++i) t->size_inflight[i] = false;
  if (user) *user = h.user;
  return XF_OK;
}

// the policies a table runs (the CLI compares a resumed table's with its environment)
int xf_table_policies(xf_table* t, xf_admission_config* admit, xf_eviction_config* evict, int* tracking) {
  if (!t) return XF_ERR_ARG;
  if (admit) *admit = t->admit;
  if (evict) *evict = t->evict;
  if (tracking) *tracking = t->d_stamp != nullptr;
  return XF_OK;
}

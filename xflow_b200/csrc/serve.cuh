// Serving model internals shared by serve.cu (freeze, predict, the XFSM file) and delta.cu (diff, apply, the XFSD file):
// the model's host structure, the device functions that read and build its rows, the host steps both use and the
// chunked sections of their files.  The kernels behind the host steps live in serve.cu only.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <mutex>

#include "internal.h"

// what a model's rows hold (xf_model::fm, xf_model_info::fm, the files' fm field)
enum { XF_SERVE_LR = 0, XF_SERVE_FM = 1, XF_SERVE_FMC = 2, XF_SERVE_MVM = 3, XF_SERVE_FFM = 4 };
// rows {key, word 8, v[K], 0...}: the canonical FM's and the field-aware FM's (word 8: w) and the multi-view machine's
// (word 8: 0, no linear term)
__host__ __device__ inline bool xf_serve_latent_rows(int fm) {
  return fm == XF_SERVE_FMC || fm == XF_SERVE_MVM || fm == XF_SERVE_FFM;
}

struct xf_model {
  XfTableView view{};      // base / mask / log2cap / bshift / stride of the model's rows; K, v_init, v_const, seed of the source;
                           // canon = 1 for canonical rows
  int device = 0;
  int fm = 0, absent = 0, optimizer = 0;  // fm: XF_SERVE_*
  int precision = XF_PRECISION_F32;       // of the latent fields (FM st, qt; canonical v): XF_PRECISION_*
  int shard_index = 0, num_shards = 0;    // a part (xf_table_freeze_part): shard_index of num_shards >= 1; 0: a whole model
  uint64_t keys = 0, source_keys = 0, pruned_keys = 0;
  cudaStream_t stream = nullptr;
  // staging of the host entry points, grown on demand; those calls are serialised by the mutex
  std::mutex mu;
  XfDevBuf s_keys, s_out, s_aux;  // s_aux: a host batch's upload image (xf_model_upload), or a lookup's outputs
  XfPinBuf h_in, h_out;
};

// the keys shard s of S owns (xf_shard_of, postoffice.cc:134-143): [s width, (s + 1) width) with width =
// floor((2^64 - 1) / S); the last shard runs to 2^64 - 2.  *lo and *hi are inclusive.
inline void xf_shard_range(int s, int S, uint64_t* lo, uint64_t* hi) {
  const uint64_t width = 0xFFFFFFFFFFFFFFFFull / (uint64_t)(S > 1 ? S : 1);
  *lo = (uint64_t)s * width;
  *hi = s + 1 >= S ? 0xFFFFFFFFFFFFFFFEull : (uint64_t)(s + 1) * width - 1ull;
}

// XF_ERR_STATE for a part passed where a whole model is needed (predict, diff, apply)
inline int xf_refuse_part(const xf_model* m, const char* fn) {
  if (m->num_shards == 0) return XF_OK;
  xf_set_error("%s: the model is a part (shard %d of %d), not a model: merge the parts with xf_model_merge", fn,
               m->shard_index, m->num_shards);
  return XF_ERR_STATE;
}

// what defines how an absent key reads: the fields two models (a model and a delta, the parts of a merge) must agree on
// (and on the layout of their rows: precision)
struct XfCompat {
  int fm, latent_dim, optimizer, absent, v_init;
  float v_const;
  uint64_t seed;
  int precision;
};
inline XfCompat xf_compat_of(const xf_model* m) {
  return XfCompat{m->fm, m->view.K, m->optimizer, m->absent, m->view.v_init, m->view.v_const, m->view.seed, m->precision};
}
// the first field that differs, or nullptr
inline const char* xf_compat_diff(const XfCompat& a, const XfCompat& b) {
  if (a.fm != b.fm) return "fm";
  if (a.latent_dim != b.latent_dim) return "latent_dim";
  if (a.precision != b.precision) return "precision";
  if (a.optimizer != b.optimizer) return "optimizer";
  if (a.absent != b.absent) return "absent";
  if (a.v_init != b.v_init) return "v_init";
  if (memcmp(&a.v_const, &b.v_const, sizeof(float)) != 0) return "v_const";
  if (a.seed != b.seed) return "seed";
  return nullptr;
}

// Bytes of a model row.  F32: LR {key, w, 0}: 16; FM {key, w, st, qt, 0...}: 32; canonical FM {key, w, 0, v[K], 0...}:
// 16 + 4K rounded up to 32, so that every row starts on a sector and lane c's piece v[4c .. 4c+3] lies at 16 + 16c.
// F16 (FM and canonical only; w stays float32): FM {key, w, st, qt}: 16, no padding; canonical {key, w, 0, v[K], 0...}:
// 16 + 2K rounded up to 32, lane c's piece at 16 + 8c.  A multi-view machine's row {key, u64 0, v[K], 0...} is the
// canonical one with w = 0; a field-aware FM's row is the canonical one.
__host__ __device__ inline uint32_t xf_model_row_bytes(int fm, int K, int precision) {
  const uint32_t vb = precision == XF_PRECISION_F16 ? 2u : 4u;
  if (xf_serve_latent_rows(fm)) return (16u + vb * (uint32_t)K + 31u) & ~31u;
  if (fm == XF_SERVE_FM) return precision == XF_PRECISION_F16 ? 16u : 32u;
  return 16u;
}
// the latent dimensions a canonical model serves: C = K / 4 lanes per token, a power of two <= 32
inline bool xf_fmc_latent_ok(int K) { return K == 4 || K == 8 || K == 16 || K == 32 || K == 64 || K == 128; }
// those a multi-view machine's model serves: the ones its trainer takes (step_mvm.cu, XF_MVM_K_MAX)
inline bool xf_mvm_latent_ok(int K) { return K == 4 || K == 8 || K == 16 || K == 32; }
// A packed row of a model (fm, K, precision, row_bytes) has zero bytes where its layout has padding: LR [12, 16); FM
// [20, 32) at F32, none at F16; canonical [12, 16) and [16 + 4K, row_bytes) at F32, [16 + 2K, row_bytes) at F16; a
// multi-view machine's as the canonical one's, and [8, 12) too; a field-aware FM's as the canonical one's.  Every model
// in memory keeps them zero (the fill writes them, freeze and convert write fields only, the other passes copy whole
// rows), so that whole rows compare and hash as their fields do.  Checked a word at a time: the 4-byte word after w (LR, canonical; for a multi-view machine's row
// the word of w too) or qt (FM), then 8-byte words to the row's end.
inline bool xf_model_padding_zero(const uint8_t* p, int fm, int K, int precision, uint32_t row_bytes) {
  if (fm == XF_SERVE_FM && precision == XF_PRECISION_F16) return true;
  const uint32_t vb = precision == XF_PRECISION_F16 ? 2u : 4u;
  uint32_t w4;
  memcpy(&w4, p + (fm == XF_SERVE_FM ? 20 : 12), 4);
  uint64_t any = w4;
  if (fm == XF_SERVE_MVM) {
    memcpy(&w4, p + 8, 4);
    any |= w4;
  }
  for (uint32_t b = xf_serve_latent_rows(fm) ? 16u + vb * (uint32_t)K : fm == XF_SERVE_FM ? 24u : 16u; b < row_bytes; b += 8) {
    uint64_t x;
    memcpy(&x, p + b, 8);
    any |= x;
  }
  return any == 0;
}
// a binary16 field's bits (the low 16 of x) widened to float32, exactly
__device__ __forceinline__ float xf_h2f(uint32_t x) { return __half2float(__ushort_as_half((unsigned short)(x & 0xFFFFu))); }

// ---- model rows: read-only for the lifetime of every kernel that looks keys up, hence the non-coherent path
// H: an F16 FM row {key, w, st, qt} of 16 bytes, one load as for LR, its fields widened after the load
template <bool FM, bool H = false>
__device__ __forceinline__ void xf_serve_load(const uint8_t* p, uint64_t& key, float& w, float& st, float& qt) {
  uint64_t q0, q1, q2 = 0ull, q3 = 0ull;
  if (FM && !H) {
    // one sector as two 128-bit loads by the same lane (sm_90 has no 256-bit load), issued back to back
    asm("ld.global.nc.v2.u64 {%0,%1}, [%4];\n\tld.global.nc.v2.u64 {%2,%3}, [%4+16];"
        : "=l"(q0), "=l"(q1), "=l"(q2), "=l"(q3) : "l"(p));
  } else {
    asm("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(q0), "=l"(q1) : "l"(p));
  }
  key = q0;
  w = __uint_as_float((uint32_t)q1);
  if (H) {
    st = xf_h2f((uint32_t)(q1 >> 32));
    qt = xf_h2f((uint32_t)(q1 >> 48));
  } else {
    st = __uint_as_float((uint32_t)(q1 >> 32));
    qt = __uint_as_float((uint32_t)q2);
  }
}

// Find `key` from its home slot `s`, whose row the caller has loaded into (k, w, st, qt); false: the model does not
// hold it.  The load is at most 0.5, so a chain ends at an empty slot long before XF_MAX_PROBE.
template <bool FM, bool H = false>
__device__ __forceinline__ bool xf_serve_find(const XfTableView& m, uint64_t key, uint64_t k, float& w, float& st, float& qt) {
  for (uint32_t i = 1; i <= XF_MAX_PROBE; ++i) {
    if (k == key) return true;
    if (k == XF_EMPTY_KEY) return false;
    xf_serve_load<FM, H>(xf_row(m, xf_probe_slot(m, key, i)), k, w, st, qt);
  }
  return false;
}

// ---- whole rows: bytes [8, stride) are opaque outside freeze, predict and lookup
// Claim a slot for `key` and return its row, for the caller to write bytes 8 .. stride; nullptr: not claimed.  A probe
// overflow sets *error.  KEEP = false: the inserted keys are unique, and a key met twice sets *error.  KEEP = true: a
// key the model already holds keeps its row, untouched (the caller orders the kernels so that the row it holds is
// complete).
template <bool KEEP = false>
__device__ __forceinline__ uint8_t* xf_model_claim(const XfTableView& m, uint64_t key, int* error) {
  for (uint32_t i = 0; i < XF_MAX_PROBE; ++i) {
    uint8_t* rowp = xf_row(m, xf_probe_slot(m, key, i));
    const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(rowp), (unsigned long long)XF_EMPTY_KEY,
                                             (unsigned long long)key);
    if (old == XF_EMPTY_KEY) return rowp;
    if (old == key) {
      if (KEEP) return nullptr;
      break;
    }
  }
  *error = 1;
  return nullptr;
}
// The row at `src` into the model `m`: `head` is its first 16 bytes {key, word 8}, which the caller has loaded to read
// the key; bytes 16 .. stride follow 16 bytes per access.  Bytes 16 .. 31 (all of an FM row's rest) are loaded before
// the claim, so that their latency overlaps the CAS's.  The claim is xf_model_claim<KEEP>'s.
template <bool KEEP = false>
__device__ __forceinline__ void xf_model_put_row(const XfTableView& m, const uint8_t* src, ulonglong2 head, int* error) {
  const bool wide = m.stride > 16u;
  const uint4 second = wide ? *reinterpret_cast<const uint4*>(src + 16) : make_uint4(0u, 0u, 0u, 0u);
  uint8_t* dst = xf_model_claim<KEEP>(m, head.x, error);
  if (!dst) return;
  *reinterpret_cast<unsigned long long*>(dst + 8) = head.y;
  if (wide) *reinterpret_cast<uint4*>(dst + 16) = second;
  for (uint32_t o = 32; o < m.stride; o += 16)
    *reinterpret_cast<uint4*>(dst + o) = *reinterpret_cast<const uint4*>(src + o);
}
// the slot that holds `key`, or -1: the key words only, through the non-coherent path
__device__ __forceinline__ int64_t xf_model_find_slot(const XfTableView& m, uint64_t key) {
  for (uint32_t i = 0; i < XF_MAX_PROBE; ++i) {
    const uint64_t s = xf_probe_slot(m, key, i);
    const uint64_t k = __ldg(reinterpret_cast<const unsigned long long*>(xf_row(m, s)));
    if (k == key) return (int64_t)s;
    if (k == XF_EMPTY_KEY) return -1;
  }
  return -1;
}

// slots of a model of `keys` keys: the smallest power of two >= 2 x keys (load <= 0.5), at least 1024; keys <= 2^62
inline uint64_t xf_model_capacity(uint64_t keys) {
  uint64_t c = 1024;
  while (c < 2 * keys) c <<= 1;
  return c;
}

// a new model on `device`, which is made current: its stream, and the fields XfCompat describes (precision included)
int xf_model_init(xf_model* m, int device, const XfCompat& c);
// the model's table on the current device: `capacity` empty rows (stride from m->fm, m->view.K, m->precision), filled on
// m->stream;
// XF_ERR_FULL past 2^32 slots
int xf_model_alloc(xf_model* m, uint64_t capacity);
// waits for the model's stream and frees everything (m may be NULL)
void xf_model_free(xf_model* m);

// Rows of a model listed as (key, slot) pairs and sorted by key on the device: the first step of a model file, and of
// a delta's upserts and deletes.  keys_in / slots_in hold the n pairs in any order; the sort leaves them in keys_out /
// slots_out.  Device scratch: 24 bytes per pair and cub's temporary storage.
struct XfSortedSlots {
  XfDevBuf keys_in, keys_out, slots_in, slots_out, tmp, count;
  int ensure(uint64_t n);  // room for n pairs and the list kernels' counter
  void release();
};
// list every row of `v` (capacity v.mask + 1) into s and sort; n = the model's keys
int xf_model_list_sorted(const XfTableView& v, uint64_t n, XfSortedSlots& s, cudaStream_t st);
// sort the n listed pairs of s by key
int xf_sort_slots(XfSortedSlots& s, uint64_t n, cudaStream_t st);
// out = the rows of `v` in slots[0 .. n), packed
int xf_model_gather(const XfTableView& v, const uint32_t* slots, uint64_t n, void* out, cudaStream_t st);
// insert n packed rows (as a model file holds them; keys unique) into `v`; a probe overflow or a key met twice sets
// *error
int xf_model_insert_rows(const XfTableView& v, const uint8_t* rows, uint64_t n, int* error, cudaStream_t st);

// Each request's top k candidates (rank.cu): request q's scores are pctr[cand_ptr[q] .. cand_ptr[q+1]); slots
// [q k, q k + k) of top_index (and of top_pctr, unless NULL) receive its ranked local indices and their scores, padded
// with 0xFFFFFFFF (and the NaN 0x7FC00000).  1 <= k <= XF_RANK_MAX_K.  Reads cand_ptr on the device only; no scratch.
void xf_launch_rank(const float* pctr, const uint32_t* cand_ptr, uint32_t requests, uint32_t k, uint32_t* top_index,
                    float* top_pctr, cudaStream_t st);

// ---- the files' chunked sections (XFSM and XFSP rows, XFSD upserts and delete keys)
// A section of n entries of `bytes` bytes is a sequence of chunks of per_chunk entries (the last may be shorter), each a
// head {u64 first entry, u64 entries, u64 checksum, u64 0} and its entries.  The checksum is xf_st_host_sum over the
// entries, their offsets tagged with the chunk's index in the file (xf_st_tag), which runs on from section to section.
#define XF_CHUNK_HEAD 32
// the section's bytes in the file
inline uint64_t xf_section_bytes(uint64_t n, uint32_t bytes, uint64_t per_chunk) {
  return (n + per_chunk - 1) / per_chunk * XF_CHUNK_HEAD + n * bytes;
}
// Write a section, chunk indices from *chunk on (advanced past it).  src(first, c, &dev) makes entries [first, first + c)
// ready at device address dev on `st`; each chunk is staged through `pin`, summed and written.
int xf_chunks_save(FILE* f, const char* name, uint64_t n, uint32_t bytes, uint64_t per_chunk, uint64_t* chunk, XfPinBuf& pin,
                   cudaStream_t st, const std::function<int(uint64_t first, uint64_t c, const void** dev)>& src);
// What a section's entries must satisfy besides their checksums: each begins with a key, and the keys ascend strictly,
// stay below 2^64 - 1 and lie in shard shard_index of num_shards (xf_shard_range; 0 of 0: any key); entries that are
// rows (fm >= 0: XF_SERVE_*, of latent_dim K and precision) have zero padding (xf_model_padding_zero).  file and what
// name the file and the entries in the errors.
struct XfChunkCheck {
  const char* file;
  const char* what;
  int fm, K, precision;
  int shard_index, num_shards;
};
// Read a section written by xf_chunks_save and check it chunk by chunk (XF_ERR_IO at the first fault), staged through
// `pin`; sink(first, c, host) takes each verified chunk, and `st` is synchronised before the next one is read into `pin`.
int xf_chunks_load(FILE* f, const char* path, uint64_t n, uint32_t bytes, uint64_t per_chunk, uint64_t* chunk,
                   const XfChunkCheck& check, XfPinBuf& pin, cudaStream_t st,
                   const std::function<int(uint64_t first, uint64_t c, const void* host)>& sink);
// XF_ERR_IO unless the file is `expect` bytes long, as its header announces; leaves it positioned at `header_bytes`
int xf_file_size_check(FILE* f, const char* path, const char* file, uint64_t expect, uint64_t header_bytes);
// the fields a model's and a delta's header share: a row kind with its latent_dim, precision (F16: FM and canonical
// only) and row_bytes, and a known absent policy, optimizer and v_init
bool xf_compat_sane(const XfCompat& c, uint32_t row_bytes);

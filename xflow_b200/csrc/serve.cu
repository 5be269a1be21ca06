// Serving model: a trained table frozen for prediction only (layer 6 of include/xflow_b200.h, which documents the
// semantics and the XFSM file format).
//
// A model row holds what the forward pass reads of a key and nothing else: LR {key, w} in 16 bytes, FM of any K
// {key, w, st = sum_k v_k, qt = sum_k v_k^2} in one 32-byte sector (fm_worker.cc:177-196 collapses the interaction over
// k, so a token contributes w, st and qt only, and in a frozen model they are constants).  The model is an
// open-addressing table of such rows with the training table's hash and probe sequence (xf_probe_slot), described by an
// XfTableView whose stride is the model's row size, so that the table's device functions serve both.
//
//   freeze   xf_k_freeze<COUNT>   one pass counts the rows kept, one inserts them (CAS on the key word); each resolves a
//                                 row as a reader does: xf_apply_pending for w, xf_fm_token for st, qt
//   predict  xf_k_serve<FM>       warp per row, two tokens per lane in flight, the mapping and the association of the
//                                 step kernels' forward pass (step.cu, step_lazy.cu), so the result is theirs bit for bit;
//                                 no insert, no atomics, no shared memory
//   file     rows sorted by key (cub radix sort of (key, slot)), gathered a chunk at a time through bounded staging;
//            xf_chunks_save / xf_chunks_load write and check the chunked sections of XFSM, XFSP and XFSD;
//            load: xf_k_model_insert_rows
//
// Outside freeze, predict and lookup a row is {key, body}: the other passes (here xf_k_model_insert_rows and xf_k_merge,
// in delta.cu fingerprint, diff and apply) copy, compare or hash bytes [8, stride) whole, one kernel for every row kind.
//
// A part (xf_table_freeze_part) is what xf_k_freeze makes of one shard table, whose counting pass also counts the keys
// outside the shard's range; its file is XFSP.  xf_model_merge makes the whole model of S parts:
//   merge    xf_k_merge            a grid-stride walk over a part's slots in place (or a 64 MiB chunk of them peer-copied
//                                  from another device), each live row put whole with xf_model_put_row
//
// A canonical model (xf_table_freeze_canonical, fm = XF_SERVE_FMC) serves the textbook FM with feature values
// (step_fmc.cu), whose per-k sums do not collapse: its row is {key, w, 0, v[K]} padded to a multiple of 32 bytes.
//   freeze   xf_k_freeze_fmc<COUNT>  the same two passes; v is the row's latent block or its initial values
//   predict  xf_k_serve_fmc<C>       xf_k_step_fmc's mapping (C = K/4 lanes per token), its per-lane order and its
//                                    arithmetic (forward.cuh: xf_fmc_add, xf_fmc_arg); the C lanes of a token load the
//                                    head and their 16-byte piece of the home slot at once; two passes in flight
//
// A multi-view machine's model (xf_table_freeze_mvm, fm = XF_SERVE_MVM) serves step_mvm.cu's forward on field ids and
// feature values: its row is the canonical one with w = 0, {key, 0, v[K]} (the machine has no linear term).
//   freeze   xf_k_freeze_fmc<COUNT, true>  v resolved as for a canonical model, w neither written nor pruned on
//   predict  xf_k_serve_mvm<C>             xf_k_serve_fmc's mapping, loads and probe; the per-(field, k) sums in shared
//                                          memory, added in token order without atomics: a pass's tokens of one field
//                                          are ranked with __match_any_sync and added a rank per round
//
// A field-aware FM's model (xf_table_freeze_ffm, fm = XF_SERVE_FFM) serves step_ffm.cu's forward on field ids and
// feature values: its row is the canonical one, piece c of v the key's vector for field c.
//   freeze   xf_k_freeze_fmc<COUNT, false>  the canonical freeze
//   predict  xf_k_serve_ffm<C>              xf_k_serve_fmc's mapping, loads and probe; the field sums T[F][F] in dynamic
//                                           shared memory, in token order, with xf_k_step_ffm's arithmetic (forward.cuh:
//                                           xf_ffm_add, xf_ffm_arg)
//
// An F16 model (xf_model_convert) holds its latent fields in binary16: FM {key, w, st, qt} in 16 bytes, canonical
// {key, w, 0, v[K]} with 2-byte v.  Its predict and lookup kernels are the F32 ones' H = true instantiations, which widen
// each field right after the load and then run the F32 arithmetic unchanged.
//   convert  xf_k_model_convert<FMC, TO_HALF>  a grid-stride walk over the source's slots as xf_k_merge's; each live row
//                                              converted and put into the result with xf_model_claim
//
// Each row kind's forward is a token loop and a finishing step: xf_serve_arg (LR, FM), xf_fmc_arg (canonical),
// xf_mvm_product (multi-view machine), xf_ffm_arg (field-aware FM), each written once; the last three are forward.cuh's,
// shared with the training steps.  A flat predict kernel runs the
// loop over each row's token indices.  A candidate kernel (xf_k_serve_cand*) runs it as a fold over positions
// (xf_serve_fold, xf_fmc_fold, xf_mvm_fold, xf_ffm_fold): once over a request's context, then over each candidate's
// tokens from that state (see "Two forms of each fold").  xf_launch_predict and xf_launch_candidates pick the instantiation (xf_with_precision, xf_with_lanes); the
// host entry points upload a batch as one image (xf_model_upload).
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cub/cub.cuh>
#include <mutex>
#include <vector>

#include "serve.cuh"
#include "forward.cuh"

#define XF_SM_VERSION 1u

// The file header (little-endian, 104 bytes; the layout is documented in include/xflow_b200.h)
struct XfModelHeader {
  char magic[4];           //   0 "XFSM"
  uint32_t version;        //   4
  uint64_t header_bytes;   //   8
  uint64_t keys;           //  16
  uint64_t capacity;       //  24
  uint32_t row_bytes;      //  32
  int32_t fm;              //  36
  int32_t latent_dim;      //  40
  int32_t optimizer;       //  44
  int32_t absent;          //  48
  int32_t v_init;          //  52 resolved
  float v_const;           //  56
  uint32_t precision;      //  60 XF_PRECISION_* (reserved as 0 before F16 models)
  uint64_t seed;           //  64
  uint64_t source_keys;    //  72
  uint64_t pruned_keys;    //  80
  uint64_t chunk_rows;     //  88
  uint64_t header_checksum;  // 96 over bytes [0, 96)
};
static_assert(sizeof(XfModelHeader) == 104 && offsetof(XfModelHeader, seed) == 64 &&
                  offsetof(XfModelHeader, header_checksum) == 96,
              "the documented header is 104 bytes");

// A part file "XFSP" (112 bytes): XFSM's header with its own magic, bytes [0, 96) as XFSM's, then the shard
struct XfPartHeader {
  uint8_t model[96];         //   0 XFSM's fields up to chunk_rows, magic "XFSP", header_bytes 112
  int32_t shard_index;       //  96
  int32_t num_shards;        // 100
  uint64_t header_checksum;  // 104 over bytes [0, 104)
};
static_assert(sizeof(XfPartHeader) == 112 && offsetof(XfPartHeader, header_checksum) == 104,
              "the documented part header is 112 bytes");

// one token's terms into the lane's sums, in the order the step kernels add them
template <bool FM, bool H>
__device__ __forceinline__ void xf_serve_token(const XfTableView& m, int absent, uint64_t key, uint64_t k, float w, float st,
                                               float qt, float& wsum, float& ssum, float& qsum) {
  if (!xf_serve_find<FM, H>(m, key, k, w, st, qt)) {
    if (absent == XF_ABSENT_ZERO) return;
    // the row the table would insert: w = 0 and, FM, a latent block that is not materialised
    w = 0.f;
    if (FM) xf_fm_token<1>(m, 0u, 0u, key, st, qt);
  }
  wsum += w;
  if (FM) { ssum += st; qsum += qt; }
}

// Two forms of each fold.  Each row kind's loop over a row's tokens is written twice: as a fold over positions
// (xf_serve_fold, xf_fmc_fold, xf_mvm_fold), which the candidate kernels run from a context's state, and in the flat
// kernel over token indices [beg, end).  Both give every token the same lane and order, so both compute the same bits.
// They stay apart because each form compiles well only for its own kernels.  As a call to the fold, a flat kernel widens
// keys + beg + p in two steps: on an H100 80GB HBM3 (700 W) the flat LR kernel took 1 - 3 % longer, and
// xf_k_serve_mvm<C, true> needed 48 registers instead of 40 at C = 2 and 4.  Rewriting the folds in token indices would
// change the candidate kernels' code instead.  A change to one form's arithmetic is a change to both.

// The positions [lo, hi) of a row whose token at position p is keys[beg + p - lo] into the lane's sums: lane l takes the
// positions = l (mod 32) in increasing order, two in flight, as xf_k_serve.  A candidate's tokens follow its context's
// n_c at [n_c mod 64, n_c mod 64 + n), each on the lane the flat row gives it.
template <bool FM, bool H>
__device__ __forceinline__ void xf_serve_fold(const XfTableView& m, int absent, const uint64_t* __restrict__ keys,
                                              uint32_t beg, uint32_t lo, uint32_t hi, float& wsum, float& ssum,
                                              float& qsum) {
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t p0 = lo & ~63u; p0 < hi; p0 += 64u) {
    const uint32_t pa = p0 + lane, pb = pa + 32u;
    const bool v0 = pa >= lo && pa < hi, v1 = pb >= lo && pb < hi;
    const uint64_t k0 = v0 ? __ldcs(keys + beg + (pa - lo)) : 0ull;  // streaming: do not displace model rows in L2
    const uint64_t k1 = v1 ? __ldcs(keys + beg + (pb - lo)) : 0ull;
    // both first looks are in flight before either is resolved
    uint64_t a = XF_EMPTY_KEY, b = XF_EMPTY_KEY;
    float wa = 0.f, sa = 0.f, qa = 0.f, wb = 0.f, sb = 0.f, qb = 0.f;
    if (v0) xf_serve_load<FM, H>(xf_row(m, xf_home_slot(m, k0)), a, wa, sa, qa);
    if (v1) xf_serve_load<FM, H>(xf_row(m, xf_home_slot(m, k1)), b, wb, sb, qb);
    if (v0) xf_serve_token<FM, H>(m, absent, k0, a, wa, sa, qa, wsum, ssum, qsum);
    if (v1) xf_serve_token<FM, H>(m, absent, k1, b, wb, sb, qb, wsum, ssum, qsum);
  }
}

// the lanes' sums reduced over the warp, then wx + (S·S - Q) op by op (fm_worker.cc:193-196): the sigmoid's argument
template <bool FM>
__device__ __forceinline__ float xf_serve_arg(float wsum, float ssum, float qsum) {
  const float wx = xf_warp_sum(wsum);
  if (!FM) return wx;
  const float S = xf_warp_sum(ssum);
  const float Q = xf_warp_sum(qsum);
  return __fadd_rn(wx, __fsub_rn(__fmul_rn(S, S), Q));
}

template <bool FM, bool H>
__global__ void __launch_bounds__(256)
xf_k_serve(XfTableView m, int absent, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys, int B,
           float* __restrict__ pctr_out) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * warps_per_block;
  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    const int chunks = (int)((end - beg + 63u) >> 6);
    float wsum = 0.f, ssum = 0.f, qsum = 0.f;
    // xf_serve_fold over [0, n) in token indices (see "Two forms of each fold" above)
    for (int ch = 0; ch < chunks; ++ch) {
      const uint32_t j0 = beg + (uint32_t)ch * 64u + (uint32_t)lane;
      const uint32_t j1 = j0 + 32u;
      const bool v0 = j0 < end, v1 = j1 < end;
      const uint64_t k0 = v0 ? __ldcs(keys + j0) : 0ull;
      const uint64_t k1 = v1 ? __ldcs(keys + j1) : 0ull;
      uint64_t a = XF_EMPTY_KEY, b = XF_EMPTY_KEY;
      float wa = 0.f, sa = 0.f, qa = 0.f, wb = 0.f, sb = 0.f, qb = 0.f;
      if (v0) xf_serve_load<FM, H>(xf_row(m, xf_home_slot(m, k0)), a, wa, sa, qa);
      if (v1) xf_serve_load<FM, H>(xf_row(m, xf_home_slot(m, k1)), b, wb, sb, qb);
      if (v0) xf_serve_token<FM, H>(m, absent, k0, a, wa, sa, qa, wsum, ssum, qsum);
      if (v1) xf_serve_token<FM, H>(m, absent, k1, b, wb, sb, qb, wsum, ssum, qsum);
    }
    const float arg = xf_serve_arg<FM>(wsum, ssum, qsum);
    if (lane == 0) pctr_out[row] = xf_sigmoid(arg);
  }
}

// ---- canonical rows {key, w, 0, v[K]}: the forward of xf_k_step_fmc (mode 1) on the model's rows
// A token's head {key, w} and lane c's latent piece v[4c .. 4c+3] of the row at p, as two non-coherent loads issued
// back to back (the C lanes of a token load the same head: one request).  H: the piece is four binary16 values, one
// 8-byte load at 16 + 8c, widened after it.
template <bool H>
__device__ __forceinline__ void xf_fmc_load(const uint8_t* p, int c, uint64_t& key, float& w, float4& v) {
  uint64_t q0, q1;
  if (H) {
    uint32_t h0, h1;
    asm("ld.global.nc.v2.u64 {%0,%1}, [%4];\n\tld.global.nc.v2.u32 {%2,%3}, [%5];"
        : "=l"(q0), "=l"(q1), "=r"(h0), "=r"(h1)
        : "l"(p), "l"(p + 16 + 8 * c));
    v = make_float4(xf_h2f(h0), xf_h2f(h0 >> 16), xf_h2f(h1), xf_h2f(h1 >> 16));
  } else {
    asm("ld.global.nc.v2.u64 {%0,%1}, [%6];\n\tld.global.nc.v4.f32 {%2,%3,%4,%5}, [%7];"
        : "=l"(q0), "=l"(q1), "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
        : "l"(p), "l"(p + 16 + 16 * c));
  }
  key = q0;
  w = __uint_as_float((uint32_t)q1);
}

// Find `key` from its home slot, whose row the caller has loaded into (k, w, v); false: the model does not hold it
template <bool H>
__device__ __forceinline__ bool xf_fmc_find(const XfTableView& m, uint64_t key, uint64_t k, float& w, float4& v, int c) {
  for (uint32_t i = 1; i <= XF_MAX_PROBE; ++i) {
    if (k == key) return true;
    if (k == XF_EMPTY_KEY) return false;
    xf_fmc_load<H>(xf_row(m, xf_probe_slot(m, key, i)), c, k, w, v);
  }
  return false;
}

// one token into the lane's sums: its row found from the home slot the caller loaded (k, w, v), or the absent policy
template <bool H>
__device__ __forceinline__ void xf_fmc_serve_token(const XfTableView& m, int absent, uint64_t key, uint64_t k, float w,
                                                   float4 v, float x, int c, float (&S)[4], float& Q, float& wx) {
  if (!xf_fmc_find<H>(m, key, k, w, v, c)) {
    if (absent == XF_ABSENT_ZERO) return;
    // the row the table would insert: w = 0 and a latent block that is not materialised
    w = 0.f;
    v = xf_v_init_piece(m, key, c);
  }
  xf_fmc_add(v, x, w, c == 0, S, Q, wx);
}

// The positions [lo, hi) of a row whose token at position p is keys[beg + p - lo] (vals NULL: every value 1) into the
// lane's sums: C = K/4 lanes per token, lane group g takes the positions = g (mod T = 32/C) in increasing order, two
// passes in flight, as xf_k_step_fmc.  A candidate's tokens start at its context's n_c mod 2T.
template <int C, bool H>
__device__ __forceinline__ void xf_fmc_fold(const XfTableView& m, int absent, const uint64_t* __restrict__ keys,
                                            const float* __restrict__ vals, uint32_t beg, uint32_t lo, uint32_t hi,
                                            float (&S)[4], float& Q, float& wx) {
  constexpr uint32_t T = 32 / C;
  const int lane = threadIdx.x & 31;
  const int c = lane & (C - 1);
  const uint32_t tg = (uint32_t)(lane / C);
  for (uint32_t p0 = lo & ~(2u * T - 1u); p0 < hi; p0 += 2u * T) {
    const uint32_t pa = p0 + tg, pb = pa + T;
    const bool va = pa >= lo && pa < hi, vb = pb >= lo && pb < hi;
    const uint32_t ja = beg + (pa - lo), jb = beg + (pb - lo);
    // streaming: do not displace model rows in L2
    const uint64_t ka = va ? __ldcs(keys + ja) : 0ull;
    const uint64_t kb = vb ? __ldcs(keys + jb) : 0ull;
    const float xa = (va && vals) ? __ldcs(vals + ja) : 1.0f;
    const float xb = (vb && vals) ? __ldcs(vals + jb) : 1.0f;
    // both home rows are in flight before either is resolved
    uint64_t ra = XF_EMPTY_KEY, rb = XF_EMPTY_KEY;
    float wa = 0.f, wb = 0.f;
    float4 qa = make_float4(0.f, 0.f, 0.f, 0.f), qb = qa;
    if (va) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, ka)), c, ra, wa, qa);
    if (vb) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, kb)), c, rb, wb, qb);
    if (va) xf_fmc_serve_token<H>(m, absent, ka, ra, wa, qa, xa, c, S, Q, wx);
    if (vb) xf_fmc_serve_token<H>(m, absent, kb, rb, wb, qb, xb, c, S, Q, wx);
  }
}

// One warp per row.  A lane adds its tokens in the order of the step kernel's passes, with its arithmetic (xf_fmc_add,
// xf_fmc_arg), so the result is the table's bit for bit.  No insert, no atomics, no shared memory.
template <int C, bool H>
__global__ void __launch_bounds__(256)
xf_k_serve_fmc(XfTableView m, int absent, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
               const float* __restrict__ vals, int B, float* __restrict__ pctr_out) {
  constexpr int T = 32 / C;
  const int lane = threadIdx.x & 31;
  const int c = lane & (C - 1);
  const int tg = lane / C;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * warps_per_block;
  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    float S[4] = {0.f, 0.f, 0.f, 0.f};
    float Q = 0.f, wx = 0.f;
    // xf_fmc_fold over [0, n) in token indices (see "Two forms of each fold" above)
    for (uint32_t j0 = beg; j0 < end; j0 += 2u * T) {
      const uint32_t ja = j0 + (uint32_t)tg, jb = ja + (uint32_t)T;
      const bool va = ja < end, vb = jb < end;
      const uint64_t ka = va ? __ldcs(keys + ja) : 0ull;
      const uint64_t kb = vb ? __ldcs(keys + jb) : 0ull;
      const float xa = (va && vals) ? __ldcs(vals + ja) : 1.0f;
      const float xb = (vb && vals) ? __ldcs(vals + jb) : 1.0f;
      uint64_t ra = XF_EMPTY_KEY, rb = XF_EMPTY_KEY;
      float wa = 0.f, wb = 0.f;
      float4 pa = make_float4(0.f, 0.f, 0.f, 0.f), pb = pa;
      if (va) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, ka)), c, ra, wa, pa);
      if (vb) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, kb)), c, rb, wb, pb);
      if (va) xf_fmc_serve_token<H>(m, absent, ka, ra, wa, pa, xa, c, S, Q, wx);
      if (vb) xf_fmc_serve_token<H>(m, absent, kb, rb, wb, pb, xb, c, S, Q, wx);
    }
    const float arg = xf_fmc_arg(C, S, Q, wx);
    if (lane == 0) pctr_out[row] = xf_sigmoid(arg);
  }
}

// ---- multi-view machine rows {key, 0, v[K]}: the forward of xf_k_step_mvm (mode 1) with its same-field adds in token
// order
// A token's latent piece v[4c .. 4c+3]: its row found from the home slot the caller loaded (k, v), or the absent
// policy's row (DEFAULT: the initial values; ZERO: zeros)
template <bool H>
__device__ __forceinline__ float4 xf_mvm_serve_token(const XfTableView& m, int absent, uint64_t key, uint64_t k, float4 v,
                                                     int c) {
  float w;
  if (xf_fmc_find<H>(m, key, k, w, v, c)) return v;
  if (absent == XF_ABSENT_ZERO) return make_float4(0.f, 0.f, 0.f, 0.f);
  return xf_v_init_piece(m, key, c);
}

// The n tokens of a row from keys[beg] (vals NULL: every value 1) into the warp's sums S, each entry in token order
// (xf_mvm_add), with xf_k_serve_fmc's mapping, loads and probe; returns the lane's fields present (the caller reduces
// them over the warp).  Every token makes its field present: under ZERO an absent key is a row of zeros, it adds 0 x.
template <int C, bool H>
__device__ __forceinline__ unsigned xf_mvm_fold(const XfTableView& m, int absent, const uint64_t* __restrict__ keys,
                                                const uint8_t* __restrict__ fields, const float* __restrict__ vals,
                                                uint32_t beg, uint32_t n, float (*S)[4 * C]) {
  constexpr uint32_t T = 32 / C;
  const int lane = threadIdx.x & 31;
  const int c = lane & (C - 1);
  const uint32_t tg = (uint32_t)(lane / C);
  unsigned present = 0u;
  for (uint32_t i0 = 0; i0 < n; i0 += 2u * T) {
    const uint32_t ia = i0 + tg, ib = ia + T;
    const bool va = ia < n, vb = ib < n;
    const uint32_t ja = beg + ia, jb = beg + ib;
    // streaming: do not displace model rows in L2
    const uint64_t ka = va ? __ldcs(keys + ja) : 0ull;
    const uint64_t kb = vb ? __ldcs(keys + jb) : 0ull;
    const uint32_t fa = va ? (uint32_t)__ldcs(fields + ja) & (XF_MVM_FIELDS - 1) : 0u;
    const uint32_t fb = vb ? (uint32_t)__ldcs(fields + jb) & (XF_MVM_FIELDS - 1) : 0u;
    const float xa = (va && vals) ? __ldcs(vals + ja) : 1.0f;
    const float xb = (vb && vals) ? __ldcs(vals + jb) : 1.0f;
    // both home rows are in flight before either is resolved
    uint64_t ra = XF_EMPTY_KEY, rb = XF_EMPTY_KEY;
    float wa, wb;  // a multi-view machine's row holds no w
    float4 pa = make_float4(0.f, 0.f, 0.f, 0.f), pb = pa;
    if (va) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, ka)), c, ra, wa, pa);
    if (vb) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, kb)), c, rb, wb, pb);
    if (va) pa = xf_mvm_serve_token<H>(m, absent, ka, ra, pa, c);
    if (vb) pb = xf_mvm_serve_token<H>(m, absent, kb, rb, pb, c);
    present |= (va ? 1u << fa : 0u) | (vb ? 1u << fb : 0u);
    xf_mvm_add<4 * C>(S, va, fa, c, pa, xa);  // pass a, then pass b
    xf_mvm_add<4 * C>(S, vb, fb, c, pb, xb);
  }
  return present;
}

// One warp per row; the per-(field, k) sums of the row in shared memory, XF_MVM_FIELDS x K floats per warp as
// xf_k_step_mvm's.  y is the warp sum of the P_k (xf_mvm_product), as in the step kernel; lane k < K then clears the
// present fields' sums for the warp's next row.  No insert, no atomics.
template <int C, bool H>
__global__ void __launch_bounds__(256)
xf_k_serve_mvm(XfTableView m, int absent, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
               const uint8_t* __restrict__ fields, const float* __restrict__ vals, int B, float* __restrict__ pctr_out) {
  constexpr int K = 4 * C;
  constexpr int T = 32 / C;
  __shared__ __align__(16) float s_sum[8][XF_MVM_FIELDS][K];  // K x 128 bytes per warp, at most 4 KB
  const int lane = threadIdx.x & 31;
  const int c = lane & (C - 1);
  const int tg = lane / C;
  const int wib = threadIdx.x >> 5;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + wib;
  const int nwarps = gridDim.x * warps_per_block;
  float (*S)[K] = s_sum[wib];
  if (lane < K)
    for (int f = 0; f < XF_MVM_FIELDS; ++f) S[f][lane] = 0.f;
  __syncwarp();
  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    unsigned present = 0u;
    // xf_mvm_fold over the row in token indices (see "Two forms of each fold" above)
    for (uint32_t j0 = beg; j0 < end; j0 += 2u * T) {
      const uint32_t ja = j0 + (uint32_t)tg, jb = ja + (uint32_t)T;
      const bool va = ja < end, vb = jb < end;
      const uint64_t ka = va ? __ldcs(keys + ja) : 0ull;
      const uint64_t kb = vb ? __ldcs(keys + jb) : 0ull;
      const uint32_t fa = va ? (uint32_t)__ldcs(fields + ja) & (XF_MVM_FIELDS - 1) : 0u;
      const uint32_t fb = vb ? (uint32_t)__ldcs(fields + jb) & (XF_MVM_FIELDS - 1) : 0u;
      const float xa = (va && vals) ? __ldcs(vals + ja) : 1.0f;
      const float xb = (vb && vals) ? __ldcs(vals + jb) : 1.0f;
      uint64_t ra = XF_EMPTY_KEY, rb = XF_EMPTY_KEY;
      float wa, wb;
      float4 pa = make_float4(0.f, 0.f, 0.f, 0.f), pb = pa;
      if (va) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, ka)), c, ra, wa, pa);
      if (vb) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, kb)), c, rb, wb, pb);
      if (va) pa = xf_mvm_serve_token<H>(m, absent, ka, ra, pa, c);
      if (vb) pb = xf_mvm_serve_token<H>(m, absent, kb, rb, pb, c);
      present |= (va ? 1u << fa : 0u) | (vb ? 1u << fb : 0u);
      xf_mvm_add<K>(S, va, fa, c, pa, xa);
      xf_mvm_add<K>(S, vb, fb, c, pb, xb);
    }
    present = __reduce_or_sync(0xffffffffu, present);
    const float P = xf_mvm_product<K>(S, present);
    if (lane < K && present)
      for (unsigned q = present; q; q &= q - 1) S[__ffs(q) - 1][lane] = 0.f;
    __syncwarp();  // the sums are clear before the warp's next row adds to them
    const float y = xf_warp_sum(P);
    if (lane == 0) pctr_out[row] = xf_sigmoid(y);
  }
}

// ---- field-aware FM rows {key, w, 0, v[L]}: the forward of xf_k_step_ffm (pass 1, pair sum, sigmoid) on the model's
// rows, with its arithmetic (xf_ffm_add, xf_ffm_arg).  Piece c of v is the key's vector for field c; F = C = L/4 fields.
// A token's w and piece c: its row found from the home slot the caller loaded (k, w, v), or the absent policy's row
// (DEFAULT: w = 0 and the initial values; ZERO: zeros, its field still present)
template <bool H>
__device__ __forceinline__ void xf_ffm_serve_token(const XfTableView& m, int absent, uint64_t key, uint64_t k, float& w,
                                                   float4& v, int c) {
  if (xf_fmc_find<H>(m, key, k, w, v, c)) return;
  w = 0.f;
  if (absent == XF_ABSENT_ZERO) v = make_float4(0.f, 0.f, 0.f, 0.f);
  else v = xf_v_init_piece(m, key, c);
}

// The n tokens of a row from keys[beg] (vals NULL: every value 1) into the warp's state T, Σwx, Q, with
// xf_k_serve_fmc's mapping, loads and probe, two passes in flight, each added as xf_ffm_add; returns the lane's fields
// present (the caller reduces them over the warp).  Every token makes its field present.
template <int C, bool H>
__device__ __forceinline__ unsigned xf_ffm_fold(const XfTableView& m, int absent, const uint64_t* __restrict__ keys,
                                                const uint8_t* __restrict__ fields, const float* __restrict__ vals,
                                                uint32_t beg, uint32_t n, float4* T, float& wx, float& Q) {
  constexpr uint32_t TP = 32 / C;
  const int lane = threadIdx.x & 31;
  const int c = lane & (C - 1);
  const uint32_t tg = (uint32_t)(lane / C);
  unsigned present = 0u;
  for (uint32_t i0 = 0; i0 < n; i0 += 2u * TP) {
    const uint32_t ia = i0 + tg, ib = ia + TP;
    const bool va = ia < n, vb = ib < n;
    const uint32_t ja = beg + ia, jb = beg + ib;
    // streaming: do not displace model rows in L2
    const uint64_t ka = va ? __ldcs(keys + ja) : 0ull;
    const uint64_t kb = vb ? __ldcs(keys + jb) : 0ull;
    const uint32_t fa = va ? (uint32_t)__ldcs(fields + ja) & (C - 1) : 0u;
    const uint32_t fb = vb ? (uint32_t)__ldcs(fields + jb) & (C - 1) : 0u;
    const float xa = (va && vals) ? __ldcs(vals + ja) : 1.0f;
    const float xb = (vb && vals) ? __ldcs(vals + jb) : 1.0f;
    // both home rows are in flight before either is resolved
    uint64_t ra = XF_EMPTY_KEY, rb = XF_EMPTY_KEY;
    float wa = 0.f, wb = 0.f;
    float4 pa = make_float4(0.f, 0.f, 0.f, 0.f), pb = pa;
    if (va) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, ka)), c, ra, wa, pa);
    if (vb) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, kb)), c, rb, wb, pb);
    if (va) xf_ffm_serve_token<H>(m, absent, ka, ra, wa, pa, c);
    if (vb) xf_ffm_serve_token<H>(m, absent, kb, rb, wb, pb, c);
    present |= (va ? 1u << fa : 0u) | (vb ? 1u << fb : 0u);
    xf_ffm_add<C, true>(T, va, 0, fa, pa, wa, xa, wx, Q);  // pass a, then pass b
    xf_ffm_add<C, true>(T, vb, 0, fb, pb, wb, xb, wx, Q);
  }
  return present;
}

// warps per CTA of the field-aware FM's flat kernel: C = 32 (L = 128) holds 16 KB of field sums per warp, 4 warps per
// CTA (64 KB, opt-in) as xf_k_step_ffm; else 8.  Its candidate kernel holds twice that per warp (T and T0): 2 warps at
// C = 32 (64 KB, opt-in), else 4.
__host__ __device__ constexpr int xf_ffm_warps(int C) { return C == 32 ? 4 : 8; }
__host__ __device__ constexpr int xf_cand_ffm_warps(int C) { return C == 32 ? 2 : 4; }

// One warp per row; the row's field sums in dynamic shared memory, F x F float4 per warp.  After a row, lane b < F
// clears T[a][b] for its present fields a.  No insert, no atomics.
template <int C, bool H>
__global__ void __launch_bounds__(32 * xf_ffm_warps(C))
xf_k_serve_ffm(XfTableView m, int absent, const uint32_t* __restrict__ row_ptr, const uint64_t* __restrict__ keys,
               const uint8_t* __restrict__ fields, const float* __restrict__ vals, int B, float* __restrict__ pctr_out) {
  constexpr int TP = 32 / C;
  extern __shared__ float4 s_ffm[];
  const int lane = threadIdx.x & 31;
  const int c = lane & (C - 1);
  const int tg = lane / C;
  const int wib = threadIdx.x >> 5;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + wib;
  const int nwarps = gridDim.x * warps_per_block;
  float4* T = s_ffm + (size_t)wib * (C * C);
  for (int i = lane; i < C * C; i += 32) T[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncwarp();
  for (int row = gwarp; row < B; row += nwarps) {
    const uint32_t beg = __ldg(row_ptr + row);
    const uint32_t end = __ldg(row_ptr + row + 1);
    unsigned present = 0u;
    float wx = 0.f, Q = 0.f;
    // xf_ffm_fold over the row in token indices (see "Two forms of each fold" above)
    for (uint32_t j0 = beg; j0 < end; j0 += 2u * TP) {
      const uint32_t ja = j0 + (uint32_t)tg, jb = ja + (uint32_t)TP;
      const bool va = ja < end, vb = jb < end;
      const uint64_t ka = va ? __ldcs(keys + ja) : 0ull;
      const uint64_t kb = vb ? __ldcs(keys + jb) : 0ull;
      const uint32_t fa = va ? (uint32_t)__ldcs(fields + ja) & (C - 1) : 0u;
      const uint32_t fb = vb ? (uint32_t)__ldcs(fields + jb) & (C - 1) : 0u;
      const float xa = (va && vals) ? __ldcs(vals + ja) : 1.0f;
      const float xb = (vb && vals) ? __ldcs(vals + jb) : 1.0f;
      uint64_t ra = XF_EMPTY_KEY, rb = XF_EMPTY_KEY;
      float wa = 0.f, wb = 0.f;
      float4 pa = make_float4(0.f, 0.f, 0.f, 0.f), pb = pa;
      if (va) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, ka)), c, ra, wa, pa);
      if (vb) xf_fmc_load<H>(xf_row(m, xf_home_slot(m, kb)), c, rb, wb, pb);
      if (va) xf_ffm_serve_token<H>(m, absent, ka, ra, wa, pa, c);
      if (vb) xf_ffm_serve_token<H>(m, absent, kb, rb, wb, pb, c);
      present |= (va ? 1u << fa : 0u) | (vb ? 1u << fb : 0u);
      xf_ffm_add<C, true>(T, va, 0, fa, pa, wa, xa, wx, Q);
      xf_ffm_add<C, true>(T, vb, 0, fb, pb, wb, xb, wx, Q);
    }
    present = __reduce_or_sync(0xffffffffu, present);
    const float arg = xf_ffm_arg<C>(T, present, wx, Q);
    if (lane == 0) pctr_out[row] = xf_sigmoid(arg);
    // clear the rows of T this row used, for the warp's next row
    __syncwarp();
    if (lane < C)
      for (unsigned q = present; q; q &= q - 1) T[(__ffs(q) - 1) * C + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncwarp();
  }
}

// f(std::bool_constant<H>()) for a model's precision: H = true for binary16 latent fields
template <typename F>
static void xf_with_precision(const xf_model* m, F&& f) {
  if (m->precision == XF_PRECISION_F16) f(std::true_type());
  else f(std::false_type());
}

// the flat forward of any model on device arrays (fields: a multi-view machine's or a field-aware FM's, which read
// nothing else)
static void xf_launch_predict(const xf_model* m, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* fields,
                              const float* vals, uint32_t rows, float* pctr_out, cudaStream_t st) {
  if (rows == 0) return;
  const int grid = xf_grid_for((uint64_t)rows * 32, 256, 8);
  const int B = (int)rows;
  xf_with_precision(m, [&](auto H) {
    if (m->fm == XF_SERVE_FFM)
      xf_with_lanes<32>(m->view.K, [&](auto C) {
        constexpr int block = 32 * xf_ffm_warps(C);
        constexpr size_t smem = (size_t)xf_ffm_warps(C) * C * C * sizeof(float4);
        xf_k_serve_ffm<C, H><<<xf_grid_smem((const void*)xf_k_serve_ffm<C, H>, (uint64_t)rows * 32, block, smem), block,
                               smem, st>>>(m->view, m->absent, row_ptr, keys, fields, vals, B, pctr_out);
      });
    else if (m->fm == XF_SERVE_MVM)
      xf_with_lanes<8>(m->view.K, [&](auto C) {
        xf_k_serve_mvm<C, H><<<grid, 256, 0, st>>>(m->view, m->absent, row_ptr, keys, fields, vals, B, pctr_out);
      });
    else if (m->fm == XF_SERVE_FMC)
      xf_with_lanes<32>(m->view.K, [&](auto C) {
        xf_k_serve_fmc<C, H><<<grid, 256, 0, st>>>(m->view, m->absent, row_ptr, keys, vals, B, pctr_out);
      });
    else if (m->fm) xf_k_serve<true, H><<<grid, 256, 0, st>>>(m->view, m->absent, row_ptr, keys, B, pctr_out);
    else xf_k_serve<false, false><<<grid, 256, 0, st>>>(m->view, m->absent, row_ptr, keys, B, pctr_out);
  });
}

// ---- candidate scoring: a request's context scored against each of its candidates (xf_model_predict_candidates_*)
// Candidate c of request q is the row "context q, then row c".  Every forward above is a per-lane (LR, FM, canonical)
// or per-entry (multi-view machine) left fold over the row's positions in increasing order, so the fold over the context
// is a prefix of the fold over every such row.  A warp folds the context once and starts each candidate's fold from
// that state: candidate token i sits at position n_c + i, on the lane (LR, FM) or lane group (canonical) that the flat
// kernel gives that position, so the result is the flat kernel's on the concatenated row, bit for bit.
//
// Work: the candidates in runs of XF_CAND_RUN, a warp per run.  A run that crosses a request boundary is scored a
// request at a time, each request's context folded once; a warp finds its first request by a binary search over
// cand_ptr.  Nothing is written but pctr_out.
#define XF_CAND_RUN 16u

struct XfCandView {
  const uint32_t* ctx_ptr;
  const uint64_t* ctx_keys;
  const float* ctx_vals;
  const uint8_t* ctx_fields;
  const uint32_t* cand_ptr;
  const uint32_t* row_ptr;
  const uint64_t* keys;
  const float* vals;
  const uint8_t* fields;
  uint32_t requests, candidates;
};

// the request that holds candidate c: the q < R with cand_ptr[q] <= c < cand_ptr[q + 1] (cand_ptr[0] = 0 <= c <
// cand_ptr[R])
__device__ __forceinline__ uint32_t xf_cand_request(const uint32_t* __restrict__ cand_ptr, uint32_t R, uint32_t c) {
  uint32_t lo = 0, hi = R;
  while (hi - lo > 1u) {
    const uint32_t mid = lo + (hi - lo) / 2u;
    if (__ldg(cand_ptr + mid) <= c) lo = mid;
    else hi = mid;
  }
  return lo;
}

// The walk every candidate kernel makes: each run of XF_CAND_RUN candidates, split at request boundaries; for each
// request q met, state = context(q) once, candidate(state, c) for its candidates in the run, then done(state).  The
// state goes by value, so that it stays in registers.
template <typename Ctx, typename Cand, typename Done>
__device__ __forceinline__ void xf_cand_walk(const XfCandView& b, int gwarp, int nwarps, Ctx context, Cand candidate,
                                             Done done) {
  const uint32_t runs = (uint32_t)(((uint64_t)b.candidates + XF_CAND_RUN - 1u) / XF_CAND_RUN);
  for (uint32_t run = (uint32_t)gwarp; run < runs; run += (uint32_t)nwarps) {
    uint32_t c = run * XF_CAND_RUN;
    const uint32_t c_end = b.candidates - c > XF_CAND_RUN ? c + XF_CAND_RUN : b.candidates;
    for (uint32_t q = xf_cand_request(b.cand_ptr, b.requests, c); c < c_end; ++q) {
      const uint32_t last = min(c_end, __ldg(b.cand_ptr + q + 1));
      if (c >= last) continue;  // a request without candidates
      const auto state = context(q);
      for (; c < last; ++c) candidate(state, c);
      done(state);
    }
  }
}

// LR and FM: the context's three sums per lane stay in registers; a candidate's tokens start at position n_c mod 64,
// which puts each on the lane xf_k_serve gives it
template <bool FM, bool H>
__global__ void __launch_bounds__(256)
xf_k_serve_cand(XfTableView m, int absent, XfCandView b, float* __restrict__ pctr_out) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  struct Ctx { float wsum, ssum, qsum; uint32_t lo; };
  xf_cand_walk(b, gwarp, gridDim.x * warps_per_block,
               [=](uint32_t q) {
                 const uint32_t beg = __ldg(b.ctx_ptr + q), n = __ldg(b.ctx_ptr + q + 1) - beg;
                 Ctx x{0.f, 0.f, 0.f, n & 63u};
                 xf_serve_fold<FM, H>(m, absent, b.ctx_keys, beg, 0u, n, x.wsum, x.ssum, x.qsum);
                 return x;
               },
               [=](const Ctx& x, uint32_t c) {
                 const uint32_t beg = __ldg(b.row_ptr + c), n = __ldg(b.row_ptr + c + 1) - beg;
                 float wsum = x.wsum, ssum = x.ssum, qsum = x.qsum;
                 xf_serve_fold<FM, H>(m, absent, b.keys, beg, x.lo, x.lo + n, wsum, ssum, qsum);
                 const float arg = xf_serve_arg<FM>(wsum, ssum, qsum);
                 if (lane == 0) pctr_out[c] = xf_sigmoid(arg);
               },
               [](const Ctx&) {});
}

// canonical: the context's S[4], Q and wx per lane stay in registers; a candidate's tokens start at position
// n_c mod 2T, which puts each on the lane group xf_k_serve_fmc gives it
template <int C, bool H>
__global__ void __launch_bounds__(256)
xf_k_serve_cand_fmc(XfTableView m, int absent, XfCandView b, float* __restrict__ pctr_out) {
  constexpr uint32_t T = 32 / C;
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int gwarp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  struct Ctx { float S[4], Q, wx; uint32_t lo; };
  xf_cand_walk(b, gwarp, gridDim.x * warps_per_block,
               [=](uint32_t q) {
                 const uint32_t beg = __ldg(b.ctx_ptr + q), n = __ldg(b.ctx_ptr + q + 1) - beg;
                 Ctx x{{0.f, 0.f, 0.f, 0.f}, 0.f, 0.f, n & (2u * T - 1u)};
                 xf_fmc_fold<C, H>(m, absent, b.ctx_keys, b.ctx_vals, beg, 0u, n, x.S, x.Q, x.wx);
                 return x;
               },
               [=](const Ctx& x, uint32_t c) {
                 const uint32_t beg = __ldg(b.row_ptr + c), n = __ldg(b.row_ptr + c + 1) - beg;
                 float S[4] = {x.S[0], x.S[1], x.S[2], x.S[3]};
                 float Q = x.Q, wx = x.wx;
                 xf_fmc_fold<C, H>(m, absent, b.keys, b.vals, beg, x.lo, x.lo + n, S, Q, wx);
                 const float arg = xf_fmc_arg(C, S, Q, wx);
                 if (lane == 0) pctr_out[c] = xf_sigmoid(arg);
               },
               [](const Ctx&) {});
}

// Multi-view machine: a warp's working sums S[f][k] and a copy S0 of the context's, both in shared memory (2 x 32 x K
// floats per warp, 4 warps per block: 32 KB at K = 32).  Each candidate adds its tokens to S in token order; then lane
// k < K forms P_k over the fields present in the context or the candidate, as xf_k_serve_mvm, and puts the candidate's
// fields back to the context's sums.  After a request's last candidate in the run, its context's fields are cleared in
// both.  The candidate tokens' lanes do not matter: S is the warp's, each entry a fold in token order.
#define XF_CAND_MVM_WARPS 4
template <int C, bool H>
__global__ void __launch_bounds__(32 * XF_CAND_MVM_WARPS)
xf_k_serve_cand_mvm(XfTableView m, int absent, XfCandView b, float* __restrict__ pctr_out) {
  constexpr int K = 4 * C;
  __shared__ __align__(16) float s_sum[XF_CAND_MVM_WARPS][2][XF_MVM_FIELDS][K];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int gwarp = blockIdx.x * XF_CAND_MVM_WARPS + wib;
  float (*S)[K] = s_sum[wib][0];
  float (*S0)[K] = s_sum[wib][1];
  if (lane < K)
    for (int f = 0; f < XF_MVM_FIELDS; ++f) S[f][lane] = S0[f][lane] = 0.f;
  __syncwarp();
  xf_cand_walk(b, gwarp, gridDim.x * XF_CAND_MVM_WARPS,
               [=](uint32_t q) {
                 const uint32_t beg = __ldg(b.ctx_ptr + q), n = __ldg(b.ctx_ptr + q + 1) - beg;
                 const unsigned ctx_present = __reduce_or_sync(
                     0xffffffffu, xf_mvm_fold<C, H>(m, absent, b.ctx_keys, b.ctx_fields, b.ctx_vals, beg, n, S));
                 __syncwarp();
                 if (lane < K)
                   for (unsigned f = ctx_present; f; f &= f - 1) S0[__ffs(f) - 1][lane] = S[__ffs(f) - 1][lane];
                 return ctx_present;
               },
               [=](unsigned ctx_present, uint32_t c) {
                 const uint32_t beg = __ldg(b.row_ptr + c), n = __ldg(b.row_ptr + c + 1) - beg;
                 __syncwarp();
                 const unsigned own = __reduce_or_sync(0xffffffffu, xf_mvm_fold<C, H>(m, absent, b.keys, b.fields,
                                                                                      b.vals, beg, n, S));
                 __syncwarp();
                 const float P = xf_mvm_product<K>(S, ctx_present | own);
                 // `lane < K` alone would do (own is 0 when nothing is present); with xf_mvm_product's own test
                 // beside it the kernel compiles to the code it had with the product written inline
                 if (lane < K && (ctx_present | own))
                   for (unsigned q = own; q; q &= q - 1) S[__ffs(q) - 1][lane] = S0[__ffs(q) - 1][lane];
                 const float y = xf_warp_sum(P);
                 if (lane == 0) pctr_out[c] = xf_sigmoid(y);
               },
               [=](unsigned ctx_present) {
                 // the context leaves both copies before the warp's next request
                 if (lane < K)
                   for (unsigned f = ctx_present; f; f &= f - 1) S[__ffs(f) - 1][lane] = S0[__ffs(f) - 1][lane] = 0.f;
                 __syncwarp();
               });
}

// Field-aware FM: a warp's working field sums T and a copy T0 of the context's, both in dynamic shared memory (2 F x F
// float4 per warp: 32 KB at L = 128), the context's Σwx, Q and present fields in registers.  Each candidate continues
// the fold from that state, forms the pair sum over the fields present in the context or the candidate, as
// xf_k_serve_ffm, and puts the rows T[f][*] of its own fields back to the context's.  After a request's last candidate
// in the run, its context's rows are cleared in both.  Every part of the state is a left fold in token order, so the
// candidate tokens' lanes do not matter.
template <int C, bool H>
__global__ void __launch_bounds__(32 * xf_cand_ffm_warps(C), 1)
xf_k_serve_cand_ffm(XfTableView m, int absent, XfCandView b, float* __restrict__ pctr_out) {
  constexpr int W = xf_cand_ffm_warps(C);
  extern __shared__ float4 s_ffm[];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int gwarp = blockIdx.x * W + wib;
  float4* T = s_ffm + (size_t)wib * (2 * C * C);
  float4* T0 = T + C * C;
  for (int i = lane; i < 2 * C * C; i += 32) T[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncwarp();
  struct Ctx { float wx, Q; unsigned present; };
  xf_cand_walk(b, gwarp, gridDim.x * W,
               [=](uint32_t q) {
                 const uint32_t beg = __ldg(b.ctx_ptr + q), n = __ldg(b.ctx_ptr + q + 1) - beg;
                 Ctx x{0.f, 0.f, 0u};
                 x.present = __reduce_or_sync(
                     0xffffffffu, xf_ffm_fold<C, H>(m, absent, b.ctx_keys, b.ctx_fields, b.ctx_vals, beg, n, T, x.wx, x.Q));
                 __syncwarp();
                 if (lane < C)
                   for (unsigned f = x.present; f; f &= f - 1) T0[(__ffs(f) - 1) * C + lane] = T[(__ffs(f) - 1) * C + lane];
                 return x;
               },
               [=](const Ctx& x, uint32_t c) {
                 const uint32_t beg = __ldg(b.row_ptr + c), n = __ldg(b.row_ptr + c + 1) - beg;
                 float wx = x.wx, Q = x.Q;
                 __syncwarp();
                 const unsigned own = __reduce_or_sync(
                     0xffffffffu, xf_ffm_fold<C, H>(m, absent, b.keys, b.fields, b.vals, beg, n, T, wx, Q));
                 __syncwarp();
                 const float arg = xf_ffm_arg<C>(T, x.present | own, wx, Q);
                 __syncwarp();  // every lane has read T before its candidate's rows go back
                 if (lane < C)
                   for (unsigned f = own; f; f &= f - 1) T[(__ffs(f) - 1) * C + lane] = T0[(__ffs(f) - 1) * C + lane];
                 if (lane == 0) pctr_out[c] = xf_sigmoid(arg);
               },
               [=](const Ctx& x) {
                 // the context leaves both copies before the warp's next request
                 __syncwarp();
                 if (lane < C)
                   for (unsigned f = x.present; f; f &= f - 1)
                     T[(__ffs(f) - 1) * C + lane] = T0[(__ffs(f) - 1) * C + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
                 __syncwarp();
               });
}

// the candidate forward of any model on device arrays
static void xf_launch_candidates(const xf_model* m, const XfCandView& b, float* pctr_out, cudaStream_t st) {
  if (b.candidates == 0) return;
  const uint64_t warps = ((uint64_t)b.candidates + XF_CAND_RUN - 1u) / XF_CAND_RUN;
  constexpr int MVM_THREADS = 32 * XF_CAND_MVM_WARPS;
  const int grid = m->fm == XF_SERVE_MVM ? xf_grid_for(warps * 32, MVM_THREADS, 16) : xf_grid_for(warps * 32, 256, 8);
  xf_with_precision(m, [&](auto H) {
    if (m->fm == XF_SERVE_FFM)
      xf_with_lanes<32>(m->view.K, [&](auto C) {
        constexpr int block = 32 * xf_cand_ffm_warps(C);
        constexpr size_t smem = (size_t)xf_cand_ffm_warps(C) * 2 * C * C * sizeof(float4);
        xf_k_serve_cand_ffm<C, H><<<xf_grid_smem((const void*)xf_k_serve_cand_ffm<C, H>, warps * 32, block, smem), block,
                                    smem, st>>>(m->view, m->absent, b, pctr_out);
      });
    else if (m->fm == XF_SERVE_MVM)
      xf_with_lanes<8>(m->view.K, [&](auto C) {
        xf_k_serve_cand_mvm<C, H><<<grid, MVM_THREADS, 0, st>>>(m->view, m->absent, b, pctr_out);
      });
    else if (m->fm == XF_SERVE_FMC)
      xf_with_lanes<32>(m->view.K, [&](auto C) {
        xf_k_serve_cand_fmc<C, H><<<grid, 256, 0, st>>>(m->view, m->absent, b, pctr_out);
      });
    else if (m->fm) xf_k_serve_cand<true, H><<<grid, 256, 0, st>>>(m->view, m->absent, b, pctr_out);
    else xf_k_serve_cand<false, false><<<grid, 256, 0, st>>>(m->view, m->absent, b, pctr_out);
  });
}

// ---- building a model's table
__global__ void xf_k_model_fill(uint4* base, uint64_t chunks16, uint32_t per_row) {
  for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < chunks16; c += (uint64_t)gridDim.x * blockDim.x)
    base[c] = (c % per_row == 0) ? make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u) : make_uint4(0u, 0u, 0u, 0u);
}

// Slot r of the training table as a reader resolves it, and whether the model keeps it.  COUNT: count the rows kept,
// the live rows and the live keys outside [lo, hi] (counts[3]: a part's foreign keys); else insert the rows kept into `m`.
template <bool COUNT, int VEC>
__global__ void __launch_bounds__(256)
xf_k_freeze(XfTableView t, XfTableView m, int absent, int prune, uint64_t lo, uint64_t hi,
            unsigned long long* __restrict__ counts, int* error) {
  const uint64_t cap = t.mask + 1;
  unsigned int kept_n = 0, live_n = 0, foreign_n = 0;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap; r += (uint64_t)gridDim.x * blockDim.x) {
    XfHead h = xf_load_head(xf_row(t, r));
    if (h.key == XF_EMPTY_KEY) continue;
    ++live_n;
    if (COUNT && (h.key < lo || h.key > hi)) ++foreign_n;
    const uint32_t flags = t.lazy ? 0u : h.flags;  // a lazy (LR) row keeps a batch tag there
    xf_apply_pending(t, h);
    float st = 0.f, qt = 0.f;
    if (t.K > 0) xf_fm_token<VEC>(t, (uint32_t)r, flags, h.key, st, qt);
    bool keep = true;
    if (prune && h.w == 0.0f)
      keep = t.K > 0 && (absent == XF_ABSENT_DEFAULT ? (flags & XF_FLAG_V_READY) != 0u : !(st == 0.0f && qt == 0.0f));
    if (!keep) continue;
    ++kept_n;
    if (COUNT) continue;
    uint8_t* p = xf_model_claim(m, h.key, error);
    if (!p) continue;
    // the fields only: the padding stays as the fill left it, zero
    if (t.K > 0) {
      *reinterpret_cast<float2*>(p + 8) = make_float2(h.w, st);
      *reinterpret_cast<float*>(p + 16) = qt;
    } else {
      *reinterpret_cast<float*>(p + 8) = h.w;
    }
  }
  if (COUNT) {
    kept_n = __reduce_add_sync(0xffffffffu, kept_n);
    live_n = __reduce_add_sync(0xffffffffu, live_n);
    foreign_n = __reduce_add_sync(0xffffffffu, foreign_n);
    if ((threadIdx.x & 31u) == 0u) {
      if (kept_n) atomicAdd(counts, (unsigned long long)kept_n);
      if (live_n) atomicAdd(counts + 1, (unsigned long long)live_n);
      if (foreign_n) atomicAdd(counts + 3, (unsigned long long)foreign_n);
    }
  }
}

// latent piece q (coordinates 4q .. 4q+3) of a canonical table's row r as a reader resolves it: the row's block if it is
// materialised, else the initial values
__device__ __forceinline__ float4 xf_fmc_piece(const XfTableView& t, uint64_t r, bool ready, uint64_t key, uint32_t q) {
  if (ready) return __ldcg(reinterpret_cast<const float4*>(xf_row(t, r) + 32) + q);
  return xf_v_init_piece(t, key, q);
}

// xf_k_freeze for a canonical table: the model row is {key, w, 0, v[K]} with v resolved as xf_fmc_piece does.  Prune:
// w == 0 and, under DEFAULT, a latent block that is not materialised; under ZERO, every resolved v_k == 0.  MVM: the
// multi-view machine's row {key, 0, v[K]}: w is neither written nor part of the prune rule.
template <bool COUNT, bool MVM>
__global__ void __launch_bounds__(256)
xf_k_freeze_fmc(XfTableView t, XfTableView m, int absent, int prune, unsigned long long* __restrict__ counts, int* error) {
  const uint64_t cap = t.mask + 1;
  const uint32_t pieces = (uint32_t)t.K >> 2;
  unsigned int kept_n = 0, live_n = 0;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap; r += (uint64_t)gridDim.x * blockDim.x) {
    const XfHead h = xf_load_head(xf_row(t, r));
    if (h.key == XF_EMPTY_KEY) continue;
    ++live_n;
    const bool ready = (h.flags & XF_FLAG_V_READY) != 0u;
    bool keep = true;
    if (prune && (MVM || h.w == 0.0f)) {
      keep = false;
      if (absent == XF_ABSENT_DEFAULT) keep = ready;
      else
        for (uint32_t q = 0; q < pieces && !keep; ++q) {
          const float4 v = xf_fmc_piece(t, r, ready, h.key, q);
          keep = v.x != 0.0f || v.y != 0.0f || v.z != 0.0f || v.w != 0.0f;
        }
    }
    if (!keep) continue;
    ++kept_n;
    if (COUNT) continue;
    uint8_t* p = xf_model_claim(m, h.key, error);
    if (!p) continue;
    if (!MVM) *reinterpret_cast<float*>(p + 8) = h.w;  // bytes 12 .. 15 (MVM: 8 .. 15) and the tail stay as the fill left them: zero
    for (uint32_t q = 0; q < pieces; ++q) reinterpret_cast<float4*>(p + 16)[q] = xf_fmc_piece(t, r, ready, h.key, q);
  }
  if (COUNT) {
    kept_n = __reduce_add_sync(0xffffffffu, kept_n);
    live_n = __reduce_add_sync(0xffffffffu, live_n);
    if ((threadIdx.x & 31u) == 0u) {
      if (kept_n) atomicAdd(counts, (unsigned long long)kept_n);
      if (live_n) atomicAdd(counts + 1, (unsigned long long)live_n);
    }
  }
}

// what a canonical model holds for keys[0 .. n): w, v[n][K] (either may be nullptr; H: v widened from binary16), present
template <bool H>
__global__ void xf_k_model_lookup_fmc(XfTableView m, const uint64_t* __restrict__ keys, uint64_t n, float* w_out, float* v_out,
                                      uint8_t* present) {
  const int K = m.K;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const int64_t s = xf_model_find_slot(m, keys[i]);
    const uint8_t* p = s >= 0 ? xf_row(m, (uint64_t)s) : nullptr;
    if (w_out) w_out[i] = p ? reinterpret_cast<const float*>(p)[2] : 0.f;
    if (v_out)
      for (int k = 0; k < K; ++k)
        v_out[i * K + k] = !p ? 0.f : H ? xf_h2f(reinterpret_cast<const uint16_t*>(p + 16)[k]) : reinterpret_cast<const float*>(p + 16)[k];
    present[i] = p ? 1 : 0;
  }
}

// insert n packed rows (a chunk of a model file, or a delta's upserts) into `m`
__global__ void __launch_bounds__(256)
xf_k_model_insert_rows(XfTableView m, const uint8_t* __restrict__ rows, uint64_t n, int* error) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* src = rows + i * m.stride;
    xf_model_put_row(m, src, __ldg(reinterpret_cast<const ulonglong2*>(src)), error);
  }
}

// merge: the live rows among n slots of a part (its own slot array, or a chunk of it staged on this device) into `m`
__global__ void __launch_bounds__(256)
xf_k_merge(const uint8_t* __restrict__ slots, uint64_t n, XfTableView m, int* error) {
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* src = slots + r * m.stride;
    const ulonglong2 head = __ldg(reinterpret_cast<const ulonglong2*>(src));
    if (head.x == XF_EMPTY_KEY) continue;
    xf_model_put_row(m, src, head, error);
  }
}

// A latent field at the result's precision: binary16 bits rounded to nearest even (TO_HALF), or the float32 value of
// binary16 bits.  *over counts a field finite in float32 and not in binary16 (|x| >= 65520); NaN stays NaN.
__device__ __forceinline__ uint32_t xf_to_half(float x, uint32_t& over) {
  const __half h = __float2half_rn(x);
  over += (isfinite(x) && __hisinf(h)) ? 1u : 0u;
  return (uint32_t)__half_as_ushort(h);
}

// convert: the live rows of a model's slots into `m`, its latent fields converted (TO_HALF: F32 -> F16, else F16 ->
// F32); w and the key are copied, the result's padding stays as the fill left it, zero.  An FM row is built in registers
// before the claim.  A canonical row (up to 544 bytes) is converted a piece v[4q .. 4q+3] at a time after the claim, as
// xf_model_put_row copies the rest of a row.  overflow[0] += the fields that do not fit binary16, overflow[1] = the
// smallest key that holds one.
template <bool FMC, bool TO_HALF>
__global__ void __launch_bounds__(256)
xf_k_model_convert(XfTableView src, XfTableView m, unsigned long long* overflow, int* error) {
  const uint64_t cap = src.mask + 1;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* p = xf_row(src, r);
    const ulonglong2 head = __ldg(reinterpret_cast<const ulonglong2*>(p));
    if (head.x == XF_EMPTY_KEY) continue;
    uint32_t over = 0;
    if (!FMC) {
      // F32 {key, w, st | qt, 0...}: head.y = w | st << 32, qt at 16; F16 {key, w | st << 32 | qt << 48}
      uint64_t body;
      float qt = 0.f;
      if (TO_HALF) {
        const float st = __uint_as_float((uint32_t)(head.y >> 32));
        qt = __ldg(reinterpret_cast<const float*>(p + 16));
        body = (head.y & 0xFFFFFFFFull) | (uint64_t)xf_to_half(st, over) << 32 | (uint64_t)xf_to_half(qt, over) << 48;
      } else {
        body = (head.y & 0xFFFFFFFFull) | (uint64_t)__float_as_uint(xf_h2f((uint32_t)(head.y >> 32))) << 32;
        qt = xf_h2f((uint32_t)(head.y >> 48));
      }
      uint8_t* dst = xf_model_claim(m, head.x, error);
      if (dst) {
        *reinterpret_cast<unsigned long long*>(dst + 8) = body;
        if (!TO_HALF) *reinterpret_cast<float*>(dst + 16) = qt;
      }
    } else {
      uint8_t* dst = xf_model_claim(m, head.x, error);
      if (dst) {
        *reinterpret_cast<unsigned long long*>(dst + 8) = head.y;  // w and the zero word
        const uint32_t pieces = (uint32_t)src.K >> 2;
        for (uint32_t q = 0; q < pieces; ++q) {
          if (TO_HALF) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(p + 16) + q);
            reinterpret_cast<uint2*>(dst + 16)[q] = make_uint2(xf_to_half(v.x, over) | xf_to_half(v.y, over) << 16,
                                                               xf_to_half(v.z, over) | xf_to_half(v.w, over) << 16);
          } else {
            const uint2 h = __ldg(reinterpret_cast<const uint2*>(p + 16) + q);
            reinterpret_cast<float4*>(dst + 16)[q] = make_float4(xf_h2f(h.x), xf_h2f(h.x >> 16), xf_h2f(h.y), xf_h2f(h.y >> 16));
          }
        }
      }
    }
    if (TO_HALF && over) {
      atomicAdd(overflow, (unsigned long long)over);
      atomicMin(overflow + 1, (unsigned long long)head.x);
    }
  }
}

// every (key, slot) the model holds, in no particular order
__global__ void xf_k_model_list(XfTableView m, uint64_t* keys_out, uint32_t* slots_out, unsigned long long* count) {
  const uint64_t cap = m.mask + 1;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < cap; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t key = *reinterpret_cast<const uint64_t*>(xf_row(m, r));
    if (key == XF_EMPTY_KEY) continue;
    const unsigned long long idx = atomicAdd(count, 1ull);
    keys_out[idx] = key;
    slots_out[idx] = (uint32_t)r;
  }
}

// out = the rows in slots[0 .. n), packed, 16 bytes per thread and access
__global__ void xf_k_model_gather(XfTableView m, const uint32_t* __restrict__ slots, uint64_t n, uint4* __restrict__ out) {
  const uint32_t q = m.stride / 16u;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n * q; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = j / q;
    out[j] = *reinterpret_cast<const uint4*>(xf_row(m, slots[i]) + 16u * (uint32_t)(j - i * q));
  }
}

template <bool H>
__global__ void xf_k_model_lookup(XfTableView m, const uint64_t* __restrict__ keys, uint64_t n, float* w_out, float* st_out,
                                  float* qt_out, uint8_t* present) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t key = keys[i];
    uint64_t k;
    float w, st, qt;
    bool have;
    if (m.K > 0) {
      xf_serve_load<true, H>(xf_row(m, xf_home_slot(m, key)), k, w, st, qt);
      have = xf_serve_find<true, H>(m, key, k, w, st, qt);
    } else {
      xf_serve_load<false>(xf_row(m, xf_home_slot(m, key)), k, w, st, qt);
      have = xf_serve_find<false>(m, key, k, w, st, qt);
      st = qt = 0.f;
    }
    w_out[i] = have ? w : 0.f;
    st_out[i] = have ? st : 0.f;
    qt_out[i] = have ? qt : 0.f;
    present[i] = have ? 1 : 0;
  }
}

// -------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------
// the model's table on the current device: `capacity` empty rows
int xf_model_alloc(xf_model* m, uint64_t capacity) {
  if (capacity > (1ull << 32)) {
    xf_set_error("a serving model of %llu slots exceeds 2^32", (unsigned long long)capacity);
    return XF_ERR_FULL;
  }
  const uint32_t stride = xf_model_row_bytes(m->fm, m->view.K, m->precision);
  m->view.canon = xf_serve_latent_rows(m->fm) ? 1 : 0;
  uint8_t* base = nullptr;
  XF_CUDA_TRY(cudaMalloc(&base, capacity * stride));
  m->view.base = base;
  m->view.mask = capacity - 1;
  uint32_t lg = 0;
  while ((1ull << lg) < capacity) ++lg;
  m->view.log2cap = lg;
  m->view.stride = stride;
  m->view.bshift = xf_bucket_shift(stride, lg);
  const uint64_t chunks16 = capacity * (stride / 16u);
  xf_k_model_fill<<<xf_grid_for(chunks16, 256, 16), 256, 0, m->stream>>>(reinterpret_cast<uint4*>(base), chunks16, stride / 16u);
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

int xf_model_init(xf_model* m, int device, const XfCompat& c) {
  m->device = device;
  XF_CUDA_TRY(cudaSetDevice(device));
  XF_CUDA_TRY(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
  m->fm = c.fm;
  m->precision = c.precision;
  m->absent = c.absent;
  m->optimizer = c.optimizer;
  m->view.K = c.latent_dim;
  m->view.opt = c.optimizer;
  m->view.v_init = c.v_init;
  m->view.v_const = c.v_const;
  m->view.seed = c.seed;
  return XF_OK;
}

void xf_model_free(xf_model* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  if (m->stream) cudaStreamSynchronize(m->stream);
  if (m->view.base) cudaFree(m->view.base);
  m->s_keys.release(); m->s_out.release(); m->s_aux.release();
  m->h_in.release(); m->h_out.release();
  if (m->stream) cudaStreamDestroy(m->stream);
  delete m;
}

int XfSortedSlots::ensure(uint64_t n) {
  XF_TRY(keys_in.ensure(std::max<uint64_t>(n, 1) * 8)); XF_TRY(keys_out.ensure(std::max<uint64_t>(n, 1) * 8));
  XF_TRY(slots_in.ensure(std::max<uint64_t>(n, 1) * 4)); XF_TRY(slots_out.ensure(std::max<uint64_t>(n, 1) * 4));
  return count.ensure(8);
}

void XfSortedSlots::release() {
  keys_in.release(); keys_out.release(); slots_in.release(); slots_out.release(); tmp.release(); count.release();
}

int xf_sort_slots(XfSortedSlots& s, uint64_t n, cudaStream_t st) {
  if (n == 0) return XF_OK;
  size_t tb = 0;
  XF_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, s.keys_in.as<uint64_t>(), s.keys_out.as<uint64_t>(), s.slots_in.as<uint32_t>(),
                                              s.slots_out.as<uint32_t>(), n, 0, 64, st));
  XF_TRY(s.tmp.ensure(std::max<size_t>(tb, 16)));
  XF_CUDA_TRY(cub::DeviceRadixSort::SortPairs(s.tmp.p, tb, s.keys_in.as<uint64_t>(), s.keys_out.as<uint64_t>(), s.slots_in.as<uint32_t>(),
                                              s.slots_out.as<uint32_t>(), n, 0, 64, st));
  return XF_OK;
}

int xf_model_list_sorted(const XfTableView& v, uint64_t n, XfSortedSlots& s, cudaStream_t st) {
  XF_TRY(s.ensure(n));
  XF_CUDA_TRY(cudaMemsetAsync(s.count.p, 0, 8, st));
  xf_k_model_list<<<xf_grid_for(v.mask + 1, 256, 8), 256, 0, st>>>(v, s.keys_in.as<uint64_t>(), s.slots_in.as<uint32_t>(),
                                                                   s.count.as<unsigned long long>());
  XF_CUDA_TRY(cudaGetLastError());
  return xf_sort_slots(s, n, st);
}

int xf_model_gather(const XfTableView& v, const uint32_t* slots, uint64_t n, void* out, cudaStream_t st) {
  if (n == 0) return XF_OK;
  xf_k_model_gather<<<xf_grid_for(n * (v.stride / 16u), 256, 8), 256, 0, st>>>(v, slots, n, reinterpret_cast<uint4*>(out));
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

int xf_model_insert_rows(const XfTableView& v, const uint8_t* rows, uint64_t n, int* error, cudaStream_t st) {
  if (n == 0) return XF_OK;
  xf_k_model_insert_rows<<<xf_grid_for(n, 256, 8), 256, 0, st>>>(v, rows, n, error);
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

XF_DLL int xf_freeze_config_default(xf_freeze_config* cfg) {
  if (!cfg) return XF_ERR_ARG;
  cfg->absent = -1;
  cfg->prune = 1;
  cfg->device = -1;
  return XF_OK;
}

// the body of xf_table_freeze (latent = XF_SERVE_LR), xf_table_freeze_canonical (XF_SERVE_FMC), xf_table_freeze_mvm
// (XF_SERVE_MVM), xf_table_freeze_ffm (XF_SERVE_FFM: the canonical freeze, its rows are the canonical ones) and
// xf_table_freeze_part (part): on failure the caller frees `m`
static int xf_freeze_into(xf_table* t, const xf_freeze_config& cfg, int latent, bool part, xf_model* m, const char* fn) {
  const int src_dev = t->cfg.device;
  XF_CUDA_TRY(cudaSetDevice(src_dev));
  XF_TRY(t->check_error());  // waits for everything enqueued on the table's stream
  const XfTableView& tv = t->view;
  const int fm = latent != XF_SERVE_LR ? latent : (tv.K > 0 ? XF_SERVE_FM : XF_SERVE_LR);
  const int absent = cfg.absent >= 0 ? cfg.absent : (t->admit.mode == XF_ADMIT_ALL ? XF_ABSENT_DEFAULT : XF_ABSENT_ZERO);
  XF_TRY(xf_model_init(m, src_dev, XfCompat{fm, tv.K, tv.opt, absent, tv.v_init, tv.v_const, tv.seed,
                                                   XF_PRECISION_F32}));
  // the build runs on the model's stream: the table's stream is idle (above) and the host calls on the table are
  // locked out by the caller, so nothing writes the table while it is read
  cudaStream_t st = m->stream;
  unsigned long long* d_counts = nullptr;  // {kept, live, error flag, foreign}
  XF_CUDA_TRY(cudaMalloc(&d_counts, 4 * sizeof(unsigned long long)));
  struct Free { void* p; ~Free() { cudaFree(p); } } free_counts{d_counts};
  XF_CUDA_TRY(cudaMemsetAsync(d_counts, 0, 4 * sizeof(unsigned long long), st));
  int* d_error = reinterpret_cast<int*>(d_counts + 2);
  const int grid = xf_grid_for(tv.mask + 1, 256, 8);
  const int prune = cfg.prune ? 1 : 0;
  // the keys the table owns: a part refuses others; a whole table (num_shards == 1) owns every key
  uint64_t lo = 0, hi = 0;
  xf_shard_range(t->cfg.shard_index, t->cfg.num_shards, &lo, &hi);
#define XF_FREEZE_LAUNCH(COUNT)                                                                                       \
  if (fm == XF_SERVE_FMC || fm == XF_SERVE_FFM) xf_k_freeze_fmc<COUNT, false><<<grid, 256, 0, st>>>(tv, m->view, m->absent, prune, d_counts, d_error); \
  else if (fm == XF_SERVE_MVM) xf_k_freeze_fmc<COUNT, true><<<grid, 256, 0, st>>>(tv, m->view, m->absent, prune, d_counts, d_error); \
  else switch (xf_vec_for(tv.K)) {                                                                                         \
    case 4: xf_k_freeze<COUNT, 4><<<grid, 256, 0, st>>>(tv, m->view, m->absent, prune, lo, hi, d_counts, d_error); break; \
    case 2: xf_k_freeze<COUNT, 2><<<grid, 256, 0, st>>>(tv, m->view, m->absent, prune, lo, hi, d_counts, d_error); break; \
    default: xf_k_freeze<COUNT, 1><<<grid, 256, 0, st>>>(tv, m->view, m->absent, prune, lo, hi, d_counts, d_error); break; \
  }
  XF_FREEZE_LAUNCH(true)
  XF_CUDA_TRY(cudaGetLastError());
  unsigned long long counts[4] = {0, 0, 0, 0};
  XF_CUDA_TRY(cudaMemcpyAsync(counts, d_counts, sizeof(counts), cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  if (part && counts[3] != 0) {
    xf_set_error("%s: the table is shard %d of %d and holds %llu keys outside its range (pulled, pushed or imported "
                 "there): a part holds its own range only", fn, t->cfg.shard_index, t->cfg.num_shards, counts[3]);
    return XF_ERR_STATE;
  }
  if (part) {
    m->shard_index = t->cfg.shard_index;
    m->num_shards = t->cfg.num_shards;
  }
  m->keys = counts[0];
  m->source_keys = counts[1];
  m->pruned_keys = counts[1] - counts[0];
  XF_TRY(xf_model_alloc(m, xf_model_capacity(m->keys)));
  XF_FREEZE_LAUNCH(false)
#undef XF_FREEZE_LAUNCH
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(counts, d_counts, sizeof(counts), cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  if ((int)counts[2] != 0) {
    xf_set_error("%s: a probe sequence of the model overflowed", fn);
    return XF_ERR_FULL;
  }
  if (cfg.device >= 0 && cfg.device != src_dev) {
    // the model lives on another device: copy its table there
    const uint64_t bytes = (m->view.mask + 1) * (uint64_t)m->view.stride;
    uint8_t* src = m->view.base;
    XF_CUDA_TRY(cudaStreamDestroy(m->stream));
    m->stream = nullptr;
    XF_CUDA_TRY(cudaSetDevice(cfg.device));
    uint8_t* dst = nullptr;
    XF_CUDA_TRY(cudaMalloc(&dst, bytes));
    m->view.base = dst;
    m->device = cfg.device;
    const cudaError_t e = cudaMemcpyPeer(dst, cfg.device, src, src_dev, bytes);
    cudaSetDevice(src_dev);
    cudaFree(src);
    XF_CUDA_TRY(e);
    XF_CUDA_TRY(cudaSetDevice(cfg.device));
    XF_CUDA_TRY(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
  }
  return XF_OK;
}

static int xf_freeze(xf_table* t, const xf_freeze_config* cfg_in, int latent, bool part, xf_model** out) {
  const bool canonical = latent == XF_SERVE_FMC, mvm = latent == XF_SERVE_MVM, ffm = latent == XF_SERVE_FFM;
  const char* fn = part ? "xf_table_freeze_part" : canonical ? "xf_table_freeze_canonical" : mvm ? "xf_table_freeze_mvm"
                 : ffm ? "xf_table_freeze_ffm" : "xf_table_freeze";
  if (out) *out = nullptr;
  if (!t || !out) { xf_set_error("null argument"); return XF_ERR_ARG; }
  xf_freeze_config cfg;
  xf_freeze_config_default(&cfg);
  if (cfg_in) cfg = *cfg_in;
  if (cfg.absent < -1 || cfg.absent > XF_ABSENT_ZERO) { xf_set_error("%s: absent = %d is not an XF_ABSENT_* policy", fn, cfg.absent); return XF_ERR_ARG; }
  if (cfg.device >= xf_device_count()) { xf_set_error("%s: no CUDA device %d", fn, cfg.device); return XF_ERR_ARG; }
  if (part && t->cfg.canonical_fm) {
    xf_set_error("xf_table_freeze_part: a canonical table (canonical_fm = 1) is never sharded: freeze it whole with "
                 "xf_table_freeze_canonical");
    return XF_ERR_ARG;
  }
  if (latent == XF_SERVE_LR && !part && t->cfg.canonical_fm) {
    xf_set_error("xf_table_freeze: a canonical table (canonical_fm = 1) has no collapsed serving model: the per-k sums of "
                 "the canonical FM and the multi-view machine do not collapse to one pair of sums per key; "
                 "xf_table_freeze_canonical serves it with the canonical FM's forward");
    return XF_ERR_ARG;
  }
  if (mvm && !t->cfg.canonical_fm) {
    xf_set_error("xf_table_freeze_mvm: the table is not canonical (canonical_fm = 0): the multi-view machine trains "
                 "canonical tables only");
    return XF_ERR_ARG;
  }
  if (mvm && !xf_mvm_latent_ok(t->cfg.latent_dim)) {
    xf_set_error("xf_table_freeze_mvm: latent_dim = %d: the multi-view machine serves K = 4, 8, 16 or 32",
                 t->cfg.latent_dim);
    return XF_ERR_ARG;
  }
  if (ffm && !t->cfg.canonical_fm) {
    xf_set_error("xf_table_freeze_ffm: the table is not canonical (canonical_fm = 0): the field-aware FM trains canonical "
                 "tables only");
    return XF_ERR_ARG;
  }
  if (ffm && !xf_fmc_latent_ok(t->cfg.latent_dim)) {
    xf_set_error("xf_table_freeze_ffm: latent_dim = %d: the field-aware FM serves L = 4, 8, 16, 32, 64 or 128",
                 t->cfg.latent_dim);
    return XF_ERR_ARG;
  }
  if (canonical && (!t->cfg.canonical_fm || !xf_fmc_latent_ok(t->cfg.latent_dim))) {
    xf_set_error("xf_table_freeze_canonical: the table is not canonical (canonical_fm = %d, latent_dim = %d): freeze it "
                 "with xf_table_freeze", t->cfg.canonical_fm, t->cfg.latent_dim);
    return XF_ERR_ARG;
  }
  if (!part && t->cfg.num_shards > 1) {
    xf_set_error("%s: the table is shard %d of %d: one shard's rows are not a model (freeze every shard with "
                 "xf_table_freeze_part and merge the parts with xf_model_merge)", fn, t->cfg.shard_index, t->cfg.num_shards);
    return XF_ERR_ARG;
  }
  std::lock_guard<std::mutex> host_lock(t->host_mu);
  xf_model* m = new xf_model;
  const int rc = xf_freeze_into(t, cfg, latent, part, m, fn);
  if (rc != XF_OK) { xf_model_free(m); return rc; }
  *out = m;
  return XF_OK;
}

XF_DLL int xf_table_freeze(xf_table* t, const xf_freeze_config* cfg, xf_model** out) {
  return xf_freeze(t, cfg, XF_SERVE_LR, false, out);
}

XF_DLL int xf_table_freeze_canonical(xf_table* t, const xf_freeze_config* cfg, xf_model** out) {
  return xf_freeze(t, cfg, XF_SERVE_FMC, false, out);
}

XF_DLL int xf_table_freeze_mvm(xf_table* t, const xf_freeze_config* cfg, xf_model** out) {
  return xf_freeze(t, cfg, XF_SERVE_MVM, false, out);
}

XF_DLL int xf_table_freeze_ffm(xf_table* t, const xf_freeze_config* cfg, xf_model** out) {
  return xf_freeze(t, cfg, XF_SERVE_FFM, false, out);
}

XF_DLL int xf_table_freeze_part(xf_table* t, const xf_freeze_config* cfg, xf_model** out) {
  return xf_freeze(t, cfg, XF_SERVE_LR, true, out);
}

XF_DLL int xf_model_part_info(xf_model* m, int* shard_index, int* num_shards) {
  if (!m) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (m->num_shards == 0) {
    xf_set_error("xf_model_part_info: the model is whole, not a part");
    return XF_ERR_STATE;
  }
  if (shard_index) *shard_index = m->shard_index;
  if (num_shards) *num_shards = m->num_shards;
  return XF_OK;
}

XF_DLL int xf_model_destroy(xf_model* m) {
  xf_model_free(m);
  return XF_OK;
}

XF_DLL int xf_model_get_info(xf_model* m, xf_model_info* out) {
  if (!m || !out) return XF_ERR_ARG;
  memset(out, 0, sizeof(*out));
  out->keys = m->keys;
  out->capacity = m->view.mask + 1;
  out->bytes = out->capacity * m->view.stride;
  out->source_keys = m->source_keys;
  out->pruned_keys = m->pruned_keys;
  out->row_bytes = m->view.stride;
  out->latent_dim = m->view.K;
  out->optimizer = m->optimizer;
  out->absent = m->absent;
  out->fm = m->fm;
  out->precision = m->precision;
  return XF_OK;
}

// ---- predict
// one host array of a host entry point's batch: `bytes` from `src` (0: the array is not uploaded)
struct XfUpload {
  const void* src;
  size_t bytes;
};

// The arrays of a host batch into one pinned image, each at a 16-byte aligned offset, and onto the device with one copy
// into s_aux on the model's stream; dev[i] = array i's device address, NULL for an empty one.  The caller holds the
// model's mutex with its device current.
template <int N>
static int xf_model_upload(xf_model* m, const XfUpload (&part)[N], const void* (&dev)[N]) {
  size_t off[N + 1];
  off[0] = 0;
  for (int i = 0; i < N; ++i) off[i + 1] = off[i] + ((part[i].bytes + 15) & ~(size_t)15);
  XF_TRY(m->h_in.ensure(off[N]));
  XF_TRY(m->s_aux.ensure(off[N]));
  for (int i = 0; i < N; ++i)
    if (part[i].bytes) memcpy(m->h_in.as<uint8_t>() + off[i], part[i].src, part[i].bytes);
  XF_CUDA_TRY(cudaMemcpyAsync(m->s_aux.p, m->h_in.p, off[N], cudaMemcpyHostToDevice, m->stream));
  for (int i = 0; i < N; ++i) dev[i] = part[i].bytes ? m->s_aux.as<uint8_t>() + off[i] : nullptr;
  return XF_OK;
}

// XF_ERR_ARG, naming the array and the index, where ptr[0 .. n] decreases
static int xf_check_nondecreasing(const uint32_t* ptr, uint32_t n, const char* what, const char* fn) {
  for (uint32_t i = 0; i < n; ++i)
    if (ptr[i] > ptr[i + 1]) {
      xf_set_error("%s: %s decreases at %u (%u > %u)", fn, what, i, ptr[i], ptr[i + 1]);
      return XF_ERR_ARG;
    }
  return XF_OK;
}

// the field ids of a model that reads them: below 32 for a multi-view machine's, below F = L / 4 for a field-aware FM's
static int xf_check_host_fields(const xf_model* m, const uint8_t* fields, uint32_t n, const char* what, const char* fn) {
  if (m->fm == XF_SERVE_FFM) {
    const uint32_t F = (uint32_t)m->view.K / 4u;
    for (uint32_t j = 0; j < n; ++j)
      if (fields[j] >= F) {
        xf_set_error("%s: %s: field id %u of token %u: a field-aware FM's model of latent_dim %d takes field ids below "
                     "F = %u", fn, what, (unsigned)fields[j], j, m->view.K, F);
        return XF_ERR_ARG;
      }
    return XF_OK;
  }
  for (uint32_t j = 0; j < n; ++j)
    if (fields[j] >= XF_MVM_FIELDS) {
      xf_set_error("%s: %s: field id %u of token %u: a multi-view machine takes field ids below %d", fn, what,
                   (unsigned)fields[j], j, XF_MVM_FIELDS);
      return XF_ERR_ARG;
    }
  return XF_OK;
}

// feature values are read by canonical, multi-view machine and field-aware FM models only: the LR and FM forwards ignore them
static int xf_check_vals(const xf_model* m, const void* vals, const char* fn) {
  if (vals && !xf_serve_latent_rows(m->fm)) {
    xf_set_error("%s: an %s model ignores feature values: pass vals = NULL (values need a model frozen with "
                 "xf_table_freeze_canonical)", fn, m->fm ? "FM" : "LR");
    return XF_ERR_ARG;
  }
  return XF_OK;
}

// the row kinds whose forward reads the tokens' field ids: the multi-view machine and the field-aware FM
static bool xf_reads_fields(const xf_model* m) { return m->fm == XF_SERVE_MVM || m->fm == XF_SERVE_FFM; }

// field ids are read by multi-view machine and field-aware FM models, and those read nothing without them: the _fields
// entry points serve them only, and every other entry point refuses them
static int xf_check_fields_kind(const xf_model* m, bool with_fields, const char* fn) {
  static const char* const kind[] = {"LR", "FM", "canonical", "multi-view machine's", "field-aware FM's"};
  static_assert(sizeof(kind) / sizeof(kind[0]) == XF_SERVE_FFM + 1, "a name for every row kind");
  if (xf_reads_fields(m) && !with_fields) {
    xf_set_error("%s: a %s model reads the tokens' field ids: use xf_model_predict_host_fields or "
                 "xf_model_predict_device_fields", fn, kind[m->fm]);
    return XF_ERR_ARG;
  }
  if (!xf_reads_fields(m) && with_fields) {
    xf_set_error("%s: an %s model reads no field ids: field ids need a model frozen with xf_table_freeze_mvm or "
                 "xf_table_freeze_ffm", fn, kind[m->fm]);
    return XF_ERR_ARG;
  }
  return XF_OK;
}

static int xf_predict_host(xf_model* m, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* fields, const float* vals,
                           uint32_t rows, uint32_t nnz, float* pctr_out, bool with_fields, const char* fn) {
  if (!m || !row_ptr || (!keys && nnz) || (!pctr_out && rows) || (with_fields && !fields && nnz)) {
    xf_set_error("null argument");
    return XF_ERR_ARG;
  }
  XF_TRY(xf_refuse_part(m, fn));
  XF_TRY(xf_check_fields_kind(m, with_fields, fn));
  XF_TRY(xf_check_vals(m, vals, fn));
  XF_TRY(xf_check_nondecreasing(row_ptr, rows, "row_ptr", fn));
  if (row_ptr[rows] > nnz) { xf_set_error("%s: row_ptr ends at %u, past nnz = %u", fn, row_ptr[rows], nnz); return XF_ERR_ARG; }
  XF_TRY(xf_check_host_keys(keys, nnz, fn));
  if (with_fields) XF_TRY(xf_check_host_fields(m, fields, nnz, "fields", fn));
  if (rows == 0) return XF_OK;
  std::lock_guard<std::mutex> lock(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  XF_TRY(m->h_out.ensure((size_t)rows * 4));
  XF_TRY(m->s_out.ensure((size_t)rows * 4));
  const XfUpload part[] = {{row_ptr, ((size_t)rows + 1) * 4},
                           {keys, (size_t)nnz * 8},
                           {vals, vals ? (size_t)nnz * 4 : 0},
                           {fields, with_fields ? (size_t)nnz : 0}};
  const void* d[4];
  XF_TRY(xf_model_upload(m, part, d));
  xf_launch_predict(m, static_cast<const uint32_t*>(d[0]), static_cast<const uint64_t*>(d[1]),
                    static_cast<const uint8_t*>(d[3]), static_cast<const float*>(d[2]), rows, m->s_out.as<float>(),
                    m->stream);
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(m->h_out.p, m->s_out.p, (size_t)rows * 4, cudaMemcpyDeviceToHost, m->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(m->stream));
  memcpy(pctr_out, m->h_out.p, (size_t)rows * 4);
  return XF_OK;
}

XF_DLL int xf_model_predict_host(xf_model* m, const uint32_t* row_ptr, const uint64_t* keys, uint32_t rows, uint32_t nnz,
                                 float* pctr_out) {
  return xf_predict_host(m, row_ptr, keys, nullptr, nullptr, rows, nnz, pctr_out, false, "xf_model_predict_host");
}

XF_DLL int xf_model_predict_host_values(xf_model* m, const uint32_t* row_ptr, const uint64_t* keys, const float* vals,
                                        uint32_t rows, uint32_t nnz, float* pctr_out) {
  return xf_predict_host(m, row_ptr, keys, nullptr, vals, rows, nnz, pctr_out, false, "xf_model_predict_host_values");
}

XF_DLL int xf_model_predict_host_fields(xf_model* m, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* fields,
                                        const float* vals, uint32_t rows, uint32_t nnz, float* pctr_out) {
  return xf_predict_host(m, row_ptr, keys, fields, vals, rows, nnz, pctr_out, true, "xf_model_predict_host_fields");
}

static int xf_predict_device(xf_model* m, const uint32_t* d_row_ptr, const uint64_t* d_keys, const uint8_t* d_fields,
                             const float* d_vals, uint32_t rows, uint32_t nnz, float* d_pctr_out, void* cuda_stream,
                             bool with_fields, const char* fn) {
  if (!m || !d_row_ptr || (!d_keys && nnz) || (!d_pctr_out && rows) || (with_fields && !d_fields && nnz)) {
    xf_set_error("null argument");
    return XF_ERR_ARG;
  }
  XF_TRY(xf_refuse_part(m, fn));
  XF_TRY(xf_check_fields_kind(m, with_fields, fn));
  XF_TRY(xf_check_vals(m, d_vals, fn));
  XF_CUDA_TRY(cudaSetDevice(m->device));
  xf_launch_predict(m, d_row_ptr, d_keys, d_fields, d_vals, rows, d_pctr_out, reinterpret_cast<cudaStream_t>(cuda_stream));
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

XF_DLL int xf_model_predict_device(xf_model* m, const uint32_t* d_row_ptr, const uint64_t* d_keys, uint32_t rows,
                                   uint32_t nnz, float* d_pctr_out, void* cuda_stream) {
  return xf_predict_device(m, d_row_ptr, d_keys, nullptr, nullptr, rows, nnz, d_pctr_out, cuda_stream, false,
                           "xf_model_predict_device");
}

XF_DLL int xf_model_predict_device_values(xf_model* m, const uint32_t* d_row_ptr, const uint64_t* d_keys, const float* d_vals,
                                          uint32_t rows, uint32_t nnz, float* d_pctr_out, void* cuda_stream) {
  return xf_predict_device(m, d_row_ptr, d_keys, nullptr, d_vals, rows, nnz, d_pctr_out, cuda_stream, false,
                           "xf_model_predict_device_values");
}

XF_DLL int xf_model_predict_device_fields(xf_model* m, const uint32_t* d_row_ptr, const uint64_t* d_keys,
                                          const uint8_t* d_fields, const float* d_vals, uint32_t rows, uint32_t nnz,
                                          float* d_pctr_out, void* cuda_stream) {
  return xf_predict_device(m, d_row_ptr, d_keys, d_fields, d_vals, rows, nnz, d_pctr_out, cuda_stream, true,
                           "xf_model_predict_device_fields");
}

// what both candidate entry points check without reading the arrays: null pointers, a part, the model's kind
static int xf_check_candidates(xf_model* m, const xf_candidate_batch* b, const void* pctr_out, const char* fn) {
  const bool reads = m && xf_reads_fields(m);
  if (!m || !b || !b->ctx_ptr || !b->cand_ptr || !b->row_ptr || (!b->ctx_keys && b->ctx_nnz) || (!b->keys && b->nnz) ||
      (!pctr_out && b->candidates) || (reads && ((!b->ctx_fields && b->ctx_nnz) || (!b->fields && b->nnz)))) {
    xf_set_error("null argument");
    return XF_ERR_ARG;
  }
  XF_TRY(xf_refuse_part(m, fn));
  XF_TRY(xf_check_fields_kind(m, reads || b->ctx_fields || b->fields, fn));
  XF_TRY(xf_check_vals(m, b->ctx_vals, fn));
  XF_TRY(xf_check_vals(m, b->vals, fn));
  return XF_OK;
}

static XfCandView xf_cand_view(const xf_candidate_batch& b) {
  return XfCandView{b.ctx_ptr, b.ctx_keys, b.ctx_vals, b.ctx_fields, b.cand_ptr, b.row_ptr, b.keys, b.vals, b.fields,
                    b.requests, b.candidates};
}

// the checks xf_model_predict_candidates_host makes on a batch's host arrays, after xf_check_candidates
static int xf_check_candidates_host(const xf_model* m, const xf_candidate_batch* b, const char* fn) {
  const uint32_t R = b->requests, N = b->candidates;
  XF_TRY(xf_check_nondecreasing(b->ctx_ptr, R, "ctx_ptr", fn));
  XF_TRY(xf_check_nondecreasing(b->cand_ptr, R, "cand_ptr", fn));
  XF_TRY(xf_check_nondecreasing(b->row_ptr, N, "row_ptr", fn));
  if (b->cand_ptr[0] != 0 || b->cand_ptr[R] != N) {
    xf_set_error("%s: cand_ptr runs from %u to %u: it must run from 0 to candidates = %u", fn, b->cand_ptr[0],
                 b->cand_ptr[R], N);
    return XF_ERR_ARG;
  }
  if (b->ctx_ptr[R] > b->ctx_nnz) {
    xf_set_error("%s: ctx_ptr ends at %u, past ctx_nnz = %u", fn, b->ctx_ptr[R], b->ctx_nnz);
    return XF_ERR_ARG;
  }
  if (b->row_ptr[N] > b->nnz) {
    xf_set_error("%s: row_ptr ends at %u, past nnz = %u", fn, b->row_ptr[N], b->nnz);
    return XF_ERR_ARG;
  }
  char what[96];
  snprintf(what, sizeof what, "%s: ctx_keys", fn);
  XF_TRY(xf_check_host_keys(b->ctx_keys, b->ctx_nnz, what));
  snprintf(what, sizeof what, "%s: keys", fn);
  XF_TRY(xf_check_host_keys(b->keys, b->nnz, what));
  if (xf_reads_fields(m)) {
    XF_TRY(xf_check_host_fields(m, b->ctx_fields, b->ctx_nnz, "ctx_fields", fn));
    XF_TRY(xf_check_host_fields(m, b->fields, b->nnz, "fields", fn));
  }
  return XF_OK;
}

// A checked host batch onto the device as one image (xf_model_upload), each context once; *v: its arrays there.  The
// caller holds the model's mutex with its device current.
static int xf_upload_candidates(xf_model* m, const xf_candidate_batch* b, XfCandView* v) {
  const uint32_t R = b->requests, N = b->candidates;
  const bool reads = xf_reads_fields(m);
  const XfUpload part[] = {
      {b->ctx_ptr, ((size_t)R + 1) * 4},
      {b->cand_ptr, ((size_t)R + 1) * 4},
      {b->row_ptr, ((size_t)N + 1) * 4},
      {b->ctx_keys, (size_t)b->ctx_nnz * 8},
      {b->keys, (size_t)b->nnz * 8},
      {b->ctx_vals, b->ctx_vals ? (size_t)b->ctx_nnz * 4 : 0},
      {b->vals, b->vals ? (size_t)b->nnz * 4 : 0},
      {b->ctx_fields, reads ? (size_t)b->ctx_nnz : 0},
      {b->fields, reads ? (size_t)b->nnz : 0},
  };
  const void* d[9];
  XF_TRY(xf_model_upload(m, part, d));
  *v = XfCandView{static_cast<const uint32_t*>(d[0]), static_cast<const uint64_t*>(d[3]), static_cast<const float*>(d[5]),
                  static_cast<const uint8_t*>(d[7]), static_cast<const uint32_t*>(d[1]), static_cast<const uint32_t*>(d[2]),
                  static_cast<const uint64_t*>(d[4]), static_cast<const float*>(d[6]), static_cast<const uint8_t*>(d[8]),
                  R, N};
  return XF_OK;
}

XF_DLL int xf_model_predict_candidates_host(xf_model* m, const xf_candidate_batch* b, float* pctr_out) {
  static const char* const fn = "xf_model_predict_candidates_host";
  XF_TRY(xf_check_candidates(m, b, pctr_out, fn));
  XF_TRY(xf_check_candidates_host(m, b, fn));
  const uint32_t N = b->candidates;
  if (N == 0) return XF_OK;
  std::lock_guard<std::mutex> lock(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  XF_TRY(m->h_out.ensure((size_t)N * 4));
  XF_TRY(m->s_out.ensure((size_t)N * 4));
  XfCandView v;
  XF_TRY(xf_upload_candidates(m, b, &v));
  xf_launch_candidates(m, v, m->s_out.as<float>(), m->stream);
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(m->h_out.p, m->s_out.p, (size_t)N * 4, cudaMemcpyDeviceToHost, m->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(m->stream));
  memcpy(pctr_out, m->h_out.p, (size_t)N * 4);
  return XF_OK;
}

XF_DLL int xf_model_predict_candidates_device(xf_model* m, const xf_candidate_batch* b, float* d_pctr_out,
                                              void* cuda_stream) {
  XF_TRY(xf_check_candidates(m, b, d_pctr_out, "xf_model_predict_candidates_device"));
  XF_CUDA_TRY(cudaSetDevice(m->device));
  xf_launch_candidates(m, xf_cand_view(*b), d_pctr_out, reinterpret_cast<cudaStream_t>(cuda_stream));
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

// what both rank entry points check besides xf_check_candidates: k, and the index output
static int xf_check_rank(const xf_candidate_batch* b, uint32_t k, const void* top_index, const char* fn) {
  if (k == 0 || k > XF_RANK_MAX_K) {
    xf_set_error("%s: k = %u: it must run from 1 to XF_RANK_MAX_K = %d", fn, k, XF_RANK_MAX_K);
    return XF_ERR_ARG;
  }
  if (b && b->requests && !top_index) {
    xf_set_error("%s: top_index is NULL with %u requests", fn, b->requests);
    return XF_ERR_ARG;
  }
  return XF_OK;
}

XF_DLL int xf_model_rank_candidates_host(xf_model* m, const xf_candidate_batch* b, uint32_t k, uint32_t* top_index,
                                         float* top_pctr) {
  static const char* const fn = "xf_model_rank_candidates_host";
  XF_TRY(xf_check_rank(b, k, top_index, fn));
  XF_TRY(xf_check_candidates(m, b, top_index, fn));
  XF_TRY(xf_check_candidates_host(m, b, fn));
  const uint32_t R = b->requests, N = b->candidates;
  if (R == 0) return XF_OK;
  const size_t slots = (size_t)R * k, back = slots * (top_pctr ? 8 : 4);
  std::lock_guard<std::mutex> lock(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  // the scores stay on the device in s_out; the outputs, indices then scores, in s_keys
  XF_TRY(m->s_out.ensure((size_t)N * 4));
  XF_TRY(m->s_keys.ensure(slots * 8));
  XF_TRY(m->h_out.ensure(back));
  XfCandView v;
  XF_TRY(xf_upload_candidates(m, b, &v));
  uint32_t* d_index = m->s_keys.as<uint32_t>();
  xf_launch_candidates(m, v, m->s_out.as<float>(), m->stream);
  xf_launch_rank(m->s_out.as<float>(), v.cand_ptr, R, k, d_index,
                 top_pctr ? reinterpret_cast<float*>(d_index + slots) : nullptr, m->stream);
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(m->h_out.p, m->s_keys.p, back, cudaMemcpyDeviceToHost, m->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(m->stream));
  memcpy(top_index, m->h_out.p, slots * 4);
  if (top_pctr) memcpy(top_pctr, m->h_out.as<uint8_t>() + slots * 4, slots * 4);
  return XF_OK;
}

XF_DLL int xf_model_rank_candidates_device(xf_model* m, const xf_candidate_batch* b, uint32_t k, float* d_pctr,
                                           uint32_t* d_top_index, float* d_top_pctr, void* cuda_stream) {
  static const char* const fn = "xf_model_rank_candidates_device";
  XF_TRY(xf_check_rank(b, k, d_top_index, fn));
  XF_TRY(xf_check_candidates(m, b, d_pctr, fn));
  XF_CUDA_TRY(cudaSetDevice(m->device));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
  xf_launch_candidates(m, xf_cand_view(*b), d_pctr, st);
  xf_launch_rank(d_pctr, b->cand_ptr, b->requests, k, d_top_index, d_top_pctr, st);
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

XF_DLL int xf_model_predict_ingested(xf_model* m, xf_trainer* tr, uint32_t row_start, uint32_t row_end, float* pctr_out,
                                     uint8_t* labels_out) {
  if (!m || !tr) { xf_set_error("null argument"); return XF_ERR_ARG; }
  XF_TRY(xf_refuse_part(m, "xf_model_predict_ingested"));
  XF_TRY(xf_check_fields_kind(m, false, "xf_model_predict_ingested"));
  if (m->fm == XF_SERVE_FMC) {
    xf_set_error("xf_model_predict_ingested: a canonical model reads feature values, which an ingested text block does "
                 "not carry: use xf_model_predict_host_values / _device_values");
    return XF_ERR_ARG;
  }
  if (tr->cfg.model != (m->fm ? XF_MODEL_FM : XF_MODEL_LR)) {
    xf_set_error("xf_model_predict_ingested: the trainer's model (%d) is not the serving model's (%s)", tr->cfg.model,
                 m->fm ? "FM" : "LR");
    return XF_ERR_ARG;
  }
  if (tr->table->cfg.device != m->device) {
    xf_set_error("xf_model_predict_ingested: the trainer's block is on device %d, the model on device %d",
                 tr->table->cfg.device, m->device);
    return XF_ERR_ARG;
  }
  XF_TRY(xf_ingested_range(tr, row_start, row_end));
  const uint32_t rows = row_end - row_start;
  if (rows == 0) return XF_OK;
  if (!pctr_out) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lock(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  xf_trainer::IngestSet& g = tr->ing[tr->ing_cur];
  cudaStream_t st = tr->table->stream;  // the block's parse is ordered before this stream's work
  XF_TRY(m->s_out.ensure((size_t)rows * 4));
  // row_ptr holds absolute token offsets: a slice is a shifted row_ptr
  xf_launch_predict(m, g.row_ptr.as<uint32_t>() + row_start, g.keys.as<uint64_t>(), nullptr, nullptr, rows,
                    m->s_out.as<float>(), st);
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(pctr_out, m->s_out.p, (size_t)rows * 4, cudaMemcpyDeviceToHost, st));
  if (labels_out) XF_CUDA_TRY(cudaMemcpyAsync(labels_out, g.labels.as<uint8_t>() + row_start, rows, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaEventRecord(g.consumed, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  return XF_OK;
}

// what a canonical model holds for n host keys: w[n], v[n][K], present[n] (any output may be NULL)
static int xf_lookup_fmc(xf_model* m, const uint64_t* keys, uint64_t n, float* w, float* v, uint8_t* present) {
  if (n == 0) return XF_OK;
  const uint64_t K = (uint64_t)m->view.K;
  std::lock_guard<std::mutex> lock(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  XF_TRY(m->s_keys.ensure(n * 8));
  XF_TRY(m->s_aux.ensure(n * (4 * K + 5)));  // v[n][K] w[n] present[n]
  float* d_v = m->s_aux.as<float>();
  float* d_w = d_v + n * K;
  uint8_t* d_present = reinterpret_cast<uint8_t*>(d_w + n);
  XF_CUDA_TRY(cudaMemcpyAsync(m->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, m->stream));
  xf_with_precision(m, [&](auto H) {
    xf_k_model_lookup_fmc<H><<<xf_grid_for(n, 256, 8), 256, 0, m->stream>>>(m->view, m->s_keys.as<uint64_t>(), n, d_w,
                                                                           v ? d_v : nullptr, d_present);
  });
  XF_CUDA_TRY(cudaGetLastError());
  if (w) XF_CUDA_TRY(cudaMemcpyAsync(w, d_w, n * 4, cudaMemcpyDeviceToHost, m->stream));
  if (v) XF_CUDA_TRY(cudaMemcpyAsync(v, d_v, n * K * 4, cudaMemcpyDeviceToHost, m->stream));
  if (present) XF_CUDA_TRY(cudaMemcpyAsync(present, d_present, n, cudaMemcpyDeviceToHost, m->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(m->stream));
  return XF_OK;
}

XF_DLL int xf_model_lookup_latent(xf_model* m, const uint64_t* keys, uint64_t n, float* w, float* v, uint8_t* present) {
  if (!m || (!keys && n)) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (!xf_serve_latent_rows(m->fm)) {
    xf_set_error("xf_model_lookup_latent: an %s model holds no latent rows: use xf_model_lookup", m->fm ? "FM" : "LR");
    return XF_ERR_ARG;
  }
  XF_TRY(xf_check_host_keys(keys, n, "xf_model_lookup_latent"));
  return xf_lookup_fmc(m, keys, n, w, v, present);
}

XF_DLL int xf_model_lookup(xf_model* m, const uint64_t* keys, uint64_t n, float* w, float* st, float* qt, uint8_t* present) {
  if (!m || (!keys && n)) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (xf_serve_latent_rows(m->fm)) {
    if (st || qt) {
      xf_set_error("xf_model_lookup: a %s model holds no st, qt: pass NULL, and read its latent rows with "
                   "xf_model_lookup_latent", m->fm == XF_SERVE_MVM ? "multi-view machine's"
                                             : m->fm == XF_SERVE_FFM ? "field-aware FM's" : "canonical");
      return XF_ERR_ARG;
    }
    XF_TRY(xf_check_host_keys(keys, n, "xf_model_lookup"));
    return xf_lookup_fmc(m, keys, n, w, nullptr, present);
  }
  XF_TRY(xf_check_host_keys(keys, n, "xf_model_lookup"));
  if (n == 0) return XF_OK;
  std::lock_guard<std::mutex> lock(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  XF_TRY(m->s_keys.ensure(n * 8));
  XF_TRY(m->s_aux.ensure(n * 13));  // w[n] st[n] qt[n] present[n]
  float* d_w = m->s_aux.as<float>();
  uint8_t* d_present = reinterpret_cast<uint8_t*>(d_w + 3 * n);
  XF_CUDA_TRY(cudaMemcpyAsync(m->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, m->stream));
  xf_with_precision(m, [&](auto H) {
    xf_k_model_lookup<H><<<xf_grid_for(n, 256, 8), 256, 0, m->stream>>>(m->view, m->s_keys.as<uint64_t>(), n, d_w, d_w + n,
                                                                       d_w + 2 * n, d_present);
  });
  XF_CUDA_TRY(cudaGetLastError());
  if (w) XF_CUDA_TRY(cudaMemcpyAsync(w, d_w, n * 4, cudaMemcpyDeviceToHost, m->stream));
  if (st) XF_CUDA_TRY(cudaMemcpyAsync(st, d_w + n, n * 4, cudaMemcpyDeviceToHost, m->stream));
  if (qt) XF_CUDA_TRY(cudaMemcpyAsync(qt, d_w + 2 * n, n * 4, cudaMemcpyDeviceToHost, m->stream));
  if (present) XF_CUDA_TRY(cudaMemcpyAsync(present, d_present, n, cudaMemcpyDeviceToHost, m->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(m->stream));
  return XF_OK;
}

// ---- file
static bool xf_write(FILE* f, const void* p, size_t n) { return n == 0 || fwrite(p, 1, n, f) == n; }
static bool xf_read(FILE* f, void* p, size_t n) { return n == 0 || fread(p, 1, n, f) == n; }

int xf_chunks_save(FILE* f, const char* name, uint64_t n, uint32_t bytes, uint64_t per_chunk, uint64_t* chunk, XfPinBuf& pin,
                   cudaStream_t st, const std::function<int(uint64_t first, uint64_t c, const void** dev)>& src) {
  if (n == 0) return XF_OK;
  XF_TRY(pin.ensure(std::min(per_chunk, n) * bytes));
  for (uint64_t first = 0; first < n; first += per_chunk, ++*chunk) {
    const uint64_t c = std::min(per_chunk, n - first);
    const void* dev = nullptr;
    XF_TRY(src(first, c, &dev));
    XF_CUDA_TRY(cudaMemcpyAsync(pin.p, dev, c * bytes, cudaMemcpyDeviceToHost, st));
    XF_CUDA_TRY(cudaStreamSynchronize(st));
    const uint64_t head[4] = {first, c, xf_st_host_sum(pin.p, c * bytes, xf_st_tag(*chunk)), 0ull};
    if (!xf_write(f, head, sizeof(head)) || !xf_write(f, pin.p, c * bytes)) {
      xf_set_error("write to %s failed", name);
      return XF_ERR_IO;
    }
  }
  return XF_OK;
}

int xf_chunks_load(FILE* f, const char* path, uint64_t n, uint32_t bytes, uint64_t per_chunk, uint64_t* chunk,
                   const XfChunkCheck& check, XfPinBuf& pin, cudaStream_t st,
                   const std::function<int(uint64_t first, uint64_t c, const void* host)>& sink) {
  if (n == 0) return XF_OK;
  XF_TRY(pin.ensure(std::min(per_chunk, n) * bytes));
  uint64_t lo = 0, hi = 0, prev = 0;
  xf_shard_range(check.shard_index, check.num_shards, &lo, &hi);
  for (uint64_t first = 0; first < n; first += per_chunk, ++*chunk) {
    const uint64_t c = std::min(per_chunk, n - first);
    uint64_t head[4];
    if (!xf_read(f, head, sizeof(head)) || !xf_read(f, pin.p, c * bytes)) {
      xf_set_error("truncated %s %s", check.file, path);
      return XF_ERR_IO;
    }
    if (head[0] != first || head[1] != c || head[3] != 0 || head[2] != xf_st_host_sum(pin.p, c * bytes, xf_st_tag(*chunk))) {
      xf_set_error("%s %s: chunk %llu is damaged (checksum mismatch)", check.file, path, (unsigned long long)*chunk);
      return XF_ERR_IO;
    }
    const uint8_t* p = pin.as<uint8_t>();
    for (uint64_t r = first; r < first + c; ++r, p += bytes) {
      uint64_t key;
      memcpy(&key, p, 8);
      if ((r > 0 && key <= prev) || key == XF_EMPTY_KEY) {
        xf_set_error("%s %s: the %s keys are not strictly ascending below 2^64 - 1 (entry %llu)", check.file, path, check.what,
                     (unsigned long long)r);
        return XF_ERR_IO;
      }
      prev = key;
      if (key < lo || key > hi) {
        xf_set_error("%s %s: key %016llx of %s %llu lies outside shard %d of %d", check.file, path, (unsigned long long)key,
                     check.what, (unsigned long long)r, check.shard_index, check.num_shards);
        return XF_ERR_IO;
      }
      if (check.fm >= 0 && !xf_model_padding_zero(p, check.fm, check.K, check.precision, bytes)) {
        xf_set_error("%s %s: %s %llu has non-zero padding", check.file, path, check.what, (unsigned long long)r);
        return XF_ERR_IO;
      }
    }
    XF_TRY(sink(first, c, pin.p));
    XF_CUDA_TRY(cudaStreamSynchronize(st));  // the pinned buffer is read again for the next chunk
  }
  return XF_OK;
}

int xf_file_size_check(FILE* f, const char* path, const char* file, uint64_t expect, uint64_t header_bytes) {
  if (fseek(f, 0, SEEK_END) != 0) { xf_set_error("cannot read %s", path); return XF_ERR_IO; }
  const long fsz = ftell(f);
  if (fsz < 0 || (uint64_t)fsz != expect) {
    xf_set_error("corrupt or truncated %s %s: %ld bytes, its header announces %llu", file, path, fsz, (unsigned long long)expect);
    return XF_ERR_IO;
  }
  if (fseek(f, (long)header_bytes, SEEK_SET) != 0) { xf_set_error("cannot read %s", path); return XF_ERR_IO; }
  return XF_OK;
}

bool xf_compat_sane(const XfCompat& c, uint32_t row_bytes) {
  if (c.precision != XF_PRECISION_F32 && c.precision != XF_PRECISION_F16) return false;
  if (c.fm == XF_SERVE_FMC || c.fm == XF_SERVE_FFM) {
    if (!xf_fmc_latent_ok(c.latent_dim)) return false;
  } else if (c.fm == XF_SERVE_MVM) {
    if (!xf_mvm_latent_ok(c.latent_dim)) return false;
  } else if (c.fm != (c.latent_dim > 0 ? 1 : 0) || c.latent_dim < 0 || (c.fm == XF_SERVE_LR && c.precision != XF_PRECISION_F32)) {
    return false;
  }
  if (row_bytes != xf_model_row_bytes(c.fm, c.latent_dim, c.precision)) return false;
  if (c.absent != XF_ABSENT_DEFAULT && c.absent != XF_ABSENT_ZERO) return false;
  if (c.optimizer != XF_OPT_FTRL && c.optimizer != XF_OPT_SGD && c.optimizer != XF_OPT_ADAGRAD) return false;
  return c.v_init == 0 || c.v_init == XF_INIT_COUNTER || c.v_init == XF_INIT_ZERO;
}

// the model header's side of the compatibility check (serve.cuh: XfCompat)
static XfCompat xf_compat_of(const XfModelHeader& h) {
  return XfCompat{h.fm, h.latent_dim, h.optimizer, h.absent, h.v_init, h.v_const, h.seed, (int)h.precision};
}

static int xf_sm_save_body(xf_model* m, FILE* f, const char* name) {
  XfModelHeader h;
  memset(&h, 0, sizeof(h));
  memcpy(h.magic, "XFSM", 4);
  h.version = XF_SM_VERSION;
  h.header_bytes = sizeof(h);
  h.keys = m->keys;
  h.capacity = m->view.mask + 1;
  h.row_bytes = m->view.stride;
  h.fm = m->fm;
  h.latent_dim = m->view.K;
  h.optimizer = m->optimizer;
  h.absent = m->absent;
  h.v_init = m->view.v_init;
  h.v_const = m->view.v_const;
  h.precision = (uint32_t)m->precision;
  h.seed = m->view.seed;
  h.source_keys = m->source_keys;
  h.pruned_keys = m->pruned_keys;
  h.chunk_rows = XF_ST_CHUNK_BYTES / h.row_bytes;
  bool wrote;
  if (m->num_shards) {
    // a part: XFSP, XFSM's fields and then the shard
    XfPartHeader p;
    memcpy(h.magic, "XFSP", 4);
    h.header_bytes = sizeof(XfPartHeader);
    memcpy(p.model, &h, sizeof(p.model));
    p.shard_index = m->shard_index;
    p.num_shards = m->num_shards;
    p.header_checksum = xf_st_host_sum(&p, offsetof(XfPartHeader, header_checksum), 0);
    wrote = xf_write(f, &p, sizeof(p));
  } else {
    h.header_checksum = xf_st_host_sum(&h, offsetof(XfModelHeader, header_checksum), 0);
    wrote = xf_write(f, &h, sizeof(h));
  }
  if (!wrote) { xf_set_error("write to %s failed", name); return XF_ERR_IO; }
  const uint64_t n = m->keys;
  if (n == 0) return XF_OK;
  // (key, slot) of every row, sorted by key on the device; then the rows in that order, a chunk at a time gathered
  cudaStream_t st = m->stream;
  XfSortedSlots sorted;
  XfDevBuf rows;
  struct Release { XfSortedSlots* s; XfDevBuf* r; ~Release() { s->release(); r->release(); } } rel{&sorted, &rows};
  XF_TRY(xf_model_list_sorted(m->view, n, sorted, st));
  XF_TRY(rows.ensure(std::min<uint64_t>(h.chunk_rows, n) * h.row_bytes));
  uint64_t chunk = 0;
  return xf_chunks_save(f, name, n, h.row_bytes, h.chunk_rows, &chunk, m->h_out, st,
                        [&](uint64_t first, uint64_t c, const void** dev) {
                          *dev = rows.p;
                          return xf_model_gather(m->view, sorted.slots_out.as<uint32_t>() + first, c, rows.p, st);
                        });
}

XF_DLL int xf_model_save(xf_model* m, const char* path) {
  if (!m || !path) { xf_set_error("null argument"); return XF_ERR_ARG; }
  std::lock_guard<std::mutex> lock(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  return xf_save_atomic(path, [&](FILE* f, const char* name) { return xf_sm_save_body(m, f, name); });
}

// the header's own consistency (after its checksum): every size derived from it is bounded before it is used
static bool xf_sm_header_sane(const XfModelHeader& h) {
  if (!xf_compat_sane(xf_compat_of(h), h.row_bytes)) return false;
  if (h.keys > (1ull << 31) || h.capacity != xf_model_capacity(h.keys) || h.keys + h.pruned_keys != h.source_keys) return false;
  return h.chunk_rows == XF_ST_CHUNK_BYTES / h.row_bytes;
}

// the rows of an XFSM or XFSP file (header of `header_bytes`) into `m` on `device`; m->shard_index, num_shards are set:
// a part's keys must lie in its shard's range
static int xf_sm_load_body(xf_model* m, int device, FILE* f, const char* path, const XfModelHeader& h, uint64_t header_bytes) {
  XF_TRY(xf_model_init(m, device, xf_compat_of(h)));
  XF_TRY(xf_file_size_check(f, path, "model file", header_bytes + xf_section_bytes(h.keys, h.row_bytes, h.chunk_rows),
                            header_bytes));
  m->keys = h.keys;
  m->source_keys = h.source_keys;
  m->pruned_keys = h.pruned_keys;
  XF_TRY(xf_model_alloc(m, h.capacity));
  if (h.keys == 0) { XF_CUDA_TRY(cudaStreamSynchronize(m->stream)); return XF_OK; }
  XfDevBuf rows, err;
  struct Release { XfDevBuf* b[2]; ~Release() { for (XfDevBuf* x : b) x->release(); } } rel{{&rows, &err}};
  XF_TRY(rows.ensure(std::min<uint64_t>(h.chunk_rows, h.keys) * h.row_bytes));
  XF_TRY(err.ensure(4));
  XF_CUDA_TRY(cudaMemsetAsync(err.p, 0, 4, m->stream));
  XfChunkCheck check{"model file", "row", h.fm, h.latent_dim, (int)h.precision, m->shard_index, m->num_shards};
  uint64_t chunk = 0;
  XF_TRY(xf_chunks_load(f, path, h.keys, h.row_bytes, h.chunk_rows, &chunk, check, m->h_in, m->stream,
                        [&](uint64_t, uint64_t c, const void* host) -> int {
                          XF_CUDA_TRY(cudaMemcpyAsync(rows.p, host, c * h.row_bytes, cudaMemcpyHostToDevice, m->stream));
                          return xf_model_insert_rows(m->view, rows.as<uint8_t>(), c, err.as<int>(), m->stream);
                        }));
  int e = 0;
  XF_CUDA_TRY(cudaMemcpy(&e, err.p, 4, cudaMemcpyDeviceToHost));
  if (e) { xf_set_error("model file %s: a probe sequence of the model overflowed", path); return XF_ERR_IO; }
  return XF_OK;
}

XF_DLL int xf_model_load(xf_model** out, const char* path, int device) {
  if (out) *out = nullptr;
  if (!out || !path) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (device < 0 || device >= xf_device_count()) { xf_set_error("xf_model_load: no CUDA device %d", device); return XF_ERR_CUDA; }
  FILE* f = fopen(path, "rb");
  if (!f) { xf_set_error("cannot open %s", path); return XF_ERR_IO; }
  XfPartHeader p;  // an XFSP header; an XFSM one is its first 104 bytes
  memset(&p, 0, sizeof(p));
  const size_t got = fread(&p, 1, sizeof(p), f);
  XfModelHeader h;
  memcpy(&h, &p, sizeof(h));
  const bool part = got >= 4 && memcmp(h.magic, "XFSP", 4) == 0;
  const size_t hbytes = part ? sizeof(XfPartHeader) : sizeof(XfModelHeader);
  int rc = XF_OK;
  if (xf_refuse_foreign(h.magic, got, path, "XFSMXFSP") != XF_OK) {
    rc = XF_ERR_IO;
  } else if (got < 4 || (memcmp(h.magic, "XFSM", 4) != 0 && !part)) {
    xf_set_error("%s is not a serving model (no XFSM or XFSP magic)", path);
    rc = XF_ERR_IO;
  } else if (got < hbytes || h.header_bytes != hbytes || h.version != XF_SM_VERSION) {
    xf_set_error("model file %s: truncated header or unknown version %u", path, h.version);
    rc = XF_ERR_IO;
  } else if (!part && (h.header_checksum != xf_st_host_sum(&h, offsetof(XfModelHeader, header_checksum), 0) ||
                       !xf_sm_header_sane(h))) {
    xf_set_error("model file %s: the header is damaged (checksum mismatch)", path);
    rc = XF_ERR_IO;
  } else if (part && (p.header_checksum != xf_st_host_sum(&p, offsetof(XfPartHeader, header_checksum), 0) ||
                      !xf_sm_header_sane(h) || xf_serve_latent_rows(h.fm))) {
    xf_set_error("model part file %s: the header is damaged (checksum mismatch)", path);
    rc = XF_ERR_IO;
  } else if (part && (p.num_shards < 1 || p.shard_index < 0 || p.shard_index >= p.num_shards)) {
    xf_set_error("model part file %s: shard %d of %d does not exist", path, p.shard_index, p.num_shards);
    rc = XF_ERR_IO;
  }
  xf_model* m = nullptr;
  if (rc == XF_OK) {
    m = new xf_model;
    if (part) {
      m->shard_index = p.shard_index;
      m->num_shards = p.num_shards;
    }
    rc = xf_sm_load_body(m, device, f, path, h, hbytes);
  }
  fclose(f);
  if (rc != XF_OK) { xf_model_free(m); return rc; }
  *out = m;
  return XF_OK;
}

// ---- merge
// the body of xf_model_merge (the parts checked): on failure the caller frees `m`
static int xf_merge_into(xf_model* const* parts, int n, int device, xf_model* m) {
  XF_TRY(xf_model_init(m, device, xf_compat_of(parts[0])));
  cudaStream_t st = m->stream;
  for (int i = 0; i < n; ++i) {
    m->keys += parts[i]->keys;
    m->source_keys += parts[i]->source_keys;
    m->pruned_keys += parts[i]->pruned_keys;
  }
  XF_TRY(xf_model_alloc(m, xf_model_capacity(m->keys)));
  XfDevBuf err, stage;
  struct Release { XfDevBuf* b[2]; ~Release() { for (XfDevBuf* x : b) x->release(); } } rel{{&err, &stage}};
  XF_TRY(err.ensure(4));
  XF_CUDA_TRY(cudaMemsetAsync(err.p, 0, 4, st));
  const uint32_t stride = m->view.stride;
  auto launch = [&](const uint8_t* slots, uint64_t c) -> int {
    xf_k_merge<<<xf_grid_for(c, 256, 8), 256, 0, st>>>(slots, c, m->view, err.as<int>());
    XF_CUDA_TRY(cudaGetLastError());
    return XF_OK;
  };
  for (int i = 0; i < n; ++i) {
    const xf_model* q = parts[i];
    const uint64_t slots = q->view.mask + 1;
    if (q->device == device) {  // read in place
      XF_TRY(launch(q->view.base, slots));
      continue;
    }
    // another device: its slots come over by peer copy, 64 MiB at a time, into one staging buffer that the stream's
    // order hands from each chunk's kernel to the next chunk's copy
    const uint64_t per = XF_ST_CHUNK_BYTES / stride;
    XF_TRY(stage.ensure(std::min(per, slots) * stride));
    for (uint64_t first = 0; first < slots; first += per) {
      const uint64_t c = std::min(per, slots - first);
      XF_CUDA_TRY(cudaMemcpyPeerAsync(stage.p, device, q->view.base + first * stride, q->device, c * stride, st));
      XF_TRY(launch(stage.as<uint8_t>(), c));
    }
  }
  int e = 0;
  XF_CUDA_TRY(cudaMemcpyAsync(&e, err.p, 4, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  if (e) {
    xf_set_error("xf_model_merge: a probe sequence of the model overflowed");
    return XF_ERR_FULL;
  }
  return XF_OK;
}

XF_DLL int xf_model_merge(xf_model* const* parts, int n, int device, xf_model** out) {
  if (out) *out = nullptr;
  if (!out || (!parts && n > 0)) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (n < 1) { xf_set_error("xf_model_merge: %d parts: a merge takes every part of one split", n); return XF_ERR_ARG; }
  std::vector<int> seen((size_t)n, -1);
  for (int i = 0; i < n; ++i) {
    const xf_model* q = parts[i];
    if (!q) { xf_set_error("null argument: parts[%d]", i); return XF_ERR_ARG; }
    if (q->num_shards == 0) {
      xf_set_error("xf_model_merge: parts[%d] is a whole model, not a part (xf_table_freeze_part makes parts)", i);
      return XF_ERR_ARG;
    }
    if (q->num_shards != n) {
      xf_set_error("xf_model_merge: parts[%d] is shard %d of a %d-way split, but %d parts were passed: a merge takes "
                   "every part of one split, each once", i, q->shard_index, q->num_shards, n);
      return XF_ERR_ARG;
    }
    if (seen[(size_t)q->shard_index] >= 0) {
      xf_set_error("xf_model_merge: shard %d is passed twice (parts[%d] and parts[%d]), so another shard is missing",
                   q->shard_index, seen[(size_t)q->shard_index], i);
      return XF_ERR_ARG;
    }
    seen[(size_t)q->shard_index] = i;
    if (const char* f = xf_compat_diff(xf_compat_of(parts[0]), xf_compat_of(q))) {
      xf_set_error("xf_model_merge: parts[0] and parts[%d] differ in %s: the parts of one model read absent keys alike", i, f);
      return XF_ERR_ARG;
    }
  }
  const int target = device < 0 ? parts[0]->device : device;
  if (target >= xf_device_count()) { xf_set_error("xf_model_merge: no CUDA device %d", target); return XF_ERR_ARG; }
  xf_model* m = new xf_model;
  const int rc = xf_merge_into(parts, n, target, m);
  if (rc != XF_OK) { xf_model_free(m); return rc; }
  *out = m;
  return XF_OK;
}

// ---- convert
// the body of xf_model_convert: on failure the caller frees `out`
static int xf_convert_into(xf_model* m, int precision, xf_model* out) {
  XfCompat c = xf_compat_of(m);
  c.precision = precision;
  XF_TRY(xf_model_init(out, m->device, c));
  out->keys = m->keys;
  out->source_keys = m->source_keys;
  out->pruned_keys = m->pruned_keys;
  out->shard_index = m->shard_index;
  out->num_shards = m->num_shards;
  cudaStream_t st = out->stream;
  XF_TRY(xf_model_alloc(out, m->view.mask + 1));
  if (precision == m->precision) {
    // a copy: the same rows at the same stride and capacity, so the same slots
    XF_CUDA_TRY(cudaMemcpyAsync(out->view.base, m->view.base, (m->view.mask + 1) * (uint64_t)m->view.stride,
                                cudaMemcpyDeviceToDevice, st));
    XF_CUDA_TRY(cudaStreamSynchronize(st));
    return XF_OK;
  }
  XfDevBuf aux;  // {overflowing fields, their smallest key, probe error}
  struct Release { XfDevBuf* a; ~Release() { a->release(); } } rel{&aux};
  XF_TRY(aux.ensure(24));
  unsigned long long* d_over = aux.as<unsigned long long>();
  int* d_error = reinterpret_cast<int*>(d_over + 2);
  XF_CUDA_TRY(cudaMemsetAsync(d_over, 0, 8, st));
  XF_CUDA_TRY(cudaMemsetAsync(d_over + 1, 0xFF, 8, st));
  XF_CUDA_TRY(cudaMemsetAsync(d_error, 0, 4, st));
  const int grid = xf_grid_for(m->view.mask + 1, 256, 8);
  const bool to_half = precision == XF_PRECISION_F16;
  if (xf_serve_latent_rows(m->fm)) {  // a multi-view machine's zero word is copied as a canonical row's w
    if (to_half) xf_k_model_convert<true, true><<<grid, 256, 0, st>>>(m->view, out->view, d_over, d_error);
    else xf_k_model_convert<true, false><<<grid, 256, 0, st>>>(m->view, out->view, d_over, d_error);
  } else {
    if (to_half) xf_k_model_convert<false, true><<<grid, 256, 0, st>>>(m->view, out->view, d_over, d_error);
    else xf_k_model_convert<false, false><<<grid, 256, 0, st>>>(m->view, out->view, d_over, d_error);
  }
  XF_CUDA_TRY(cudaGetLastError());
  unsigned long long h[3] = {0, 0, 0};
  XF_CUDA_TRY(cudaMemcpyAsync(h, d_over, 24, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  if ((int)h[2] != 0) {
    xf_set_error("xf_model_convert: a probe sequence of the model overflowed");
    return XF_ERR_FULL;
  }
  if (h[0] != 0) {
    xf_set_error("xf_model_convert: %llu latent fields are finite in float32 but not in binary16 (|x| >= 65520), the "
                 "smallest key that holds one is %llu (%016llx): conversion never saturates", h[0], h[1], h[1]);
    return XF_ERR_STATE;
  }
  return XF_OK;
}

XF_DLL int xf_model_convert(xf_model* m, int precision, xf_model** out) {
  if (out) *out = nullptr;
  if (!m || !out) { xf_set_error("null argument"); return XF_ERR_ARG; }
  if (precision != XF_PRECISION_F32 && precision != XF_PRECISION_F16) {
    xf_set_error("xf_model_convert: precision = %d is not an XF_PRECISION_* value", precision);
    return XF_ERR_ARG;
  }
  if (m->fm == XF_SERVE_LR) {
    xf_set_error("xf_model_convert: an LR model has no latent fields to narrow (its row is a key and w in 16 bytes)");
    return XF_ERR_ARG;
  }
  xf_model* c = new xf_model;
  const int rc = xf_convert_into(m, precision, c);
  if (rc != XF_OK) { xf_model_free(c); return rc; }
  *out = c;
  return XF_OK;
}

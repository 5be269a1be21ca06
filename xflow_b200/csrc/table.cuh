// Device-side layout and primitives of the GPU-resident parameter table.
//
// The table replaces the reference's server-side state — the two
// std::unordered_map<ps::Key, FTRLEntry/SGDEntry> stores behind KV apps 0 (w) and 1 (v)
// (src/optimizer/ftrl.h:27-36,84,87-96,151 ; src/optimizer/sgd.h:23-28,61,67-72,105) —
// with ONE open-addressing hash table in HBM whose row holds everything a key owns:
//
//   byte  0  u64  key            (EMPTY = 2^64-1; never a legal key in the reference either:
//                                 it lies outside every server range, postoffice.cc:134-143)
//   byte  8  f64  g              per-batch gradient accumulator of w; -0.0 == "untouched this batch".
//                                Double, so that the sum over a key's occurrences is exact to float
//                                precision whatever order the L2 atomics land in (deterministic, and
//                                more accurate than the reference's own sequential float sum).
//                                (LAZY tables keep their sum elsewhere, see below)
//   byte 16  f32  w              app-0 weight                         (FTRLEntry_w::w / SGDEntry_w::w)
//   byte 20  f32  n              FTRL / AdaGrad accumulator of w (unused by SGD)
//   byte 24  f32  z              FTRL accumulator of w (unused by SGD; 0 under AdaGrad)
//   byte 28  u32  flags          bit0 = latent block materialised (V_READY)
//   LAZY tables (LR, K == 0, "update on next touch", step_lazy.cu) use bytes 16..31 differently, so that ONE
//   128-bit compare-and-swap on that aligned word can fold a pending optimizer step in, stamp the row for the
//   current batch and deposit the first residual, all at once:
//     byte 16  f32 n, byte 20 f32 z   (FTRL; the weight is not stored: w = f(z, n), the closed form the
//                                      reference's handle evaluates after every push, ftrl.h:66-74)
//              f32 w, byte 20 unused  (SGD)
//              f32 w, byte 20 f32 n   (AdaGrad)
//     byte  8  f32 w_given, u32 check   a weight set from outside (xf_table_import) that is NOT f(z, n): it stands
//                                      for w until the first optimizer step after the import is folded in
//                                      (check = a digest of bytes 16..23, re-marked by the batch that first opens
//                                      the row: xf_lazy_given; the reference would likewise use the stored w in its
//                                      next step and then overwrite it with f(z', n'))
//     byte 24  u64 { tag : 16 (low) | g : 48 (high) }   tag = the batch whose residual sum is pending in g
//                                      (0: none); g = that sum as a signed FIXED-POINT integer of the batch's
//                                      unit 2^-s (xf_fix_shift: s = 27 below 2^20 tokens, smaller above, so
//                                      that no sum can leave the 48 bits): integer adds are exactly
//                                      associative, so the result does not depend on the order the atomics
//                                      land in (bit-reproducible), and an add of x << 16 never disturbs the
//                                      tag below it.
//   ---- 32 B = one DRAM sector: an LR pull, gradient accumulate or update touches exactly one ----
//   byte 32            f32 v[K]    app-1 latent row
//   byte A             f64 L, f64 Aq   per-batch latent-gradient accumulators, A = round_up(32 + 4K, 16).
//                                  The reference's gv[i,k] = sum_occ loss_s * (S_s - v[i,k])
//                                  (fm_worker.cc:141-142) factorises as Aq_i - v[i,k] * L_i with
//                                  L_i = sum_occ loss_s and Aq_i = sum_occ loss_s * S_s: two f64
//                                  accumulators per key instead of K float ones (3 atomics per token
//                                  instead of 1 + K/4 vector ones, and no second read of v).
//   byte A + 16        f32 nv[K]   (FTRL and AdaGrad)
//   byte A + 16 + 4K   f32 zv[K]   (FTRL only)
//   row stride = round_up(A + 16 + (FTRL ? 8K : AdaGrad ? 4K : 0), 32): K = 16 FTRL -> 256 B, AdaGrad -> 192 B.
//
// Missing keys are inserted on first touch by a pull OR a push, like `store[key]`
// (ftrl.h:56,114-120 ; sgd.h:48,92).  Default contents: w = n = z = 0 ; v per init mode.  The latent
// block is materialised lazily by the first update of the key (a row is only ever written by
// kernels that own the key exclusively); until then readers compute the same deterministic
// initial value from (key, k, seed), so "insert on pull" is observably identical.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define XF_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull
#define XF_FLAG_V_READY 1u
#define XF_NEG_ZERO_BITS 0x80000000u
#define XF_NEG_ZERO_BITS64 0x8000000000000000ull
#define XF_MAX_PROBE 8192

enum { XF_OPT_FTRL = 0, XF_OPT_SGD = 1, XF_OPT_ADAGRAD = 2 };  // = XF_OPTIMIZER_*
enum { XF_INIT_DEFAULT = 0, XF_INIT_COUNTER = 1, XF_INIT_ZERO = 3 };

struct XfTableView {
  uint8_t* base;
  uint64_t mask;      // capacity - 1
  uint32_t log2cap;
  uint32_t bshift;    // log2 of the slots per probing bucket (see xf_probe_slot)
  uint32_t stride;    // bytes per row
  int K;
  int opt;
  int v_init;         // resolved: 0 const(v_const), 1 counter normal, 3 zero
  float v_const;
  uint64_t seed;
  float alpha, beta, lambda1, lambda2, learning_rate;
  unsigned long long* size;   // number of keys present
  int* error;                 // set to 1 when a probe sequence overflows (table full)
  // "update on next touch" (K == 0 tables, see step.cu): the flags word of a row is then a TAG =
  // sequence number of the batch whose residual sum sits in g (0: nothing pending, XF_TAG_LOCKED: a
  // thread is folding the pending step into the row right now); rows_by_seq[tag] is that batch's row
  // count (the divisor of lr_worker.cc:116-118) in the low 32 bits and the fixed-point shift s of its residual
  // sums (xf_fix_shift) above them.  Every reader applies a pending step on the fly.
  int lazy;
  const uint64_t* rows_by_seq;
  // canonical per-k FM (step_fmc.cu; not the reference's model, SURVEY 8f-4): rows carry K more float
  // accumulators A[k] = sum_occ loss x S_k behind the optimizer state
  int canon;
};
// Feature admission (admit.cu): which ABSENT keys a training step may insert.  Only the admitting instantiations
// of the step kernels take it; a token whose key is absent and not admitted is "rejected": it reads as a row of
// zeros, updates nothing, and its key is appended to the rejected-token list for the Bloom filter's count pass.
#define XF_ADM_POISSON 1  // = XF_ADMIT_POISSON: admit iff top 24 bits of splitmix64(key ^ batch_mix) < p24
#define XF_ADM_BLOOM 2    // = XF_ADMIT_BLOOM: admit iff min over the key's cells >= threshold
#define XF_ADM_NEVER 3    // predict with a policy set: insert nothing, count nothing
#define XF_ADM_MAX_HASHES 8
struct XfAdmitView {
  int mode;
  uint32_t p24;                          // floor(p * 2^24)
  uint64_t batch_mix;                    // splitmix64(seed + b), b = the table's training-batch number
  uint32_t threshold, log2_cells, hashes;
  uint64_t seed;                         // the policy's seed (the Bloom cells: xf_admit_cell)
  const uint8_t* cells;                  // 2^log2_cells one-byte saturating counters
  unsigned long long* rej_n;             // append position of the rejected-token list (Poisson: the stats counter)
  uint64_t* rej_keys;                    // the list (nullptr: count only)
  unsigned long long* admitted;          // keys inserted by admission (stats)
};
// Feature eviction (evict.cu): which keys a sweep keeps, as one predicate on (stamp, key).  Order: a larger stamp is
// more recent, and between equal stamps the smaller key is.  A key is kept iff stamp >= cutoff and, if bounded, it is
// at least as recent as the boundary (s_star, k_star).  Growth keeps every key (cutoff 0, not bounded).
struct XfKeep {
  uint32_t cutoff;
  int bounded;
  uint32_t s_star;
  uint64_t k_star;
};
// Feature eviction (xf_table_set_eviction, evict.cu): stamp[slot] = the training-batch number that last touched the
// slot's key (nullptr: tracking off); now = the table's batch number when the kernel was launched.  A kernel
// parameter of its own, passed last: inside XfTableView it changed how ptxas allocates the FM step's registers.
struct XfStampView {
  uint32_t* stamp;
  uint32_t now;
};
// Importance weighting (weight.cu): e[row] = the effective weight of each row of the step (0: the row is skipped) and
// *W = sum over trained rows of ceil(e) x tokens, the bound the lazy step derives its fixed-point unit from.  Only the
// weighting instantiations of the step kernels read it; a kernel parameter of its own, passed last, like XfStampView.
struct XfWeightView {
  const float* e;
  const unsigned long long* W;
};
__host__ __device__ __forceinline__ bool xf_keeps(const XfKeep& k, uint32_t stamp, uint64_t key) {
  return stamp >= k.cutoff && (!k.bounded || stamp > k.s_star || (stamp == k.s_star && key <= k.k_star));
}
#define XF_TAG_LOCKED 0xFFFFFFFFu  // never a batch number (the sequence ring is far smaller)
#define XF_FIX_MAX_SHIFT 27    // the finest unit of a lazy table's residual sums: 2^-27
#define XF_TAG_MASK 0xFFFFull  // lazy rows: low 16 bits of the word at byte 24

// The unit 2^-s of a lazy batch's residual sums, from a bound on its token count: every |residual| <= 1, so a key's
// sum over the batch is at most nnz in magnitude, and each token's residual is rounded to a multiple of 2^-s before it
// is added, which keeps every partial sum within nnz * 2^s units.  The largest s <= 27 with nnz * 2^s <= 2^47 - 1 keeps
// that inside the 48-bit signed field: s = 27 below 2^20 tokens, 24 for 6.5 M.
__host__ __device__ inline int xf_fix_shift(uint64_t nnz) {
  int bits = 0;  // bit length of nnz: nnz < 2^bits
  while (bits < 64 && (nnz >> bits) != 0ull) ++bits;
  const int s = 47 - bits;
  return s > XF_FIX_MAX_SHIFT ? XF_FIX_MAX_SHIFT : (s < 0 ? 0 : s);
}

__host__ __device__ inline uint32_t xf_acc_off(int K) { return (32u + 4u * (uint32_t)K + 15u) & ~15u; }
// floats of optimizer state per latent coordinate behind the accumulators: nv, zv (FTRL), nv (AdaGrad), none (SGD)
__host__ __device__ inline uint32_t xf_latent_state(int opt) { return opt == XF_OPT_FTRL ? 2u : (opt == XF_OPT_ADAGRAD ? 1u : 0u); }
__host__ __device__ inline uint32_t xf_ca_off(int K, int opt) {  // canonical FM: the A[K] accumulators
  return xf_acc_off(K) + 16u + 4u * xf_latent_state(opt) * (uint32_t)K;
}
__host__ __device__ inline uint32_t xf_row_stride(int K, int opt, int canon = 0) {
  if (K <= 0) return 32u;
  uint32_t bytes = xf_ca_off(K, opt) + (canon ? 4u * (uint32_t)K : 0u);
  return (bytes + 31u) & ~31u;
}

#ifdef __CUDACC__

// Probe sequence: BUCKETISED linear probing.  Slots are grouped in aligned buckets of B = 2^bshift slots
// that share one 128-byte line (LR: 4 rows of 32 B; FM rows are longer than a line: B = 1 = plain linear
// probing).  Probe i of a key visits its home bucket first — starting at a key-dependent slot and wrapping
// inside the bucket — and then the following buckets slot by slot.  Why: a warp waits for the slowest of its
// lanes, and every step of a linear-probing chain used to be one more DEPENDENT DRAM access (on the 1e8-id
// table at load 0.37 the longest chain among the 64 tokens a warp has in flight is several DRAM round trips).
// Inside a bucket the further probes hit the line the first one fetched (L2 fetch granularity = the bucket,
// xf_table_create); chains that leave the home bucket are rare
// (1.6 % of the keys at load 0.37 with B = 4, simulated; expected longest chain among 64 tokens 1.7 lines).
__device__ __forceinline__ uint64_t xf_probe_slot(const XfTableView& t, uint64_t key, uint32_t i) {
  const uint64_t m = key * 0x9E3779B97F4A7C15ull;
  const uint32_t bs = t.bshift;
  const uint64_t hb = m >> (64 - (t.log2cap - bs));  // home bucket
  const uint32_t b1 = (1u << bs) - 1u;
  const uint32_t j0 = (uint32_t)(m >> 9) & b1;       // where the walk through the home bucket starts
  const uint32_t k = i >> bs;
  const uint32_t j = (k == 0) ? ((j0 + i) & b1) : (i & b1);
  return (((hb + k) << bs) | j) & t.mask;
}
__device__ __forceinline__ uint64_t xf_home_slot(const XfTableView& t, uint64_t key) { return xf_probe_slot(t, key, 0); }

// ---- counter-based initial value of the latent table; must stay bit-identical to
// ---- oracle/xflow_oracle.cc: xo_counter_normal (integer ops + two exactly rounded float ops)
__host__ __device__ __forceinline__ uint64_t xf_splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// ---- admission hashes; must stay bit-identical to tests/admission_model.py (bloom_cells, poisson_admits)
// cell j of `key`: the top log2_cells bits of splitmix64(key ^ splitmix64(seed + (j + 1) * 0x9E3779B97F4A7C15))
__host__ __device__ __forceinline__ uint64_t xf_admit_cell(uint64_t key, uint64_t seed, uint32_t j, uint32_t log2_cells) {
  return xf_splitmix64(key ^ xf_splitmix64(seed + (uint64_t)(j + 1) * 0x9E3779B97F4A7C15ull)) >> (64 - log2_cells);
}
__device__ __forceinline__ bool xf_admit(const XfAdmitView& a, uint64_t key) {
  if (a.mode == XF_ADM_POISSON) return (uint32_t)(xf_splitmix64(key ^ a.batch_mix) >> 40) < a.p24;
  if (a.mode != XF_ADM_BLOOM) return false;
  uint32_t m = 255u;
  for (uint32_t j = 0; j < a.hashes; ++j) m = min(m, (uint32_t)__ldcg(a.cells + xf_admit_cell(key, a.seed, j, a.log2_cells)));
  return m >= a.threshold;
}
// Warp-aggregated append of the rejected tokens (r0: k0, r1: k1) to the list: one atomic per warp and chunk that has
// rejections, none otherwise.  All 32 lanes of the warp must call it together.
__device__ __forceinline__ void xf_admit_append(const XfAdmitView& a, bool r0, uint64_t k0, bool r1, uint64_t k1) {
  const unsigned m0 = __ballot_sync(0xffffffffu, r0), m1 = __ballot_sync(0xffffffffu, r1);
  if ((m0 | m1) == 0u) return;
  const unsigned lane = threadIdx.x & 31u;
  unsigned long long base = 0ull;
  if (lane == 0u) base = atomicAdd(a.rej_n, (unsigned long long)(__popc(m0) + __popc(m1)));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (a.rej_keys) {
    const unsigned lt = (1u << lane) - 1u;
    if (r0) a.rej_keys[base + __popc(m0 & lt)] = k0;
    if (r1) a.rej_keys[base + __popc(m0) + __popc(m1 & lt)] = k1;
  }
}
// The same for one token per lane (rejected: r, key k): one atomic per warp and 32 tokens that have rejections.
__device__ __forceinline__ void xf_admit_append(const XfAdmitView& a, bool r, uint64_t k) {
  const unsigned m = __ballot_sync(0xffffffffu, r);
  if (m == 0u) return;
  const unsigned lane = threadIdx.x & 31u;
  unsigned long long base = 0ull;
  if (lane == 0u) base = atomicAdd(a.rej_n, (unsigned long long)__popc(m));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (a.rej_keys && r) a.rej_keys[base + __popc(m & ((1u << lane) - 1u))] = k;
}

__device__ __forceinline__ float xf_counter_normal(uint64_t key, uint32_t k, uint64_t seed) {
  uint64_t base = xf_splitmix64(key ^ xf_splitmix64(seed + 0x632BE59BD9B4E019ull * (uint64_t)(k + 1)));
  uint32_t sum = 0;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    uint64_t x = xf_splitmix64(base + (uint64_t)r);
    sum += (uint32_t)(x & 0xFFFF) + (uint32_t)((x >> 16) & 0xFFFF) + (uint32_t)((x >> 32) & 0xFFFF) +
           (uint32_t)((x >> 48) & 0xFFFF);
  }
  float u = __fmul_rn((float)((int32_t)sum - 6 * 65535), 1.0f / 65536.0f);
  return __fmul_rn(u, 1e-2f);
}
__device__ __forceinline__ float xf_v_init(const XfTableView& t, uint64_t key, uint32_t k) {
  if (t.v_init == XF_INIT_COUNTER) return xf_counter_normal(key, k, t.seed);
  if (t.v_init == XF_INIT_ZERO) return 0.0f;
  return t.v_const;
}
// the initial values of latent piece q, coordinates 4q .. 4q+3 (the piece a lane of the canonical kernels holds)
__device__ __forceinline__ float4 xf_v_init_piece(const XfTableView& t, uint64_t key, uint32_t q) {
  return make_float4(xf_v_init(t, key, 4 * q), xf_v_init(t, key, 4 * q + 1), xf_v_init(t, key, 4 * q + 2),
                     xf_v_init(t, key, 4 * q + 3));
}

// ---- row accessors
__device__ __forceinline__ uint8_t* xf_row(const XfTableView& t, uint64_t slot) {
  return t.base + slot * (uint64_t)t.stride;
}
__device__ __forceinline__ double* xf_row_g(uint8_t* row) { return reinterpret_cast<double*>(row + 8); }
#define XF_OFF_STATE 16  // {w, n, z, flags}: one aligned 16-byte word
#define XF_OFF_FLAGS 28
__device__ __forceinline__ float* xf_row_v(uint8_t* row) { return reinterpret_cast<float*>(row + 32); }
__device__ __forceinline__ double* xf_row_acc(uint8_t* row, int K) { return reinterpret_cast<double*>(row + xf_acc_off(K)); }
__device__ __forceinline__ float* xf_row_nv(uint8_t* row, int K) { return reinterpret_cast<float*>(row + xf_acc_off(K) + 16); }
__device__ __forceinline__ float* xf_row_zv(uint8_t* row, int K) { return xf_row_nv(row, K) + K; }
__device__ __forceinline__ float* xf_row_ca(const XfTableView& t, uint8_t* row) { return reinterpret_cast<float*>(row + xf_ca_off(t.K, t.opt)); }

struct XfHead {
  uint64_t key;
  uint32_t flags;
  float w, n, z;
  double g;
};

// One 32-byte sector as two 128-bit loads from the same lane (sm_90 has no 256-bit LDG).  That is two
// instructions, and so two memory requests, per row: on a random multi-GB table it costs twice what one row look
// could (tools/membench.cu, "read" against "read pair"); xf_ld32_pair below reads the same rows with each
// instruction serving half the lanes' rows.  Each half is one 16-byte access, which is what the lazy protocol's
// 128-bit CAS on bytes 16..31 compares against.
__device__ __forceinline__ void xf_ld32_cg(const void* p, uint64_t& q0, uint64_t& q1, uint64_t& q2, uint64_t& q3) {
  asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%4];\n\tld.global.cg.v2.u64 {%2,%3}, [%4+16];"
               : "=l"(q0), "=l"(q1), "=l"(q2), "=l"(q3) : "l"(p));
}
__device__ __forceinline__ void xf_ld32_ca(const void* p, uint64_t& q0, uint64_t& q1, uint64_t& q2, uint64_t& q3) {
  asm volatile("ld.global.ca.v2.u64 {%0,%1}, [%4];\n\tld.global.ca.v2.u64 {%2,%3}, [%4+16];"
               : "=l"(q0), "=l"(q1), "=l"(q2), "=l"(q3) : "l"(p));
}
// The row at `mine` (nullptr: none; the result is then zero) read by lane PAIRS, through L2: lanes 2i and 2i+1
// each load one 16-byte half of the even lane's row in one instruction and of the odd lane's row in a second, then
// swap halves, so each lane ends up with its own whole row.  Still two LDG.128 per lane, but each instruction
// touches 16 rows rather than 32, which halves the requests per row (tools/membench.cu).  Both loads are issued
// before the swap, so they are in flight together.  All 32 lanes of the warp must call it together.
__device__ __forceinline__ void xf_ld32_pair(const uint8_t* mine, uint64_t& q0, uint64_t& q1, uint64_t& q2, uint64_t& q3) {
  const uint32_t odd = threadIdx.x & 1u;
  const uint8_t* other = (const uint8_t*)__shfl_xor_sync(0xffffffffu, (unsigned long long)mine, 1);
  const uint8_t* r0 = odd ? other : mine;  // the even lane's row
  const uint8_t* r1 = odd ? mine : other;  // the odd lane's row
  uint64_t x0 = 0, x1 = 0, y0 = 0, y1 = 0;
  asm volatile("{\n .reg .pred p0, p1;\n setp.ne.u64 p0, %4, 0;\n setp.ne.u64 p1, %5, 0;\n"
               " @p0 ld.global.cg.v2.u64 {%0,%1}, [%6];\n @p1 ld.global.cg.v2.u64 {%2,%3}, [%7];\n}"
               : "+l"(x0), "+l"(x1), "+l"(y0), "+l"(y1)
               : "l"(r0), "l"(r1), "l"(r0 + 16 * odd), "l"(r1 + 16 * odd));
  const uint64_t m0 = odd ? y0 : x0, m1 = odd ? y1 : x1;  // this lane's half of its own row
  const uint64_t t0 = __shfl_xor_sync(0xffffffffu, odd ? x0 : y0, 1);
  const uint64_t t1 = __shfl_xor_sync(0xffffffffu, odd ? x1 : y1, 1);
  q0 = odd ? t0 : m0; q1 = odd ? t1 : m1;
  q2 = odd ? m0 : t0; q3 = odd ? m1 : t1;
}
// the whole sector written by two 128-bit stores (no read-for-fill: L2 merges them into one full sector)
__device__ __forceinline__ void xf_st32(void* p, uint64_t q0, uint64_t q1, uint64_t q2, uint64_t q3) {
  asm volatile("st.global.v2.u64 [%0], {%1,%2};\n\tst.global.v2.u64 [%0+16], {%3,%4};" ::"l"(p), "l"(q0), "l"(q1),
               "l"(q2), "l"(q3)
               : "memory");
}

__device__ __forceinline__ XfHead xf_load_head(const uint8_t* row) {
  // the row's first 32-byte sector straight from L2 (L1 is useless for random rows)
  uint64_t q0, q1, q2, q3;
  xf_ld32_cg(row, q0, q1, q2, q3);
  XfHead h;
  h.key = q0;
  h.g = __longlong_as_double((long long)q1);
  h.w = __uint_as_float((uint32_t)q2);
  h.n = __uint_as_float((uint32_t)(q2 >> 32));
  h.z = __uint_as_float((uint32_t)q3);
  h.flags = (uint32_t)(q3 >> 32);
  return h;
}

// Same sector through L1 (ld.global.ca).  Only for kernels in which w / n / z / flags of existing rows do
// not change while the kernel runs (the eager step: it adds to g / gv with L2 atomics and inserts keys,
// nothing else).  A stale copy can then differ from L2 only by showing EMPTY for a slot that was claimed
// during this kernel — the insert CAS resolves that (xf_probe_from), and a row inserted during the kernel
// still has its default parameters.  With skewed ids this keeps each SM's reads of the hot rows local:
// through L2 every token of the hottest key queues on one slice (DESIGN.md section 4).
__device__ __forceinline__ XfHead xf_load_head_l1(const uint8_t* row) {
  uint64_t q0, q1, q2, q3;
  xf_ld32_ca(row, q0, q1, q2, q3);
  XfHead h;
  h.key = q0;
  h.g = __longlong_as_double((long long)q1);
  h.w = __uint_as_float((uint32_t)q2);
  h.n = __uint_as_float((uint32_t)(q2 >> 32));
  h.z = __uint_as_float((uint32_t)q3);
  h.flags = (uint32_t)(q3 >> 32);
  return h;
}

// eight consecutive floats of a latent row (one 32-byte sector) through L1 (read-only-for-the-kernel data,
// see xf_load_head_l1)
__device__ __forceinline__ void xf_ld8_l1(const float* p, float (&o)[8]) {
  uint64_t q0, q1, q2, q3;
  xf_ld32_ca(p, q0, q1, q2, q3);
  o[0] = __uint_as_float((uint32_t)q0); o[1] = __uint_as_float((uint32_t)(q0 >> 32));
  o[2] = __uint_as_float((uint32_t)q1); o[3] = __uint_as_float((uint32_t)(q1 >> 32));
  o[4] = __uint_as_float((uint32_t)q2); o[5] = __uint_as_float((uint32_t)(q2 >> 32));
  o[6] = __uint_as_float((uint32_t)q3); o[7] = __uint_as_float((uint32_t)(q3 >> 32));
}

template <int VEC>
__device__ __forceinline__ void xf_ldv_step(const float* p, float (&o)[VEC]) {
  // through L1: v does not change during the step kernel (see xf_load_head_l1), hot rows stay SM-local
  if (VEC == 4) { float4 t = __ldca(reinterpret_cast<const float4*>(p)); o[0] = t.x; o[1 % VEC] = t.y; o[2 % VEC] = t.z; o[3 % VEC] = t.w; }
  else if (VEC == 2) { float2 t = __ldca(reinterpret_cast<const float2*>(p)); o[0] = t.x; o[1 % VEC] = t.y; }
  else { o[0] = __ldca(p); }
}
// FM: (sum_k v, sum_k v^2) of one token's latent row  (fm_worker.cc:178-192, per-token part).  The step kernels
// (step.cu) and the freeze of a serving model (serve.cu) both reduce a row through this one function, so that a
// frozen row holds, bit for bit, what the forward pass computes.
template <int VEC>
__device__ __forceinline__ void xf_fm_token(const XfTableView& t, uint32_t slot, uint32_t flags, uint64_t key,
                                            float& st, float& qt) {
  const int K = t.K;
  st = 0.f;
  qt = 0.f;
  if ((flags & XF_FLAG_V_READY) && (K & 7) == 0) {
    // a sector at a time (the row starts 32-byte aligned)
    const float* vp = reinterpret_cast<const float*>(xf_row(t, slot) + 32);
    for (int k = 0; k < K; k += 8) {
      float v[8];
      xf_ld8_l1(vp + k, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) { st += v[e]; qt = __fadd_rn(qt, __fmul_rn(v[e], v[e])); }
    }
  } else if (flags & XF_FLAG_V_READY) {
    const float* vp = reinterpret_cast<const float*>(xf_row(t, slot) + 32);
    for (int k = 0; k < K; k += VEC) {
      float v[VEC];
      xf_ldv_step<VEC>(vp + k, v);
#pragma unroll
      for (int e = 0; e < VEC; ++e) { st += v[e]; qt = __fadd_rn(qt, __fmul_rn(v[e], v[e])); }
    }
  } else {
    for (int k = 0; k < K; ++k) {
      const float v = xf_v_init(t, key, (uint32_t)k);
      st += v;
      qt = __fadd_rn(qt, __fmul_rn(v, v));
    }
  }
}

// full-sector store of the head
__device__ __forceinline__ void xf_store_head(uint8_t* row, const XfHead& h) {
  const uint64_t q1 = (uint64_t)__double_as_longlong(h.g);
  const uint64_t q2 = (uint64_t)__float_as_uint(h.w) | ((uint64_t)__float_as_uint(h.n) << 32);
  const uint64_t q3 = (uint64_t)__float_as_uint(h.z) | ((uint64_t)h.flags << 32);
  xf_st32(row, h.key, q1, q2, q3);
}

// Find `key` starting at its home slot `s` (= xf_home_slot) whose head `h` the caller has already loaded; if
// INSERT, claim an empty slot for it when absent (store[key] semantics).  Returns the slot index, or -1 (not found
// without INSERT, or probe overflow -> *t.error = 1).  On return `h` is the row's first sector as it
// was when the key matched (or the default contents on insert).
// ADMIT (INSERT only): an absent key is inserted only if the policy `*adm` admits it; otherwise the call returns -1
// and sets *rejected (unless the policy is XF_ADM_NEVER).  Every token of one key decides the same way in a batch.
// STAMP (INSERT only): the inserting thread stamps the new key with sv->now when the table tracks stamps.
template <bool INSERT, bool ADMIT = false, bool STAMP = false>
__device__ __forceinline__ int64_t xf_probe_from(const XfTableView& t, uint64_t key, uint64_t s, XfHead& h,
                                                 const XfAdmitView* adm = nullptr, bool* rejected = nullptr,
                                                 const XfStampView* sv = nullptr) {
  for (int probes = 0; probes < XF_MAX_PROBE; ++probes) {
    if (h.key == key) return (int64_t)s;
    if (h.key == XF_EMPTY_KEY) {
      if (!INSERT) return -1;
      if (ADMIT && !xf_admit(*adm, key)) {
        *rejected = adm->mode != XF_ADM_NEVER;
        return -1;
      }
      unsigned long long old =
          atomicCAS(reinterpret_cast<unsigned long long*>(xf_row(t, s)), (unsigned long long)XF_EMPTY_KEY,
                    (unsigned long long)key);
      if (old == XF_EMPTY_KEY) {
        // we created the entry: count it (warp-aggregated) and report default contents
        unsigned m = __activemask();
        int leader = __ffs(m) - 1;
        if ((int)(threadIdx.x & 31) == leader) {
          atomicAdd(t.size, (unsigned long long)__popc(m));
          if (ADMIT) atomicAdd(adm->admitted, (unsigned long long)__popc(m));
        }
        if (STAMP && sv->stamp != nullptr) sv->stamp[s] = sv->now;
        h.key = key; h.flags = 0; h.w = 0.f; h.n = 0.f; h.z = 0.f;
        h.g = t.lazy ? 0.0 : -0.0;  // what xf_k_fill left in the row (lazy: the integer 0)
        return (int64_t)s;
      }
      if (old == key) {
        // raced with another inserter of the same key: the parameter fields are still defaults
        h.key = key;
        return (int64_t)s;
      }
      // a different key took the slot: fall through to the next one
    }
    s = xf_probe_slot(t, key, (uint32_t)probes + 1u);
    h = xf_load_head(xf_row(t, s));
  }
  *t.error = 1;
  return -1;
}

template <bool INSERT, bool STAMP = false>
__device__ __forceinline__ int64_t xf_probe(const XfTableView& t, uint64_t key, XfHead* head,
                                            const XfStampView* sv = nullptr) {
  const uint64_t s = xf_home_slot(t, key);
  XfHead h = xf_load_head(xf_row(t, s));
  const int64_t r = xf_probe_from<INSERT, false, STAMP>(t, key, s, h, nullptr, nullptr, sv);
  *head = h;
  return r;
}

// ---- arithmetic restated from the reference, IEEE-rounded op by op (no FMA contraction) ----

// Base::sigmoid  src/base/base.h:54-63
__device__ __forceinline__ float xf_sigmoid(float x) {
  if (x < -30.f) return (float)1e-6;
  if (x > 30.f) return 1.0f;
  // pow(2.718281828, x) as exp(x * ln 2.718281828) in double: same value to ~3e-15 relative (far below
  // the final float rounding), a third of the registers and instructions of the generic double pow
  const double ex = exp((double)x * 0.9999999998311266);
  return (float)(ex / (1.0 + ex));
}

// FTRL-proximal coordinate update  src/optimizer/ftrl.h:59-74 (== :126-141)
__device__ __forceinline__ void xf_ftrl_coord(const XfTableView& t, float g, float& w, float& n, float& z) {
  float old_n = n;
  float nn = __fadd_rn(old_n, __fmul_rn(g, g));
  float sig = __fdiv_rn(__fsub_rn(__fsqrt_rn(nn), __fsqrt_rn(old_n)), t.alpha);
  z = __fadd_rn(z, __fsub_rn(g, __fmul_rn(sig, w)));
  n = nn;
  if (fabsf(z) <= t.lambda1) {
    w = 0.0f;
  } else {
    float tmpr = 0.0f;
    if (z > 0.0f) tmpr = __fsub_rn(z, t.lambda1);
    if (z < 0.0f) tmpr = __fadd_rn(z, t.lambda1);
    float tmpl = -__fadd_rn(__fdiv_rn(__fadd_rn(t.beta, __fsqrt_rn(n)), t.alpha), t.lambda2);
    w = __fdiv_rn(tmpr, tmpl);
  }
}

// SGD coordinate update  src/optimizer/sgd.h:52,96
__device__ __forceinline__ void xf_sgd_coord(const XfTableView& t, float g, float& w) {
  w = __fsub_rn(w, __fmul_rn(t.learning_rate, g));
}

// AdaGrad coordinate update (include/xflow_b200.h, section 2): eta = learning_rate, beta = the accumulator's start
//   n' = n + g*g,  w' = w - eta*g / sqrt(beta + n'),  every operation rounded to nearest on its own (no FMA)
__device__ __forceinline__ void xf_adagrad_coord(const XfTableView& t, float g, float& w, float& n) {
  n = __fadd_rn(n, __fmul_rn(g, g));
  w = __fsub_rn(w, __fdiv_rn(__fmul_rn(t.learning_rate, g), __fsqrt_rn(__fadd_rn(t.beta, n))));
}

__device__ __forceinline__ void xf_opt_coord(const XfTableView& t, float g, float& w, float& n, float& z) {
  if (t.opt == XF_OPT_FTRL) xf_ftrl_coord(t, g, w, n, z);
  else if (t.opt == XF_OPT_ADAGRAD) xf_adagrad_coord(t, g, w, n);
  else xf_sgd_coord(t, g, w);
}

// push_gradient[i] /= 1.0 * loss.size()  lr_worker.cc:116-118 ; fm_worker.cc:150-156 (double divide)
__device__ __forceinline__ float xf_div_rows_plain(float g, double rows) { return (float)((double)g / rows); }
__device__ __forceinline__ float xf_div_rows(float g, double rows) {
  // A power-of-two row count (the usual batch size) makes the quotient an exact scaling: multiplying by
  // the exact reciprocal gives the same double, hence the same float, without a double division (the
  // update kernel was instruction-bound on it).
  const long long b = __double_as_longlong(rows);
  if ((b & 0x000FFFFFFFFFFFFFll) == 0ll && b > 0ll) {
    const double inv = __longlong_as_double((2046ll << 52) - b);  // 2^-e for rows = 2^e
    return (float)((double)g * inv);
  }
  return (float)((double)g / rows);
}

// FTRL's weight as a function of its accumulators: the last lines of the reference's update (ftrl.h:66-74),
// which it evaluates after every push — so (w, n, z) of a key always satisfy w == xf_ftrl_w(z, n).
__device__ __forceinline__ float xf_ftrl_w(const XfTableView& t, float z, float n) {
  if (fabsf(z) <= t.lambda1) return 0.0f;
  float tmpr = 0.0f;
  if (z > 0.0f) tmpr = __fsub_rn(z, t.lambda1);
  if (z < 0.0f) tmpr = __fadd_rn(z, t.lambda1);
  const float tmpl = -__fadd_rn(__fdiv_rn(__fadd_rn(t.beta, __fsqrt_rn(n)), t.alpha), t.lambda2);
  return __fdiv_rn(tmpr, tmpl);
}
// 2^e as a double, exactly (-1022 <= e <= 1023)
__device__ __forceinline__ double xf_pow2(int e) { return __longlong_as_double((long long)(1023 + e) << 52); }
// a residual in units of 2^-shift, rounded to nearest (xf_fix_shift)
__device__ __forceinline__ long long xf_fix_of(float residual, int shift) {
  return __double2ll_rn((double)residual * xf_pow2(shift));
}

// ---- lazy rows: the raw second half {q2 = bytes 16..23, q3 = bytes 24..31} of a row loaded with xf_load_head
__device__ __forceinline__ uint64_t xf_raw_q2(const XfHead& h) {
  return (uint64_t)__float_as_uint(h.w) | ((uint64_t)__float_as_uint(h.n) << 32);
}
__device__ __forceinline__ uint64_t xf_raw_q3(const XfHead& h) {
  return (uint64_t)__float_as_uint(h.z) | ((uint64_t)h.flags << 32);
}
__device__ __forceinline__ uint64_t xf_raw_q1(const XfHead& h) { return (uint64_t)__double_as_longlong(h.g); }
// digest of a lazy row's state word that validates an imported weight kept in bytes 8..15; never 0, so a row
// without an imported weight (bytes 8..15 all zero) can never pass for one, whatever its state
__device__ __forceinline__ uint32_t xf_lazy_check(uint64_t q2) {
  const uint32_t c = (uint32_t)q2 ^ (uint32_t)(q2 >> 32) ^ 0xA5A5A5A5u;
  return c ? c : 1u;
}
// The imported weight stands for w until the first optimizer step after the import folds in; that step can leave the
// state word as it was (a residual sum of exactly 0), so the check alone cannot end it.  The batch that first opens
// the row therefore re-marks it with its own tag (xf_lazy_mark_open): check = (top half of the digest, complemented)
// << 16 | tag, valid only while the row's tag is still that batch's, i.e. until the next batch opens the row and folds
// the step.  A row that was never opened since the import keeps the plain digest (tag 0).
__device__ __forceinline__ uint32_t xf_lazy_open_check(uint64_t q2, uint32_t tag) {
  return (((xf_lazy_check(q2) >> 16) ^ 0xFFFFu) << 16) | tag;
}
// does bytes 8..15 (q1) hold a weight that stands for w of the lazy row (q2, q3)?
__device__ __forceinline__ bool xf_lazy_given(uint64_t q1, uint64_t q2, uint64_t q3) {
  const uint32_t c = (uint32_t)(q1 >> 32), tag = (uint32_t)(q3 & XF_TAG_MASK);
  return c == xf_lazy_check(q2) || (tag != 0u && c == xf_lazy_open_check(q2, tag));
}
// After the deposit that opened a row for batch `seq` from the look (q1, q2, q3): a row still carrying its imported
// weight unopened (tag 0) is re-marked for seq (a 32-bit store of the check; readers in between accept either form).
__device__ __forceinline__ void xf_lazy_mark_open(uint8_t* rowp, uint64_t q1, uint64_t q2, uint64_t q3, uint32_t seq) {
  if ((q3 & XF_TAG_MASK) == 0ull && (uint32_t)(q1 >> 32) == xf_lazy_check(q2))
    *reinterpret_cast<uint32_t*>(rowp + 12) = xf_lazy_open_check(q2, seq);
}
// What batch `seq` pulls from a lazy row whose second half is (q2, q3): the weight with the pending optimizer
// step (the Push of the batch named by the tag, gradient = (float)(residual sum) / rows, lr_worker.cc:116-118)
// applied.  q2_new = the first word the row gets when it is opened (its state after that step).  Pure.
// ADAGRAD: the table's optimizer is AdaGrad; otherwise it is FTRL or SGD, told apart at run time.  The lazy LR step
// instantiates both, so that its FTRL and SGD code does not carry AdaGrad's branch.
template <bool ADAGRAD>
__device__ __forceinline__ float xf_lazy_fold_t(const XfTableView& t, uint64_t q1, uint64_t q2, uint64_t q3, uint32_t seq,
                                                uint64_t& q2_new) {
  const uint32_t tag = (uint32_t)(q3 & XF_TAG_MASK);
  const bool pending = tag != 0u && tag != seq;
  float g = 0.f;
  if (pending) {
    const long long gfix = (long long)q3 >> 16;
    // the residual sum, in the unit its batch deposited it with, is rounded to float once (push_gradient is a
    // float vector), then divided in double
    const uint64_t rs = __ldg(t.rows_by_seq + tag);
    g = xf_div_rows_plain((float)((double)gfix * xf_pow2(-(int)(rs >> 32))), (double)(uint32_t)rs);
  }
  const float a = __uint_as_float((uint32_t)q2), b = __uint_as_float((uint32_t)(q2 >> 32));
  if (ADAGRAD) {  // the weight itself and its accumulator
    float w = a, n = b;
    if (pending) xf_adagrad_coord(t, g, w, n);
    q2_new = (uint64_t)__float_as_uint(w) | ((uint64_t)__float_as_uint(n) << 32);
    return w;
  }
  if (t.opt == XF_OPT_FTRL) {
    float n = a, z = b;
    float w = xf_lazy_given(q1, q2, q3) ? __uint_as_float((uint32_t)q1) : xf_ftrl_w(t, z, n);
    if (pending) xf_ftrl_coord(t, g, w, n, z);
    q2_new = (uint64_t)__float_as_uint(n) | ((uint64_t)__float_as_uint(z) << 32);
    return w;
  }
  float w = a;
  if (pending) xf_sgd_coord(t, g, w);
  q2_new = (uint64_t)__float_as_uint(w);
  return w;
}
__device__ __forceinline__ float xf_lazy_fold(const XfTableView& t, uint64_t q1, uint64_t q2, uint64_t q3, uint32_t seq,
                                              uint64_t& q2_new) {
  return t.opt == XF_OPT_ADAGRAD ? xf_lazy_fold_t<true>(t, q1, q2, q3, seq, q2_new)
                                 : xf_lazy_fold_t<false>(t, q1, q2, q3, seq, q2_new);
}
// A raw-loaded head of a lazy row -> the row as the reference's server would hold it right now (pending step
// applied): canonical fields w, n, z; flags = 0; g = 0.  Every reader outside the step kernels goes through this.
__device__ __forceinline__ void xf_apply_pending(const XfTableView& t, XfHead& h) {
  if (!t.lazy) return;
  uint64_t q2n;
  const float w = xf_lazy_fold(t, xf_raw_q1(h), xf_raw_q2(h), xf_raw_q3(h), 0xFFFFFFFFu, q2n);
  h.w = w;
  if (t.opt == XF_OPT_FTRL) {
    h.n = __uint_as_float((uint32_t)q2n);
    h.z = __uint_as_float((uint32_t)(q2n >> 32));
  } else {
    h.n = t.opt == XF_OPT_ADAGRAD ? __uint_as_float((uint32_t)(q2n >> 32)) : 0.f;
    h.z = 0.f;
  }
  h.flags = 0u;
  h.g = 0.0;
}
__device__ __forceinline__ bool xf_lazy_has_pending(const XfHead& raw) { return (xf_raw_q3(raw) & XF_TAG_MASK) != 0ull; }
// store a canonical head (no pending step) into a lazy row.  keep_w: the weight was set from outside and need
// not be f(z, n) (xf_table_import): keep it beside the state
__device__ __forceinline__ void xf_lazy_store(const XfTableView& t, uint8_t* rowp, const XfHead& h, bool keep_w = false) {
  const bool ftrl = t.opt == XF_OPT_FTRL;
  const uint64_t q2 = ftrl ? ((uint64_t)__float_as_uint(h.n) | ((uint64_t)__float_as_uint(h.z) << 32))
                    : t.opt == XF_OPT_ADAGRAD ? ((uint64_t)__float_as_uint(h.w) | ((uint64_t)__float_as_uint(h.n) << 32))
                                              : (uint64_t)__float_as_uint(h.w);
  uint64_t q1 = 0ull;
  if (keep_w && ftrl && __float_as_uint(h.w) != __float_as_uint(xf_ftrl_w(t, h.z, h.n)))
    q1 = (uint64_t)__float_as_uint(h.w) | ((uint64_t)xf_lazy_check(q2) << 32);
  xf_st32(rowp, h.key, q1, q2, 0ull);
}
// store a canonical head into a row of either kind
__device__ __forceinline__ void xf_store_head_t(const XfTableView& t, uint8_t* rowp, const XfHead& h) {
  if (t.lazy) xf_lazy_store(t, rowp, h);
  else xf_store_head(rowp, h);
}

// ---- lazy tables: fold + open + deposit with ONE 128-bit compare-and-swap ------------------------------------
// On a multi-GB table every instruction that touches a random row costs about the same whatever it is — load,
// store, CAS or RED, hit or miss: the request path saturates first (tools/membench.cu measures it) — so the number
// of row-touching instructions per token is what sets the speed of these kernels.  Round 1's protocol needed four (load, CAS on the tag, 256-bit store, RED).  Here a
// token needs two: the load, and this deposit — which for the FIRST token of a batch on a row is a CAS.128 of
// {state, tag, g}: (pending state, p, sum_p) -> (state after the step of p, seq, its own residual), and for a
// later token of the same batch (duplicate keys) a 64-bit integer add into g.  Nobody ever waits or polls.
__device__ __forceinline__ bool xf_cas128(uint8_t* addr, uint64_t e0, uint64_t e1, uint64_t d0, uint64_t d1, uint64_t& o0,
                                          uint64_t& o1) {
  asm volatile(
      "{\n .reg .b128 cmp, swp, old;\n mov.b128 cmp, {%2, %3};\n mov.b128 swp, {%4, %5};\n"
      " atom.global.cas.b128 old, [%6], cmp, swp;\n mov.b128 {%0, %1}, old;\n}"
      : "=l"(o0), "=l"(o1)
      : "l"(e0), "l"(e1), "l"(d0), "l"(d1), "l"(addr)
      : "memory");
  return o0 == e0 && o1 == e1;
}
__device__ __forceinline__ void xf_lazy_add(uint8_t* rowp, long long fix) {
  atomicAdd(reinterpret_cast<unsigned long long*>(rowp + 24), (unsigned long long)fix << 16);  // never carries into the tag
}
// Deposit `fix` units of residual of batch `seq` into the row whose second half was (q2, q3) when the caller
// looked; q2_new from xf_lazy_fold.  Returns true when this call opened the row (= the key's first token of the
// batch: the unique-key count).  *stale (optional): the caller's look may be OLDER than this batch (the sharded
// owner works from the look its Pull took); a row that meanwhile moved on to another batch is then reported
// instead of flagged as an error, and the caller looks again.
// The same in two halves, for callers that keep several deposits in flight: _issue sends the CAS (or, for a row
// already seen open, the RED) and returns what came back; _resolve acts on it.
__device__ __forceinline__ bool xf_lazy_deposit_issue(uint8_t* rowp, uint64_t q2, uint64_t q3, uint64_t q2_new, uint32_t seq,
                                                      long long fix, uint64_t& o2, uint64_t& o3) {
  if ((uint32_t)(q3 & XF_TAG_MASK) == seq) {  // already open for this batch: nothing comes back
    xf_lazy_add(rowp, fix);
    o2 = q2; o3 = q3;
    return false;
  }
  xf_cas128(rowp + XF_OFF_STATE, q2, q3, q2_new, ((unsigned long long)fix << 16) | (uint64_t)seq, o2, o3);
  return true;
}
// returns true when the issued CAS opened the row.  *stale reports a row that moved on to another batch since the
// caller's look (as in xf_lazy_deposit): the sharded owner, which works from the look its Pull stashed, looks again;
// for the lazy step kernel, whose look is from this batch, it is an error.
__device__ __forceinline__ bool xf_lazy_deposit_resolve(uint8_t* rowp, bool issued, uint64_t q2, uint64_t q3, uint64_t o2,
                                                        uint64_t o3, uint32_t seq, long long fix, bool* stale) {
  *stale = false;
  if (!issued) return false;
  if (o2 == q2 && o3 == q3) return true;
  if ((uint32_t)(o3 & XF_TAG_MASK) == seq) {  // another token of this batch was first
    xf_lazy_add(rowp, fix);
    return false;
  }
  *stale = true;
  return false;
}
__device__ __forceinline__ bool xf_lazy_deposit(const XfTableView& t, uint8_t* rowp, uint64_t q2, uint64_t q3, uint64_t q2_new,
                                                uint32_t seq, long long fix, bool* stale = nullptr) {
  if (stale) *stale = false;
  if ((uint32_t)(q3 & XF_TAG_MASK) == seq) {  // already open for this batch
    xf_lazy_add(rowp, fix);
    return false;
  }
  uint64_t o2, o3;
  if (xf_cas128(rowp + XF_OFF_STATE, q2, q3, q2_new, ((unsigned long long)fix << 16) | (uint64_t)seq, o2, o3)) return true;
  if ((uint32_t)(o3 & XF_TAG_MASK) == seq) {  // another token of this batch was first
    xf_lazy_add(rowp, fix);
    return false;
  }
  if (stale) *stale = true;
  else *t.error = 2;  // inside a batch a row only ever goes from "pending" to "open for seq"
  return false;
}

__device__ __forceinline__ float xf_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

#endif  // __CUDACC__

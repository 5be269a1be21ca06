// Grouped test metric on the device (include/xflow_b200.h section 9): every group's exact AUC and logloss, and their
// row-weighted mean (GAUC), for held-out predictions that carry a uint64 group id per row (a user, a request).
//
//   add      copies the rows (p, y, g) into the metric's buffers on the caller's stream
//   finish   DeviceSelect     each non-NaN row's key {g, -p, y} (-0 made +0 first), NaN rows dropped
//            DeviceRadixSort  ascending on (g, -p) through a decomposer: by group, then by descending prediction; the
//                             label rides in the key's padding.  Not stable: every per-group quantity is a sum over tie
//                             runs, so the order inside a run does not matter
//            DeviceScan       one inclusive scan of {positives, run start, group start} under (sum, max, max)
//            DeviceReduce::ReduceByKey  per group {n + 2^32 P, U2, S} in integers: each row adds 1, y and its logloss
//                             units L_i, and the last row of a tie run adds gn (2 pb + gp) to U2
//            xf_k_gm_groups   per group auc_g, logloss_g, T_g and M_g; the global integer sums by block reduction and
//                             integer atomics
//   topk     DeviceReduce::ReduceByKey  per group {H, G} over the finish's sorted rows and scan: the last row of a tie
//                             run adds its overlap with the top k (xf_gm_run_end, as the U2 term)
//            xf_k_gm_topk     per group ndcg_g, precision_g and recall_g, and the global sums as xf_k_gm_groups
//   The host only copies and turns the global sums into correctly rounded ratios (xf_ratio).  Every
// accumulator is an integer and every double a fixed function of integers, so the report and the per-group arrays
// depend only on the multiset of rows: not on add cuts, streams, grid or atomic order.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <cub/cub.cuh>
#include <cuda/std/tuple>
#include <mutex>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <vector>

#include "metric.cuh"

typedef unsigned long long u64;

namespace {

constexpr u64 XF_GM_MAX_ROWS = 1ull << 31;  // a metric holds fewer rows (xf_metric's limit)
constexpr int XF_GM_THREADS = 256;

struct XfGmKey {
  uint64_t g;
  float negp;  // -p, with both zeros as +0
  uint32_t y;  // 1 for a positive row: not part of the sort key
};
struct XfGmDecomposer {  // the sort key, most significant first
  __host__ __device__ ::cuda::std::tuple<uint64_t&, float&> operator()(XfGmKey& k) const { return {k.g, k.negp}; }
};

struct XfGmMakeKey {
  const float* p;
  const uint8_t* y;
  const uint64_t* g;
  __host__ __device__ XfGmKey operator()(uint32_t i) const {
    const float pi = p[i];
    return XfGmKey{g[i], pi == 0.f ? 0.f : -pi, y[i] != 0 ? 1u : 0u};
  }
};
struct XfGmScored {
  __host__ __device__ bool operator()(const XfGmKey& k) const { return k.negp == k.negp; }
};

// positives up to the row, the start of its tie run and of its group (sorted positions)
struct XfGmScan {
  uint32_t pos, run, grp;
};
struct XfGmScanOp {
  __host__ __device__ XfGmScan operator()(const XfGmScan& a, const XfGmScan& b) const {
    return XfGmScan{a.pos + b.pos, a.run > b.run ? a.run : b.run, a.grp > b.grp ? a.grp : b.grp};
  }
};
struct XfGmHeads {
  const XfGmKey* k;
  __host__ __device__ XfGmScan operator()(uint32_t i) const {
    const XfGmKey c = k[i];
    bool grp = i == 0, run = grp;
    if (!grp) {
      const XfGmKey b = k[i - 1];
      grp = b.g != c.g;
      run = grp || b.negp != c.negp;
    }
    return XfGmScan{c.y, run ? i : 0u, grp ? i : 0u};
  }
};

// a group's integer sums: np = n + 2^32 P (each below 2^31), U2, and S = s_lo + 2^64 s_hi
struct XfGmAgg {
  u64 np, u2, s_lo, s_hi;
};
struct XfGmAggOp {
  __host__ __device__ XfGmAgg operator()(const XfGmAgg& a, const XfGmAgg& b) const {
    XfGmAgg r{a.np + b.np, a.u2 + b.u2, a.s_lo + b.s_lo, a.s_hi + b.s_hi};
    r.s_hi += r.s_lo < a.s_lo ? 1ull : 0ull;
    return r;
  }
};
// the group's results, written over its XfGmAgg by xf_k_gm_groups
struct XfGmOut {
  u64 rows, positives;
  double auc, logloss;
};
static_assert(sizeof(XfGmAgg) == sizeof(XfGmOut), "a group's results take its sums' place");

struct XfGmGroupOf {
  const XfGmKey* k;
  __host__ __device__ uint64_t operator()(uint32_t i) const { return k[i].g; }
};

// the tie run [start, i] that sorted row i ends, from the scan: its position in its group, its group's positives
// before it (pb), its positives (gp) and rows
struct XfGmRun {
  u64 at, pb, gp, rows;
};
// false when row i is not the last row of its tie run (of n sorted rows)
__device__ __forceinline__ bool xf_gm_run_end(const XfGmScan* s, uint32_t n, uint32_t i, XfGmRun& r) {
  if (i + 1 != n && s[i + 1].run != i + 1) return false;
  const XfGmScan h = s[i];
  const u64 before_run = h.run ? s[h.run - 1].pos : 0u, before_grp = h.grp ? s[h.grp - 1].pos : 0u;
  r.at = h.run - h.grp;
  r.pb = before_run - before_grp;
  r.gp = h.pos - before_run;
  r.rows = i - h.run + 1;
  return true;
}

struct XfGmRowTerms {
  const XfGmKey* k;
  const XfGmScan* s;
  uint32_t n;
  __device__ XfGmAgg operator()(uint32_t i) const {
    const XfGmKey c = k[i];
    XfGmAgg a{1ull | (u64)c.y << 32, 0ull, 0ull, 0ull};
    xf_loss_units(1.f, -c.negp, (int)c.y, a.s_lo, a.s_hi);
    XfGmRun r;
    if (xf_gm_run_end(s, n, i, r)) a.u2 = (r.rows - r.gp) * (2 * r.pb + r.gp);
    return a;
  }
};

// ---- top k (xf_group_metric_topk): a group's integers H and G in units of 2^-32, summed over its tie runs
struct XfGmTopkSums {
  u64 h, g, zero;  // the third word keeps a group's sums in the place of its XfGmTopkOut
};
struct XfGmTopkSumOp {
  __host__ __device__ XfGmTopkSums operator()(const XfGmTopkSums& a, const XfGmTopkSums& b) const {
    return XfGmTopkSums{a.h + b.h, a.g + b.g, 0ull};
  }
};
// the group's top-k results, written over its XfGmTopkSums by xf_k_gm_topk
struct XfGmTopkOut {
  double ndcg, precision, recall;
};
static_assert(sizeof(XfGmTopkSums) == sizeof(XfGmTopkOut), "a group's results take its sums' place");

// x / c rounded to the nearest integer, ties to even; the quotient fits 64 bits
__device__ __forceinline__ u64 xf_div_rn(unsigned __int128 x, u64 c) {
  if (c == 1) return (u64)x;
  const u64 q = (u64)(x / c), r = (u64)(x - (unsigned __int128)q * c);
  return q + ((2 * r > c || (2 * r == c && (q & 1))) ? 1ull : 0ull);
}

// a tie run's terms at its last row: its m positives spread evenly over its c rows, o of which lie in the top k,
// give rn(m o 2^32 / c) hits and rn(m (D(a + o) - D(a)) / c) DCG (D: the cumulative discounts, k <= 65536 entries)
struct XfGmTopkTerms {
  const XfGmScan* s;
  const u64* D;
  uint32_t n, k;
  __device__ XfGmTopkSums operator()(uint32_t i) const {
    XfGmTopkSums a{0ull, 0ull, 0ull};
    XfGmRun r;
    if (xf_gm_run_end(s, n, i, r) && r.gp && r.at < k) {
      const u64 o = min((u64)k - r.at, r.rows);
      a.h = xf_div_rn((unsigned __int128)(r.gp * o) << 32, r.rows);
      a.g = xf_div_rn((unsigned __int128)r.gp * (D[r.at + o] - D[r.at]), r.rows);
    }
    return a;
  }
};

// the global sums (words of struct XfGmSums on the device)
struct XfGmSums {
  u64 groups, rows, positives, scored_groups, scored_rows, t, m, s_lo, s_hi;
};
constexpr int XF_GM_SUM_WORDS = 9;
struct XfGmSumOp {
  __device__ XfGmSums operator()(const XfGmSums& a, const XfGmSums& b) const {
    XfGmSums r{a.groups + b.groups, a.rows + b.rows, a.positives + b.positives, a.scored_groups + b.scored_groups,
               a.scored_rows + b.scored_rows, a.t + b.t, a.m + b.m, a.s_lo, a.s_hi};
    xf_add128(r.s_lo, r.s_hi, b.s_lo, b.s_hi);
    return r;
  }
};

// lo + 2^64 hi correctly rounded to double (round to nearest even): the top 64 bits with the rest as a sticky bit
__device__ __forceinline__ double xf_u128_to_double_rn(u64 lo, u64 hi) {
  if (!hi) return __ull2double_rn(lo);
  const int k = 64 - __clzll(hi);  // hi's bits; S < 2^70 keeps k below 64
  const u64 v = hi << (64 - k) | lo >> k | ((lo & ((1ull << k) - 1)) ? 1ull : 0ull);
  return ldexp(__ull2double_rn(v), k);
}

__global__ void __launch_bounds__(XF_GM_THREADS)
xf_k_gm_groups(XfGmAgg* __restrict__ groups, const uint32_t* __restrict__ n_groups, u64* __restrict__ sums) {
  const uint32_t G = *n_groups;
  XfGmSums acc{0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < G; g += gridDim.x * blockDim.x) {
    const XfGmAgg a = groups[g];
    const u64 n = a.np & 0xFFFFFFFFull, P = a.np >> 32, N = n - P;
    XfGmOut o;
    o.rows = n;
    o.positives = P;
    o.auc = (P && N) ? (double)a.u2 / ((2.0 * (double)P) * (double)N) : NAN;
    o.logloss = xf_u128_to_double_rn(a.s_lo, a.s_hi) / ((double)n * 4294967296.0);
    reinterpret_cast<XfGmOut*>(groups)[g] = o;
    ++acc.groups;
    acc.rows += n;
    acc.positives += P;
    xf_add128(acc.s_lo, acc.s_hi, a.s_lo, a.s_hi);
    if (P && N) {
      ++acc.scored_groups;
      acc.scored_rows += n;
      acc.t += __double2ull_rn(((double)n * o.auc) * 4294967296.0);
      acc.m += __double2ull_rn(o.auc * 4294967296.0);
    }
  }
  typedef cub::BlockReduce<XfGmSums, XF_GM_THREADS> R;
  __shared__ typename R::TempStorage tmp;
  const XfGmSums b = R(tmp).Reduce(acc, XfGmSumOp());
  if (threadIdx.x == 0) {
    const u64 w[XF_GM_SUM_WORDS - 2] = {b.groups, b.rows, b.positives, b.scored_groups, b.scored_rows, b.t, b.m};
    for (int k = 0; k < XF_GM_SUM_WORDS - 2; ++k)
      if (w[k]) atomicAdd(sums + k, w[k]);
    xf_atomic_add128(sums + XF_GM_SUM_WORDS - 2, b.s_lo, b.s_hi);
  }
}

// the top k's global sums (words of struct XfGmTopkTotals on the device): t and m of ndcg, precision and recall
struct XfGmTopkTotals {
  u64 groups, scored_groups, scored_rows, t[3], m[3];
};
constexpr int XF_GM_TOPK_WORDS = 9;
static_assert(sizeof(XfGmTopkTotals) == 8 * XF_GM_TOPK_WORDS, "the top k's global sums are words");
struct XfGmTopkTotalOp {
  __device__ XfGmTopkTotals operator()(const XfGmTopkTotals& a, const XfGmTopkTotals& b) const {
    XfGmTopkTotals r;
    r.groups = a.groups + b.groups;
    r.scored_groups = a.scored_groups + b.scored_groups;
    r.scored_rows = a.scored_rows + b.scored_rows;
    for (int x = 0; x < 3; ++x) {
      r.t[x] = a.t[x] + b.t[x];
      r.m[x] = a.m[x] + b.m[x];
    }
    return r;
  }
};

// per group ndcg_g, precision_g and recall_g over its {H, G} (in place), from its rows and positives in the finish's
// per-group results; the global integer sums by block reduction and integer atomics
__global__ void __launch_bounds__(XF_GM_THREADS)
xf_k_gm_topk(XfGmTopkSums* __restrict__ topk, const XfGmOut* __restrict__ groups, uint32_t G,
             const u64* __restrict__ D, uint32_t k, u64* __restrict__ sums) {
  XfGmTopkTotals acc{0, 0, 0, {0, 0, 0}, {0, 0, 0}};
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < G; g += gridDim.x * blockDim.x) {
    const XfGmTopkSums a = topk[g];
    const u64 n = groups[g].rows, P = groups[g].positives, N = n - P;
    XfGmTopkOut o;
    o.ndcg = P ? (double)a.g / (double)D[P < k ? P : k] : NAN;
    o.precision = P ? (double)a.h / ((double)(n < k ? n : k) * 4294967296.0) : NAN;
    o.recall = P ? (double)a.h / ((double)P * 4294967296.0) : NAN;
    reinterpret_cast<XfGmTopkOut*>(topk)[g] = o;
    ++acc.groups;
    if (P && N) {
      ++acc.scored_groups;
      acc.scored_rows += n;
      const double x[3] = {o.ndcg, o.precision, o.recall};
      for (int j = 0; j < 3; ++j) {
        acc.t[j] += __double2ull_rn(((double)n * x[j]) * 4294967296.0);
        acc.m[j] += __double2ull_rn(x[j] * 4294967296.0);
      }
    }
  }
  typedef cub::BlockReduce<XfGmTopkTotals, XF_GM_THREADS> R;
  __shared__ typename R::TempStorage tmp;
  const XfGmTopkTotals b = R(tmp).Reduce(acc, XfGmTopkTotalOp());
  if (threadIdx.x == 0) {
    const u64* w = reinterpret_cast<const u64*>(&b);
    for (int j = 0; j < XF_GM_TOPK_WORDS; ++j)
      if (w[j]) atomicAdd(sums + j, w[j]);
  }
}

// d(i) = 2^32 / log2(i + 2) rounded to the nearest integer, and D(i) = sum of d(j), j < i: the header's table
// (section 9), built once from long double log2l (64-bit mantissa)
constexpr uint32_t XF_GM_TOPK_MAX_K = XF_GROUP_TOPK_MAX_K;
const std::vector<u64>& xf_gm_discounts() {
  static std::mutex mu;
  static std::vector<u64> D;
  std::lock_guard<std::mutex> lk(mu);
  if (D.empty()) {
    std::vector<u64> t(XF_GM_TOPK_MAX_K + 1, 0ull);
    for (uint32_t i = 0; i < XF_GM_TOPK_MAX_K; ++i)
      t[i + 1] = t[i] + (u64)llroundl(4294967296.0L / log2l((long double)i + 2.0L));
    D.swap(t);
  }
  return D;
}

}  // namespace

struct xf_group_metric {
  int device = 0;
  cudaStream_t stream = nullptr;    // finishes; waits for every add
  cudaEvent_t added = nullptr;      // recorded on an add's stream after the add
  cudaEvent_t cleared = nullptr;    // recorded on `stream` by a reset: later adds wait for it
  XfDevBuf pctr, lab, grp;          // the rows held: 13 bytes each
  // finish's scratch, kept for later calls: the sort's two key buffers (the group ids of the last finish end up in
  // the one the sort leaves free), the scan, the per-group sums and results, CUB's storage and the global sums
  XfDevBuf keys_a, keys_b, scan, agg, tmp, acc;
  XfDevBuf topk, disc;              // the last topk's per-group results; the cumulative discounts D (uploaded once)
  const uint64_t* d_ids = nullptr;  // the last finish's group ids, in keys_a or keys_b
  const XfGmKey* d_sorted = nullptr;  // the last finish's sorted rows, in the other one
  uint64_t n = 0;
  uint64_t groups = 0;              // of the last finish
  uint32_t scored = 0;              // the last finish's sorted rows (its non-NaN rows)
  bool finished = false;            // a finish with no reset or add after it
  bool topk_done = false;           // a topk with no finish, reset or add after it
  std::mutex mu;
};

XF_DLL int xf_group_metric_create(xf_group_metric** out, int device) {
  if (!out) return XF_ERR_ARG;
  *out = nullptr;
  XF_CUDA_TRY(cudaSetDevice(device));
  xf_group_metric* m = new xf_group_metric;
  m->device = device;
  cudaError_t e = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&m->added, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&m->cleared, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventRecord(m->cleared, m->stream);
  if (e != cudaSuccess) {
    xf_group_metric_destroy(m);
    xf_set_error("xf_group_metric_create: %s", cudaGetErrorString(e));
    return XF_ERR_CUDA;
  }
  *out = m;
  return XF_OK;
}

XF_DLL int xf_group_metric_destroy(xf_group_metric* m) {
  if (!m) return XF_OK;
  cudaSetDevice(m->device);
  if (m->stream) cudaStreamSynchronize(m->stream);
  XfDevBuf* bufs[] = {&m->pctr, &m->lab, &m->grp, &m->keys_a, &m->keys_b, &m->scan, &m->agg, &m->tmp, &m->acc,
                      &m->topk, &m->disc};
  for (XfDevBuf* b : bufs) b->release();
  if (m->added) cudaEventDestroy(m->added);
  if (m->cleared) cudaEventDestroy(m->cleared);
  if (m->stream) cudaStreamDestroy(m->stream);
  delete m;
  return XF_OK;
}

XF_DLL int xf_group_metric_reset(xf_group_metric* m) {
  if (!m) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  // `stream` waits for every add so far; later adds wait for this
  XF_CUDA_TRY(cudaEventRecord(m->cleared, m->stream));
  m->n = 0;
  m->finished = m->topk_done = false;
  return XF_OK;
}

XF_DLL int xf_group_metric_add_device(xf_group_metric* m, const float* d_pctr, const uint8_t* d_labels,
                                      const uint64_t* d_groups, uint64_t n, void* cuda_stream) {
  if (!m) return XF_ERR_ARG;
  if (n && (!d_pctr || !d_labels || !d_groups)) {
    xf_set_error("xf_group_metric_add_device: a NULL array (d_pctr %s, d_labels %s, d_groups %s) with n = %llu",
                 d_pctr ? "set" : "NULL", d_labels ? "set" : "NULL", d_groups ? "set" : "NULL", (unsigned long long)n);
    return XF_ERR_ARG;
  }
  std::lock_guard<std::mutex> lk(m->mu);
  if (n >= XF_GM_MAX_ROWS - m->n) {
    xf_set_error("xf_group_metric_add_device: %llu rows held and %llu added would reach 2^31 rows (a metric holds "
                 "fewer)", (unsigned long long)m->n, (unsigned long long)n);
    return XF_ERR_ARG;
  }
  if (n == 0) return XF_OK;
  XF_CUDA_TRY(cudaSetDevice(m->device));
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const uint64_t total = m->n + n;
  if (total * 8 > m->grp.cap || total * 4 > m->pctr.cap || total > m->lab.cap) {
    // earlier adds, on any stream, may still be copying into the old buffers
    XF_CUDA_TRY(cudaStreamSynchronize(m->stream));
    XF_TRY(xf_grow_keep(m->pctr, m->n * 4, total * 4, m->stream));
    XF_TRY(xf_grow_keep(m->lab, m->n, total, m->stream));
    XF_TRY(xf_grow_keep(m->grp, m->n * 8, total * 8, m->stream));
  }
  XF_CUDA_TRY(cudaStreamWaitEvent(st, m->cleared, 0));
  XF_CUDA_TRY(cudaMemcpyAsync(m->pctr.as<float>() + m->n, d_pctr, n * 4, cudaMemcpyDeviceToDevice, st));
  XF_CUDA_TRY(cudaMemcpyAsync(m->lab.as<uint8_t>() + m->n, d_labels, n, cudaMemcpyDeviceToDevice, st));
  XF_CUDA_TRY(cudaMemcpyAsync(m->grp.as<uint64_t>() + m->n, d_groups, n * 8, cudaMemcpyDeviceToDevice, st));
  XF_CUDA_TRY(cudaEventRecord(m->added, st));
  XF_CUDA_TRY(cudaStreamWaitEvent(m->stream, m->added, 0));
  m->n = total;
  m->finished = m->topk_done = false;
  return XF_OK;
}

XF_DLL int xf_group_metric_finish(xf_group_metric* m, struct xf_group_report* out) {
  if (!m || !out) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(m->mu);
  XF_CUDA_TRY(cudaSetDevice(m->device));
  cudaStream_t st = m->stream;
  const uint64_t n = m->n;
  m->finished = m->topk_done = false;
  memset(out, 0, sizeof(*out));
  out->logloss = out->gauc = out->gauc_mean = NAN;
  // {XfGmSums, rows selected, groups}
  XF_TRY(m->acc.ensure(sizeof(XfGmSums) + 8));
  uint32_t* d_counts = reinterpret_cast<uint32_t*>(m->acc.as<char>() + sizeof(XfGmSums));
  XfGmSums h{0, 0, 0, 0, 0, 0, 0, 0, 0};
  uint32_t scored = 0;
  if (n) {
    XF_TRY(m->keys_a.ensure(n * sizeof(XfGmKey)));
    XF_TRY(m->keys_b.ensure(n * sizeof(XfGmKey)));
    XF_TRY(m->scan.ensure(n * sizeof(XfGmScan)));
    XF_TRY(m->agg.ensure(n * sizeof(XfGmAgg)));
    XfGmKey* ka = m->keys_a.as<XfGmKey>();
    const auto rows_in = thrust::make_transform_iterator(
        thrust::counting_iterator<uint32_t>(0),
        XfGmMakeKey{m->pctr.as<float>(), m->lab.as<uint8_t>(), m->grp.as<uint64_t>()});
    size_t need = 0;
    XF_CUDA_TRY(cub::DeviceSelect::If(nullptr, need, rows_in, ka, d_counts, (int)n, XfGmScored(), st));
    XF_TRY(m->tmp.ensure(need));
    size_t tb = m->tmp.cap;
    XF_CUDA_TRY(cub::DeviceSelect::If(m->tmp.p, tb, rows_in, ka, d_counts, (int)n, XfGmScored(), st));
    XF_CUDA_TRY(cudaMemcpyAsync(&scored, d_counts, 4, cudaMemcpyDeviceToHost, st));
    XF_CUDA_TRY(cudaStreamSynchronize(st));
  }
  if (scored) {
    const int nv = (int)scored;
    cub::DoubleBuffer<XfGmKey> keys(m->keys_a.as<XfGmKey>(), m->keys_b.as<XfGmKey>());
    XfGmScan* scan = m->scan.as<XfGmScan>();
    XfGmAgg* agg = m->agg.as<XfGmAgg>();
    size_t need_sort = 0, need_scan = 0, need_reduce = 0;
    XF_CUDA_TRY(cub::DeviceRadixSort::SortKeys(nullptr, need_sort, keys, nv, XfGmDecomposer(), st));
    const auto heads = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), XfGmHeads{nullptr});
    XF_CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, need_scan, heads, scan, XfGmScanOp(), nv, st));
    const auto ids_in = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), XfGmGroupOf{nullptr});
    const auto terms = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0),
                                                       XfGmRowTerms{nullptr, nullptr, 0u});
    XF_CUDA_TRY(cub::DeviceReduce::ReduceByKey(nullptr, need_reduce, ids_in, (uint64_t*)nullptr, terms, agg,
                                               d_counts + 1, XfGmAggOp(), nv, st));
    XF_TRY(m->tmp.ensure(std::max(need_sort, std::max(need_scan, need_reduce))));
    size_t tb = m->tmp.cap;
    XF_CUDA_TRY(cub::DeviceRadixSort::SortKeys(m->tmp.p, tb, keys, nv, XfGmDecomposer(), st));
    const XfGmKey* sorted = keys.Current();
    uint64_t* ids = reinterpret_cast<uint64_t*>(keys.Alternate());  // free after the sort: 16 bytes per row
    tb = m->tmp.cap;
    XF_CUDA_TRY(cub::DeviceScan::InclusiveScan(
        m->tmp.p, tb, thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), XfGmHeads{sorted}), scan,
        XfGmScanOp(), nv, st));
    tb = m->tmp.cap;
    XF_CUDA_TRY(cub::DeviceReduce::ReduceByKey(
        m->tmp.p, tb, thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), XfGmGroupOf{sorted}),
        ids, thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0),
                                             XfGmRowTerms{sorted, scan, (uint32_t)nv}),
        agg, d_counts + 1, XfGmAggOp(), nv, st));
    XF_CUDA_TRY(cudaMemsetAsync(m->acc.p, 0, sizeof(XfGmSums), st));
    xf_k_gm_groups<<<xf_grid_for((uint64_t)nv, XF_GM_THREADS, 4), XF_GM_THREADS, 0, st>>>(agg, d_counts + 1,
                                                                                          m->acc.as<u64>());
    XF_CUDA_TRY(cudaGetLastError());
    XF_CUDA_TRY(cudaMemcpyAsync(&h, m->acc.p, sizeof(XfGmSums), cudaMemcpyDeviceToHost, st));
    XF_CUDA_TRY(cudaStreamSynchronize(st));
    m->d_ids = ids;
    m->d_sorted = sorted;
  }
  out->rows = h.rows;
  out->positives = h.positives;
  out->negatives = h.rows - h.positives;
  out->nan_rows = n - scored;
  out->groups = h.groups;
  out->scored_groups = h.scored_groups;
  out->scored_rows = h.scored_rows;
  XfU256 s, t, mm, rows, srows, sgroups;  // units of 2^-32
  s.w[0] = h.s_lo;
  s.w[1] = h.s_hi;
  t.w[0] = h.t;
  mm.w[0] = h.m;
  rows.w[0] = h.rows << 32;  // every count is below 2^31
  srows.w[0] = h.scored_rows << 32;
  sgroups.w[0] = h.scored_groups << 32;
  out->logloss = xf_ratio(s, rows);
  out->gauc = xf_ratio(t, srows);
  out->gauc_mean = xf_ratio(mm, sgroups);
  m->groups = h.groups;
  m->scored = scored;
  m->finished = true;
  return XF_OK;
}

XF_DLL int xf_group_metric_groups(xf_group_metric* m, uint64_t n, uint64_t* ids, uint64_t* rows, uint64_t* positives,
                                  double* auc, double* logloss) {
  if (!m) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(m->mu);
  if (!m->finished) {
    xf_set_error("xf_group_metric_groups: no finish since the last reset or add (the groups are those of a finish)");
    return XF_ERR_STATE;
  }
  if (n != m->groups) {
    xf_set_error("xf_group_metric_groups: n = %llu, but the last finish found %llu groups", (unsigned long long)n,
                 (unsigned long long)m->groups);
    return XF_ERR_ARG;
  }
  if (n == 0) return XF_OK;
  XF_CUDA_TRY(cudaSetDevice(m->device));
  cudaStream_t st = m->stream;
  if (ids) XF_CUDA_TRY(cudaMemcpyAsync(ids, m->d_ids, n * 8, cudaMemcpyDeviceToHost, st));
  const char* base = m->agg.as<char>();
  void* dst[4] = {rows, positives, auc, logloss};
  for (int f = 0; f < 4; ++f)  // field f of every XfGmOut
    if (dst[f])
      XF_CUDA_TRY(cudaMemcpy2DAsync(dst[f], 8, base + 8 * f, sizeof(XfGmOut), 8, n, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  return XF_OK;
}

XF_DLL int xf_group_metric_topk(xf_group_metric* m, uint32_t k, struct xf_group_topk_report* out) {
  if (!m || !out) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(m->mu);
  if (!m->finished) {
    xf_set_error("xf_group_metric_topk: no finish since the last reset or add (the top k ranks the rows of a finish)");
    return XF_ERR_STATE;
  }
  if (k == 0 || k > XF_GM_TOPK_MAX_K) {
    xf_set_error("xf_group_metric_topk: k = %u, outside 1 .. %u", k, XF_GM_TOPK_MAX_K);
    return XF_ERR_ARG;
  }
  XF_CUDA_TRY(cudaSetDevice(m->device));
  cudaStream_t st = m->stream;
  const uint64_t G = m->groups;
  m->topk_done = false;
  memset(out, 0, sizeof(*out));
  out->ndcg = out->ndcg_mean = out->precision = out->precision_mean = out->recall = out->recall_mean = NAN;
  XfGmTopkTotals h{0, 0, 0, {0, 0, 0}, {0, 0, 0}};
  if (G) {
    if (!m->disc.p) {
      const std::vector<u64>& D = xf_gm_discounts();
      XF_TRY(m->disc.ensure(D.size() * 8));
      XF_CUDA_TRY(cudaMemcpyAsync(m->disc.p, D.data(), D.size() * 8, cudaMemcpyHostToDevice, st));
    }
    XF_TRY(m->topk.ensure(G * sizeof(XfGmTopkSums)));
    // {XfGmTopkTotals, groups found}: the finish's global sums, read already, leave room for these
    XF_TRY(m->acc.ensure(sizeof(XfGmTopkTotals) + 4));
    uint32_t* d_runs = reinterpret_cast<uint32_t*>(m->acc.as<char>() + sizeof(XfGmTopkTotals));
    XfGmTopkSums* sums = m->topk.as<XfGmTopkSums>();
    const u64* D = m->disc.as<u64>();
    const int nv = (int)m->scored;
    // the unique ids go to the free half of the ids' buffer: 16 bytes per sorted row hold 8 per group twice
    uint64_t* ids_again = const_cast<uint64_t*>(m->d_ids) + G;
    const auto ids_in = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), XfGmGroupOf{m->d_sorted});
    const auto terms = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0),
                                                       XfGmTopkTerms{m->scan.as<XfGmScan>(), D, (uint32_t)nv, k});
    size_t need = 0;
    XF_CUDA_TRY(cub::DeviceReduce::ReduceByKey(nullptr, need, ids_in, ids_again, terms, sums, d_runs, XfGmTopkSumOp(),
                                               nv, st));
    XF_TRY(m->tmp.ensure(need));
    size_t tb = m->tmp.cap;
    XF_CUDA_TRY(cub::DeviceReduce::ReduceByKey(m->tmp.p, tb, ids_in, ids_again, terms, sums, d_runs, XfGmTopkSumOp(),
                                               nv, st));
    XF_CUDA_TRY(cudaMemsetAsync(m->acc.p, 0, sizeof(XfGmTopkTotals), st));
    xf_k_gm_topk<<<xf_grid_for(G, XF_GM_THREADS, 4), XF_GM_THREADS, 0, st>>>(sums, m->agg.as<XfGmOut>(), (uint32_t)G,
                                                                           D, k, m->acc.as<u64>());
    XF_CUDA_TRY(cudaGetLastError());
    XF_CUDA_TRY(cudaMemcpyAsync(&h, m->acc.p, sizeof(XfGmTopkTotals), cudaMemcpyDeviceToHost, st));
    XF_CUDA_TRY(cudaStreamSynchronize(st));
  }
  out->k = k;
  out->groups = h.groups;
  out->scored_groups = h.scored_groups;
  out->scored_rows = h.scored_rows;
  XfU256 srows, sgroups;  // units of 2^-32; every count is below 2^31
  srows.w[0] = h.scored_rows << 32;
  sgroups.w[0] = h.scored_groups << 32;
  double* ratios[3][2] = {{&out->ndcg, &out->ndcg_mean}, {&out->precision, &out->precision_mean},
                          {&out->recall, &out->recall_mean}};
  for (int x = 0; x < 3; ++x) {
    XfU256 t, mm;
    t.w[0] = h.t[x];
    mm.w[0] = h.m[x];
    *ratios[x][0] = xf_ratio(t, srows);
    *ratios[x][1] = xf_ratio(mm, sgroups);
  }
  m->topk_done = true;
  return XF_OK;
}

XF_DLL int xf_group_metric_groups_topk(xf_group_metric* m, uint64_t n, double* ndcg, double* precision,
                                       double* recall) {
  if (!m) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(m->mu);
  if (!m->topk_done) {
    xf_set_error("xf_group_metric_groups_topk: no topk since the last finish, reset or add (the values are those of "
                 "a topk)");
    return XF_ERR_STATE;
  }
  if (n != m->groups) {
    xf_set_error("xf_group_metric_groups_topk: n = %llu, but the last finish found %llu groups", (unsigned long long)n,
                 (unsigned long long)m->groups);
    return XF_ERR_ARG;
  }
  if (n == 0) return XF_OK;
  XF_CUDA_TRY(cudaSetDevice(m->device));
  cudaStream_t st = m->stream;
  const char* base = m->topk.as<char>();
  double* dst[3] = {ndcg, precision, recall};
  for (int f = 0; f < 3; ++f)  // field f of every XfGmTopkOut
    if (dst[f])
      XF_CUDA_TRY(cudaMemcpy2DAsync(dst[f], 8, base + 8 * f, sizeof(XfGmTopkOut), 8, n, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  return XF_OK;
}

XF_DLL int xf_group_metric_discounts(uint64_t* d, uint32_t n) {
  if (n > XF_GM_TOPK_MAX_K || (n && !d)) {
    xf_set_error("xf_group_metric_discounts: n = %u with d %s (n <= %u and d set when n > 0)", n, d ? "set" : "NULL",
                 XF_GM_TOPK_MAX_K);
    return XF_ERR_ARG;
  }
  const std::vector<u64>& D = xf_gm_discounts();
  for (uint32_t i = 0; i < n; ++i) d[i] = D[i + 1] - D[i];
  return XF_OK;
}

// Progressive validation on the device (include/xflow_b200.h section 8): a streaming, binned metric whose
// accumulators are all integers, so that its report is a function of the multiset of rows added to it.
//
//   xf_k_pv_add     one row per thread: classify it (skipped, overflow, NaN, scored), bin it, round its weight and
//                   its e * l and e * pc terms to the 2^-32 unit; the warp's rows that share a (bin, class) are summed
//                   and added by one lane (__match_any_sync), the global sums once per block
//   xf_k_pv_report  one block: per-thread chunks of bins, an exact suffix scan of W+ over the chunks, then each thread
//                   walks its chunk downwards in double and one fixed-order tree reduces the AUC numerators
// The host turns the exact sums into correctly rounded doubles (xf_ratio).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <mutex>

#include "internal.h"

typedef unsigned long long u64;

namespace {

struct XfPvBin {
  u64 n[2];     // rows of class 0 (negative) / 1 (positive)
  u64 w[2][2];  // their weight mass in units of 2^-32: {low word, high word}
};
struct XfPvSums {
  u64 nan_rows, overflow_rows;
  u64 el[3];  // sum e * l, 192 bits
  u64 ep[2];  // sum e * pc, 128 bits
};
constexpr int XF_PV_SUM_WORDS = 7;
struct XfPvOut {
  XfPvSums s;
  u64 n[2];
  u64 w[2][2];
  double auc_lo, auc_tie;  // sum_b W-_b W+_{>b} and sum_b W-_b W+_b, units 2^-64
};

constexpr int XF_PV_THREADS = 256;
constexpr int XF_PV_REPORT_THREADS = 1024;

}  // namespace

struct xf_pv {
  int device = 0;
  uint32_t m = 10;
  uint32_t nbins = 0;
  XfPvBin* d_bins = nullptr;
  XfPvSums* d_sums = nullptr;
  XfPvOut* d_out = nullptr;
  XfPvOut* h_out = nullptr;         // page-locked
  cudaStream_t stream = nullptr;    // resets and reports; waits for every add
  cudaEvent_t added = nullptr;      // recorded on an add's stream after the add
  cudaEvent_t cleared = nullptr;    // recorded on `stream` after the last reset: adds wait for it
  int attached = 0;                 // trainers feeding this pv
  std::mutex mu;
};

__device__ __forceinline__ void xf_add128(u64& lo, u64& hi, u64 alo, u64 ahi) {
  lo += alo;
  hi += ahi + (lo < alo ? 1ull : 0ull);
}

// a multi-word atomic add: every word's carry is decided by the old value its own atomic returned, so the words hold
// the exact sum (mod 2^(64 n)) whatever the order of the adds
__device__ __forceinline__ void xf_atomic_add128(u64* w, u64 lo, u64 hi) {
  if (lo) {
    const u64 old = atomicAdd(w, lo);
    if (old + lo < old) ++hi;
  }
  if (hi) atomicAdd(w + 1, hi);
}
__device__ __forceinline__ void xf_atomic_add192(u64* w, u64 a0, u64 a1, u64 a2) {
  if (a0) {
    const u64 old = atomicAdd(w, a0);
    if (old + a0 < old) ++a1;  // a1 < 2^64 - 1: a block's sum stays far below 2^191
  }
  if (a1) {
    const u64 old = atomicAdd(w + 1, a1);
    if (old + a1 < old) ++a2;
  }
  if (a2) atomicAdd(w + 2, a2);
}

__device__ __forceinline__ double xf_u128_to_double(u64 lo, u64 hi) { return (double)hi * 0x1p64 + (double)lo; }

__global__ void __launch_bounds__(XF_PV_THREADS)
xf_k_pv_add(const float* __restrict__ pctr, const uint8_t* __restrict__ labels, const float* __restrict__ weights,
            uint64_t n, uint32_t m, XfPvBin* __restrict__ bins, XfPvSums* __restrict__ sums) {
  const int lane = threadIdx.x & 31;
  u64 nan_rows = 0, overflow_rows = 0, el0 = 0, el1 = 0, el2 = 0, ep0 = 0, ep1 = 0;
  const uint32_t first_bin = 107u << m;  // bits(2^-20) >> (23 - m)
  // whole warps run every iteration: the bin match below needs all 32 lanes
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = base + threadIdx.x;
    int cls = -1;
    uint32_t bin = 0;
    u64 u = 0;
    if (i < n) {
      const float e = weights ? weights[i] : 1.f;
      if (e != 0.f) {
        if (!(e >= 0.f && e < 2147483648.f)) {
          ++overflow_rows;
        } else {
          const float p = pctr[i];
          if (p != p) {
            ++nan_rows;
          } else {
            cls = labels[i] != 0 ? 1 : 0;
            const float pc = fminf(fmaxf(p, 0x1p-20f), 1.f);
            bin = (__float_as_uint(pc) >> (23 - m)) - first_bin;
            u = __double2ull_rn((double)e * 4294967296.0);
            const u64 t = __double2ull_rn((double)e * (double)pc * 4294967296.0);  // e * pc exact, < 2^63 units
            ep0 += t;
            ep1 += ep0 < t ? 1ull : 0ull;
            const double q = fmin(fmax((double)p, 1e-15), 1.0 - 1e-15);
            const double l = cls ? -log(q) : -log(1.0 - q);
            const double x = (double)e * l * 4294967296.0;  // < 2^69 units
            u64 xl, xh = 0;
            if (x < 0x1p64) {
              xl = __double2ull_rn(x);
            } else {  // an integer: the split is exact
              xh = (u64)(x * 0x1p-64);
              xl = (u64)(x - (double)xh * 0x1p64);
            }
            el0 += xl;
            const u64 c = el0 < xl ? 1ull : 0ull;
            el1 += xh + c;
            el2 += el1 < xh + c ? 1ull : 0ull;
          }
        }
      }
    }
    // the warp's rows of one (bin, class) are summed and added by their lowest lane; rows that are not scored get
    // keys no scored row has (scored keys are < 2^22)
    const unsigned key = cls >= 0 ? (bin << 1 | (unsigned)cls) : (0xFFFFFFE0u | (unsigned)lane);
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    const uint32_t ulo = (uint32_t)u, uhi = (uint32_t)(u >> 32);
    u64 slo = 0, shi = 0;  // < 2^37 each
#pragma unroll
    for (int l = 0; l < 32; ++l) {
      const uint32_t a = __shfl_sync(0xffffffffu, ulo, l), b = __shfl_sync(0xffffffffu, uhi, l);
      if ((peers >> l) & 1u) { slo += a; shi += b; }
    }
    if (cls >= 0 && lane == __ffs(peers) - 1) {
      XfPvBin* bp = bins + bin;
      atomicAdd(&bp->n[cls], (u64)__popc(peers));
      const u64 lo = slo + (shi << 32);
      const u64 hi = (shi >> 32) + (lo < slo ? 1ull : 0ull);
      xf_atomic_add128(bp->w[cls], lo, hi);
    }
  }
  // the block's global sums: warp shuffles with carries, then warp 0 over the warps' sums
  __shared__ u64 s_part[XF_PV_THREADS / 32][XF_PV_SUM_WORDS];
  u64 v[XF_PV_SUM_WORDS] = {nan_rows, overflow_rows, el0, el1, el2, ep0, ep1};
  auto reduce = [&](u64* a) {
    for (int o = 16; o > 0; o >>= 1) {
      u64 b[XF_PV_SUM_WORDS];
#pragma unroll
      for (int k = 0; k < XF_PV_SUM_WORDS; ++k) b[k] = __shfl_down_sync(0xffffffffu, a[k], o);
      a[0] += b[0];
      a[1] += b[1];
      a[2] += b[2];
      const u64 c0 = a[2] < b[2] ? 1ull : 0ull;
      a[3] += b[3] + c0;
      const u64 c1 = a[3] < b[3] + c0 ? 1ull : 0ull;
      a[4] += b[4] + c1;
      xf_add128(a[5], a[6], b[5], b[6]);
    }
  };
  reduce(v);
  const int warp = threadIdx.x >> 5;
  if (lane == 0)
    for (int k = 0; k < XF_PV_SUM_WORDS; ++k) s_part[warp][k] = v[k];
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < XF_PV_SUM_WORDS; ++k) v[k] = lane < XF_PV_THREADS / 32 ? s_part[lane][k] : 0ull;
    reduce(v);
    if (lane == 0) {
      if (v[0]) atomicAdd(&sums->nan_rows, v[0]);
      if (v[1]) atomicAdd(&sums->overflow_rows, v[1]);
      xf_atomic_add192(sums->el, v[2], v[3], v[4]);
      xf_atomic_add128(sums->ep, v[5], v[6]);
    }
  }
}

// one block; out zeroed before
__global__ void __launch_bounds__(XF_PV_REPORT_THREADS)
xf_k_pv_report(const XfPvBin* __restrict__ bins, uint32_t nbins, const XfPvSums* __restrict__ sums,
               XfPvOut* __restrict__ out) {
  __shared__ u64 s_lo[XF_PV_REPORT_THREADS], s_hi[XF_PV_REPORT_THREADS];
  __shared__ double s_a[XF_PV_REPORT_THREADS], s_t[XF_PV_REPORT_THREADS];
  const int t = threadIdx.x;
  const uint32_t chunk = (nbins + XF_PV_REPORT_THREADS - 1) / XF_PV_REPORT_THREADS;
  const uint32_t b0 = min((uint32_t)t * chunk, nbins), b1 = min(b0 + chunk, nbins);
  u64 n0 = 0, n1 = 0, wn_lo = 0, wn_hi = 0, wp_lo = 0, wp_hi = 0;
  for (uint32_t b = b0; b < b1; ++b) {
    n0 += bins[b].n[0];
    n1 += bins[b].n[1];
    xf_add128(wn_lo, wn_hi, bins[b].w[0][0], bins[b].w[0][1]);
    xf_add128(wp_lo, wp_hi, bins[b].w[1][0], bins[b].w[1][1]);
  }
  if (n0) atomicAdd(&out->n[0], n0);
  if (n1) atomicAdd(&out->n[1], n1);
  xf_atomic_add128(out->w[0], wn_lo, wn_hi);
  xf_atomic_add128(out->w[1], wp_lo, wp_hi);
  s_lo[t] = wp_lo;
  s_hi[t] = wp_hi;
  __syncthreads();
  if (t == 0) {  // exclusive suffix sums: W+ of the chunks above each chunk, exact
    u64 lo = 0, hi = 0;
    for (int k = XF_PV_REPORT_THREADS - 1; k >= 0; --k) {
      const u64 clo = s_lo[k], chi = s_hi[k];
      s_lo[k] = lo;
      s_hi[k] = hi;
      xf_add128(lo, hi, clo, chi);
    }
  }
  __syncthreads();
  u64 above_lo = s_lo[t], above_hi = s_hi[t];
  double a = 0.0, tie = 0.0;
  for (uint32_t b = b1; b-- > b0;) {
    const double wn = xf_u128_to_double(bins[b].w[0][0], bins[b].w[0][1]);
    a += wn * xf_u128_to_double(above_lo, above_hi);
    tie += wn * xf_u128_to_double(bins[b].w[1][0], bins[b].w[1][1]);
    xf_add128(above_lo, above_hi, bins[b].w[1][0], bins[b].w[1][1]);
  }
  s_a[t] = a;
  s_t[t] = tie;
  __syncthreads();
  for (int s = XF_PV_REPORT_THREADS / 2; s > 0; s >>= 1) {
    if (t < s) {
      s_a[t] += s_a[t + s];
      s_t[t] += s_t[t + s];
    }
    __syncthreads();
  }
  if (t == 0) {
    out->auc_lo = s_a[0];
    out->auc_tie = s_t[0];
    out->s = *sums;
  }
}

// ---- exact ratios on the host: num / den correctly rounded to double (round to nearest even), num and den < 2^192
namespace {
struct U256 {
  uint64_t w[4] = {0, 0, 0, 0};
};
int bitlen(const U256& a) {
  for (int k = 3; k >= 0; --k)
    if (a.w[k]) return 64 * k + 64 - __builtin_clzll(a.w[k]);
  return 0;
}
bool bit(const U256& a, int i) { return (a.w[i >> 6] >> (i & 63)) & 1u; }
U256 shl(const U256& a, int s) {
  U256 r;
  for (int i = 255; i >= s; --i)
    if (bit(a, i - s)) r.w[i >> 6] |= 1ull << (i & 63);
  return r;
}
bool geq(const U256& a, const U256& b) {
  for (int k = 3; k >= 0; --k)
    if (a.w[k] != b.w[k]) return a.w[k] > b.w[k];
  return true;
}
void sub(U256& a, const U256& b) {
  uint64_t borrow = 0;
  for (int k = 0; k < 4; ++k) {
    const uint64_t x = a.w[k], y = b.w[k];
    const uint64_t d = x - y - borrow;
    borrow = (x < y || (x == y && borrow)) ? 1 : 0;
    a.w[k] = d;
  }
}
U256 u256(const u64* words, int n) {
  U256 r;
  for (int k = 0; k < n; ++k) r.w[k] = words[k];
  return r;
}
}  // namespace

static double xf_ratio(U256 num, U256 den) {
  if (bitlen(den) == 0) return NAN;
  if (bitlen(num) == 0) return 0.0;
  // scale so that the quotient has 55 or 56 bits, then round it to 53 with the remainder as sticky bit
  const int s = 55 - (bitlen(num) - bitlen(den));
  if (s >= 0) num = shl(num, s);
  else den = shl(den, -s);
  U256 r;
  uint64_t q = 0;
  for (int i = bitlen(num) - 1; i >= 0; --i) {
    r = shl(r, 1);
    if (bit(num, i)) r.w[0] |= 1u;
    if (geq(r, den)) {
      sub(r, den);
      q |= 1ull << i;  // the quotient is below 2^56: only i < 56 sets a bit
    }
  }
  const int extra = 64 - __builtin_clzll(q) - 53;
  uint64_t keep = q >> extra;
  const uint64_t rem = q & ((1ull << extra) - 1), half = 1ull << (extra - 1);
  const bool sticky = bitlen(r) != 0;
  if (rem > half || (rem == half && (sticky || (keep & 1)))) ++keep;
  return ldexp((double)keep, extra - s);
}

// ---- API
XF_DLL int xf_pv_create(xf_pv** out, int device, uint32_t mantissa_bits) {
  if (!out) return XF_ERR_ARG;
  *out = nullptr;
  if (mantissa_bits < 4 || mantissa_bits > 16) {
    xf_set_error("xf_pv_create: mantissa_bits must be 4 .. 16, got %u", mantissa_bits);
    return XF_ERR_ARG;
  }
  XF_CUDA_TRY(cudaSetDevice(device));
  xf_pv* pv = new xf_pv;
  pv->device = device;
  pv->m = mantissa_bits;
  pv->nbins = (20u << mantissa_bits) + 1u;
  int rc = XF_OK;
  auto fail = [&](cudaError_t e) {
    if (e != cudaSuccess && rc == XF_OK) {
      xf_set_error("xf_pv_create: %s", cudaGetErrorString(e));
      rc = XF_ERR_CUDA;
    }
  };
  fail(cudaMalloc(&pv->d_bins, (size_t)pv->nbins * sizeof(XfPvBin)));
  if (rc == XF_OK) fail(cudaMalloc(&pv->d_sums, sizeof(XfPvSums)));
  if (rc == XF_OK) fail(cudaMalloc(&pv->d_out, sizeof(XfPvOut)));
  if (rc == XF_OK) fail(cudaHostAlloc(&pv->h_out, sizeof(XfPvOut), cudaHostAllocDefault));
  if (rc == XF_OK) fail(cudaStreamCreateWithFlags(&pv->stream, cudaStreamNonBlocking));
  if (rc == XF_OK) fail(cudaEventCreateWithFlags(&pv->added, cudaEventDisableTiming));
  if (rc == XF_OK) fail(cudaEventCreateWithFlags(&pv->cleared, cudaEventDisableTiming));
  if (rc == XF_OK) rc = xf_pv_reset(pv);
  if (rc == XF_OK) fail(cudaStreamSynchronize(pv->stream));
  if (rc != XF_OK) {
    const std::string err = xf_last_error();
    pv->attached = 0;
    xf_pv_destroy(pv);
    xf_set_error("%s", err.c_str());
    return rc;
  }
  *out = pv;
  return XF_OK;
}

XF_DLL int xf_pv_destroy(xf_pv* pv) {
  if (!pv) return XF_OK;
  if (pv->attached) {
    xf_set_error("xf_pv_destroy: %d trainer(s) still feed this pv (xf_trainer_set_validation(tr, NULL) detaches)",
                 pv->attached);
    return XF_ERR_STATE;
  }
  cudaSetDevice(pv->device);
  if (pv->stream) cudaStreamSynchronize(pv->stream);
  cudaFree(pv->d_bins);
  cudaFree(pv->d_sums);
  cudaFree(pv->d_out);
  if (pv->h_out) cudaFreeHost(pv->h_out);
  if (pv->added) cudaEventDestroy(pv->added);
  if (pv->cleared) cudaEventDestroy(pv->cleared);
  if (pv->stream) cudaStreamDestroy(pv->stream);
  delete pv;
  return XF_OK;
}

XF_DLL int xf_pv_reset(xf_pv* pv) {
  if (!pv) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(pv->mu);
  XF_CUDA_TRY(cudaSetDevice(pv->device));
  XF_CUDA_TRY(cudaMemsetAsync(pv->d_bins, 0, (size_t)pv->nbins * sizeof(XfPvBin), pv->stream));
  XF_CUDA_TRY(cudaMemsetAsync(pv->d_sums, 0, sizeof(XfPvSums), pv->stream));
  XF_CUDA_TRY(cudaEventRecord(pv->cleared, pv->stream));
  return XF_OK;
}

XF_DLL int xf_pv_add_device(xf_pv* pv, const float* d_pctr, const uint8_t* d_labels, const float* d_weights,
                            uint64_t n, void* cuda_stream) {
  if (!pv || ((!d_pctr || !d_labels) && n)) return XF_ERR_ARG;
  if (n == 0) return XF_OK;
  std::lock_guard<std::mutex> lk(pv->mu);
  XF_CUDA_TRY(cudaSetDevice(pv->device));
  cudaStream_t st = (cudaStream_t)cuda_stream;
  // after the last reset; the pv's stream (resets, reports) after this add
  XF_CUDA_TRY(cudaStreamWaitEvent(st, pv->cleared, 0));
  xf_k_pv_add<<<xf_grid_for(n, XF_PV_THREADS, 4), XF_PV_THREADS, 0, st>>>(d_pctr, d_labels, d_weights, n, pv->m,
                                                                          pv->d_bins, pv->d_sums);
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaEventRecord(pv->added, st));
  XF_CUDA_TRY(cudaStreamWaitEvent(pv->stream, pv->added, 0));
  return XF_OK;
}

XF_DLL int xf_pv_report(xf_pv* pv, struct xf_pv_report* out) {
  if (!pv || !out) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(pv->mu);
  XF_CUDA_TRY(cudaSetDevice(pv->device));
  XF_CUDA_TRY(cudaMemsetAsync(pv->d_out, 0, sizeof(XfPvOut), pv->stream));
  xf_k_pv_report<<<1, XF_PV_REPORT_THREADS, 0, pv->stream>>>(pv->d_bins, pv->nbins, pv->d_sums, pv->d_out);
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(pv->h_out, pv->d_out, sizeof(XfPvOut), cudaMemcpyDeviceToHost, pv->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(pv->stream));
  const XfPvOut& h = *pv->h_out;
  memset(out, 0, sizeof(*out));
  out->negatives = h.n[0];
  out->positives = h.n[1];
  out->rows = h.n[0] + h.n[1];
  out->nan_rows = h.s.nan_rows;
  out->overflow_rows = h.s.overflow_rows;
  U256 one;
  one.w[0] = 1ull << 32;  // 2^32 units = weight 1
  const U256 wn = u256(h.w[0], 2), wp = u256(h.w[1], 2);
  U256 w = wn;  // W = W- + W+ < 2^128
  uint64_t lo = w.w[0] + wp.w[0];
  w.w[1] = w.w[1] + wp.w[1] + (lo < w.w[0] ? 1 : 0);
  w.w[0] = lo;
  out->weight_neg = xf_ratio(wn, one);
  out->weight_pos = xf_ratio(wp, one);
  out->logloss = xf_ratio(u256(h.s.el, 3), w);
  out->mean_pctr = xf_ratio(u256(h.s.ep, 2), w);
  out->ctr = xf_ratio(wp, w);
  const double pn = out->weight_pos * out->weight_neg * 0x1p64;  // in the units of the device's numerators
  if (pn > 0.0) {
    out->auc_lo = h.auc_lo / pn;
    out->auc_hi = (h.auc_lo + h.auc_tie) / pn;
    out->auc = 0.5 * (out->auc_lo + out->auc_hi);
  } else {
    out->auc_lo = out->auc_hi = out->auc = NAN;
  }
  return XF_OK;
}

// ---- the trainers' side (capi.cu)
int xf_pv_attach(xf_pv* pv, int device) {
  if (pv->device != device) {
    xf_set_error("xf_trainer_set_validation: the pv lives on device %d, the trainer's table on device %d", pv->device,
                 device);
    return XF_ERR_ARG;
  }
  std::lock_guard<std::mutex> lk(pv->mu);
  ++pv->attached;
  return XF_OK;
}

void xf_pv_detach(xf_pv* pv) {
  std::lock_guard<std::mutex> lk(pv->mu);
  --pv->attached;
}

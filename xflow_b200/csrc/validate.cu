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
#include <vector>

#include "metric.cuh"

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

constexpr u64 XF_PV_EMPTY_KEY = ~0ull;  // the reserved key
constexpr uint32_t XF_PV_NO_SLICE = 0xFFFFFFFFu;
constexpr uint32_t XF_PV_MAP_PROBES = 8;  // buckets past the home one
struct XfPvSliceMap {
  const u64* keys = nullptr;          // 4 per bucket, XF_PV_EMPTY_KEY where free
  const uint32_t* slice = nullptr;    // per slot
  u64 seed = 0;
  uint32_t shift = 63, mask = 1;      // bucket = mix(key ^ seed) >> shift, 2^(64 - shift) buckets
  uint32_t probes = 0;                // the longest probe of a present key: buckets past its home
};

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
  // slices (xf_pv_set_slices): n_slices sets of nbins_s bins and sums, and the map on the device
  uint32_t n_slices = 0, ms = 0, nbins_s = 0;
  XfPvBin* d_sbins = nullptr;
  XfPvSums* d_ssums = nullptr;
  XfPvOut* d_sout = nullptr;
  XfPvOut* h_sout = nullptr;        // page-locked
  u64* d_map_keys = nullptr;
  uint32_t* d_map_slice = nullptr;
  XfPvSliceMap map;
  std::mutex mu;
};

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

// a row's class and fixed-point terms (section 8): cls 0 / 1 for a scored negative / positive row, else one of the codes
// below; bin, u (e), t (e * pc) and xl + 2^64 xh (e * l) are set for a scored row only.  The slice kernel's; xf_k_pv_add
// keeps its own inline copy of the classification and binning (through this function it compiles to 36 registers
// instead of 32), and the tests hold the two to equal report bytes.  Both take e * l from xf_loss_units (metric.cuh).
enum { XF_PV_SKIP = -1, XF_PV_OVERFLOW = -2, XF_PV_NAN = -3 };
struct XfPvRow {
  int cls;
  uint32_t bin;
  u64 u, t, xl, xh;
};
__device__ __forceinline__ XfPvRow xf_pv_row(float e, const float* __restrict__ pctr, const uint8_t* __restrict__ labels,
                                             uint64_t i, uint32_t m) {
  XfPvRow v{XF_PV_SKIP, 0u, 0ull, 0ull, 0ull, 0ull};
  if (e == 0.f) return v;
  if (!(e >= 0.f && e < 2147483648.f)) {
    v.cls = XF_PV_OVERFLOW;
    return v;
  }
  const float p = pctr[i];
  if (p != p) {
    v.cls = XF_PV_NAN;
    return v;
  }
  v.cls = labels[i] != 0 ? 1 : 0;
  const uint32_t first_bin = 107u << m;  // bits(2^-20) >> (23 - m)
  const float pc = fminf(fmaxf(p, 0x1p-20f), 1.f);
  v.bin = (__float_as_uint(pc) >> (23 - m)) - first_bin;
  v.u = __double2ull_rn((double)e * 4294967296.0);
  v.t = __double2ull_rn((double)e * (double)pc * 4294967296.0);  // e * pc exact, < 2^63 units
  xf_loss_units(e, p, v.cls, v.xl, v.xh);
  return v;
}

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
            u64 xl, xh;
            xf_loss_units(e, p, cls, xl, xh);
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

// ---- slices (xf_pv_set_slices): an open-addressing map key -> slice in buckets of 4 keys, one 32-byte sector each.
// A key's home bucket comes from a mix of all its bits; it sits in the first bucket from there with a free slot, and
// slots fill in order, so a bucket whose last slot is free ends every probe through it.  The host builds the map and
// bounds the longest probe (XF_PV_MAP_PROBES) by reseeding or doubling it.
__host__ __device__ __forceinline__ u64 xf_pv_mix(u64 z) {  // splitmix64's finalizer: a bijection on 64 bits
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ uint32_t xf_pv_slice_of(const XfPvSliceMap& mp, u64 key) {
  if (key == XF_PV_EMPTY_KEY) return XF_PV_NO_SLICE;
  uint32_t b = (uint32_t)(xf_pv_mix(key ^ mp.seed) >> mp.shift);
  for (uint32_t p = 0; p <= mp.probes; ++p, b = (b + 1) & mp.mask) {
    const ulonglong2* q = reinterpret_cast<const ulonglong2*>(mp.keys + 4 * (size_t)b);
    const ulonglong2 k01 = __ldg(q), k23 = __ldg(q + 1);
    if (k01.x == key) return __ldg(mp.slice + 4 * (size_t)b);
    if (k01.y == key) return __ldg(mp.slice + 4 * (size_t)b + 1);
    if (k23.x == key) return __ldg(mp.slice + 4 * (size_t)b + 2);
    if (k23.y == key) return __ldg(mp.slice + 4 * (size_t)b + 3);
    if (k23.y == XF_PV_EMPTY_KEY) break;
  }
  return XF_PV_NO_SLICE;
}

// does a token in keys[beg, end) name slice s?  (warp-uniform arguments; the whole warp runs it)
__device__ __forceinline__ bool xf_pv_named_in(XfPvSliceMap mp, const uint64_t* __restrict__ keys, uint32_t beg,
                                            uint32_t end, uint32_t s, int lane) {
  for (uint32_t base = beg; base < end; base += 32) {
    const uint32_t j = base + lane;
    if (__any_sync(0xffffffffu, j < end && xf_pv_slice_of(mp, keys[j]) == s)) return true;
  }
  return false;
}

// one warp per row, its lanes over 32-token chunks.  Each (row, slice) pair is added once, by the lowest lane of the
// first chunk whose tokens name the slice: __match_any_sync finds a chunk's distinct slices, and the slices the row
// has added so far sit one per lane in `seen` (the first 32; past those, earlier chunks are looked up again).
__global__ void __launch_bounds__(XF_PV_THREADS)
xf_k_pv_slice_add(const float* __restrict__ pctr, const uint8_t* __restrict__ labels,
                  const float* __restrict__ weights, const uint32_t* __restrict__ row_ptr,
                  const uint64_t* __restrict__ keys, uint64_t rows, XfPvSliceMap mp, uint32_t ms, uint32_t nbins_s,
                  XfPvBin* __restrict__ bins, XfPvSums* __restrict__ sums) {
  const int lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += warps) {
    const float e = weights ? weights[r] : 1.f;
    if (e == 0.f) continue;  // adds nothing anywhere
    const uint32_t beg = row_ptr[r], end = row_ptr[r + 1];
    uint32_t seen = XF_PV_NO_SLICE, n_seen = 0;
    for (uint32_t base = beg; base < end; base += 32) {
      const uint32_t j = base + lane;
      const uint32_t s = j < end ? xf_pv_slice_of(mp, keys[j]) : XF_PV_NO_SLICE;
      if (!__any_sync(0xffffffffu, s != XF_PV_NO_SLICE)) continue;
      const unsigned peers = __match_any_sync(0xffffffffu, s);
      unsigned leaders = __ballot_sync(0xffffffffu, s != XF_PV_NO_SLICE && lane == __ffs(peers) - 1);
      unsigned fresh = 0;
      while (leaders) {
        const int l = __ffs(leaders) - 1;
        leaders &= leaders - 1;
        const uint32_t sl = __shfl_sync(0xffffffffu, s, l);
        bool added = __any_sync(0xffffffffu, seen == sl);
        if (!added && n_seen > 32) added = xf_pv_named_in(mp, keys, beg, base, sl, lane);
        if (!added) {
          if (lane == (int)n_seen) seen = sl;
          ++n_seen;
          fresh |= 1u << l;
        }
      }
      if ((fresh >> lane) & 1u) {
        const XfPvRow v = xf_pv_row(e, pctr, labels, r, ms);
        XfPvSums* sp = sums + s;
        if (v.cls == XF_PV_OVERFLOW) {
          atomicAdd(&sp->overflow_rows, 1ull);
        } else if (v.cls == XF_PV_NAN) {
          atomicAdd(&sp->nan_rows, 1ull);
        } else {
          // the low words first, all three in flight at once; each carry then goes on as in xf_atomic_add128
          XfPvBin* bp = bins + (size_t)s * nbins_s + v.bin;
          atomicAdd(&bp->n[v.cls], 1ull);
          const u64 ow = atomicAdd(&bp->w[v.cls][0], v.u);
          const u64 oe = atomicAdd(&sp->el[0], v.xl);
          const u64 op = atomicAdd(&sp->ep[0], v.t);
          if (ow + v.u < ow) atomicAdd(&bp->w[v.cls][1], 1ull);
          xf_atomic_add128(sp->el + 1, v.xh + (oe + v.xl < oe ? 1ull : 0ull), 0ull);
          if (op + v.t < op) atomicAdd(&sp->ep[1], 1ull);
        }
      }
    }
  }
}

// one block per accumulator set (the global one, or one per slice); out zeroed before
__global__ void __launch_bounds__(XF_PV_REPORT_THREADS)
xf_k_pv_report(const XfPvBin* __restrict__ bins, uint32_t nbins, const XfPvSums* __restrict__ sums,
               XfPvOut* __restrict__ out) {
  bins += (size_t)blockIdx.x * nbins;
  sums += blockIdx.x;
  out += blockIdx.x;
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
typedef XfU256 U256;
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

double xf_ratio(U256 num, U256 den) {
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

static void xf_pv_free_slices(xf_pv* pv) {
  cudaFree(pv->d_sbins);
  cudaFree(pv->d_ssums);
  cudaFree(pv->d_sout);
  if (pv->h_sout) cudaFreeHost(pv->h_sout);
  cudaFree(pv->d_map_keys);
  cudaFree(pv->d_map_slice);
  pv->d_sbins = nullptr;
  pv->d_ssums = nullptr;
  pv->d_sout = nullptr;
  pv->h_sout = nullptr;
  pv->d_map_keys = nullptr;
  pv->d_map_slice = nullptr;
  pv->map = XfPvSliceMap();
  pv->n_slices = pv->ms = pv->nbins_s = 0;
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
  xf_pv_free_slices(pv);
  if (pv->added) cudaEventDestroy(pv->added);
  if (pv->cleared) cudaEventDestroy(pv->cleared);
  if (pv->stream) cudaStreamDestroy(pv->stream);
  delete pv;
  return XF_OK;
}

// under pv->mu
static int xf_pv_clear(xf_pv* pv) {
  XF_CUDA_TRY(cudaSetDevice(pv->device));
  XF_CUDA_TRY(cudaMemsetAsync(pv->d_bins, 0, (size_t)pv->nbins * sizeof(XfPvBin), pv->stream));
  XF_CUDA_TRY(cudaMemsetAsync(pv->d_sums, 0, sizeof(XfPvSums), pv->stream));
  if (pv->n_slices) {
    XF_CUDA_TRY(cudaMemsetAsync(pv->d_sbins, 0, (size_t)pv->n_slices * pv->nbins_s * sizeof(XfPvBin), pv->stream));
    XF_CUDA_TRY(cudaMemsetAsync(pv->d_ssums, 0, (size_t)pv->n_slices * sizeof(XfPvSums), pv->stream));
  }
  XF_CUDA_TRY(cudaEventRecord(pv->cleared, pv->stream));
  return XF_OK;
}

XF_DLL int xf_pv_reset(xf_pv* pv) {
  if (!pv) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(pv->mu);
  return xf_pv_clear(pv);
}

// The slice map on the host: 2^log2b buckets of 4 slots, the key in the first bucket from its home with a free slot.
// XF_ERR_ARG, naming the key, for a key listed twice.  probes: the longest walk past a key's home bucket.
static int xf_pv_build_map(const uint64_t* keys, const uint32_t* slice_of, uint64_t n, uint32_t log2b, u64 seed,
                           std::vector<u64>& mk, std::vector<uint32_t>& ms, uint32_t* probes) {
  const uint64_t nb = 1ull << log2b, mask = nb - 1;
  mk.assign(4 * nb, XF_PV_EMPTY_KEY);
  ms.assign(4 * nb, XF_PV_NO_SLICE);
  *probes = 0;
  for (uint64_t i = 0; i < n; ++i) {
    uint64_t b = xf_pv_mix(keys[i] ^ seed) >> (64 - log2b);
    for (uint32_t p = 0;; ++p, b = (b + 1) & mask) {
      int k = 0;
      while (k < 4 && mk[4 * b + k] != XF_PV_EMPTY_KEY && mk[4 * b + k] != keys[i]) ++k;
      if (k == 4) continue;
      if (mk[4 * b + k] == keys[i]) {
        xf_set_error("xf_pv_set_slices: key %llu is listed twice (a key names at most one slice)",
                     (unsigned long long)keys[i]);
        return XF_ERR_ARG;
      }
      mk[4 * b + k] = keys[i];
      ms[4 * b + k] = slice_of[i];
      if (p > *probes) *probes = p;
      break;
    }
  }
  return XF_OK;
}

XF_DLL int xf_pv_set_slices(xf_pv* pv, const uint64_t* keys, const uint32_t* slice_of, uint64_t n_keys,
                            uint32_t n_slices, uint32_t slice_mantissa_bits) {
  if (!pv || ((!keys || !slice_of) && n_keys)) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(pv->mu);
  if (pv->attached) {
    xf_set_error("xf_pv_set_slices: %d trainer(s) feed this pv; detach it (xf_trainer_set_validation(tr, NULL)), set "
                 "the slices, then attach it again", pv->attached);
    return XF_ERR_STATE;
  }
  if (n_slices > 65536) {
    xf_set_error("xf_pv_set_slices: n_slices must be at most 65536, got %u", n_slices);
    return XF_ERR_ARG;
  }
  if (n_keys > (1ull << 24)) {
    xf_set_error("xf_pv_set_slices: n_keys must be at most 2^24, got %llu", (unsigned long long)n_keys);
    return XF_ERR_ARG;
  }
  const uint32_t ms = slice_mantissa_bits;
  if (n_slices && (ms < 4 || ms > 16)) {
    xf_set_error("xf_pv_set_slices: slice_mantissa_bits must be 4 .. 16, got %u", ms);
    return XF_ERR_ARG;
  }
  const uint64_t nbins_s = n_slices ? (20ull << ms) + 1 : 0;
  const uint64_t bytes = (uint64_t)n_slices * (nbins_s * sizeof(XfPvBin) + sizeof(XfPvSums));
  if (bytes > (1ull << 30)) {
    xf_set_error("xf_pv_set_slices: %u slices at slice_mantissa_bits %u need %llu bytes of accumulators, over 1 GiB "
                 "(fewer slices or fewer mantissa bits)", n_slices, ms, (unsigned long long)bytes);
    return XF_ERR_ARG;
  }
  for (uint64_t i = 0; i < n_keys; ++i) {
    if (slice_of[i] >= n_slices) {
      xf_set_error("xf_pv_set_slices: slice_of[%llu] = %u is not below n_slices = %u", (unsigned long long)i,
                   slice_of[i], n_slices);
      return XF_ERR_ARG;
    }
    if (keys[i] == XF_PV_EMPTY_KEY) {
      xf_set_error("xf_pv_set_slices: keys[%llu] is the reserved key 2^64 - 1", (unsigned long long)i);
      return XF_ERR_ARG;
    }
  }
  // at least twice the slots as keys; reseeded, then doubled, while a key sits more than XF_PV_MAP_PROBES buckets
  // past its home (a bound that only an adversarial key set should reach; past it lookups stay exact, only longer)
  std::vector<u64> mk;
  std::vector<uint32_t> msl;
  uint32_t log2b = 1, probes = 0;
  u64 seed = 0;
  if (n_slices) {
    uint32_t base = 1;
    while ((4ull << base) < 2 * n_keys) ++base;
    for (int attempt = 0; attempt < 8; ++attempt) {
      seed = xf_pv_mix(0x9e3779b97f4a7c15ull * (u64)(attempt + 1));
      log2b = base + (uint32_t)attempt / 4;
      XF_TRY(xf_pv_build_map(keys, slice_of, n_keys, log2b, seed, mk, msl, &probes));
      if (probes <= XF_PV_MAP_PROBES) break;
    }
  }
  // the adds enqueued so far (pv->stream waits for each) may still read the old map and accumulators
  XF_CUDA_TRY(cudaSetDevice(pv->device));
  XF_CUDA_TRY(cudaStreamSynchronize(pv->stream));
  xf_pv_free_slices(pv);
  if (n_slices) {
    int rc = XF_OK;
    auto fail = [&](cudaError_t e) {
      if (e != cudaSuccess && rc == XF_OK) {
        xf_set_error("xf_pv_set_slices: %s", cudaGetErrorString(e));
        rc = XF_ERR_CUDA;
      }
    };
    fail(cudaMalloc(&pv->d_sbins, (size_t)n_slices * nbins_s * sizeof(XfPvBin)));
    if (rc == XF_OK) fail(cudaMalloc(&pv->d_ssums, (size_t)n_slices * sizeof(XfPvSums)));
    if (rc == XF_OK) fail(cudaMalloc(&pv->d_sout, (size_t)n_slices * sizeof(XfPvOut)));
    if (rc == XF_OK) fail(cudaHostAlloc(&pv->h_sout, (size_t)n_slices * sizeof(XfPvOut), cudaHostAllocDefault));
    if (rc == XF_OK) fail(cudaMalloc(&pv->d_map_keys, mk.size() * sizeof(u64)));
    if (rc == XF_OK) fail(cudaMalloc(&pv->d_map_slice, msl.size() * sizeof(uint32_t)));
    if (rc == XF_OK) fail(cudaMemcpy(pv->d_map_keys, mk.data(), mk.size() * sizeof(u64), cudaMemcpyHostToDevice));
    if (rc == XF_OK)
      fail(cudaMemcpy(pv->d_map_slice, msl.data(), msl.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    if (rc != XF_OK) {  // the pv is left without slices, its sums cleared
      xf_pv_free_slices(pv);
      xf_pv_clear(pv);
      return rc;
    }
    pv->n_slices = n_slices;
    pv->ms = ms;
    pv->nbins_s = (uint32_t)nbins_s;
    pv->map.keys = pv->d_map_keys;
    pv->map.slice = pv->d_map_slice;
    pv->map.seed = seed;
    pv->map.shift = 64 - log2b;
    pv->map.mask = (1u << log2b) - 1;
    pv->map.probes = probes;
  }
  return xf_pv_clear(pv);
}

XF_DLL int xf_pv_add_device(xf_pv* pv, const float* d_pctr, const uint8_t* d_labels, const float* d_weights,
                            uint64_t n, void* cuda_stream) {
  if (!pv || ((!d_pctr || !d_labels) && n)) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(pv->mu);
  if (pv->n_slices) {
    xf_set_error("xf_pv_add_device: a sliced pv needs each row's keys: xf_pv_add_device_rows");
    return XF_ERR_STATE;
  }
  if (n == 0) return XF_OK;
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

XF_DLL int xf_pv_add_device_rows(xf_pv* pv, const float* d_pctr, const uint8_t* d_labels, const float* d_weights,
                                 const uint32_t* d_row_ptr, const uint64_t* d_keys, uint64_t rows, void* cuda_stream) {
  if (!pv || ((!d_pctr || !d_labels) && rows)) return XF_ERR_ARG;
  if (rows == 0) return XF_OK;
  {
    std::lock_guard<std::mutex> lk(pv->mu);
    if (pv->n_slices) {
      if (!d_row_ptr || !d_keys) return XF_ERR_ARG;
      XF_CUDA_TRY(cudaSetDevice(pv->device));
      cudaStream_t st = (cudaStream_t)cuda_stream;
      XF_CUDA_TRY(cudaStreamWaitEvent(st, pv->cleared, 0));
      xf_k_pv_add<<<xf_grid_for(rows, XF_PV_THREADS, 4), XF_PV_THREADS, 0, st>>>(d_pctr, d_labels, d_weights, rows,
                                                                                 pv->m, pv->d_bins, pv->d_sums);
      XF_CUDA_TRY(cudaGetLastError());
      xf_k_pv_slice_add<<<xf_grid_for(rows * 32, XF_PV_THREADS, 8), XF_PV_THREADS, 0, st>>>(
          d_pctr, d_labels, d_weights, d_row_ptr, d_keys, rows, pv->map, pv->ms, pv->nbins_s, pv->d_sbins,
          pv->d_ssums);
      XF_CUDA_TRY(cudaGetLastError());
      XF_CUDA_TRY(cudaEventRecord(pv->added, st));
      XF_CUDA_TRY(cudaStreamWaitEvent(pv->stream, pv->added, 0));
      return XF_OK;
    }
  }
  return xf_pv_add_device(pv, d_pctr, d_labels, d_weights, rows, cuda_stream);
}

// one report record from the device's exact sums
static void xf_pv_fill_report(const XfPvOut& h, struct xf_pv_report* out) {
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
  xf_pv_fill_report(*pv->h_out, out);
  return XF_OK;
}

XF_DLL int xf_pv_report_slices(xf_pv* pv, struct xf_pv_report* out, uint32_t n) {
  if (!pv || (!out && n)) return XF_ERR_ARG;
  std::lock_guard<std::mutex> lk(pv->mu);
  if (n != pv->n_slices || n == 0) {
    xf_set_error("xf_pv_report_slices: n = %u, but the pv has %u slices%s", n, pv->n_slices,
                 pv->n_slices ? "" : " (xf_pv_set_slices sets them)");
    return XF_ERR_ARG;
  }
  XF_CUDA_TRY(cudaSetDevice(pv->device));
  const size_t bytes = (size_t)n * sizeof(XfPvOut);
  XF_CUDA_TRY(cudaMemsetAsync(pv->d_sout, 0, bytes, pv->stream));
  xf_k_pv_report<<<n, XF_PV_REPORT_THREADS, 0, pv->stream>>>(pv->d_sbins, pv->nbins_s, pv->d_ssums, pv->d_sout);
  XF_CUDA_TRY(cudaGetLastError());
  XF_CUDA_TRY(cudaMemcpyAsync(pv->h_sout, pv->d_sout, bytes, cudaMemcpyDeviceToHost, pv->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(pv->stream));
  for (uint32_t s = 0; s < n; ++s) xf_pv_fill_report(pv->h_sout[s], out + s);
  return XF_OK;
}

// ---- the trainers' side (capi.cu)
bool xf_pv_sliced(xf_pv* pv) {
  std::lock_guard<std::mutex> lk(pv->mu);
  return pv->n_slices != 0;
}

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

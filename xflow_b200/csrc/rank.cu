// Candidate ranking (xf_model_rank_candidates_*): each request's top k candidates by pctr, selected on the device from
// the scores the candidate kernels (serve.cu) wrote.
//
// The order.  Candidate i of a request (its local index) with score p has the key r = ord(p) << 32 | (2^32 - 1 - i),
// where ord(NaN) = 0 and, for a number, ord(p) = bits(p) ^ 2^31 with the sign bit clear and ~bits(p) with it set.  ord
// is increasing in p over the numbers (-inf < ... < -0 < +0 < ... < +inf) and above 0 for each of them, so NaN of
// either sign ranks last; the low word orders equal score bits by smaller index and makes a request's keys distinct.
// A candidate ranks before another iff its key is larger.  Distinct keys leave exactly one correct output, so no thread
// or atomic order can show in it.  No key is 0 (i <= 2^32 - 2), so 0 pads a sort and stands for an empty slot.
//
// Two kernels on the caller's stream, each with a grid sized from R alone; each reads n_q = cand_ptr[q+1] - cand_ptr[q]
// on the device and takes the requests of its size class:
//   xf_k_rank_warp  n_q <= XF_RANK_SMALL: a warp per request.  E = 1, 2, 4 or 8 keys per lane in registers (position
//                   r * 32 + lane) and a bitonic network over them: shuffles below distance 32, register pairs above.
//   xf_k_rank_cta   n_q > XF_RANK_SMALL: a CTA of 1024 threads per request, the CTAs striding over the requests.  A
//                   radix select finds the k-th largest key 8 bits a pass from the top, each pass a shared histogram of
//                   one digit over the keys that match the digits found so far, re-read from pctr (L2-resident).  It
//                   stops at the first digit whose bin is taken whole, so it reaches the index word only when equal
//                   scores span position k, and there it skips the digits above the largest index.  The keys at or
//                   above the threshold (k of them; all n_q when n_q <= k) are compacted into shared memory and sorted
//                   there by a bitonic network.
// Neither kernel uses global memory but its inputs and outputs.
#include <cuda_runtime.h>
#include <stdint.h>

#include "serve.cuh"

namespace {

constexpr uint32_t XF_RANK_SMALL = 256;  // the largest request a warp ranks: 8 keys per lane
constexpr int XF_RANK_WARPS = 8;         // requests per CTA of xf_k_rank_warp
constexpr int XF_RANK_THREADS = 1024;    // threads of an xf_k_rank_cta CTA (its histogram sum takes 4 per bin)
constexpr uint32_t XF_RANK_GRID = 256;   // CTAs of xf_k_rank_cta at most: about two per SM
constexpr int XF_RANK_UNROLL = 8;        // scores in flight per thread in a pass over a request
constexpr uint32_t XF_RANK_PAD_PCTR = 0x7FC00000u;  // the pctr bits of an empty slot (its index: 0xFFFFFFFF)

__device__ __forceinline__ uint64_t xf_rank_key(uint32_t bits, uint32_t i) {
  const uint32_t o = (bits & 0x7FFFFFFFu) > 0x7F800000u ? 0u : (bits & 0x80000000u) ? ~bits : bits ^ 0x80000000u;
  return (uint64_t)o << 32 | (uint32_t)~i;
}

// slot j of a request's output from its key (0: an empty slot); the pctr is re-read, so a NaN keeps its bits
__device__ __forceinline__ void xf_rank_put(const uint32_t* __restrict__ pq, uint32_t* __restrict__ ti,
                                            uint32_t* __restrict__ tp, uint32_t j, uint64_t key) {
  const uint32_t i = ~(uint32_t)key;
  ti[j] = key ? i : 0xFFFFFFFFu;
  if (tp) tp[j] = key ? __ldg(pq + i) : XF_RANK_PAD_PCTR;
}

__device__ __forceinline__ uint64_t xf_max64(uint64_t a, uint64_t b) { return a > b ? a : b; }
__device__ __forceinline__ uint64_t xf_min64(uint64_t a, uint64_t b) { return a > b ? b : a; }

// one request of n <= 32 E candidates, ranked by the warp
template <int E>
__device__ __forceinline__ void xf_rank_warp(const uint32_t* __restrict__ pq, uint32_t n, uint32_t k,
                                             uint32_t* __restrict__ ti, uint32_t* __restrict__ tp, uint32_t lane) {
  uint64_t x[E];
#pragma unroll
  for (int r = 0; r < E; ++r) {
    const uint32_t e = r * 32u + lane;
    x[r] = e < n ? xf_rank_key(__ldg(pq + e), e) : 0ull;
  }
  // descending: in a block of s positions with (e & s) == 0 the lower position of each pair keeps the larger key
#pragma unroll
  for (uint32_t s = 2; s <= 32u * E; s <<= 1) {
#pragma unroll
    for (uint32_t j = s >> 1; j > 0; j >>= 1) {
      if (j >= 32u) {
        const int jr = (int)(j >> 5);
#pragma unroll
        for (int r = 0; r < E; ++r) {
          if (r & jr) continue;
          const bool desc = ((r * 32u) & s) == 0;
          const uint64_t a = x[r], b = x[r | jr];
          x[r] = desc ? xf_max64(a, b) : xf_min64(a, b);
          x[r | jr] = desc ? xf_min64(a, b) : xf_max64(a, b);
        }
      } else {
#pragma unroll
        for (int r = 0; r < E; ++r) {
          const uint64_t o = __shfl_xor_sync(0xFFFFFFFFu, x[r], (int)j);
          const bool desc = ((r * 32u + lane) & s) == 0;
          const bool lower = (lane & j) == 0;
          x[r] = lower == desc ? xf_max64(x[r], o) : xf_min64(x[r], o);
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < E; ++r) {
    const uint32_t e = r * 32u + lane;
    if (e < k) xf_rank_put(pq, ti, tp, e, x[r]);
  }
  for (uint32_t e = 32u * E + lane; e < k; e += 32u) xf_rank_put(pq, ti, tp, e, 0ull);
}

__global__ void __launch_bounds__(XF_RANK_WARPS * 32) xf_k_rank_warp(const uint32_t* __restrict__ pctr,
                                                                     const uint32_t* __restrict__ cand_ptr, uint32_t R,
                                                                     uint32_t k, uint32_t* __restrict__ top_index,
                                                                     uint32_t* __restrict__ top_pctr) {
  const uint64_t q = (uint64_t)blockIdx.x * XF_RANK_WARPS + (threadIdx.x >> 5);
  if (q >= R) return;
  const uint32_t lo = __ldg(cand_ptr + q), n = __ldg(cand_ptr + q + 1) - lo;
  if (n > XF_RANK_SMALL) return;
  const uint32_t* pq = pctr + lo;
  uint32_t* ti = top_index + q * k;
  uint32_t* tp = top_pctr ? top_pctr + q * k : nullptr;
  const uint32_t lane = threadIdx.x & 31u;
  if (n <= 32u) xf_rank_warp<1>(pq, n, k, ti, tp, lane);
  else if (n <= 64u) xf_rank_warp<2>(pq, n, k, ti, tp, lane);
  else if (n <= 128u) xf_rank_warp<4>(pq, n, k, ti, tp, lane);
  else xf_rank_warp<8>(pq, n, k, ti, tp, lane);
}

struct XfRankShared {
  uint32_t hist[256][32];           // a digit's histogram, one copy per lane: a warp's increments hit 32 banks
  uint64_t keys[XF_RANK_MAX_K];     // the selected keys
  uint32_t sum[256];                // the histogram, summed over the lanes
  uint32_t list[XF_RANK_THREADS];   // the large requests of a round, as offsets
  uint64_t prefix;                  // the digits found so far
  uint32_t need, done, count, nlist;
};

// A pass over a request: f(true, key) for every candidate, XF_RANK_UNROLL loads in flight per thread.  The trip count
// is the same for every thread, so f may use warp votes; it is called with (false, 0) past the request's end.
template <class F>
__device__ __forceinline__ void xf_rank_pass(const uint32_t* __restrict__ pq, uint32_t n, F f) {
  constexpr uint32_t T = XF_RANK_THREADS, U = XF_RANK_UNROLL;
  for (uint64_t i0 = threadIdx.x; i0 < (uint64_t)n + threadIdx.x; i0 += (uint64_t)T * U) {
    uint32_t bits[U];
#pragma unroll
    for (uint32_t u = 0; u < U; ++u) {
      const uint64_t i = i0 + (uint64_t)u * T;
      bits[u] = i < n ? __ldg(pq + i) : 0u;
    }
#pragma unroll
    for (uint32_t u = 0; u < U; ++u) {
      const uint64_t i = i0 + (uint64_t)u * T;
      f(i < n, i < n ? xf_rank_key(bits[u], (uint32_t)i) : 0ull);
    }
  }
}

// one request of n > XF_RANK_SMALL candidates, ranked by the CTA
__device__ void xf_rank_cta(XfRankShared& s, const uint32_t* __restrict__ pq, uint32_t n, uint32_t k,
                            uint32_t* __restrict__ ti, uint32_t* __restrict__ tp) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  uint64_t thr = 0;  // the keys selected: those >= thr (all when n <= k)
  if (n > k) {
    uint64_t prefix = 0, mask = 0;
    uint32_t need = k;  // the rank of the k-th largest key among those that match prefix under mask
    for (int shift = 56;; shift -= 8) {
      if (shift < 32 && (uint64_t)(n - 1u) >> shift == 0) {
        // every i < n has digit 0 here, every ~i digit 255: the bin holds all the matching keys, no pass needed
        prefix |= 0xFFull << shift;
        mask |= 0xFFull << shift;
        continue;
      }
      uint4* h4 = reinterpret_cast<uint4*>(&s.hist[0][0]);
      for (uint32_t w = tid; w < 256u * 32u / 4u; w += XF_RANK_THREADS) h4[w] = make_uint4(0u, 0u, 0u, 0u);
      __syncthreads();
      // a thread's run of keys in one bin is counted in a register and added once: equal scores (a clamped sigmoid)
      // put most keys of a request in one bin, whose increments would otherwise queue on its 32 words
      uint32_t run_bin = 0, run = 0;
      xf_rank_pass(pq, n, [&](bool valid, uint64_t key) {
        if (!valid || (key & mask) != prefix) return;
        const uint32_t bin = (uint32_t)(key >> shift) & 255u;
        if (run && bin != run_bin) {
          atomicAdd(&s.hist[run_bin][lane], run);
          run = 0;
        }
        run_bin = bin;
        ++run;
      });
      if (run) atomicAdd(&s.hist[run_bin][lane], run);
      __syncthreads();
      {
        // bin tid / 4, lanes 8 (tid % 4) .. +7, read in an order that keeps a warp's loads on 32 banks
        const uint32_t bin = tid >> 2, part = tid & 3u;
        uint32_t c = 0;
#pragma unroll
        for (uint32_t j = 0; j < 8u; ++j) c += s.hist[bin][part * 8u + ((j + bin) & 7u)];
        c += __shfl_xor_sync(0xFFFFFFFFu, c, 1);
        c += __shfl_xor_sync(0xFFFFFFFFu, c, 2);
        if (part == 0) s.sum[bin] = c;
      }
      __syncthreads();
      if (warp == 0) {
        // lane l holds bins 255 - 8l .. 248 - 8l, from the top; `acc` counts the keys in the bins above its first
        uint32_t c[8], tot = 0;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          c[r] = s.sum[255u - 8u * lane - r];
          tot += c[r];
        }
        uint32_t incl = tot;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, d);
          if ((int)lane >= d) incl += y;
        }
        uint32_t acc = incl - tot;
        if (acc < need && need <= incl) {
          bool found = false;
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            if (found) continue;
            if (need <= acc + c[r]) {
              found = true;
              s.prefix = prefix | (uint64_t)(255u - 8u * lane - r) << shift;
              s.need = need - acc;
              s.done = c[r] == need - acc;
            } else {
              acc += c[r];
            }
          }
        }
      }
      __syncthreads();
      prefix = s.prefix;
      need = s.need;
      mask |= 0xFFull << shift;
      if (s.done) break;  // bin taken whole: the selection is every key >= prefix, k of them
    }
    thr = prefix;
  }
  if (tid == 0) s.count = 0;
  __syncthreads();
  xf_rank_pass(pq, n, [&](bool valid, uint64_t key) {
    const bool take = valid && key >= thr;
    const uint32_t vote = __ballot_sync(0xFFFFFFFFu, take);
    uint32_t at = 0;
    if (lane == 0 && vote) at = atomicAdd(&s.count, (uint32_t)__popc(vote));
    at = __shfl_sync(0xFFFFFFFFu, at, 0);
    if (take) s.keys[at + __popc(vote & ((1u << lane) - 1u))] = key;
  });
  __syncthreads();
  const uint32_t m = s.count;  // min(n, k)
  uint32_t P = 2;
  while (P < m) P <<= 1;
  for (uint32_t e = m + tid; e < P; e += XF_RANK_THREADS) s.keys[e] = 0ull;
  __syncthreads();
  for (uint32_t sz = 2; sz <= P; sz <<= 1) {
    for (uint32_t j = sz >> 1; j > 0; j >>= 1) {
      for (uint32_t t = tid; t < P / 2u; t += XF_RANK_THREADS) {
        const uint32_t e = 2u * t - (t & (j - 1u));  // the lower position of pair t at distance j
        const uint64_t a = s.keys[e], b = s.keys[e + j];
        const bool desc = (e & sz) == 0;
        if (desc ? a < b : a > b) {
          s.keys[e] = b;
          s.keys[e + j] = a;
        }
      }
      __syncthreads();
    }
  }
  for (uint32_t e = tid; e < k; e += XF_RANK_THREADS) xf_rank_put(pq, ti, tp, e, e < P ? s.keys[e] : 0ull);
  __syncthreads();  // the next request reuses s
}

__global__ void __launch_bounds__(XF_RANK_THREADS) xf_k_rank_cta(const uint32_t* __restrict__ pctr,
                                                                 const uint32_t* __restrict__ cand_ptr, uint32_t R,
                                                                 uint32_t k, uint32_t* __restrict__ top_index,
                                                                 uint32_t* __restrict__ top_pctr) {
  __shared__ XfRankShared s;
  const uint64_t G = gridDim.x;
  // a round: thread t looks at request q0 + t G, and the CTA ranks the large ones it found
  for (uint64_t q0 = blockIdx.x; q0 < R; q0 += G * XF_RANK_THREADS) {
    const uint64_t q = q0 + threadIdx.x * G;
    bool large = false;
    if (q < R) large = __ldg(cand_ptr + q + 1) - __ldg(cand_ptr + q) > XF_RANK_SMALL;
    if (threadIdx.x == 0) s.nlist = 0;
    __syncthreads();
    if (large) s.list[atomicAdd(&s.nlist, 1u)] = threadIdx.x;  // the ranking order of the requests shows nowhere
    __syncthreads();
    const uint32_t nlist = s.nlist;
    for (uint32_t j = 0; j < nlist; ++j) {
      const uint64_t qq = q0 + (uint64_t)s.list[j] * G;
      const uint32_t lo = __ldg(cand_ptr + qq), n = __ldg(cand_ptr + qq + 1) - lo;
      xf_rank_cta(s, pctr + lo, n, k, top_index + qq * k, top_pctr ? top_pctr + qq * k : nullptr);
    }
    __syncthreads();  // s.list and s.nlist are read before the next round writes them
  }
}

}  // namespace

void xf_launch_rank(const float* pctr, const uint32_t* cand_ptr, uint32_t R, uint32_t k, uint32_t* top_index,
                    float* top_pctr, cudaStream_t st) {
  if (R == 0) return;
  const uint32_t* p = reinterpret_cast<const uint32_t*>(pctr);
  uint32_t* tp = reinterpret_cast<uint32_t*>(top_pctr);
  const uint64_t warp_grid = ((uint64_t)R + XF_RANK_WARPS - 1) / XF_RANK_WARPS;
  xf_k_rank_warp<<<(unsigned)warp_grid, XF_RANK_WARPS * 32, 0, st>>>(p, cand_ptr, R, k, top_index, tp);
  xf_k_rank_cta<<<R < XF_RANK_GRID ? R : XF_RANK_GRID, XF_RANK_THREADS, 0, st>>>(p, cand_ptr, R, k, top_index, tp);
}

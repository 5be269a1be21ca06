// Micro-benchmarks behind the round-2 kernel decisions: which access PRIMITIVES limit the table kernels?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/membench tools/membench.cu
//   tools/membench [table_MB=8192] [accesses_M=6.5]
// Table of 32-byte rows (the LR row), `n` distinct-ish random rows per launch (one batch's worth).
//   read        one 32-byte load per access (two 128-bit loads from one lane, as xf_load_head)
//   read pair   the same rows, each 128-bit load instruction serving two lanes' halves of one row (xf_ld32_pair)
//   rmw         load + 32-byte store
//   lazy        load + CAS on the tag word + 32-byte store + f64 RED   (the "open + accumulate" of step_lazy.cu)
//   lazy_sync   the same with __syncwarp between the stages (warp-synchronous, like the row kernel)
//   red         f64 RED only
//   pf+read     prefetch.global.L2 of n2 rows in one kernel, then the read kernel over the same rows
//   chain-k     k dependent loads per access (probe chains)
// On one H100 80GB HBM3 (SXM, power limit 400 W), 8 GiB table, 6.5 M rows per launch, best of 3, the same at L2
// fetch granularity 32, 64 and 128 B (to within 1 %), in G rows/s: read 21.9, read pair 30.4-30.7 (1.40x),
// CAS.128 only 12.0, load + CAS.128 10.3-10.4, read pair + CAS.128 10.3-10.5.  A paired look costs fewer requests
// than a one-lane one, but a row that is also CAS'd is bound by the atomic.
//   look, then CAS.128 after D MB (klag)  a lane-pair look at a row, and the CAS.128 on that row only after every
//               thread of the grid has made `lag` more looks: D = the lines those looks bring into L2
// On one H100 80GB HBM3 (SXM, power limit 700 W, SM clock 1980 MHz read after the run), 8 GiB table, 2 CTAs of 256
// per SM (67 584 threads), 32 M rows per launch, best of 3; look alone 31.2 G rows/s; "CAS" = per-row time over the
// look alone:
//   D (MB of 128-B lines)   0      8.2    16.5   24.8   33.0   49.5   66.0
//   G rows/s                12.34  11.06  9.51   8.89   8.76   8.74   8.73
//   CAS, ps per row         49.0   58.4   73.1   80.4   82.0   82.3   82.5
// At 32-B fetch granularity the CAS costs 81.9 ps already at 4 rounds (270 k other looks: 8.2 MB of sectors, but
// 33 MB of 128-B lines) and 84.1 at 31 rounds: L2 room is counted in lines, so a finer fetch makes none.  The more
// other lines were looked at since a row's look, the less often its CAS finds the line; past about 25 MB, almost never.
//   look, then CAS.128 after one round  the same at 4 CTAs of 256 per SM (135 168 threads), lag 0 and 1 round: what
//               the lazy LR step's row groups see, one token per thread, depositing one round of looks after the look
// Same card (700 W, 1980 MHz), 128-B fetch, look alone 31.5 G rows/s: 51.4 ps per row at lag 0, 75.2 at lag 1 (D = 16.5
// MB: one round at 1 024 threads per SM brings in as many lines as two rounds at 512).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

__device__ __forceinline__ uint64_t mix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// a 32-byte sector as two 128-bit accesses (sm_90 has no 256-bit LDG / STG), as table.cuh does
__device__ __forceinline__ void ld256(const uint8_t* p, uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d) {
  asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%4];\n\tld.global.cg.v2.u64 {%2,%3}, [%4+16];"
               : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p));
}
// The same 32-byte rows read by lane PAIRS (as xf_ld32_pair in table.cuh): lanes 2i and 2i+1 each load one 16-byte
// half of the even lane's row in one instruction and of the odd lane's row in a second one, then swap halves.  Still
// two LDG.128 per lane, but each instruction touches 16 rows instead of 32.  p == nullptr: no row (returns zeros).
__device__ __forceinline__ void ld256_pair(const uint8_t* p, uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d) {
  const uint32_t odd = threadIdx.x & 1u;
  const uint8_t* o = (const uint8_t*)__shfl_xor_sync(0xffffffffu, (unsigned long long)p, 1);
  const uint8_t* r0 = odd ? o : p;
  const uint8_t* r1 = odd ? p : o;
  uint64_t x0 = 0, x1 = 0, y0 = 0, y1 = 0;
  asm volatile("{\n .reg .pred p0, p1;\n setp.ne.u64 p0, %4, 0;\n setp.ne.u64 p1, %5, 0;\n"
               " @p0 ld.global.cg.v2.u64 {%0,%1}, [%6];\n @p1 ld.global.cg.v2.u64 {%2,%3}, [%7];\n}"
               : "+l"(x0), "+l"(x1), "+l"(y0), "+l"(y1)
               : "l"(r0), "l"(r1), "l"(r0 + 16 * odd), "l"(r1 + 16 * odd));
  const uint64_t m0 = odd ? y0 : x0, m1 = odd ? y1 : x1;  // this lane's half of its own row
  const uint64_t t0 = __shfl_xor_sync(0xffffffffu, odd ? x0 : y0, 1), t1 = __shfl_xor_sync(0xffffffffu, odd ? x1 : y1, 1);
  a = odd ? t0 : m0; b = odd ? t1 : m1; c = odd ? m0 : t0; d = odd ? m1 : t1;
}
__device__ __forceinline__ void st256(uint8_t* p, uint64_t a, uint64_t b, uint64_t c, uint64_t d) {
  asm volatile("st.global.v2.u64 [%0], {%1,%2};\n\tst.global.v2.u64 [%0+16], {%3,%4};" ::"l"(p), "l"(a), "l"(b), "l"(c),
               "l"(d) : "memory");
}

enum { M_READ = 0, M_RMW, M_LAZY, M_LAZY_SYNC, M_RED, M_PF, M_CHAIN2, M_CHAIN4, M_READ64, M_READ128, M_LD2, M_ST, M_LD_RED, M_RED2, M_CAS, M_LD_CAS_ST, M_LD_ST_RED, M_ST16, M_RED_F32, M_LD_ST16, M_CAS128, M_LD_CAS128, M_LD_CAS128_RED, M_READ_PAIR, M_READ_PAIR_CAS128 };

template <int MODE>
__global__ void __launch_bounds__(256) k(uint8_t* base, uint64_t mask, uint64_t n, uint64_t seed, uint32_t tag, uint64_t* sink) {
  uint64_t acc = 0;
  const bool pair = MODE == M_READ_PAIR || MODE == M_READ_PAIR_CAS128;
  const uint64_t n_it = pair ? (n + 31) & ~31ull : n;  // the pair modes keep whole warps in the loop
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_it; i += (uint64_t)gridDim.x * blockDim.x) {
    uint8_t* p = base + ((mix(seed + i) & mask) << 5);
    uint64_t a, b, c, d;
    if (pair) {
      ld256_pair(i < n ? p : nullptr, a, b, c, d);
      acc += a ^ b ^ c ^ d;
      if (MODE == M_READ_PAIR_CAS128 && i < n) {
        uint64_t o0, o1;
        const uint64_t n0 = c + 1, n1 = (d & 0xFFFFFFFFull) | ((uint64_t)tag << 32);
        asm volatile("{\n .reg .b128 cmp, swp, old;\n mov.b128 cmp, {%2, %3};\n mov.b128 swp, {%4, %5};\n"
                     " atom.global.cas.b128 old, [%6], cmp, swp;\n mov.b128 {%0, %1}, old;\n}"
                     : "=l"(o0), "=l"(o1) : "l"(c), "l"(d), "l"(n0), "l"(n1), "l"(p + 16) : "memory");
        acc += o0 ^ o1;
      }
    } else if (MODE == M_PF) {
      asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
    } else if (MODE == M_RED) {
      atomicAdd(reinterpret_cast<double*>(p + 24), 1.0);
    } else if (MODE == M_READ) {
      ld256(p, a, b, c, d);
      acc += a ^ b ^ c ^ d;
    } else if (MODE == M_READ64 || MODE == M_READ128) {
      // the whole 64 / 128-byte aligned group around the row (bucket probing)
      const int nb = MODE == M_READ64 ? 2 : 4;
      uint8_t* q = (uint8_t*)((uint64_t)p & ~(uint64_t)(nb * 32 - 1));
      for (int j = 0; j < nb; ++j) { ld256(q + 32 * j, a, b, c, d); acc += a ^ b ^ c ^ d; }
    } else if (MODE == M_LD2) {          // the same sector twice, the second load depends on the first
      ld256(p, a, b, c, d);
      uint8_t* q = p + ((a >> 63) << 5);  // a is 0 or small: q == p, but the address depends on the data
      ld256(q, a, b, c, d);
      acc += a ^ d;
    } else if (MODE == M_ST) {           // blind full-sector store (no load)
      st256(p, i, 1, 2, 3);
    } else if (MODE == M_ST16) {         // blind 16-byte store (half a sector)
      *reinterpret_cast<uint4*>(p + 16) = make_uint4(1, 2, 3, (uint32_t)i);
    } else if (MODE == M_LD_ST16) {      // load + 16-byte store
      ld256(p, a, b, c, d);
      *reinterpret_cast<uint4*>(p + 16) = make_uint4((uint32_t)a, 2, 3, (uint32_t)i);
    } else if (MODE == M_LD_RED) {
      ld256(p, a, b, c, d);
      atomicAdd(reinterpret_cast<double*>(p + 24), 1.0 + (double)(a & 1));
    } else if (MODE == M_RED2) {
      atomicAdd(reinterpret_cast<double*>(p + 24), 1.0);
      atomicAdd(reinterpret_cast<double*>(p + 24), 2.0);
    } else if (MODE == M_RED_F32) {
      atomicAdd(reinterpret_cast<float*>(p + 24), 1.0f);
    } else if (MODE == M_CAS) {
      acc += atomicCAS(reinterpret_cast<unsigned int*>(p + 20), 0u, 7u);
    } else if (MODE == M_LD_CAS_ST) {
      ld256(p, a, b, c, d);
      const uint32_t old_tag = (uint32_t)(c >> 32);
      const uint32_t got = atomicCAS(reinterpret_cast<unsigned int*>(p + 20), old_tag, 0xFFFFFFFFu);
      if (got == old_tag) st256(p, a, b + 1, (c & 0xFFFFFFFFull) | ((uint64_t)tag << 32), 0);
    } else if (MODE == M_LD_ST_RED) {
      ld256(p, a, b, c, d);
      st256(p, a, b + 1, (c & 0xFFFFFFFFull) | ((uint64_t)tag << 32), 0);
      atomicAdd(reinterpret_cast<double*>(p + 24), 1.0);
    } else if (MODE == M_CAS128 || MODE == M_LD_CAS128 || MODE == M_LD_CAS128_RED) {
      // claim + publish in ONE 128-bit compare-and-swap on the row's second half {w,n,z,tag}
      c = 0; d = 0;
      if (MODE != M_CAS128) ld256(p, a, b, c, d);
      uint64_t o0, o1;
      const uint64_t n0 = c + 1, n1 = (d & 0xFFFFFFFFull) | ((uint64_t)tag << 32);
      asm volatile("{\n .reg .b128 cmp, swp, old;\n mov.b128 cmp, {%2, %3};\n mov.b128 swp, {%4, %5};\n"
                   " atom.global.cas.b128 old, [%6], cmp, swp;\n mov.b128 {%0, %1}, old;\n}"
                   : "=l"(o0), "=l"(o1) : "l"(c), "l"(d), "l"(n0), "l"(n1), "l"(p + 16) : "memory");
      acc += o0 ^ o1;
      if (MODE == M_LD_CAS128_RED) atomicAdd(reinterpret_cast<unsigned long long*>(p + 8), 12345ull + (o0 & 1));
    } else if (MODE == M_RMW) {
      ld256(p, a, b, c, d);
      st256(p, a + 1, b, c, d);
    } else if (MODE == M_LAZY || MODE == M_LAZY_SYNC) {
      ld256(p, a, b, c, d);
      const uint32_t old_tag = (uint32_t)(c >> 32);
      if (MODE == M_LAZY_SYNC) __syncwarp();
      const uint32_t got = atomicCAS(reinterpret_cast<unsigned int*>(p + 20), old_tag, 0xFFFFFFFFu);
      if (MODE == M_LAZY_SYNC) __syncwarp();
      if (got == old_tag) st256(p, a, b + 1, (c & 0xFFFFFFFFull) | ((uint64_t)tag << 32), 0);
      if (MODE == M_LAZY_SYNC) __syncwarp();
      atomicAdd(reinterpret_cast<double*>(p + 24), 1.0);
    } else if (MODE == M_CHAIN2 || MODE == M_CHAIN4) {
      const int kk = MODE == M_CHAIN2 ? 2 : 4;
      for (int j = 0; j < kk; ++j) {
        ld256(p, a, b, c, d);
        acc += a;
        p = base + ((mix(seed + i + (a & 1) + 1000003ull * (j + 1)) & mask) << 5);  // depends on the loaded value
      }
    }
  }
  if (acc == 0x123456789ull) *sink = acc;
}

// A lane-pair look at a row, then a CAS.128 on that row after `lag` more rounds of looks by every thread of the grid:
// between a row's look and its CAS the GPU makes lag x (grid threads) other random looks, and D = that x the L2 fetch
// granularity (the bytes those looks fetch).  The CAS compares against the newest look, so it waits for it (as the
// step kernel's CAS waits for the row's looks); on the zeroed table both rows are almost always untouched and it
// succeeds.  The last `lag` rounds look past n (fill and drain: at most 7 % more looks in the sweep below).
__global__ void __launch_bounds__(256) klag(uint8_t* base, uint64_t mask, uint64_t n, uint64_t seed, uint32_t tag, int lag,
                                            uint64_t* sink) {
  const uint64_t T = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t K = (n + T - 1) / T;
  uint64_t acc = 0;
  for (uint64_t k = 0; k < K + (uint64_t)lag; ++k) {
    const uint64_t i = t + k * T;
    uint64_t a, b, c, d;
    ld256_pair(base + ((mix(seed + i) & mask) << 5), a, b, c, d);
    acc += a ^ b;
    if (k >= (uint64_t)lag && i - (uint64_t)lag * T < n) {
      uint8_t* p = base + ((mix(seed + i - (uint64_t)lag * T) & mask) << 5);
      uint64_t o0, o1;
      const uint64_t n0 = c + 1, n1 = (d & 0xFFFFFFFFull) | ((uint64_t)tag << 32);
      asm volatile("{\n .reg .b128 cmp, swp, old;\n mov.b128 cmp, {%2, %3};\n mov.b128 swp, {%4, %5};\n"
                   " atom.global.cas.b128 old, [%6], cmp, swp;\n mov.b128 {%0, %1}, old;\n}"
                   : "=l"(o0), "=l"(o1) : "l"(c), "l"(d), "l"(n0), "l"(n1), "l"(p + 16) : "memory");
      acc += o0 ^ o1;
    }
  }
  if (acc == 0x123456789ull) *sink = acc;
}

// V: 0 read 4 lanes x 4 x uint4 | 1 read 16 lanes x uint4 | 2 rmw 4 lanes | 3 rmw 16 lanes
template <int V>
__global__ void __launch_bounds__(256) krow(uint8_t* base, uint64_t mask, uint64_t n, uint64_t seed, uint64_t* sink) {
  const int G = (V & 1) ? 16 : 4;
  const uint64_t gid = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const uint64_t ngrp = (uint64_t)gridDim.x * blockDim.x / G;
  const int q = threadIdx.x % G;
  uint32_t acc = 0;
  for (uint64_t i = gid; i < n; i += ngrp) {
    uint4* row = reinterpret_cast<uint4*>(base + ((mix(seed + i) & mask) << 8));
    if (G == 16) {
      uint4 v = __ldcg(row + q);
      acc += v.x ^ v.w;
      if (V >= 2) { v.x += 1; row[q] = v; }
    } else {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = __ldcg(row + 4 * j + q);
#pragma unroll
      for (int j = 0; j < 4; ++j) { acc += v[j].x ^ v[j].w; if (V >= 2) { v[j].x += 1; row[4 * j + q] = v[j]; } }
    }
  }
  if (acc == 0x12345u) *sink = acc;
}

static int g_sms = 132;

template <int MODE>
static float run(const char* name, uint8_t* base, uint64_t nsect, uint64_t n, uint64_t* sink, int bps = 8, uint64_t seed0 = 77,
                 bool print = true, int reps = 3) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) {
    cudaEventRecord(e0);
    k<MODE><<<g_sms * bps, 256>>>(base, nsect - 1, n, seed0 + 1000 * r, 5 + r, sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  if (print) printf("  %-40s CTAs/SM %d  %8.1f us   %7.2f G accesses/s\n", name, bps, best * 1e3, (double)n / (best * 1e-3) / 1e9);
  return best;
}

// best of 3 launches of klag, each on the zeroed table (every CAS finds the zeros it compares against, as on the first
// launch)
static float run_lag(uint8_t* base, uint64_t nsect, uint64_t nl, int bps, int lag, uint64_t seed0, uint64_t* sink) {
  float best = 1e30f;
  for (int r = 0; r < 3; ++r) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaMemset(base, 0, nsect * 32);
    cudaEventRecord(e0);
    klag<<<g_sms * bps, 256>>>(base, nsect - 1, nl, seed0 + 1000 * r, 9 + r, lag, sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  return best;
}

int main(int argc, char** argv) {
  uint64_t mb = argc > 1 ? strtoull(argv[1], 0, 10) : 8192;
  double acc_m = argc > 2 ? atof(argv[2]) : 6.5;
  uint64_t n = (uint64_t)(acc_m * 1e6);
  uint64_t nsect = 1;
  cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0);
  while (nsect * 32 < mb * 1048576ull) nsect <<= 1;
  uint8_t* base;
  uint64_t* sink;
  cudaMalloc(&base, nsect * 32);
  cudaMalloc(&sink, 8);
  cudaMemset(base, 0, nsect * 32);
  for (int fetch = 32; fetch <= 128; fetch *= 2) {
    cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, fetch);
    printf("table %llu MiB, %llu accesses per launch, L2 fetch granularity %d B\n", (unsigned long long)(nsect * 32 >> 20),
           (unsigned long long)n, fetch);
    for (int bps = 2; bps <= 8; bps *= 2) run<M_READ>("read", base, nsect, n, sink, bps);
    for (int bps = 2; bps <= 8; bps *= 2) run<M_READ_PAIR>("read pair", base, nsect, n, sink, bps);
    run<M_READ64>("read 64-B group (2 loads)", base, nsect, n, sink);
    run<M_READ128>("read 128-B group (4 loads)", base, nsect, n, sink);
    for (int bps = 4; bps <= 8; bps *= 2) run<M_RMW>("rmw (load + store)", base, nsect, n, sink, bps);
    run<M_RED>("red f64", base, nsect, n, sink);
    for (int bps = 4; bps <= 8; bps *= 2) run<M_LAZY>("lazy (load + CAS + store + RED)", base, nsect, n, sink, bps);
    run<M_LAZY_SYNC>("lazy, warp-synchronous stages", base, nsect, n, sink);
    run<M_LD2>("load the same row twice (dependent)", base, nsect, n, sink);
    run<M_ST>("blind 32-B store", base, nsect, n, sink);
    run<M_ST16>("blind 16-B store", base, nsect, n, sink);
    run<M_LD_ST16>("load + 16-B store", base, nsect, n, sink);
    run<M_LD_RED>("load + RED", base, nsect, n, sink);
    run<M_RED2>("RED twice on the row", base, nsect, n, sink);
    run<M_RED_F32>("red f32", base, nsect, n, sink);
    run<M_CAS>("CAS only (returning)", base, nsect, n, sink);
    run<M_LD_CAS_ST>("load + CAS + store", base, nsect, n, sink);
    run<M_LD_ST_RED>("load + store + RED", base, nsect, n, sink);
    run<M_CAS128>("CAS.128 only", base, nsect, n, sink);
    run<M_LD_CAS128>("load + CAS.128", base, nsect, n, sink);
    run<M_READ_PAIR_CAS128>("read pair + CAS.128", base, nsect, n, sink);
    run<M_LD_CAS128_RED>("load + CAS.128 + RED.u64", base, nsect, n, sink);
    run<M_CHAIN2>("chain of 2 dependent loads", base, nsect, 2 * n / 2, sink);
    run<M_CHAIN4>("chain of 4 dependent loads", base, nsect, n, sink);
    // prefetch effectiveness: rows that fit L2 (64 MB), prefetched by one kernel and read by the next
    {
      const uint64_t n2 = 2000000;
      float cold = 1e30f, warm = 1e30f, pf = 1e30f;
      for (int r = 0; r < 3; ++r) {
        run<M_RED>("", base, nsect, 8000000, sink, 8, 9000 + r, false, 1);  // wipe L2 with other rows
        float c = run<M_READ>("", base, nsect, n2, sink, 8, 555 + r, false, 1);
        run<M_RED>("", base, nsect, 8000000, sink, 8, 9100 + r, false, 1);
        float p = run<M_PF>("", base, nsect, n2, sink, 8, 777 + r, false, 1);
        float w = run<M_READ>("", base, nsect, n2, sink, 8, 777 + r, false, 1);
        if (c < cold) cold = c;
        if (w < warm) warm = w;
        if (p < pf) pf = p;
      }
      printf("  prefetch.global.L2 check (2 M rows = 64 MB): cold read %.1f us, prefetch kernel %.1f us, read after prefetch %.1f us\n",
             cold * 1e3, pf * 1e3, warm * 1e3);
    }
  }
  // look, then CAS.128 on the same row after D MB of other looks (klag): does the CAS find the row's line in L2?
  {
    const uint64_t nl = 32000000;  // rows per launch: about 470 rounds of the 2-CTA-per-SM grid, 12 % of the table
    const int bps = 2;
    const uint64_t T = (uint64_t)g_sms * bps * 256;
    const int dmb[] = {0, 8, 16, 24, 32, 48, 64};
    for (int fetch = 128; fetch >= 32; fetch /= 4) {
      cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, fetch);
      const float look = run<M_READ_PAIR>("", base, nsect, nl, sink, bps, 31, false);
      printf("look, then CAS.128 after D MB of other looks: L2 fetch granularity %d B, %llu threads, %llu rows per launch,"
             " look alone %.2f G rows/s\n", fetch, (unsigned long long)T, (unsigned long long)nl, (double)nl / (look * 1e-3) / 1e9);
      for (int di = 0; di < (int)(sizeof(dmb) / sizeof(dmb[0])); ++di) {
        const int lag = (int)((double)dmb[di] * 1048576.0 / ((double)T * fetch) + 0.5);
        const float best = run_lag(base, nsect, nl, bps, lag, 4242 + 100 * di + fetch, sink);
        const double rate = (double)nl / (best * 1e-3) / 1e9;
        printf("  D %5.1f MB (lag %2d rounds)  %8.1f us  %6.2f G rows/s  CAS after the look %5.1f ps per row\n",
               (double)lag * T * fetch / 1048576.0, lag, best * 1e3, rate, 1e3 / rate - (double)look * 1e9 / nl);
      }
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(e));
  }
  // the same after exactly one round of looks by every thread, at 4 CTAs of 256 per SM: the lazy LR step's row groups
  // (one token per thread) look at all of a row's first rows in one round and deposit after it
  {
    const uint64_t nl = 32000000;
    const int bps = 4;
    const uint64_t T = (uint64_t)g_sms * bps * 256;
    cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 128);
    const float look = run<M_READ_PAIR>("", base, nsect, nl, sink, bps, 31, false);
    printf("look, then CAS.128 after one round of looks, 4 CTAs of 256 per SM (%llu threads), L2 fetch granularity 128 B,"
           " look alone %.2f G rows/s\n", (unsigned long long)T, (double)nl / (look * 1e-3) / 1e9);
    for (int lag = 0; lag <= 1; ++lag) {
      const float best = run_lag(base, nsect, nl, bps, lag, 5353 + 100 * lag, sink);
      const double rate = (double)nl / (best * 1e-3) / 1e9;
      printf("  D %5.1f MB (lag %d round)  %8.1f us  %6.2f G rows/s  CAS after the look %5.1f ps per row\n",
             (double)lag * T * 128 / 1048576.0, lag, best * 1e3, rate, 1e3 / rate - (double)look * 1e9 / nl);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(e));
  }
  // 256-byte rows (the FM k=16 FTRL row): per-thread pieces vs one cooperative instruction per row
  {
    const uint64_t nrow = nsect / 8;
    printf("256-B rows, %llu rows, %llu random rows per launch\n", (unsigned long long)nrow, (unsigned long long)n);
    void (*kern[4])(uint8_t*, uint64_t, uint64_t, uint64_t, uint64_t*) = {krow<0>, krow<1>, krow<2>, krow<3>};
    const char* names[4] = {"read row: 4 lanes x 4 x 16 B (as xf_k_update)", "read row: 16 lanes x 16 B, one instruction",
                            "rmw row: 4 lanes x 4 x 16 B", "rmw row: 16 lanes x 16 B, one instruction"};
    for (int v = 0; v < 4; ++v) {
      cudaEvent_t e0, e1;
      cudaEventCreate(&e0); cudaEventCreate(&e1);
      float best = 1e30f;
      for (int r = 0; r < 3; ++r) {
        cudaEventRecord(e0);
        kern[v]<<<g_sms * 8, 256>>>(base, nrow - 1, n, 99 + r, sink);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
      }
      printf("  %-52s %8.1f us   %7.2f G rows/s\n", names[v], best * 1e3, (double)n / (best * 1e-3) / 1e9);
    }
  }
  return 0;
}

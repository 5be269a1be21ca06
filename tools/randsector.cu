// Micro-benchmark: what can the H100's HBM3 + L2 sustain for RANDOM 32-byte sector traffic?
// The xflow hot path is exactly that access pattern (one table row = one sector), so this number —
// not the streaming-copy peak — is the practical ceiling of the probe and update kernels.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/randsector tools/randsector.cu
//   tools/randsector [table_MB=1024] [accesses_M=16]
// Prints G sectors/s and GB/s for: random 32-byte reads at several loads-in-flight per thread,
// random read-modify-write of the sector, random f64 atomic adds, with 32 B and 64 B L2 fetch granularity.
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
__device__ __forceinline__ void st256(uint8_t* p, uint64_t a, uint64_t b, uint64_t c, uint64_t d) {
  asm volatile("st.global.v2.u64 [%0], {%1,%2};\n\tst.global.v2.u64 [%0+16], {%3,%4};" ::"l"(p), "l"(a), "l"(b), "l"(c),
               "l"(d) : "memory");
}
static int g_sms = 132;

template <int MLP, int MODE>  // MODE 0 read, 1 read+write, 2 atomic f64 add
__global__ void k_rand(uint8_t* base, uint64_t nsect_mask, uint64_t per_thread, uint64_t seed, uint64_t* sink) {
  uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t acc = 0;
  for (uint64_t i = 0; i < per_thread; i += MLP) {
    uint64_t a[MLP], b[MLP], c[MLP], d[MLP];
    uint8_t* p[MLP];
#pragma unroll
    for (int m = 0; m < MLP; ++m) p[m] = base + ((mix(seed + tid * per_thread + i + m) & nsect_mask) << 5);
    if (MODE == 2) {
#pragma unroll
      for (int m = 0; m < MLP; ++m) atomicAdd(reinterpret_cast<double*>(p[m] + 24), 1.0);
    } else {
#pragma unroll
      for (int m = 0; m < MLP; ++m) ld256(p[m], a[m], b[m], c[m], d[m]);
#pragma unroll
      for (int m = 0; m < MLP; ++m) {
        acc += a[m] ^ b[m] ^ c[m] ^ d[m];
        if (MODE == 1) st256(p[m], a[m] + 1, b[m], c[m], d[m]);
      }
    }
  }
  if (acc == 0x123456789ull) *sink = acc;
}

// Ordered variants: what does address ORDER buy?  ORDER 1 = sorted sparse: access number n goes to sector
// n*S + (hash(n) mod S) — ascending addresses, one touched sector in every S (what a full sort of the
// batch by table slot would produce).  ORDER 2 = windowed: accesses are random inside a window of W
// sectors that advances with n (what a one-pass bucketing of the batch by slot prefix would produce).
template <int MLP, int MODE, int ORDER>
__global__ void k_ord(uint8_t* base, uint64_t nsect, uint64_t per_thread, uint64_t S, uint64_t W, uint64_t seed,
                      uint64_t* sink) {
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t threads = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t total = per_thread * threads;
  uint64_t acc = 0;
  for (uint64_t i = 0; i < per_thread; i += MLP) {
    uint64_t a[MLP], b[MLP], c[MLP], d[MLP];
    uint8_t* p[MLP];
#pragma unroll
    for (int m = 0; m < MLP; ++m) {
      const uint64_t n = (i + m) * threads + tid;  // all threads sweep the table together
      uint64_t sect;
      if (ORDER == 1) sect = n * S + mix(seed + n) % S;
      else sect = (n * (nsect - W) / total) + mix(seed + n) % W;
      p[m] = base + ((sect % nsect) << 5);
    }
    if (MODE == 2) {
#pragma unroll
      for (int m = 0; m < MLP; ++m) atomicAdd(reinterpret_cast<double*>(p[m] + 24), 1.0);
    } else {
#pragma unroll
      for (int m = 0; m < MLP; ++m) ld256(p[m], a[m], b[m], c[m], d[m]);
#pragma unroll
      for (int m = 0; m < MLP; ++m) {
        acc += a[m] ^ b[m] ^ c[m] ^ d[m];
        if (MODE == 1) st256(p[m], a[m] + 1, b[m], c[m], d[m]);
      }
    }
  }
  if (acc == 0x123456789ull) *sink = acc;
}

template <int MLP, int MODE, int ORDER>
static void run_ord(const char* name, uint8_t* base, uint64_t nsect, uint64_t total, uint64_t S, uint64_t W,
                    uint64_t* sink) {
  const int block = 256, grid = g_sms * 8;
  uint64_t threads = (uint64_t)block * grid;
  uint64_t per_thread = (total / threads / MLP) * MLP;
  if (per_thread == 0) per_thread = MLP;
  if (ORDER == 1) S = nsect / (per_thread * threads);  // spread the accesses over the whole table
  if (S == 0) S = 1;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  k_ord<MLP, MODE, ORDER><<<grid, block>>>(base, nsect, per_thread, S, W, 1, sink);
  float best = 1e30f;
  for (int r = 0; r < 3; ++r) {
    cudaEventRecord(e0);
    k_ord<MLP, MODE, ORDER><<<grid, block>>>(base, nsect, per_thread, S, W, 77 + r, sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  double n = (double)per_thread * threads;
  double gs = n / (best * 1e-3) / 1e9;
  printf("  %-44s S=%-3llu W=%-8llu %8.2f G sectors/s  %8.1f GB/s%s\n", name, (unsigned long long)S,
         (unsigned long long)W, gs, gs * 32 * (MODE == 1 ? 2 : 1), MODE == 1 ? " (read+write)" : "");
}

template <int MLP, int MODE>
static void run(const char* name, uint8_t* base, uint64_t nsect, uint64_t total, uint64_t* sink) {
  const int block = 256, grid = g_sms * 8;
  uint64_t threads = (uint64_t)block * grid;
  uint64_t per_thread = (total / threads / MLP) * MLP;
  if (per_thread == 0) per_thread = MLP;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  k_rand<MLP, MODE><<<grid, block>>>(base, nsect - 1, per_thread, 1, sink);  // warm-up
  float best = 1e30f;
  for (int r = 0; r < 3; ++r) {
    cudaEventRecord(e0);
    k_rand<MLP, MODE><<<grid, block>>>(base, nsect - 1, per_thread, 77 + r, sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  double n = (double)per_thread * threads;
  double gs = n / (best * 1e-3) / 1e9;
  printf("  %-34s %8.2f G sectors/s  %8.1f GB/s%s\n", name, gs, gs * 32 * (MODE == 1 ? 2 : 1),
         MODE == 1 ? " (read+write)" : "");
}

int main(int argc, char** argv) {
  uint64_t mb = argc > 1 ? strtoull(argv[1], 0, 10) : 1024;
  uint64_t total = (argc > 2 ? strtoull(argv[2], 0, 10) : 16) * 1000000ull;
  uint64_t nsect = 1;
  cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0);
  while (nsect * 32 < mb * 1048576ull) nsect <<= 1;
  uint8_t* base;
  uint64_t* sink;
  cudaMalloc(&base, nsect * 32);
  cudaMalloc(&sink, 8);
  cudaMemset(base, 0, nsect * 32);
  for (int gran = 64; gran >= 32; gran -= 32) {
    cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran);
    size_t got = 0;
    cudaDeviceGetLimit(&got, cudaLimitMaxL2FetchGranularity);
    printf("table %llu MB, %llu M accesses, L2 fetch granularity requested %d got %zu\n",
           (unsigned long long)(nsect * 32 >> 20), (unsigned long long)(total / 1000000), gran, got);
    run<1, 0>("random 32B read, 1 in flight/thread", base, nsect, total, sink);
    run<2, 0>("random 32B read, 2 in flight/thread", base, nsect, total, sink);
    run<4, 0>("random 32B read, 4 in flight/thread", base, nsect, total, sink);
    run<8, 0>("random 32B read, 8 in flight/thread", base, nsect, total, sink);
    run<4, 1>("random 32B read-modify-write, 4", base, nsect, total, sink);
    run<4, 2>("random f64 atomicAdd (RED), 4", base, nsect, total, sink);
  }
  // address-order experiments at the default granularity: `total` accesses spread over the table
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  printf("ordered access, table %llu MB, %llu M accesses\n", (unsigned long long)(nsect * 32 >> 20),
         (unsigned long long)(total / 1000000));
  run_ord<4, 0, 1>("sorted sparse read", base, nsect, total, 0, 0, sink);
  run_ord<4, 1, 1>("sorted sparse read-modify-write", base, nsect, total, 0, 0, sink);
  run_ord<4, 2, 1>("sorted sparse f64 atomicAdd", base, nsect, total, 0, 0, sink);
  for (uint64_t wmb = 1; wmb <= 256; wmb *= 4) {
    const uint64_t W = wmb * 1048576ull / 32;
    if (W >= nsect) break;
    run_ord<4, 0, 2>("windowed random read", base, nsect, total, 0, W, sink);
    run_ord<4, 1, 2>("windowed random read-modify-write", base, nsect, total, 0, W, sink);
    run_ord<4, 2, 2>("windowed random f64 atomicAdd", base, nsect, total, 0, W, sink);
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("CUDA error %s\n", cudaGetErrorString(e)); return 1; }
  return 0;
}

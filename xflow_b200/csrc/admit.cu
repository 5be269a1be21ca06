// Feature admission (McMahan et al., "Ad Click Prediction: a View from the Trenches", section 5.1): the counting
// Bloom filter behind XF_ADMIT_BLOOM.  The step kernels decide (xf_admit, table.cuh) and append every rejected
// token's key to the trainer's rejected-token list; these two kernels then run on the table's stream after the step:
//   xf_k_admit_count  each rejected token adds 1 to each of its `hashes` cells, saturating at 255.  A cell is a
//                     byte: the add is a CAS on the aligned 32-bit word that holds it.  Saturating increments
//                     commute, so the filter after a batch does not depend on the order the atomics land in.
//   xf_k_admit_decay  halves every cell (the "rolling" filter, every decay_batches batches).
// Poisson admission needs neither: it has no state.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "table.cuh"

__device__ __forceinline__ void xf_admit_add(uint8_t* cells, uint64_t c) {
  unsigned int* word = reinterpret_cast<unsigned int*>(cells + (c & ~3ull));
  const unsigned int shift = (unsigned int)(c & 3ull) * 8u;
  unsigned int old = *reinterpret_cast<volatile unsigned int*>(word);
  for (;;) {
    if (((old >> shift) & 0xFFu) == 0xFFu) return;  // saturated
    const unsigned int prev = atomicCAS(word, old, old + (1u << shift));
    if (prev == old) return;
    old = prev;
  }
}

__global__ void xf_k_admit_count(XfAdmitView a, uint8_t* cells, const uint64_t* __restrict__ rej_keys,
                                 const unsigned long long* rej_n, unsigned long long* rejected_total,
                                 unsigned long long* next_rej_n) {
  const unsigned long long n = *rej_n;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    atomicAdd(rejected_total, n);
    *next_rej_n = 0ull;  // the list position of the next batch (its previous user was the batch before this one)
  }
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const uint64_t key = rej_keys[i];
    for (uint32_t j = 0; j < a.hashes; ++j) xf_admit_add(cells, xf_admit_cell(key, a.seed, j, a.log2_cells));
  }
}

__global__ void xf_k_admit_decay(uint4* cells, uint64_t n16) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (uint64_t)gridDim.x * blockDim.x) {
    uint4 v = cells[i];
    v.x = (v.x >> 1) & 0x7F7F7F7Fu;
    v.y = (v.y >> 1) & 0x7F7F7F7Fu;
    v.z = (v.z >> 1) & 0x7F7F7F7Fu;
    v.w = (v.w >> 1) & 0x7F7F7F7Fu;
    cells[i] = v;
  }
}

void xf_launch_admit_count(const XfAdmitView& a, uint8_t* cells, const uint64_t* rej_keys, const unsigned long long* rej_n,
                           uint32_t nnz, unsigned long long* rejected_total, unsigned long long* next_rej_n,
                           cudaStream_t st) {
  const int grid = xf_grid_for(nnz ? (uint64_t)nnz : 1ull, 256, 8);
  xf_k_admit_count<<<grid, 256, 0, st>>>(a, cells, rej_keys, rej_n, rejected_total, next_rej_n);
}

void xf_launch_admit_decay(uint8_t* cells, uint32_t log2_cells, cudaStream_t st) {
  const uint64_t n16 = (1ull << log2_cells) / 16;  // log2_cells >= 10
  xf_k_admit_decay<<<xf_grid_for(n16, 256, 8), 256, 0, st>>>(reinterpret_cast<uint4*>(cells), n16);
}

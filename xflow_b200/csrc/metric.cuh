// Pieces shared by the device metrics: xf_metric (metric.cu), progressive validation (validate.cu) and the grouped
// test metric (group_metric.cu).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "internal.h"

// ---- device: exact multi-word sums
__device__ __forceinline__ void xf_add128(unsigned long long& lo, unsigned long long& hi, unsigned long long alo,
                                          unsigned long long ahi) {
  lo += alo;
  hi += ahi + (lo < alo ? 1ull : 0ull);
}

// a multi-word atomic add: every word's carry is decided by the old value its own atomic returned, so the words hold
// the exact sum (mod 2^(64 n)) whatever the order of the adds
__device__ __forceinline__ void xf_atomic_add128(unsigned long long* w, unsigned long long lo, unsigned long long hi) {
  if (lo) {
    const unsigned long long old = atomicAdd(w, lo);
    if (old + lo < old) ++hi;
  }
  if (hi) atomicAdd(w + 1, hi);
}

// A row's logloss term in units of 2^-32 (include/xflow_b200.h sections 8 and 9): q = p clamped to [1e-15, 1 - 1e-15]
// in double, l = -ln(q) for a positive row (pos != 0) and -ln(1 - q) for a negative one, and e * l * 2^32 rounded once
// in double, then to the nearest integer xl + 2^64 xh (e < 2^31: below 2^69 units).
__device__ __forceinline__ void xf_loss_units(float e, float p, int pos, unsigned long long& xl,
                                              unsigned long long& xh) {
  const double q = fmin(fmax((double)p, 1e-15), 1.0 - 1e-15);
  const double l = pos ? -log(q) : -log(1.0 - q);
  const double x = (double)e * l * 4294967296.0;  // < 2^69 units
  if (x < 0x1p64) {
    xl = __double2ull_rn(x);
    xh = 0;
  } else {  // an integer: the split is exact
    xh = (unsigned long long)(x * 0x1p-64);
    xl = (unsigned long long)(x - (double)xh * 0x1p64);
  }
}

// ---- host
// an unsigned 256-bit integer, least significant word first
struct XfU256 {
  uint64_t w[4] = {0, 0, 0, 0};
};
// num / den correctly rounded to double (round to nearest even); NaN when den = 0; num, den < 2^192 (validate.cu)
double xf_ratio(XfU256 num, XfU256 den);
// grow a device buffer to at least `want` bytes keeping its first `used`: the copy is stream-ordered after everything
// queued on `st`, and the call waits for `st` before it frees the old buffer (metric.cu)
int xf_grow_keep(XfDevBuf& b, size_t used, size_t want, cudaStream_t st);

"""numpy restatement of the deterministic training step's per-key sums (xf_trainer_set_deterministic, csrc/step_det.cu;
include/xflow_b200.h section 3): each key's terms in token order, cut into runs of 32; a run summed by the xor
butterfly over 32 lanes with -0.0 in the lanes past it; the run sums added in order onto the accumulator.  float32
terms add in float32, float64 terms in float64, every add rounded to nearest.  Also the optimizer's SGD step of the
canonical rows (xf_k_update, kernels.cu), for a table after one deterministic step."""
from fractions import Fraction

import numpy as np

RUN = 32


def butterfly(terms):
    """a_0 of the butterfly over one run: terms[i] in lane i (i < 32, along axis 0), -0.0 past them; for o = 16 .. 1
    a_i = a_i + a_(i^o)."""
    terms = np.asarray(terms)
    assert 1 <= terms.shape[0] <= RUN
    a = np.full((RUN,) + terms.shape[1:], -0.0, terms.dtype)
    a[:terms.shape[0]] = terms
    lanes = np.arange(RUN)
    for o in (16, 8, 4, 2, 1):
        a = a + a[lanes ^ o]  # same dtype: one rounding per add
    return a[0]


def key_sum(terms, start):
    """The accumulator after adding a key's terms (token order, along axis 0) run by run onto `start`."""
    terms = np.asarray(terms)
    acc = np.array(start, terms.dtype)
    for i in range(0, terms.shape[0], RUN):
        acc = acc + butterfly(terms[i:i + RUN])
    return acc


def fmc_terms(r, x, S):
    """Canonical FM terms of tokens with residual r, value x and row sums S[., K]: A = fl(fl(r x) S_k) (float32),
    G = r x and L2 = r x x (float64)."""
    r, x = np.asarray(r, np.float32), np.asarray(x, np.float32)
    A = (r * x)[:, None] * np.asarray(S, np.float32)
    G = r.astype(np.float64) * x.astype(np.float64)
    return A, G, G * x.astype(np.float64)


def sums_by_key(keys, A, G=None, L=None):
    """{key: (A, G, L2)} accumulators after one step: tokens grouped by key in token order; A and L2 from +0, G from
    -0.0.  G / L None: the multi-view machine (g terms +0.0, L2 untouched)."""
    out = {}
    for k in np.unique(keys):
        idx = np.nonzero(keys == k)[0]
        a = key_sum(A[idx], np.zeros(A.shape[1], np.float32))
        if G is None:
            out[int(k)] = (a, key_sum(np.zeros(idx.size), -0.0), 0.0)
        else:
            out[int(k)] = (a, key_sum(G[idx], -0.0), key_sum(L[idx], 0.0))
    return out


def _fma(a, b, c):
    """fl(a b + c) in float64 (the update kernel's contracted multiply-add), exactly rounded once"""
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def sgd_update(w, v, acc, rows, lr):
    """One SGD step of a canonical row from its accumulators (A, G, L2): gw = (float)G / rows, gv_k =
    (float)fma(-v_k, L2, A_k) / rows, each quotient rounded to float; w - lr gw and v_k - lr gv_k in float32."""
    A, G, L = acc
    lr = np.float32(lr)
    gw = np.float32(np.float64(np.float32(G)) / rows)
    gv = np.array([np.float32(np.float64(np.float32(_fma(-vk, L, ak))) / rows) for vk, ak in zip(v, A)], np.float32)
    return np.float32(w) - lr * gw, np.asarray(v, np.float32) - lr * gv

"""CPU statement of importance-weighted training (include/xflow_b200.h: xf_trainer_step_host_weighted,
xf_trainer_set_negative_sampling) on top of the oracle's table and the admission model.

`WeightingTable` is an `AdmittingTable` whose step takes optional row weights and applies the trainer's
negative-sampling policy:
  * every row gets its effective weight e_r = c_r * s_r (float32 product, `row_weights`);
  * if every e_r is 1 the step is the unweighted one, and the oracle's own arithmetic runs (AdmittingTable.step);
  * otherwise only the rows with e_r > 0 are trained: the admission decisions, the pull and the push see only their
    keys, and only their rejected tokens count into the Bloom filter.  The forward pass is the oracle's
    (xo_worker_compute_given on the trained rows); the gradients are the oracle's calculate_gradient in its exact_sums
    arithmetic (xo_gradient_exact) with loss_r = e_r * (pctr_r - label_r) (float32): the same float32 terms, FM's
    S_r restated in the oracle's summation order, summed per key in float64 and divided by the batch's full row count
    B.  With weights of 1 (always_weighted=True) this path equals the oracle's exact_sums step bit for bit.
step returns (keys pushed, unweighted residuals with 0 for skipped rows, mean_abs_loss), so `oracle.train_file` /
`predict_file` drive it unchanged.
"""
import numpy as np

from admission_model import ADMIT_BLOOM, AdmittingTable, bloom_cells
from oracle import oracle as O
from xflow_b200 import datagen

M64 = (1 << 64) - 1


def p24_of(rate):
    return int(np.floor(np.float64(np.float32(rate)) * 16777216.0))


def row_hash_sums(row_ptr, keys):
    """F_r = sum over the row's tokens of splitmix64(key) mod 2^64 (0 for a row without tokens)."""
    row_ptr = np.asarray(row_ptr, np.int64)
    h = datagen.splitmix64(np.ascontiguousarray(keys, np.uint64)) if len(keys) else np.zeros(0, np.uint64)
    with np.errstate(over="ignore"):
        cs = np.concatenate([np.zeros(1, np.uint64), np.cumsum(h, dtype=np.uint64)])
        return cs[row_ptr[1:]] - cs[row_ptr[:-1]]


def kept_negatives(row_ptr, keys, rate, seed):
    """Per row: would a negative row be kept (top 24 bits of splitmix64(seed ^ F_r) < floor(rate * 2^24))."""
    F = row_hash_sums(row_ptr, keys)
    with np.errstate(over="ignore"):
        return (datagen.splitmix64(F ^ np.uint64(seed)) >> np.uint64(40)) < np.uint64(p24_of(rate))


def row_weights(row_ptr, keys, labels, weights=None, rate=1.0, seed=0):
    """e_r = c_r * s_r in float32 (c_r = weights or 1; s_r from the negative-sampling policy)."""
    B = np.asarray(labels).size
    c = np.ones(B, np.float32) if weights is None else np.asarray(weights, np.float32)
    s = np.ones(B, np.float32)
    if rate < 1.0:
        inv = np.float32(1.0 / np.float64(np.float32(rate)))
        neg = np.asarray(labels) == 0
        kept = kept_negatives(row_ptr, keys, rate, seed)
        s[neg] = np.where(kept[neg], inv, np.float32(0))
    return (c * s).astype(np.float32)


def fix_bound(row_ptr, e):
    """W = sum over the trained rows of ceil(e_r) * tokens_r (ceil capped at 2^31), the lazy step's bound."""
    lens = np.diff(np.asarray(row_ptr, np.int64))
    m = np.minimum(np.ceil(e.astype(np.float64)), 2.0 ** 31).astype(np.int64)
    return int(np.sum(np.where(e > 0, m * lens, 0)))


def fix_shift(n):
    """include: xf_fix_shift"""
    s = 47 - int(n).bit_length()
    return max(0, min(27, s))


def oracle_row_sums(K, row_ptr, vt):
    """The oracle's v_sum (xo_forward): per row, float32 sums over k (outer) and the row's tokens in ascending key
    order (inner).  vt[j] = the latent row of token j, tokens already in that order within each row."""
    row_ptr = np.asarray(row_ptr, np.int64)
    rows = row_ptr.size - 1
    lens = np.diff(row_ptr)
    S = np.zeros(rows, np.float32)
    for k in range(K):
        for p in range(int(lens.max()) if rows else 0):
            r = np.flatnonzero(lens > p)
            S[r] = (S[r] + vt[row_ptr[r] + p, k]).astype(np.float32)
    return S


def weighted_gradients(K, row_ptr, keys, e, pctr_minus_label, w, v, B):
    """The oracle's calculate_gradient in its exact_sums arithmetic (xo_gradient_exact) with loss_r = e_r * residual_r,
    over the SORTED unique keys of the (trained) rows: float32 terms (FM: loss_r * (S_r - v_ik), S_r the oracle's
    v_sum; the w-term the K-fold float32 sum of loss_r), summed per key in float64, rounded to float32 and divided by B
    as lr_worker.cc:116-118 does.  Returns (gw[U], gv[U, K], loss_w[rows])."""
    row_ptr = np.asarray(row_ptr, np.int64)
    keys = np.ascontiguousarray(keys, np.uint64)
    rows = row_ptr.size - 1
    lw = (e.astype(np.float32) * pctr_minus_label.astype(np.float32)).astype(np.float32)
    sid = np.repeat(np.arange(rows), np.diff(row_ptr))
    order = np.lexsort((keys, sid))      # within each row, ascending key: the oracle's sorted all_keys
    keys, sid = keys[order], sid[order]
    uk, inv = np.unique(keys, return_inverse=True)
    lk = lw
    if K > 0:
        lk = np.zeros(rows, np.float32)
        for _ in range(K):
            lk = (lk + lw).astype(np.float32)
    gw = np.zeros(uk.size, np.float64)
    np.add.at(gw, inv, lk[sid].astype(np.float64))
    gv = np.zeros((uk.size, K), np.float64)
    if K > 0:
        vt = v[inv]                                      # [tokens, K]
        S = oracle_row_sums(K, row_ptr, vt)              # the row's v summed over tokens AND k (fm_worker.cc:178-192)
        term = (lw[sid, None] * (S[sid, None] - vt).astype(np.float32)).astype(np.float32)
        np.add.at(gv, inv, term.astype(np.float64))
    gw = (gw.astype(np.float32) / np.float64(B)).astype(np.float32)
    gv = (gv.astype(np.float32) / np.float64(B)).astype(np.float32)
    return uk, gw, gv, lw


class WeightingTable(AdmittingTable):
    def __init__(self, always_weighted=False, **table_kwargs):
        """always_weighted: take the weighted path even when every e_r is 1 (to check it against the oracle)."""
        super().__init__(**table_kwargs)
        self.rate, self.seed_neg, self.skipped = 1.0, 0, 0
        self.always_weighted = always_weighted

    def set_negative_sampling(self, rate, seed=0):
        self.rate, self.seed_neg = float(np.float32(rate)), seed

    def step(self, row_ptr, keys, labels, weights=None):
        """One weighted update() on a slice; returns (keys pushed, residual[B], mean_abs_loss)."""
        row_ptr = np.asarray(row_ptr, np.int64)
        keys = np.ascontiguousarray(keys, np.uint64)
        labels = np.asarray(labels, np.int32)
        B = labels.size
        if B == 0:
            U, loss = super().step(row_ptr, keys, labels)
            return U, loss, 0.0
        e = row_weights(row_ptr, keys, labels, weights, self.rate, self.seed_neg)
        if np.all(e == 1) and not self.always_weighted:
            U, loss = super().step(row_ptr, keys, labels)
            return U, loss, float(np.sum(np.abs(loss.astype(np.float64))) / B)
        trained = np.flatnonzero(e > 0)
        self.skipped += B - trained.size
        lens = np.diff(row_ptr)
        sub_rp = np.concatenate([[0], np.cumsum(lens[trained])]).astype(np.int64)
        sub_keys = keys[np.concatenate([np.arange(row_ptr[r], row_ptr[r + 1]) for r in trained])] \
            if trained.size else np.zeros(0, np.uint64)
        sub_keys = np.ascontiguousarray(sub_keys, np.uint64)
        sub_lab = labels[trained]
        uk = np.unique(sub_keys)
        if self.mode == 0:
            keep = np.ones(uk.size, bool)
        else:
            present = self.t.export(uk)["present"].astype(bool)
            admit = self._admits(uk[~present])
            keep = present.copy()
            keep[~present] = admit
            self.admitted += int(admit.sum())
        w, v = self._values(uk, keep)
        residual = np.zeros(B, np.float32)
        U = 0
        if trained.size:
            # the oracle's forward on the trained rows (its gradient, divided by their count, is not used)
            _, _, res = O.worker_compute_given(self.K, sub_rp, sub_keys, sub_lab, w, v if self.K else None)
            residual[trained] = res
            _, gw, gv, _ = weighted_gradients(self.K, sub_rp, sub_keys, e[trained], res, w, v, B)
            if keep.any():
                self.t.push(uk[keep], gw=gw[keep])
                if self.K:
                    self.t.push(uk[keep], gv=gv[keep])
            U = int(keep.sum())
        if self.mode != 0:
            rej_tokens = sub_keys[~keep[np.searchsorted(uk, sub_keys)]] if sub_keys.size else sub_keys
            self.rejected += int(rej_tokens.size)
            if self.mode == ADMIT_BLOOM:
                if rej_tokens.size:
                    np.add.at(self.cells, bloom_cells(rej_tokens, self.seed, self.hashes, self.log2_cells).ravel(), 1)
                    np.minimum(self.cells, 255, out=self.cells)
                if self.decay and (self.batches + 1) % self.decay == 0:
                    self.cells >>= 1
        self.batches += 1
        mal = float(np.sum(e.astype(np.float64) * np.abs(residual.astype(np.float64))) / B)
        return U, residual, mal

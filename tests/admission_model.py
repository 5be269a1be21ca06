"""CPU statement of feature admission (include/xflow_b200.h: xf_table_set_admission) on top of the oracle's table.

`AdmittingTable` wraps an `oracle.Table` and runs a training step the way the device does with a policy set:
  * split the slice's sorted unique keys into present, admitted and rejected (the Bloom filter as it stood before
    the batch, or the Poisson draw of (key, batch));
  * pull only the present and admitted keys (w, then v, in key order, as xo_worker_compute does); rejected keys read
    as w = 0, v = 0;
  * residuals and gradients from those values (xo_worker_compute_given: the oracle's calculate_loss /
    calculate_gradient);
  * push only the present and admitted keys;
  * then count every rejected token into the filter (saturating at 255) and apply the decay.
Predict with a policy never inserts: absent keys contribute 0.  Without a policy every call is the oracle's own.
It has `init_push`, `step` and `predict` with the oracle's signatures, so `oracle.train_file` / `predict_file`
drive it unchanged.
"""
import numpy as np

from oracle import oracle as O
from xflow_b200 import datagen

ADMIT_ALL, ADMIT_POISSON, ADMIT_BLOOM = 0, 1, 2
GOLDEN_GAMMA = np.uint64(0x9E3779B97F4A7C15)


def _mix(x):
    return datagen.splitmix64(np.array([x], np.uint64))[0]


def bloom_cells(keys, seed, hashes, log2_cells):
    """[hashes, n] cell indices: top log2_cells bits of splitmix64(key ^ splitmix64(seed + (j + 1) * golden))."""
    keys = np.asarray(keys, np.uint64)
    with np.errstate(over="ignore"):
        mixes = [_mix(np.uint64(seed) + np.uint64(j + 1) * GOLDEN_GAMMA) for j in range(hashes)]
        return np.stack([(datagen.splitmix64(keys ^ m) >> np.uint64(64 - log2_cells)).astype(np.int64) for m in mixes])


def poisson_admits(keys, seed, batch, p24):
    """top 24 bits of splitmix64(key ^ splitmix64(seed + b)) < p24"""
    keys = np.asarray(keys, np.uint64)
    with np.errstate(over="ignore"):
        mix = _mix(np.uint64(seed) + np.uint64(batch))
        return (datagen.splitmix64(keys ^ mix) >> np.uint64(40)) < np.uint64(p24)


class AdmittingTable:
    def __init__(self, **table_kwargs):
        self.t = O.Table(**table_kwargs)
        self.K = self.t.K
        self.mode = ADMIT_ALL
        self.cells = np.zeros(0, np.int64)
        self.batches = self.rejected = self.admitted = 0

    def set_admission(self, mode, probability=1.0, threshold=2, log2_cells=30, hashes=3, decay_batches=0, seed=0):
        """Replaces the policy and clears the filter; the counters run on."""
        self.mode, self.threshold, self.log2_cells, self.hashes = mode, threshold, log2_cells, hashes
        self.decay, self.seed = decay_batches, seed
        self.p24 = int(np.floor(np.float64(np.float32(probability)) * 16777216.0))
        self.cells = np.zeros(1 << log2_cells if mode == ADMIT_BLOOM else 0, np.int64)

    def admission_stats(self):
        return dict(batches=self.batches, rejected_tokens=self.rejected, admitted_keys=self.admitted)

    def admission_filter(self):
        return self.cells.astype(np.uint8)

    # ---- the oracle.Table surface used by the tests and by oracle.train_file / predict_file
    def size(self):
        return self.t.size()

    def export(self, keys):
        return self.t.export(keys)

    def init_push(self):
        self.t.init_push()

    def _admits(self, absent):
        if self.mode == ADMIT_POISSON:
            return poisson_admits(absent, self.seed, self.batches, self.p24)
        if absent.size == 0:
            return np.zeros(0, bool)
        return self.cells[bloom_cells(absent, self.seed, self.hashes, self.log2_cells)].min(0) >= self.threshold

    def _values(self, uk, keep):
        """w, v of the sorted unique keys: pulled for `keep` (inserting admitted keys), 0 elsewhere."""
        w = np.zeros(uk.size, np.float32)
        v = np.zeros((uk.size, self.K), np.float32)
        if keep.any():
            pw, pv = self.t.pull(uk[keep])
            w[keep] = pw
            if self.K:
                v[keep] = pv
        return w, v

    def step(self, row_ptr, keys, labels):
        """One update() on a slice; returns (keys pushed, loss[B])."""
        B = np.asarray(labels).size
        if B == 0:  # an empty slice is not a training batch
            return self.t.step(row_ptr, keys, labels)
        if self.mode == ADMIT_ALL:
            self.batches += 1
            return self.t.step(row_ptr, keys, labels)
        keys = np.ascontiguousarray(keys, np.uint64)
        uk = np.unique(keys)
        present = self.t.export(uk)["present"].astype(bool)
        admit = self._admits(uk[~present])
        keep = present.copy()
        keep[~present] = admit
        self.admitted += int(admit.sum())
        w, v = self._values(uk, keep)
        gw, gv, loss = O.worker_compute_given(self.K, row_ptr, keys, labels, w, v if self.K else None)
        if keep.any():
            self.t.push(uk[keep], gw=gw[keep])
            if self.K:
                self.t.push(uk[keep], gv=gv[keep])
        rej_tokens = keys[~keep[np.searchsorted(uk, keys)]] if keys.size else keys
        self.rejected += int(rej_tokens.size)
        if self.mode == ADMIT_BLOOM:
            if rej_tokens.size:
                np.add.at(self.cells, bloom_cells(rej_tokens, self.seed, self.hashes, self.log2_cells).ravel(), 1)
                np.minimum(self.cells, 255, out=self.cells)  # saturating adds commute: min(255, c + count)
            if self.decay and (self.batches + 1) % self.decay == 0:
                self.cells >>= 1
        self.batches += 1
        return int(keep.sum()), loss

    def predict(self, row_ptr, keys):
        if self.mode == ADMIT_ALL:
            return self.t.predict(row_ptr, keys)
        keys = np.ascontiguousarray(keys, np.uint64)
        B = np.asarray(row_ptr).size - 1
        uk = np.unique(keys)
        e = self.t.export(uk)  # no insert
        keep = e["present"].astype(bool)
        w = np.where(keep, e["w"], np.float32(0)).astype(np.float32)
        v = np.where(keep[:, None], e["v"], np.float32(0)).astype(np.float32) if self.K else None
        # calculate_loss with labels 0: the residual pctr - 0 is pctr
        _, _, pctr = O.worker_compute_given(self.K, row_ptr, keys, np.zeros(B, np.int32), w, v)
        return pctr

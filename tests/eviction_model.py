"""CPU statement of feature eviction (include/xflow_b200.h: xf_table_set_eviction / xf_table_evict) on top of the
oracle's table and the admission model.

`EvictingTable` wraps an `AdmittingTable` (so admission and eviction combine) and keeps a stamp per present key:
  * a training step of batch b stamps every key that one of its tokens reads from a row (present before the step,
    or inserted / admitted by it) with b; a rejected token stamps nothing;
  * any other insertion (predict's insert-on-pull, pull, push, import, init_push) stamps the new key with the number
    of training batches run so far; an existing key keeps its stamp;
  * when tracking starts, every present key gets the number of training batches run so far.
A sweep at batch number B keeps the keys with stamp >= B - T (T > 0, B > T) and then, with max_keys = N > 0, the N
most recent of them (larger stamp first, then smaller key).  The oracle's table is rebuilt as a fresh `O.Table` with
the same parameters and the survivors' full state (w, n, z, v, nv, zv) imported.
It has `init_push`, `step` and `predict` with the oracle's signatures, and with `every = E` it sweeps after each
training step that makes the batch number a multiple of E, so `oracle.train_file` runs it as the CLI does.
"""
import numpy as np

from admission_model import AdmittingTable
from oracle import oracle as O

UNTOUCHED = np.uint64(0xFFFFFFFFFFFFFFFF)


def survivors(keys, stamps, B, max_idle_batches, max_keys):
    """The keep mask of a sweep at batch number B over present keys with their stamps."""
    keys = np.asarray(keys, np.uint64)
    stamps = np.asarray(stamps, np.int64)
    keep = np.ones(keys.size, bool)
    if max_idle_batches > 0 and B > max_idle_batches:
        keep &= stamps >= B - max_idle_batches
    if max_keys > 0 and keep.sum() > max_keys:
        idx = np.flatnonzero(keep)
        order = np.lexsort((keys[idx], -stamps[idx]))  # most recent first: larger stamp, then smaller key
        keep[:] = False
        keep[idx[order[:max_keys]]] = True
    return keep


class EvictingTable:
    def __init__(self, **table_kwargs):
        self.kw = table_kwargs
        self.a = AdmittingTable(**table_kwargs)
        self.K = self.a.K
        self.stamp = {}  # present key -> stamp (kept whether or not tracking is on; reset when it starts)
        self.tracking = False
        self.T = self.N = self.every = 0
        self.sweeps = self.evicted = 0

    # ---- policies
    def set_admission(self, *a, **k):
        self.a.set_admission(*a, **k)

    def admission_stats(self):
        return self.a.admission_stats()

    @property
    def batches(self):
        return self.a.batches

    def set_eviction(self, max_idle_batches=0, max_keys=0, every=0):
        if not self.tracking:
            self.stamp = {k: self.batches for k in self.stamp}
        self.tracking = True
        self.T, self.N, self.every = max_idle_batches, max_keys, every

    def last_touch(self, keys):
        return np.array([self.stamp.get(int(k), UNTOUCHED) for k in np.asarray(keys, np.uint64)], np.uint64)

    def keys(self):
        return np.array(sorted(self.stamp), np.uint64)

    # ---- insertion bookkeeping
    def _inserted(self, keys):
        """Stamp the keys of `keys` that are present now and were not before with the current batch number."""
        uk = np.unique(np.asarray(keys, np.uint64))
        if uk.size == 0:
            return
        present = self.a.t.export(uk)["present"].astype(bool)
        for k in uk[present]:
            self.stamp.setdefault(int(k), self.batches)

    # ---- the oracle.Table surface
    def size(self):
        return self.a.size()

    def export(self, keys):
        return self.a.export(keys)

    def init_push(self):
        self.a.init_push()
        self._inserted(np.zeros(1, np.uint64))

    def pull(self, keys):
        out = self.a.t.pull(keys)
        self._inserted(keys)
        return out

    def push(self, keys, gw=None, gv=None):
        self.a.t.push(keys, gw, gv)
        self._inserted(keys)

    def import_(self, keys, **fields):
        self.a.t.import_(keys, **fields)
        self._inserted(keys)

    def step(self, row_ptr, keys, labels):
        B = np.asarray(labels).size
        if B == 0:
            return self.a.step(row_ptr, keys, labels)
        b = self.batches
        out = self.a.step(row_ptr, keys, labels)
        uk = np.unique(np.asarray(keys, np.uint64))
        if uk.size:
            read = self.a.t.export(uk)["present"].astype(bool)  # keys with a row: present or admitted
            for k in uk[read]:
                self.stamp[int(k)] = b
        if self.every and self.batches % self.every == 0:
            self.evict()
        return out

    def predict(self, row_ptr, keys):
        p = self.a.predict(row_ptr, keys)
        self._inserted(keys)
        return p

    # ---- the sweep
    def evict(self):
        assert self.tracking
        self.sweeps += 1
        keys = self.keys()
        if keys.size == 0:
            return 0
        stamps = np.array([self.stamp[int(k)] for k in keys], np.int64)
        keep = survivors(keys, stamps, self.batches, self.T, self.N)
        if keep.all():
            return 0
        kept = keys[keep]
        e = self.a.t.export(kept)
        t = O.Table(**self.kw)
        if kept.size:
            v = dict(v=e["v"], nv=e["nv"], zv=e["zv"]) if self.K else {}
            t.import_(kept, w=e["w"], nw=e["nw"], zw=e["zw"], **v)
        self.a.t = t
        for k in keys[~keep]:
            del self.stamp[int(k)]
        self.evicted += int((~keep).sum())
        return int((~keep).sum())

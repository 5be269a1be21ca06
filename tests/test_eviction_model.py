"""The CPU statement of feature eviction (tests/eviction_model.py, the yardstick of tests/test_gpu_eviction.py)
against a scalar restatement written token by token in plain Python: the stamps of training steps, predict inserts and
init_push, and the sweep's idle edge, its key-budget boundary with ties broken by key, a budget above the key count,
and both limits together."""
import numpy as np

from eviction_model import EvictingTable, survivors
from xflow_b200 import datagen


class ScalarStamps:
    """One token at a time: a dict of present keys and their stamps, and a sweep by sorting."""

    def __init__(self):
        self.stamp = {}
        self.b = 0

    def train(self, keys):
        keys = [int(k) for k in keys]
        if not keys:
            return
        for k in keys:
            self.stamp[k] = self.b
        self.b += 1

    def insert(self, keys):
        for k in keys:
            self.stamp.setdefault(int(k), self.b)

    def sweep(self, T, N):
        live = sorted(self.stamp.items(), key=lambda kv: (-kv[1], kv[0]))
        if T > 0 and self.b > T:
            live = [(k, s) for k, s in live if s >= self.b - T]
        if N > 0:
            live = live[:N]
        before = len(self.stamp)
        self.stamp = dict(live)
        return before - len(self.stamp)


def _batch(seed, B=64, d=6, space=400):
    rp, keys, lab = datagen.make_csr_keys(seed, B, d, space, lambda ids: np.asarray(ids, np.uint64) + 1, dist="zipf",
                                          zipf_s=1.1)
    return rp.astype(np.int64), keys, lab.astype(np.int32)


def _agree(m, s):
    assert sorted(m.stamp.items()) == sorted(s.stamp.items())
    assert m.size() == len(s.stamp)
    keys = np.array(sorted(s.stamp), np.uint64)
    assert np.array_equal(m.last_touch(keys), np.array([s.stamp[int(k)] for k in keys], np.uint64))


def test_stamps_follow_training_predict_and_init_push():
    m, s = EvictingTable(K=0), ScalarStamps()
    m.init_push()
    s.insert([0])
    m.step(*_batch(1))  # before tracking: stamps restart when it starts
    s.train(_batch(1)[1])
    m.set_eviction()
    s.stamp = {k: s.b for k in s.stamp}
    _agree(m, s)
    for i in range(2, 6):
        rp, keys, lab = _batch(i)
        m.step(rp, keys, lab)
        s.train(keys)
        prp, pkeys, _ = _batch(100 + i, space=800)
        m.predict(prp, pkeys)
        s.insert(pkeys)
        _agree(m, s)
    m.step(np.zeros(1, np.int64), np.zeros(0, np.uint64), np.zeros(0, np.int32))  # an empty batch is not a batch
    assert m.batches == s.b
    m.push(np.array([5000, 5001], np.uint64), gw=np.zeros(2, np.float32))
    s.insert([5000, 5001])
    _agree(m, s)


def test_idle_edge():
    """A key touched exactly T batches before the sweep (stamp B - T) stays; one batch earlier goes."""
    T = 3
    m, s = EvictingTable(K=0), ScalarStamps()
    m.set_eviction(max_idle_batches=T)
    for i in range(6):
        keys = np.array([10 + i, 100], np.uint64)
        m.step(np.array([0, 2], np.int64), keys, np.array([1], np.int32))
        s.train(keys)
    assert m.batches == 6
    # the last T batches are 3, 4, 5: keys 10, 11, 12 (stamps 0-2) go; 13 (stamp 3 = B - T) stays
    assert m.evict() == s.sweep(T, 0) == 3
    assert set(m.stamp) == {13, 14, 15, 100}
    _agree(m, s)


def test_budget_ties_broken_by_key():
    m, s = EvictingTable(K=0), ScalarStamps()
    m.set_eviction(max_keys=5)
    for keys in ([7, 3, 9], [40, 20, 30, 10, 50]):  # the second batch's 5 keys share a stamp: the boundary is inside it
        keys = np.array(keys, np.uint64)
        m.step(np.array([0, keys.size], np.int64), keys, np.array([0], np.int32))
        s.train(keys)
    m.set_eviction(max_keys=3)
    assert m.evict() == s.sweep(0, 3) == 5
    assert set(m.stamp) == {10, 20, 30}
    _agree(m, s)


def test_budget_above_key_count_is_a_no_op():
    m, s = EvictingTable(K=8), ScalarStamps()
    m.set_eviction(max_keys=10 ** 6, max_idle_batches=100)
    for i in range(3):
        rp, keys, lab = _batch(i)
        m.step(rp, keys, lab)
        s.train(keys)
    before = m.export(m.keys())
    assert m.evict() == s.sweep(100, 10 ** 6) == 0
    after = m.export(m.keys())
    for f in before:
        assert np.array_equal(before[f], after[f]), f
    _agree(m, s)


def test_both_limits_and_periodic_sweeps():
    m, s = EvictingTable(K=4), ScalarStamps()
    m.set_eviction(max_idle_batches=2, max_keys=60, every=3)
    for i in range(10):
        rp, keys, lab = _batch(i)
        m.step(rp, keys, lab)
        s.train(keys)
        if s.b % 3 == 0:
            s.sweep(2, 60)
        _agree(m, s)
    assert m.sweeps == 3


def test_survivors_matches_a_sort():
    rng = np.random.default_rng(5)
    keys = rng.choice(1 << 40, 3000, replace=False).astype(np.uint64)
    stamps = rng.integers(0, 20, keys.size)
    for T, N in [(0, 0), (5, 0), (0, 100), (7, 1000), (30, 3000), (0, 2999)]:
        keep = survivors(keys, stamps, 20, T, N)
        live = sorted(zip(stamps.tolist(), keys.tolist()), key=lambda x: (-x[0], x[1]))
        if T > 0 and 20 > T:
            live = [x for x in live if x[0] >= 20 - T]
        if N > 0:
            live = live[:N]
        assert set(keys[keep].tolist()) == {k for _, k in live}, (T, N)

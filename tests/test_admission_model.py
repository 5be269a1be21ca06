"""The CPU statement of feature admission (tests/admission_model.py, the yardstick of tests/test_gpu_admission.py)
against a scalar restatement written token by token in plain Python integers: the Bloom filter's cells, saturating
counts and decay, the Poisson draw, and the extreme Poisson probabilities against the oracle without a policy."""
import numpy as np

from admission_model import ADMIT_BLOOM, ADMIT_POISSON, AdmittingTable
from oracle import oracle as O
from xflow_b200 import datagen

M64 = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15


def splitmix64(x):
    x = (x + GOLD) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


class ScalarBloom:
    """One token at a time, one saturating increment at a time."""

    def __init__(self, n, L, h, D, seed):
        self.n, self.L, self.h, self.D, self.seed = n, L, h, D, seed
        self.cells = [0] * (1 << L)
        self.b = 0
        self.present = set()
        self.rejected = self.admitted = 0

    def cell(self, key, j):
        return splitmix64(key ^ splitmix64((self.seed + (j + 1) * GOLD) & M64)) >> (64 - self.L)

    def batch(self, keys):
        keys = [int(k) for k in keys]
        decided = {}
        for k in keys:
            if k not in self.present and k not in decided:
                decided[k] = min(self.cells[self.cell(k, j)] for j in range(self.h)) >= self.n
        for k, ok in decided.items():
            if ok:
                self.present.add(k)
                self.admitted += 1
        for k in keys:
            if decided.get(k) is False:
                self.rejected += 1
                for j in range(self.h):
                    c = self.cell(k, j)
                    self.cells[c] = min(255, self.cells[c] + 1)
        if self.D and (self.b + 1) % self.D == 0:
            self.cells = [c >> 1 for c in self.cells]
        self.b += 1


def _batches(n, B=128, d=12, space=2000):
    return [datagen.make_csr_keys(40 + s, B, d, space, O.hash_decimal_ids, dist="zipf", zipf_s=1.1) for s in range(n)]


def test_bloom_filter_matches_scalar_restatement():
    """Tiny filter (2^10 cells: false positives and saturation matter), 3 hashes, decay every 2 batches; the tokens
    of each batch shuffled for the scalar restatement, whose result therefore must not depend on token order."""
    for policy_seed in (5, 6):
        t = AdmittingTable()
        t.set_admission(ADMIT_BLOOM, threshold=2, log2_cells=10, hashes=3, decay_batches=2, seed=policy_seed)
        ref = ScalarBloom(2, 10, 3, 2, policy_seed)
        rng = np.random.default_rng(policy_seed)
        for rp, keys, lab in _batches(6):
            t.step(rp.astype(np.int64), keys, lab.astype(np.int32))
            ref.batch(keys[rng.permutation(keys.size)])
            assert np.array_equal(t.admission_filter(), np.array(ref.cells, np.uint8))
            assert t.admission_stats() == dict(batches=ref.b, rejected_tokens=ref.rejected, admitted_keys=ref.admitted)
            assert t.size() == len(ref.present)
        assert max(ref.cells) > 0 and ref.rejected > 0 and ref.admitted > 0


def test_bloom_filter_saturates_at_255():
    t = AdmittingTable()
    t.set_admission(ADMIT_BLOOM, threshold=255, log2_cells=10, hashes=2, seed=1)
    ref = ScalarBloom(255, 10, 2, 0, 1)
    rp = np.arange(0, 301, dtype=np.int64)
    keys = np.full(300, 12345, np.uint64)  # one key, 300 occurrences per batch
    for _ in range(2):
        t.step(rp, keys, np.zeros(300, np.int32))
        ref.batch(keys)
    f = t.admission_filter()
    assert np.array_equal(f, np.array(ref.cells, np.uint8)) and f.max() == 255
    assert t.size() == 1  # admitted in the second batch


def test_poisson_extremes():
    """p = 1 equals the oracle without a policy (every table field, every batch); p = 0 inserts nothing and predicts
    sigmoid(0); predict with a policy does not insert."""
    for K in (0, 4):
        a = O.Table(K=K, init_mode=O.INIT_COUNTER, seed=2)
        b, z = (AdmittingTable(K=K, init_mode=O.INIT_COUNTER, seed=2) for _ in range(2))
        b.set_admission(ADMIT_POISSON, probability=1.0, seed=9)
        z.set_admission(ADMIT_POISSON, probability=0.0, seed=9)
        all_keys = []
        for rp, keys, lab in _batches(4):
            ua, la = a.step(rp.astype(np.int64), keys, lab.astype(np.int32))
            ub, lb = b.step(rp.astype(np.int64), keys, lab.astype(np.int32))
            z.step(rp.astype(np.int64), keys, lab.astype(np.int32))
            assert ua == ub and np.array_equal(la.view(np.uint32), lb.view(np.uint32))
            all_keys.append(keys)
        uk = np.unique(np.concatenate(all_keys))
        ea, eb = a.export(uk), b.export(uk)
        for k in ea:
            assert np.array_equal(ea[k], eb[k]), k
        # every key of a trained batch is present: the same prediction
        rp, keys, _ = _batches(4)[-1]
        assert np.array_equal(b.predict(rp.astype(np.int64), keys), a.predict(rp.astype(np.int64), keys))
        rp, keys, _ = datagen.make_csr_keys(99, 128, 12, 2000, O.hash_decimal_ids)
        size = b.size()
        b.predict(rp.astype(np.int64), keys)
        assert b.size() == size
        assert z.size() == 0 and z.admission_stats()["rejected_tokens"] == sum(k.size for k in all_keys)
        assert np.all(z.predict(rp.astype(np.int64), keys) == np.float32(O.sigmoid(0.0)))
        assert z.size() == 0


def test_poisson_decision_is_per_key_and_batch():
    """u24(key, b) < floor(p 2^24), restated with plain integers; the admitted share follows p."""
    t = AdmittingTable()
    t.set_admission(ADMIT_POISSON, probability=0.3, seed=4)
    rp, keys, lab = datagen.make_csr_keys(7, 512, 16, 10 ** 7, O.hash_decimal_ids)
    t.step(rp.astype(np.int64), keys, lab.astype(np.int32))
    uk = np.unique(keys)
    p24 = int(np.floor(float(np.float32(0.3)) * 2.0 ** 24))
    want = np.array([(splitmix64(int(k) ^ splitmix64(4 + 0)) >> 40) < p24 for k in uk])  # batch b = 0
    assert np.array_equal(t.export(uk)["present"].astype(bool), want)
    assert abs(want.mean() - 0.3) < 0.03

"""CPU checks of the importance-weighting model (tests/weighting_model.py): with weights of 1 it is the oracle's step,
its negative-sampling decision is the one include/xflow_b200.h states token by token, and the lazy step's fixed-point
unit chosen from W = sum ceil(e_r) * tokens_r keeps every key's weighted residual sum inside its 48-bit field."""
import numpy as np
import pytest

from oracle import oracle as O
from test_lazy_fixed_point_model import field_sum, fix_of, wrap48
from weighting_model import (WeightingTable, fix_bound, fix_shift, kept_negatives, p24_of, row_hash_sums,
                             row_weights, weighted_gradients)
from xflow_b200 import datagen

M64 = (1 << 64) - 1


def _splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def _batch(seed, B=600, d=12, space=4000, ragged=True):
    return datagen.make_csr_keys(seed, B, d, space, O.hash_decimal_ids, dist="zipf", zipf_s=1.2, ragged=ragged)


@pytest.mark.parametrize("K", [0, 8, 10])
@pytest.mark.parametrize("opt", [O.OPT_FTRL, O.OPT_SGD])
def test_weights_of_one_are_the_oracle_step(K, opt):
    # the model's weighted path, forced on at weights of 1, against the oracle's own step in its exact_sums arithmetic
    a = WeightingTable(always_weighted=True, K=K, opt=opt, init_mode=O.INIT_COUNTER, seed=3)
    b = O.Table(K=K, opt=opt, init_mode=O.INIT_COUNTER, seed=3)
    seen = []
    for s in range(3):
        rp, keys, lab = _batch(10 + s)
        rp, lab = rp.astype(np.int64), lab.astype(np.int32)
        _, la, mal = a.step(rp, keys, lab, np.ones(lab.size, np.float32))
        with O.exact_sums():
            _, lb = b.step(rp, keys, lab)
        assert np.array_equal(la.view(np.uint32), lb.view(np.uint32))
        assert mal == pytest.approx(float(np.abs(lb.astype(np.float64)).mean()), rel=1e-12)
        seen.append(keys)
    uk = np.unique(np.concatenate(seen))
    ea, eb = a.export(uk), b.export(uk)
    for f in ea:
        assert np.array_equal(np.asarray(ea[f]).view(np.uint8), np.asarray(eb[f]).view(np.uint8)), f


def test_weighted_gradient_with_weights_of_one_is_the_exact_oracle_gradient():
    # the general path of the model (float64 sums of the weighted residuals) against the oracle's own exact_sums
    # arithmetic on the same pulled values, bit for bit
    for K in (0, 8, 10):
        t = O.Table(K=K, init_mode=O.INIT_COUNTER, seed=1)
        rp, keys, lab = _batch(5, B=300)
        rp, lab = rp.astype(np.int64), lab.astype(np.int32)
        t.step(rp, keys, lab)  # non-zero state
        with O.exact_sums():
            uk, gw_o, gv_o, res = t.worker_compute(rp, keys, lab)
        w, v = t.pull(uk)
        uk2, gw, gv, lw = weighted_gradients(K, rp, keys, np.ones(lab.size, np.float32), res, w, v, lab.size)
        assert np.array_equal(uk, uk2) and np.array_equal(lw, res)
        assert np.array_equal(gw.view(np.uint32), gw_o.view(np.uint32))
        assert np.array_equal(gv.view(np.uint32), gv_o.view(np.uint32))


def test_sampling_decision_matches_a_token_by_token_statement():
    rng = np.random.default_rng(4)
    for trial in range(6):
        rp, keys, lab = _batch(40 + trial, B=400, ragged=True)
        rp = rp.astype(np.int64)
        rp[5] = rp[4]  # an empty row somewhere (its successors keep their tokens)
        rate = float(rng.choice([0.5, 0.1, 0.013, 2.0 ** -24, 1.0 - 2.0 ** -20]))
        seed = int(rng.integers(0, 2 ** 63))
        got = kept_negatives(rp, keys, rate, seed)
        p24 = p24_of(rate)
        F = row_hash_sums(rp, keys)
        for r in range(lab.size):
            f = 0
            for j in range(rp[r], rp[r + 1]):
                f = (f + _splitmix64(int(keys[j]))) & M64
            assert int(F[r]) == f
            assert bool(got[r]) == ((_splitmix64(seed ^ f) >> 40) < p24), (trial, r)
        # order of the tokens does not matter; equal key multisets decide alike
        perm = np.concatenate([rng.permutation(np.arange(rp[r], rp[r + 1])) for r in range(lab.size)]).astype(np.int64)
        assert np.array_equal(kept_negatives(rp, keys[perm], rate, seed), got)
        e = row_weights(rp, keys, lab, None, rate, seed)
        inv = np.float32(1.0 / np.float64(np.float32(rate)))
        assert np.all(e[lab != 0] == 1)
        assert np.array_equal(e[lab == 0], np.where(got[lab == 0], inv, np.float32(0)))
    # about rate of the negatives are kept
    rp, keys, lab = _batch(99, B=20000, ragged=False)
    kept = kept_negatives(rp.astype(np.int64), keys, 0.1, 7)
    assert abs(kept.mean() - 0.1) < 0.01


def test_caller_weights_multiply_the_policy():
    rp, keys, lab = _batch(3, B=200)
    rp = rp.astype(np.int64)
    c = np.random.default_rng(0).uniform(0, 8, lab.size).astype(np.float32)
    e = row_weights(rp, keys, lab, c, 0.25, 11)
    s = row_weights(rp, keys, lab, None, 0.25, 11)
    assert np.array_equal(e, (c * s).astype(np.float32))
    assert fix_bound(rp, np.ones(lab.size, np.float32)) == int(rp[-1])  # weights 1: W = nnz, the unweighted unit


@pytest.mark.parametrize("weight", [1.0, 1.5, 4.0, 8.0, 1000.0, 2.0 ** 20])
def test_unit_from_W_keeps_every_sum_inside_the_field(weight):
    # the largest sum a batch can make on one key: every token of every trained row on it, |residual| = 1, at the
    # row's weight.  W replaces nnz in the bound of tests/test_lazy_fixed_point_model.py.
    for k in range(0, 33):
        for tokens in {max(1, (1 << k) - 1), 1 << k, (1 << k) + 1}:
            if tokens >= 1 << 32:
                continue
            e = np.float32(weight)
            W = int(np.ceil(np.float64(e))) * tokens
            s = fix_shift(W)
            per = fix_of(np.float32(np.float32(e) * np.float32(1.0)), s)
            exact = tokens * per
            if W <= 2 ** 47 - 1:
                assert wrap48(exact) == exact, (weight, tokens, s)
            else:
                assert s == 0  # outside the step's range: documented, not exact
    # mixed weights, random residuals: the field sum equals the exact integer sum
    rng = np.random.default_rng(1)
    for _ in range(30):
        n = int(rng.integers(1, 4000))
        e = rng.uniform(0, 8, n).astype(np.float32)
        r = rng.uniform(-1, 1, n).astype(np.float32)
        wl = (e * r).astype(np.float32)
        W = int(np.sum(np.ceil(e.astype(np.float64))))
        s = fix_shift(W)
        fixes = np.rint(wl.astype(np.float64) * 2.0 ** s).astype(np.int64)
        assert field_sum(wl, s) == int(fixes.sum())
        assert abs(int(fixes.sum())) <= W * 2 ** s


def test_skipped_rows_change_nothing_in_the_model():
    t = WeightingTable(K=0)
    rp, keys, lab = _batch(8, B=100)
    rp, lab = rp.astype(np.int64), lab.astype(np.int32)
    wts = np.ones(lab.size, np.float32)
    wts[::2] = 0
    _, res, mal = t.step(rp, keys, lab, wts)
    assert np.all(res[::2] == 0) and np.all(res[1::2] != 0)
    only_skipped = np.setdiff1d(np.concatenate([keys[rp[r]:rp[r + 1]] for r in range(0, lab.size, 2)]),
                                np.concatenate([keys[rp[r]:rp[r + 1]] for r in range(1, lab.size, 2)]))
    assert only_skipped.size > 0
    assert not t.export(only_skipped)["present"].any()
    assert t.skipped == lab.size // 2
    assert mal == pytest.approx(float(np.abs(res[1::2].astype(np.float64)).sum() / lab.size))

"""tests/lr_ledger.py on the CPU: its optimizer arithmetic is the oracle's bit for bit, its fixed-point sums stay within
the quantisation bound of the oracle's exact-sum step, its residual intervals hold the oracle's residuals, and it
tells a wrong deposit apart from a right one."""
import numpy as np
import pytest

import lr_ledger as L
from oracle import oracle as O
from xflow_b200 import datagen

OPTS = {"ftrl": O.OPT_FTRL, "sgd": O.OPT_SGD}


def _states(rng, n):
    """Random FTRL states: n >= 0 over many scales, z of both signs, some exactly at and next to the L1 threshold,
    and a few of zero."""
    nw = (10.0 ** rng.uniform(-12, 2, n)).astype(np.float32)
    nw[::11] = 0.0
    zw = (rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 0, n)).astype(np.float32)
    l1 = np.float32(L.L1)
    zw[1::13] = l1
    zw[2::13] = -l1
    zw[3::13] = np.nextafter(l1, np.float32(1))
    zw[4::13] = np.nextafter(-l1, np.float32(-1))
    zw[5::13] = 0.0
    return nw, zw


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("imported", [False, True], ids=["w=f(z,n)", "imported-w"])
def test_coordinate_step_equals_oracle_push(opt, imported):
    """The ledger's float32 FTRL / SGD coordinate equals the oracle's push handle bit for bit: random states, gradients
    of both signs and zero, states at the L1 threshold, and weights imported from outside that are not f(z, n)."""
    rng = np.random.default_rng(5 + imported)
    n = 4000
    keys = np.arange(1, n + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    nw, zw = _states(rng, n)
    if imported or opt == "sgd":
        w = (rng.standard_normal(n) * 10.0 ** rng.uniform(-5, 0, n)).astype(np.float32)
        w[::17] = 0.0
    else:
        w = L.ftrl_w(zw, nw)
    if opt == "sgd":
        nw = zw = np.zeros(n, np.float32)
    g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-9, 0, n)).astype(np.float32)
    g[::7] = 0.0
    g[1::7] = -g[1::7]
    ot = O.Table(K=0, opt=OPTS[opt])
    ot.import_(keys, w=w, nw=nw, zw=zw)
    if imported and opt == "ftrl":
        assert np.mean(w != L.ftrl_w(zw, nw)) > 0.9
    ot.push(keys, gw=g)
    want = ot.export(keys)
    got = L.apply_step(dict(w=w, nw=nw, zw=zw), g, np.ones(n, bool), opt)
    for f in ("w", "nw", "zw"):
        assert np.array_equal(got[f].view(np.uint32), want[f].view(np.uint32)), f
    # and a second step from there, where w = f(z, n) again
    ot.push(keys, gw=-g)
    got2 = L.apply_step(got, -g, np.ones(n, bool), opt)
    want2 = ot.export(keys)
    for f in ("w", "nw", "zw"):
        assert np.array_equal(got2[f].view(np.uint32), want2[f].view(np.uint32)), f


def _oracle_batches(seed, B=512, d=24, space=4000):
    h = O.hash_decimal_ids
    return [datagen.make_csr_keys(seed, B, d, space, h),
            datagen.make_csr_keys(seed + 1, B // 2, d, space, h, dist="zipf", zipf_s=1.1),
            datagen.make_csr_keys(seed + 2, B, d, space, h, ragged=True),
            datagen.make_csr_keys(seed + 3, B, 2 * d, space, h, dist="zipf", zipf_s=1.3, ragged=True)]


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
def test_fixed_point_sums_match_exact_sum_steps_within_the_bound(opt):
    """With s = 27 the ledger's fold on the oracle's residuals stays within count * 2^-s / 2 (over the row count) of the
    oracle's exact-sum gradient, and the ledger's optimizer step with that exact gradient is the oracle's post-step
    state bit for bit: the claim of test_quantised_sums_match_eager_steps_within_the_bound, through the ledger."""
    xt = O.Table(K=0, opt=OPTS[opt])
    for rp, keys, lab in _oracle_batches(3):
        B = lab.size
        uk, cnt = np.unique(keys, return_counts=True)
        pre = xt.export(uk)
        with O.exact_sums():
            _, res = xt.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        post = xt.export(uk)
        led = L.ledger_step(pre, rp, keys, res, B, opt)
        assert led.s == 27 and led.trained.all()
        exact = np.zeros(uk.size)
        row_of = np.repeat(np.arange(B), np.diff(rp.astype(np.int64)))
        np.add.at(exact, np.searchsorted(uk, keys), res[row_of].astype(np.float64))
        g_exact = (exact.astype(np.float32).astype(np.float64) / B).astype(np.float32)
        want = L.apply_step(pre, g_exact, led.trained, opt)
        for f in ("w", "nw", "zw"):
            assert np.array_equal(want[f].view(np.uint32), post[f].view(np.uint32)), f
        unit = 2.0 ** -led.s
        assert np.all(np.abs(led.sums * unit - exact) <= cnt * unit / 2 * (1 + 1e-12))
        tol = cnt * unit / 2 / B + 2 * np.spacing(np.abs(g_exact)).astype(np.float64) + 1e-45
        assert np.all(np.abs(led.g.astype(np.float64) - g_exact) <= tol)


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
def test_oracle_residuals_lie_inside_the_residual_bounds(opt):
    """Over several steps of uniform, Zipf and ragged batches, every residual of the oracle lies in residual_bounds from
    the oracle's own pre-step state, and the intervals are narrow."""
    ot = O.Table(K=0, opt=OPTS[opt])
    for step, (rp, keys, lab) in enumerate(_oracle_batches(7) * 2):
        uk = np.unique(keys)
        pre = ot.export(uk)
        _, res = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        lo, hi = L.residual_bounds(pre["w"][np.searchsorted(uk, keys)], rp, keys, lab)
        r = res.astype(np.float64)
        assert np.all((r >= lo) & (r <= hi)), step
        assert np.all(hi - lo <= 1e-5)
        if step >= 4:
            assert np.any(hi - lo > 0)   # the weights are no longer all zero


def _dup_batch(seed):
    """Rows with a key repeated inside one warp chunk (for group_count_1) and in rows of both labels."""
    rng = np.random.default_rng(seed)
    rp, keys, lab = datagen.make_csr_keys(seed, 256, 40, 2000, O.hash_decimal_ids)
    keys = keys.copy()
    keys[rp[5] + 3] = keys[rp[5] + 9]
    return rp, keys, lab, rng


@pytest.mark.parametrize("perturb", L.PERTURBATIONS)
@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
def test_ledger_tells_wrong_deposits_apart(perturb, opt):
    """One token dropped or doubled, a warp group's count taken as 1, the unit off by one bit, or the divisor off by one
    row: each changes at least one key's post-step bits, on a state that earlier steps made nonzero."""
    ot = O.Table(K=0, opt=OPTS[opt])
    for rp, keys, lab in _oracle_batches(11)[:2]:
        ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
    rp, keys, lab, _ = _dup_batch(13)
    uk = np.unique(keys)
    pre = ot.export(uk)
    _, res = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
    right = L.ledger_step(pre, rp, keys, res, lab.size, opt)
    wrong = L.ledger_step(pre, rp, keys, res, lab.size, opt, perturb=perturb)
    differs = np.zeros(uk.size, bool)
    for f in ("w", "nw", "zw"):
        differs |= right[f].view(np.uint32) != wrong[f].view(np.uint32)
    assert differs.any(), perturb


def test_weights_and_rejections_enter_the_ledger():
    """Rows of weight 0 deposit nothing and a key only they hold takes no step; a fractional or larger weight scales
    the deposit and sets the unit from W; a rejected token deposits nothing."""
    rp = np.array([0, 2, 4, 5], np.int64)
    keys = np.array([10, 11, 10, 12, 13], np.uint64)
    res = np.array([0.25, -0.75, 0.5], np.float32)
    uk = np.unique(keys)
    pre = dict(keys=uk, w=np.zeros(4, np.float32), nw=np.zeros(4, np.float32), zw=np.zeros(4, np.float32))
    e = np.array([1.5, 0.0, 3.0], np.float32)
    led = L.ledger_step(pre, rp, keys, res, 3, "sgd", e=e)
    assert led.s == L.fix_shift(2 * 2 + 3 * 1)
    assert list(led.trained) == [True, True, False, True]
    u = 2 ** led.s
    assert list(led.sums) == [int(0.375 * u), int(0.375 * u), 0, int(1.5 * u)]
    keep = np.array([True, False, True, True, True])
    led = L.ledger_step(pre, rp, keys, res, 3, "sgd", keep=keep)
    assert list(led.trained) == [True, False, True, True] and led.s == 27
    assert list(led.sums) == [int((0.25 - 0.75) * 2 ** 27), 0, int(-0.75 * 2 ** 27), int(0.5 * 2 ** 27)]

"""CPU checks of progressive validation's model (tests/validation_model.py): the binning rule of
include/xflow_b200.h section 8 orders the bins as the predictions, and the report's [auc_lo, auc_hi] brackets the
exact weighted AUC of the raw floats, closing on it when every distinct prediction has a bin of its own."""
import math
from fractions import Fraction

import numpy as np
import pytest

import validation_model as V


@pytest.mark.parametrize("m", [4, 10, 16])
def test_bins_follow_the_order_of_p(m):
    assert V.bin_of(2.0 ** -20, m) == 0 and V.bin_of(1.0, m) == V.nbins(m) - 1
    # clamped: anything below 2^-20 (zero, negatives, -inf) and above 1 (+inf) share the end bins
    for p in (0.0, -0.0, -3.0, -math.inf, 1e-30, 2.0 ** -21):
        assert V.bin_of(p, m) == 0
    for p in (1.5, 7.0, math.inf):
        assert V.bin_of(p, m) == V.nbins(m) - 1
    rng = np.random.default_rng(m)
    p = np.sort(np.concatenate([rng.random(2000, dtype=np.float32), np.float32(2.0) ** -rng.integers(0, 21, 200)]))
    b = [V.bin_of(x, m) for x in p.tolist()]
    assert all(b0 <= b1 for b0, b1 in zip(b, b[1:]))
    assert max(b) < V.nbins(m)
    # a bin is 2^(23 - m) consecutive floats: the first float of a bin starts it
    edge = np.array([V.bits(0.25) >> (23 - m) << (23 - m)], np.uint32).view(np.float32)[0]
    below = np.nextafter(edge, np.float32(0))
    assert V.bin_of(edge, m) == V.bin_of(below, m) + 1


def test_fixed_point_units_round_to_nearest_even():
    assert V.units(1.0) == 2 ** 32
    assert V.units(2.0 ** -30) == 4
    assert V.units(2.0 ** 24) == 2 ** 56
    assert V.units(2.0 ** -33) == 0          # half a unit: to even
    assert V.units(3 * 2.0 ** -33) == 2      # one and a half: to even
    assert V.units(2.0 ** -40) == 0


def test_report_formulas_on_a_small_stream():
    pv = V.Pv(4).add([0.25, 0.25, 0.75, np.nan, 0.5, 0.5], [1, 0, 1, 1, 0, 1], [1.0, 2.0, 0.5, 1.0, 0.0, np.inf])
    r = pv.exact()
    assert (r["rows"], r["positives"], r["negatives"], r["nan_rows"], r["overflow_rows"]) == (3, 2, 1, 1, 1)
    assert r["weight_pos"] == Fraction(3, 2) and r["weight_neg"] == 2
    assert r["ctr"] == Fraction(3, 7)
    assert r["mean_pctr"] == (Fraction(1, 4) + 2 * Fraction(1, 4) + Fraction(3, 8)) / Fraction(7, 2)
    # the negative (0.25, weight 2) ties the positive of weight 1 and lies below the one of weight 1/2
    assert r["auc_lo"] == Fraction(2 * Fraction(1, 2), Fraction(3, 2) * 2)
    assert r["auc_hi"] == Fraction(2 * Fraction(3, 2), Fraction(3, 2) * 2) == 1
    want_ll = (V.units(-math.log(0.25)) + V.units(2.0 * -math.log(0.75)) + V.units(0.5 * -math.log(0.75)))
    assert r["logloss"] == Fraction(want_ll, 7 * 2 ** 31)
    rep = pv.report()
    assert rep["auc"] == 2 / 3 and rep["ctr"] == 3 / 7
    # one class empty: the AUC is NaN, the rest is defined
    rep = V.Pv(10).add([0.1, 0.2], [0, 0]).report()
    assert math.isnan(rep["auc"]) and math.isnan(rep["auc_lo"]) and rep["ctr"] == 0.0
    rep = V.Pv(10).report()
    assert rep["rows"] == 0 and math.isnan(rep["logloss"]) and math.isnan(rep["auc"])


def _stream(rng, n, levels):
    """Predictions with many exact ties and near-ties (neighbouring floats), weights with zeros and wide ranges."""
    base = rng.random(levels).astype(np.float32) * np.float32(0.3)
    p = base[rng.integers(0, levels, n)]
    near = rng.random(n) < 0.3
    p[near] = np.nextafter(p[near], np.float32(1))
    y = (rng.random(n) < 0.35).astype(np.uint8)
    w = rng.choice(np.array([0.0, 2.0 ** -30, 0.5, 1.0, 3.0, 10.0, 2.0 ** 24], np.float32), n)
    return p, y, w


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("m", [4, 10])
def test_exact_auc_lies_in_the_bracket(seed, m):
    rng = np.random.default_rng(seed)
    p, y, w = _stream(rng, 300, 12)
    pv = V.Pv(m).add(p, y, w)
    r = pv.exact()
    exact = V.exact_auc(p, y, w)
    assert exact is not None
    assert r["auc_lo"] <= exact <= r["auc_hi"]
    # unweighted too
    r = V.Pv(m).add(p, y).exact()
    exact = V.exact_auc(p, y)
    assert r["auc_lo"] <= exact <= r["auc_hi"]


@pytest.mark.parametrize("seed", range(4))
def test_one_prediction_per_bin_closes_the_bracket(seed):
    """Distinct predictions in distinct bins: the bins' order is the floats' order, ties are exact ties."""
    m = 8
    rng = np.random.default_rng(100 + seed)
    starts = rng.choice(V.nbins(m) - 1, 40, replace=False)
    # the first float of each chosen bin
    first = (np.uint32(V.bits(2.0 ** -20)) >> np.uint32(23 - m)) + starts.astype(np.uint32)
    levels = (first << np.uint32(23 - m)).view(np.float32)
    assert len({V.bin_of(x, m) for x in levels.tolist()}) == levels.size
    p = levels[rng.integers(0, levels.size, 400)]
    y = (rng.random(400) < 0.5).astype(np.uint8)
    w = rng.choice(np.array([0.0, 0.25, 1.0, 7.0], np.float32), 400)
    r = V.Pv(m).add(p, y, w).exact()
    exact = V.exact_auc(p, y, w)
    assert r["auc_lo"] < r["auc_hi"]  # ties exist: the bracket is their half
    assert r["auc"] == exact

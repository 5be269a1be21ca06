"""CPU checks of tests/group_metric_model.py, the statement of the grouped test metric (include/xflow_b200.h section
9): U2 against pair counting, AUC against scipy's Mann-Whitney U, logloss against the progressive-validation model,
and invariance under permutation and re-cutting."""
import math

import numpy as np
import pytest
from scipy.stats import mannwhitneyu

import group_metric_model as G
import validation_model as V

SPECIAL = np.array([0.0, -0.0, np.inf, -np.inf, 0.5, 0.25, 1.0, 1e-20, 1.0 - 2 ** -24, 0.75], np.float32)


def _rows(seed, n, n_groups, levels=None):
    rng = np.random.default_rng(seed)
    p = rng.random(n).astype(np.float32)
    if levels is not None:
        p = levels[rng.integers(0, levels.size, n)]
    y = rng.choice(np.array([0, 1, 2, 255], np.uint8), n, p=[0.55, 0.35, 0.05, 0.05])
    g = rng.integers(0, n_groups, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)  # ids across all 64 bits
    return p, y, g


@pytest.mark.parametrize("seed", range(6))
def test_u2_counts_pairs_in_small_groups_full_of_ties(seed):
    p, y, g = _rows(seed, 400, 12, SPECIAL)
    p[:5] = np.nan
    rep, per = G.evaluate(p, y, g)
    keep = ~np.isnan(p)
    assert rep["nan_rows"] == 5 and rep["rows"] == int(keep.sum())
    assert per["ids"].tolist() == sorted(set(g[keep].tolist()))
    for k, gid in enumerate(per["ids"].tolist()):
        sel = keep & (g == np.uint64(gid))
        assert int(per["u2"][k]) == G.u2_pairs(p[sel], y[sel] != 0)
        assert int(per["rows"][k]) == int(sel.sum()) and int(per["positives"][k]) == int((y[sel] != 0).sum())


def test_negative_zero_ties_with_positive_zero():
    # one positive at -0.0 and one negative at +0.0: a tie, U2 = 1
    rep, per = G.evaluate(np.array([-0.0, 0.0], np.float32), np.array([1, 0], np.uint8), np.zeros(2, np.uint64))
    assert per["u2"].tolist() == [1] and per["auc"][0] == 0.5
    rep, per = G.evaluate(np.array([np.inf, np.inf, -np.inf], np.float32), np.array([1, 0, 0], np.uint8),
                          np.zeros(3, np.uint64))
    assert per["u2"].tolist() == [3]   # the tie at +Inf counts 1, the win over -Inf counts 2


@pytest.mark.parametrize("seed", range(4))
def test_auc_is_scipys_mann_whitney_u(seed):
    p, y, g = _rows(100 + seed, 3000, 7, np.round(np.linspace(0, 1, 16), 3).astype(np.float32))
    p[::97] = np.random.default_rng(seed).random(p[::97].size).astype(np.float32)
    rep, per = G.evaluate(p, y, g)
    for k, gid in enumerate(per["ids"].tolist()):
        sel = g == np.uint64(gid)
        pos, neg = p[sel & (y != 0)].astype(np.float64), p[sel & (y == 0)].astype(np.float64)
        u = mannwhitneyu(pos, neg, alternative="two-sided", method="asymptotic").statistic
        assert 2 * u == int(per["u2"][k])
        assert per["auc"][k] == int(per["u2"][k]) / ((2.0 * pos.size) * neg.size)
        assert abs(per["auc"][k] - u / (pos.size * neg.size)) <= 1e-15


def test_report_definitions():
    p, y, g = _rows(7, 5000, 40, SPECIAL)
    g[:50] = np.uint64(2 ** 64 - 1)
    y[g == g[60]] = 1                       # one all-positive group
    rep, per = G.evaluate(p, y, g)
    scored = ~np.isnan(per["auc"])
    assert rep["groups"] == per["ids"].size and rep["scored_groups"] == int(scored.sum()) < rep["groups"]
    assert rep["scored_rows"] == int(per["rows"][scored].sum())
    assert per["ids"][-1] == np.uint64(2 ** 64 - 1)
    t = sum(round((float(r) * a) * G.UNIT) for r, a in zip(per["rows"][scored].tolist(), per["auc"][scored].tolist()))
    assert abs(rep["gauc"] - t / G.UNIT / rep["scored_rows"]) <= 1e-15
    assert abs(rep["gauc"] - float(np.average(per["auc"][scored], weights=per["rows"][scored]))) <= 1e-9
    assert abs(rep["gauc_mean"] - float(np.mean(per["auc"][scored]))) <= 1e-9
    for k in range(per["ids"].size):
        assert per["logloss"][k] == float(int(per["s"][k])) / (float(per["rows"][k]) * G.UNIT)
    # the logloss is the unweighted pv's, to the bit (both are one correctly rounded ratio of the same integers)
    assert rep["logloss"] == V.Pv(4).add(p, y).report()["logloss"]


def test_empty_and_nan_only():
    for p in (np.zeros(0, np.float32), np.full(3, np.nan, np.float32)):
        rep, per = G.evaluate(p, np.zeros(p.size, np.uint8), np.arange(p.size, dtype=np.uint64))
        assert rep["rows"] == rep["groups"] == rep["scored_groups"] == 0 and rep["nan_rows"] == p.size
        assert all(math.isnan(rep[k]) for k in ("logloss", "gauc", "gauc_mean")) and per["ids"].size == 0


def test_permuting_and_recutting_leave_the_output_unchanged():
    p, y, g = _rows(11, 20000, 300, SPECIAL)
    p[::113] = np.nan
    want = G.GroupMetric().add(p, y, g).finish()
    rng = np.random.default_rng(12)
    perm = rng.permutation(p.size)
    m = G.GroupMetric()
    cuts = [0, 1, 17, 5000, 5001, 13000, p.size]
    for a, b in zip(cuts, cuts[1:]):
        m.add(p[perm[a:b]], y[perm[a:b]], g[perm[a:b]])
    got = m.finish()
    assert got[0] == want[0] or all(got[0][k] == want[0][k] or (got[0][k] != got[0][k] and want[0][k] != want[0][k])
                                    for k in want[0])
    for k in want[1]:
        assert np.array_equal(got[1][k], want[1][k], equal_nan=k in ("auc", "logloss")), k

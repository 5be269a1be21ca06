"""CPU checks of tests/group_topk_model.py, the statement of the grouped metric's ranking quality at a cutoff (include/
xflow_b200.h section 9): H and G against the average over every order of every tie run, the textbook NDCG@k,
precision@k and recall@k with distinct scores, invariance under permutation and re-cutting, the edges, and the
library's discount table against the 50-digit one."""
import itertools
import math
from fractions import Fraction

import numpy as np
import pytest

import group_metric_model as GM
import group_topk_model as T

LEVELS = np.array([0.9, 0.8, 0.8, 0.5, 0.5, 0.5, 0.2, -0.0, 0.0], np.float32)


def _rows(seed, n, n_groups, levels=None):
    rng = np.random.default_rng(seed)
    p = rng.random(n).astype(np.float32) if levels is None else levels[rng.integers(0, levels.size, n)]
    y = rng.choice(np.array([0, 1, 2, 255], np.uint8), n, p=[0.55, 0.35, 0.05, 0.05])
    g = rng.integers(0, n_groups, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    return p, y, g


def _brute(p, y, k, D):
    """Exact expected hits and DCG (in units, with the integer discounts) over every order inside every tie run of one
    group: (E[hits], E[DCG], runs that round)."""
    order = np.argsort(-p, kind="stable")
    p, y = p[order], (y[order] != 0).astype(int)
    runs = [list(y[p == v]) for v in sorted(set(p.tolist()), reverse=True)]
    hits = dcg = Fraction(0)
    count = 0
    for combo in itertools.product(*[list(itertools.permutations(r)) for r in runs]):
        labels = [v for r in combo for v in r]
        hits += sum(labels[:k])
        dcg += sum(D[i + 1] - D[i] for i, v in enumerate(labels[:k]) if v)
        count += 1
    rounding = 0
    a = 0
    for r in runs:
        o = min(max(k - a, 0), len(r))
        rounding += 1 if (0 < o and sum(r) and len(r) > 1) else 0
        a += len(r)
    return hits / count, dcg / count, rounding


@pytest.mark.parametrize("seed", range(4))
def test_h_and_g_are_the_average_over_every_order_of_every_tie_run(seed):
    D = T.cumulative(16)
    p, y, g = _rows(seed, 90, 12, LEVELS)   # about 7 rows a group in runs of up to 4
    for k in (1, 2, 3, 5, 8, 16):
        rep, per = T.evaluate(p, y, g, k)
        for j, gid in enumerate(per["ids"].tolist()):
            sel = g == np.uint64(gid)
            gp, gy = np.where(p[sel] == 0, np.float32(0), p[sel]), y[sel]
            hits, dcg, rounding = _brute(gp, gy, k, D)
            H, G = int(per["H"][j]), int(per["G"][j])
            if rounding == 0:
                assert H == hits * T.UNIT and G == dcg
            assert abs(H - hits * T.UNIT) <= Fraction(rounding, 2)
            assert abs(G - dcg) <= Fraction(rounding, 2)
            # exact when no run straddles k: every run is wholly in or wholly out of the top k
            a, straddles = 0, False
            for v in sorted(set(gp.tolist()), reverse=True):
                c = int((gp == v).sum())
                straddles |= a < k < a + c
                a += c
            if not straddles:
                assert H == hits * T.UNIT


@pytest.mark.parametrize("k", [1, 3, 10, 100])
def test_distinct_scores_give_the_textbook_formulas(k):
    rng = np.random.default_rng(k)
    n = 4000
    p = rng.permutation(np.linspace(0.001, 0.999, n).astype(np.float32))
    assert np.unique(p).size == n
    y = (rng.random(n) < 0.3).astype(np.uint8)
    g = rng.integers(0, 60, n).astype(np.uint64)
    rep, per = T.evaluate(p, y, g, k)
    for j, gid in enumerate(per["ids"].tolist()):
        sel = g == np.uint64(gid)
        ys = (y[sel][np.argsort(-p[sel])] != 0).astype(float)
        P = int(ys.sum())
        if P == 0:
            assert math.isnan(per["ndcg"][j]) and math.isnan(per["precision"][j]) and math.isnan(per["recall"][j])
            continue
        disc = 1.0 / np.log2(np.arange(2, ys.size + 2))
        dcg = float((ys[:k] * disc[:k]).sum())
        idcg = float(disc[:min(P, k)].sum())
        hits = float(ys[:k].sum())
        for name, want in (("ndcg", dcg / idcg), ("precision", hits / min(k, ys.size)), ("recall", hits / P)):
            assert abs(per[name][j] - want) <= 1e-9 * want + 1e-300, (name, per[name][j], want)
    scored = ~np.isnan(per["ndcg"]) & (per["rows"] > per["positives"])
    for name in ("ndcg", "precision", "recall"):
        x, w = per[name][scored], per["rows"][scored]
        assert abs(rep[name] - float(np.average(x, weights=w))) <= 1e-9
        assert abs(rep[name + "_mean"] - float(np.mean(x))) <= 1e-9


def test_permuting_and_recutting_leave_the_output_unchanged():
    p, y, g = _rows(11, 20000, 300, LEVELS)
    p[::113] = np.nan
    want = T.evaluate(p, y, g, 10)
    perm = np.random.default_rng(12).permutation(p.size)
    m = GM.GroupMetric()
    cuts = [0, 1, 17, 5000, 5001, 13000, p.size]
    for a, b in zip(cuts, cuts[1:]):
        m.add(p[perm[a:b]], y[perm[a:b]], g[perm[a:b]])
    got = T.evaluate(*(np.concatenate([pt[i] for pt in m.parts]) for i in range(3)), 10)
    for key in want[0]:
        assert got[0][key] == want[0][key] or (math.isnan(got[0][key]) and math.isnan(want[0][key])), key
    for key in want[1]:
        assert np.array_equal(got[1][key], want[1][key], equal_nan=key in ("ndcg", "precision", "recall")), key


def test_edges():
    f = np.float32
    # one group: positives at ranks 0 and 2 of 4 distinct scores
    p = np.array([0.9, 0.7, 0.5, 0.3], f)
    y = np.array([1, 0, 1, 0], np.uint8)
    g = np.zeros(4, np.uint64)
    D = T.cumulative(8)
    d = [D[i + 1] - D[i] for i in range(8)]
    rep, per = T.evaluate(p, y, g, 1)                     # k = 1
    assert per["H"][0] == T.UNIT and per["G"][0] == d[0] and per["ndcg"][0] == 1.0
    assert per["precision"][0] == 1.0 and per["recall"][0] == 0.5
    for k in (4, 7, 65536):                                # k >= n_g: precision divides by n_g, recall is 1
        rep, per = T.evaluate(p, y, g, k)
        assert per["precision"][0] == 0.5 and per["recall"][0] == 1.0
        assert per["ndcg"][0] == float(d[0] + d[2]) / float(d[0] + d[1])
    # P_g = 0: NaN, and the group is not scored; N_g = 0: ndcg and precision 1, and not scored either
    rep, per = T.evaluate(np.array([0.2, 0.1, 0.4, 0.4], f), np.array([0, 0, 1, 1], np.uint8),
                          np.array([5, 5, 6, 6], np.uint64), 1)
    assert math.isnan(per["ndcg"][0]) and math.isnan(per["precision"][0]) and math.isnan(per["recall"][0])
    assert per["ndcg"][1] == per["precision"][1] == 1.0 and per["recall"][1] == 0.5   # two tied positives, k = 1
    assert rep["scored_groups"] == 0 and rep["scored_rows"] == 0 and math.isnan(rep["ndcg"])
    assert math.isnan(rep["precision_mean"]) and rep["groups"] == 2
    # one-row groups
    rep, per = T.evaluate(np.array([0.3, 0.6], f), np.array([1, 0], np.uint8), np.array([1, 2], np.uint64), 10)
    assert per["ndcg"][0] == per["precision"][0] == per["recall"][0] == 1.0 and math.isnan(per["ndcg"][1])
    # a run of 3 rows holding 1 positive straddles k = 2: H = rn(2^33 / 3), G = rn((d0 + d1) / 3)
    rep, per = T.evaluate(np.array([0.5, 0.5, 0.5, 0.1], f), np.array([0, 1, 0, 1], np.uint8), np.zeros(4, np.uint64), 2)
    assert per["H"][0] == T.rn(2 * T.UNIT, 3) and per["G"][0] == T.rn(d[0] + d[1], 3)
    # an empty set
    rep, per = T.evaluate(np.zeros(0, f), np.zeros(0, np.uint8), np.zeros(0, np.uint64), 5)
    assert rep["groups"] == rep["scored_rows"] == 0 and all(math.isnan(rep[k]) for k in ("ndcg", "recall_mean"))


def test_rounding_is_to_nearest_even():
    assert [T.rn(x, 2) for x in (1, 3, 5, 7)] == [0, 2, 2, 4]
    assert T.rn(2, 3) == 1 and T.rn(1, 3) == 0 and T.rn(10 ** 30 + 1, 2) == 10 ** 30 // 2


def test_the_librarys_discounts_are_the_50_digit_table():
    from xflow_b200 import api
    want = T.discounts()
    got = api.group_discounts()
    assert got.dtype == np.uint64 and np.array_equal(got, want)
    assert int(want[0]) == 2 ** 32 and int(want[2]) == 2 ** 31
    assert math.log2(T.cumulative()[-1]) < 44.2
    assert np.array_equal(api.group_discounts(7), want[:7]) and api.group_discounts(0).size == 0
    with pytest.raises(api.XflowError, match="65537"):
        api.group_discounts(65537)

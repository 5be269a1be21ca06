"""CPU statement of the grouped metric's ranking quality at a cutoff (include/xflow_b200.h section 9,
xf_group_metric_topk): the discounts from 50-digit decimal logarithms, each group's H and G as exact integers, the
per-group doubles in IEEE float64 and the report's means as exact Fractions rounded to float.  The rows, sort and tie
runs are those of tests/group_metric_model.py."""
import math
from decimal import Decimal, ROUND_HALF_EVEN, localcontext
from fractions import Fraction

import numpy as np

UNIT = 2 ** 32
MAX_K = 65536
_D = [0]   # the cumulative discounts D(0 ..) computed so far


def _extend(n):
    """D(0 .. n), computed once: d(i) = 2^32 ln 2 / ln(i + 2) at 50 significant digits, rounded half to even."""
    with localcontext() as ctx:
        ctx.prec = 50
        ln2 = Decimal(2).ln()
        for i in range(len(_D) - 1, n):
            d = (Decimal(UNIT) * ln2 / Decimal(i + 2).ln()).to_integral_value(ROUND_HALF_EVEN)
            _D.append(_D[-1] + int(d))


def cumulative(n=MAX_K):
    """D(0 .. n) as Python ints (n <= 65536)."""
    assert 0 <= n <= MAX_K
    if len(_D) <= n:
        _extend(n)
    return _D[:n + 1]


def discounts(n=MAX_K):
    """d(0 .. n-1) as uint64."""
    D = cumulative(n)
    return np.array([b - a for a, b in zip(D, D[1:])], np.uint64)


def rn(num, den):
    """The exact rational num / den (integers, den > 0) rounded to the nearest integer, ties to even."""
    q, r = divmod(num, den)
    return q + (1 if 2 * r > den or (2 * r == den and q & 1) else 0)


def runs(pctr, labels, groups):
    """The finish's sorted non-NaN rows as tie runs: (ids of the groups, per-group n and P, and per run its group index,
    start a within its group, rows c and positives m), all numpy int64 but the ids."""
    p = np.asarray(pctr, np.float32).ravel()
    y = np.asarray(labels).ravel() != 0
    g = np.asarray(groups, np.uint64).ravel()
    keep = ~np.isnan(p)
    p, y, g = p[keep], y[keep], g[keep]
    p = np.where(p == 0, np.float32(0), p)
    order = np.lexsort((-p, g))
    p, y, g = p[order], y[order].astype(np.int64), g[order]
    n = p.size
    if n == 0:
        z = np.zeros(0, np.int64)
        return np.zeros(0, np.uint64), z, z, z, z, z, z
    gs = np.flatnonzero(np.r_[True, g[1:] != g[:-1]])
    rs = np.flatnonzero(np.r_[True, (g[1:] != g[:-1]) | (p[1:] != p[:-1])])
    c = np.diff(np.r_[rs, n])
    m = np.add.reduceat(y, rs)
    rg = np.searchsorted(gs, rs, side="right") - 1
    a = rs - gs[rg]
    rows = np.diff(np.r_[gs, n])
    P = np.add.reduceat(y, gs)
    return g[gs], rows, P, rg, a, c, m


def evaluate(pctr, labels, groups, k):
    """(report dict, per-group dict in ascending id order) of topk(k) on the rows (p, y, g)."""
    assert 1 <= k <= MAX_K
    D = cumulative(k)
    ids, rows, P, rg, a, c, m = runs(pctr, labels, groups)
    G_ = ids.size
    o = np.minimum(np.maximum(k - a, 0), c)
    H = [0] * G_
    Gs = [0] * G_
    live = np.flatnonzero((o > 0) & (m > 0))
    for r in live.tolist():
        ar, cr, mr, orr, gi = int(a[r]), int(c[r]), int(m[r]), int(o[r]), int(rg[r])
        H[gi] += rn(mr * orr * UNIT, cr)
        Gs[gi] += rn(mr * (D[ar + orr] - D[ar]), cr)
    Pk = np.minimum(P, k)
    I = [D[v] for v in Pk.tolist()]
    hasp = P > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        ndcg = np.where(hasp, np.array(Gs, np.float64) / np.array(I, np.float64), np.nan)
        precision = np.where(hasp, np.array(H, np.float64) / (np.minimum(rows, k).astype(np.float64) * float(UNIT)),
                             np.nan)
        recall = np.where(hasp, np.array(H, np.float64) / (P.astype(np.float64) * float(UNIT)), np.nan)
    scored = hasp & (rows - P > 0)
    srows = int(rows[scored].sum())
    sgroups = int(scored.sum())
    report = dict(k=k, groups=G_, scored_groups=sgroups, scored_rows=srows)
    for name, x in (("ndcg", ndcg), ("precision", precision), ("recall", recall)):
        t = sum(round((float(r) * v) * UNIT) for r, v in zip(rows[scored].tolist(), x[scored].tolist()))
        mm = sum(round(v * UNIT) for v in x[scored].tolist())
        report[name] = math.nan if srows == 0 else float(Fraction(t, srows * UNIT))
        report[name + "_mean"] = math.nan if sgroups == 0 else float(Fraction(mm, sgroups * UNIT))
    per_group = dict(ids=ids, rows=rows, positives=P, H=np.array(H, dtype=object), G=np.array(Gs, dtype=object),
                     I=np.array(I, dtype=object), ndcg=ndcg, precision=precision, recall=recall)
    return report, per_group

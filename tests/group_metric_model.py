"""CPU statement of the grouped test metric (include/xflow_b200.h section 9, xf_group_metric_*): each group's U2, AUC
and logloss in exact integers and IEEE float64, and the report's ratios as exact Fractions rounded to float.  The
sorting and per-run sums are numpy int64 (every sum stays below 2^63 at the sizes the tests use; the model checks
it), so that it runs at millions of rows."""
import math
from fractions import Fraction

import numpy as np

UNIT = 2 ** 32                  # the logloss and mean sums' unit is 2^-32
Q_MIN, Q_MAX = 1e-15, 1.0 - 1e-15
I63 = 2 ** 63


def loss_units(p, y):
    """L: l * 2^32 rounded to the nearest integer, l = -ln q (y != 0) or -ln(1 - q), q = p clamped to [1e-15, 1 - 1e-15]
    in double (the pv's per-row term at weight 1)."""
    q = min(max(float(np.float32(p)), Q_MIN), Q_MAX)
    return round(Fraction(-math.log(q) if y else -math.log(1.0 - q)) * UNIT)


def ratio(num, den):
    """num / den correctly rounded to double; NaN for den = 0."""
    return math.nan if den == 0 else float(Fraction(int(num), int(den)))


def u2_pairs(p, y):
    """U2 of one group by counting pairs: 2 #{pos > neg} + #{pos == neg}, floats compared as floats."""
    p = [float(v) for v in np.asarray(p, np.float32)]
    pos = [v for v, c in zip(p, np.asarray(y).tolist()) if c]
    neg = [v for v, c in zip(p, np.asarray(y).tolist()) if not c]
    return sum(2 * (a > b) + (a == b) for b in neg for a in pos)


def evaluate(pctr, labels, groups):
    """(report dict, per-group dict of arrays in ascending id order) for the rows (p, y, g)."""
    p = np.asarray(pctr, np.float32).ravel()
    y = np.asarray(labels).ravel() != 0
    g = np.asarray(groups, np.uint64).ravel()
    keep = ~np.isnan(p)
    nan_rows = int(p.size - keep.sum())
    p, y, g = p[keep], y[keep], g[keep]
    p = np.where(p == 0, np.float32(0), p)       # -0.0 ties with +0.0
    order = np.lexsort((-p, g))                   # by group, then by descending prediction
    p, y, g = p[order], y[order].astype(np.int64), g[order]
    n = p.size
    gs = np.flatnonzero(np.r_[True, g[1:] != g[:-1]]) if n else np.zeros(0, np.int64)
    rs = np.flatnonzero(np.r_[True, (g[1:] != g[:-1]) | (p[1:] != p[:-1])]) if n else np.zeros(0, np.int64)
    # tie runs: their positives gp, negatives gn, and the group's positives before them pb
    run_len = np.diff(np.r_[rs, n])
    gp = np.add.reduceat(y, rs) if n else np.zeros(0, np.int64)
    gn = run_len - gp
    run_group = np.searchsorted(gs, rs, side="right") - 1
    before = np.cumsum(gp) - gp                                   # positives before the run, over all groups
    first_run = np.searchsorted(rs, gs)                            # each group's first run
    pb = before - before[first_run][run_group]
    u2 = np.add.reduceat(gn * (2 * pb + gp), first_run) if n else np.zeros(0, np.int64)
    # logloss units: math.log once per distinct (p, y)
    uniq, inv = np.unique(p, return_inverse=True)
    lpos = np.array([loss_units(v, 1) for v in uniq.tolist()], np.int64)
    lneg = np.array([loss_units(v, 0) for v in uniq.tolist()], np.int64)
    L = np.where(y != 0, lpos[inv], lneg[inv])
    s = np.add.reduceat(L, gs) if n else np.zeros(0, np.int64)
    rows = np.diff(np.r_[gs, n]).astype(np.int64)
    P = np.add.reduceat(y, gs) if n else np.zeros(0, np.int64)
    N = rows - P
    assert n < 2 ** 31 and (L.sum() if n else 0) < I63 // 2 and (u2.max() if n else 0) < I63 // 2
    scored = (P > 0) & (N > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        auc = np.where(scored, u2.astype(np.float64) / ((2.0 * P.astype(np.float64)) * N.astype(np.float64)), np.nan)
    logloss = s.astype(np.float64) / (rows.astype(np.float64) * float(UNIT))
    T = [round((float(r) * a) * UNIT) for r, a in zip(rows[scored].tolist(), auc[scored].tolist())]
    M = [round(a * UNIT) for a in auc[scored].tolist()]
    R = int(rows.sum())
    report = dict(rows=R, positives=int(P.sum()), negatives=int(N.sum()), nan_rows=nan_rows, groups=int(gs.size),
                  scored_groups=int(scored.sum()), scored_rows=int(rows[scored].sum()))
    report["logloss"] = ratio(sum(int(v) for v in s.tolist()), R * UNIT)
    report["gauc"] = ratio(sum(T), report["scored_rows"] * UNIT)
    report["gauc_mean"] = ratio(sum(M), report["scored_groups"] * UNIT)
    per_group = dict(ids=g[gs] if n else np.zeros(0, np.uint64), rows=rows.astype(np.uint64),
                     positives=P.astype(np.uint64), auc=auc, logloss=logloss, u2=u2, s=s)
    return report, per_group


class GroupMetric:
    """The metric's calls: add appends rows, finish evaluates every row added since the last reset."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.parts = []

    def add(self, pctr, labels, groups):
        self.parts.append((np.asarray(pctr, np.float32), np.asarray(labels, np.uint8), np.asarray(groups, np.uint64)))
        return self

    def finish(self):
        if not self.parts:
            return evaluate(np.zeros(0, np.float32), np.zeros(0, np.uint8), np.zeros(0, np.uint64))
        return evaluate(*(np.concatenate([pt[k] for pt in self.parts]) for k in range(3)))

"""CPU statement of progressive validation's metric (include/xflow_b200.h section 8, xf_pv_*): the bins and fixed-point
sums in Python integers, the report as exact rationals rounded to double, and the exact weighted AUC of the raw
floats (ties counted 1/2) that the report's [auc_lo, auc_hi] must bracket."""
import math
from fractions import Fraction

import numpy as np

UNIT = 2 ** 32           # the sums' unit is 2^-32
P_MIN = 2.0 ** -20       # the binning clamp [2^-20, 1]
Q_MIN, Q_MAX = 1e-15, 1.0 - 1e-15


def f32(x):
    return float(np.float32(x))


def nbins(m):
    return 20 * 2 ** m + 1


def bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def clamp_p(p):
    """pc: p clamped to [2^-20, 1] in float (p not NaN)."""
    return min(max(f32(p), P_MIN), 1.0)


def bin_of(p, m):
    pc = clamp_p(p)
    return (bits(pc) >> (23 - m)) - (bits(P_MIN) >> (23 - m))


def loss_term(p, y):
    """l = -ln(q) (positive) or -ln(1 - q) (negative), q = p clamped to [1e-15, 1 - 1e-15] in double."""
    q = min(max(float(np.float32(p)), Q_MIN), Q_MAX)
    return -math.log(q) if y else -math.log(1.0 - q)


def units(x):
    """x (a double, >= 0) in units of 2^-32, rounded to nearest even after the exact scaling."""
    return round(Fraction(x) * UNIT)


class Pv:
    def __init__(self, m=10):
        self.m = m
        self.n = [[0, 0] for _ in range(nbins(m))]   # [bin][class]
        self.w = [[0, 0] for _ in range(nbins(m))]
        self.nan_rows = self.overflow_rows = 0
        self.el = self.ep = 0

    def add(self, pctr, labels, weights=None):
        pctr = np.asarray(pctr, np.float32)
        labels = np.asarray(labels)
        weights = np.ones(pctr.size, np.float32) if weights is None else np.asarray(weights, np.float32)
        for p, y, e in zip(pctr.tolist(), labels.tolist(), weights.tolist()):
            if e == 0.0:
                continue
            if not (e >= 0.0 and e < 2.0 ** 31):
                self.overflow_rows += 1
                continue
            if p != p:
                self.nan_rows += 1
                continue
            c = 1 if y != 0 else 0
            b = bin_of(p, self.m)
            self.n[b][c] += 1
            self.w[b][c] += units(e)
            self.ep += units(e * clamp_p(p))           # exact in double
            self.el += units(e * loss_term(p, c))      # e * l rounded once in double
        return self

    def exact(self):
        """The report's fields as exact rationals (None where the report has NaN)."""
        wn = sum(w[0] for w in self.w)
        wp = sum(w[1] for w in self.w)
        W = wn + wp
        r = dict(positives=sum(n[1] for n in self.n), negatives=sum(n[0] for n in self.n),
                 nan_rows=self.nan_rows, overflow_rows=self.overflow_rows,
                 weight_pos=Fraction(wp, UNIT), weight_neg=Fraction(wn, UNIT))
        r["rows"] = r["positives"] + r["negatives"]
        r["logloss"] = Fraction(self.el, W) if W else None
        r["mean_pctr"] = Fraction(self.ep, W) if W else None
        r["ctr"] = Fraction(wp, W) if W else None
        if wp and wn:
            above, lo, tie = 0, 0, 0
            for b in range(len(self.w) - 1, -1, -1):
                lo += self.w[b][0] * above
                tie += self.w[b][0] * self.w[b][1]
                above += self.w[b][1]
            r["auc_lo"] = Fraction(lo, wp * wn)
            r["auc_hi"] = Fraction(lo + tie, wp * wn)
            r["auc"] = (r["auc_lo"] + r["auc_hi"]) / 2
        else:
            r["auc_lo"] = r["auc_hi"] = r["auc"] = None
        return r

    def report(self):
        """The report as the library states it: every ratio correctly rounded to double, NaN where undefined."""
        return {k: (v if isinstance(v, int) else (math.nan if v is None else float(v))) for k, v in self.exact().items()}


def exact_auc(pctr, labels, weights=None):
    """Weighted AUC of the raw floats with ties counted 1/2, over the rows a pv scores (exact rational; None if a
    class has no weight)."""
    pctr = np.asarray(pctr, np.float32)
    weights = np.ones(pctr.size, np.float32) if weights is None else np.asarray(weights, np.float32)
    rows = [(float(p), 1 if y else 0, units(float(e))) for p, y, e in zip(pctr.tolist(), np.asarray(labels).tolist(),
                                                                            weights.tolist())
            if e != 0.0 and e >= 0.0 and e < 2.0 ** 31 and p == p]
    pos = [(p, u) for p, c, u in rows if c]
    neg = [(p, u) for p, c, u in rows if not c]
    wp, wn = sum(u for _, u in pos), sum(u for _, u in neg)
    if not wp or not wn:
        return None
    num = Fraction(0)
    for pn, un in neg:
        for pp, up in pos:
            if pp > pn:
                num += un * up
            elif pp == pn:
                num += Fraction(un * up, 2)
    return num / (wp * wn)

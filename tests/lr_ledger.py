"""Exact ledger of one lazy LR training step (xflow_b200/csrc/step_lazy.cu: xf_k_step_lr_lazy) from any table state.

A lazy LR step sums each key's residuals as integers: every token of row r deposits xf_fix_of(e_r * residual_r, s),
the residual in units of 2^-s rounded to nearest (ties to even), and the deposits of a key add up in a 48-bit field.
Integer adds do not depend on the order in which they land, so once the kernel's own float32 residuals are known the
post-step table is a deterministic function of the pre-step state:
  * s = xf_fix_shift(nnz) for an unweighted step (nnz = the batch's token count), xf_fix_shift(W) for a weighted one
    (W = sum over the rows with e_r > 0 of ceil(e_r) * len_r, weighting_model.fix_bound);
  * a key's gradient is the sum scaled back with that unit, rounded to float once, divided in double by the batch's
    row count and rounded again (xf_lazy_fold);
  * one FTRL (xf_ftrl_coord) or SGD (xf_sgd_coord) step in float32, operation for operation as table.cuh writes it,
    from the pre-step weight, which may be an imported one that is not f(z, n).
ledger_step() states that function; a step whose export differs from it in one bit lost, doubled or mis-scaled a
deposit somewhere.  The residuals themselves depend on the order a row's weights are summed in, so they are held to
an order-free interval instead (residual_bounds)."""
import numpy as np

from fm_model import ALPHA, BETA, L1, L2, LR, U, gamma, sigmoid_range
from test_lazy_fixed_point_model import fix_shift
from weighting_model import fix_bound

F = np.float32
FIELD_LIMIT = (1 << 47) - 1
PERTURBATIONS = ("drop_token", "double_token", "group_count_1", "unit_off_by_one", "rows_plus_1", "rows_minus_1")


def ftrl_w(z, n):
    """xf_ftrl_w in float32: the FTRL weight of the accumulators (ftrl.h:66-74)."""
    z, n = np.asarray(z, F), np.asarray(n, F)
    tmpr = np.where(z > 0, z - F(L1), np.where(z < 0, z + F(L1), F(0))).astype(F)
    tmpl = -((F(BETA) + np.sqrt(n)) / F(ALPHA) + F(L2))
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(np.abs(z) <= F(L1), F(0), tmpr / tmpl).astype(F)


def ftrl_coord(g, w, n, z):
    """xf_ftrl_coord in float32: (w, n, z) after one step with gradient g."""
    g, w, n, z = (np.asarray(a, F) for a in (g, w, n, z))
    nn = n + g * g
    sig = (np.sqrt(nn) - np.sqrt(n)) / F(ALPHA)
    z2 = z + (g - sig * w)
    return ftrl_w(z2, nn), nn.astype(F), z2.astype(F)


def sgd_coord(g, w):
    """xf_sgd_coord in float32."""
    return (np.asarray(w, F) - F(LR) * np.asarray(g, F)).astype(F)


def fix_of(x, s):
    """xf_fix_of of float32 values: units of 2^-s, rounded to nearest with ties to even (__double2ll_rn)."""
    return np.rint(np.asarray(x, F).astype(np.float64) * 2.0 ** s).astype(np.int64)


def fold_gradient(sums, s, rows):
    """xf_lazy_fold's gradient: (float)((double)(float)(sum * 2^-s) / rows)."""
    return (np.asarray(sums, np.int64).astype(np.float64) * 2.0 ** -s).astype(F).astype(np.float64) / float(rows)


def apply_step(pre, g, trained, opt):
    """One optimizer step with gradients g (float32) on the trained keys of the exported state `pre`; the others keep
    their state."""
    w, n, z = (np.array(pre[f], F) for f in ("w", "nw", "zw"))
    g = np.asarray(g, np.float64).astype(F)
    t = np.asarray(trained, bool)
    if opt == "ftrl":
        w2, n2, z2 = ftrl_coord(g[t], w[t], n[t], z[t])
        w[t], n[t], z[t] = w2, n2, z2
    else:
        w[t] = sgd_coord(g[t], w[t])
    return dict(w=w, nw=n, zw=z)


class Ledger(dict):
    """The post-step {w, nw, zw} of the sorted unique keys; also .uk, .trained (the keys the step trained), .sums (their
    integer residual sums), .s (the unit's shift) and .g (the gradients)."""


def ledger_step(pre, rp, keys, residuals, rows, opt, e=None, keep=None, perturb=None):
    """The post-step state of every key of the batch.

    pre: the exported state before the step (dict with keys = the batch's sorted unique keys, w, nw, zw; absent keys
    export zeros).  residuals: the step's float32 residual per row, unweighted, as get_loss returns them.  rows: the
    divisor, the batch's full row count.  e: the rows' effective weights (None: an unweighted step).  keep: per token,
    False where admission rejected the key (it deposits nothing).  perturb: one of PERTURBATIONS, a deliberately wrong
    deposit or fold, to show that the ledger tells it apart."""
    assert perturb is None or perturb in PERTURBATIONS
    uk = np.asarray(pre["keys"], np.uint64)
    keys = np.ascontiguousarray(keys, np.uint64)
    rp = np.asarray(rp, np.int64)
    B = rp.size - 1
    assert np.all(uk[:-1] < uk[1:]), "pre must hold the sorted unique keys"
    inv = np.searchsorted(uk, keys)
    assert np.array_equal(uk[np.minimum(inv, uk.size - 1)], keys), "pre must hold every key of the batch"
    row_of = np.repeat(np.arange(B), np.diff(rp))
    res = np.asarray(residuals, F)
    if e is None:
        s = fix_shift(keys.size)
        loss = res
        live_row = np.ones(B, bool)
    else:
        e = np.asarray(e, F)
        s = fix_shift(fix_bound(rp, e))
        loss = (e * res).astype(F)
        live_row = e > 0
    tok = live_row[row_of]
    if keep is not None:
        tok &= np.asarray(keep, bool)
    dep = fix_of(loss[row_of], s + 1 if perturb == "unit_off_by_one" else s)
    dep = np.where(tok, dep, 0)
    if perturb in ("drop_token", "double_token"):
        j = int(np.argmax(np.where(tok, np.abs(dep), -1)))
        dep[j] = 0 if perturb == "drop_token" else 2 * dep[j]
    if perturb == "group_count_1":
        # the first key that occurs more than once in one 32-token warp chunk of a row deposits as if it occurred once
        chunk = row_of.astype(np.int64) * (1 << 32) + (np.arange(keys.size) - rp[row_of]) // 32
        pair = np.stack([chunk, inv]).T[tok]
        u, c = np.unique(pair, axis=0, return_counts=True)
        assert (c > 1).any(), "group_count_1 needs a key twice in one warp chunk"
        ch, k = u[np.argmax(c > 1)]
        hit = np.flatnonzero(tok & (chunk == ch) & (inv == k))
        dep[hit[1:]] = 0
    sums = np.zeros(uk.size, np.int64)
    np.add.at(sums, inv, dep)
    assert np.all(np.abs(sums) <= FIELD_LIMIT), "a residual sum left the 48-bit field"
    trained = np.zeros(uk.size, bool)
    trained[inv[tok]] = True
    div = rows + (1 if perturb == "rows_plus_1" else -1 if perturb == "rows_minus_1" else 0)
    g = fold_gradient(sums, s, div).astype(F)
    out = Ledger(apply_step(pre, g, trained, opt))
    out.uk, out.trained, out.sums, out.s, out.g = uk, trained, sums, s, g
    return out


def residual_bounds(pre_w, rp, keys, labels):
    """[lo, hi] (float64) of each row's residual, whatever order the row's weights are summed in.  pre_w: the weight
    each token pulls (0 for a token whose key admission rejected)."""
    rp = np.asarray(rp, np.int64)
    B = rp.size - 1
    row_of = np.repeat(np.arange(B), np.diff(rp))
    w = np.asarray(pre_w, F).astype(np.float64)
    t = np.diff(rp).astype(np.float64)
    wx = np.bincount(row_of, w, minlength=B)
    wabs = np.bincount(row_of, np.abs(w), minlength=B)
    e = gamma(t) * wabs
    pl, ph = sigmoid_range(wx - e, wx + e)
    pl, ph = pl * (1 - 1.5 * U), ph * (1 + 1.5 * U)   # the rounding to float (and exp's own error, ~1e-15)
    lab = np.asarray(labels, np.float64)
    lo, hi = pl - lab, ph - lab
    r = U * np.maximum(np.abs(lo), np.abs(hi))         # the float subtraction of the label
    return lo - r, hi + r

"""float64 model of one training step of the reference's FM (XF_MODEL_FM: step.cu's xf_k_step and kernels.cu's
xf_k_update) from ANY table state, with a-priori rounding bounds that hold for every summation order.

Semantics (DESIGN.md section 1, fm_worker.cc:126-245): x = 1 for every token; a row's argument is
wx + (sum v)^2 - sum v^2 with both sums over all tokens and all k (no 1/2); the residual is
sigmoid(arg) - label with the reference's clamped sigmoid (pow(2.718281828, x), 1e-6 below -30, 1 above 30);
a key's w-gradient adds the residual K times per occurrence (fm_worker.cc:140); its latent gradient is
sum_occ residual * (S_row - v_k) = Aq - v_k L; both are divided by the batch's row count in double; then one FTRL
(ftrl.h:59-74) or SGD (sgd.h) step per coordinate.  Importance weights multiply the residual in the gradients only.

The centre is that arithmetic in float64 on the float32 state.  The bounds follow the standard float error
analysis with u = 2^-24 and gamma(n) = n u / (1 - n u), so they hold whatever order an implementation sums in, as
long as it sums in float32 or better:
  * a row of t tokens: wx, S and Q are sums of t, tK and tK terms, each within gamma(terms) * sum |terms| of exact;
  * that carries into arg = wx + S^2 - Q (with the rounding of the three operations), into the residual through the
    sigmoid evaluated at both ends of arg's interval (plus its own rounding and the clamp at -30), and into the
    subtraction of the label;
  * a key's sums over its m occurrences carry each occurrence's residual and S error, plus gamma(m + 2) of the summed
    magnitudes: a float sum of the reference's per-k terms residual * (S - v_k), or of the factorised L and Aq;
  * the K-fold w-gradient carries gamma(K m) of K sum |residual|: the reference adds the residual K m times in
    float;
  * the quotient by the row count and the cast to float add a rounding each;
  * through one optimizer step the gradient's interval is mapped exactly (FTRL's n' and z' at both ends of the
    interval and at their extrema inside it; w' at the corners of the (z', n') box, which bound it because w' is
    monotone in each), then widened by an operation-by-operation bound of the kernel's own float32 FTRL / SGD
    arithmetic.  At the L1 threshold (|z'| ~ lambda1) the box holds both sides, so either is accepted.

fm_step() computes one step; check_step() holds an implementation's residuals and post-step state to it;
run_steps() drives an implementation step by step from its own pre-step state (so errors never compound)."""
import numpy as np

U = 2.0 ** -24
ALPHA, BETA, L1, L2 = float(np.float32(5e-2)), 1.0, float(np.float32(5e-5)), 10.0  # ftrl.h:17-20 (float members)
LR = float(np.float32(1e-3))  # sgd.h:16
P_MIN = float(np.float32(1e-6))  # base.h:56: the sigmoid below -30
SAFETY = 1.01  # covers the second-order terms the first-order bounds below leave out
FIELDS = ("w", "nw", "zw", "v", "nv", "zv")
PERTURBATIONS = ("div_b_plus_1", "no_k_fold", "half", "post_step_v", "drop_hot_occurrence", "previous_n")


def gamma(n):
    nu = np.maximum(np.asarray(n, np.float64), 0.0) * U
    assert np.all(nu < 0.5), "too many terms for the float error bounds"
    return nu / (1.0 - nu)


def sigmoid(x):
    """Base::sigmoid (base.h:54-63) in float64, before the rounding to float."""
    x = np.asarray(x, np.float64)
    e = np.power(2.718281828, np.clip(x, -30.0, 30.0))
    return np.where(x < -30.0, P_MIN, np.where(x > 30.0, 1.0, e / (1.0 + e)))


def sigmoid_range(lo, hi):
    """[min, max] of the clamped sigmoid over [lo, hi]: monotone except for the drop from 1e-6 to sigmoid(-30)."""
    a, b = sigmoid(lo), sigmoid(hi)
    pl, ph = np.minimum(a, b), np.maximum(a, b)
    across = (lo < -30.0) & (hi >= -30.0)
    pl = np.where(across, np.minimum(pl, sigmoid(-30.0)), pl)
    ph = np.where(across, np.maximum(ph, P_MIN), ph)
    return pl, ph


def ftrl_w(z, n):
    """FTRL's weight from its accumulators (ftrl.h:66-74), float64; continuous, non-increasing in z."""
    d = (BETA + np.sqrt(np.maximum(n, 0.0))) / ALPHA + L2
    return np.where(np.abs(z) <= L1, 0.0, -(z - np.sign(z) * L1) / d)


def _ftrl_z(g, w, n, z, n_sig):
    return z + g - (np.sqrt(n + g * g) - np.sqrt(n_sig)) / ALPHA * w


def ftrl_step(g, eg, w, n, z, n_sig=None):
    """One FTRL coordinate step for a gradient in [g - eg, g + eg] from the float state (w, n, z).
    Returns {w, n, z: (centre, lo, hi)}.  n_sig (a wrong previous n) changes the centre only."""
    n_sig = n if n_sig is None else n_sig
    glo, ghi = g - eg, g + eg
    n_c = n + g * g
    z_c = _ftrl_z(g, w, n, z, n_sig)
    w_c = ftrl_w(z_c, n_c)
    # n' = n + g^2 over the interval
    g2lo = np.where((glo <= 0) & (ghi >= 0), 0.0, np.minimum(glo * glo, ghi * ghi))
    g2hi = np.maximum(glo * glo, ghi * ghi)
    nlo, nhi = n + g2lo, n + g2hi
    # z'(g) at both ends, at 0 (its kink when n = 0) and where dz'/dg = 1 - (w / alpha) g / sqrt(n + g^2) vanishes
    cands = [_ftrl_z(glo, w, n, z, n), _ftrl_z(ghi, w, n, z, n)]
    inside0 = (glo <= 0) & (ghi >= 0)
    cands.append(np.where(inside0, _ftrl_z(np.zeros_like(g), w, n, z, n), cands[0]))
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.where(w != 0, ALPHA / np.where(w != 0, w, 1.0), np.inf)
        crit = np.abs(c) < 1
        gs = np.where(crit, np.sign(c) * np.abs(c) * np.sqrt(n) / np.sqrt(np.where(crit, 1 - c * c, 1.0)), 0.0)
    use = crit & (gs >= glo) & (gs <= ghi)
    cands.append(np.where(use, _ftrl_z(gs, w, n, z, n), cands[0]))
    cands = np.stack(cands)
    zlo, zhi = cands.min(0), cands.max(0)
    # the kernel's float32 arithmetic, operation by operation (xf_ftrl_coord / xo_ftrl_coord)
    G = np.maximum(np.abs(glo), np.abs(ghi))
    e_nn = U * nhi + U * G * G                       # g*g, n + g*g
    s1 = np.sqrt(nhi)
    with np.errstate(divide="ignore", invalid="ignore"):
        e_s1 = U * s1 + np.where(nlo > 0, np.minimum(e_nn / np.sqrt(np.where(nlo > 0, nlo, 1.0)), np.sqrt(e_nn)),
                                 np.sqrt(e_nn))
    e_s0 = U * np.sqrt(n)
    dhi = s1 - np.sqrt(n)
    e_d = e_s1 + e_s0 + U * (dhi + e_s1 + e_s0)
    e_sig = e_d / ALPHA + U * (dhi + e_d) / ALPHA
    sw = (dhi + e_d) / ALPHA * np.abs(w)
    e_sw = e_sig * np.abs(w) + U * sw
    e_t = e_sw + U * (G + sw)
    zmag = np.maximum(np.abs(zlo), np.abs(zhi))
    e_z = SAFETY * (e_t + U * (zmag + e_t))
    e_n = SAFETY * e_nn
    zlo, zhi = zlo - e_z, zhi + e_z
    nlo, nhi = np.maximum(nlo - e_n, 0.0), nhi + e_n
    corners = np.stack([ftrl_w(zz, nn) for zz in (zlo, zhi) for nn in (nlo, nhi)])
    wlo, whi = corners.min(0), corners.max(0)
    e_w = SAFETY * 6 * U * np.maximum(np.abs(wlo), np.abs(whi))  # tmpr, sqrt, +beta, /alpha, +lambda2, /
    return dict(w=(w_c, wlo - e_w, whi + e_w), n=(n_c, nlo, nhi), z=(z_c, zlo, zhi))


def sgd_step(g, eg, w):
    """w - lr g for a gradient in [g - eg, g + eg]; float32 rounding of the product and the difference."""
    lo, hi = w - LR * (g + eg), w - LR * (g - eg)
    e = SAFETY * U * (LR * (np.abs(g) + eg) + np.maximum(np.abs(lo), np.abs(hi)))
    return w - LR * g, lo - e, hi + e


class Step:
    """One modelled step: residuals (centre, half-width), pctr interval, and per field (centre, lo, hi) over uk."""


def fm_step(uk, state, rp, keys, lab, K, opt, weights=None, keep=None, perturb=None, n_prev=None):
    """Model one step from `state` (float32 arrays w, nw, zw [U] and v, nv, zv [U, K] of the sorted keys uk, which
    must hold every key of a kept token).  keep: tokens the step trains on (admission: rejected tokens read as zero
    and are left out); rows with weight 0 are left out too, and the divisor stays the batch's row count.
    perturb: one of PERTURBATIONS, a deliberately wrong arithmetic (only the centres change; n_prev: the state's
    nw / nv of the step before, for "previous_n")."""
    assert perturb is None or perturb in PERTURBATIONS
    B = lab.size
    rp = np.asarray(rp, np.int64)
    row_of = np.repeat(np.arange(B), np.diff(rp))
    e_row = np.ones(B) if weights is None else np.asarray(weights, np.float32).astype(np.float64)
    tok = np.ones(keys.size, bool) if keep is None else np.asarray(keep, bool).copy()
    tok &= e_row[row_of] != 0
    rows, inv = row_of[tok], np.searchsorted(uk, keys[tok])
    assert np.array_equal(uk[inv], keys[tok]), "uk must hold every trained key"
    nU = uk.size
    W = state["w"].astype(np.float64)
    V = state["v"].astype(np.float64).reshape(nU, K)
    # ---- forward: per-row sums and their error bounds
    t = np.bincount(rows, minlength=B).astype(np.float64)

    def rsum(x):
        return np.bincount(rows, x[inv], minlength=B)

    wx, wabs = rsum(W), rsum(np.abs(W))
    S, Sabs, Q = rsum(V.sum(1)), rsum(np.abs(V).sum(1)), rsum((V * V).sum(1))
    y = 0.5 * (S * S - Q) if perturb == "half" else S * S - Q
    arg = wx + y
    eS = gamma(t * K - 1) * Sabs
    eQ = gamma(t * K) * Q
    e_y = 2 * np.abs(S) * eS + eS * eS + U * (np.abs(S) + eS) ** 2 + eQ
    e_y += U * (np.abs(y) + e_y)
    e_arg = gamma(t - 1) * wabs + e_y
    e_arg = SAFETY * (e_arg + U * (np.abs(arg) + e_arg))
    pl, ph = sigmoid_range(arg - e_arg, arg + e_arg)
    pl, ph = pl * (1 - 1.5 * U), ph * (1 + 1.5 * U)  # the rounding to float (and pow's own error, ~1e-15)
    st = Step()
    st.B, st.uk = B, uk
    st.pctr = (sigmoid(arg), pl, ph)
    lab64 = lab.astype(np.float64)
    res = sigmoid(arg) - lab64
    e_res = np.maximum(ph - lab64 - res, res - (pl - lab64))
    e_res = e_res + U * (np.abs(res) + e_res)
    trained = e_row != 0
    st.loss = (np.where(trained, res, 0.0), np.where(trained, e_res, 0.0))
    ell, e_ell = e_row * res, e_row * e_res
    if weights is not None:
        e_ell = e_ell + U * (np.abs(ell) + e_ell)
    # ---- backward: per-key sums of the occurrences
    l, el, s, es = ell[rows], e_ell[rows], S[rows], eS[rows]

    def ksum(x):
        return np.bincount(inv, x, minlength=nU)

    m = np.bincount(inv, minlength=nU).astype(np.float64)
    a1, a2, a3 = ksum(el * (np.abs(s) + es)), ksum(el), ksum(np.abs(l) * es)
    b1, b2 = ksum((np.abs(l) + el) * (np.abs(s) + es)), ksum(np.abs(l) + el)
    eg = (a1[:, None] + np.abs(V) * a2[:, None] + a3[:, None]) / B
    eg += gamma(m + 2)[:, None] * (b1[:, None] + np.abs(V) * b2[:, None]) / B
    if perturb == "drop_hot_occurrence":
        # lose one occurrence's terms: of the most frequent key among those where one occurrence's term
        # |l| |S| / B exceeds the bound of its sums (a key of m occurrences carries m u of m terms, so a lost term is
        # only visible while m^2 u stays small), the occurrence with the largest term
        term = np.abs(l) * np.abs(s) / B
        big = np.zeros(nU)
        np.maximum.at(big, inv, term)
        seen = big > 4 * eg.max(1)
        hot = np.argmax(np.where(seen, m, 0)) if seen.any() else np.argmax(m)
        j0 = np.nonzero(inv == hot)[0][np.argmax(term[inv == hot])]
        l = l.copy()
        l[j0] = 0.0
    L, Aq = ksum(l), ksum(l * s)
    Bd = B + 1.0 if perturb == "div_b_plus_1" else float(B)
    g = (Aq[:, None] - V * L[:, None]) / Bd
    eg = SAFETY * (eg + 2 * U * (np.abs(g) + eg))
    gw = (1.0 if perturb == "no_k_fold" else K) * L / Bd
    egw = (K * a2 + gamma(K * m) * K * b2) / B
    egw = SAFETY * (egw + 2 * U * (np.abs(gw) + egw))
    # ---- optimizer; keys without a trained occurrence stay as they are
    live = m > 0
    out = {}

    def put(name, cen, lo, hi, old):
        keep_old = live if np.ndim(old) == 1 else live[:, None]
        out[name] = tuple(np.where(keep_old, a, old) for a in (cen, lo, hi))

    st64 = {k: state[k].astype(np.float64).reshape(nU, -1) if k in ("v", "nv", "zv") else state[k].astype(np.float64)
            for k in FIELDS}
    if opt == "ftrl":
        np_w = np_v = None
        if perturb == "previous_n":
            np_w, np_v = n_prev["nw"].astype(np.float64), n_prev["nv"].astype(np.float64).reshape(nU, K)
        rw = ftrl_step(gw, egw, st64["w"], st64["nw"], st64["zw"], np_w)
        rv = ftrl_step(g, eg, V, st64["nv"], st64["zv"], np_v)
        if perturb == "post_step_v":
            g2 = (Aq[:, None] - rv["w"][0] * L[:, None]) / Bd
            rv2 = ftrl_step(g2, eg, V, st64["nv"], st64["zv"])
            rv = {k: (rv2[k][0],) + rv[k][1:] for k in rv}
        for f, r in (("w", rw["w"]), ("nw", rw["n"]), ("zw", rw["z"]), ("v", rv["w"]), ("nv", rv["n"]), ("zv", rv["z"])):
            put(f, *r, st64[f])
    else:
        put("w", *sgd_step(gw, egw, st64["w"]), st64["w"])
        rv = sgd_step(g, eg, V)
        if perturb == "post_step_v":
            g2 = (Aq[:, None] - rv[0] * L[:, None]) / Bd
            rv = (sgd_step(g2, eg, V)[0],) + rv[1:]
        put("v", *rv, V)
        for f in ("nw", "zw", "nv", "zv"):
            put(f, st64[f], st64[f], st64[f], st64[f])
    st.fields = out
    st.touched = live
    return st


def _report(what, got, lo, hi, cen):
    bad = ~((got >= lo) & (got <= hi))
    if bad.any():
        idx = [tuple(i) for i in np.argwhere(bad)[:4]]
        det = ", ".join("%s: got %.9g in [%.9g, %.9g] centre %.9g" % (i, got[i], lo[i], hi[i], cen[i]) for i in idx)
        return "%s: %d/%d outside the bounds (%s)" % (what, int(bad.sum()), bad.size, det)
    return None


def violations(st, loss=None, post=None, pctr=None, what=""):
    """Messages for every group of elements outside the step's bounds (empty: all inside)."""
    msgs = []
    if loss is not None:
        c, e = st.loss
        m = _report(what + " residuals", np.asarray(loss, np.float64), c - e, c + e, c)
        msgs += [m] if m else []
    if pctr is not None:
        m = _report(what + " pctr", np.asarray(pctr, np.float64), st.pctr[1], st.pctr[2], st.pctr[0])
        msgs += [m] if m else []
    if post is not None:
        for f in FIELDS:
            cen, lo, hi = st.fields[f]
            got = np.asarray(post[f], np.float64).reshape(cen.shape)
            m = _report("%s %s" % (what, f), got, lo, hi, cen)
            msgs += [m] if m else []
    return msgs


def check_step(st, loss=None, post=None, pctr=None, what=""):
    msgs = violations(st, loss, post, pctr, what)
    assert not msgs, "\n".join(msgs)


def centre_state(st):
    """The centres as float32 state and residuals: a perturbed model's answer, for checks that bounds have teeth."""
    return st.loss[0], {f: st.fields[f][0] for f in FIELDS}


def rel_tolerance(st, field):
    """Half-width over |centre| of every element with a nonzero centre ("loss" for the residuals)."""
    if field == "loss":
        c, e = st.loss
    else:
        c, lo, hi = (a[st.touched] for a in st.fields[field])  # keys the step trained
        e = (hi - lo) / 2
    c, e = np.ravel(c), np.ravel(e)
    nz = c != 0
    return e[nz] / np.abs(c[nz])


def pre_state(export, init_v, keys, K):
    """An implementation's state of `keys` (sorted, unique) before a step: its export, and for keys it does not hold
    the values the step gives a new key (w = n = z = 0, v = init_v(keys))."""
    e = export(keys)
    absent = e["present"] == 0
    st = {f: np.array(e[f], np.float32).reshape(keys.size, -1) if f in ("v", "nv", "zv") else np.array(e[f], np.float32)
          for f in FIELDS}
    if absent.any():
        for f in ("w", "nw", "zw"):
            st[f][absent] = 0.0
        st["v"][absent] = np.asarray(init_v(keys[absent]), np.float32).reshape(-1, K)
        st["nv"][absent] = 0.0
        st["zv"][absent] = 0.0
    return st, e["present"].astype(bool)


def run_steps(export, step, init_v, batches, K, opt, weights=None, on_step=None, admitted=False):
    """Drive an implementation step by step and hold each step to the model from the implementation's own pre-step
    state.  export(keys) -> dict(w, nw, zw, v, nv, zv, present); step(i, rp, keys, lab) -> float32 residuals;
    init_v(keys) -> v of new keys.  admitted: the step may reject absent keys (a key absent before and after the step
    was rejected; its tokens are left out).  on_step(i, st, post, loss) sees every checked step.  Returns the
    steps."""
    out = []
    for i, (rp, keys, lab) in enumerate(batches):
        uk = np.unique(keys)
        pre, _ = pre_state(export, init_v, uk, K)
        loss = step(i, rp, keys, lab)
        post_e = export(uk)
        keep = None
        if admitted:
            keep = (post_e["present"] != 0)[np.searchsorted(uk, keys)]
        st = fm_step(uk, pre, rp, keys, lab, K, opt, weights=None if weights is None else weights[i], keep=keep)
        post = {f: post_e[f] for f in FIELDS}
        absent = post_e["present"] == 0
        assert not (absent & st.touched).any(), "step %d: a key the step trained has no row" % i
        for f in FIELDS:  # a key no trained token reached (rejected, or only in rows of weight 0) may have no row
            post[f] = np.where(absent.reshape((-1,) + (1,) * (np.ndim(post[f]) - 1)), st.fields[f][0], post[f])
        check_step(st, loss, post, what="step %d:" % i)
        if on_step:
            on_step(i, st, post, loss)
        out.append(st)
    return out

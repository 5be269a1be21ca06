"""tests/fm_model.py on the CPU: its bounds contain the reference and exclude wrong arithmetic.

The oracle (the reference's arithmetic restated, pinned bit for bit to the reference) sums in one legal order, in
float32, so its run must lie inside the model's bounds element for element, every step starting from the oracle's
own pre-step state.  A wrong arithmetic must not: every perturbation of fm_model.PERTURBATIONS has to put elements
outside the bounds on the same cases.  And the bounds must stay tight enough to mean something."""
import numpy as np
import pytest

import fm_model as M
from common import data_prefixes, golden, ftrl64
from cases import CASES
from oracle import oracle as O
from test_gpu_edges import _long_batch
from xflow_b200 import datagen

SEED = 11
WIDTHS = [1, 3, 8, 10, 16, 33, 132]
SHAPES = ["ragged", "zipf1.05", "zipf1.3", "long"]
STEPS = 4


def batches(shape, seed=0, B=256, d=16, space=3000):
    """STEPS batches: uniform ragged rows; Zipf(1.05) rows of d; Zipf(1.3) ragged rows; the long-row mix of
    test_gpu_edges (every length of LONG_LENS, up to 4097 tokens, keys repeating inside and across rows)."""
    h = O.hash_decimal_ids
    if shape == "long":
        return [_long_batch(1 + s // 2, 1 << 30) for s in range(STEPS)]  # the keys of a step return in the next
    if shape == "ragged":
        return [datagen.make_csr_keys(seed + s, B, d, space, h, ragged=True) for s in range(STEPS)]
    z = float(shape[4:])
    return [datagen.make_csr_keys(seed + s, B, d, space, h, dist="zipf", zipf_s=z, ragged=(z > 1.1)) for s in range(STEPS)]


class Oracle:
    """The oracle as the implementation under test: its table, its step, and the values a new key enters with."""

    def __init__(self, K, opt, init_mode=O.INIT_COUNTER, seed=SEED, exact=False):
        self.K, self.opt, self.exact = K, opt, exact
        self.args = dict(K=K, opt=O.OPT_FTRL if opt == "ftrl" else O.OPT_SGD, init_mode=init_mode, seed=seed)
        self.t = O.Table(**self.args)

    def init_v(self, keys):
        return O.Table(**self.args).pull(keys)[1]

    def step(self, i, rp, keys, lab):
        a = (np.asarray(rp, np.int64), keys, lab.astype(np.int32))
        if self.exact:
            with O.exact_sums():
                return self.t.step(*a)[1]
        return self.t.step(*a)[1]

    def run(self, bs, on_step=None):
        return M.run_steps(self.t.export, self.step, self.init_v, bs, self.K, self.opt, on_step=on_step)


def golden_run(case, syn_data, steps=STEPS):
    """The first `steps` slices of a golden FM case's training, on an oracle table set up as the case sets it up."""
    c = CASES[case]
    o = Oracle(c["K"], c["opt"], init_mode=O.INIT_ZERO if c.get("preinit") else O.INIT_DEFAULT)
    if c.get("preinit"):
        g = golden(case)
        o.t.import_(g["keys"], w=g["init_w"], v=g["init_v"])
    train, _ = data_prefixes(case, syn_data)
    bs = []
    while len(bs) < steps:
        for rp, keys, lab in O.load_blocks(train + "-00000", c.get("block_mb", 2) << 20):
            bs.append((rp, keys, lab.astype(np.uint8)))
    return o, bs[:steps]


FM_GOLDEN = sorted(k for k, c in CASES.items() if c["model"] == "fm")


# ---------------------------------------------------------------------------------------------------------------------
# the reference lies inside the bounds
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", FM_GOLDEN)
def test_golden_cases_inside_bounds(case, syn_data):
    o, bs = golden_run(case, syn_data)
    o.run(bs)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("K", WIDTHS)
def test_oracle_inside_bounds(K, opt, shape):
    Oracle(K, opt).run(batches(shape, seed=K))


@pytest.mark.parametrize("shape", ["zipf1.3", "long"])
@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
def test_oracle_exact_sums_inside_bounds(opt, shape):
    """The oracle with its per-key sums in double (oracle.exact_sums), another legal order."""
    Oracle(16, opt, exact=True).run(batches(shape, seed=3))


# ---------------------------------------------------------------------------------------------------------------------
# the centre is the reference's algorithm
# ---------------------------------------------------------------------------------------------------------------------
def _loops64(pre, uk, rp, keys, lab, K, opt):
    """The reference's step written as its loops (fm_worker.cc:126-245: k-outer row sums, per-occurrence per-k
    gradient terms residual * (S - v_k), the w-gradient added K times, / rows; ftrl.h:59-74, sgd.h) in float64."""
    B = lab.size
    idx = {int(k): i for i, k in enumerate(uk)}
    W, V = pre["w"].astype(np.float64), pre["v"].astype(np.float64)
    loss, S = np.zeros(B), np.zeros(B)
    for r in range(B):
        toks = [idx[int(k)] for k in keys[rp[r]:rp[r + 1]]]
        wx = sum(W[i] for i in toks)
        s = q = 0.0
        for k in range(K):
            for i in toks:
                s += V[i, k]
                q += V[i, k] * V[i, k]
        S[r] = s
        loss[r] = float(M.sigmoid(wx + s * s - q)) - lab[r]
    gw, gv = np.zeros(uk.size), np.zeros((uk.size, K))
    for r in range(B):
        for k in range(K):
            for key in keys[rp[r]:rp[r + 1]]:
                i = idx[int(key)]
                gw[i] += loss[r]
                gv[i, k] += loss[r] * (S[r] - V[i, k])
    gw, gv = gw / B, gv / B
    out = {}
    if opt == "ftrl":
        out["w"], out["nw"], out["zw"] = ftrl64(gw, W, pre["nw"].astype(np.float64), pre["zw"].astype(np.float64),
                                                alpha=M.ALPHA, l1=M.L1)
        out["v"], out["nv"], out["zv"] = ftrl64(gv, V, pre["nv"].astype(np.float64), pre["zv"].astype(np.float64),
                                                alpha=M.ALPHA, l1=M.L1)
    else:
        out["w"], out["v"] = W - M.LR * gw, V - M.LR * gv
    return loss, out


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("K", [3, 10])
def test_centre_is_the_reference_loops_in_float64(K, opt):
    """The model's centre (factorised latent gradient Aq - v L, vectorised) equals the reference's loops run in float64,
    to 1e-12 relative, from a state three oracle steps in (n, z, w all nonzero).  The oracle itself rounds every stage
    to float32, so no float32 run can be compared at that precision; the oracle runs above are held to the bounds."""
    o = Oracle(K, opt)
    bs = batches("ragged", seed=40, B=48, d=6, space=200)
    o.run(bs[:3])
    rp, keys, lab = bs[3]
    uk = np.unique(keys)
    pre, _ = M.pre_state(o.t.export, o.init_v, uk, K)
    st = M.fm_step(uk, pre, rp, keys, lab, K, opt)
    loss, ref = _loops64(pre, uk, rp.astype(np.int64), keys, lab, K, opt)
    assert opt == "sgd" or ((pre["nv"] > 0).mean() > 0.5 and (pre["zw"] != 0).mean() > 0.5)
    np.testing.assert_allclose(st.loss[0], loss, rtol=1e-12, atol=1e-15)
    for f, r in ref.items():
        np.testing.assert_allclose(st.fields[f][0], r, rtol=1e-12, atol=1e-15, err_msg=f)


# ---------------------------------------------------------------------------------------------------------------------
# teeth: wrong arithmetic falls outside
# ---------------------------------------------------------------------------------------------------------------------
def applicable(perturb, K, opt, shape=None):
    """no_k_fold is the identity at K = 1; SGD has no n; and SGD's post-step v differs from v by lr * g, far below
    any float32 resolution of the gradient it feeds.  In the long-row mix at K = 132 every key also sits in a row of
    4097 tokens, whose S sums 540 804 terms: their worst-case float error (3 % of sum |v|) hides a lost occurrence and
    a gradient formed on the post-step v, while the forward and the divisor perturbations stay visible."""
    if shape == "long" and K > 64 and perturb in ("drop_hot_occurrence", "post_step_v"):
        return False
    if perturb == "no_k_fold":
        return K > 1
    if perturb in ("previous_n", "post_step_v"):
        return opt == "ftrl"
    return True


def caught_perturbations(o, bs):
    """Run the oracle over the batches; at every step model the step correctly and under each perturbation (from the
    same pre-step state), and collect the perturbations whose centres leave the correct bounds somewhere."""
    allk = np.unique(np.concatenate([b[1] for b in bs]))
    caught, prev = set(), None
    for i, (rp, keys, lab) in enumerate(bs):
        snap, _ = M.pre_state(o.t.export, o.init_v, allk, o.K)
        uk = np.unique(keys)
        at = np.searchsorted(allk, uk)
        pre = {f: snap[f][at] for f in M.FIELDS}
        loss = o.step(i, rp, keys, lab)
        post = o.t.export(uk)
        st = M.fm_step(uk, pre, rp, keys, lab, o.K, o.opt)
        M.check_step(st, loss, post, what="step %d:" % i)
        for p in M.PERTURBATIONS:
            if p in caught or not applicable(p, o.K, o.opt) or (p == "previous_n" and prev is None):
                continue
            n_prev = {f: prev[f][at] for f in ("nw", "nv")} if prev is not None else None
            bad = M.fm_step(uk, pre, rp, keys, lab, o.K, o.opt, perturb=p, n_prev=n_prev)
            l_bad, s_bad = M.centre_state(bad)
            if M.violations(st, np.float32(l_bad), {f: np.float32(s_bad[f]) for f in M.FIELDS}):
                caught.add(p)
        prev = snap
    return caught


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("K", WIDTHS)
def test_perturbations_fall_outside(K, opt, shape):
    caught = caught_perturbations(Oracle(K, opt), batches(shape, seed=K))
    want = {p for p in M.PERTURBATIONS if applicable(p, K, opt, shape)}
    assert want <= caught, "not caught: %s" % sorted(want - caught)


@pytest.mark.parametrize("case", FM_GOLDEN)
def test_perturbations_fall_outside_golden(case, syn_data):
    o, bs = golden_run(case, syn_data)
    caught = caught_perturbations(o, bs)
    want = {p for p in M.PERTURBATIONS if applicable(p, o.K, o.opt)}
    assert want <= caught, "not caught: %s" % sorted(want - caught)


# ---------------------------------------------------------------------------------------------------------------------
# tightness
# ---------------------------------------------------------------------------------------------------------------------
# The largest median half-width, relative to the value, on rows of at most 64 tokens.  The worst-case error of a float
# sum of n terms is (n - 1) u sum |terms|, and a row's S sums t K latent values of random sign, so the residual's bound
# grows like (t K)^2 u |v|^2: below 1e-5 up to K = 8, not at K = 64 (t K = 4096: about 2.4e-4 of sum |v|).
TIGHT = {1: 1e-5, 8: 1e-5, 16: 5e-5, 33: 2e-4, 64: 1e-3}


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("K", sorted(TIGHT))
def test_bounds_are_tight_on_short_rows(K, opt):
    """Rows of at most 64 tokens: the median half-width of the residuals, w and v (and z, n with FTRL) stays below
    TIGHT[K] of the value.  Bounds that accept everything fail here."""
    meds = {}

    def on_step(i, st, post, loss):
        for f in ("loss", "w", "v") + (("zw", "zv", "nv") if opt == "ftrl" else ()):
            meds.setdefault(f, []).append(M.rel_tolerance(st, f))

    bs = batches("ragged", seed=K, d=24) + batches("zipf1.05", seed=K, d=32)
    assert max(np.diff(b[0]).max() for b in bs) <= 64
    Oracle(K, opt).run(bs, on_step)
    for f, v in meds.items():
        med = float(np.median(np.concatenate(v)))
        assert med < TIGHT[K], "%s: median relative half-width %.3g" % (f, med)


def test_sigmoid_range_holds_the_clamp():
    lo, hi = M.sigmoid_range(np.array([-30.5, -31.0, 29.9]), np.array([-29.5, -30.5, 30.1]))
    assert lo[0] <= M.sigmoid(-30.0) and hi[0] >= M.P_MIN
    assert lo[1] == hi[1] == M.P_MIN
    assert hi[2] == 1.0

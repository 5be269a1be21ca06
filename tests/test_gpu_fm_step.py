"""The device's FM training step (step.cu's xf_k_step, kernels.cu's xf_k_update) against the float64 model of
tests/fm_model.py (pytest -m gpu), one step at a time from the device's own state: before each step the batch's keys
are exported from the device (keys it does not hold enter with the oracle's initial values), and after it the
residuals and the exported state (w, n, z, v, nv, zv) must lie inside the model's bounds.  The state is re-read
before every step, so errors never compound and every step is held to the same tight bounds.

The matrix: K = 1 ... 256 (VEC 1 / 2 / 4, 1 ... 32 lanes per key, and K / VEC > 32 where a lane of xf_k_update
owns several chunks), FTRL and SGD, fixed-length and ragged rows of uniform and Zipf ids; the long-row mix of
test_gpu_edges (up to 4097 tokens, a key in chunk 0 and again in chunks 2+) with FTRL; key layouts aimed at the
step's hot-key cache (placement_model: hot keys whose slots alias a few cache entries, and every entry of every CTA
claimed); an imported state with large n and partly unmaterialised latent rows; Bloom admission, eviction stamps and
sweeps, importance weights, predict; both ends of XFLOW_FM_CACHE_LOG2 in a child process; and a B = 65 536 batch in
the cfg5 shape."""
import os
import subprocess
import sys

import numpy as np
import pytest

import fm_model as M
import placement_model as P
from oracle import oracle as O
from test_gpu_edges import _long_batch
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SEED = 29
WIDTHS = [1, 2, 3, 4, 8, 10, 16, 32, 33, 64, 128, 132, 256]
STEPS = 4
CACHE_LOG2 = 9  # step.cu: XF_STEP_CACHE_LOG2, the default


def _gopt(opt):
    return api.OPT_FTRL if opt == "ftrl" else api.OPT_SGD


class Device:
    """A device table and FM trainer, run step by step against the model."""

    def __init__(self, K, opt, max_rows, max_nnz, capacity=0, seed=SEED):
        self.K, self.opt, self.seed = K, opt, seed
        self.t = api.Table(latent_dim=K, optimizer=_gopt(opt), v_init=api.VINIT_COUNTER, seed=seed, capacity=capacity)
        self.tr = api.Trainer(self.t, model=api.MODEL_FM, max_rows=max_rows, max_nnz=max_nnz, keep_loss=True)
        self.weights = None

    def init_v(self, keys):
        oopt = O.OPT_FTRL if self.opt == "ftrl" else O.OPT_SGD
        return O.Table(K=self.K, opt=oopt, init_mode=O.INIT_COUNTER, seed=self.seed).pull(keys)[1]

    def step(self, i, rp, keys, lab):
        if self.weights is None:
            self.tr.step_host(rp, keys, lab)
        else:
            self.tr.step_host_weighted(rp, keys, lab, self.weights[i])
        return self.tr.get_loss(lab.size)

    def run(self, bs, on_step=None, admitted=False):
        return M.run_steps(self.t.export, self.step, self.init_v, bs, self.K, self.opt, weights=self.weights,
                           on_step=on_step, admitted=admitted)

    def close(self):
        self.tr.close()
        self.t.close()


def _batches(dist, K, B=1024, d=16, space=20000):
    """STEPS batches; odd steps ragged (0 ... 2d - 1 tokens a row)."""
    return [datagen.make_csr_keys(100 * K + s, B, d, space, api.hash_decimal_ids, dist=dist, zipf_s=1.05,
                                  ragged=(s % 2 == 1)) for s in range(STEPS)]


def _run(K, opt, bs, **kw):
    d = Device(K, opt, max(b[2].size for b in bs), max(b[1].size for b in bs), **kw)
    try:
        return d.run(bs)
    finally:
        d.close()


# ---------------------------------------------------------------------------------------------------------------------
# widths x optimizers x id distributions; the long rows
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist", ["uniform", "zipf"])
@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("K", WIDTHS)
def test_fm_step_within_bounds(K, opt, dist):
    _run(K, opt, _batches(dist, K))


@pytest.mark.parametrize("K", WIDTHS)
def test_fm_long_rows_within_bounds(K):
    """FTRL on rows of every length in LONG_LENS up to 4097 tokens: from 129 tokens on, phase B re-probes the slots
    of chunks 2+; a key sits in chunk 0 and again in chunks 2+ of the same row."""
    _run(K, "ftrl", [_long_batch(1 + s // 2, 1 << 30) for s in range(STEPS)])


# ---------------------------------------------------------------------------------------------------------------------
# the hot-key cache
# ---------------------------------------------------------------------------------------------------------------------
LOG2CAP = 18


def cache_entry(slot, log2nc=CACHE_LOG2):
    """step.cu: the hot-key cache entry of a slot."""
    return ((np.asarray(slot, np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - log2nc)


def key_at(slot, log2cap, bshift):
    """A key whose home slot is `slot` (placement_model's inversion of xf_probe_slot's multiplier)."""
    hb, j0 = slot >> bshift, slot & ((1 << bshift) - 1)
    return np.uint64(P.key_of((hb << (64 - (log2cap - bshift))) | (j0 << 9) | 1))


def cache_layout(layout, K, opt, seed):
    """Keys at chosen slots of a 2^LOG2CAP table, and STEPS batches of them.
    alias: 640 hot keys whose slots map to 4 cache entries; rows of 32 of them (Zipf-weighted), so in every CTA one key
           per entry claims it and the others' tokens take the global atomics.
    claim_all: 3 keys per cache entry; the 8 rows of a CTA (64 tokens each; 512 rows make 64 CTAs of one row per warp)
           cover all 512 entries, so every entry of every CTA is claimed and flushed.
    The table must not grow (a step reserves room for its token count): 2^18 slots hold either."""
    bshift = P.bucket_log2(P.row_stride(K, opt == "ftrl"), LOG2CAP)
    slots = np.arange(1, 1 << LOG2CAP, dtype=np.uint64)
    ent = cache_entry(slots)
    rng = np.random.default_rng(seed)
    bs = []
    if layout == "alias":
        pick = np.concatenate([slots[ent == e][:160] for e in (3, 77, 300, 511)])
        keys = np.array([key_at(int(s), LOG2CAP, bshift) for s in pick], np.uint64)
        p = 1.0 / np.arange(1, keys.size + 1) ** 0.8
        p /= p.sum()
        for s in range(STEPS):
            B, d = 2048, 32
            toks = keys[rng.choice(keys.size, (B, d), p=p)]
            bs.append(((np.arange(B + 1) * d).astype(np.uint32), toks.reshape(-1), rng.integers(0, 2, B).astype(np.uint8)))
    else:
        per = [slots[ent == e][rng.choice(200, 3, replace=False)] for e in range(1 << CACHE_LOG2)]
        keys = np.array([[key_at(int(s), LOG2CAP, bshift) for s in row] for row in per], np.uint64)  # [512, 3]
        for s in range(STEPS):
            B, d = 512, 64
            rows = []
            for r in range(B):
                e = (r % 8) * 64 + rng.permutation(64)
                rows.append(keys[e, rng.integers(0, 3, 64)])
            bs.append(((np.arange(B + 1) * d).astype(np.uint32), np.concatenate(rows), rng.integers(0, 2, B).astype(np.uint8)))
    return bs


@pytest.mark.parametrize("layout", ["alias", "claim_all"])
@pytest.mark.parametrize("K,opt", [(1, "ftrl"), (4, "sgd"), (16, "ftrl"), (33, "sgd"), (132, "ftrl")])
def test_fm_hot_key_cache_layouts_within_bounds(K, opt, layout):
    bs = cache_layout(layout, K, opt, seed=K)
    d = Device(K, opt, max(b[2].size for b in bs), max(b[1].size for b in bs), capacity=1 << LOG2CAP)
    try:
        assert d.t.capacity() == 1 << LOG2CAP
        d.run(bs)
        assert d.t.capacity() == 1 << LOG2CAP  # no growth: the keys stayed at the slots they were built for
    finally:
        d.close()


# ---------------------------------------------------------------------------------------------------------------------
# imported state, admission, eviction, weights, predict
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("K", [8, 33, 132])
def test_fm_imported_state_within_bounds(K, opt):
    """Half of the keys start from an imported state with large n (so FTRL's sigma = (sqrt(n') - sqrt(n)) / alpha is
    not 0 on the first step) and nonzero w and z; half of those have no latent row materialised (the import sets only
    w, n, z), the other half a full imported latent state.  The rest are absent."""
    bs = _batches("zipf", K, B=1024, d=16, space=6000)
    rng = np.random.default_rng(K)
    allk = np.unique(np.concatenate([b[1] for b in bs]))
    imp = allk[rng.random(allk.size) < 0.5]
    mat = imp[rng.random(imp.size) < 0.5]
    head = imp[~np.isin(imp, mat)]
    d = Device(K, opt, 2048, 2048 * 32)
    try:
        n = imp.size

        def f32(x):
            return np.asarray(x, np.float32)

        w, nw, zw = f32(rng.normal(0, 0.05, n)), f32(rng.uniform(10, 1000, n)), f32(rng.normal(0, 0.5, n))
        at = np.searchsorted(imp, head)
        d.t.import_(head, w=w[at], nw=nw[at], zw=zw[at])
        at = np.searchsorted(imp, mat)
        m = mat.size
        d.t.import_(mat, w=w[at], nw=nw[at], zw=zw[at], v=f32(rng.normal(0, 0.02, (m, K))),
                    nv=f32(rng.uniform(10, 1000, (m, K))), zv=f32(rng.normal(0, 0.5, (m, K))))
        steps = d.run(bs)
        assert steps[0].touched[np.searchsorted(steps[0].uk, imp[np.isin(imp, steps[0].uk)])].any()
    finally:
        d.close()


def test_fm_bloom_admission_within_bounds():
    """Bloom admission: a key enters only once it has been counted twice; rejected tokens read as zero and are left
    out of the model (a key absent before and after a step was rejected)."""
    K = 16
    bs = _batches("zipf", K, B=1024, d=16, space=6000)
    d = Device(K, "ftrl", 1024, 1024 * 32)
    try:
        d.t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=14, hashes=3, decay_batches=0, seed=5)
        steps = d.run(bs, admitted=True)
        assert d.t.admission_stats()["rejected_tokens"] > 0
        assert len(steps) == STEPS
    finally:
        d.close()


def test_fm_eviction_within_bounds():
    """Eviction stamps on, and a sweep after every step that drops keys idle for 1 batch: they come back as new keys."""
    K = 10
    bs = _batches("uniform", K, B=1024, d=16, space=4000)
    d = Device(K, "ftrl", 1024, 1024 * 32)
    try:
        d.t.set_eviction(max_idle_batches=1)
        dropped = []
        d.run(bs, lambda i, st, post, loss: dropped.append(d.t.evict()))
        assert sum(dropped) > 0
    finally:
        d.close()


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
def test_fm_weighted_within_bounds(opt):
    """Random row weights, a fifth of them exactly 0: the gradients use e_r x residual, the divisor stays B, and a row
    of weight 0 trains nothing and reports a residual of 0."""
    K = 16
    bs = _batches("zipf", K, B=1024, d=16, space=6000)
    rng = np.random.default_rng(3)
    d = Device(K, opt, 1024, 1024 * 32)
    try:
        d.weights = []
        for b in bs:
            w = rng.uniform(0, 3, b[2].size).astype(np.float32)
            w[rng.random(w.size) < 0.2] = 0.0
            d.weights.append(w)
        d.run(bs)
    finally:
        d.close()


def test_fm_predict_within_bounds():
    """Predict (the step kernel's mode 1) against the model's forward pass, after training steps, on rows with keys the
    table holds and keys it does not."""
    K = 16
    bs = _batches("zipf", K, B=1024, d=16, space=6000)
    d = Device(K, "ftrl", 1024, 1024 * 32)
    try:
        d.run(bs[:3])
        rp, keys, _ = datagen.make_csr_keys(7, 1024, 16, 12000, api.hash_decimal_ids, dist="zipf", ragged=True)
        uk = np.unique(keys)
        pre, _ = M.pre_state(d.t.export, d.init_v, uk, K)
        st = M.fm_step(uk, pre, rp, keys, np.zeros(rp.size - 1, np.uint8), K, "ftrl")
        M.check_step(st, pctr=d.tr.predict_host(rp, keys), what="predict:")
    finally:
        d.close()


# ---------------------------------------------------------------------------------------------------------------------
# XFLOW_FM_CACHE_LOG2 (read once per process) and the full batch size
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log2", ["0", "10"])
def test_fm_cache_size_setting_within_bounds(log2, tmp_path):
    """A zipf case, the long rows and both cache layouts, in a child process with the setting at both ends."""
    r = subprocess.run([sys.executable, os.path.join(HERE, "edge_child.py"), "fm_bounds", str(tmp_path / "out.npz")],
                       env=dict(os.environ, XFLOW_FM_CACHE_LOG2=log2), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr


def cache_setting_cases():
    """What the child runs (edge_child.py fm_bounds)."""
    _run(16, "ftrl", _batches("zipf", 16))
    _run(33, "sgd", _batches("zipf", 33))
    _run(8, "ftrl", [_long_batch(1 + s // 2, 1 << 30) for s in range(STEPS)])
    for layout in ("alias", "claim_all"):
        bs = cache_layout(layout, 16, "ftrl", seed=1)
        _run(16, "ftrl", bs, capacity=1 << LOG2CAP)


def test_fm_full_batch_cfg5_shape_within_bounds():
    """B = 65 536 rows of 64 Zipf(1.05) ids over 1e8 (the cfg5 shape), K = 16, FTRL: steps 1 to 3."""
    B, d, K = 65536, 64, 16
    bs = [datagen.make_csr_keys(40 + s, B, d, 10 ** 8, api.hash_decimal_ids, dist="zipf") for s in range(3)]
    dev = Device(K, "ftrl", B, B * d, capacity=1 << 23)
    try:
        dev.run(bs)
    finally:
        dev.close()

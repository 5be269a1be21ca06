"""AdaGrad tables (XF_OPTIMIZER_ADAGRAD, include/xflow_b200.h section 2) on the device: the optimizer alone bit for bit
against the numpy float32 statement (tests/adagrad_model.py) on every row layout, training against the oracle's
gradients, the lazy LR step against the eager one, exact resume, serving, the table features, and the refusals."""
import os

import numpy as np
import pytest

import adagrad_model as A
import deterministic_model as DM
from common import assert_close, bits_equal
from ffm_model import FFM64
from oracle import oracle as O
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

LR, BETA = A.LR, 1.0
HP = dict(learning_rate=LR, beta=BETA)


def _table(monkeypatch, K=0, eager=False, canonical=False, ring=None, **kw):
    if eager:
        monkeypatch.setenv("XFLOW_EAGER", "1")
    else:
        monkeypatch.delenv("XFLOW_EAGER", raising=False)
    if ring is None:
        monkeypatch.delenv("XFLOW_SEQ_RING", raising=False)
    else:
        monkeypatch.setenv("XFLOW_SEQ_RING", str(ring))
    args = dict(HP, v_init=api.VINIT_COUNTER, seed=5, capacity=1 << 15)
    args.update(kw)
    return api.Table(latent_dim=K, optimizer=api.OPT_ADAGRAD, canonical_fm=1 if canonical else 0, **args)


def _grads(rng, shape):
    """Random gradients with zeros, subnormals and large values."""
    g = (rng.standard_normal(shape) * 10.0 ** rng.integers(-5, 2, shape)).astype(np.float32)
    flat = g.reshape(-1)
    flat[::9] = 0.0
    flat[1::17] = np.float32(2e-39)
    flat[2::23] = np.float32(-7e-41)
    flat[3::29] = np.float32(3e3)
    return g


def _keys(n, seed=0):
    return np.unique(api.hash_decimal_ids(np.arange(seed, seed + n, dtype=np.uint64)))


def _bits_equal(a, b, what):
    assert bits_equal(a, b), "%s: %d elements differ" % (what, int((np.asarray(a, np.float32).view(np.uint32) !=
                                                                    np.asarray(b, np.float32).view(np.uint32)).sum()))


# ---- 1. the optimizer alone, exact ------------------------------------------------------------------------------------
CASES = [("lr_lazy", 0, False, False), ("lr_eager", 0, True, False)] + [("fm", K, False, False) for K in (4, 10, 16)] + \
        [("canonical", K, False, True) for K in (4, 8, 16, 32, 64, 128)]


@pytest.mark.parametrize("name,K,eager,canonical", CASES)
def test_push_equals_the_float32_statement(monkeypatch, name, K, eager, canonical):
    t = _table(monkeypatch, K, eager, canonical)
    keys = _keys(3000)
    rng = np.random.default_rng(K + 7 * eager)
    e0 = t.export(keys)
    assert not e0["present"].any()
    w, n = np.zeros(keys.size, np.float32), np.zeros(keys.size, np.float32)
    v = t.pull(keys)[1]  # inserts the keys; FM: their initial latent rows
    nv = np.zeros((keys.size, K), np.float32) if K else None
    for r in range(5):
        sub = np.sort(rng.choice(keys.size, keys.size * 2 // 3, replace=False))
        gw = _grads(rng, sub.size)
        gv = _grads(rng, (sub.size, K)) if K else None
        t.push(keys[sub], gw=gw, gv=gv)
        w[sub], n[sub] = A.step32(gw, w[sub], n[sub], LR, BETA)
        if K:
            v[sub], nv[sub] = A.step32(gv, v[sub], nv[sub], LR, BETA)
        e = t.export(keys)
        _bits_equal(e["w"], w, "push %d w" % r)
        _bits_equal(e["nw"], n, "push %d nw" % r)
        assert not e["zw"].any()
        if K:
            _bits_equal(e["v"], v, "push %d v" % r)
            _bits_equal(e["nv"], nv, "push %d nv" % r)
            assert not e["zv"].any()
    # the row is what xf_row_stride says: v, the two accumulators, nv (and A on canonical tables), no zv
    expect = 32 if K == 0 else (((32 + 4 * K + 15) & ~15) + 16 + 4 * K * (2 if canonical else 1) + 31) & ~31
    assert t.row_bytes() == expect
    t.close()


def test_row_sizes():
    for K, canon, ftrl, ada, sgd in ((16, 0, 256, 192, 128), (128, 1, 2112, 1600, 1088)):
        got = []
        for opt in (api.OPT_FTRL, api.OPT_ADAGRAD, api.OPT_SGD):
            t = api.Table(latent_dim=K, optimizer=opt, canonical_fm=canon, capacity=1024)
            got.append(t.row_bytes())
            t.close()
        assert got == [ftrl, ada, sgd]


# ---- 2. training ------------------------------------------------------------------------------------------------------
def _oracle_run(t, tr, K, batches):
    """Train the device and, beside it, the oracle's gradients from the model's own values followed by step32.
    Returns (keys, model state, device export)."""
    state = {}
    for rp, keys, lab in batches:
        uk = np.unique(keys)
        new = np.array([int(k) not in state for k in uk])
        if K and new.any():  # the initial latent rows, as the table gives a key on insert
            t0 = api.Table(latent_dim=K, optimizer=api.OPT_ADAGRAD, v_init=api.VINIT_COUNTER, seed=5, capacity=1 << 15,
                           **HP)
            _, vin = t0.pull(uk[new])
            t0.close()
            for k, row in zip(uk[new], vin):
                state[int(k)] = [np.float32(0), np.float32(0), row.copy(), np.zeros(K, np.float32)]
        for k in uk[new]:
            state.setdefault(int(k), [np.float32(0), np.float32(0), None, None])
        w = np.array([state[int(k)][0] for k in uk], np.float32)
        n = np.array([state[int(k)][1] for k in uk], np.float32)
        v = np.stack([state[int(k)][2] for k in uk]) if K else None
        nv = np.stack([state[int(k)][3] for k in uk]) if K else None
        gw, gv, _ = O.worker_compute_given(K, rp.astype(np.int64), keys, lab.astype(np.int32), w, v)
        w2, n2 = A.step32(gw, w, n, LR, BETA)
        if K:
            v2, nv2 = A.step32(gv, v, nv, LR, BETA)
        for i, k in enumerate(uk):
            state[int(k)] = [w2[i], n2[i], v2[i] if K else None, nv2[i] if K else None]
        tr.step_host(rp, keys, lab)
    keys = np.array(sorted(state), np.uint64)
    return keys, state, t.export(keys)


@pytest.mark.parametrize("K,dist", [(0, "uniform"), (0, "zipf"), (8, "uniform"), (8, "zipf")])
def test_training_matches_the_oracle(monkeypatch, K, dist):
    t = _table(monkeypatch, K)
    tr = api.Trainer(t, model=api.MODEL_FM if K else api.MODEL_LR, max_rows=1024, max_nnz=1024 * 16)
    batches = []
    for i in range(4):
        rp, keys, lab = datagen.make_csr_keys(40 + i, 1024, 16, 50000, api.hash_decimal_ids, dist=dist)
        batches.append((rp, keys, lab))
    keys, state, e = _oracle_run(t, tr, K, batches)
    w = np.array([state[int(k)][0] for k in keys], np.float32)
    n = np.array([state[int(k)][1] for k in keys], np.float32)
    assert e["present"].all()
    # Zipf keys: a hot key's gradient is a long sum whose order differs between the device and the oracle
    frac = 0.0 if dist == "uniform" else 2e-3
    assert_close(e["w"], w, "w", max_bad_frac=frac)
    assert_close(e["nw"], n, "nw", max_bad_frac=frac)
    if K:
        v = np.stack([state[int(k)][2] for k in keys])
        nv = np.stack([state[int(k)][3] for k in keys])
        assert_close(e["v"], v, "v", max_bad_frac=frac)
        assert_close(e["nv"], nv, "nv", max_bad_frac=frac)
    tr.close()
    t.close()


@pytest.mark.parametrize("mvm", [False, True])
def test_deterministic_canonical_exact(monkeypatch, mvm):
    """Deterministic canonical FM and MVM steps on one-token rows that repeat four keys hundreds of times (and a tail of
    single keys): every step's table equals deterministic_model's per-key sums of the device's residuals, divided by
    the rows as xf_k_update divides them, followed by step32, bit for bit."""
    K, B = 8, 1024
    t = _table(monkeypatch, K, canonical=True)
    tr = api.Trainer(t, model=api.MODEL_MVM if mvm else api.MODEL_FM_CANONICAL, max_rows=B, max_nnz=B, keep_loss=True)
    tr.set_deterministic(True)
    rng = np.random.default_rng(14 + mvm)
    ids = np.where(rng.random(B) < 0.8, rng.integers(0, 4, B), rng.integers(100, 100000, B)).astype(np.uint64)
    keys = api.hash_decimal_ids(ids)
    uk = np.unique(keys)
    pos = np.searchsorted(uk, keys)
    t.pull(uk)
    v0 = (rng.normal(0, 1, (uk.size, K)) * 2.0 ** rng.integers(-12, 4, (uk.size, 1))).astype(np.float32)
    t.import_(uk, w=rng.normal(0, 0.1, uk.size).astype(np.float32), v=v0)
    rp = np.arange(B + 1, dtype=np.uint32)
    for step in range(3):
        x = rng.uniform(-2.0, 2.0, B).astype(np.float32)
        lab = (rng.random(B) < 0.5).astype(np.uint8)
        fields = rng.integers(0, 5, B).astype(np.uint8)
        before = t.export(uk)
        if mvm:
            tr.step_host_fields(rp, keys, fields, x, lab)
        else:
            tr.step_host_values(rp, keys, x, lab)
        r = tr.get_loss(B)
        after = t.export(uk)
        V = before["v"][pos].astype(np.float32)
        if mvm:  # o_k = 1: a one-token row has no other field
            sums = DM.sums_by_key(keys, ((r * x)[:, None] * np.ones((1, K), np.float32)).astype(np.float32))
        else:
            S = np.float32(0.0) + V * x[:, None]  # the row's S_k: its one token's v_k x from +0
            sums = DM.sums_by_key(keys, *DM.fmc_terms(r, x, S))
        for i, k in enumerate(uk):
            Ak, G, L2 = sums[int(k)]
            vb = before["v"][i].astype(np.float32)
            gv = np.array([np.float32(np.float64(np.float32(DM._fma(-vk, L2, ak))) / B) for vk, ak in zip(vb, Ak)],
                          np.float32)
            v2, nv2 = A.step32(gv, vb, before["nv"][i], LR, BETA)
            if mvm:  # the machine has no w: it stays as it was
                w2, n2 = before["w"][i], before["nw"][i]
            else:
                w2, n2 = A.step32(np.float32(np.float64(np.float32(G)) / B), before["w"][i], before["nw"][i], LR, BETA)
            for f, want in (("w", w2), ("nw", n2), ("v", v2), ("nv", nv2)):
                _bits_equal(after[f][i], want, "step %d key %d %s" % (step, i, f))
    tr.close()
    t.close()


def test_ffm_within_the_bounds(monkeypatch):
    """Field-aware FM steps on batches in which no key repeats (keys recur across batches, so n grows): the gradients
    of ffm_model.FFM64 from the device's residuals, with a bound on the device's float32 sums, then step64."""
    L, B = 16, 384
    F = L // 4
    rng = np.random.default_rng(21)
    pool = api.hash_decimal_ids(np.arange(1, 6001, dtype=np.uint64))
    t = _table(monkeypatch, L, canonical=True)
    tr = api.Trainer(t, model=api.MODEL_FFM, max_rows=B, max_nnz=B * 14, keep_loss=True)
    t.import_(np.sort(pool), w=rng.normal(0, 0.2, pool.size).astype(np.float32),
              v=rng.normal(0, 0.12, (pool.size, L)).astype(np.float32))
    for step in range(3):
        lens = rng.integers(1, 14, B)
        rp = np.zeros(B + 1, np.uint32)
        rp[1:] = np.cumsum(lens)
        n = int(rp[-1])
        keys = pool[rng.permutation(pool.size)[:n]]
        fields = rng.integers(0, F, n).astype(np.uint8)
        x = rng.uniform(0.25, 1.75, n).astype(np.float32)
        x[::5] *= -1.0
        lab = (rng.random(B) < 0.35).astype(np.uint8)
        uk = np.unique(keys)
        assert uk.size == n
        before = t.export(uk)
        tr.step_host_fields(rp, keys, fields, x, lab)
        r = tr.get_loss(B).astype(np.float64)
        after = t.export(uk)
        idx = np.searchsorted(uk, keys)
        gw, gv = FFM64(before["w"], before["v"], "sgd").gradients(idx, rp, fields, x, r)
        # magnitudes: the same sums over |terms|, plus each token's own piece (which the device may add and take away)
        aw, av = FFM64(np.abs(before["w"]), np.abs(before["v"]), "sgd").gradients(idx, rp, fields, np.abs(x), np.abs(r))
        own = np.abs(r[np.repeat(np.arange(B), lens)]) * x.astype(np.float64) ** 2
        av = av.reshape(n, F, 4)
        av[idx, fields] += own[:, None] * np.abs(before["v"][idx].reshape(n, F, 4)[np.arange(n), fields])
        c = 2.0 * (lens.max() + 4) * A.U
        bw = A.step64(gw / B, c * aw / B, before["w"], before["nw"])
        bv = A.step64(gv / B, c * av.reshape(n, L) / B, before["v"], before["nv"])
        for f, b, key in (("w", bw, "w"), ("nw", bw, "n"), ("v", bv, "w"), ("nv", bv, "n")):
            _, lo, hi = b[key]
            got = after[f].astype(np.float64)
            bad = ~((got >= lo) & (got <= hi))
            assert not bad.any(), "step %d %s: %d outside the bounds" % (step, f, int(bad.sum()))
        moved = np.abs(after["v"].astype(np.float64) - before["v"]).max()
        assert moved > 1e-6, moved
    tr.close()
    t.close()


# ---- 3. the lazy LR step equals the eager one -------------------------------------------------------------------------
@pytest.mark.parametrize("ring", [None, 5])
def test_lazy_equals_eager(monkeypatch, ring):
    lazy = _table(monkeypatch, ring=ring)
    eager = _table(monkeypatch, eager=True)
    trs = [api.Trainer(t, model=api.MODEL_LR, max_rows=512, max_nnz=512 * 8) for t in (lazy, eager)]
    seen = []
    for i in range(12):
        rp, keys, lab = datagen.make_csr_keys(70 + i, 512, 8, 5000, api.hash_decimal_ids, dist="zipf")
        seen.append(keys)
        for tr in trs:
            tr.step_host(rp, keys, lab)
        uk = np.unique(np.concatenate(seen))
        a, b = lazy.export(uk), eager.export(uk)
        for f in ("w", "nw", "zw"):
            _bits_equal(a[f], b[f], "batch %d %s" % (i, f))
    for tr in trs:
        tr.close()
    lazy.close()
    eager.close()


# ---- 4. resume --------------------------------------------------------------------------------------------------------
def _resume_batches(model, i):
    canonical = model == api.MODEL_FM_CANONICAL
    rng = np.random.default_rng(300 + i)
    if canonical:  # every key once per batch: comparable bit for bit even without the deterministic mode
        ids = rng.permutation(20000)[:512 * 8].astype(np.uint64)
        rp = np.arange(513, dtype=np.uint32) * 8
        lab = (rng.random(512) < 0.3).astype(np.uint8)
    else:
        rp, ids, lab = datagen.make_ids(300 + i, 512, 8, 20000, dist="zipf")
    return rp, api.hash_decimal_ids(np.asarray(ids, np.uint64)), lab, rng.uniform(0.5, 1.5, ids.size).astype(np.float32)


def _resume_run(monkeypatch, K, model, steps, save_at=None, load=None, path=None):
    t = _table(monkeypatch, K, canonical=model == api.MODEL_FM_CANONICAL)
    if load:
        t.load_state(load)
    tr = api.Trainer(t, model=model, max_rows=512, max_nnz=512 * 8)
    if model == api.MODEL_FM_CANONICAL:
        tr.set_deterministic(True)
    for i in steps:
        rp, keys, lab, vals = _resume_batches(model, i)
        if model == api.MODEL_FM_CANONICAL:
            tr.step_host_values(rp, keys, vals, lab)
        else:
            tr.step_host(rp, keys, lab)
        if save_at == i:
            t.save_state(path)
    keys = np.sort(t.list_keys())
    e = t.export(keys)
    tr.close()
    t.close()
    return keys, e


@pytest.mark.parametrize("K,model", [(0, api.MODEL_LR), (8, api.MODEL_FM), (8, api.MODEL_FM_CANONICAL)])
def test_resume_is_exact(monkeypatch, tmp_path, K, model):
    path = str(tmp_path / "state.xfst")
    k0, e0 = _resume_run(monkeypatch, K, model, range(8), save_at=3, path=path)
    k1, e1 = _resume_run(monkeypatch, K, model, range(4, 8), load=path)
    assert np.array_equal(k0, k1)
    for f in ("w", "nw", "zw", "v", "nv", "zv"):
        _bits_equal(e0[f], e1[f], f)


def test_image_refused_by_another_optimizer(monkeypatch, tmp_path):
    path = str(tmp_path / "state.xfst")
    _resume_run(monkeypatch, 0, api.MODEL_LR, range(2), save_at=1, path=path)
    t = api.Table(optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=5, capacity=1 << 15)
    with pytest.raises(api.XflowError, match="optimizer"):
        t.load_state(path)
    assert t.size() == 0
    t.close()


@pytest.mark.parametrize("K", [0, 10])
def test_xftb_round_trip(monkeypatch, tmp_path, K):
    t = _table(monkeypatch, K)
    keys = _keys(2000)
    rng = np.random.default_rng(3)
    t.pull(keys)
    for _ in range(3):
        t.push(keys, gw=_grads(rng, keys.size), gv=_grads(rng, (keys.size, K)) if K else None)
    path = str(tmp_path / "t.xftb")
    t.save(path)
    u = _table(monkeypatch, K, v_init=api.VINIT_ZERO)
    u.load(path)
    a, b = t.export(keys), u.export(keys)
    for f in ("w", "nw", "zw", "v", "nv", "zv", "present"):
        assert np.array_equal(np.asarray(a[f]), np.asarray(b[f])), f
    # and both go on alike
    g = _grads(rng, keys.size)
    for x in (t, u):
        x.push(keys, gw=g)
    _bits_equal(t.export(keys)["w"], u.export(keys)["w"], "after a push")
    t.close()
    u.close()


@pytest.mark.parametrize("K,eager", [(0, False), (0, True), (8, False)])
def test_import_ignores_z(monkeypatch, K, eager):
    """An import with FTRL's z fields (an FTRL-written file, say) keeps w, n, v and nv and drops zw and zv."""
    t = _table(monkeypatch, K, eager)
    keys = _keys(500)
    rng = np.random.default_rng(8)
    f = {"w": rng.normal(0, 0.3, keys.size), "nw": rng.uniform(0.5, 2, keys.size), "zw": rng.normal(0, 1, keys.size)}
    if K:
        f.update(v=rng.normal(0, 0.3, (keys.size, K)), nv=rng.uniform(0.5, 2, (keys.size, K)),
                 zv=rng.normal(0, 1, (keys.size, K)))
    f = {k: np.asarray(a, np.float32) for k, a in f.items()}
    t.import_(keys, **f)
    e = t.export(keys)
    for name in ("w", "nw") + (("v", "nv") if K else ()):
        _bits_equal(e[name], f[name], name)
    assert not e["zw"].any() and not e["zv"].any()
    t.close()


# ---- 5. serving -------------------------------------------------------------------------------------------------------
def _serving_table(monkeypatch, kind, seed):
    K = {"lr": 0, "fm": 8, "canonical": 8, "mvm": 8, "ffm": 16}[kind]
    model = {"lr": api.MODEL_LR, "fm": api.MODEL_FM, "canonical": api.MODEL_FM_CANONICAL, "mvm": api.MODEL_MVM,
             "ffm": api.MODEL_FFM}[kind]
    t = _table(monkeypatch, K, canonical=kind in ("canonical", "mvm", "ffm"))
    tr = api.Trainer(t, model=model, max_rows=512, max_nnz=512 * 8)
    if kind == "mvm":
        tr.set_deterministic(True)
    F = 3 if kind != "ffm" else K // 4
    for i in range(seed, seed + 3):
        rp, keys, lab, vals = _resume_batches(api.MODEL_FM_CANONICAL, i)
        fields = (np.arange(keys.size) % F).astype(np.uint8)
        if kind in ("lr", "fm"):
            tr.step_host(rp, keys, lab)
        elif kind == "canonical":
            tr.step_host_values(rp, keys, vals, lab)
        else:
            tr.step_host_fields(rp, keys, fields, vals, lab)
    return t, tr, F


def _freeze(t, kind):
    return {"lr": t.freeze, "fm": t.freeze, "canonical": t.freeze_canonical, "mvm": t.freeze_mvm,
            "ffm": t.freeze_ffm}[kind]()


def _predict_both(tr, m, kind, F):
    rp, keys, _, vals = _resume_batches(api.MODEL_FM_CANONICAL, 99)
    keys = keys[:2048]
    rp = rp[rp <= 2048]
    vals = vals[:2048]
    fields = (np.arange(keys.size) % F).astype(np.uint8)
    if kind in ("lr", "fm"):
        return tr.predict_host(rp, keys), m.predict_host(rp, keys)
    if kind == "canonical":
        return tr.predict_host_values(rp, keys, vals), m.predict_host(rp, keys, vals)
    return tr.predict_host_fields(rp, keys, fields, vals), m.predict_host_fields(rp, keys, fields, vals)


@pytest.mark.parametrize("kind", ["lr", "fm", "canonical", "mvm", "ffm"])
def test_serving(monkeypatch, tmp_path, kind):
    t, tr, F = _serving_table(monkeypatch, kind, 0)
    m = _freeze(t, kind)
    got_t, got_m = _predict_both(tr, m, kind, F)
    _bits_equal(got_m, got_t, "predict")
    assert m.info()["optimizer"] == api.OPT_ADAGRAD
    path = str(tmp_path / "m.xfsm")
    m.save(path)
    m2 = api.Model.load(path)
    assert m2.info()["optimizer"] == api.OPT_ADAGRAD
    assert m2.fingerprint() == m.fingerprint()
    # a delta between two AdaGrad models of the same table
    rp, keys, lab, vals = _resume_batches(api.MODEL_FM_CANONICAL, 50)
    if kind in ("lr", "fm"):
        tr.step_host(rp, keys, lab)
    elif kind == "canonical":
        tr.step_host_values(rp, keys, vals, lab)
    else:
        tr.step_host_fields(rp, keys, (np.arange(keys.size) % F).astype(np.uint8), vals, lab)
    nxt = _freeze(t, kind)
    d = m.diff(nxt)
    rebuilt = m.apply(d)
    assert rebuilt.fingerprint() == nxt.fingerprint()
    p1, p2 = _predict_both(tr, rebuilt, kind, F)
    _bits_equal(p2, p1, "predict after the delta")
    tr.close()
    t.close()


# ---- 6. features on AdaGrad tables -------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [0, 8])
def test_features(monkeypatch, K):
    model = api.MODEL_FM if K else api.MODEL_LR
    # admission and eviction run, and keep what they keep
    t = _table(monkeypatch, K)
    t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=12, hashes=3, seed=5)
    t.set_eviction(max_idle_batches=2, max_keys=3000)
    tr = api.Trainer(t, model=model, max_rows=512, max_nnz=512 * 8)
    pv = api.ProgressiveValidation()
    tr.set_validation(pv)
    for i in range(6):
        rp, keys, lab = datagen.make_csr_keys(90 + i, 512, 8, 20000, api.hash_decimal_ids, dist="zipf")
        tr.step_host(rp, keys, lab)
        if i % 2:
            t.evict()
    assert t.admission_stats()["rejected_tokens"] > 0
    assert 0 < t.size() <= 3000
    assert pv.report()["rows"] == 6 * 512
    keys = np.sort(t.list_keys())
    e = t.export(keys)
    assert np.all(np.isfinite(e["w"])) and np.all(e["nw"] >= 0)
    tr.close()
    t.close()
    # weights of 1 equal the plain step bit for bit
    outs = []
    for weighted in (False, True):
        t = _table(monkeypatch, K)
        tr = api.Trainer(t, model=model, max_rows=512, max_nnz=512 * 8)
        for i in range(4):
            rp, keys, lab = datagen.make_csr_keys(120 + i, 512, 8, 20000, api.hash_decimal_ids, dist="zipf")
            if weighted:
                tr.step_host_weighted(rp, keys, lab, np.ones(512, np.float32))
            else:
                tr.step_host(rp, keys, lab)
        keys = np.sort(t.list_keys())
        outs.append((keys, t.export(keys)))
        tr.close()
        t.close()
    assert np.array_equal(outs[0][0], outs[1][0])
    for f in ("w", "nw", "v", "nv"):
        _bits_equal(outs[0][1][f], outs[1][1][f], "weighted " + f)


# ---- 7. sharded ------------------------------------------------------------------------------------------------------
ROUNDS = 3


def _shard_batch(rank, rnd):
    return datagen.make_csr_keys(600 + 10 * rnd + rank, 2048, 16, 100000, api.hash_decimal_ids)


def _shard_worker(rank, world, id_path, K, ret):
    from xflow_b200 import api as X
    if rank == 0:
        cid = X.Comm.new_id()
        np.save(id_path + ".tmp.npy", cid)
        os.replace(id_path + ".tmp.npy", id_path)
    else:
        import time
        while not os.path.exists(id_path):
            time.sleep(0.05)
        cid = np.load(id_path)
    comm = X.Comm(cid, rank, world, rank)
    table = X.Table(latent_dim=K, optimizer=X.OPT_ADAGRAD, device=rank, v_init=X.VINIT_COUNTER, seed=9,
                    shard_index=rank, num_shards=world, capacity=1 << 17, **HP)
    tr = X.Trainer(table, model=X.MODEL_FM if K else X.MODEL_LR, max_rows=2048, max_nnz=2048 * 16, comm=comm)
    for rnd in range(ROUNDS):
        rp, keys, lab = _shard_batch(rank, rnd)
        tr.step_host(rp, keys, lab)
    tr.sync()
    comm.barrier()
    allk = np.unique(np.concatenate([_shard_batch(r, rnd)[1] for r in range(world) for rnd in range(ROUNDS)]))
    mine = np.array([X.shard_of(int(k), world) == rank for k in allk])
    ret[rank] = dict(keys=allk[mine], e=table.export(allk[mine]))
    comm.barrier()
    tr.close()
    table.close()
    comm.close()


@pytest.mark.parametrize("K", [0, 8])
def test_sharded_equals_single_table(K, tmp_path):
    """Two ranks training on the range-sharded table equal one table driven in the sharded step's lock-step schedule:
    every rank pulls and computes its gradients (the oracle's, from the pulled values) before any push of the round,
    and the pushes land in rank order."""
    world = 2
    if api.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    import torch.multiprocessing as mp
    ret = mp.Manager().dict()
    mp.spawn(_shard_worker, args=(world, str(tmp_path / "ncclid.npy"), K, ret), nprocs=world, join=True)
    ref = api.Table(latent_dim=K, optimizer=api.OPT_ADAGRAD, v_init=api.VINIT_COUNTER, seed=9, capacity=1 << 18, **HP)
    for rnd in range(ROUNDS):
        pend = []
        for r in range(world):
            rp, keys, lab = _shard_batch(r, rnd)
            uk = np.unique(keys)
            w, v = ref.pull(uk)
            gw, gv, _ = O.worker_compute_given(K, rp.astype(np.int64), keys, lab.astype(np.int32), w, v if K else None)
            pend.append((uk, gw, gv))
        for uk, gw, gv in pend:
            ref.push(uk, gw=gw, gv=gv if K else None)
    for r in range(world):
        got = ret[r]
        want = ref.export(got["keys"])
        assert got["e"]["present"].all() and want["present"].all()
        for f in ("w", "nw") + (("v", "nv") if K else ()):
            assert_close(got["e"][f], want[f], "rank %d %s" % (r, f))
        assert not got["e"]["zw"].any()
    ref.close()


# ---- 8. refusals ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("field,value", [("beta", 0.0), ("beta", -1.0), ("beta", float("nan")), ("beta", float("inf")),
                                         ("learning_rate", float("inf")), ("learning_rate", float("-inf")),
                                         ("learning_rate", float("nan"))])
def test_refusals(field, value):
    with pytest.raises(api.XflowError, match=field):
        api.Table(optimizer=api.OPT_ADAGRAD, **{field: value})


def test_unknown_optimizer_refused():
    with pytest.raises(api.XflowError, match="bad table config"):
        api.Table(optimizer=3)

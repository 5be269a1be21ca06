"""Deterministic mode of the canonical FM and multi-view machine trainers (xf_trainer_set_deterministic,
csrc/step_det.cu): the same bits on every run under contention, each key's sums in the documented association (the
numpy restatement in deterministic_model.py), the default step's bits where that is reproducible, the float64 models'
tolerances, the frozen model's predict, exact resume, and the interface (refusals, launch counts, allocation failure)."""
import functools

import numpy as np
import pytest

import deterministic_model as DM
from common import MVM64, CanonicalFM64, assert_close
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

BIG = 65536
ERR_ARG, ERR_CUDA = "error -1:", "error -2:"


def _keys(ids):
    return api.hash_decimal_ids(np.asarray(ids, np.uint64))


def _csr(lens):
    rp = np.zeros(len(lens) + 1, np.uint32)
    rp[1:] = np.cumsum(lens)
    return rp


@functools.lru_cache(maxsize=None)
def _contended(seed, B=BIG, mvm=False):
    """Hot keys in every row and repeats inside rows: each row has key 0, two keys of a 64-key hot set, one key twice
    and 4 .. 10 Zipf keys; multi-view machine rows put 4 .. 12 of their tokens in field 0."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(8, 15, B)
    rp = _csr(lens)
    n = int(rp[-1])
    _, zipf, _ = datagen.make_ids(seed, 1, n, 200000, dist="zipf")
    ids = zipf.astype(np.uint64) + 1000
    starts = rp[:-1].astype(np.int64)
    ids[starts] = 0
    ids[starts + 1] = rng.integers(1, 65, B)
    ids[starts + 2] = rng.integers(1, 65, B)
    ids[starts + 4] = ids[starts + 3]
    keys = _keys(ids)
    x = rng.uniform(-1.5, 2.0, n).astype(np.float32)
    x[rng.random(n) < 0.05] = 0.0
    lab = (rng.random(B) < 0.3).astype(np.uint8)
    fields = None
    if mvm:
        fields = rng.integers(1, 6, n).astype(np.uint8)
        nf0 = rng.integers(4, 13, B)
        pos = np.arange(n) - np.repeat(starts, lens)
        fields[pos < np.repeat(np.minimum(nf0, lens), lens)] = 0
    return rp, keys, fields, x, lab


def _table(K, opt, canon_model, lr=None, capacity=1 << 20, seed=5):
    kw = dict(latent_dim=K, optimizer=opt, v_init=api.VINIT_COUNTER, seed=seed, capacity=capacity, canonical_fm=1)
    if lr is not None:
        kw["learning_rate"] = lr
    t = api.Table(**kw)
    tr = api.Trainer(t, model=canon_model, max_rows=BIG, max_nnz=BIG * 16, keep_loss=True)
    return t, tr


def _step(tr, mvm, batch):
    rp, keys, fields, x, lab = batch
    if mvm:
        return tr.step_host_fields(rp, keys, fields, x, lab)
    return tr.step_host_values(rp, keys, x, lab)


def _predict(tr, mvm, batch):
    rp, keys, fields, x, _ = batch
    return tr.predict_host_fields(rp, keys, fields, x) if mvm else tr.predict_host_values(rp, keys, x)


def _export_bytes(t):
    keys = np.sort(t.list_keys())
    e = t.export(keys)
    return keys, {k: np.ascontiguousarray(v).tobytes() for k, v in e.items()}


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


CASES = [(False, K, o) for K in (4, 16, 128) for o in (api.OPT_FTRL, api.OPT_SGD)] + \
        [(True, K, o) for K in (4, 32) for o in (api.OPT_FTRL, api.OPT_SGD)]


@pytest.mark.parametrize("mvm,K,opt", CASES)
def test_reproducible_under_contention(mvm, K, opt, tmp_path):
    """Two tables train on the same contended 65 536-row batches, one of them with another trainer's steps interleaved
    on a second stream: exports, key sets, residuals, losses, predictions, stats, pv reports and the frozen models'
    files are identical byte for byte."""
    model = api.MODEL_MVM if mvm else api.MODEL_FM_CANONICAL
    batches = [_contended(11 + i, mvm=mvm) for i in range(3)]
    runs = []
    other_t, other_tr = _table(K, opt, model, seed=9)
    for run in range(2):
        t, tr = _table(K, opt, model)
        tr.set_deterministic(True)
        pv = api.ProgressiveValidation(device=0, mantissa_bits=12)
        tr.set_validation(pv)
        out = {"loss": [], "res": [], "pred": []}
        for i, b in enumerate(batches):
            if run == 1:
                _step(other_tr, mvm, batches[(i + 1) % 3])  # its own table and stream, in flight beside ours
            out["loss"].append(np.float32(_step(tr, mvm, b)).tobytes())
            out["res"].append(tr.get_loss(b[4].size).tobytes())
        out["pred"] = _predict(tr, mvm, batches[0]).tobytes()
        out["keys"], out["export"] = _export_bytes(t)
        out["stats"] = tr.stats()
        out["pv"] = pv.report_bytes()
        m = t.freeze_mvm() if mvm else t.freeze_canonical()
        path = str(tmp_path / ("m%d.xfsm" % run))
        m.save(path)
        out["model"] = open(path, "rb").read()
        runs.append(out)
        tr.set_validation(None)
    a, b = runs
    assert a["keys"].tobytes() == b["keys"].tobytes()
    for k in a["export"]:
        assert a["export"][k] == b["export"][k], k
    for k in ("loss", "res", "pred", "stats", "pv", "model"):
        assert a[k] == b[k], k
    assert a["stats"]["unique_keys"] > 0


@pytest.mark.parametrize("mvm", [False, True])
def test_bit_exact_order(mvm):
    """One SGD step on one-token rows that repeat four keys hundreds of times (and a tail of single keys): the table
    after the step equals the numpy restatement of the association and the update, fed the device's residuals."""
    K, B, lr = 8, 1024, 0.5
    t, tr = _table(K, api.OPT_SGD, api.MODEL_MVM if mvm else api.MODEL_FM_CANONICAL, lr=lr)
    tr.set_deterministic(True)
    rng = np.random.default_rng(4)
    ids = np.where(rng.random(B) < 0.8, rng.integers(0, 4, B), rng.integers(100, 100000, B)).astype(np.uint64)
    keys = _keys(ids)
    x = rng.uniform(-2.0, 2.0, B).astype(np.float32)
    lab = (rng.random(B) < 0.5).astype(np.uint8)
    rp = _csr(np.ones(B, np.int64))
    fields = rng.integers(0, 5, B).astype(np.uint8)
    uk = np.unique(keys)
    t.pull(uk)
    before = t.export(uk)
    # spread the latent values so that the terms differ in magnitude and the association shows
    v0 = (rng.normal(0, 1, (uk.size, K)) * 2.0 ** rng.integers(-12, 4, (uk.size, 1))).astype(np.float32)
    t.import_(uk, w=before["w"].astype(np.float32), v=v0)
    if mvm:
        tr.step_host_fields(rp, keys, fields, x, lab)
    else:
        tr.step_host_values(rp, keys, x, lab)
    r = tr.get_loss(B)
    after = t.export(uk)
    pos = np.searchsorted(uk, keys)
    V = v0[pos]
    if mvm:
        A = (r * x)[:, None] * np.ones((1, K), np.float32)      # o_k = 1: a one-token row has no other field
        sums = DM.sums_by_key(keys, A.astype(np.float32))
    else:
        S = np.float32(0.0) + V * x[:, None]                   # the row's S_k: its one token's v_k x from +0
        A, G, L = DM.fmc_terms(r, x, S)
        sums = DM.sums_by_key(keys, A, G, L)
    hot = 0
    for i, k in enumerate(uk):
        w2, v2 = DM.sgd_update(before["w"][i], v0[i], sums[int(k)], float(B), lr)
        if mvm:
            w2 = np.float32(before["w"][i])
        assert _bits(np.float32(after["w"][i])) == _bits(np.float32(w2)), i
        assert (_bits(after["v"][i].astype(np.float32)) == _bits(v2)).all(), i
        hot += int((keys == k).sum() > 32)
    assert hot == 4


def _once_batch(seed, B, mvm):
    """Every key once in the batch; machine rows have at most 5 tokens, all in different fields."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 6, B)
    rp = _csr(lens)
    n = int(rp[-1])
    ids = rng.permutation(10 ** 6)[:n].astype(np.uint64) + 10 ** 6 * seed
    x = rng.uniform(-1.5, 2.0, n).astype(np.float32)
    lab = (rng.random(B) < 0.3).astype(np.uint8)
    fields = None
    if mvm:
        fields = np.concatenate([rng.permutation(8)[:m] for m in lens]).astype(np.uint8)
    return rp, _keys(ids), fields, x, lab


@pytest.mark.parametrize("mvm,K,opt", [(False, 16, api.OPT_FTRL), (False, 128, api.OPT_SGD), (True, 8, api.OPT_FTRL),
                                       (True, 32, api.OPT_SGD)])
def test_agrees_with_the_atomic_path(mvm, K, opt):
    """Where the default step is reproducible (every key once, no field twice in a row) both modes give the same bits."""
    model = api.MODEL_MVM if mvm else api.MODEL_FM_CANONICAL
    (ta, tra), (tb, trb) = _table(K, opt, model), _table(K, opt, model)
    trb.set_deterministic(True)
    for s in range(3):
        b = _once_batch(30 + s, 8192, mvm)
        _step(tra, mvm, b)
        _step(trb, mvm, b)
        assert tra.get_loss(8192).tobytes() == trb.get_loss(8192).tobytes()
    b = _once_batch(40, 4096, mvm)
    assert _predict(tra, mvm, b).tobytes() == _predict(trb, mvm, b).tobytes()
    ka, ea = _export_bytes(ta)
    kb, eb = _export_bytes(tb)
    assert ka.tobytes() == kb.tobytes()
    for k in ea:
        assert ea[k] == eb[k], k
    assert tra.stats() == trb.stats()


@pytest.mark.parametrize("K,opt", [(8, "ftrl"), (16, "sgd")])
def test_canonical_fm_accuracy(K, opt):
    """On batches with repeated keys the deterministic canonical FM stays within the parity tolerances of CanonicalFM64."""
    gopt = api.OPT_FTRL if opt == "ftrl" else api.OPT_SGD
    B, d, space = 512, 12, 3000
    t = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=4, canonical_fm=1)
    tr = api.Trainer(t, model=api.MODEL_FM_CANONICAL, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
    tr.set_deterministic(True)
    rng = np.random.default_rng(K)
    model = CanonicalFM64(K, opt, t.pull)
    for step in range(3):
        rp, keys, lab = datagen.make_csr_keys(70 + step, B, d, space, api.hash_decimal_ids, ragged=(step == 1))
        x = (rng.random(keys.size) * 1.5 + 0.25).astype(np.float32)
        x[::7] *= -1.0
        loss = model.step(rp, keys, x, lab)
        tr.step_host_values(rp, keys, x, lab)
        assert_close(tr.get_loss(B), loss, "residuals, step %d" % step, rel=2e-5, abs_floor=2e-6)
    allk = model.keys()
    e, ref = t.export(allk), model.export(allk)
    for k in ("w", "v") + (("nw", "zw", "nv", "zv") if opt == "ftrl" else ()):
        assert_close(e[k].reshape(allk.size, -1), ref[k], k, rel=2e-4, abs_floor=2e-7)


@pytest.mark.parametrize("K,opt", [(8, "sgd"), (16, "ftrl")])
def test_mvm_accuracy(K, opt):
    """On batches with repeated keys and fields the deterministic machine stays within the tolerances of MVM64."""
    gopt = api.OPT_FTRL if opt == "ftrl" else api.OPT_SGD
    B, d, space, F, lr = 384, 9, 2500, 5, 20.0
    t = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=4, canonical_fm=1, learning_rate=lr)
    tr = api.Trainer(t, model=api.MODEL_MVM, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
    tr.set_deterministic(True)
    rng = np.random.default_rng(100 + K)
    batches = []
    for step in range(3):
        rp, keys, lab = datagen.make_csr_keys(170 + step, B, d, space, api.hash_decimal_ids, ragged=(step == 1))
        fields = rng.integers(0, F, keys.size).astype(np.uint8)
        x = (rng.random(keys.size) * 1.5 + 0.25).astype(np.float32)
        batches.append((rp, keys, fields, x, lab))
    allk = np.unique(np.concatenate([b[1] for b in batches]))
    V0 = rng.normal(0.0, 0.6, (allk.size, K)).astype(np.float32)
    t.import_(allk, v=V0)
    model = MVM64(V0, opt, lr)
    for step, (rp, keys, fields, x, lab) in enumerate(batches):
        loss = model.step(np.searchsorted(allk, keys), rp, fields, x, lab)
        tr.step_host_fields(rp, keys, fields, x, lab)
        assert_close(tr.get_loss(B), loss, "residuals, step %d" % step, rel=5e-5, abs_floor=5e-6)
    e = t.export(allk)
    if opt == "ftrl":
        for name, ref in (("v", model.V), ("nv", model.NV), ("zv", model.ZV)):
            assert_close(e[name].reshape(allk.size, -1), ref, name, rel=5e-4, abs_floor=5e-7)
    else:
        moved = np.abs(model.V - V0).max()
        assert moved > 1e-3
        assert_close(e["v"].reshape(allk.size, -1) - V0, model.V - V0, "v - v0", rel=2e-3,
                     abs_floor=2e-6 + 1e-4 * moved)


def test_mvm_predict_equals_frozen_model():
    """With the mode on the table's predict is the frozen model's forward on every row, many same-field tokens
    included."""
    K = 16
    t, tr = _table(K, api.OPT_FTRL, api.MODEL_MVM)
    tr.set_deterministic(True)
    b = _contended(21, B=4096, mvm=True)
    _step(tr, True, b)
    keys = np.sort(t.list_keys())
    rng = np.random.default_rng(5)
    t.import_(keys, w=np.zeros(keys.size, np.float32), v=rng.normal(0, 0.7, (keys.size, K)).astype(np.float32))
    m = t.freeze_mvm()
    rp, k, fields, x, _ = _contended(22, B=4096, mvm=True)
    got = tr.predict_host_fields(rp, k, fields, x)
    want = m.predict_host_fields(rp, k, fields, x)
    assert got.tobytes() == want.tobytes()
    assert np.unique(got).size > 100


@pytest.mark.parametrize("mvm", [False, True])
def test_exact_resume(mvm, tmp_path):
    """A state image saved mid-run with repeated keys, resumed: every export, residual and prediction equals the run
    that never saved."""
    K, model = 16, (api.MODEL_MVM if mvm else api.MODEL_FM_CANONICAL)
    batches = [_contended(50 + i, B=8192, mvm=mvm) for i in range(4)]
    ta, tra = _table(K, api.OPT_FTRL, model)
    tra.set_deterministic(True)
    res_a = []
    for b in batches:
        _step(tra, mvm, b)
        res_a.append(tra.get_loss(8192).tobytes())
    tb, trb = _table(K, api.OPT_FTRL, model)
    trb.set_deterministic(True)
    for b in batches[:2]:
        _step(trb, mvm, b)
    path = str(tmp_path / "mid.xfst")
    tb.save_state(path)
    tc, trc = _table(K, api.OPT_FTRL, model)
    tc.load_state(path)
    trc.set_deterministic(True)
    for i, b in enumerate(batches[2:]):
        _step(trc, mvm, b)
        assert trc.get_loss(8192).tobytes() == res_a[2 + i]
    assert _predict(trc, mvm, batches[0]).tobytes() == _predict(tra, mvm, batches[0]).tobytes()
    ka, ea = _export_bytes(ta)
    kc, ec = _export_bytes(tc)
    assert ka.tobytes() == kc.tobytes()
    for k in ea:
        assert ea[k] == ec[k], k


def test_refused_on_lr_and_fm():
    t = api.Table(latent_dim=0)
    tr = api.Trainer(t, model=api.MODEL_LR, max_rows=64, max_nnz=1024)
    with pytest.raises(api.XflowError, match="fixed point or f64"):
        tr.set_deterministic(True)
    t2 = api.Table(latent_dim=8)
    tr2 = api.Trainer(t2, model=api.MODEL_FM, max_rows=64, max_nnz=1024)
    with pytest.raises(api.XflowError, match="fixed point or f64"):
        tr2.set_deterministic(True)


def _sort_launches(n, log2cap):
    if n <= 256 * 19:
        return 1
    return 2 + -(-(log2cap + 1) // 8)


@pytest.mark.parametrize("mvm", [False, True])
def test_launch_counts(mvm):
    """The documented kernels per deterministic step; predict one; on = 0 gives the default step's count back."""
    K, model = 8, (api.MODEL_MVM if mvm else api.MODEL_FM_CANONICAL)
    # room for every key, so that no growth (whose rehash kernels the table counts) happens inside a step
    ref_t, ref_tr = _table(K, api.OPT_FTRL, model, capacity=1 << 20)
    t, tr = _table(K, api.OPT_FTRL, model, capacity=1 << 20)
    small, big = _contended(60, B=256, mvm=mvm), _contended(61, B=8192, mvm=mvm)
    n0 = ref_tr.launches()
    _step(ref_tr, mvm, small)
    default_step = ref_tr.launches() - n0
    n0 = ref_tr.launches()
    _predict(ref_tr, mvm, small)
    default_predict = ref_tr.launches() - n0
    tr.set_deterministic(True)
    for b in (small, big):
        n0 = tr.launches()
        cap = t.capacity()
        _step(tr, mvm, b)
        assert t.capacity() == cap
        log2cap = int(cap).bit_length() - 1
        assert tr.launches() - n0 == 1 + _sort_launches(b[1].size, log2cap) + 3 + 1 + 1
    n0 = tr.launches()
    _predict(tr, mvm, small)
    assert tr.launches() - n0 == 1 == default_predict
    tr.set_deterministic(False)
    n0 = tr.launches()
    _step(tr, mvm, small)
    assert tr.launches() - n0 == default_step == 2


def test_allocation_failure_leaves_the_trainer_unchanged():
    """Scratch for 2^28 rows of K = 128 does not fit in device memory: XF_ERR_CUDA, and the trainer keeps training
    with the default kernels, as a twin that never asked."""
    K = 128
    mk = lambda: api.Table(latent_dim=K, optimizer=api.OPT_SGD, v_init=api.VINIT_COUNTER, seed=5, canonical_fm=1)
    t, twin_t = mk(), mk()
    tr = api.Trainer(t, model=api.MODEL_FM_CANONICAL, max_rows=1 << 28, max_nnz=1 << 16, keep_loss=True)
    twin = api.Trainer(twin_t, model=api.MODEL_FM_CANONICAL, max_rows=1 << 28, max_nnz=1 << 16, keep_loss=True)
    with pytest.raises(api.XflowError, match=ERR_CUDA):
        tr.set_deterministic(True)
    b = _once_batch(70, 2048, False)
    n0 = tr.launches()
    _step(tr, False, b)
    _step(twin, False, b)
    assert tr.launches() - n0 == 2
    assert tr.get_loss(2048).tobytes() == twin.get_loss(2048).tobytes()
    ka, ea = _export_bytes(t)
    kb, eb = _export_bytes(twin_t)
    assert ka.tobytes() == kb.tobytes()
    for k in ea:
        assert ea[k] == eb[k], k

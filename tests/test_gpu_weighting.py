"""Importance-weighted training on the device (pytest -m gpu): xf_trainer_step_host_weighted / _device_weighted and
xf_trainer_set_negative_sampling (include/xflow_b200.h) against the CPU model tests/weighting_model.py, and weights of
1 against the unweighted step bit for bit."""
import os
import re
import subprocess

import numpy as np
import pytest

from common import GOLDEN, assert_close
from oracle import oracle as O
from weighting_model import WeightingTable, row_weights
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN = os.path.join(GOLDEN, "data", "small_train")
TEST = os.path.join(GOLDEN, "data", "small_test")

CONFIGS = {  # name: (model, optimizer, K, eager LR)
    "lr_ftrl": (api.MODEL_LR, api.OPT_FTRL, 0, False),
    "lr_sgd": (api.MODEL_LR, api.OPT_SGD, 0, False),
    "lr_ftrl_eager": (api.MODEL_LR, api.OPT_FTRL, 0, True),
    "lr_sgd_eager": (api.MODEL_LR, api.OPT_SGD, 0, True),
    "fm_sgd_k8": (api.MODEL_FM, api.OPT_SGD, 8, False),
    "fm_ftrl_k16": (api.MODEL_FM, api.OPT_FTRL, 16, False),
}


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()


def _sync():
    import torch
    torch.cuda.synchronize()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _table(cfg, monkeypatch, bloom=False, evict=False, capacity=0):
    m, opt, K, eager = CONFIGS[cfg]
    monkeypatch.setenv("XFLOW_EAGER", "1" if eager else "0")
    t = api.Table(latent_dim=K, optimizer=opt, v_init=api.VINIT_COUNTER, seed=11, capacity=capacity)
    if bloom:
        t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=12, hashes=3, decay_batches=2, seed=7)
    if evict:
        t.set_eviction(max_keys=0)
    return t, m, K


def _model(cfg, bloom=False):
    _, opt, K, _ = CONFIGS[cfg]
    t = WeightingTable(K=K, opt=O.OPT_FTRL if opt == api.OPT_FTRL else O.OPT_SGD, init_mode=O.INIT_COUNTER, seed=11)
    if bloom:
        t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=12, hashes=3, decay_batches=2, seed=7)
    return t


def _batches(n, B, d, space, dist="uniform", seed=100):
    return [datagen.make_csr_keys(seed + s, B, d, space, api.hash_decimal_ids, dist=dist, zipf_s=1.2,
                                  ragged=(s % 2 == 1)) for s in range(n)]


def _export(t, keys):
    return t.export(np.unique(np.concatenate([np.zeros(1, np.uint64)] + list(keys))))


# ---- 1. weights of 1 are the unweighted step, bit for bit
@pytest.mark.parametrize("extras", ["plain", "bloom_evict"])
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_weights_of_one_are_the_unweighted_step(cfg, path, extras, monkeypatch):
    B, d = 1024, 20
    bl = extras == "bloom_evict"
    batches = _batches(4, B, d, 6000, dist="zipf")
    out = []
    for weighted in (False, True):
        t, m, K = _table(cfg, monkeypatch, bloom=bl, evict=bl)
        tr = api.Trainer(t, model=m, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
        tr.init_push()
        l0 = tr.launches()
        losses, mals = [], []
        for rp, keys, lab in batches:
            ones = np.ones(lab.size, np.float32)
            if path == "host":
                mal = tr.step_host_weighted(rp, keys, lab, ones) if weighted else tr.step_host(rp, keys, lab)
                mals.append(mal)
            else:
                arrs = [_dev(a) for a in (rp.astype(np.uint32), keys, lab.astype(np.uint8), ones)]
                _sync()
                p = [a.data_ptr() for a in arrs]
                if weighted:
                    tr.step_device_weighted(p[0], p[1], p[2], p[3], lab.size, keys.size)
                else:
                    tr.step_device(p[0], p[1], p[2], lab.size, keys.size)
                tr.sync()
                del arrs
            losses.append(tr.get_loss(lab.size))
        launches = tr.launches() - l0
        keys_all = [k for _, k, _ in batches]
        uk = np.unique(np.concatenate(keys_all + [np.zeros(1, np.uint64)]))
        stamps = t.last_touch(uk) if bl else None
        out.append((t.export(uk), losses, mals, tr.stats()["unique_keys"], stamps, t.size(),
                    t.admission_stats(), launches))
        tr.close()
        t.close()
    (e0, l0, m0, u0, s0, n0, a0, c0), (e1, l1, m1, u1, s1, n1, a1, c1) = out
    for f in e0:
        assert np.array_equal(_bits(e0[f]), _bits(e1[f])), f
    for x, y in zip(l0, l1):
        assert np.array_equal(_bits(x), _bits(y))
    # the loss sum is added in float with one atomic per block, in any order: equal within float rounding
    assert np.allclose(m0, m1, rtol=1e-5, atol=0)
    assert u0 == u1 and n0 == n1 and a0 == a1
    if bl:
        assert np.array_equal(s0, s1)
    assert c1 == c0 + len(batches)  # one weighting pass per weighted step


# ---- 2. random weights in [0, 8] with exact zeros against the model
@pytest.mark.parametrize("dist", ["uniform", "zipf"])
@pytest.mark.parametrize("cfg", ["lr_ftrl", "lr_sgd", "lr_ftrl_eager", "fm_sgd_k8", "fm_ftrl_k16"])
def test_random_weights_match_model(cfg, dist, monkeypatch):
    B, d = 2048, 24
    t, m, K = _table(cfg, monkeypatch)
    mt = _model(cfg)
    tr = api.Trainer(t, model=m, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
    tr.init_push()
    mt.init_push()
    rng = np.random.default_rng(5)
    seen = [np.zeros(1, np.uint64)]
    skipped = 0
    for s, (rp, keys, lab) in enumerate(_batches(5, B, d, 30000, dist=dist, seed=300)):
        wts = rng.uniform(0, 8, lab.size).astype(np.float32)
        wts[rng.random(lab.size) < 0.15] = 0
        mal = tr.step_host_weighted(rp, keys, lab, wts)
        _, res, mmal = mt.step(rp.astype(np.int64), keys, lab.astype(np.int32), wts)
        skipped += int((wts == 0).sum())
        gl = tr.get_loss(B)
        assert np.all(gl[wts == 0] == 0)
        frac = 0.0 if dist == "uniform" else 0.01
        assert_close(gl, res, "loss step %d" % s, abs_floor=1e-6, max_bad_frac=frac)
        assert abs(mal - mmal) <= 1e-5 * mmal + 1e-6
        seen.append(keys)
        uk = np.unique(np.concatenate(seen))
        ge, me = t.export(uk), mt.export(uk)
        assert np.array_equal(ge["present"], me["present"]), s
        for f in ("w", "nw", "zw") + (("v", "nv", "zv") if K else ()):
            assert_close(ge[f], me[f], "%s step %d" % (f, s), rel=2e-5, abs_floor=2e-7, max_bad_frac=frac)
    assert t.size() == mt.size()
    assert tr.skipped_rows() == skipped == mt.skipped


# ---- 3. rows with e_r = 0 change nothing
@pytest.mark.parametrize("cfg", ["lr_ftrl", "lr_ftrl_eager", "fm_ftrl_k16"])
def test_zero_weight_rows_change_nothing(cfg, monkeypatch):
    B, d = 512, 16
    t, m, K = _table(cfg, monkeypatch, bloom=True, evict=True)
    mt = _model(cfg, bloom=True)
    tr = api.Trainer(t, model=m, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
    batches = _batches(4, B, d, 3000, dist="zipf", seed=20)
    for s, (rp, keys, lab) in enumerate(batches):
        wts = np.ones(lab.size, np.float32)
        wts[s % 3::3] = 0
        tr.step_host_weighted(rp, keys, lab, wts)
        _, res, _ = mt.step(rp.astype(np.int64), keys, lab.astype(np.int32), wts)
        gl = tr.get_loss(B)
        assert np.all(gl[wts == 0] == 0) and np.all(res[wts == 0] == 0)
        assert t.size() == mt.size()
        assert t.admission_stats() == mt.admission_stats()
    # keys that occur only in skipped rows are absent
    fresh = datagen.make_csr_keys(999, 64, d, 10 ** 7, api.hash_decimal_ids)
    before = t.size()
    tr.step_host_weighted(fresh[0], fresh[1], fresh[2], np.zeros(64, np.float32))
    assert t.size() == before
    assert not t.export(np.unique(fresh[1]))["present"].any()
    assert tr.skipped_rows() == mt.skipped + 64
    assert t.admission_stats()["batches"] == 5  # still a training batch


# ---- 4. the fixed-point edge: one key over 2^20 and 3 * 2^20 tokens with weight 4
@pytest.mark.parametrize("tokens", [(1 << 20) + 64, 3 << 20])
def test_fixed_point_edge_with_weights(tokens, monkeypatch):
    rows, per = tokens // 64, 64
    rp = (np.arange(rows + 1) * per).astype(np.uint32)
    keys = np.full(rows * per, 12345, np.uint64)
    lab = np.zeros(rows, np.uint8)
    lab[::3] = 1
    wts = np.full(rows, 4.0, np.float32)
    res = {}
    for eager in (False, True):
        monkeypatch.setenv("XFLOW_EAGER", "1" if eager else "0")
        t = api.Table(capacity=1 << 12)
        tr = api.Trainer(t, model=api.MODEL_LR, max_rows=rows, max_nnz=rows * per)
        for _ in range(2):
            tr.step_host_weighted(rp, keys, lab, wts, want_loss=False)
        tr.sync()
        res[eager] = t.export(np.array([12345], np.uint64))
    mt = WeightingTable(K=0)
    for _ in range(2):
        mt.step(rp.astype(np.int64), keys, lab.astype(np.int32), wts)
    me = mt.export(np.array([12345], np.uint64))
    for f in ("w", "nw", "zw"):
        assert_close(res[False][f], me[f], "lazy " + f, rel=1e-5)
        assert_close(res[True][f], me[f], "eager " + f, rel=1e-5)
    # a row of more than 128 tokens (the lazy step's long-row path) with weights
    B, d = 64, 300
    rp, keys, lab = datagen.make_csr_keys(77, B, d, 5000, api.hash_decimal_ids)
    wts = np.random.default_rng(2).uniform(0, 3, B).astype(np.float32)
    wts[::7] = 0
    monkeypatch.setenv("XFLOW_EAGER", "0")
    t = api.Table(latent_dim=0)
    tr = api.Trainer(t, model=api.MODEL_LR, max_rows=B, max_nnz=B * d, keep_loss=True)
    mt = WeightingTable(K=0)
    for _ in range(3):
        tr.step_host_weighted(rp, keys, lab, wts)
        _, r, _ = mt.step(rp.astype(np.int64), keys, lab.astype(np.int32), wts)
        assert_close(tr.get_loss(B), r, "long-row loss", abs_floor=1e-6)
    uk = np.unique(keys)
    ge, me = t.export(uk), mt.export(uk)
    for f in ("w", "nw", "zw"):
        assert_close(ge[f], me[f], "long-row " + f, rel=2e-5, abs_floor=2e-7)


# ---- 5. negative sampling: every entry point decides alike
def _pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).pin_memory()


def _text(rp, ids, lab):
    lines = []
    for r in range(lab.size):
        toks = " ".join("0:%d:1" % int(i) for i in ids[rp[r]:rp[r + 1]])
        lines.append("%d\t%s" % (lab[r], toks))
    return ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("rate", [0.5, 0.1])
@pytest.mark.parametrize("cfg", ["lr_ftrl", "fm_sgd_k8"])
def test_negative_sampling_entry_points_agree(cfg, rate, monkeypatch):
    B, d, nb = 1000, 12, 4
    data = [datagen.make_ids(500 + s, B, d, 20000, "uniform", 1.05, False) for s in range(nb)]
    batches = [(rp, api.hash_decimal_ids(ids), lab) for rp, ids, lab in data]
    results = {}
    for path in ("host", "device", "async", "ids_async", "ingest1", "ingest2", "weighted", "model"):
        if path == "model":
            mt = _model(cfg)
            mt.set_negative_sampling(rate, 9)
            for rp, keys, lab in batches:
                mt.step(rp.astype(np.int64), keys, lab.astype(np.int32))
            results[path] = (mt, mt.skipped)
            continue
        t, m, K = _table(cfg, monkeypatch)
        tr = api.Trainer(t, model=m, max_rows=2 * B, max_nnz=2 * B * d)
        tr.set_negative_sampling(rate, 9)
        if path.startswith("ingest"):
            per = 1 if path == "ingest1" else 2  # one batch per block, or two batches per block, stepped as slices
            for i in range(0, nb, per):
                text = b"".join(_text(*data[j]) for j in range(i, i + per))
                rows, _ = tr.ingest_text(text)
                assert rows == per * B
                for c in range(per):
                    tr.step_ingested(c * B, (c + 1) * B)
        else:
            for (rp, keys, lab), (_, ids, _) in zip(batches, data):
                if path == "host":
                    tr.step_host(rp, keys, lab, want_loss=False)
                elif path == "weighted":
                    tr.step_host_weighted(rp, keys, lab, np.ones(lab.size, np.float32), want_loss=False)
                elif path == "device":
                    arrs = [_dev(a) for a in (rp.astype(np.uint32), keys, lab.astype(np.uint8))]
                    _sync()
                    tr.step_device(arrs[0].data_ptr(), arrs[1].data_ptr(), arrs[2].data_ptr(), lab.size, keys.size)
                    tr.sync()
                else:
                    src = keys if path == "async" else ids.astype(np.uint32)
                    pins = [_pinned(a) for a in (rp.astype(np.uint32), src, lab.astype(np.uint8))]
                    fn = tr.step_host_async if path == "async" else tr.step_host_ids_async
                    fn(pins[0].data_ptr(), pins[1].data_ptr(), pins[2].data_ptr(), lab.size, keys.size)
                    tr.sync()
        tr.sync()
        results[path] = (t, tr.skipped_rows())
        results[path + "_tr"] = tr
    all_keys = np.unique(np.concatenate([np.zeros(1, np.uint64)] + [k for _, k, _ in batches]))
    ref_t, ref_skip = results["host"]
    ref = ref_t.export(all_keys)
    exp_skip = sum(int((row_weights(rp.astype(np.int64), k, l, None, rate, 9) == 0).sum()) for rp, k, l in batches)
    assert ref_skip == exp_skip == results["model"][1]
    assert 0.3 * (1 - rate) * B * nb < exp_skip
    for path in ("device", "async", "ids_async", "ingest1", "ingest2", "weighted"):
        t, skip = results[path]
        e = t.export(all_keys)
        assert skip == ref_skip, path
        for f in e:
            assert np.array_equal(_bits(e[f]), _bits(ref[f])), (path, f)
    me = results["model"][0].export(all_keys)
    assert np.array_equal(ref["present"], me["present"])
    K = CONFIGS[cfg][2]
    for f in ("w", "nw", "zw") + (("v", "nv", "zv") if K else ()):
        assert_close(ref[f], me[f], f, rel=2e-5, abs_floor=2e-7)


# ---- 6. bit-reproducible at B = 65 536 with weights and sampling
@pytest.mark.parametrize("cfg", ["lr_ftrl", "lr_ftrl_eager", "fm_ftrl_k16"])
def test_reproducible_at_65536_rows(cfg, monkeypatch):
    B, d = 65536, 24
    batches = _batches(3, B, d, 1 << 22, dist="zipf", seed=40)
    rng = np.random.default_rng(3)
    wts = [rng.uniform(0, 4, B).astype(np.float32) for _ in batches]
    exps = []
    for _ in range(2):
        t, m, K = _table(cfg, monkeypatch)
        tr = api.Trainer(t, model=m, max_rows=B, max_nnz=B * d * 2)
        tr.set_negative_sampling(0.3, 1)
        for (rp, keys, lab), w in zip(batches, wts):
            tr.step_host_weighted(rp, keys, lab, w, want_loss=False)
        tr.sync()
        exps.append((_export(t, [k for _, k, _ in batches]), t.size(), tr.skipped_rows()))
        tr.close()
        t.close()
    (a, na, sa), (b, nb, sb) = exps
    assert na == nb and sa == sb
    for f in a:
        assert np.array_equal(_bits(a[f]), _bits(b[f])), f


# ---- 7. the CLI
def _cli(env, tmp_path, model="0", epochs="3", world="1"):
    exe = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
    e = dict(os.environ, XFLOW_OPTIMIZER="ftrl", XFLOW_WORLD=world, XFLOW_RANK="0",
             XFLOW_COMM_FILE=str(tmp_path / "comm.id"), **env)
    for k in ("WORLD_SIZE", "XFLOW_ADMIT", "XFLOW_EVICT_MAX_KEYS", "XFLOW_EVICT_IDLE", "XFLOW_EVICT_EVERY"):
        e.pop(k, None)
    return subprocess.run([exe, TRAIN, TEST, model, epochs], cwd=str(tmp_path), env=e, capture_output=True, text=True,
                          timeout=600)


@pytest.mark.parametrize("model,K", [("0", 0), ("1", 10)])
def test_cli_negative_sampling_matches_model(model, K, tmp_path):
    r = _cli(dict(XFLOW_NEG_SAMPLE="0.25", XFLOW_SEED="3"), tmp_path, model=model)
    assert r.returncode == 0, r.stdout + r.stderr
    m = re.search(r"logloss: (\S+)\s+auc = (\S+)\s+tp = (\d+) fp = (\d+)", r.stdout)
    assert m, r.stdout
    ll, auc = float(m.group(1)), float(m.group(2))
    # XFLOW_SEED seeds the sampling policy AND the CLI's tables (the FM latent initialisation)
    t = WeightingTable(K=K, seed=3)
    t.set_negative_sampling(0.25, 3)
    O.train_file(t, TRAIN + "-00000", 2 << 20, 3)
    assert t.skipped > 0
    lab, p = O.predict_file(t, TEST + "-00000", (4 << 20) if K == 0 else (2 << 20))
    want = O.auc_logloss(lab, p)
    assert abs(ll - want["logloss"]) <= 2e-5 * abs(want["logloss"]) + 1e-6
    assert abs(auc - want["auc"]) <= 2e-5
    pred = np.loadtxt(str(tmp_path / "pred_0_0.txt"), ndmin=2)
    assert np.array_equal(pred[:, 2].astype(np.int32), lab)
    assert np.all(np.abs(pred[:, 0] - p) <= 2e-5 * np.abs(p) + 1.1e-6)


@pytest.mark.parametrize("value,world", [("0.5", "2"), ("x", "1"), ("0", "1"), ("1.5", "1"), ("-0.1", "1"),
                                         ("1e-9", "1")])
def test_cli_refuses_bad_negative_sampling(value, world, tmp_path):
    r = _cli(dict(XFLOW_NEG_SAMPLE=value), tmp_path, epochs="1", world=world)
    assert r.returncode != 0 and "XFLOW_NEG_SAMPLE" in (r.stdout + r.stderr), r.stdout + r.stderr


# ---- 8. refusals
def test_refusals(monkeypatch):
    monkeypatch.setenv("XFLOW_EAGER", "0")
    rp = np.array([0, 2, 3], np.uint32)
    keys = np.array([1, 2, 3], np.uint64)
    lab = np.array([1, 0], np.uint8)
    ct = api.Table(latent_dim=8, canonical_fm=1)
    for model in (api.MODEL_FM_CANONICAL, api.MODEL_MVM):
        tr = api.Trainer(ct, model=model, max_rows=4, max_nnz=8)
        with pytest.raises(api.XflowError, match="importance weighting"):
            tr.set_negative_sampling(0.5)
        with pytest.raises(api.XflowError, match="importance weighting"):
            tr.step_host_weighted(rp, keys, lab, np.ones(2, np.float32))
        tr.close()
    t = api.Table()
    tr = api.Trainer(t, model=api.MODEL_LR, max_rows=4, max_nnz=8)
    for bad in (np.nan, -1.0, np.inf):
        with pytest.raises(api.XflowError, match="weight"):
            tr.step_host_weighted(rp, keys, lab, np.array([1.0, bad], np.float32))
    assert t.size() == 0
    # a lazy table's residual sums hold less than 2^47 units: W = 2^40 x 256 tokens is refused, 2^30 x 256 is trained
    tr2 = api.Trainer(t, model=api.MODEL_LR, max_rows=4, max_nnz=512)
    rpb, kb = np.array([0, 256, 257], np.uint32), np.arange(1, 258, dtype=np.uint64)
    with pytest.raises(api.XflowError, match="too large"):
        tr2.step_host_weighted(rpb, kb, lab, np.array([2.0 ** 40, 1.0], np.float32))
    assert t.size() == 0
    tr2.step_host_weighted(rpb, kb, lab, np.array([2.0 ** 30, 1.0], np.float32))
    assert t.size() == 257
    tr2.close()
    for rate in (0.0, 1.5, 2.0 ** -25, -0.5, float("nan")):
        with pytest.raises(api.XflowError, match="rate"):
            tr.set_negative_sampling(rate)
    tr.set_negative_sampling(2.0 ** -24)  # the smallest rate
    tr.set_negative_sampling(1.0)         # off
    assert tr.skipped_rows() == 0
    # a one-rank comm forced onto the sharded step
    import torch  # noqa: F401  (maps PyTorch's NCCL for the comm's bootstrap)
    monkeypatch.setenv("XFLOW_MG_FORCE", "1")
    cid = api.Comm.new_id()
    comm = api.Comm(cid, 0, 1, 0)
    st = api.Table()
    mtr = api.Trainer(st, model=api.MODEL_LR, max_rows=4, max_nnz=8, comm=comm)
    with pytest.raises(api.XflowError, match="single-GPU"):
        mtr.set_negative_sampling(0.5)
    with pytest.raises(api.XflowError, match="single-GPU"):
        mtr.step_host_weighted(rp, keys, lab, np.ones(2, np.float32))
    mtr.close()
    st.close()
    comm.close()

"""Sliced progressive validation on the device (pytest -m gpu): xf_pv_set_slices / xf_pv_add_device_rows /
xf_pv_report_slices against the CPU model tests/pv_slices_model.py and against unsliced pvs fed each slice's rows, a
trainer feeding a sliced pv on every training entry point, a frozen model evaluated per slice, and the CLI's
XFLOW_PV_SLICES."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import pv_slices_model as S
import validation_model as V
from common import GOLDEN
from weighting_model import row_weights
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN = os.path.join(GOLDEN, "data", "small_train")
TEST = os.path.join(GOLDEN, "data", "small_test")
B, D, SPACE = 256, 6, 4000
INTS = ("rows", "positives", "negatives", "nan_rows", "overflow_rows")

CONFIGS = {  # name: (model, optimizer, K, eager LR)
    "lr_ftrl": (api.MODEL_LR, api.OPT_FTRL, 0, False),
    "lr_ftrl_eager": (api.MODEL_LR, api.OPT_FTRL, 0, True),
    "lr_sgd": (api.MODEL_LR, api.OPT_SGD, 0, False),
    "fm_ftrl_k16": (api.MODEL_FM, api.OPT_FTRL, 16, False),
    "fm_sgd_k8": (api.MODEL_FM, api.OPT_SGD, 8, False),
    "fmc_ftrl_k8": (api.MODEL_FM_CANONICAL, api.OPT_FTRL, 8, False),
    "mvm_ftrl_k8": (api.MODEL_MVM, api.OPT_FTRL, 8, False),
}
CANONICAL = (api.MODEL_FM_CANONICAL, api.MODEL_MVM)
ENTRIES = {api.MODEL_LR: ["host", "device", "async", "ids_async", "ingested"],
           api.MODEL_FM: ["host", "device", "async", "ids_async", "ingested"],
           api.MODEL_FM_CANONICAL: ["host_values", "device_values"],
           api.MODEL_MVM: ["host_fields"]}
CASES = ([(c, e, 1.0) for c in CONFIGS for e in ENTRIES[CONFIGS[c][0]]] +
         [(c, e, 0.1) for c in ("lr_ftrl", "lr_ftrl_eager", "fm_ftrl_k16") for e in ("weighted", "device_weighted")])


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()


def _ok(rc):
    assert rc == 0, (rc, api.lib().xf_last_error().decode(errors="replace"))


def _report(raw):
    r = api.PvReport.from_buffer_copy(raw)
    return {n: getattr(r, n) for n, _ in api.PvReport._fields_}


def _plain_bytes(ms, p, y, w, rows):
    """The report bytes of an unsliced pv with mantissa_bits = ms fed rows `rows` through add_device."""
    torch = _torch()
    pv = api.ProgressiveValidation(mantissa_bits=ms)
    if rows.size:
        d = [_dev(p[rows]), _dev(y[rows]), _dev(w[rows])]
        torch.cuda.synchronize()
        pv.add_device(d[0].data_ptr(), d[1].data_ptr(), rows.size, d[2].data_ptr())
    raw = pv.report_bytes()
    pv.close()
    return raw


# ---- 1. add_device_rows against the model and against plain pvs
def _special_stream(seed, n):
    rng = np.random.default_rng(seed)
    p = rng.random(n).astype(np.float32)
    m = 10
    edges = ((np.arange(50, dtype=np.uint32) * np.uint32(997) % np.uint32(20 << m) + np.uint32(107 << m))
             << np.uint32(23 - m)).view(np.float32)
    special = np.array([2.0 ** -20, 1e-6, 1.0, np.nan, -0.5, 1.5, np.inf, -np.inf, 0.0, -0.0, 2.0 ** -21, 1e-30,
                        0.5, np.nextafter(np.float32(0.5), np.float32(0))], np.float32)
    pool = np.concatenate([special, edges, np.nextafter(edges, np.float32(0))])
    pick = rng.random(n) < 0.3
    p[pick] = pool[rng.integers(0, pool.size, int(pick.sum()))]
    y = rng.choice(np.array([0, 1, 2], np.uint8), n, p=[0.6, 0.3, 0.1])
    w = rng.choice(np.array([0.0, 2.0 ** -30, 2.0 ** 24, 1.0, 0.37, 3.0, -1.0, np.inf, np.nan, 2.0 ** 31, -0.0],
                            np.float32), n, p=[0.1, 0.1, 0.05, 0.4, 0.1, 0.15, 0.02, 0.02, 0.02, 0.02, 0.02])
    return p, y, w


def _sliced_rows(seed, n, n_slices):
    """Rows of 0 .. 120 tokens over random keys; slice keys 1 .. 2 n_slices (two per slice) in about half the rows,
    some repeated across 32-token chunks; a few rows name more than 32 distinct slices (when there are that many)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 121, n)
    lens[:5] = [0, 1, 32, 33, 120]
    rp = np.zeros(n + 1, np.uint32)
    rp[1:] = np.cumsum(lens)
    keys = (rng.integers(1 << 40, 1 << 62, int(rp[-1]), dtype=np.int64).astype(np.uint64))
    slice_keys = np.arange(1, 2 * n_slices + 1, dtype=np.uint64)
    for r in range(n):
        a, b = int(rp[r]), int(rp[r + 1])
        if b == a or rng.random() < 0.4:
            continue  # in no slice
        k = slice_keys[rng.integers(0, slice_keys.size)]
        for pos in {int(x) for x in rng.integers(a, b, 3)}:  # up to three times, anywhere in the row
            keys[pos] = k
        if rng.random() < 0.3:  # and a second slice's key
            keys[int(rng.integers(a, b))] = slice_keys[rng.integers(0, slice_keys.size)]
        if b - a >= 100 and n_slices > 40 and rng.random() < 0.3:
            keys[a:a + 80] = np.repeat(slice_keys[rng.permutation(slice_keys.size)[:40]], 2)  # 40 distinct slices
    smap = {int(k): (int(k) - 1) // 2 for k in slice_keys}
    return rp, keys, smap


@pytest.mark.parametrize("ms,n_slices", [(4, 48), (8, 48), (16, 6)])
def test_add_device_rows_matches_the_model_and_plain_pvs(ms, n_slices):
    torch = _torch()
    n = 3000
    p, y, w = _special_stream(ms, n)
    rp, keys, smap = _sliced_rows(ms + 1, n, n_slices)
    members = S.slice_rows(rp, keys, smap, n_slices)
    in_some = np.unique(np.concatenate(members))
    assert 0 < in_some.size < n and min(m.size for m in members) > 0
    assert max(len({smap[k] for k in keys[rp[r]:rp[r + 1]].tolist() if k in smap}) for r in range(n)) > \
        (32 if n_slices > 32 else 1)
    dp, dy, dw, drp, dk = _dev(p), _dev(y), _dev(w), _dev(rp), _dev(keys)
    torch.cuda.synchronize()
    pv = api.ProgressiveValidation(mantissa_bits=10)
    pv.set_slices(np.array(list(smap), np.uint64), np.array(list(smap.values()), np.uint32), n_slices, ms)
    pv.add_device_rows(dp.data_ptr(), dy.data_ptr(), drp.data_ptr(), dk.data_ptr(), n, dw.data_ptr())
    raw = pv.report_slices_bytes()
    assert len(raw) == n_slices
    # the global report: a plain pv's
    assert pv.report_bytes() == _plain_bytes(10, p, y, w, np.arange(n))
    # each slice: a plain pv (mantissa_bits = ms) fed only its rows, and the model
    want = S.slice_reports(p, y, w, rp, keys, smap, n_slices, ms)
    for s in range(n_slices):
        assert raw[s] == _plain_bytes(ms, p, y, w, members[s]), s
        got = _report(raw[s])
        for k in INTS:
            assert got[k] == want[s][k], (s, k)
        for k in ("weight_pos", "weight_neg", "mean_pctr", "ctr"):
            assert np.float64(got[k]).tobytes() == np.float64(want[s][k]).tobytes(), (s, k)
        for k in ("logloss", "auc", "auc_lo", "auc_hi"):
            if math.isnan(want[s][k]):
                assert math.isnan(got[k]), (s, k)
            else:
                assert abs(got[k] - want[s][k]) <= 1e-12 * abs(want[s][k]), (s, k, got[k], want[s][k])
    assert sum(_report(r)["nan_rows"] for r in raw) > 0 and sum(_report(r)["overflow_rows"] for r in raw) > 0
    glob = pv.report_bytes()
    # uneven cuts (row_ptr[0] != 0: the offsets stay absolute into the same keys), then two streams: the same bytes
    cuts = [0, 1, 33, 700, 701, 2500, 2999, n]
    seven = api.ProgressiveValidation(mantissa_bits=10)
    seven.set_slices(np.array(list(smap), np.uint64), np.array(list(smap.values()), np.uint32), n_slices, ms)
    for a, b in zip(cuts, cuts[1:]):
        seven.add_device_rows(dp.data_ptr() + 4 * a, dy.data_ptr() + a, drp.data_ptr() + 4 * a, dk.data_ptr(), b - a,
                              dw.data_ptr() + 4 * a)
    assert seven.report_slices_bytes() == raw and seven.report_bytes() == glob
    two = api.ProgressiveValidation(mantissa_bits=10)
    two.set_slices(np.array(list(smap), np.uint64), np.array(list(smap.values()), np.uint32), n_slices, ms)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    h = n // 2
    two.add_device_rows(dp.data_ptr(), dy.data_ptr(), drp.data_ptr(), dk.data_ptr(), h, dw.data_ptr(),
                        stream=s1.cuda_stream)
    two.add_device_rows(dp.data_ptr() + 4 * h, dy.data_ptr() + h, drp.data_ptr() + 4 * h, dk.data_ptr(), n - h,
                        dw.data_ptr() + 4 * h, stream=s2.cuda_stream)
    assert two.report_slices_bytes() == raw and two.report_bytes() == glob
    for x in (pv, seven, two):
        x.close()


# ---- 2. training feeds each slice exactly its rows' pre-update predictions
class Batch:
    """One CSR batch in every form the entry points take (as tests/test_gpu_validation.py's)."""

    def __init__(self, seed, canonical):
        torch = _torch()
        rng = np.random.default_rng(seed)
        if canonical:
            ids = (np.arange(B * D, dtype=np.uint64) * np.uint64(7) + np.uint64(seed * 13)) % np.uint64(3 * B * D)
            self.rp = np.arange(B + 1, dtype=np.uint32) * D
            self.lab = (rng.random(B) < 0.3).astype(np.uint8)
        else:
            self.rp, ids, self.lab = datagen.make_ids(seed, B, D, SPACE)
        self.keys = api.hash_decimal_ids(np.asarray(ids, np.uint64))
        self.ids = np.asarray(ids).astype(np.uint32)
        self.nnz = int(self.keys.size)
        self.vals = rng.uniform(0.5, 1.5, self.nnz).astype(np.float32)
        self.fields = (np.arange(self.nnz) % 3).astype(np.uint8)
        self.w = rng.choice(np.array([0.0, 0.5, 1.0, 2.0, 7.5], np.float32), B)
        arrays = dict(rp=self.rp, keys=self.keys, ids=self.ids, lab=self.lab, vals=self.vals, w=self.w)
        self.pin = {n: torch.from_numpy(a.view(np.uint8)).pin_memory() for n, a in arrays.items()}
        self.dev = {n: torch.from_numpy(a.view(np.uint8)).cuda() for n, a in arrays.items()}
        torch.cuda.synchronize()
        self.text = b"".join(b"%d\t%s\n" % (int(self.lab[r]), b" ".join(
            b"%d:%d:1" % (j, int(ids[self.rp[r] + j])) for j in range(int(self.rp[r + 1] - self.rp[r]))))
            for r in range(B))

    def d(self, n):
        return self.dev[n].data_ptr()

    def p(self, n):
        return self.pin[n].data_ptr()


def _table(cfg, monkeypatch):
    model, opt, K, eager = CONFIGS[cfg]
    monkeypatch.setenv("XFLOW_EAGER", "1" if eager else "0")
    return api.Table(latent_dim=K, optimizer=opt, v_init=api.VINIT_COUNTER, seed=11, capacity=1 << 15,
                     canonical_fm=1 if model in CANONICAL else 0)


def _train(tr, b, entry):
    if entry == "host":
        tr.step_host(b.rp, b.keys, b.lab, want_loss=False)
    elif entry == "device":
        tr.step_device(b.d("rp"), b.d("keys"), b.d("lab"), B, b.nnz)
    elif entry == "async":
        tr.step_host_async(b.p("rp"), b.p("keys"), b.p("lab"), B, b.nnz)
    elif entry == "ids_async":
        tr.step_host_ids_async(b.p("rp"), b.p("ids"), b.p("lab"), B, b.nnz)
    elif entry == "ingested":
        assert tr.ingest_text(b.text) == (B, b.nnz)
        tr.step_ingested(0, B)
    elif entry == "host_values":
        tr.step_host_values(b.rp, b.keys, b.vals, b.lab)
    elif entry == "device_values":
        _ok(api.lib().xf_trainer_step_device_values(tr.h, C.c_void_p(b.d("rp")), C.c_void_p(b.d("keys")),
                                                    C.c_void_p(b.d("vals")), C.c_void_p(b.d("lab")), B, b.nnz))
    elif entry == "host_fields":
        tr.step_host_fields(b.rp, b.keys, b.fields, b.vals, b.lab)
    elif entry == "weighted":
        tr.step_host_weighted(b.rp, b.keys, b.lab, b.w, want_loss=False)
    elif entry == "device_weighted":
        tr.step_device_weighted(b.d("rp"), b.d("keys"), b.d("lab"), b.d("w"), B, b.nnz)
    tr.sync()
    _torch().cuda.synchronize()


def _twin_pred(t, cfg, b, path, monkeypatch):
    """The predictions of a copy of `t` as it stands now."""
    model = CONFIGS[cfg][0]
    t.save_state(path)
    t2 = _table(cfg, monkeypatch)
    t2.load_state(path)
    tr2 = api.Trainer(t2, model=model, max_rows=B, max_nnz=B * D)
    if model == api.MODEL_FM_CANONICAL:
        p = tr2.predict_host_values(b.rp, b.keys, b.vals)
    elif model == api.MODEL_MVM:
        p = tr2.predict_host_fields(b.rp, b.keys, b.fields, b.vals)
    else:
        p = tr2.predict_host(b.rp, b.keys)
    tr2.close()
    t2.close()
    return p


def _contents(t):
    keys = np.sort(t.list_keys())
    ex = t.export(keys)
    parts = [keys] + [ex[k] for k in ("w", "nw", "zw", "v", "nv", "zv", "present")]
    return b"".join(np.ascontiguousarray(a).tobytes() for a in parts)


TRAIN_SLICES, TRAIN_MS = 5, 8


def _train_map():
    """Ids 0 .. 1199 name slices 0 .. 4 (id % 5): most rows of either batch kind name one or more, some none."""
    ids = np.arange(1200, dtype=np.uint64)
    return api.hash_decimal_ids(ids), (ids % np.uint64(TRAIN_SLICES)).astype(np.uint32)


def _run(cfg, entry, rate, monkeypatch, tmp_path, sliced, n_batches=4):
    """Train n_batches with a pv attached (sliced or not); returns (global bytes, slice bytes or None, the plain pvs'
    bytes per slice, the table's contents, stats)."""
    model = CONFIGS[cfg][0]
    t = _table(cfg, monkeypatch)
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * D)
    if rate < 1.0:
        tr.set_negative_sampling(rate, 5)
    pv = api.ProgressiveValidation()
    mk, ms = _train_map()
    smap = dict(zip(mk.tolist(), ms.tolist()))
    if sliced:
        pv.set_slices(mk, ms, TRAIN_SLICES, TRAIN_MS)
    tr.set_validation(pv)
    preds, labs, ws, members = [], [], [], [[] for _ in range(TRAIN_SLICES)]
    for i in range(n_batches):
        b = Batch(300 + i, model in CANONICAL)
        if sliced:
            pred = _twin_pred(t, cfg, b, str(tmp_path / "twin.xfst"), monkeypatch)
            if "weighted" in entry or rate < 1.0:
                e = row_weights(b.rp, b.keys, b.lab, b.w if "weighted" in entry else None, rate, 5)
            else:
                e = np.ones(B, np.float32)
            for s, rows in enumerate(S.slice_rows(b.rp, b.keys, smap, TRAIN_SLICES)):
                members[s].append(rows + i * B)
            preds.append(pred)
            labs.append(b.lab)
            ws.append(e)
        n0 = tr.launches()
        _train(tr, b, entry)
        if i == 0:
            launches = tr.launches() - n0
    glob = pv.report_bytes()
    slices = plain = None
    if sliced:
        slices = pv.report_slices_bytes()
        p, y, w = np.concatenate(preds), np.concatenate(labs), np.concatenate(ws)
        plain = [_plain_bytes(TRAIN_MS, p, y, w, np.concatenate(m)) for m in members]
    out = (glob, slices, plain, _contents(t), tr.stats(), launches)
    tr.close()
    pv.close()
    t.close()
    return out


@pytest.mark.parametrize("cfg,entry,rate", CASES)
def test_training_feeds_each_slice_its_rows(cfg, entry, rate, monkeypatch, tmp_path):
    glob, slices, plain, state, stats, launches = _run(cfg, entry, rate, monkeypatch, tmp_path, sliced=True)
    reps = [_report(r) for r in slices]
    assert all(r["rows"] > 0 for r in reps), [r["rows"] for r in reps]
    assert slices == plain
    glob0, _, _, state0, stats0, launches0 = _run(cfg, entry, rate, monkeypatch, tmp_path, sliced=False)
    assert glob == glob0 and state == state0 and stats == stats0
    assert launches == launches0 + 1  # +2 per step with a sliced pv, +1 with an unsliced one


# ---- 3. full size
def test_full_size_one_call_equals_four_and_a_second_run():
    torch = _torch()
    rows, d = 65536, 100
    rp, keys, _ = datagen.make_csr_keys(77, rows, d, 10 ** 7, api.hash_decimal_ids, dist="zipf", zipf_s=1.1)
    rng = np.random.default_rng(77)
    p = rng.random(rows).astype(np.float32)
    y = (rng.random(rows) < 0.03).astype(np.uint8)
    uniq, counts = np.unique(keys, return_counts=True)
    mk = uniq[np.argsort(-counts, kind="stable")[:1000]]  # the most frequent keys: most rows name a slice
    ms = (np.arange(1000) % 100).astype(np.uint32)
    d_all = [_dev(a) for a in (p, y, rp, keys)]
    torch.cuda.synchronize()
    dp, dy, drp, dk = (a.data_ptr() for a in d_all)
    out = []
    for cut in (1, 4, 1):
        pv = api.ProgressiveValidation()
        pv.set_slices(mk, ms, 100, 8)
        step = rows // cut
        for a in range(0, rows, step):
            pv.add_device_rows(dp + 4 * a, dy + a, drp + 4 * a, dk, step)
        out.append((pv.report_slices_bytes(), pv.report_bytes()))
        pv.close()
    assert out[0] == out[1] == out[2]
    reps = [_report(r) for r in out[0][0]]
    smap = dict(zip(mk.tolist(), ms.tolist()))
    want = [m.size for m in S.slice_rows(rp, keys, smap, 100)]
    assert [r["rows"] for r in reps] == want and sum(want) > rows // 2


# ---- 4. refusals and lifecycle
def test_refusals_and_lifecycle(monkeypatch):
    torch = _torch()
    pv = api.ProgressiveValidation()
    k = np.arange(1, 11, dtype=np.uint64)
    s = (np.arange(10) % 3).astype(np.uint32)
    cases = [
        (dict(keys=k, slice_of=np.where(s == 2, 3, s).astype(np.uint32), num_slices=3), "not below n_slices"),
        (dict(keys=np.concatenate([k, k[3:4]]), slice_of=np.concatenate([s, s[:1]]), num_slices=3), "listed twice"),
        (dict(keys=np.concatenate([k, np.array([2 ** 64 - 1], np.uint64)]), slice_of=np.concatenate([s, s[:1]]),
              num_slices=3), "reserved key"),
        (dict(keys=k, slice_of=s, num_slices=65537), "at most 65536"),
        (dict(keys=k, slice_of=s, num_slices=3, mantissa_bits=3), "slice_mantissa_bits"),
        (dict(keys=k, slice_of=s, num_slices=3, mantissa_bits=17), "slice_mantissa_bits"),
        (dict(keys=k, slice_of=s, num_slices=18, mantissa_bits=16), "1 GiB"),  # 17 fit
    ]
    for kw, msg in cases:
        with pytest.raises(api.XflowError, match=msg):
            pv.set_slices(**kw)
    big = np.arange(1, (1 << 24) + 2, dtype=np.uint64)
    with pytest.raises(api.XflowError, match="n_keys"):
        pv.set_slices(big, np.zeros(big.size, np.uint32), 1)
    del big
    with pytest.raises(api.XflowError, match="slices"):
        pv.report_slices_bytes(0)  # an unsliced pv has none
    # a sliced pv: add_device refused, report_slices needs its n, reset clears the slices
    b = Batch(9, False)
    p = np.random.default_rng(1).random(B).astype(np.float32)
    dp = _dev(p)
    torch.cuda.synchronize()
    pv.set_slices(api.hash_decimal_ids(np.arange(SPACE, dtype=np.uint64)),
                  (np.arange(SPACE) % 4).astype(np.uint32), 4, 4)
    with pytest.raises(api.XflowError, match="xf_pv_add_device_rows"):
        pv.add_device(dp.data_ptr(), b.d("lab"), B)
    pv.add_device_rows(dp.data_ptr(), b.d("lab"), b.d("rp"), b.d("keys"), B)
    assert sum(_report(r)["rows"] for r in pv.report_slices_bytes()) >= B  # every key names a slice
    for n in (3, 5):
        with pytest.raises(api.XflowError, match="slices"):
            pv.report_slices_bytes(n)
    pv.reset()
    assert all(_report(r)["rows"] == 0 for r in pv.report_slices_bytes())
    assert _report(pv.report_bytes())["rows"] == 0
    # set_slices clears every sum too
    pv.add_device_rows(dp.data_ptr(), b.d("lab"), b.d("rp"), b.d("keys"), B)
    pv.set_slices(api.hash_decimal_ids(np.arange(SPACE, dtype=np.uint64)),
                  (np.arange(SPACE) % 2).astype(np.uint32), 2, 8)
    assert [_report(r)["rows"] for r in pv.report_slices_bytes()] == [0, 0] and _report(pv.report_bytes())["rows"] == 0
    # refused while a trainer feeds it; launches +2 per step
    monkeypatch.setenv("XFLOW_EAGER", "0")
    t = api.Table(seed=1)
    tr = api.Trainer(t, model=api.MODEL_LR, max_rows=B, max_nnz=B * D)
    n0 = tr.launches()
    tr.step_host(b.rp, b.keys, b.lab)
    n1 = tr.launches()
    tr.set_validation(pv)
    tr.step_host(b.rp, b.keys, b.lab)
    assert tr.launches() - n1 == n1 - n0 + 2
    with pytest.raises(api.XflowError, match="detach"):
        pv.set_slices(np.zeros(0, np.uint64), np.zeros(0, np.uint32), 0)
    tr.set_validation(None)
    # zero slices: add_device works again, report_slices is refused
    pv.set_slices(np.zeros(0, np.uint64), np.zeros(0, np.uint32), 0)
    pv.add_device(dp.data_ptr(), b.d("lab"), B)
    assert _report(pv.report_bytes())["rows"] == B
    with pytest.raises(api.XflowError, match="slices"):
        pv.report_slices_bytes(0)
    tr.set_validation(pv)
    n2 = tr.launches()
    tr.step_host(b.rp, b.keys, b.lab)
    assert tr.launches() - n2 == n1 - n0 + 1
    tr.close()
    t.close()
    pv.close()


# ---- 5. a frozen model evaluated per slice
def _libffm(path):
    """(row_ptr, keys, labels, {field: ids per row}) of a libffm text file, ids hashed as the loader hashes them."""
    rp, keys, lab, fields = [0], [], [], {}
    for r, line in enumerate(open(path, "rb")):
        parts = line.split()
        lab.append(1 if int(parts[0]) else 0)
        for tok in parts[1:]:
            f, fid, _ = tok.split(b":")
            keys.append(api.hash_bytes(fid))
            fields.setdefault(int(f), {}).setdefault(r, []).append(fid)
        rp.append(len(keys))
    return np.array(rp, np.uint32), np.array(keys, np.uint64), np.array(lab, np.uint8), fields


def test_frozen_model_per_slice_auc_is_bracketed(monkeypatch):
    torch = _torch()
    monkeypatch.setenv("XFLOW_EAGER", "0")
    rp, keys, lab, _ = _libffm(TRAIN + "-00000")
    t = api.Table(latent_dim=8, optimizer=api.OPT_FTRL, seed=3, capacity=1 << 16)
    tr = api.Trainer(t, model=api.MODEL_FM, max_rows=256, max_nnz=1 << 14)
    for _ in range(5):
        tr.step_host(rp, keys, lab, want_loss=False)
    m = t.freeze()
    trp, tkeys, tlab, fields = _libffm(TEST + "-00000")
    ids = sorted({fid for row in fields[2].values() for fid in row})  # field 2: one id in every row
    mk = np.array([api.hash_bytes(x) for x in ids], np.uint64)
    ms = (np.arange(len(ids)) % 4).astype(np.uint32)
    d = [_dev(a) for a in (trp, tkeys, tlab)]
    out = torch.empty(tlab.size, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    m.predict_device(d[0].data_ptr(), d[1].data_ptr(), tlab.size, tkeys.size, out.data_ptr())
    torch.cuda.synchronize()
    pv = api.ProgressiveValidation(mantissa_bits=16)
    pv.set_slices(mk, ms, 4, 16)
    pv.add_device_rows(out.data_ptr(), d[2].data_ptr(), d[0].data_ptr(), d[1].data_ptr(), tlab.size)
    reps = pv.report_slices()
    pred = out.cpu().numpy()
    members = S.slice_rows(trp, tkeys, dict(zip(mk.tolist(), ms.tolist())), 4)
    # every row names one or more slices (a field-2 id may also be another field's id: ids hash without the field)
    assert np.unique(np.concatenate(members)).size == tlab.size
    for s, rows in enumerate(members):
        assert reps[s]["rows"] == rows.size > 0
        exact = V.exact_auc(pred[rows], tlab[rows])
        if exact is None:
            assert math.isnan(reps[s]["auc"])
        else:
            assert reps[s]["auc_lo"] <= float(exact) <= reps[s]["auc_hi"], (s, float(exact), reps[s])
    pv.close()
    m.close()
    tr.close()
    t.close()


# ---- 6. the CLI
def _cli(env, tmp_path, epochs="2", world="1"):
    exe = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
    e = dict(os.environ, XFLOW_OPTIMIZER="ftrl", XFLOW_WORLD=world, XFLOW_RANK="0",
             XFLOW_COMM_FILE=str(tmp_path / "comm.id"), **env)
    for k in ("WORLD_SIZE", "XFLOW_ADMIT", "XFLOW_EVICT_MAX_KEYS", "XFLOW_EVICT_IDLE", "XFLOW_EVICT_EVERY",
              "XFLOW_NEG_SAMPLE", "XFLOW_EAGER", "XFLOW_HOST_PARSE", "XFLOW_CORE_NUM", "XFLOW_BLOCK_MB", "XFLOW_SEED"):
        e.pop(k, None)
    if "XFLOW_PROGRESSIVE" not in env:
        e.pop("XFLOW_PROGRESSIVE", None)
    return subprocess.run([exe, TRAIN, TEST, "0", epochs], cwd=str(tmp_path), env=e, capture_output=True, text=True,
                          timeout=600)


LINE = re.compile(r"^progressive epoch (\d+) : .*rows = (\d+)$")
SLICE = re.compile(r"^progressive epoch (\d+) slice (\d+) : logloss = (\S+)  auc = (\S+) \[(\S+), (\S+)\]  "
                   r"mean_pctr = (\S+)  ctr = (\S+)  rows = (\d+)$")


def test_cli_prints_one_line_per_slice(tmp_path):
    _, _, _, fields = _libffm(TRAIN + "-00000")
    ids = sorted({fid for row in fields[3].values() for fid in row})  # field 3: one id in every row (a partition)
    path = tmp_path / "slices.txt"
    path.write_text("".join("%s %d\n" % (x.decode(), i % 3) for i, x in enumerate(ids)))
    r = _cli(dict(XFLOW_PROGRESSIVE="1", XFLOW_PV_SLICES=str(path)), tmp_path)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [s for s in r.stdout.splitlines() if s.startswith("progressive")]
    assert len(lines) == 2 * 4
    for epoch in range(2):
        g = LINE.match(lines[4 * epoch])
        assert g and int(g.group(1)) == epoch, lines
        sl = [SLICE.match(x) for x in lines[4 * epoch + 1:4 * epoch + 4]]
        assert all(sl) and [(int(x.group(1)), int(x.group(2))) for x in sl] == [(epoch, 0), (epoch, 1), (epoch, 2)]
        assert sum(int(x.group(9)) for x in sl) == int(g.group(2)) > 0
    # without the variable: the lines of a run without slices
    plain = _cli(dict(XFLOW_PROGRESSIVE="1"), tmp_path)
    assert [s for s in plain.stdout.splitlines() if s.startswith("progressive")] == lines[::4]


@pytest.mark.parametrize("content,env,world,needle", [
    ("123 0\n456\n", dict(XFLOW_PROGRESSIVE="1"), "1", "XFLOW_PV_SLICES"),
    ("123 0\n123 1\n", dict(XFLOW_PROGRESSIVE="1"), "1", "XFLOW_PV_SLICES"),
    ("123 0\n", dict(), "1", "XFLOW_PROGRESSIVE"),
    ("123 0\n", dict(XFLOW_PROGRESSIVE="1"), "2", "XFLOW_PV_SLICES"),
])
def test_cli_refuses_bad_slices_at_startup(content, env, world, needle, tmp_path):
    path = tmp_path / "slices.txt"
    path.write_text(content)
    r = _cli(dict(env, XFLOW_PV_SLICES=str(path)), tmp_path, epochs="1", world=world)
    assert r.returncode != 0 and needle in (r.stdout + r.stderr), r.stdout + r.stderr
    assert "progressive epoch" not in r.stdout

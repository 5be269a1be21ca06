"""Progressive validation on the device (pytest -m gpu): xf_pv_* against the CPU model tests/validation_model.py, and
xf_trainer_set_validation on every training entry point against a twin: a second pv fed the predictions of a copy of
the table taken (xf_table_save_state / _load_state) before each step."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import validation_model as V
from common import GOLDEN
from weighting_model import row_weights
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN = os.path.join(GOLDEN, "data", "small_train")
TEST = os.path.join(GOLDEN, "data", "small_test")
B, D, SPACE = 256, 6, 4000

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
CASES = [(c, e) for c in CONFIGS for e in ENTRIES[CONFIGS[c][0]]]


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()


def _ok(rc):
    assert rc == 0, (rc, api.lib().xf_last_error().decode(errors="replace"))


class Batch:
    """One CSR batch in every form the entry points take.  The canonical FM and the MVM add a batch's contributions
    to a key with float atomics: there every key occurs once per batch, and the MVM's fields (token j of a row has
    field j % 3) hold two tokens per row, where its shared-memory sums are order-free."""

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


def _table(cfg, monkeypatch, policy=None):
    model, opt, K, eager = CONFIGS[cfg]
    monkeypatch.setenv("XFLOW_EAGER", "1" if eager else "0")
    t = api.Table(latent_dim=K, optimizer=opt, v_init=api.VINIT_COUNTER, seed=11, capacity=1 << 15,
                  canonical_fm=1 if model in CANONICAL else 0)
    if policy == "bloom":
        t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=12, hashes=3, decay_batches=2, seed=7)
    elif policy == "evict":
        t.set_eviction(max_idle_batches=2, max_keys=600)
    return t


def _train(tr, b, entry):
    torch = _torch()
    L = api.lib()
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
        _ok(L.xf_trainer_step_device_values(tr.h, C.c_void_p(b.d("rp")), C.c_void_p(b.d("keys")),
                                            C.c_void_p(b.d("vals")), C.c_void_p(b.d("lab")), B, b.nnz))
    elif entry == "host_fields":
        tr.step_host_fields(b.rp, b.keys, b.fields, b.vals, b.lab)
    elif entry == "weighted":
        tr.step_host_weighted(b.rp, b.keys, b.lab, b.w, want_loss=False)
    elif entry == "device_weighted":
        tr.step_device_weighted(b.d("rp"), b.d("keys"), b.d("lab"), b.d("w"), B, b.nnz)
    tr.sync()
    torch.cuda.synchronize()


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


def _contents(t, policy):
    """What the table holds: its keys in order with every optimizer field (pending lazy steps folded in) and, with
    eviction tracking, their stamps.  Not the state image's bytes: which slot a key takes when the step inserts
    several at once is the order the hardware lets them in, in a run with or without a pv alike."""
    keys = np.sort(t.list_keys())
    ex = t.export(keys)
    parts = [keys] + [ex[k] for k in ("w", "nw", "zw", "v", "nv", "zv", "present")]
    if policy == "evict":
        parts.append(t.last_touch(keys))
    return b"".join(np.ascontiguousarray(a).tobytes() for a in parts)


def _run(cfg, entry, monkeypatch, tmp_path, policy=None, rate=1.0, n_batches=4, with_pv=True):
    """Train n_batches; returns (trainer's pv report bytes, twin pv report bytes, the table's final contents, rows with
    e > 0)."""
    model = CONFIGS[cfg][0]
    t = _table(cfg, monkeypatch, policy)
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * D)
    if rate < 1.0:
        tr.set_negative_sampling(rate, 5)
    pv = twin = None
    if with_pv:
        pv, twin = api.ProgressiveValidation(), api.ProgressiveValidation()
        tr.set_validation(pv)
    keep = []  # the adds are asynchronous: their inputs stay alive until the report
    trained = 0
    for i in range(n_batches):
        b = Batch(300 + i, model in CANONICAL)
        if with_pv:
            pred = _twin_pred(t, cfg, b, str(tmp_path / "twin.xfst"), monkeypatch)
            if entry in ("weighted", "device_weighted") or rate < 1.0:
                e = row_weights(b.rp, b.keys, b.lab, b.w if "weighted" in entry else None, rate, 5)
            else:
                e = np.ones(B, np.float32)
            trained += int(np.count_nonzero(e))
            d = [_dev(pred), _dev(b.lab), _dev(e)]
            _torch().cuda.synchronize()
            twin.add_device(d[0].data_ptr(), d[1].data_ptr(), B, d[2].data_ptr())
            keep.append((d, b))
        _train(tr, b, entry)
        if policy == "evict" and i % 2 == 1:
            t.evict()
    contents = _contents(t, policy)
    out = (pv.report_bytes(), twin.report_bytes()) if with_pv else (None, None)
    tr.close()
    t.close()
    if with_pv:
        pv.close()
        twin.close()
    return out[0], out[1], contents, trained


def _report(raw):
    r = api.PvReport.from_buffer_copy(raw)
    return {n: getattr(r, n) for n, _ in api.PvReport._fields_}


# ---- 1. xf_pv_add_device against the model
def _special_stream(seed, n=6000):
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


@pytest.mark.parametrize("m", [4, 10, 16])
def test_add_device_matches_the_model(m):
    torch = _torch()
    p, y, w = _special_stream(m)
    want = V.Pv(m).add(p, y, w).report()
    dp, dy, dw = _dev(p), _dev(y), _dev(w)
    torch.cuda.synchronize()
    one = api.ProgressiveValidation(mantissa_bits=m)
    one.add_device(dp.data_ptr(), dy.data_ptr(), p.size, dw.data_ptr())
    raw = one.report_bytes()
    got = _report(raw)
    for k in ("rows", "positives", "negatives", "nan_rows", "overflow_rows"):
        assert got[k] == want[k], k
    for k in ("weight_pos", "weight_neg", "mean_pctr", "ctr"):
        assert np.float64(got[k]).tobytes() == np.float64(want[k]).tobytes(), (k, got[k], want[k])
    for k in ("logloss", "auc", "auc_lo", "auc_hi"):
        assert abs(got[k] - want[k]) <= 1e-12 * abs(want[k]), (k, got[k], want[k])
    assert got["nan_rows"] > 0 and got["overflow_rows"] > 0 and got["auc_lo"] <= got["auc_hi"]
    # seven uneven calls, then two streams: the same bytes
    cuts = [0, 1, 33, 700, 701, 2500, 4999, p.size]
    seven = api.ProgressiveValidation(mantissa_bits=m)
    for a, b in zip(cuts, cuts[1:]):
        seven.add_device(dp.data_ptr() + 4 * a, dy.data_ptr() + a, b - a, dw.data_ptr() + 4 * a)
    assert seven.report_bytes() == raw
    two = api.ProgressiveValidation(mantissa_bits=m)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    h = p.size // 2
    two.add_device(dp.data_ptr(), dy.data_ptr(), h, dw.data_ptr(), stream=s1.cuda_stream)
    two.add_device(dp.data_ptr() + 4 * h, dy.data_ptr() + h, p.size - h, dw.data_ptr() + 4 * h, stream=s2.cuda_stream)
    assert two.report_bytes() == raw
    # report does not reset; reset does; NULL weights are all 1
    assert two.report_bytes() == raw
    two.reset()
    assert _report(two.report_bytes())["rows"] == 0
    two.add_device(dp.data_ptr(), dy.data_ptr(), p.size)
    want1 = V.Pv(m).add(p, y).report()
    got1 = _report(two.report_bytes())
    assert got1["rows"] == want1["rows"] and got1["ctr"] == want1["ctr"] and got1["mean_pctr"] == want1["mean_pctr"]
    for pv in (one, seven, two):
        pv.close()


# ---- 2. training feeds exactly its pre-update predictions
@pytest.mark.parametrize("cfg,entry", CASES)
def test_training_feeds_its_pre_update_predictions(cfg, entry, monkeypatch, tmp_path):
    got, twin, state, trained = _run(cfg, entry, monkeypatch, tmp_path)
    r = _report(got)
    assert r["rows"] == trained == 4 * B and not math.isnan(r["auc"])
    assert got == twin
    _, _, state0, _ = _run(cfg, entry, monkeypatch, tmp_path, with_pv=False)
    assert state == state0


# ---- 3. weighting: negative sampling at 0.1 plus caller weights
@pytest.mark.parametrize("entry", ["weighted", "device_weighted"])
@pytest.mark.parametrize("cfg", ["lr_ftrl", "lr_ftrl_eager", "fm_ftrl_k16"])
def test_weighted_steps_feed_their_effective_weights(cfg, entry, monkeypatch, tmp_path):
    got, twin, state, trained = _run(cfg, entry, monkeypatch, tmp_path, rate=0.1)
    r = _report(got)
    assert 0 < r["rows"] == trained < 4 * B
    assert got == twin
    _, _, state0, _ = _run(cfg, entry, monkeypatch, tmp_path, rate=0.1, with_pv=False)
    assert state == state0


# ---- 4. admission (LR, Bloom) and eviction tracking
@pytest.mark.parametrize("cfg,policy", [("lr_ftrl", "bloom"), ("lr_ftrl_eager", "bloom"), ("lr_ftrl", "evict"),
                                        ("fm_ftrl_k16", "evict")])
def test_admission_and_eviction(cfg, policy, monkeypatch, tmp_path):
    got, twin, state, trained = _run(cfg, "host", monkeypatch, tmp_path, policy=policy)
    assert got == twin and _report(got)["rows"] == trained
    _, _, state0, _ = _run(cfg, "host", monkeypatch, tmp_path, policy=policy, with_pv=False)
    assert state == state0


# ---- 5. full size: identical report bytes from two runs
@pytest.mark.parametrize("cfg", ["lr_ftrl", "fm_ftrl_k16"])
def test_full_size_runs_give_identical_reports(cfg, monkeypatch):
    torch = _torch()
    model, opt, K, _ = CONFIGS[cfg]
    rows, d = 65536, 100
    batches = [datagen.make_csr_keys(50 + s, rows, d, 10 ** 7, api.hash_decimal_ids, dist="zipf", zipf_s=1.1)
               for s in range(3)]
    dev = [[_dev(a) for a in bt] for bt in batches]
    torch.cuda.synchronize()
    out = []
    for _ in range(2):
        monkeypatch.setenv("XFLOW_EAGER", "0")
        t = api.Table(latent_dim=K, optimizer=opt, seed=3)
        tr = api.Trainer(t, model=model, max_rows=rows, max_nnz=rows * d)
        pv = api.ProgressiveValidation()
        tr.set_validation(pv)
        for bt, dv in zip(batches, dev):
            tr.step_device(dv[0].data_ptr(), dv[1].data_ptr(), dv[2].data_ptr(), rows, bt[1].size)
        out.append(pv.report_bytes())
        tr.close()
        pv.close()
        t.close()
    assert out[0] == out[1]
    r = _report(out[0])
    assert r["rows"] == 3 * rows and 0.0 < r["auc_lo"] <= r["auc"] <= r["auc_hi"] < 1.0


# ---- 6. refusals, detaching, launches
def test_refusals_detach_and_launches(monkeypatch):
    monkeypatch.setenv("XFLOW_EAGER", "0")
    for m in (3, 17):
        with pytest.raises(api.XflowError, match="mantissa_bits"):
            api.ProgressiveValidation(mantissa_bits=m)
    b = Batch(7, False)
    t = api.Table(seed=1)
    tr = api.Trainer(t, model=api.MODEL_LR, max_rows=B, max_nnz=B * D)
    pv = api.ProgressiveValidation()
    n0 = tr.launches()
    tr.step_host(b.rp, b.keys, b.lab)
    n1 = tr.launches()
    tr.set_validation(pv)
    tr.step_host(b.rp, b.keys, b.lab)
    n2 = tr.launches()
    assert n2 - n1 == n1 - n0 + 1
    tr.predict_host(b.rp, b.keys)  # predict never adds
    assert _report(pv.report_bytes())["rows"] == B
    with pytest.raises(api.XflowError, match="still feed"):
        pv.close()
    tr.set_validation(None)
    tr.step_host(b.rp, b.keys, b.lab)
    assert tr.launches() - n2 == n1 - n0 + 1  # the predict's one launch; nothing for the pv
    assert _report(pv.report_bytes())["rows"] == B
    pv.close()
    # a trainer's destroy detaches
    pv = api.ProgressiveValidation()
    tr.set_validation(pv)
    tr.close()
    pv.close()
    t.close()
    # a one-rank comm forced onto the sharded step
    import torch  # noqa: F401  (maps PyTorch's NCCL for the comm's bootstrap)
    monkeypatch.setenv("XFLOW_MG_FORCE", "1")
    comm = api.Comm(api.Comm.new_id(), 0, 1, 0)
    st = api.Table()
    mtr = api.Trainer(st, model=api.MODEL_LR, max_rows=4, max_nnz=8, comm=comm)
    pv = api.ProgressiveValidation()
    with pytest.raises(api.XflowError, match="single-GPU"):
        mtr.set_validation(pv)
    mtr.close()
    pv.close()
    st.close()
    comm.close()


# ---- 7. the CLI
def _cli(env, tmp_path, epochs="3", world="1"):
    exe = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
    e = dict(os.environ, XFLOW_OPTIMIZER="ftrl", XFLOW_WORLD=world, XFLOW_RANK="0",
             XFLOW_COMM_FILE=str(tmp_path / "comm.id"), **env)
    for k in ("WORLD_SIZE", "XFLOW_ADMIT", "XFLOW_EVICT_MAX_KEYS", "XFLOW_EVICT_IDLE", "XFLOW_EVICT_EVERY",
              "XFLOW_NEG_SAMPLE", "XFLOW_EAGER", "XFLOW_HOST_PARSE", "XFLOW_CORE_NUM", "XFLOW_BLOCK_MB", "XFLOW_SEED"):
        e.pop(k, None)
    return subprocess.run([exe, TRAIN, TEST, "0", epochs], cwd=str(tmp_path), env=e, capture_output=True, text=True,
                          timeout=600)


LINE = re.compile(r"progressive epoch (\d+) : logloss = (\S+)  auc = (\S+) \[(\S+), (\S+)\]  mean_pctr = (\S+)  "
                  r"ctr = (\S+)  rows = (\d+)")


def test_cli_prints_one_line_per_epoch(monkeypatch, tmp_path):
    r = _cli(dict(XFLOW_PROGRESSIVE="1"), tmp_path)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [LINE.search(s) for s in r.stdout.splitlines() if s.startswith("progressive")]
    assert len(lines) == 3 and all(lines) and [int(x.group(1)) for x in lines] == [0, 1, 2]
    # the same epochs through api: device-parsed blocks of 2 MiB, the init push, one step per block
    monkeypatch.setenv("XFLOW_EAGER", "0")
    t = api.Table(latent_dim=0, optimizer=api.OPT_FTRL, capacity=1 << 20)
    tr = api.Trainer(t, model=api.MODEL_LR, max_rows=(2 << 20) // 8 + 2, max_nnz=(2 << 20) // 6 + 2)
    tr.init_push()
    pv = api.ProgressiveValidation()
    tr.set_validation(pv)
    for epoch in range(3):
        loader = api.Loader(TRAIN + "-00000", 2 << 20)
        while True:
            text = loader.next_raw()
            if not text:
                break
            rows, _ = tr.ingest_text(text)
            tr.step_ingested(0, rows)
        loader.close()
        rep = pv.report()
        g = lines[epoch].groups()
        assert [float(x) for x in g[1:7]] == [rep["logloss"], rep["auc"], rep["auc_lo"], rep["auc_hi"],
                                             rep["mean_pctr"], rep["ctr"]], (epoch, g, rep)
        assert int(g[7]) == rep["rows"] > 0
        pv.reset()
    tr.close()
    pv.close()
    t.close()


def test_cli_refuses_progressive_with_two_ranks(tmp_path):
    r = _cli(dict(XFLOW_PROGRESSIVE="1"), tmp_path, epochs="1", world="2")
    assert r.returncode != 0 and "XFLOW_PROGRESSIVE" in (r.stdout + r.stderr), r.stdout + r.stderr

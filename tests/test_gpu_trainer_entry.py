"""The trainer's batch entry points (pytest -m gpu): what each one refuses, counts, launches and returns.

The same batch reaches the table through many entry points: host arrays (step_host, with _values / _fields forms),
page-locked arrays (step_host_async, step_host_ids_async with u32 ids hashed on the device), device arrays
(step_device, step_device_values) and device-parsed text (ingest + step_ingested), and likewise for prediction.  They
differ on purpose in a few places, pinned here one by one:

  * an empty batch (rows == 0) returns at once and counts nothing, except step_device, which counts the step;
  * step_ingested counts steps and rows but not tokens;
  * step_host, the async forms, step_device and step_ingested do not read the table's sticky error; the _values and
    _fields steps and every predict with host outputs do;
  * the async forms refuse pageable buffers (after the empty-batch return);
  * a predict launches the step kernel alone, ids_async adds the hash, ingest the 5 parse launches, a Bloom policy
    the count (and its decay) after every training step.

Every training entry point leaves the same table, bit for bit, as step_host on the same batches; every predict
entry point returns the same pctr.  Loss sums, and the canonical FM's latent state, are compared within float
rounding: the kernels add those in float with atomics, in whatever order the blocks get there."""
import ctypes as C

import numpy as np
import pytest

import placement_model as P
from common import assert_close, bits_equal
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_FULL = -1, -3
B, D, SPACE = 256, 16, 5000
FIELDS = 32  # XF_MVM_FIELDS

MODELS = {
    "lr": dict(model=api.MODEL_LR, K=0),
    "lr_eager": dict(model=api.MODEL_LR, K=0, eager=True),
    "fm": dict(model=api.MODEL_FM, K=4),
    "fmc": dict(model=api.MODEL_FM_CANONICAL, K=4, canonical_fm=1),
    "mvm": dict(model=api.MODEL_MVM, K=4, canonical_fm=1),
}


def L():
    return api.lib()


def _p(a):
    return api._p(a)


class Batch:
    """One CSR batch in every form the entry points take: pageable numpy arrays, page-locked and device copies, and
    the libffm text whose device parse gives the same keys."""

    def __init__(self, seed, rows=B):
        import torch
        self.rp, ids, self.lab = datagen.make_ids(seed, rows, D, SPACE)
        self.keys = api.hash_decimal_ids(ids)
        self.ids = ids.astype(np.uint32)
        self.rows, self.nnz = rows, int(self.keys.size)
        u = datagen.uniform_u64(seed, self.nnz, stream=7)
        self.vals = (u >> np.uint64(40)).astype(np.float32) / np.float32(1 << 24) + np.float32(0.5)
        self.fields = (u % np.uint64(FIELDS)).astype(np.uint8)
        arrays = dict(rp=self.rp, keys=self.keys, ids=self.ids, lab=self.lab, vals=self.vals, fields=self.fields)
        self.pin = {n: torch.from_numpy(a.view(np.uint8)).pin_memory() for n, a in arrays.items()}
        self.dev = {n: torch.from_numpy(a.view(np.uint8)).cuda() for n, a in arrays.items()}
        torch.cuda.synchronize()
        self.text = b"".join(b"%d\t%s\n" % (int(self.lab[r]), b" ".join(b"%d:%d:1" % (j, int(ids[self.rp[r] + j]))
                                                                           for j in range(D))) for r in range(rows))

    def p(self, name):
        return self.pin[name].data_ptr()

    def d(self, name):
        return self.dev[name].data_ptr()


def _trainer(name, monkeypatch, admission=None):
    m = MODELS[name]
    if m.get("eager"):
        monkeypatch.setenv("XFLOW_EAGER", "1")  # read when the table is created
    else:
        monkeypatch.delenv("XFLOW_EAGER", raising=False)
    t = api.Table(latent_dim=m["K"], optimizer=api.OPT_FTRL, capacity=1 << 17, seed=3,
                  **({"canonical_fm": 1} if m.get("canonical_fm") else {}))
    if admission:
        t.set_admission(**admission)
    tr = api.Trainer(t, model=m["model"], max_rows=B, max_nnz=B * D)
    return t, tr


def _ok(rc):
    assert rc == 0, (rc, L().xf_last_error().decode(errors="replace"))


def _pinned_float():
    import torch
    return torch.full((1,), -1.0, dtype=torch.float32).pin_memory()


# ---- training entry points: fn(trainer, batch) -> mean |pctr - label| of the batch (np.float32) or None


def _step_host(tr, b):
    m = C.c_float(-1.0)
    _ok(L().xf_trainer_step_host(tr.h, _p(b.rp), _p(b.keys), _p(b.lab), b.rows, b.nnz, C.byref(m)))
    return np.float32(m.value)


def _async_mean(tr, b, s):
    import torch
    torch.cuda.synchronize()  # not xf_trainer_sync: it would report the table's sticky error
    return np.float32(s.item()) / np.float32(b.rows)


def _step_host_async(tr, b):
    s = _pinned_float()
    _ok(L().xf_trainer_step_host_async(tr.h, _p(b.p("rp")), _p(b.p("keys")), _p(b.p("lab")), b.rows, b.nnz,
                                       _p(s.data_ptr())))
    return _async_mean(tr, b, s)


def _step_host_ids_async(tr, b):
    s = _pinned_float()
    _ok(L().xf_trainer_step_host_ids_async(tr.h, _p(b.p("rp")), _p(b.p("ids")), _p(b.p("lab")), b.rows, b.nnz,
                                           _p(s.data_ptr())))
    return _async_mean(tr, b, s)


def _step_device(tr, b):
    _ok(L().xf_trainer_step_device(tr.h, _p(b.d("rp")), _p(b.d("keys")), _p(b.d("lab")), b.rows, b.nnz))


def _step_ingested(tr, b):
    assert tr.ingest_text(b.text) == (b.rows, b.nnz)
    _ok(L().xf_trainer_step_ingested(tr.h, 0, b.rows))


def _step_host_values(tr, b):
    m = C.c_float(-1.0)
    _ok(L().xf_trainer_step_host_values(tr.h, _p(b.rp), _p(b.keys), _p(b.vals), _p(b.lab), b.rows, b.nnz,
                                        C.byref(m)))
    return np.float32(m.value)


def _step_device_values(tr, b):
    _ok(L().xf_trainer_step_device_values(tr.h, _p(b.d("rp")), _p(b.d("keys")), _p(b.d("vals")), _p(b.d("lab")),
                                          b.rows, b.nnz))


def _step_host_fields(tr, b):
    m = C.c_float(-1.0)
    _ok(L().xf_trainer_step_host_fields(tr.h, _p(b.rp), _p(b.keys), _p(b.fields), _p(b.vals), _p(b.lab), b.rows,
                                        b.nnz, C.byref(m)))
    return np.float32(m.value)


STEPS = {
    "step_host": _step_host, "step_host_async": _step_host_async, "step_host_ids_async": _step_host_ids_async,
    "step_device": _step_device, "step_ingested": _step_ingested, "step_host_values": _step_host_values,
    "step_device_values": _step_device_values, "step_host_fields": _step_host_fields,
}
# the entry points each model trains through; the first is the one the others are compared with
MODEL_STEPS = {
    "lr": ["step_host", "step_host_async", "step_host_ids_async", "step_device", "step_ingested"],
    "lr_eager": ["step_host", "step_host_async", "step_host_ids_async", "step_device", "step_ingested"],
    "fm": ["step_host", "step_host_async", "step_device", "step_ingested"],
    "fmc": ["step_host_values", "step_device_values"],
    "mvm": ["step_host_fields"],
}


# ---- predict entry points: fn(trainer, batch) -> pctr (np.float32[rows])


def _predict_host(tr, b):
    out = np.full(b.rows, -1, np.float32)
    _ok(L().xf_trainer_predict_host(tr.h, _p(b.rp), _p(b.keys), b.rows, b.nnz, _p(out)))
    return out


def _predict_ingested(tr, b):
    assert tr.ingest_text(b.text) == (b.rows, b.nnz)
    out, lab = np.full(b.rows, -1, np.float32), np.full(b.rows, 9, np.uint8)
    _ok(L().xf_trainer_predict_ingested(tr.h, 0, b.rows, _p(out), _p(lab)))
    assert np.array_equal(lab, b.lab)
    return out


def _predict_ingested_metric(tr, b):
    assert tr.ingest_text(b.text) == (b.rows, b.nnz)
    m = C.c_void_p()
    _ok(L().xf_metric_create(C.byref(m), 0))
    try:
        out, lab = np.full(b.rows, -1, np.float32), np.full(b.rows, 9, np.uint8)
        _ok(L().xf_trainer_predict_ingested_metric(tr.h, 0, b.rows, m, _p(out), _p(lab)))
        assert np.array_equal(lab, b.lab)
    finally:
        L().xf_metric_destroy(m)
    return out


def _predict_host_values(tr, b):
    out = np.full(b.rows, -1, np.float32)
    _ok(L().xf_trainer_predict_host_values(tr.h, _p(b.rp), _p(b.keys), _p(b.vals), b.rows, b.nnz, _p(out)))
    return out


def _predict_host_fields(tr, b):
    out = np.full(b.rows, -1, np.float32)
    _ok(L().xf_trainer_predict_host_fields(tr.h, _p(b.rp), _p(b.keys), _p(b.fields), _p(b.vals), b.rows, b.nnz,
                                           _p(out)))
    return out


PREDICTS = {"predict_host": _predict_host, "predict_ingested": _predict_ingested,
            "predict_ingested_metric": _predict_ingested_metric, "predict_host_values": _predict_host_values,
            "predict_host_fields": _predict_host_fields}
MODEL_PREDICTS = {
    "lr": ["predict_host", "predict_ingested", "predict_ingested_metric"],
    "lr_eager": ["predict_host", "predict_ingested", "predict_ingested_metric"],
    "fm": ["predict_host", "predict_ingested", "predict_ingested_metric"],
    "fmc": ["predict_host_values"],
    "mvm": ["predict_host_fields"],
}


@pytest.fixture(scope="module")
def batches():
    return [Batch(seed) for seed in (11, 12, 13)]


def _train(name, entry, batches, monkeypatch):
    t, tr = _trainer(name, monkeypatch)
    means = [STEPS[entry](tr, b) for b in batches]
    tr.sync()
    return t, tr, means


@pytest.mark.parametrize("name,entry", [(n, e) for n, es in MODEL_STEPS.items() for e in es[1:]])
def test_every_training_entry_point_leaves_the_same_table(name, entry, batches, monkeypatch):
    ta, tra, ma = _train(name, MODEL_STEPS[name][0], batches, monkeypatch)
    tb, trb, mb = _train(name, entry, batches, monkeypatch)
    keys = np.unique(np.concatenate([b.keys for b in batches]))
    a, b = ta.export(keys), tb.export(keys)
    assert a["present"].all()
    for k in ("w", "nw", "zw", "v", "nv", "zv"):
        if MODELS[name].get("canonical_fm") and k in ("v", "nv", "zv"):
            # the canonical FM sums the latent gradients in float with atomics: equal up to their order
            assert_close(b[k], a[k], k, abs_floor=1e-6 * float(np.abs(a[k]).max()))
        else:
            assert bits_equal(a[k], b[k]), k
    assert ta.size() == tb.size()
    for x, y in zip(ma, mb):
        if y is not None:
            assert_close(y, x, "mean |pctr - label|")
    assert tra.stats()["unique_keys"] == trb.stats()["unique_keys"]


@pytest.mark.parametrize("name", sorted(MODEL_PREDICTS))
def test_every_predict_entry_point_returns_the_same_pctr(name, batches, monkeypatch):
    probe = Batch(21)
    got = []
    for entry in MODEL_PREDICTS[name]:
        t, tr, _ = _train(name, MODEL_STEPS[name][0], batches, monkeypatch)
        got.append(PREDICTS[entry](tr, probe))
        assert tr.stats()["steps"] == len(batches)
    assert ((got[0] > 0) & (got[0] < 1)).all()
    for g in got[1:]:
        assert bits_equal(g, got[0])


# ---- launches per call (xf_trainer_launches): the step kernel(s) and nothing else

STEP_LAUNCHES = {"lr": 1, "lr_eager": 2, "fm": 2, "fmc": 2, "mvm": 2}
EXTRA = {"step_host_ids_async": 1}  # the device hash of the ids
INGEST = 5                          # the device parse of a text block


def _launches_of(tr, fn):
    before = tr.launches()
    fn()
    tr.sync()
    return tr.launches() - before


@pytest.mark.parametrize("name", sorted(MODELS))
def test_launches_per_call(name, batches, monkeypatch):
    b = batches[0]
    t, tr = _trainer(name, monkeypatch)
    for entry in MODEL_STEPS[name]:
        want = STEP_LAUNCHES[name] + EXTRA.get(entry, 0) + (INGEST if entry == "step_ingested" else 0)
        assert _launches_of(tr, lambda: STEPS[entry](tr, b)) == want, entry
    for entry in MODEL_PREDICTS[name]:
        want = 1 + (INGEST if "ingested" in entry else 0)
        assert _launches_of(tr, lambda: PREDICTS[entry](tr, b)) == want, entry


@pytest.mark.parametrize("name", ["lr", "fm"])
def test_launches_with_bloom_admission(name, batches, monkeypatch):
    """A Bloom policy counts the rejected tokens after every training step (+1) and halves the filter every
    decay_batches steps (+1); a predict does neither."""
    t, tr = _trainer(name, monkeypatch, admission=dict(mode=api.ADMIT_BLOOM, log2_cells=16, decay_batches=2))
    step = STEP_LAUNCHES[name]
    got = [_launches_of(tr, lambda e=e: STEPS[e](tr, batches[0])) for e in MODEL_STEPS[name]]
    want = [step + 1 + (i % 2) + EXTRA.get(e, 0) + (INGEST if e == "step_ingested" else 0)
            for i, e in enumerate(MODEL_STEPS[name])]
    assert got == want
    assert _launches_of(tr, lambda: _predict_host(tr, batches[0])) == 1
    assert t.admission_stats()["batches"] == len(MODEL_STEPS[name])


# ---- counters and empty batches


@pytest.mark.parametrize("name", sorted(MODELS))
def test_step_counters(name, batches, monkeypatch):
    """Every training step counts one step, its rows and its tokens; step_ingested does not count tokens; a predict
    counts nothing."""
    b = batches[0]
    t, tr = _trainer(name, monkeypatch)
    for entry in MODEL_STEPS[name]:
        s0 = tr.stats()
        STEPS[entry](tr, b)
        s1 = tr.stats()
        assert (s1["steps"] - s0["steps"], s1["rows"] - s0["rows"]) == (1, b.rows), entry
        assert s1["nnz"] - s0["nnz"] == (0 if entry == "step_ingested" else b.nnz), entry
    for entry in MODEL_PREDICTS[name]:
        s0 = tr.stats()
        PREDICTS[entry](tr, b)
        s1 = tr.stats()
        assert (s1["steps"], s1["rows"], s1["nnz"]) == (s0["steps"], s0["rows"], s0["nnz"]), entry


@pytest.mark.parametrize("name", sorted(MODELS))
def test_empty_batches(name, batches, monkeypatch):
    """rows == 0: every entry point returns XF_OK at once, with a zero mean where it returns one, launches nothing
    and counts nothing -- except step_device / step_device_values, which count the (empty) step.  The async forms
    return before they look at their buffers, so pageable ones are accepted here."""
    import torch
    t, tr = _trainer(name, monkeypatch)
    rp = np.zeros(1, np.uint32)
    z64, z8, zf = np.zeros(1, np.uint64), np.zeros(1, np.uint8), np.zeros(1, np.float32)
    d = torch.zeros(16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    out = np.full(1, -1, np.float32)
    m = C.c_float(-1.0)
    calls = {
        "step_host": lambda: L().xf_trainer_step_host(tr.h, _p(rp), _p(z64), _p(z8), 0, 0, C.byref(m)),
        "step_host_async": lambda: L().xf_trainer_step_host_async(tr.h, _p(rp), _p(z64), _p(z8), 0, 0, None),
        "step_host_ids_async": lambda: L().xf_trainer_step_host_ids_async(tr.h, _p(rp), _p(z64), _p(z8), 0, 0, None),
        "step_device": lambda: L().xf_trainer_step_device(tr.h, _p(d.data_ptr()), _p(d.data_ptr()),
                                                          _p(d.data_ptr()), 0, 0),
        "step_host_values": lambda: L().xf_trainer_step_host_values(tr.h, _p(rp), _p(z64), _p(zf), _p(z8), 0, 0,
                                                                    C.byref(m)),
        "step_device_values": lambda: L().xf_trainer_step_device_values(tr.h, _p(d.data_ptr()), _p(d.data_ptr()),
                                                                        _p(d.data_ptr()), _p(d.data_ptr()), 0, 0),
        "step_host_fields": lambda: L().xf_trainer_step_host_fields(tr.h, _p(rp), _p(z64), _p(z8), _p(zf), _p(z8), 0,
                                                                    0, C.byref(m)),
        "predict_host": lambda: L().xf_trainer_predict_host(tr.h, _p(rp), _p(z64), 0, 0, _p(out)),
        "predict_host_values": lambda: L().xf_trainer_predict_host_values(tr.h, _p(rp), _p(z64), _p(zf), 0, 0,
                                                                          _p(out)),
        "predict_host_fields": lambda: L().xf_trainer_predict_host_fields(tr.h, _p(rp), _p(z64), _p(z8), _p(zf), 0,
                                                                          0, _p(out)),
        "step_ingested": lambda: L().xf_trainer_step_ingested(tr.h, 3, 3),
        "predict_ingested": lambda: L().xf_trainer_predict_ingested(tr.h, 3, 3, None, None),
        "predict_ingested_metric": lambda: L().xf_trainer_predict_ingested_metric(tr.h, 3, 3, metric, None, None),
    }
    # the model's own entry points, and the async / device / ingest ones that every model takes
    names = set(MODEL_STEPS[name]) | set(MODEL_PREDICTS[name]) | {"step_host_async", "step_host_ids_async",
                                                                  "step_device", "step_ingested", "predict_ingested",
                                                                  "predict_ingested_metric"}
    if MODELS[name]["model"] == api.MODEL_FM_CANONICAL:
        names.add("step_device_values")
    assert tr.ingest_text(batches[0].text) == (B, B * D)  # an ingested block for the empty row ranges
    metric = C.c_void_p()
    _ok(L().xf_metric_create(C.byref(metric), 0))
    try:
        for entry in sorted(names):
            m.value = -1.0
            out[0] = -1
            s0, n0 = tr.stats(), tr.launches()
            _ok(calls[entry]())
            tr.sync()
            s1 = tr.stats()
            assert tr.launches() == n0, entry
            if entry.startswith("step_host") and not entry.endswith("async"):
                assert m.value == 0.0, entry
            assert out[0] == -1, entry
            counted = 1 if entry.startswith("step_device") else 0
            assert (s1["steps"] - s0["steps"], s1["rows"], s1["nnz"]) == (counted, s0["rows"], s0["nnz"]), entry
    finally:
        L().xf_metric_destroy(metric)
    assert t.size() == 0


# ---- refusals: XF_ERR_ARG, nothing counted


def _steps(tr):
    return tr.stats()["steps"]


def _with(b, **changes):
    c = object.__new__(Batch)
    c.__dict__.update(b.__dict__, **changes)
    return c


def test_batches_over_the_trainer_limits_are_refused(monkeypatch):
    """A batch over max_rows or max_nnz is refused by every entry point before anything happens (an oversized text
    block is refused by its parse: test_gpu_ingest)."""
    big = Batch(31, rows=B + 1)
    for name in sorted(MODELS):
        t, tr = _trainer(name, monkeypatch)
        entries = set(MODEL_STEPS[name] + MODEL_PREDICTS[name]) | {"step_host_async", "step_host_ids_async",
                                                                   "step_device"}
        if name == "fmc":
            entries.add("step_device_values")
        for entry in sorted(e for e in entries if "ingested" not in e):
            fn = STEPS.get(entry) or PREDICTS.get(entry)
            for rows, nnz in ((B + 1, B * D), (B, B * D + 1)):
                with pytest.raises(AssertionError, match=r"^\(-1, '.*exceeds trainer limits"):
                    fn(tr, _with(big, rows=rows, nnz=nnz))
        assert _steps(tr) == 0 and t.size() == 0, name


def test_model_mismatch_is_refused(batches, monkeypatch):
    """Feature values need the canonical FM, field ids the multi-view machine."""
    b = batches[0]
    for name in sorted(MODELS):
        t, tr = _trainer(name, monkeypatch)
        wrong = []
        if MODELS[name]["model"] != api.MODEL_FM_CANONICAL:
            wrong += [_step_host_values, _predict_host_values, _step_device_values]
        if MODELS[name]["model"] != api.MODEL_MVM:
            wrong += [_step_host_fields, _predict_host_fields]
        for fn in wrong:
            with pytest.raises(AssertionError, match=r"^\(-1, "):
                fn(tr, b)
        assert _steps(tr) == 0 and t.size() == 0, name


def test_field_ids_of_32_and_over_are_refused(batches, monkeypatch):
    b = batches[0]
    t, tr = _trainer("mvm", monkeypatch)
    bad = _with(b, fields=b.fields.copy())
    bad.fields[b.nnz - 1] = FIELDS
    for fn in (_step_host_fields, _predict_host_fields):
        with pytest.raises(AssertionError, match=r"^\(-1, '.*field id 32"):
            fn(tr, bad)
    assert _steps(tr) == 0 and t.size() == 0
    _step_host_fields(tr, b)  # the trainer goes on working
    assert _steps(tr) == 1


def test_row_ranges_outside_the_ingested_block_are_refused(batches, monkeypatch):
    b = batches[0]
    t, tr = _trainer("lr", monkeypatch)
    assert tr.ingest_text(b.text) == (B, B * D)
    metric = C.c_void_p()
    _ok(L().xf_metric_create(C.byref(metric), 0))
    out = np.empty(B + 1, np.float32)
    try:
        for lo, hi in ((0, B + 1), (5, 4), (B + 1, B + 1)):
            assert L().xf_trainer_step_ingested(tr.h, lo, hi) == ERR_ARG
            assert L().xf_trainer_predict_ingested(tr.h, lo, hi, _p(out), None) == ERR_ARG
            assert L().xf_trainer_predict_ingested_metric(tr.h, lo, hi, metric, None, None) == ERR_ARG
            assert b"outside the ingested block" in L().xf_last_error()
        # a non-empty range needs pctr_out in the plain predict
        assert L().xf_trainer_predict_ingested(tr.h, 0, B, None, None) == ERR_ARG
    finally:
        L().xf_metric_destroy(metric)
    assert _steps(tr) == 0 and t.size() == 0


def test_async_entry_points_refuse_pageable_buffers(batches, monkeypatch):
    b = batches[0]
    t, tr = _trainer("lr", monkeypatch)
    s = _pinned_float()
    pageable = np.zeros(1, np.float32)
    for fn, keys in ((L().xf_trainer_step_host_async, "keys"), (L().xf_trainer_step_host_ids_async, "ids")):
        assert fn(tr.h, _p(b.rp), _p(b.p(keys)), _p(b.p("lab")), b.rows, b.nnz, _p(s.data_ptr())) == ERR_ARG
        assert b"page-locked" in L().xf_last_error()
        assert fn(tr.h, _p(b.p("rp")), _p(b.p(keys)), _p(b.p("lab")), b.rows, b.nnz, _p(pageable)) == ERR_ARG
        assert b"page-locked" in L().xf_last_error()
    assert _steps(tr) == 0 and t.size() == 0


# ---- which entry points report the table's sticky error


@pytest.mark.parametrize("name", sorted(MODELS))
def test_which_entry_points_report_the_sticky_table_error(name, batches, monkeypatch):
    """With the table's error set (a probe overflow, sticky), the training steps on host, page-locked, device and
    ingested batches return XF_OK -- the error shows at the next synchronising call -- while the _values / _fields
    steps and every predict that returns host data report XF_ERR_FULL.  The metric predict without host outputs
    is asynchronous and returns XF_OK."""
    b = batches[0]
    t, tr = _trainer(name, monkeypatch)
    chain = P.one_chain(8192 + 1)
    with pytest.raises(api.XflowError, match="error %d:" % ERR_FULL):
        t.import_(chain, w=np.ones(chain.size, np.float32))
    expect = {e: (ERR_FULL if e in ("step_host_values", "step_host_fields") else 0) for e in MODEL_STEPS[name]}
    expect.update({e: ERR_FULL for e in MODEL_PREDICTS[name]})
    for entry, code in sorted(expect.items()):
        fn = STEPS.get(entry) or PREDICTS.get(entry)
        if code == 0:
            fn(tr, b)
        else:
            with pytest.raises(AssertionError, match=r"^\(%d, '.*probe sequence overflowed" % code):
                fn(tr, b)
    if "predict_ingested_metric" in expect:
        metric = C.c_void_p()
        _ok(L().xf_metric_create(C.byref(metric), 0))
        try:
            assert tr.ingest_text(b.text) == (B, B * D)
            _ok(L().xf_trainer_predict_ingested_metric(tr.h, 0, B, metric, None, None))
        finally:
            L().xf_trainer_sync(tr.h)
            L().xf_metric_destroy(metric)
    assert L().xf_trainer_sync(tr.h) == ERR_FULL


# ---- profiling


@pytest.mark.parametrize("name", ["lr", "fm"])
def test_profile_counts_every_step_host_call(name, batches, monkeypatch):
    t, tr = _trainer(name, monkeypatch)
    tr.set_profile(True)
    n = 5
    for i in range(n):
        _step_host(tr, batches[i % len(batches)])
    prof = tr.profile()
    assert prof["steps"] == n

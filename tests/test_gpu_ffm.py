"""The field-aware FM trainer (XF_MODEL_FFM, csrc/step_ffm.cu) on the device: parity with the float64 statement
(ffm_model.FFM64) at every latent_dim and optimizer, the canonical FM at one field, the fixed-order forward, progressive
validation, exact resume, launch counts, two host threads training at once and the refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest

from common import assert_close
from ffm_model import FFM64
from xflow_b200 import api

pytestmark = pytest.mark.gpu

ERR_ARG = "error -1:"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _csr(lens):
    rp = np.zeros(len(lens) + 1, np.uint32)
    rp[1:] = np.cumsum(lens)
    return rp


def _batch(rng, B, F, space, vals=True, long_rows=True):
    """Ragged rows over `space` ids (keys repeat inside rows and across them): an empty row, rows longer than 32
    tokens, a row of 40 tokens in the largest field F - 1 (more than one pass holds at any L), negative values."""
    lens = rng.integers(0, 14, B)
    if long_rows:
        lens[3::41] = rng.integers(33, 48, lens[3::41].size)
        lens[1] = 40
    lens[0] = 0
    rp = _csr(lens)
    n = int(rp[-1])
    keys = api.hash_decimal_ids(rng.integers(1, space, n).astype(np.uint64))
    fields = rng.integers(0, F, n).astype(np.uint8)
    if long_rows:
        fields[rp[1]:rp[2]] = F - 1
    x = None
    if vals:
        x = rng.uniform(0.25, 1.75, n).astype(np.float32)
        x[::5] *= -1.0
    lab = (rng.random(B) < 0.35).astype(np.uint8)
    return rp, keys, fields, x, lab


def _table(L, opt, lr=1e-3, capacity=0, seed=4):
    return api.Table(latent_dim=L, optimizer=opt, v_init=api.VINIT_COUNTER, seed=seed, canonical_fm=1,
                     learning_rate=lr, capacity=capacity)


def _start(t, rng, allk, L, frac=0.8):
    """Import scaled w and v for most keys (y stays within a few units); the rest enter by a pull (insert-on-pull,
    counter-based v).  Returns the starting W0 [n], V0 [n, L] of allk."""
    imp = rng.random(allk.size) < frac
    W0 = rng.normal(0.0, 0.2, allk.size).astype(np.float32)
    V0 = rng.normal(0.0, 0.12, (allk.size, L)).astype(np.float32)
    t.import_(allk[imp], w=W0[imp], v=V0[imp])
    if (~imp).any():
        w, v = t.pull(allk[~imp])
        W0[~imp] = w
        V0[~imp] = np.asarray(v).reshape(-1, L)
    return W0, V0


def _export_bytes(t):
    keys = np.sort(t.list_keys())
    e = t.export(keys)
    return keys.tobytes(), {k: np.ascontiguousarray(v).tobytes() for k, v in e.items()}


def _compare(t, allk, model, W0, V0, opt, what):
    e = t.export(allk)
    assert e["present"].all()
    n = allk.size
    if opt == "ftrl":
        for name, ref in (("w", model.W), ("nw", model.NW), ("zw", model.ZW), ("v", model.V), ("nv", model.NV),
                          ("zv", model.ZV)):
            assert_close(e[name].reshape(n, -1), ref.reshape(n, -1), "%s %s" % (what, name), rel=5e-4, abs_floor=5e-7)
    else:
        # what the steps moved, not the (much larger) starting values
        for name, ref, start in (("w", model.W, W0), ("v", model.V, V0)):
            got = e[name].reshape(n, -1).astype(np.float64) - start.reshape(n, -1)
            want = ref.reshape(n, -1) - start.reshape(n, -1)
            moved = np.abs(want).max()
            assert moved > 1e-3, (what, name, moved)
            assert_close(got, want, "%s %s - %s0" % (what, name, name), rel=2e-3, abs_floor=2e-6 + 1e-4 * moved)


@pytest.mark.parametrize("with_vals", [True, False])
@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("L", [4, 8, 16, 32, 64, 128])
def test_matches_float64_model(L, opt, with_vals):
    """Three steps against FFM64: residuals, then w, v and the FTRL state of every key (SGD: what the steps moved)."""
    F = L // 4
    gopt = api.OPT_FTRL if opt == "ftrl" else api.OPT_SGD
    lr = 20.0                                                  # SGD: large enough for the steps to show in float32
    B, space = 384, 3000
    rng = np.random.default_rng(1000 + 10 * L + (opt == "sgd") * 3 + with_vals)
    batches = [_batch(rng, B, F, space, vals=with_vals) for _ in range(3)]
    allk = np.unique(np.concatenate([b[1] for b in batches]))
    t = _table(L, gopt, lr=lr)
    tr = api.Trainer(t, model=api.MODEL_FFM, max_rows=B, max_nnz=max(b[1].size for b in batches), keep_loss=True)
    W0, V0 = _start(t, rng, allk, L)
    model = FFM64(W0, V0, opt, lr=lr)
    for step, (rp, keys, fields, x, lab) in enumerate(batches):
        loss = model.step(np.searchsorted(allk, keys), rp, fields, x, lab)
        tr.step_host_fields(rp, keys, fields, x, lab)
        assert_close(tr.get_loss(B), loss, "FFM residuals L=%d, step %d" % (L, step), rel=5e-5, abs_floor=5e-6)
    _compare(t, allk, model, W0, V0, opt, "FFM L=%d" % L)
    assert tr.stats()["steps"] == 3


def test_full_size_batch():
    """65 536 rows at L = 128 (32 fields), FTRL with values, two steps."""
    L, B, space = 128, 65536, 20000
    rng = np.random.default_rng(77)
    batches = []
    for _ in range(2):
        lens = rng.integers(1, 9, B)
        lens[5::997] = 36
        rp = _csr(lens)
        n = int(rp[-1])
        keys = api.hash_decimal_ids(rng.integers(1, space, n).astype(np.uint64))
        fields = rng.integers(0, 32, n).astype(np.uint8)
        x = rng.uniform(0.3, 1.5, n).astype(np.float32)
        batches.append((rp, keys, fields, x, (rng.random(B) < 0.3).astype(np.uint8)))
    allk = np.unique(np.concatenate([b[1] for b in batches]))
    t = _table(L, api.OPT_FTRL)
    tr = api.Trainer(t, model=api.MODEL_FFM, max_rows=B, max_nnz=max(b[1].size for b in batches), keep_loss=True)
    W0, V0 = _start(t, rng, allk, L)
    model = FFM64(W0, V0, "ftrl")
    for step, (rp, keys, fields, x, lab) in enumerate(batches):
        loss = model.step(np.searchsorted(allk, keys), rp, fields, x, lab)
        tr.step_host_fields(rp, keys, fields, x, lab)
        assert_close(tr.get_loss(B), loss, "FFM residuals, full batch, step %d" % step, rel=5e-5, abs_floor=5e-6)
    _compare(t, allk, model, W0, V0, "ftrl", "FFM full batch")


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
def test_one_field_agrees_with_canonical_fm(opt):
    """L = 4 is one field: an FFM trainer and an XF_MODEL_FM_CANONICAL trainer at K = 4, given the same import and
    the same batches, agree within the parity tolerances."""
    gopt = api.OPT_FTRL if opt == "ftrl" else api.OPT_SGD
    B, space = 512, 2000
    rng = np.random.default_rng(31)
    batches = [_batch(rng, B, 1, space) for _ in range(3)]
    allk = np.unique(np.concatenate([b[1] for b in batches]))
    W0 = rng.normal(0.0, 0.2, allk.size).astype(np.float32)
    V0 = rng.normal(0.0, 0.2, (allk.size, 4)).astype(np.float32)
    nnz = max(b[1].size for b in batches)
    ta, tb = _table(4, gopt, lr=20.0), _table(4, gopt, lr=20.0)
    ta.import_(allk, w=W0, v=V0)
    tb.import_(allk, w=W0, v=V0)
    ffm = api.Trainer(ta, model=api.MODEL_FFM, max_rows=B, max_nnz=nnz, keep_loss=True)
    fm = api.Trainer(tb, model=api.MODEL_FM_CANONICAL, max_rows=B, max_nnz=nnz, keep_loss=True)
    for step, (rp, keys, fields, x, lab) in enumerate(batches):
        ffm.step_host_fields(rp, keys, fields, x, lab)
        fm.step_host_values(rp, keys, x, lab)
        assert_close(ffm.get_loss(B), fm.get_loss(B), "residuals, step %d" % step, rel=5e-5, abs_floor=5e-6)
    ea, eb = ta.export(allk), tb.export(allk)
    names = ("w", "v", "nw", "zw", "nv", "zv") if opt == "ftrl" else ("w", "v")
    for k in names:
        assert_close(ea[k], eb[k], "FFM vs canonical FM %s" % k, rel=5e-4, abs_floor=5e-7)


def _subset(batch, rows):
    rp, keys, fields, x, lab = batch
    parts = [np.arange(rp[r], rp[r + 1]) for r in rows]
    tok = np.concatenate(parts) if parts else np.zeros(0, np.int64)
    return (_csr([p.size for p in parts]), keys[tok], fields[tok], None if x is None else x[tok], lab[rows])


@pytest.mark.parametrize("L", [4, 16, 128])
def test_forward_has_a_fixed_order(L):
    """Each row's prediction is the same bits across calls, with the batch's rows permuted, and alone in a batch."""
    F, B = L // 4, 2048
    rng = np.random.default_rng(500 + L)
    t = _table(L, api.OPT_FTRL)
    tr = api.Trainer(t, model=api.MODEL_FFM, max_rows=B, max_nnz=B * 48, keep_loss=True)
    train = _batch(rng, B, F, 1500)
    tr.step_host_fields(*train)                               # a trained table, with some keys never imported
    b = _batch(rng, B, F, 1500)
    rp, keys, fields, x, _ = b
    p1 = tr.predict_host_fields(rp, keys, fields, x)
    p2 = tr.predict_host_fields(rp, keys, fields, x)
    assert p1.tobytes() == p2.tobytes()
    assert np.unique(p1).size > 100
    perm = rng.permutation(B)
    q = _subset(b, perm)
    pp = tr.predict_host_fields(q[0], q[1], q[2], q[3])
    assert pp.tobytes() == p1[perm].tobytes()
    for r in list(range(6)) + list(rng.choice(B, 40, replace=False)):
        s = _subset(b, [r])
        one = tr.predict_host_fields(s[0], s[1], s[2], s[3])
        assert one.tobytes() == p1[r:r + 1].tobytes(), r


def test_progressive_validation_sees_the_predict():
    """A pv fed by an FFM trainer reports the same bytes as a pv fed predict_host_fields of each batch just before
    its step."""
    import torch
    L, B = 32, 4096
    rng = np.random.default_rng(9)
    batches = [_batch(rng, B, L // 4, 5000) for _ in range(3)]
    nnz = max(b[1].size for b in batches)
    ta, tb = _table(L, api.OPT_FTRL), _table(L, api.OPT_FTRL)
    tra = api.Trainer(ta, model=api.MODEL_FFM, max_rows=B, max_nnz=nnz)
    trb = api.Trainer(tb, model=api.MODEL_FFM, max_rows=B, max_nnz=nnz)
    pva, pvb = api.ProgressiveValidation(device=0), api.ProgressiveValidation(device=0)
    tra.set_validation(pva)
    for rp, keys, fields, x, lab in batches:
        tra.step_host_fields(rp, keys, fields, x, lab)
        p = trb.predict_host_fields(rp, keys, fields, x)
        d_p, d_l = torch.from_numpy(p).cuda(), torch.from_numpy(lab).cuda()
        torch.cuda.synchronize()
        pvb.add_device(d_p.data_ptr(), d_l.data_ptr(), B)
        torch.cuda.synchronize()
        trb.step_host_fields(rp, keys, fields, x, lab)
    tra.set_validation(None)
    assert pva.report_bytes() == pvb.report_bytes()


def test_exact_resume(tmp_path):
    """No key repeats within a batch: save_state after two steps, load into a fresh table, two more steps; every
    export and residual equals the run that never stopped."""
    L, B, space = 32, 4096, 400000
    rng = np.random.default_rng(21)
    batches = []
    for _ in range(4):
        lens = rng.integers(1, 12, B)
        rp = _csr(lens)
        n = int(rp[-1])
        keys = api.hash_decimal_ids(rng.choice(space, n, replace=False).astype(np.uint64) + 1)
        fields = rng.integers(0, L // 4, n).astype(np.uint8)
        x = rng.uniform(-1.0, 1.5, n).astype(np.float32)
        batches.append((rp, keys, fields, x, (rng.random(B) < 0.3).astype(np.uint8)))
    nnz = max(b[1].size for b in batches)
    mk = lambda: _table(L, api.OPT_FTRL, capacity=1 << 18)
    ta = mk()
    tra = api.Trainer(ta, model=api.MODEL_FFM, max_rows=B, max_nnz=nnz, keep_loss=True)
    res_a = []
    for b in batches:
        tra.step_host_fields(*b)
        res_a.append(tra.get_loss(B).tobytes())
    tb = mk()
    trb = api.Trainer(tb, model=api.MODEL_FFM, max_rows=B, max_nnz=nnz, keep_loss=True)
    for b in batches[:2]:
        trb.step_host_fields(*b)
    path = str(tmp_path / "mid.xfst")
    tb.save_state(path)
    tc = mk()
    tc.load_state(path)
    trc = api.Trainer(tc, model=api.MODEL_FFM, max_rows=B, max_nnz=nnz, keep_loss=True)
    for i, b in enumerate(batches[2:]):
        trc.step_host_fields(*b)
        assert trc.get_loss(B).tobytes() == res_a[2 + i]
    ka, ea = _export_bytes(ta)
    kc, ec = _export_bytes(tc)
    assert ka == kc
    for k in ea:
        assert ea[k] == ec[k], k


def test_launch_counts_match_the_mvm():
    """The step kernel and the optimizer pass per training step, one kernel per predict, +1 with a pv: as the MVM."""
    L, B = 16, 1024
    rng = np.random.default_rng(3)
    b = _batch(rng, B, 4, 3000)
    counts = []
    for model in (api.MODEL_FFM, api.MODEL_MVM):
        t = _table(L, api.OPT_FTRL, capacity=1 << 20)
        tr = api.Trainer(t, model=model, max_rows=B, max_nnz=b[1].size)
        got = []
        n0 = tr.launches(); tr.step_host_fields(*b); got.append(tr.launches() - n0)
        n0 = tr.launches(); tr.predict_host_fields(b[0], b[1], b[2], b[3]); got.append(tr.launches() - n0)
        pv = api.ProgressiveValidation(device=0)
        tr.set_validation(pv)
        n0 = tr.launches(); tr.step_host_fields(*b); got.append(tr.launches() - n0)
        tr.set_validation(None)
        counts.append(got)
    assert counts[0] == counts[1] == [2, 1, 3]


# Two host threads take the first L = 128 step of a fresh process at once (the step kernel's 64 KB shared-memory opt-in
# is made then), each on its own table; the keys are distinct, so the state after the step has one value.
_THREADS = r"""
import threading
import numpy as np
from xflow_b200 import api
L, B = 128, 4096
rng = np.random.default_rng(11)
lens = rng.integers(1, 40, B)
rp = np.zeros(B + 1, np.uint32)
rp[1:] = np.cumsum(lens)
n = int(rp[-1])
keys = api.hash_decimal_ids(rng.permutation(4 * n)[:n].astype(np.uint64) + 1)
fields = rng.integers(0, 32, n).astype(np.uint8)
x = rng.uniform(0.3, 1.5, n).astype(np.float32)
lab = (rng.random(B) < 0.3).astype(np.uint8)

def run(out, i, barrier=None):
    t = api.Table(latent_dim=L, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=4, canonical_fm=1, capacity=1 << 18)
    tr = api.Trainer(t, model=api.MODEL_FFM, max_rows=B, max_nnz=n, keep_loss=True)
    if barrier is not None:
        barrier.wait()
    tr.step_host_fields(rp, keys, fields, x, lab)
    ks = np.sort(t.list_keys())
    e = t.export(ks)
    out[i] = (tr.get_loss(B).tobytes(), ks.tobytes(), {k: np.ascontiguousarray(v).tobytes() for k, v in e.items()})
    tr.close()
    t.close()

out = [None] * 3
barrier = threading.Barrier(2)
threads = [threading.Thread(target=run, args=(out, i, barrier)) for i in range(2)]
for th in threads:
    th.start()
for th in threads:
    th.join()
run(out, 2)
assert out[2] is not None and len(out[2][1]) == 8 * n
assert out[0] == out[2] and out[1] == out[2]
print("ok")
"""


def test_two_threads_first_step_on_the_device():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", _THREADS], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


def test_refusals_leave_the_table_unchanged():
    import torch
    L, B = 16, 64
    F = L // 4
    rng = np.random.default_rng(8)
    rp, keys, fields, x, lab = _batch(rng, B, F, 500, long_rows=False)
    nnz = keys.size
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*XF_MODEL_FFM needs a table created with canonical_fm = 1"):
        api.Trainer(api.Table(latent_dim=L), model=api.MODEL_FFM, max_rows=B, max_nnz=nnz)
    t = _table(L, api.OPT_FTRL)
    tr = api.Trainer(t, model=api.MODEL_FFM, max_rows=B, max_nnz=nnz, keep_loss=True)
    tr.step_host_fields(rp, keys, fields, x, lab)
    before = _export_bytes(t)
    stats = tr.stats()
    lib = api.lib()
    need = ERR_ARG + ".*XF_MODEL_FFM steps need the tokens' field ids"
    with pytest.raises(api.XflowError, match=need):
        tr.step_host(rp, keys, lab)
    with pytest.raises(api.XflowError, match=need):
        tr.predict_host(rp, keys)
    d = {n: torch.from_numpy(a.view(np.uint8)).cuda() for n, a in (("rp", rp), ("keys", keys), ("lab", lab), ("x", x))}
    torch.cuda.synchronize()
    with pytest.raises(api.XflowError, match=need):
        tr.step_device(d["rp"].data_ptr(), d["keys"].data_ptr(), d["lab"].data_ptr(), B, nnz)
    vals_msg = ERR_ARG + ".*feature values need XF_MODEL_FM_CANONICAL"
    with pytest.raises(api.XflowError, match=vals_msg):
        tr.step_host_values(rp, keys, x, lab)
    with pytest.raises(api.XflowError, match=vals_msg):
        tr.predict_host_values(rp, keys, x)
    with pytest.raises(api.XflowError, match=vals_msg):
        api._check(lib.xf_trainer_step_device_values(tr.h, api._p(d["rp"].data_ptr()), api._p(d["keys"].data_ptr()),
                                                     api._p(d["x"].data_ptr()), api._p(d["lab"].data_ptr()), B, nnz))
    pin = {n: torch.from_numpy(a.view(np.uint8)).pin_memory()
           for n, a in (("rp", rp), ("keys", keys), ("ids", (np.arange(nnz) + 1).astype(np.uint32)), ("lab", lab))}
    with pytest.raises(api.XflowError, match=need):
        tr.step_host_async(pin["rp"].data_ptr(), pin["keys"].data_ptr(), pin["lab"].data_ptr(), B, nnz)
    with pytest.raises(api.XflowError, match=need):
        tr.step_host_ids_async(pin["rp"].data_ptr(), pin["ids"].data_ptr(), pin["lab"].data_ptr(), B, nnz)
    text = b"1 0:10:1 1:20:1 2:30:1\n0 1:40:1\n1 3:50:1 0:60:1\n"
    rows, n_ing = tr.ingest_text(text)
    assert (rows, n_ing) == (3, 6)
    with pytest.raises(api.XflowError, match=need):
        tr.step_ingested(0, rows)
    with pytest.raises(api.XflowError, match=need):
        tr.predict_ingested(0, rows)
    bad = fields.copy()
    bad[5] = F
    with pytest.raises(api.XflowError, match=ERR_ARG + " field id %d of token 5: XF_MODEL_FFM at latent_dim %d takes "
                       "field ids below %d" % (F, L, F)):
        tr.step_host_fields(rp, keys, bad, x, lab)
    with pytest.raises(api.XflowError, match=ERR_ARG + " field id"):
        tr.predict_host_fields(rp, keys, bad, x)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*XF_MODEL_FFM has no deterministic mode"):
        tr.set_deterministic(True)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*importance weighting needs XF_MODEL_LR or XF_MODEL_FM"):
        tr.step_host_weighted(rp, keys, lab, np.ones(B, np.float32))
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*importance weighting needs XF_MODEL_LR or XF_MODEL_FM"):
        tr.set_negative_sampling(0.5)
    tr.sync()
    assert _export_bytes(t) == before
    assert tr.stats() == stats
    # the trainer still trains
    tr.step_host_fields(rp, keys, fields, x, lab)
    assert tr.stats()["steps"] == stats["steps"] + 1
    # the MVM keeps its own bound of 32 fields
    tm = _table(L, api.OPT_FTRL)
    trm = api.Trainer(tm, model=api.MODEL_MVM, max_rows=B, max_nnz=nnz)
    trm.step_host_fields(rp, keys, bad, x, lab)
    bad[5] = 32
    with pytest.raises(api.XflowError, match=ERR_ARG + " field id 32 of token 5: XF_MODEL_MVM takes field ids below 32"):
        trm.step_host_fields(rp, keys, bad, x, lab)

"""Candidate ranking on serving models (xf_model_rank_candidates_*, csrc/rank.cu): each request's top k candidates by
pctr, compared byte for byte with the numpy model (tests/rank_model.py) over the scores xf_model_predict_candidates_*
returns, on every model kind, size class, tie and NaN, through both entry points."""
import re

import numpy as np
import pytest

from rank_model import PAD_INDEX, PAD_PCTR_BITS, rank_model
from test_gpu_candidates import (ERR_ARG, HELD, KINDS, POOL, UNSEEN, Batch, DeviceBatch, _bits, _device, _host, _ids,
                                 _models, _ptr, _random_batch)
from xflow_b200 import api

pytestmark = pytest.mark.gpu

SMALL = 256  # the largest request a warp ranks in rank.cu (XF_RANK_SMALL)


def _rank_host(m, b, k):
    return m.rank_candidates(b.ctx_ptr, b.ctx_keys, b.cand_ptr, b.row_ptr, b.keys, k, ctx_vals=b.ctx_vals, vals=b.vals,
                             ctx_fields=b.ctx_fields, fields=b.fields)


def _launch(m, d, k, outs, stream, with_pctr=True):
    b = d.b
    d_pctr, d_idx, d_top = outs
    m.rank_candidates_device(b.R, d.addr("ctx_ptr"), d.addr("ctx_keys"), b.ctx_keys.size, d.addr("cand_ptr"), b.N,
                             d.addr("row_ptr"), d.addr("keys"), b.keys.size, k, d_pctr.data_ptr(), d_idx.data_ptr(),
                             d_top.data_ptr() if with_pctr else 0, stream=stream.cuda_stream,
                             d_ctx_vals=d.addr("ctx_vals"), d_vals=d.addr("vals"), d_ctx_fields=d.addr("ctx_fields"),
                             d_fields=d.addr("fields"))


def _outs(torch, b, k):
    """Device outputs filled with bytes that no correct call leaves: d_pctr, d_top_index, d_top_pctr."""
    return (torch.full((max(b.N, 1),), 7.0, dtype=torch.float32, device="cuda"),
            torch.full((max(b.R * k, 1),), 12345, dtype=torch.int32, device="cuda"),
            torch.full((max(b.R * k, 1),), 3.0, dtype=torch.float32, device="cuda"))


def _fetch(b, k, outs):
    d_pctr, d_idx, d_top = outs
    n = b.R * k
    return (d_idx.cpu().numpy()[:n].view(np.uint32).reshape(b.R, k), d_top.cpu().numpy()[:n].reshape(b.R, k),
            d_pctr.cpu().numpy()[:b.N])


def _rank_dev(m, b, k, with_pctr=True):
    torch = pytest.importorskip("torch")
    d = DeviceBatch(b, torch)
    outs = _outs(torch, b, k)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    _launch(m, d, k, outs, s, with_pctr)
    s.synchronize()
    return _fetch(b, k, outs)


def _check(m, b, k, what="", scores=None):
    """Both entry points against rank_model(predict_candidates); returns (index, pctr)."""
    if scores is None:
        scores = _host(m, b)
    want_i, want_p = rank_model(scores, b.cand_ptr, k)
    got_i, got_p = _rank_host(m, b, k)
    dev_i, dev_p, dev_s = _rank_dev(m, b, k)
    assert np.array_equal(got_i, want_i), what
    assert np.array_equal(_bits(got_p), _bits(want_p)), what
    assert np.array_equal(dev_i, want_i), what
    assert np.array_equal(_bits(dev_p), _bits(want_p)), what
    assert np.array_equal(_bits(dev_s), _bits(scores)), what
    return want_i, want_p


def _plain_batch(counts, rng, ctx_len=8, cand_len=3, pool=None):
    """An LR / FM batch built without Batch's per-candidate loop: random keys, no values."""
    pool = POOL if pool is None else pool
    b = Batch.__new__(Batch)
    R, N = len(counts), int(np.sum(counts))
    b.ctx_ptr = _ptr([ctx_len] * R)
    b.cand_ptr = _ptr(counts)
    b.row_ptr = _ptr(np.full(N, cand_len))
    b.ctx_keys = pool[rng.integers(0, pool.size, int(b.ctx_ptr[-1]))].astype(np.uint64)
    b.keys = pool[rng.integers(0, pool.size, int(b.row_ptr[-1]))].astype(np.uint64)
    b.ctx_vals = b.vals = b.ctx_fields = b.fields = None
    return b


# ---- 1. every model ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,K", KINDS, ids=_ids(KINDS))
def test_every_model(kind, K):
    rng = np.random.default_rng(K + 41)
    for key, m in _models(kind, K).items():
        b = _random_batch(rng, kind, max_cands=300)
        for k in (1, 16):
            scores = _device(m, b)  # predict_candidates_device's bytes: d_pctr must equal them
            assert np.array_equal(_bits(scores), _bits(_host(m, b))), key
            _check(m, b, k, (key, k), scores)


# ---- 2. size classes ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 7, 16, 128, 1024])
def test_size_classes(k):
    rng = np.random.default_rng(k)
    sizes = {0, 1, 2, k - 1, k, k + 1, 31, 32, 33, SMALL - 1, SMALL, SMALL + 1, 1023, 1024, 1025, 4096, 65537}
    counts = [s for s in sorted(sizes) if s >= 0]
    counts = [counts[i] for i in rng.permutation(len(counts))]
    for kind, K in (("lr", 0), ("fm", 8)):
        m = _models(kind, K)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
        _check(m, _plain_batch(counts, rng), k, (kind, counts))


def test_many_requests_and_one_huge():
    rng = np.random.default_rng(43)
    m = _models("lr", 0)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    _check(m, _plain_batch([1] * 65536, rng), 16, "65536 x 1")
    idx, _ = _check(m, _plain_batch([1 << 20], rng, ctx_len=4, cand_len=4), 1024, "1 x 2^20")
    assert len(set(idx[0].tolist())) == 1024


# ---- 3. ties -----------------------------------------------------------------------------------------------------------
def test_identical_candidates():
    rng = np.random.default_rng(47)
    m = _models("lr", 0)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    b = _plain_batch([50000], rng, cand_len=5)
    b.keys = np.tile(b.keys[:5], 50000)
    idx, _ = _check(m, b, 1024, "50 000 identical rows")
    assert idx[0].tolist() == list(range(1024))


def _clamp_model():
    """An LR model with a key of w = 50 (pctr exactly 1.0) and one of w = -50 (pctr 1e-6) besides HELD[:500]."""
    hi, lo = UNSEEN[0], UNSEEN[1]
    keys = np.concatenate([[hi, lo], HELD[:500]]).astype(np.uint64)
    w = np.concatenate([[50.0, -50.0], np.random.default_rng(53).normal(0, 0.3, 500)]).astype(np.float32)
    t = api.Table(capacity=1 << 12)
    t.import_(keys, w=w)
    m = t.freeze()
    t.close()
    return m, hi, lo


def test_clamped_ties_straddle_k():
    rng = np.random.default_rng(59)
    m, hi, lo = _clamp_model()
    # n = 600 (CTA class) and 200 (warp class): every second candidate at 1.0, every fifth 1e-6 otherwise; n = 300 all
    # but ten at 1e-6, so that k reaches into the 1e-6 group
    counts = [600, 200, 300]
    b = _plain_batch(counts, rng, ctx_len=2, pool=HELD[:500])
    c = 0
    for q, n in enumerate(counts):
        for i in range(n):
            row = b.keys[3 * c:3 * c + 3]
            if q < 2 and i % 2 == 0:
                row[0] = hi
            elif q < 2 and i % 5 == 1:
                row[0] = lo
            elif q == 2 and i >= 10:
                row[0] = lo
            c += 1
    scores = _host(m, b)
    assert (scores == 1.0).sum() == 400 and (scores == np.float32(1e-6)).sum() > 290
    for k in (64, 128):
        idx, top = _check(m, b, k, k, scores)
        n1 = min(k, 100)  # request 1 has 100 scores of 1.0
        assert idx[0].tolist() == list(range(0, 2 * k, 2)) and idx[1].tolist()[:n1] == list(range(0, 2 * n1, 2))
        assert (top[0] == 1.0).all()
        low = idx[2][10:]
        assert (top[2][10:] == np.float32(1e-6)).all() and low.tolist() == list(range(10, 10 + k - 10))
    m.close()


# ---- 4. NaN and inf ----------------------------------------------------------------------------------------------------
def test_nan_and_inf():
    rng = np.random.default_rng(61)
    m = _models("canon", 8)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    counts = [40, 400, 10, 300]
    b = Batch([5] * len(counts), counts, [4] * sum(counts), rng, "canon", keys_from=HELD)
    bad = rng.random(b.N)
    for c in range(b.N):
        x = int(b.row_ptr[c])
        if bad[c] < 0.25 or c >= counts[0] + counts[1] and c < sum(counts[:3]):
            b.vals[x] = np.nan
        elif bad[c] < 0.35:
            b.vals[x] = np.inf
        elif bad[c] < 0.45:
            b.vals[x] = -np.inf
    scores = _host(m, b)
    assert np.isnan(scores).sum() > 100
    for k in (16, 128):
        idx, top = _check(m, b, k, k, scores)
        for q in range(b.R):
            n = min(k, counts[q])
            nan = np.isnan(scores[b.cand_ptr[q]:b.cand_ptr[q + 1]])
            numbers = int((~nan).sum())
            # the numbers first; then the NaN scores in index order
            assert not np.isnan(top[q, :min(numbers, n)]).any()
            tail = idx[q, numbers:n].tolist()
            assert tail == np.flatnonzero(nan)[:len(tail)].tolist()
        assert counts[2] < k and np.isnan(scores[b.cand_ptr[2]:b.cand_ptr[3]]).all()


# ---- 5. padding --------------------------------------------------------------------------------------------------------
def test_padding():
    rng = np.random.default_rng(67)
    m = _models("fm", 8)[(api.ABSENT_DEFAULT, False, api.PRECISION_F16)]
    b = _plain_batch([3, 0, 300, 1], rng)
    idx, top = _check(m, b, 512, "short requests")
    for q, n in enumerate([3, 0, 300, 1]):
        assert (idx[q, n:] == PAD_INDEX).all() and (_bits(top[q, n:]) == PAD_PCTR_BITS).all()
    b = _plain_batch([0, 0, 0], rng)
    for idx, top in (_rank_host(m, b, 5), _rank_dev(m, b, 5)[:2]):
        assert (idx == PAD_INDEX).all() and (_bits(top) == PAD_PCTR_BITS).all() and idx.shape == (3, 5)
    b = _plain_batch([], rng)
    assert _rank_host(m, b, 5)[0].shape == (0, 5)


# ---- 6. refusals -------------------------------------------------------------------------------------------------------
def _raw(m, b, k, index=True, **over):
    arr = {x: getattr(b, x) for x in ("ctx_ptr", "ctx_keys", "ctx_vals", "ctx_fields", "cand_ptr", "row_ptr", "keys",
                                      "vals", "fields")}
    addr = {x: (None if v is None else v.ctypes.data) for x, v in arr.items()}
    f = dict(requests=b.R, ctx_nnz=b.ctx_keys.size, candidates=b.N, nnz=b.keys.size, **addr)
    f.update(over)
    s = api.CandidateBatch(**f)
    out = np.empty(max(b.R * max(k, 1), 1), np.uint32)
    rc = api.lib().xf_model_rank_candidates_host(m.h, api.C.byref(s), k, api._p(out) if index else None, None)
    return rc, api.lib().xf_last_error().decode()


def _refused(m, b, k, code, pattern, index=True, **over):
    rc, msg = _raw(m, b, k, index, **over)
    assert rc == code and re.search(pattern, msg), (rc, msg, over)


def test_refusals():
    rng = np.random.default_rng(71)
    lr = _models("lr", 0)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    mv = _models("mvm", 8)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    b = Batch([3, 4], [2, 1], [2, 3, 1], rng, "lr")
    bm = Batch([3, 4], [2, 1], [2, 3, 1], rng, "mvm")
    assert _raw(lr, b, 4)[0] == 0 and _raw(mv, bm, 4)[0] == 0
    fn = "xf_model_rank_candidates_host"
    _refused(lr, b, 0, -1, fn + ": k = 0")
    _refused(lr, b, 1025, -1, fn + ": k = 1025")
    _refused(lr, b, 4, -1, fn + ": top_index is NULL", index=False)
    assert _raw(lr, Batch([], [], [], rng, "lr"), 4, index=False)[0] == 0
    # the checks of predict_candidates_host, one of each
    _refused(lr, b, 4, -1, "null argument", keys=None)
    _refused(mv, bm, 4, -1, "null argument", fields=None)
    _refused(lr, b, 4, -1, "cand_ptr decreases", cand_ptr=np.array([0, 4, 3], np.uint32).ctypes.data)
    _refused(lr, b, 4, -1, fn + ": cand_ptr runs from 0 to 2", cand_ptr=np.array([0, 2, 2], np.uint32).ctypes.data)
    _refused(lr, b, 4, -1, fn + ": ctx_ptr ends at 7, past ctx_nnz = 6", ctx_nnz=6)
    _refused(lr, b, 4, -1, fn + ": row_ptr ends at 6, past nnz = 5", nnz=5)
    bad = b.keys.copy()
    bad[1] = np.uint64(0xFFFFFFFFFFFFFFFF)
    _refused(lr, b, 4, -1, fn + ": keys: key .* at position 1 is reserved", keys=bad.ctypes.data)
    badf = bm.fields.copy()
    badf[2] = 32
    _refused(mv, bm, 4, -1, fn + ": fields: field id 32 of token 2", fields=badf.ctypes.data)
    _refused(lr, b, 4, -1, "ignores feature values", vals=np.ones(b.keys.size, np.float32).ctypes.data)
    _refused(lr, b, 4, -1, "xf_table_freeze_mvm", fields=np.zeros(16, np.uint8).ctypes.data)
    # a part
    t = api.Table(capacity=1 << 12)
    t.import_(HELD[:10], w=np.ones(10, np.float32))
    part = t.freeze_part()
    _refused(part, b, 4, -6, fn + ": the model is a part")
    part.close()
    t.close()
    # the device entry point
    torch = pytest.importorskip("torch")
    d = DeviceBatch(b, torch)
    outs = _outs(torch, b, 4)
    s = torch.cuda.current_stream()
    call = lambda k, idx=True, pc=True: lr.rank_candidates_device(
        b.R, d.addr("ctx_ptr"), d.addr("ctx_keys"), 7, d.addr("cand_ptr"), b.N, d.addr("row_ptr"), d.addr("keys"), 6,
        k, outs[0].data_ptr() if pc else 0, outs[1].data_ptr() if idx else 0, stream=s.cuda_stream)
    dfn = "xf_model_rank_candidates_device"
    for args, pattern in (((0,), dfn + ": k = 0"), ((1025,), dfn + ": k = 1025"),
                          ((4, False), dfn + ": top_index is NULL"), ((4, True, False), "null argument")):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*" + pattern):
            call(*args)
    call(4)
    torch.cuda.synchronize()


# ---- 7. the device entry point: streams in flight, no score output ----------------------------------------------------
def test_streams_and_no_pctr():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(73)
    m = _models("canon", 16)[(api.ABSENT_DEFAULT, False, api.PRECISION_F32)]
    b = Batch([9] * 6, [5, 700, 0, 250, 40, 3000], [6] * 3995, rng, "canon")
    k = 128
    want_i, want_p = _check(m, b, k, "first")
    d = DeviceBatch(b, torch)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    runs = []
    torch.cuda.synchronize()
    for _ in range(3):
        o1, o2 = _outs(torch, b, k), _outs(torch, b, k)
        torch.cuda.synchronize()
        _launch(m, d, k, o1, s1)
        _launch(m, d, k, o2, s2, with_pctr=False)
        runs.append((o1, o2))
    s1.synchronize()
    s2.synchronize()
    for o1, o2 in runs:
        i1, p1, _ = _fetch(b, k, o1)
        i2, p2, _ = _fetch(b, k, o2)
        assert np.array_equal(i1, want_i) and np.array_equal(_bits(p1), _bits(want_p))
        assert np.array_equal(i2, want_i) and (p2 == 3.0).all()  # d_top_pctr = NULL: nothing written there

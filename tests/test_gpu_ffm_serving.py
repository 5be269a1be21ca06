"""Field-aware FM serving models (xf_table_freeze_ffm, csrc/serve.cu): an FFM-trained canonical table frozen into rows
{key, w, 0, v[L]} predicts on field ids and feature values, bit for bit, what the table's own predict returns at the
moment of the freeze, on every row; scores candidates as the flat predict of "context, then candidate"; leaves the table
alone; never inserts; and its files, deltas and F16 conversion are the canonical rows' with fm = 4."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

import canonical_serving_model as CM
import compact_serving_model as CS
import ffm_serving_model as FS
import serving_model as SM
from ffm_model import FFM64, sigmoid_ref
from rank_model import rank_model
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

B, D, SPACE, N = 256, 12, 6000, 3  # training rows, tokens per row, id space, batches
CAP = 1 << 15
MAX_NNZ = 1 << 15
ROW_LENS = [0, 1, 3, 31, 32, 33, 65, 129, 300] + [8] * 25
ERR_ARG, ERR_IO, ERR_STATE = "error -1:", "error -4:", "error -6:"
CASES = [(L, api.OPT_FTRL) for L in FS.LATENT_DIMS] + [(L, api.OPT_SGD) for L in (16, 128)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _keys_of(ids):
    return api.hash_decimal_ids(np.asarray(ids, np.uint64))


def _pulled():
    """Keys a Pull inserted and no batch trained: default rows, latent block not materialised."""
    return _keys_of(np.arange(5 * SPACE, 5 * SPACE + 200))


def _unseen():
    return _keys_of(np.arange(9 * SPACE, 9 * SPACE + 300))


def _vals(rng, n):
    """Feature values with negatives and exact zeros."""
    x = rng.uniform(-1.5, 2.0, n).astype(np.float32)
    x[rng.random(n) < 0.1] = 0.0
    return x


def _make(L, opt, capacity=CAP, max_rows=1024, max_nnz=MAX_NNZ):
    t = api.Table(latent_dim=L, optimizer=opt, v_init=api.VINIT_COUNTER, seed=7, capacity=capacity, canonical_fm=1)
    tr = api.Trainer(t, model=api.MODEL_FFM, max_rows=max_rows, max_nnz=max_nnz)
    return t, tr


def _train(t, tr, first=0, n=N, pull=True):
    """Train n batches, then give the trained keys w and latent rows of N(0, 0.5): the initial values (N(0, 0.01)) and
    a few steps leave pair sums so close to 0 that most predictions would round alike."""
    F = t.K // 4
    seen = []
    for i in range(first, first + n):
        rp, ids, _ = datagen.make_ids(500 + i, B, D, SPACE, dist="zipf")
        rng = np.random.default_rng(500 + i)
        keys = _keys_of(ids)
        tr.step_host_fields(rp, keys, rng.integers(0, F, ids.size).astype(np.uint8), _vals(rng, ids.size),
                            (rng.random(B) < 0.3).astype(np.uint8))
        seen.append(keys)
    trained = np.unique(np.concatenate(seen))
    rng = np.random.default_rng(first)
    t.import_(trained, w=rng.normal(0, 0.5, trained.size).astype(np.float32),
              v=rng.normal(0, 0.5, (trained.size, t.K)).astype(np.float32))
    if pull:
        t.pull(_pulled(), want_v=False)
    return trained


def _csr(lens):
    rp = np.zeros(len(lens) + 1, np.uint32)
    rp[1:] = np.cumsum(lens)
    return rp


def _query(seed, trained, L, lens=ROW_LENS):
    """Rows of every length over trained, pulled and unseen keys, several tokens per field and every field id below F,
    one key four times in the longer rows; values scaled by 1 / sqrt(row length)."""
    rng = np.random.default_rng(seed)
    F = L // 4
    pool = np.concatenate([trained, _pulled(), _unseen()])
    rows = []
    for n in lens:
        k = pool[rng.integers(0, pool.size, n)]
        if n >= 8:
            k[n // 2:n // 2 + 3] = k[0]
        rows.append(k)
    rp = _csr([r.size for r in rows])
    keys = np.concatenate(rows).astype(np.uint64)
    f = rng.integers(0, F, keys.size).astype(np.uint8)
    f[:min(F, f.size)] = np.arange(min(F, f.size))
    scale = np.repeat(1.0 / np.sqrt(np.maximum(np.diff(rp.astype(np.int64)), 1)), np.diff(rp.astype(np.int64)))
    return rp, keys, f, (_vals(rng, keys.size) * scale).astype(np.float32)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _device(m, rp, keys, f, vals, stream=None):
    torch = pytest.importorskip("torch")
    s = stream or torch.cuda.Stream()
    d_rp, d_keys = torch.from_numpy(rp.astype(np.int32)).cuda(), torch.from_numpy(keys.view(np.int64)).cuda()
    d_f = torch.from_numpy(np.ascontiguousarray(f, np.uint8)).cuda()
    d_vals = None if vals is None else torch.from_numpy(vals).cuda()
    d_out = torch.full((rp.size - 1,), -1.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    m.predict_device_fields(d_rp.data_ptr(), d_keys.data_ptr(), d_f.data_ptr(), rp.size - 1, keys.size, d_out.data_ptr(),
                            stream=s.cuda_stream, d_vals=0 if d_vals is None else d_vals.data_ptr())
    s.synchronize()
    return d_out.cpu().numpy()


@pytest.fixture
def trained16():
    t, tr = _make(16, api.OPT_FTRL)
    yield t, tr, _train(t, tr)
    tr.close()
    t.close()


# ---- 1. bit for bit with the table's predict, every row -------------------------------------------------------------
@pytest.mark.parametrize("L,opt", CASES)
def test_predict_equals_the_tables_bit_for_bit(L, opt):
    t, tr = _make(L, opt)
    trained = _train(t, tr)
    rp, keys, f, vals = _query(L + 3, trained, L)
    models = {p: t.freeze_ffm(prune=p) for p in (False, True)}
    got = {}
    for p, m in models.items():
        for v in (None, 1):
            x = None if v is None else vals
            got[(p, v, "host")] = m.predict_host_fields(rp, keys, f, x)
            got[(p, v, "device")] = _device(m, rp, keys, f, x)
    # after the models: the table's predict inserts the unseen keys
    want = {None: tr.predict_host_fields(rp, keys, f, None), 1: tr.predict_host_fields(rp, keys, f, vals)}
    for (p, v, path), g in got.items():
        assert np.array_equal(_bits(g), _bits(want[v])), (p, v, path)
    assert len(set(want[1].tolist())) > 10 and len(set(want[None].tolist())) > 10
    info = models[True].info()
    assert info["fm"] == FS.FM_FFM and info["absent"] == api.ABSENT_DEFAULT and info["pruned_keys"] >= _pulled().size
    assert info["row_bytes"] == CM.row_bytes(L) and models[False].info()["pruned_keys"] == 0
    # field ids are read & (F - 1) on the device
    F = L // 4
    assert np.array_equal(_bits(_device(models[True], rp, keys, f + np.uint8(F) * (f < 2), vals)), _bits(want[1]))
    # the float64 definition
    uk, idx = np.unique(keys, return_inverse=True)
    e = t.export(uk)
    y64 = FFM64(e["w"], e["v"].reshape(uk.size, L), "ftrl").forward(idx, rp.astype(np.int64), f, vals)
    p64 = sigmoid_ref(y64)
    assert np.all(np.abs(got[(True, 1, "host")] - p64) <= 1e-4 + 1e-4 * np.abs(p64))
    for m in models.values():
        m.close()
    tr.close()
    t.close()


def test_large_batch_at_128():
    """65 536 rows of one token per field and Zipf ids at L = 128, host and device, against the table and float64."""
    L, F, rows = 128, 32, 65536
    t, tr = _make(L, api.OPT_FTRL, capacity=1 << 17, max_rows=rows, max_nnz=rows * F)
    trained = _train(t, tr)
    _, ids, _ = datagen.make_ids(77, rows, F, 4 * SPACE, dist="zipf")
    rp = _csr([F] * rows)
    keys = _keys_of(ids).astype(np.uint64)
    f = np.tile(np.arange(F, dtype=np.uint8), rows)
    vals = _vals(np.random.default_rng(3), keys.size) * np.float32(0.2)
    m = t.freeze_ffm()
    got_h, got_d = m.predict_host_fields(rp, keys, f, vals), _device(m, rp, keys, f, vals)
    want = tr.predict_host_fields(rp, keys, f, vals)
    assert np.array_equal(_bits(got_h), _bits(want)) and np.array_equal(_bits(got_d), _bits(want))
    assert np.unique(want).size > 1000 and trained.size > 0
    uk, idx = np.unique(keys, return_inverse=True)
    e = t.export(uk)
    p64 = sigmoid_ref(FFM64(e["w"], e["v"].reshape(uk.size, L), "ftrl").forward(idx, rp.astype(np.int64), f, vals))
    assert np.all(np.abs(got_h - p64) <= 1e-4 + 1e-4 * np.abs(p64))
    m.close()
    tr.close()
    t.close()


# ---- 2. absent keys under ZERO read as rows of zeros ---------------------------------------------------------------
def test_absent_zero_equals_the_table_with_zero_rows(trained16):
    t, tr, trained = trained16
    rp, keys, f, vals = _query(21, trained, 16)
    vals[5], vals[50] = np.nan, -np.inf
    mz, md = t.freeze_ffm(absent=api.ABSENT_ZERO), t.freeze_ffm()
    assert mz.info()["absent"] == api.ABSENT_ZERO
    got_z, got_d = mz.predict_host_fields(rp, keys, f, vals), md.predict_host_fields(rp, keys, f, vals)
    got_zd = _device(mz, rp, keys, f, vals)
    uk = np.unique(keys)
    lacks = uk[mz.lookup_latent(uk)["present"] == 0]
    assert lacks.size > 10
    t.import_(lacks, w=np.zeros(lacks.size, np.float32), v=np.zeros((lacks.size, 16), np.float32))
    want = tr.predict_host_fields(rp, keys, f, vals)
    assert np.array_equal(_bits(got_z), _bits(want)) and np.array_equal(_bits(got_zd), _bits(want))
    assert not np.array_equal(_bits(got_d), _bits(want))


# ---- 3. contents and prune ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [8, 64])
def test_contents_and_prune(L):
    t, tr = _make(L, api.OPT_FTRL)
    trained = _train(t, tr)
    zeros = _keys_of(np.arange(7 * SPACE, 7 * SPACE + 50))  # materialised rows of zeros: ZERO prunes them, DEFAULT not
    zv = np.zeros((zeros.size, L), np.float32)
    zv[::2, 1] = -0.0
    zw = np.zeros(zeros.size, np.float32)
    zw[1::2] = -0.0
    t.import_(zeros, w=zw, v=zv)
    src = t.list_keys()
    e = t.export(src)
    v_ready = ~np.isin(src, _pulled())
    rp, keys, f, vals = _query(77, np.concatenate([trained, zeros]), L)
    vals[3], vals[40], vals[41] = np.nan, np.inf, -np.inf
    for absent in (api.ABSENT_DEFAULT, api.ABSENT_ZERO):
        m_all = t.freeze_ffm(absent=absent, prune=False)
        a = m_all.lookup_latent(src)
        assert a["present"].all()
        assert np.array_equal(_bits(a["w"]), _bits(e["w"])) and np.array_equal(_bits(a["v"]), _bits(e["v"].reshape(src.size, L)))
        m = t.freeze_ffm(absent=absent)
        got = m.lookup_latent(src)
        rule = CM.pruned(e["w"], absent, v_ready, e["v"].reshape(src.size, L))
        assert np.array_equal(got["present"] == 0, rule)
        assert rule.sum() >= (_pulled().size if absent == api.ABSENT_DEFAULT else zeros.size)
        info = m.info()
        assert info["keys"] + info["pruned_keys"] == info["source_keys"] == src.size
        assert info["fm"] == FS.FM_FFM and info["latent_dim"] == L and info["row_bytes"] == CM.row_bytes(L)
        # pruning never changes a prediction, NaN and Inf values included, on either path
        for x in (None, vals):
            pa, pp = m_all.predict_host_fields(rp, keys, f, x), m.predict_host_fields(rp, keys, f, x)
            assert np.array_equal(_bits(pa), _bits(pp)), absent
            assert np.array_equal(_bits(_device(m, rp, keys, f, x)), _bits(pp)), absent
        assert np.isnan(pp).any()
        m.close()
        m_all.close()
    tr.close()
    t.close()


# ---- 4. the table is left alone, the model never inserts -----------------------------------------------------------
def test_freeze_leaves_the_table_alone(trained16, tmp_path):
    t, tr, trained = trained16
    src = t.list_keys()
    ex = {k: np.asarray(v).tobytes() for k, v in t.export(src).items()}
    t.save_state(str(tmp_path / "a"))
    canon_before, mvm_before = t.freeze_canonical(), t.freeze_mvm()
    m1 = t.freeze_ffm()
    m2 = t.freeze_ffm(absent=api.ABSENT_ZERO, prune=False)
    t.save_state(str(tmp_path / "b"))
    assert (tmp_path / "a").read_bytes() == (tmp_path / "b").read_bytes()
    assert {k: np.asarray(v).tobytes() for k, v in t.export(src).items()} == ex
    size, info = t.size(), m1.info()
    rp, keys, f, vals = _query(5, trained, 16)
    m1.predict_host_fields(rp, keys, f, vals)
    _device(m2, rp, keys, f, vals)
    assert t.size() == size and m1.info() == info
    # the canonical and MVM freezes of the same table are what they were
    canon, mvm = t.freeze_canonical(), t.freeze_mvm()
    assert canon.info()["fm"] == 2 and mvm.info()["fm"] == 3
    assert np.array_equal(_bits(canon.predict_host(rp, keys, vals)), _bits(canon_before.predict_host(rp, keys, vals)))
    assert np.array_equal(_bits(mvm.predict_host_fields(rp, keys, f, vals)), _bits(mvm_before.predict_host_fields(rp, keys, f, vals)))
    for m in (m1, m2, canon, mvm, canon_before, mvm_before):
        m.close()


# ---- 5. F16 ------------------------------------------------------------------------------------------------------
def test_f16_models(trained16, tmp_path):
    t, tr, trained = trained16
    m = t.freeze_ffm()
    h16 = m.convert(api.PRECISION_F16)
    info = h16.info()
    assert info["precision"] == 1 and info["fm"] == FS.FM_FFM and info["row_bytes"] == FS.row_bytes(16, api.PRECISION_F16)
    rp, keys, f, vals = _query(9, trained, 16)
    got = {"host": h16.predict_host_fields(rp, keys, f, vals), "device": _device(h16, rp, keys, f, vals)}
    cb = FS.candidate_batch(np.random.default_rng(4), np.concatenate([trained, _pulled(), _unseen()]), 4,
                            [0, 3, 17, 2], [0, 5, 2, 9], [0, 1, 4, 40])
    got_c = h16.predict_candidates(*cb)
    # the F32 model of a table holding the binary16-rounded v of the model's keys
    src = t.list_keys()
    held = src[m.lookup_latent(src)["present"] == 1]
    e = t.export(held)
    t.import_(held, w=e["w"], v=CS.to_half(e["v"].reshape(held.size, 16)).astype(np.float32))
    ref = t.freeze_ffm()
    for path, g in got.items():
        assert np.array_equal(_bits(g), _bits(ref.predict_host_fields(rp, keys, f, vals))), path
    assert np.array_equal(_bits(got_c), _bits(ref.predict_candidates(*cb)))
    back = h16.convert(api.PRECISION_F32)
    assert np.array_equal(_bits(back.predict_host_fields(rp, keys, f, vals)), _bits(got["host"]))
    p = str(tmp_path / "h.xfsm")
    h16.save(p)
    assert struct.unpack_from("<i", open(p, "rb").read(), 36)[0] == FS.FM_FFM
    loaded = api.Model.load(p)
    assert np.array_equal(_bits(loaded.predict_host_fields(rp, keys, f, vals)), _bits(got["host"]))
    # conversion never saturates
    big = _keys_of(np.arange(11 * SPACE, 11 * SPACE + 3))
    v = np.zeros((3, 16), np.float32)
    v[1, 7] = 70000.0
    t.import_(big, w=np.ones(3, np.float32), v=v)
    mb = t.freeze_ffm()
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*65520"):
        mb.convert(api.PRECISION_F16)
    for x in (m, h16, ref, back, loaded, mb):
        x.close()


# ---- 6. files ----------------------------------------------------------------------------------------------------
def _header(data):
    return dict(zip(SM.FIELDS, SM.HEADER.unpack(data[:SM.HEADER.size])))


def _with_header(data, **fields):
    """The file with header fields replaced and the header checksum recomputed."""
    head = list(SM.HEADER.unpack(data[:SM.HEADER.size]))
    for k, v in fields.items():
        head[SM.FIELDS.index(k)] = v
    head[-1] = SM.section_sum(SM.HEADER.pack(*head)[:96])
    return SM.HEADER.pack(*head) + data[SM.HEADER.size:]


def test_file_round_trip_layout_and_damage(trained16, tmp_path):
    t, tr, trained = trained16
    m = t.freeze_ffm()
    p = str(tmp_path / "m.xfsm")
    m.save(p)
    data = open(p, "rb").read()
    h, rows = FS.parse_model_file(data)
    info = m.info()
    assert struct.unpack_from("<i", data, 36)[0] == 4 and h["row_bytes"] == 96 and h["keys"] == info["keys"]
    lk = m.lookup_latent(rows["key"])
    assert lk["present"].all() and np.array_equal(_bits(lk["v"]), _bits(rows["v"])) and np.array_equal(_bits(lk["w"]), _bits(rows["w"]))
    args = (h["optimizer"], h["absent"], h["v_init"], h["v_const"], h["seed"], h["source_keys"])
    assert FS.model_file(CM.rows_array(rows["key"], lk["w"], lk["v"]), 16, api.PRECISION_F32, *args) == data
    assert CM.fingerprint(rows) == m.fingerprint()
    back = api.Model.load(p)
    assert back.info() == info
    rp, keys, f, vals = _query(31, trained, 16)
    assert np.array_equal(_bits(back.predict_host_fields(rp, keys, f, vals)), _bits(m.predict_host_fields(rp, keys, f, vals)))
    p2 = str(tmp_path / "m2.xfsm")
    back.save(p2)
    assert open(p2, "rb").read() == data
    back.close()
    bad = str(tmp_path / "bad")

    def refused(blob):
        open(bad, "wb").write(blob)
        with pytest.raises(api.XflowError, match=ERR_IO):
            api.Model.load(bad)

    for byte in (12, 15, 16 + 64 + 5):  # padding, with checksums that pass
        raw = bytearray(rows.tobytes())
        raw[CM.row_bytes(16) * (rows.size // 2) + byte] = 1
        refused(FS.model_file(np.frombuffer(bytes(raw), rows.dtype), 16, api.PRECISION_F32, *args))
    refused(_with_header(data, latent_dim=12))
    refused(_with_header(data, latent_dim=256))
    refused(_with_header(data, row_bytes=128))
    refused(_with_header(data, fm=5))
    api.Model.load(p).close()
    m.close()


# ---- 7. deltas ---------------------------------------------------------------------------------------------------
def _saved(m, path):
    m.save(str(path))
    return path.read_bytes()


def test_delta_chain(tmp_path):
    L = 32
    t, tr = _make(L, api.OPT_FTRL)
    _train(t, tr, 0, 2)
    models = [t.freeze_ffm()]
    for i in range(3):
        _train(t, tr, 10 + i, 1, pull=False)
        models.append(t.freeze_ffm())
    for i in range(3):
        base, nxt = models[i], models[i + 1]
        d = base.diff(nxt)
        dp = str(tmp_path / ("d%d.xfsd" % i))
        d.save(dp)
        data = open(dp, "rb").read()
        assert struct.unpack_from("<i", data, 16)[0] == FS.FM_FFM
        dl = api.Delta.load(dp)
        r = base.apply(dl)
        assert _saved(r, tmp_path / "r") == _saved(nxt, tmp_path / "n")
        assert r.fingerprint() == nxt.fingerprint() == d.info()["result_fingerprint"]
        r.close()
    # a canonical model and a field-aware FM's of one table: equal L, equal bytes, different fm
    c = t.freeze_canonical()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*fm"):
        c.diff(models[-1])
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*fm"):
        models[-1].diff(c)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*fm"):
        models[-1].apply(c.diff(t.freeze_canonical()))
    for m in models + [c]:
        m.close()
    tr.close()
    t.close()


# ---- 8. candidates and ranking -----------------------------------------------------------------------------------
def _cand_device(m, ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals, vals, ctx_fields, fields, k=None):
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(
        {1: np.uint8, 4: np.int32, 8: np.int64}[np.asarray(a).dtype.itemsize])).cuda()
    a = [dev(x) for x in (ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals, vals, ctx_fields, fields)]
    N = row_ptr.size - 1
    out = torch.full((max(N, 1),), -1.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    m.predict_candidates_device(cand_ptr.size - 1, a[0].data_ptr(), a[1].data_ptr(), ctx_keys.size, a[2].data_ptr(), N,
                                a[3].data_ptr(), a[4].data_ptr(), keys.size, out.data_ptr(), stream=s.cuda_stream,
                                d_ctx_vals=a[5].data_ptr(), d_vals=a[6].data_ptr(), d_ctx_fields=a[7].data_ptr(),
                                d_fields=a[8].data_ptr())
    s.synchronize()
    return out.cpu().numpy()[:N]


@pytest.mark.parametrize("L", FS.LATENT_DIMS)
def test_candidates_equal_flat_predict(L):
    t, tr = _make(L, api.OPT_FTRL)
    trained = _train(t, tr)
    pool = np.concatenate([trained, _pulled(), _unseen()])
    rng = np.random.default_rng(L)
    # empty contexts and candidates, requests across runs of 16, several tokens per field on both sides
    counts = [0, 1, 16, 17, 40, 3, 0, 33]
    ctx_lens = [0, 5, 9, 0, 31, 70, 2, 12]
    cb = FS.candidate_batch(rng, pool, L // 4, counts, ctx_lens, [0, 1, 2, 3, 8, 33, 65])
    m = t.freeze_ffm()
    h16 = m.convert(api.PRECISION_F16)
    for model in (m, h16):
        want = model.predict_host_fields(*FS.concatenated(*cb))
        got_h = model.predict_candidates(*cb)
        got_d = _cand_device(model, *cb)
        assert np.array_equal(_bits(got_h), _bits(want)) and np.array_equal(_bits(got_d), _bits(want))
        for k in (1, 5, 64):
            idx, pc = model.rank_candidates(*cb[:5], k, *cb[5:])
            wi, wp = rank_model(got_h, cb[2], k)
            assert np.array_equal(idx, wi) and np.array_equal(_bits(pc), _bits(wp))
    assert len(set(want.tolist())) > 20
    for x in (m, h16):
        x.close()
    tr.close()
    t.close()


def test_one_request_of_65536_candidates(trained16):
    t, tr, trained = trained16
    pool = np.concatenate([trained, _pulled(), _unseen()])
    cb = FS.candidate_batch(np.random.default_rng(8), pool, 4, [65536], [8], [8])
    m = t.freeze_ffm()
    want = m.predict_host_fields(*FS.concatenated(*cb))
    got = m.predict_candidates(*cb)
    assert np.array_equal(_bits(got), _bits(want)) and np.array_equal(_bits(_cand_device(m, *cb)), _bits(want))
    idx, pc = m.rank_candidates(*cb[:5], 100, *cb[5:])
    wi, wp = rank_model(got, cb[2], 100)
    assert np.array_equal(idx, wi) and np.array_equal(_bits(pc), _bits(wp))
    m.close()


# ---- 9. concurrency: device predicts in flight on two streams, the first call on the device at L = 128 ---------------
_STREAMS = r"""
import numpy as np, torch
from xflow_b200 import api
t = api.Table(latent_dim=128, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=7, capacity=1 << 15, canonical_fm=1)
rng = np.random.default_rng(1)
keys = api.hash_decimal_ids(np.arange(3000, dtype=np.uint64))
t.import_(keys, w=rng.normal(0, 0.5, keys.size).astype(np.float32), v=rng.normal(0, 0.5, (keys.size, 128)).astype(np.float32))
m = t.freeze_ffm()
rows = 4096
rp = np.arange(rows + 1, dtype=np.uint32) * 32
q = keys[rng.integers(0, keys.size + 500, rows * 32) % keys.size]
f = np.tile(np.arange(32, dtype=np.uint8), rows)
d_rp, d_k, d_f = (torch.from_numpy(a).cuda() for a in (rp.astype(np.int32), q.view(np.int64), f))
outs = [torch.full((rows,), -1.0, device="cuda") for _ in range(2)]
streams = [torch.cuda.Stream() for _ in range(2)]
torch.cuda.synchronize()
for s, o in zip(streams, outs):
    m.predict_device_fields(d_rp.data_ptr(), d_k.data_ptr(), d_f.data_ptr(), rows, q.size, o.data_ptr(), stream=s.cuda_stream)
torch.cuda.synchronize()
want = m.predict_host_fields(rp, q, f)
for o in outs:
    assert np.array_equal(o.cpu().numpy().view(np.uint32), want.view(np.uint32))
print("ok")
"""


def test_two_streams_first_call_on_the_device():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", _STREAMS], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


# ---- 10. refusals ------------------------------------------------------------------------------------------------
def test_refusals(trained16):
    torch = pytest.importorskip("torch")
    t, tr, trained = trained16
    # canonical_fm = 0 (a canonical table's latent_dim and shard count are checked at its creation, so no table
    # reaches the freeze's latent_dim and num_shards refusals)
    lr = api.Table(capacity=1 << 12)
    shard = api.Table(latent_dim=8, shard_index=0, num_shards=2, capacity=1 << 12)
    for x in (lr, shard):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*xf_table_freeze_ffm.*canonical_fm = 0"):
            x.freeze_ffm()
        x.close()
    m = t.freeze_ffm()
    rp = np.array([0, 2], np.uint32)
    keys = trained[:2].copy()
    ones = np.ones(2, np.float32)
    fields_fn = "predict_host_fields or xf_model_predict_device_fields"
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*field-aware FM.*" + fields_fn):
        m.predict_host(rp, keys)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*" + fields_fn):
        m.predict_host(rp, keys, ones)
    d_rp = torch.from_numpy(rp.astype(np.int32)).cuda()
    d_keys = torch.from_numpy(keys.view(np.int64)).cuda()
    d_out = torch.empty(1, dtype=torch.float32, device="cuda")
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*" + fields_fn):
        m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), 1, 2, d_out.data_ptr())
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*" + fields_fn):
        m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), 1, 2, d_out.data_ptr(), d_vals=d_out.data_ptr())
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*xf_model_predict_ingested.*" + fields_fn):
        m.predict_ingested(tr, 0, 0)
    # field ids below F = L / 4, on every side, naming the token, the id and the bound
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*field id 4 of token 1.*F = 4"):
        m.predict_host_fields(rp, keys, np.array([0, 4], np.uint8))
    cb = FS.candidate_batch(np.random.default_rng(1), trained, 4, [2], [3], [2])
    bad_ctx = list(cb)
    bad_ctx[7] = cb[7].copy()
    bad_ctx[7][2] = 9
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*ctx_fields: field id 9 of token 2.*F = 4"):
        m.predict_candidates(*bad_ctx)
    bad = list(cb)
    bad[8] = cb[8].copy()
    bad[8][1] = 200
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*fields: field id 200 of token 1.*F = 4"):
        m.rank_candidates(*bad[:5], 1, *bad[5:])
    # a NULL fields array with tokens
    assert api.lib().xf_model_predict_device_fields(m.h, api._p(d_rp.data_ptr()), api._p(d_keys.data_ptr()), None, None,
                                                    1, 2, api._p(d_out.data_ptr()), None) == -1
    with pytest.raises(api.XflowError, match=ERR_ARG):
        m.predict_candidates(*cb[:7], None, cb[8])
    # lookup: st, qt are not in a field-aware FM's row
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*field-aware FM.*xf_model_lookup_latent"):
        m.lookup(keys)
    lk = m.lookup_latent(keys)
    assert lk["present"].all() and lk["v"].shape == (2, 16)
    # models without field ids still refuse them, naming both freezes
    f = np.zeros(2, np.uint8)
    for o in (t.freeze_canonical(), api.Table(latent_dim=8, capacity=1 << 12).freeze(), api.Table(capacity=1 << 12).freeze()):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*xf_table_freeze_mvm or xf_table_freeze_ffm"):
            o.predict_host_fields(rp, keys, f)
        o.close()
    m.close()

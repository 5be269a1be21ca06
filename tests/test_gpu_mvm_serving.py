"""Multi-view machine serving models (xf_table_freeze_mvm, csrc/serve.cu): an MVM-trained canonical table frozen into
rows {key, 0, v[K]} predicts on field ids and feature values, bit for bit, what the table's own predict does wherever
that is reproducible, and the numpy float32 statement (mvm_serving_model.py) everywhere; holds what xf_table_export
returns; leaves the table alone; never inserts; and its files, deltas and F16 conversion follow the numpy statement."""
import struct

import numpy as np
import pytest

import compact_serving_model as CS
import fm_model as FMM
import mvm_serving_model as MV
import serving_model as SM
from common import assert_close
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

B, D, SPACE, N, F = 256, 12, 6000, 3, 5  # training rows, tokens per row, id space, batches, fields
CAP = 1 << 15
MAX_NNZ = 1 << 15
ROW_LENS = [0, 1, 3, 31, 32, 33, 65, 129, 300] + [8] * 25
ERR_ARG, ERR_IO, ERR_STATE = "error -1:", "error -4:", "error -6:"
CASES = [(K, api.OPT_FTRL) for K in MV.LATENT_DIMS] + [(K, api.OPT_SGD) for K in (8, 32)]


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


def _batch(seed):
    rp, ids, _ = datagen.make_ids(seed, B, D, SPACE, dist="zipf")
    rng = np.random.default_rng(seed)
    lab = (rng.random(B) < 0.3).astype(np.uint8)
    return rp, _keys_of(ids), rng.integers(0, F, ids.size).astype(np.uint8), _vals(rng, ids.size), lab


def _make(K, opt, capacity=CAP):
    t = api.Table(latent_dim=K, optimizer=opt, v_init=api.VINIT_COUNTER, seed=7, capacity=capacity, canonical_fm=1)
    tr = api.Trainer(t, model=api.MODEL_MVM, max_rows=1024, max_nnz=MAX_NNZ)
    return t, tr


def _train(t, tr, first=0, n=N, pull=True):
    """Train n batches, then give the trained keys latent rows of N(0, 0.7): the initial values (N(0, 0.01)) and a few
    steps leave products over fields so close to 0 that every prediction would round to sigmoid(0)."""
    seen = []
    for i in range(first, first + n):
        rp, keys, fields, vals, lab = _batch(500 + i)
        tr.step_host_fields(rp, keys, fields, vals, lab)
        seen.append(keys)
    trained = np.unique(np.concatenate(seen))
    rng = np.random.default_rng(first)
    t.import_(trained, w=np.zeros(trained.size, np.float32), v=rng.normal(0, 0.7, (trained.size, t.K)).astype(np.float32))
    if pull:
        t.pull(_pulled(), want_v=False)
    return trained


def _csr(lens):
    rp = np.zeros(len(lens) + 1, np.uint32)
    rp[1:] = np.cumsum(lens)
    return rp


def _query_cf(seed, trained, K, rows=48):
    """Rows the table predicts reproducibly, over at most 8 fields each (ids up to 31): half with fields cycling within
    each pass of T = 128 / K tokens (three passes where T <= 8, else one pass of up to 8 tokens), half with at most two
    tokens per field; keys trained, pulled and never seen."""
    rng = np.random.default_rng(seed)
    T = 128 // K
    pool = np.concatenate([trained, _pulled(), _unseen()])
    lens, fields = [], []
    for r in range(rows):
        if r % 2:
            n = int(rng.integers(1, (3 * T if T <= 8 else 8) + 1))
            fields.append(((np.arange(n) % min(T, 8) + r) % MV.FIELDS).astype(np.uint8))
        else:
            n = int(rng.integers(1, 17))
            fields.append(((rng.permutation(np.repeat(np.arange(8), 2))[:n] + 3 * r) % MV.FIELDS).astype(np.uint8))
        lens.append(n)
    rp = _csr(lens)
    keys = pool[rng.integers(0, pool.size, int(rp[-1]))].astype(np.uint64)
    f = np.concatenate(fields)
    assert MV.collision_free(rp, f, K).all()
    return rp, keys, f, _vals(rng, keys.size)


def _query_all(seed, trained, lens=ROW_LENS):
    """Rows of every length with many tokens per field (ids 0 .. 3 and 31), one key four times in the longer rows; the
    values are scaled by 1 / sqrt(row length), so that a field's sum stays near 1 in rows of any length."""
    rng = np.random.default_rng(seed)
    pool = np.concatenate([trained, _pulled(), _unseen()])
    rows = []
    for n in lens:
        k = pool[rng.integers(0, pool.size, n)]
        if n >= 8:
            k[n // 2:n // 2 + 3] = k[0]
        rows.append(k)
    rp = _csr([r.size for r in rows])
    keys = np.concatenate(rows).astype(np.uint64)
    f = rng.choice(np.array([0, 1, 2, 3, 31], np.uint8), keys.size)
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


# ---- 1. bit for bit with the table where the table is reproducible -----------------------------------------------
@pytest.mark.parametrize("K,opt", CASES)
def test_predict_equals_the_tables_bit_for_bit(K, opt):
    t, tr = _make(K, opt)
    trained = _train(t, tr)
    rp, keys, f, vals = _query_cf(K + 3, trained, K)
    models = {p: t.freeze_mvm(prune=p) for p in (False, True)}
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
    assert info["fm"] == MV.FM_MVM and info["absent"] == api.ABSENT_DEFAULT and info["pruned_keys"] >= _pulled().size
    assert info["row_bytes"] == MV.row_bytes(K) and models[False].info()["pruned_keys"] == 0
    for m in models.values():
        m.close()
    tr.close()
    t.close()


# ---- 2. every row: the numpy statement, the float64 definition, and the same bits on every path --------------------
@pytest.mark.parametrize("K", [4, 16, 32])
def test_all_rows_follow_the_statement(K):
    torch = pytest.importorskip("torch")
    t, tr = _make(K, api.OPT_FTRL)
    trained = _train(t, tr)
    m = t.freeze_mvm()
    rp, keys, f, vals = _query_all(40 + K, trained)
    assert not MV.collision_free(rp, f, K).all()
    got = {v: m.predict_host_fields(rp, keys, f, None if v is None else vals) for v in (None, 1)}
    tr.predict_host_fields(rp, keys, f, vals)  # inserts the unseen keys: export then reads what the model read
    v = t.export(keys)["v"].reshape(keys.size, K)
    for key, x in ((None, None), (1, vals)):
        _, p32 = MV.forward(rp, f, x, v)
        gap = np.abs(_bits(got[key]).astype(np.int64) - _bits(p32).astype(np.int64))
        assert gap.max() <= 1, (key, gap.max())
        p64 = FMM.sigmoid(MV.forward64(rp, f, x, v))
        assert_close(got[key], p64, "MVM model vs float64, K=%d" % K, rel=1e-4, abs_floor=1e-6)
    # repeated calls, the device path on a non-default stream, and the rows in another order give the same bits
    assert np.array_equal(_bits(m.predict_host_fields(rp, keys, f, vals)), _bits(got[1]))
    s = torch.cuda.Stream()
    assert np.array_equal(_bits(_device(m, rp, keys, f, vals, s)), _bits(got[1]))
    assert np.array_equal(_bits(_device(m, rp, keys, f, None, s)), _bits(got[None]))
    order = np.random.default_rng(K).permutation(rp.size - 1)
    lens = np.diff(rp.astype(np.int64))[order]
    idx = np.concatenate([np.arange(rp[r], rp[r + 1]) for r in order]).astype(np.int64)
    shuffled = m.predict_host_fields(_csr(lens), keys[idx], f[idx], vals[idx])
    assert np.array_equal(_bits(shuffled), _bits(got[1][order]))
    # field ids are read & 31 on the device
    assert np.array_equal(_bits(_device(m, rp, keys, f + np.uint8(32) * (f < 8), vals, s)), _bits(got[1]))
    m.close()
    tr.close()
    t.close()


# ---- 3. absent keys under ZERO read as rows of zeros ------------------------------------------------------------
def test_absent_zero_equals_the_table_with_zero_rows(trained16):
    t, tr, trained = trained16
    rp, keys, f, vals = _query_cf(21, trained, 16)
    mz = t.freeze_mvm(absent=api.ABSENT_ZERO)
    md = t.freeze_mvm()
    assert mz.info()["absent"] == api.ABSENT_ZERO
    got_z, got_d = mz.predict_host_fields(rp, keys, f, vals), md.predict_host_fields(rp, keys, f, vals)
    uk = np.unique(keys)
    lacks = uk[mz.lookup_latent(uk)["present"] == 0]
    assert lacks.size > 10
    t.import_(lacks, w=np.zeros(lacks.size, np.float32), v=np.zeros((lacks.size, 16), np.float32))
    want = tr.predict_host_fields(rp, keys, f, vals)
    assert np.array_equal(_bits(got_z), _bits(want))
    assert not np.array_equal(_bits(got_d), _bits(want))


# ---- 4. contents and prune ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [8, 32])
def test_contents_and_prune(K):
    t, tr = _make(K, api.OPT_FTRL)
    trained = _train(t, tr)
    zeros = _keys_of(np.arange(7 * SPACE, 7 * SPACE + 50))  # materialised rows of zeros: ZERO prunes them, DEFAULT not
    zv = np.zeros((zeros.size, K), np.float32)
    zv[::2, 1] = -0.0
    t.import_(zeros, w=np.ones(zeros.size, np.float32), v=zv)  # w plays no part
    src = t.list_keys()
    e = t.export(src)
    v_ready = ~np.isin(src, _pulled())  # every trained key's block is materialised by its first update
    rp, keys, f, vals = _query_all(77, np.concatenate([trained, zeros]))
    vals[3], vals[40] = np.nan, np.inf
    for absent in (api.ABSENT_DEFAULT, api.ABSENT_ZERO):
        m_all = t.freeze_mvm(absent=absent, prune=False)
        a = m_all.lookup_latent(src)
        assert a["present"].all() and not a["w"].any()
        assert np.array_equal(_bits(a["v"]), _bits(e["v"].reshape(src.size, K)))
        m = t.freeze_mvm(absent=absent)
        got = m.lookup_latent(src)
        rule = MV.pruned(absent, v_ready, e["v"].reshape(src.size, K))
        assert np.array_equal(got["present"] == 0, rule)
        assert rule.sum() >= (_pulled().size if absent == api.ABSENT_DEFAULT else zeros.size)
        info = m.info()
        assert info["keys"] + info["pruned_keys"] == info["source_keys"] == src.size
        assert info["keys"] == int((~rule).sum())
        assert info["fm"] == MV.FM_MVM and info["latent_dim"] == K and info["row_bytes"] == MV.row_bytes(K)
        assert info["capacity"] == SM.capacity_for(info["keys"]) and info["bytes"] == info["capacity"] * MV.row_bytes(K)
        # pruning never changes a prediction, NaN and Inf values included
        for x in (None, vals):
            pa, pp = m_all.predict_host_fields(rp, keys, f, x), m.predict_host_fields(rp, keys, f, x)
            assert np.array_equal(_bits(pa), _bits(pp)), absent
        assert np.isnan(pp).any()
        m.close()
        m_all.close()
    tr.close()
    t.close()


# ---- 5. the table is left alone, the model stands on its own -------------------------------------------------------
def test_freeze_leaves_the_table_alone(trained16, tmp_path):
    t, tr, trained = trained16
    t.save_state(str(tmp_path / "a"))
    m1 = t.freeze_mvm()
    m2 = t.freeze_mvm(absent=api.ABSENT_ZERO, prune=False)
    t.save_state(str(tmp_path / "b"))
    assert (tmp_path / "a").read_bytes() == (tmp_path / "b").read_bytes()
    # the model never inserts
    size, info = t.size(), m1.info()
    rp, keys, f, vals = _query_all(5, trained)
    m1.predict_host_fields(rp, keys, f, vals)
    _device(m2, rp, keys, f, vals)
    assert t.size() == size and m1.info() == info
    m1.close()
    m2.close()


def test_model_outlives_its_table():
    t, tr = _make(8, api.OPT_FTRL)
    trained = _train(t, tr)
    m = t.freeze_mvm()
    rp, keys, f, vals = _query_all(6, trained)
    before = m.predict_host_fields(rp, keys, f, vals)
    tr.close()
    t.close()
    keys_before = m.info()["keys"]
    m.predict_host_fields(np.array([0, 300], np.uint32), _unseen()[:300], np.zeros(300, np.uint8))
    assert m.info()["keys"] == keys_before and not m.lookup_latent(_unseen())["present"].any()
    assert np.array_equal(_bits(m.predict_host_fields(rp, keys, f, vals)), _bits(before))
    # empty rows: sigmoid(0); no rows at all
    assert m.predict_host_fields(np.zeros(4, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.uint8)).tolist() == [0.5] * 3
    assert m.predict_host_fields(np.zeros(1, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.uint8)).size == 0
    m.close()


# ---- 6. files ----------------------------------------------------------------------------------------------------
def _refused_io(fn):
    with pytest.raises(api.XflowError, match=ERR_IO):
        fn()


def _header(data):
    return dict(zip(SM.FIELDS, SM.HEADER.unpack(data[:SM.HEADER.size])))


def _file_args(h):
    return h["optimizer"], h["absent"], h["v_init"], h["v_const"], h["seed"], h["source_keys"]


def test_file_round_trip_layout_and_damage(trained16, tmp_path):
    t, tr, trained = trained16
    m = t.freeze_mvm()
    p = str(tmp_path / "m.xfsm")
    m.save(p)
    data = open(p, "rb").read()
    h, rows = MV.parse_model_file(data)
    info = m.info()
    assert struct.unpack_from("<i", data, 36)[0] == 3 and h["row_bytes"] == 96 and h["keys"] == info["keys"]
    lk = m.lookup_latent(rows["key"])
    assert lk["present"].all() and np.array_equal(_bits(lk["v"]), _bits(rows["v"]))
    # the file is the numpy builder's, and so is the fingerprint
    assert MV.model_file(MV.rows_array(rows["key"], lk["v"]), 16, 0, *_file_args(h)) == data
    assert MV.fingerprint(rows) == m.fingerprint()
    back = api.Model.load(p)
    assert back.info() == info
    rp, keys, f, vals = _query_all(31, trained)
    assert np.array_equal(_bits(back.predict_host_fields(rp, keys, f, vals)), _bits(m.predict_host_fields(rp, keys, f, vals)))
    p2 = str(tmp_path / "m2.xfsm")
    back.save(p2)
    assert open(p2, "rb").read() == data
    back.close()
    bad = str(tmp_path / "bad")
    for blob in (data[:-1], data[:200], data[:104 + 16]):
        open(bad, "wb").write(blob)
        _refused_io(lambda: api.Model.load(bad))
    # a non-zero byte 8 .. 15 or tail byte, with checksums that pass
    for byte in (8, 12, 15, 16 + 64 + 5):
        raw = bytearray(rows.tobytes())
        raw[MV.row_bytes(16) * (rows.size // 2) + byte] = 1
        dirty = np.frombuffer(bytes(raw), rows.dtype)
        open(bad, "wb").write(MV.model_file(dirty, 16, 0, *_file_args(h)))
        _refused_io(lambda: api.Model.load(bad))
    open(bad, "wb").write(MV.model_file(rows, 16, 0, *_file_args(h)))
    api.Model.load(bad).close()
    m.close()


# ---- 7. deltas ---------------------------------------------------------------------------------------------------
def _saved(m, path):
    m.save(str(path))
    return path.read_bytes()


@pytest.mark.parametrize("K", [16, 32])
def test_delta_chain(K, tmp_path):
    t, tr = _make(K, api.OPT_FTRL)
    _train(t, tr, 0, 2)
    models = [t.freeze_mvm()]
    for i in range(3):
        _train(t, tr, 10 + i, 1, pull=False)
        models.append(t.freeze_mvm())
    for i in range(3):
        base, nxt = models[i], models[i + 1]
        d = base.diff(nxt)
        dp = str(tmp_path / ("d%d.xfsd" % i))
        d.save(dp)
        dl = api.Delta.load(dp)
        assert dl.info()["row_bytes"] == MV.row_bytes(K) and dl.info()["upserts"] > 0
        r = base.apply(dl)
        nb = _saved(nxt, tmp_path / "n")
        assert _saved(r, tmp_path / "r") == nb
        assert r.fingerprint() == nxt.fingerprint() == d.info()["result_fingerprint"]
        ha, ra = MV.parse_model_file(_saved(base, tmp_path / "o"))
        hb, rb = MV.parse_model_file(nb)
        want = MV.delta_file(ra, rb, hb["source_keys"], K, 0, hb["optimizer"], hb["absent"], hb["v_init"], hb["v_const"],
                             hb["seed"])
        assert open(dp, "rb").read() == want and struct.unpack_from("<i", want, 16)[0] == 3
        for x in (d, dl, r):
            x.close()
    # a canonical model and a multi-view machine's of one table: equal K, equal bytes, different fm
    c = t.freeze_canonical()
    assert c.info()["row_bytes"] == models[-1].info()["row_bytes"]
    for a, b in ((c, models[-1]), (models[-1], c)):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*fm"):
            a.diff(b)
    dd = c.diff(t.freeze_canonical())
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*fm"):
        models[-1].apply(dd)
    for x in models + [c, dd]:
        x.close()
    tr.close()
    t.close()


# ---- 8. F16 ------------------------------------------------------------------------------------------------------
def test_f16_models(trained16, tmp_path):
    t, tr, trained = trained16
    m = t.freeze_mvm()
    h16 = m.convert(api.PRECISION_F16)
    info = h16.info()
    assert info["precision"] == api.PRECISION_F16 and info["fm"] == 3 and info["row_bytes"] == MV.row_bytes(16, 1) == 64
    h, rows = MV.parse_model_file(_saved(m, tmp_path / "m"))
    lk = h16.lookup_latent(rows["key"])
    assert lk["present"].all() and not lk["w"].any()
    assert np.array_equal(_bits(lk["v"]), _bits(CS.rounded(rows["v"])))
    # the F16 file is the numpy conversion's
    h16b, rows16 = MV.parse_model_file(_saved(h16, tmp_path / "h"))
    assert rows16.tobytes() == MV.convert(rows, MV.PRECISION_F16).tobytes() and h16b["precision"] == 1
    # every predict equals an F32 model of the rounded fields, loaded from a numpy-built file
    ref_path = tmp_path / "ref"
    ref_path.write_bytes(MV.model_file(MV.rows_array(rows["key"], CS.rounded(rows["v"])), 16, 0, *_file_args(h)))
    ref = api.Model.load(str(ref_path))
    for rp, keys, f, vals in (_query_all(8, trained), _query_cf(9, trained, 16)):
        for x in (None, vals):
            want = ref.predict_host_fields(rp, keys, f, x)
            assert np.array_equal(_bits(h16.predict_host_fields(rp, keys, f, x)), _bits(want))
            assert np.array_equal(_bits(_device(h16, rp, keys, f, x)), _bits(want))
    # F16 -> F32 widens exactly
    back = h16.convert(api.PRECISION_F32)
    assert _saved(back, tmp_path / "b") == ref_path.read_bytes()
    # mixed precisions are never diffed
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*precision"):
        m.diff(h16)
    # the 65520 refusal
    big = _keys_of(np.arange(8 * SPACE, 8 * SPACE + 3))
    bv = np.zeros((3, 16), np.float32)
    bv[1, 5] = 70000.0
    t.import_(big, w=np.zeros(3, np.float32), v=bv)
    mb = t.freeze_mvm()
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*65520"):
        mb.convert(api.PRECISION_F16)
    for x in (m, h16, ref, back, mb):
        x.close()


# ---- 9. refusals -------------------------------------------------------------------------------------------------
def test_refusals(trained16):
    torch = pytest.importorskip("torch")
    t, tr, trained = trained16
    fm = api.Table(latent_dim=8, capacity=1 << 12)
    lr = api.Table(capacity=1 << 12)
    c64 = api.Table(latent_dim=64, canonical_fm=1, capacity=1 << 12)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*canonical_fm = 0"):
        fm.freeze_mvm()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*canonical_fm = 0"):
        lr.freeze_mvm()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*latent_dim = 64"):
        c64.freeze_mvm()
    m = t.freeze_mvm()
    rp = np.array([0, 2], np.uint32)
    keys = trained[:2]
    f = np.array([0, 1], np.uint8)
    ones = np.ones(2, np.float32)
    d_rp = torch.from_numpy(rp.astype(np.int32)).cuda()
    d_keys = torch.from_numpy(keys.view(np.int64)).cuda()
    d_vals = torch.from_numpy(ones).cuda()
    d_out = torch.empty(1, dtype=torch.float32, device="cuda")
    fields_fn = "predict_host_fields or xf_model_predict_device_fields"
    for call in (lambda: m.predict_host(rp, keys), lambda: m.predict_host(rp, keys, ones),
                 lambda: m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), 1, 2, d_out.data_ptr()),
                 lambda: m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), 1, 2, d_out.data_ptr(), d_vals=d_vals.data_ptr()),
                 lambda: m.predict_ingested(tr, 0, 0)):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*" + fields_fn):
            call()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*xf_model_lookup_latent"):
        m.lookup(keys)  # asks for st and qt
    w = np.full(2, 7.0, np.float32)
    pres = np.zeros(2, np.uint8)
    api._check(api.lib().xf_model_lookup(m.h, api._p(keys), 2, api._p(w), None, None, api._p(pres)))
    assert pres.all() and not w.any()
    # field ids of 32 and more, and no field ids at all
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*field id 32 of token 1"):
        m.predict_host_fields(rp, keys, np.array([3, 32], np.uint8))
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*field id 255 of token 0"):
        m.predict_host_fields(rp, keys, np.array([255, 0], np.uint8), ones)
    out = np.empty(1, np.float32)
    assert api.lib().xf_model_predict_host_fields(m.h, api._p(rp), api._p(keys), None, None, 1, 2, api._p(out)) == -1
    assert api.lib().xf_model_predict_device_fields(m.h, api._p(d_rp.data_ptr()), api._p(d_keys.data_ptr()), None, None,
                                                    1, 2, api._p(d_out.data_ptr()), None) == -1
    m.predict_host_fields(rp, keys, f)  # the same call with field ids is served
    # the _fields entry points refuse every other model
    d_f = torch.from_numpy(f).cuda()
    fm.pull(keys)
    lr.pull(keys)
    others = [fm.freeze(), lr.freeze(), t.freeze_canonical()]
    for o in others:
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*xf_table_freeze_mvm"):
            o.predict_host_fields(rp, keys, f)
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*xf_table_freeze_mvm"):
            o.predict_device_fields(d_rp.data_ptr(), d_keys.data_ptr(), d_f.data_ptr(), 1, 2, d_out.data_ptr())
        o.close()
    m.close()
    for x in (fm, lr, c64):
        x.close()

"""Canonical serving models (xf_table_freeze_canonical, csrc/serve.cu): a canonical FM table frozen into rows
{key, w, 0, v[K]} predicts on feature values, bit for bit, what the table's own predict does; holds what xf_table_export
returns; leaves the table alone; never inserts; and its files and deltas follow canonical_serving_model.py."""
import struct

import numpy as np
import pytest

import canonical_serving_model as CM
import serving_model as SM
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

B, D, SPACE, N = 256, 12, 6000, 3  # rows and tokens per row of a training batch, id space, batches
CAP = 1 << 15
ROW_LENS = [0, 1, 3, 31, 32, 33, 65, 129, 300] + [8] * 25
ERR_ARG, ERR_IO = "error -1:", "error -4:"
KS = list(CM.LATENT_DIMS)
CASES = [(K, api.OPT_FTRL) for K in KS] + [(K, api.OPT_SGD) for K in (4, 16, 64)]


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
    return rp, _keys_of(ids), _vals(rng, ids.size), lab


def _make(K, opt, capacity=CAP):
    # lambda1 above a once-seen key's |z|, so that FTRL leaves exact zeros in w
    t = api.Table(latent_dim=K, optimizer=opt, v_init=api.VINIT_COUNTER, seed=7, capacity=capacity, canonical_fm=1,
                  lambda1=2e-3)
    tr = api.Trainer(t, model=api.MODEL_FM_CANONICAL, max_rows=B, max_nnz=8192)
    return t, tr


def _train(t, tr, first=0, n=N, pull=True):
    seen = []
    for i in range(first, first + n):
        rp, keys, vals, lab = _batch(500 + i)
        tr.step_host_values(rp, keys, vals, lab)
        seen.append(keys)
    if pull:
        t.pull(_pulled(), want_v=False)
    return np.unique(np.concatenate(seen))


def _query(seed, trained, lens=ROW_LENS):
    """Rows over trained, pulled and never-seen keys, one key four times in the longer rows, and their values"""
    rng = np.random.default_rng(seed)
    pool = np.concatenate([trained, _pulled(), _unseen()])
    rows = []
    for n in lens:
        k = pool[rng.integers(0, pool.size, n)]
        if n >= 8:
            k[n // 2:n // 2 + 3] = k[0]
        rows.append(k)
    rp = np.zeros(len(rows) + 1, np.uint32)
    rp[1:] = np.cumsum([r.size for r in rows])
    keys = np.concatenate(rows).astype(np.uint64)
    return rp, keys, _vals(rng, keys.size)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture
def trained16():
    t, tr = _make(16, api.OPT_FTRL)
    yield t, tr, _train(t, tr)
    tr.close()
    t.close()


# ---- 1. predictions ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,opt", CASES)
def test_predict_equals_the_tables_bit_for_bit(K, opt):
    t, tr = _make(K, opt)
    trained = _train(t, tr)
    rp, keys, vals = _query(K + 3, trained)
    models = {p: t.freeze_canonical(prune=p) for p in (False, True)}
    got = {(p, v): models[p].predict_host(rp, keys, None if v is None else vals) for p in models for v in (None, 1)}
    ones = models[True].predict_host(rp, keys, np.ones(keys.size, np.float32))
    plain = models[True].predict_host(rp, keys)
    # after the freezes: the table's predict inserts the unseen keys
    want = {None: tr.predict_host_values(rp, keys, None), 1: tr.predict_host_values(rp, keys, vals)}
    for (p, v), g in got.items():
        assert np.array_equal(_bits(g), _bits(want[v])), (p, v)
    assert np.array_equal(_bits(ones), _bits(want[None])) and np.array_equal(_bits(plain), _bits(want[None]))
    assert len(set(want[1].tolist())) > 10 and len(set(want[None].tolist())) > 10
    info = models[True].info()
    assert info["fm"] == 2 and info["absent"] == api.ABSENT_DEFAULT and info["pruned_keys"] >= _pulled().size
    assert models[False].info()["pruned_keys"] == 0
    for m in models.values():
        m.close()
    tr.close()
    t.close()


# ---- 2. absent keys read as nothing ------------------------------------------------------------------------------
def test_absent_zero_equals_the_table_with_zero_rows(trained16):
    t, tr, trained = trained16
    rp, keys, vals = _query(21, trained)
    mz = t.freeze_canonical(absent=api.ABSENT_ZERO)
    md = t.freeze_canonical()
    assert mz.info()["absent"] == api.ABSENT_ZERO
    got_z, got_d = mz.predict_host(rp, keys, vals), md.predict_host(rp, keys, vals)
    uk = np.unique(keys)
    lacks = uk[mz.lookup_latent(uk)["present"] == 0]
    assert lacks.size > 10
    t.import_(lacks, w=np.zeros(lacks.size, np.float32), v=np.zeros((lacks.size, 16), np.float32))
    want = tr.predict_host_values(rp, keys, vals)
    assert np.array_equal(_bits(got_z), _bits(want))
    assert not np.array_equal(_bits(got_d), _bits(want))


# ---- 3. contents and prune ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [8, 32])
def test_contents_and_prune(K):
    t, tr = _make(K, api.OPT_FTRL)
    _train(t, tr)
    zeros = _keys_of(np.arange(7 * SPACE, 7 * SPACE + 50))  # materialised rows of zeros: ZERO prunes them, DEFAULT not
    t.import_(zeros, w=np.zeros(zeros.size, np.float32), v=np.zeros((zeros.size, K), np.float32))
    src = t.list_keys()
    e = t.export(src)
    v_ready = ~np.isin(src, _pulled())  # every trained key's block is materialised by its first update
    for absent in (api.ABSENT_DEFAULT, api.ABSENT_ZERO):
        m_all = t.freeze_canonical(absent=absent, prune=False)
        a = m_all.lookup_latent(src)
        assert a["present"].all()
        assert np.array_equal(_bits(a["w"]), _bits(e["w"])) and np.array_equal(_bits(a["v"]), _bits(e["v"]))
        m = t.freeze_canonical(absent=absent)
        got = m.lookup_latent(src)
        rule = CM.pruned(e["w"], absent, v_ready, e["v"])
        assert np.array_equal(got["present"] == 0, rule)
        assert rule.sum() >= (_pulled().size if absent == api.ABSENT_DEFAULT else zeros.size)
        info = m.info()
        assert info["keys"] + info["pruned_keys"] == info["source_keys"] == src.size
        assert info["keys"] == int((~rule).sum())
        assert info["fm"] == 2 and info["latent_dim"] == K and info["row_bytes"] == CM.row_bytes(K)
        assert info["capacity"] == SM.capacity_for(info["keys"]) and info["bytes"] == info["capacity"] * CM.row_bytes(K)
        # lookup reads w and present; the kept rows hold export's bits
        lk = m.lookup_latent(src[~rule])
        assert np.array_equal(_bits(lk["v"]), _bits(e["v"][~rule]))
        w = np.zeros(src.size, np.float32)
        pres = np.zeros(src.size, np.uint8)
        api._check(api.lib().xf_model_lookup(m.h, api._p(src), src.size, api._p(w), None, None, api._p(pres)))
        assert np.array_equal(pres, got["present"]) and np.array_equal(_bits(w), _bits(got["w"]))
        m.close()
        m_all.close()
    tr.close()
    t.close()


# ---- 4. the table is left alone ----------------------------------------------------------------------------------
def test_freeze_leaves_the_table_alone(trained16, tmp_path):
    t, tr, _ = trained16
    t.save_state(str(tmp_path / "a"))
    m1 = t.freeze_canonical()
    m2 = t.freeze_canonical(absent=api.ABSENT_ZERO, prune=False)
    t.save_state(str(tmp_path / "b"))
    assert (tmp_path / "a").read_bytes() == (tmp_path / "b").read_bytes()
    m1.close()
    m2.close()


# ---- 5. the model stands on its own ------------------------------------------------------------------------------
def test_model_outlives_its_table_and_never_inserts():
    t, tr = _make(8, api.OPT_FTRL)
    trained = _train(t, tr)
    m = t.freeze_canonical()
    rp, keys, vals = _query(5, trained)
    before = m.predict_host(rp, keys, vals)
    tr.close()
    t.close()
    keys_before = m.info()["keys"]
    rpu = np.array([0, 300], np.uint32)
    m.predict_host(rpu, _unseen()[:300], np.ones(300, np.float32))
    assert m.info()["keys"] == keys_before
    assert not m.lookup_latent(_unseen())["present"].any()
    assert np.array_equal(_bits(m.predict_host(rp, keys, vals)), _bits(before))
    m.close()


# ---- 6. batch shapes ---------------------------------------------------------------------------------------------
def test_device_entry_and_batch_shapes(trained16):
    torch = pytest.importorskip("torch")
    t, tr, trained = trained16
    m = t.freeze_canonical()
    rp, keys, vals = _query(9, trained)
    want = m.predict_host(rp, keys, vals)
    s = torch.cuda.Stream()
    d_rp, d_keys = torch.from_numpy(rp.astype(np.int32)).cuda(), torch.from_numpy(keys.view(np.int64)).cuda()
    d_vals, d_out = torch.from_numpy(vals).cuda(), torch.empty(rp.size - 1, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), rp.size - 1, keys.size, d_out.data_ptr(), stream=s.cuda_stream,
                     d_vals=d_vals.data_ptr())
    s.synchronize()
    assert np.array_equal(_bits(d_out.cpu().numpy()), _bits(want))
    m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), rp.size - 1, keys.size, d_out.data_ptr(), stream=s.cuda_stream)
    s.synchronize()
    assert np.array_equal(_bits(d_out.cpu().numpy()), _bits(m.predict_host(rp, keys)))
    # empty rows: sigmoid(0); no rows at all
    assert m.predict_host(np.zeros(4, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.float32)).tolist() == [0.5] * 3
    assert m.predict_host(np.zeros(1, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.float32)).size == 0
    # a row of 4097 tokens
    rng = np.random.default_rng(2)
    long_k = np.concatenate([trained, _pulled(), _unseen()])[rng.integers(0, trained.size + 500, 4097)]
    long_v = _vals(rng, 4097)
    rp1 = np.array([0, 4097], np.uint32)
    got = m.predict_host(rp1, long_k, long_v)
    assert np.array_equal(_bits(got), _bits(tr.predict_host_values(rp1, long_k, long_v)))
    # 65 536 rows of 100 tokens: a row predicted alone gives the same bits
    R, L = 65536, 100
    pool = np.concatenate([trained, _pulled(), _unseen()])
    bk = pool[rng.integers(0, pool.size, R * L)]
    bv = _vals(rng, R * L)
    brp = (np.arange(R + 1, dtype=np.uint64) * L).astype(np.uint32)
    big = m.predict_host(brp, bk, bv)
    for r in (0, 1, 4097, 33333, R - 1):
        one = m.predict_host(np.array([0, L], np.uint32), bk[r * L:(r + 1) * L], bv[r * L:(r + 1) * L])
        assert _bits(one)[0] == _bits(big)[r]
    m.close()


# ---- 7. files ----------------------------------------------------------------------------------------------------
def _refused_io(fn):
    with pytest.raises(api.XflowError, match=ERR_IO):
        fn()


def test_file_round_trip_layout_and_damage(trained16, tmp_path):
    t, tr, trained = trained16
    m = t.freeze_canonical()
    p = str(tmp_path / "m.xfsm")
    m.save(p)
    data = open(p, "rb").read()
    h, rows = CM.parse_model_file(data)
    info = m.info()
    for f, want in (("fm", 2), ("latent_dim", 16), ("row_bytes", 96), ("keys", info["keys"]), ("capacity", info["capacity"]),
                    ("source_keys", info["source_keys"]), ("pruned_keys", info["pruned_keys"]),
                    ("absent", api.ABSENT_DEFAULT), ("chunk_rows", (64 << 20) // 96)):
        assert h[f] == want and struct.unpack_from("<q" if f in ("keys", "capacity", "source_keys", "pruned_keys",
                                                                 "chunk_rows") else "<i", data, SM.OFFSETS[f])[0] == want, f
    lk = m.lookup_latent(rows["key"])
    assert lk["present"].all() and np.array_equal(_bits(lk["w"]), _bits(rows["w"]))
    assert np.array_equal(_bits(lk["v"]), _bits(rows["v"]))
    assert CM.fingerprint(rows) == m.fingerprint()
    back = api.Model.load(p)
    rp, keys, vals = _query(31, trained)
    assert np.array_equal(_bits(back.predict_host(rp, keys, vals)), _bits(m.predict_host(rp, keys, vals)))
    p2 = str(tmp_path / "m2.xfsm")
    back.save(p2)
    assert open(p2, "rb").read() == data
    back.close()
    bad = str(tmp_path / "bad")
    for blob in (data[:-1], data[:200], data[:104 + 16]):
        open(bad, "wb").write(blob)
        _refused_io(lambda: api.Model.load(bad))
    for pos in (36, 40, 104 + 40, len(data) - 3):
        flip = bytearray(data)
        flip[pos] ^= 0x04
        open(bad, "wb").write(bytes(flip))
        _refused_io(lambda: api.Model.load(bad))
    # padding that is not zero, with checksums that pass
    for field, idx in (("zero", 0), ("pad", (rows.size - 1, 15))):
        dirty = rows.copy()
        dirty[field][idx] = 1
        open(bad, "wb").write(CM.model_file(dirty, 16, api.OPT_FTRL, api.ABSENT_DEFAULT, h["v_init"], h["v_const"],
                                             h["seed"], h["source_keys"]))
        _refused_io(lambda: api.Model.load(bad))
    # the same file built clean loads
    open(bad, "wb").write(CM.model_file(rows, 16, api.OPT_FTRL, api.ABSENT_DEFAULT, h["v_init"], h["v_const"], h["seed"],
                                        h["source_keys"]))
    api.Model.load(bad).close()
    # other formats
    t.save_state(bad)
    _refused_io(lambda: api.Model.load(bad))
    m.close()


# ---- 8. deltas ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [16, 64])
def test_delta_chain(K, tmp_path):
    t, tr = _make(K, api.OPT_FTRL)
    _train(t, tr, 0, 2)
    models = [t.freeze_canonical()]
    for i in range(3):
        _train(t, tr, 10 + i, 1, pull=False)
        models.append(t.freeze_canonical())
    for i in range(3):
        base, nxt = models[i], models[i + 1]
        d = base.diff(nxt)
        dp = str(tmp_path / ("d%d.xfsd" % i))
        d.save(dp)
        dl = api.Delta.load(dp)
        assert dl.info()["row_bytes"] == CM.row_bytes(K) and dl.info()["upserts"] > 0
        hdr = open(dp, "rb").read()[:144]
        assert struct.unpack_from("<iiI", hdr, 16)[:2] == (2, K) and struct.unpack_from("<I", hdr, 48)[0] == CM.row_bytes(K)
        r = base.apply(dl)
        r.save(str(tmp_path / "r"))
        nxt.save(str(tmp_path / "n"))
        assert (tmp_path / "r").read_bytes() == (tmp_path / "n").read_bytes()
        assert r.fingerprint() == nxt.fingerprint() == d.info()["result_fingerprint"]
        # the file is the numpy statement's
        _, ra = CM.parse_model_file(open_model(base, tmp_path))
        _, rb = CM.parse_model_file((tmp_path / "n").read_bytes())
        assert open(dp, "rb").read() == CM.delta_file(ra, rb, nxt.info()["source_keys"], K, api.OPT_FTRL,
                                                      api.ABSENT_DEFAULT, *_vinit_of(tmp_path / "n"))
        for x in (d, dl, r):
            x.close()
    # a padding-dirty upsert with checksums that pass is refused
    _, ra = CM.parse_model_file(open_model(models[0], tmp_path))
    _, rb = CM.parse_model_file(open_model(models[1], tmp_path))
    dirty = rb.copy()
    dirty["zero"][0] = 1
    bad = str(tmp_path / "bad.xfsd")
    open(bad, "wb").write(CM.delta_file(ra, dirty, models[1].info()["source_keys"], K, api.OPT_FTRL, api.ABSENT_DEFAULT,
                                        *_vinit_of(tmp_path / "n")))
    _refused_io(lambda: api.Delta.load(bad))
    for m in models:
        m.close()
    tr.close()
    t.close()


def open_model(m, tmp_path):
    p = str(tmp_path / "o.xfsm")
    m.save(p)
    return open(p, "rb").read()


def _vinit_of(path):
    h = dict(zip(SM.FIELDS, SM.HEADER.unpack(open(path, "rb").read()[:SM.HEADER.size])))
    return h["v_init"], h["v_const"], h["seed"]


def test_delta_refusals():
    c16, c16tr = _make(16, api.OPT_FTRL, capacity=1 << 12)
    c8, c8tr = _make(8, api.OPT_FTRL, capacity=1 << 12)
    f16 = api.Table(latent_dim=16, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=7, capacity=1 << 12)
    m16, m8, fm = c16.freeze_canonical(), c8.freeze_canonical(), f16.freeze()
    with pytest.raises(api.XflowError, match="fm"):
        m16.diff(fm)
    with pytest.raises(api.XflowError, match="latent_dim"):
        m16.diff(m8)
    for x in (m16, m8, fm, c16tr, c8tr, c16, c8, f16):
        x.close()


# ---- 9. refusals -------------------------------------------------------------------------------------------------
def test_refusals(trained16):
    t, tr, trained = trained16
    lr = api.Table(capacity=1 << 12)
    fm = api.Table(latent_dim=8, capacity=1 << 12)
    shard = api.Table(latent_dim=8, shard_index=0, num_shards=2, capacity=1 << 12)
    for x in (lr, fm, shard):
        with pytest.raises(api.XflowError, match=ERR_ARG):
            x.freeze_canonical()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*canonical"):
        t.freeze()
    rp = np.array([0, 2], np.uint32)
    keys = trained[:2]
    for plain in (lr.freeze(), fm.freeze()):
        plain.predict_host(rp, keys)
        with pytest.raises(api.XflowError, match=ERR_ARG):
            plain.predict_host(rp, keys, np.ones(2, np.float32))
        with pytest.raises(api.XflowError, match=ERR_ARG):
            plain.lookup_latent(keys)
        plain.close()
    m = t.freeze_canonical()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*xf_model_lookup_latent"):
        m.lookup(keys)  # asks for st and qt
    with pytest.raises(api.XflowError, match=ERR_ARG):
        m.predict_ingested(tr, 0, 0)
    with pytest.raises(api.XflowError, match=ERR_ARG):
        m.predict_host(rp, np.array([keys[0], 2 ** 64 - 1], np.uint64), np.ones(2, np.float32))
    with pytest.raises(api.XflowError, match=ERR_ARG):
        m.predict_host(np.array([0, 3], np.uint32), keys, np.ones(2, np.float32))
    m.close()
    for x in (lr, fm, shard):
        x.close()

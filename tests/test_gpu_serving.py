"""The serving model (xf_table_freeze / xf_model_*, csrc/serve.cu): a model frozen from a trained table predicts, bit for
bit, what the table's own predict does; holds what xf_table_export returns; leaves the table alone; never inserts;
survives its table; and its file is a function of its contents."""
import os
import struct
import subprocess

import numpy as np
import pytest

import serving_model as M
from common import GOLDEN
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
TRAIN = os.path.join(GOLDEN, "data", "small_train")
TEST = os.path.join(GOLDEN, "data", "small_test")

TABLES = {  # name: (model, optimizer, K, eager LR)
    "lr_ftrl": (api.MODEL_LR, api.OPT_FTRL, 0, False),
    "lr_sgd": (api.MODEL_LR, api.OPT_SGD, 0, False),
    "lr_ftrl_eager": (api.MODEL_LR, api.OPT_FTRL, 0, True),
    "lr_sgd_eager": (api.MODEL_LR, api.OPT_SGD, 0, True),
    "fm_ftrl_k8": (api.MODEL_FM, api.OPT_FTRL, 8, False),
    "fm_ftrl_k10": (api.MODEL_FM, api.OPT_FTRL, 10, False),
    "fm_ftrl_k16": (api.MODEL_FM, api.OPT_FTRL, 16, False),
    "fm_sgd_k8": (api.MODEL_FM, api.OPT_SGD, 8, False),
    "fm_sgd_k10": (api.MODEL_FM, api.OPT_SGD, 10, False),
    "fm_sgd_k16": (api.MODEL_FM, api.OPT_SGD, 16, False),
}
ALL = sorted(TABLES)
SOME = ["lr_ftrl", "lr_sgd_eager", "fm_ftrl_k16", "fm_sgd_k10"]
B, D, SPACE, N = 512, 8, 20000, 4  # rows and tokens per row of a training batch, id space, batches
CAP = 1 << 16
ROW_LENS = [0, 1, 63, 64, 65, 129, 300] + [8] * 25
ERR_ARG, ERR_IO = "error -1:", "error -4:"


def _batch(seed):
    rp, ids, _ = datagen.make_ids(seed, B, D, SPACE, dist="zipf")
    lab = (np.random.default_rng(seed).random(B) < 0.3).astype(np.uint8)
    return rp, api.hash_decimal_ids(np.asarray(ids, np.uint64)), lab


def _keys_of(ids):
    return api.hash_decimal_ids(np.asarray(ids, np.uint64))


def _pulled():
    """Keys a Pull inserted and no batch trained: default rows (FM: the latent block is not materialised)."""
    return _keys_of(np.arange(5 * SPACE, 5 * SPACE + 300))


def _unseen():
    return _keys_of(np.arange(9 * SPACE, 9 * SPACE + 400))


def _make(name, monkeypatch, max_rows=B, max_nnz=B * D, capacity=CAP):
    model, opt, K, eager = TABLES[name]
    if eager:
        monkeypatch.setenv("XFLOW_EAGER", "1")
    else:
        monkeypatch.delenv("XFLOW_EAGER", raising=False)
    # lambda1 well above a once-seen key's |z|, so that FTRL's L1 term leaves many exact zeros
    t = api.Table(latent_dim=K, optimizer=opt, seed=11, capacity=capacity, lambda1=2e-3)
    tr = api.Trainer(t, model=model, max_rows=max_rows, max_nnz=max_nnz)
    return t, tr


def _train(t, tr, first=0, n=N):
    """n Zipf batches (lazy tables end with pending steps) and a Pull of keys no batch trains; returns the trained keys"""
    seen = []
    for i in range(first, first + n):
        rp, keys, lab = _batch(1000 + i)
        tr.step_host(rp, keys, lab, want_loss=False)
        seen.append(keys)
    t.pull(_pulled(), want_v=False)
    return np.unique(np.concatenate(seen))


def _query(seed, trained):
    """Rows of 0, 1, 63, 64, 65, 129, 300 and 8 tokens over trained, pulled and never-seen keys, with repeats in a row"""
    rng = np.random.default_rng(seed)
    pool = np.concatenate([trained, _pulled(), _unseen()])
    rows = []
    for n in ROW_LENS:
        k = pool[rng.integers(0, pool.size, n)]
        if n >= 8:
            k[n // 2:n // 2 + 3] = k[0]  # one key four times in the row
        rows.append(k)
    rp = np.zeros(len(rows) + 1, np.uint32)
    rp[1:] = np.cumsum([r.size for r in rows])
    return rp, np.concatenate(rows).astype(np.uint64)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture
def frozen(request, monkeypatch):
    """(name, table, trainer, trained keys) after training; closed afterwards"""
    name = request.param
    t, tr = _make(name, monkeypatch)
    trained = _train(t, tr)
    yield name, t, tr, trained
    tr.close()
    t.close()


# ---- 1. predictions ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frozen", ALL, indirect=True)
@pytest.mark.parametrize("absent", ["default", "zero"])
def test_predict_equals_the_tables_bit_for_bit(frozen, absent):
    name, t, tr, trained = frozen
    if absent == "zero":
        t.set_admission(api.ADMIT_POISSON, probability=0.0)  # from here on the table's predict inserts nothing
    rp, keys = _query(7, trained)
    m = t.freeze()
    m_all = t.freeze(prune=False)
    assert m.info()["absent"] == (api.ABSENT_ZERO if absent == "zero" else api.ABSENT_DEFAULT)
    # the other policy, stated: absent keys read differently under it (FM: their initial latent values count or do not)
    other = t.freeze(absent=api.ABSENT_ZERO if absent == "default" else api.ABSENT_DEFAULT)
    got, got_all = m.predict_host(rp, keys), m_all.predict_host(rp, keys)
    want = tr.predict_host(rp, keys)  # after the freezes: without a policy it inserts the unseen keys
    assert np.array_equal(_bits(got), _bits(want))
    assert np.array_equal(_bits(got_all), _bits(want))
    assert len(set(got.tolist())) > 10  # the rows do differ
    assert m_all.info()["pruned_keys"] == 0
    # an SGD FM row never reads as nothing: no L1 term zeroes it, and its initial latent values are not zero
    sgd_fm = TABLES[name][1] == api.OPT_SGD and TABLES[name][2] > 0
    assert (m.info()["pruned_keys"] > 0) == (not (absent == "zero" and sgd_fm))
    assert other.info()["absent"] != m.info()["absent"]
    if TABLES[name][2]:
        assert not np.array_equal(_bits(other.predict_host(rp, keys)), _bits(want))
    for x in (m, m_all, other):
        x.close()


def test_empty_batches_and_rows(monkeypatch):
    t, tr = _make("fm_ftrl_k8", monkeypatch)
    _train(t, tr, n=1)
    m = t.freeze()
    assert m.predict_host(np.zeros(1, np.uint32), np.zeros(0, np.uint64)).size == 0
    p = m.predict_host(np.zeros(4, np.uint32), np.zeros(0, np.uint64))
    assert np.array_equal(_bits(p), _bits(np.full(3, 0.5, np.float32)))
    m.close(); tr.close(); t.close()


# ---- 2. contents -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frozen", ALL, indirect=True)
@pytest.mark.parametrize("absent", [api.ABSENT_DEFAULT, api.ABSENT_ZERO])
def test_contents_are_the_tables(frozen, absent):
    name, t, tr, trained = frozen
    K = TABLES[name][2]
    keys = np.sort(t.list_keys())
    assert np.array_equal(keys, np.unique(np.concatenate([trained, _pulled()])))
    ex = t.export(keys)
    st, qt = M.fm_sums(ex["v"]) if K else (np.zeros(keys.size, np.float32),) * 2
    m_all, m = t.freeze(absent=absent, prune=False), t.freeze(absent=absent)
    la = m_all.lookup(keys)
    assert la["present"].all()
    assert np.array_equal(_bits(la["w"]), _bits(ex["w"]))
    assert np.array_equal(_bits(la["st"]), _bits(st)) and np.array_equal(_bits(la["qt"]), _bits(qt))
    # pruned: exactly the rows that read as an absent key; a trained FM key's latent block is materialised, a pulled one's not
    gone = M.pruned(ex["w"], K > 0, absent, v_ready=np.isin(keys, trained), st=st, qt=qt)
    lp = m.lookup(keys)
    assert np.array_equal(lp["present"], (~gone).astype(np.uint8))
    sgd_fm_zero = K > 0 and TABLES[name][1] == api.OPT_SGD and absent == api.ABSENT_ZERO  # such a row never reads as nothing
    assert gone.any() == (not sgd_fm_zero) and not gone.all()
    for f, ref in (("w", ex["w"]), ("st", st), ("qt", qt)):
        assert np.array_equal(_bits(lp[f][~gone]), _bits(ref[~gone])) and not lp[f][gone].any()
    assert not m.lookup(_unseen())["present"].any() and not m_all.lookup(_unseen())["present"].any()
    for x, pruned in ((m, int(gone.sum())), (m_all, 0)):
        i = x.info()
        assert i["keys"] + i["pruned_keys"] == i["source_keys"] == t.size() == keys.size
        assert i["pruned_keys"] == pruned
        assert i["row_bytes"] == (32 if K else 16) and i["bytes"] == i["capacity"] * i["row_bytes"]
        assert i["capacity"] == M.capacity_for(i["keys"]) and 2 * i["keys"] <= i["capacity"]
        assert (i["latent_dim"], i["optimizer"], i["fm"], i["absent"]) == (K, TABLES[name][1], int(K > 0), absent)
        x.close()


# ---- 3. the table is left alone ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SOME)
def test_freeze_changes_nothing_in_the_table(name, monkeypatch, tmp_path):
    finals = []
    for run in ("plain", "frozen"):
        t, tr = _make(name, monkeypatch)
        t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=12, hashes=3, decay_batches=3, seed=5)
        t.set_eviction(max_idle_batches=3, max_keys=1500)
        _train(t, tr)
        if run == "frozen":
            # a state image holds every row, stamp, filter cell, the batch number and the pending-step ring
            before, after = str(tmp_path / "before"), str(tmp_path / "after")
            t.save_state(before, user=1)
            m = t.freeze()
            m2 = t.freeze(absent=api.ABSENT_DEFAULT, prune=False)
            t.save_state(after, user=1)
            assert open(before, "rb").read() == open(after, "rb").read()
            assert m.info()["absent"] == api.ABSENT_ZERO  # the table has a policy
            m.close(); m2.close()
        _train(t, tr, first=N, n=3)
        tr.sync()
        # which slot a key lies in depends on the order its inserting threads ran in: two runs compare by key
        keys = np.sort(t.list_keys())
        ex = t.export(keys)
        finals.append([keys, t.last_touch(keys), np.array(sorted(t.admission_stats().items()), object)] +
                      [ex[f].view(np.uint32) for f in ("w", "nw", "zw", "v", "nv", "zv")])
        tr.close(); t.close()
    assert len(finals[0][0]) > 100
    for a, b in zip(*finals):
        assert np.array_equal(a, b)


# ---- 4. never inserts; independent of its source -------------------------------------------------------------------
@pytest.mark.parametrize("name", SOME)
def test_model_never_inserts_and_outlives_its_table(name, monkeypatch, tmp_path):
    t, tr = _make(name, monkeypatch)
    trained = _train(t, tr)
    rp, keys = _query(3, trained)
    m = t.freeze()
    f0, f1 = str(tmp_path / "m0"), str(tmp_path / "m1")
    m.save(f0)
    info, size = m.info(), t.size()
    p0 = m.predict_host(rp, keys)
    for _ in range(2):
        assert np.array_equal(_bits(m.predict_host(rp, keys)), _bits(p0))
    assert m.info() == info and t.size() == size and not m.lookup(_unseen())["present"].any()
    m.save(f1)
    assert open(f0, "rb").read() == open(f1, "rb").read()
    _train(t, tr, first=N, n=2)  # the source moves on
    assert not np.array_equal(_bits(tr.predict_host(rp, keys)), _bits(p0))
    assert np.array_equal(_bits(m.predict_host(rp, keys)), _bits(p0))
    tr.close(); t.close()
    assert np.array_equal(_bits(m.predict_host(rp, keys)), _bits(p0))
    m.close()


# ---- 5. device pointers, ingested blocks ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", SOME)
def test_predict_device_on_a_stream(name, monkeypatch):
    import torch
    t, tr = _make(name, monkeypatch)
    trained = _train(t, tr)
    rp, keys = _query(5, trained)
    m = t.freeze()
    want = m.predict_host(rp, keys)
    dev = torch.device("cuda:0")
    d_rp = torch.from_numpy(rp.astype(np.int32)).to(dev)
    d_keys = torch.from_numpy(keys.view(np.int64)).to(dev)
    d_out = torch.full((rp.size - 1,), -1.0, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    s = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(s):
        m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), rp.size - 1, keys.size, d_out.data_ptr(), stream=s.cuda_stream)
        m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), 0, keys.size, d_out.data_ptr(), stream=s.cuda_stream)
    s.synchronize()
    assert np.array_equal(_bits(d_out.cpu().numpy()), _bits(want))
    m.close(); tr.close(); t.close()


@pytest.mark.parametrize("name", SOME)
def test_predict_ingested_reads_the_model(name, monkeypatch):
    t, tr = _make(name, monkeypatch, max_rows=1 << 12, max_nnz=1 << 18)
    text = open(TRAIN + "-00000", "rb").read()
    rows, nnz = tr.ingest_text(text)
    tr.step_ingested(0, rows)
    rows, nnz = tr.ingest_text(open(TEST + "-00000", "rb").read())
    assert rows > 100
    m = t.freeze()
    got, got_lab = m.predict_ingested(tr, 0, rows)
    part, part_lab = m.predict_ingested(tr, 10, 50)
    want, want_lab = tr.predict_ingested(0, rows)
    assert np.array_equal(_bits(got), _bits(want)) and np.array_equal(got_lab, want_lab)
    assert np.array_equal(_bits(part), _bits(want[10:50])) and np.array_equal(part_lab, want_lab[10:50])
    assert len(set(want.tolist())) > 10 and want_lab.any()
    m.close(); tr.close(); t.close()


# ---- 6. the file ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frozen", SOME, indirect=True)
def test_file_round_trip_and_determinism(frozen, tmp_path):
    name, t, tr, trained = frozen
    K = TABLES[name][2]
    rp, keys = _query(9, trained)
    a, b, c = (str(tmp_path / x) for x in "abc")
    m, m2 = t.freeze(), t.freeze()
    m.save(a)
    m2.save(b)
    data = open(a, "rb").read()
    assert data == open(b, "rb").read()
    back = api.Model.load(a)
    back.save(c)
    assert data == open(c, "rb").read()
    assert back.info() == m.info()
    assert np.array_equal(_bits(back.predict_host(rp, keys)), _bits(m.predict_host(rp, keys)))
    allk = np.concatenate([np.sort(t.list_keys()), _unseen()])
    la, lb = m.lookup(allk), back.lookup(allk)
    for f in ("w", "st", "qt", "present"):
        assert np.array_equal(la[f].view(np.uint8), lb[f].view(np.uint8))
    # the documented layout, and the numpy statement of the format builds the same bytes from the model's contents
    i = m.info()
    h, rows = M.parse_file(data)
    assert struct.unpack_from("<4sIQQQI", data, 0) == (b"XFSM", 1, 104, i["keys"], i["capacity"], i["row_bytes"])
    assert struct.unpack_from("<iiii", data, 36) == (i["fm"], K, TABLES[name][1], i["absent"])
    assert struct.unpack_from("<QQQ", data, 64) == (11, i["source_keys"], i["pruned_keys"])
    assert struct.unpack_from("<Q", data, 88)[0] == (64 << 20) // i["row_bytes"]
    kept = la["present"].astype(bool)
    mine = M.rows_array(allk[kept], la["w"][kept], la["st"][kept] if K else None, la["qt"][kept] if K else None)
    assert mine.tobytes() == rows.tobytes()
    assert M.build_file(mine, K, TABLES[name][1], i["absent"], h["v_init"], h["v_const"], 11, i["source_keys"]) == data
    for x in (m, m2, back):
        x.close()


@pytest.mark.parametrize("frozen", ["lr_ftrl", "fm_ftrl_k16"], indirect=True)
def test_damaged_and_foreign_files_are_refused(frozen, tmp_path):
    name, t, tr, trained = frozen
    good = str(tmp_path / "good")
    m = t.freeze()
    m.save(good)
    m.close()
    data = open(good, "rb").read()
    bad = str(tmp_path / "bad")

    def refused(content):
        open(bad, "wb").write(content)
        with pytest.raises(api.XflowError, match=ERR_IO):
            api.Model.load(bad)

    for cut in (0, 3, 50, 104, 104 + 32 + 5, len(data) - 16, len(data) - 1):
        refused(data[:cut])
    refused(data + b"\0" * 16)
    for pos in (5, 17, 37, 49, 90, 97, 104 + 1, 104 + 17, 104 + 32 + 3, 104 + 32 + 9, len(data) - 20):
        x = bytearray(data)
        x[pos] ^= 0x04
        refused(bytes(x))
    # checksums that pass over a row whose padding is not zero (LR bytes 12 .. 15, FM 20 .. 31)
    row_bytes = struct.unpack_from("<I", data, 32)[0]
    assert len(data) == 104 + 32 + struct.unpack_from("<Q", data, 16)[0] * row_bytes  # one chunk
    x = bytearray(data)
    x[104 + 32 + row_bytes - 1] = 1
    struct.pack_into("<Q", x, 104 + 16, M.section_sum(bytes(x[104 + 32:]), 0))
    open(bad, "wb").write(bytes(x))
    with pytest.raises(api.XflowError, match=ERR_IO + ".*padding"):
        api.Model.load(bad)
    xftb, xfst = str(tmp_path / "xftb"), str(tmp_path / "xfst")
    t.save(xftb)
    t.save_state(xfst)
    for other in (xftb, xfst):
        refused(open(other, "rb").read())
    with pytest.raises(api.XflowError, match=ERR_IO):
        api.Model.load(str(tmp_path / "missing"))
    api.Model.load(good).close()


def test_unwritable_path_leaves_no_tmp(monkeypatch, tmp_path):
    t, tr = _make("lr_ftrl", monkeypatch)
    _train(t, tr, n=1)
    m = t.freeze()
    path = str(tmp_path / "no_such_dir" / "model.xfsm")
    with pytest.raises(api.XflowError, match=ERR_IO):
        m.save(path)
    assert not os.path.exists(path) and not os.path.exists(path + ".tmp")
    m.close(); tr.close(); t.close()


# ---- 7. the staging grows ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lr_ftrl", "fm_ftrl_k16"])
def test_staging_grows_with_the_batch(name, monkeypatch):
    t, tr = _make(name, monkeypatch)
    trained = _train(t, tr)
    m = t.freeze()
    rp, keys = _query(1, trained)
    rp, keys = rp[:17], keys[:rp[16]]
    small = m.predict_host(rp, keys)
    rows, d = 65536, 100
    pool = np.concatenate([trained, _unseen()])
    big_keys = pool[np.random.default_rng(2).integers(0, pool.size, rows * d)]
    big = m.predict_host(np.arange(rows + 1, dtype=np.uint32) * d, big_keys)
    assert np.isfinite(big).all() and len(set(big[:1000].tolist())) > 100
    # row r of the big batch alone gives the same value
    for r in (0, 777, rows - 1):
        one = m.predict_host(np.array([0, d], np.uint32), big_keys[r * d:(r + 1) * d])
        assert _bits(one)[0] == _bits(big)[r]
    assert np.array_equal(_bits(m.predict_host(rp, keys)), _bits(small))
    m.close(); tr.close(); t.close()


# ---- 8. refusals ---------------------------------------------------------------------------------------------------
def test_refusals(monkeypatch):
    monkeypatch.delenv("XFLOW_EAGER", raising=False)
    canon = api.Table(latent_dim=8, canonical_fm=1)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*canonical"):
        canon.freeze()
    canon.close()
    shard = api.Table(shard_index=0, num_shards=2)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*shard"):
        shard.freeze()
    shard.close()
    t, tr = _make("lr_ftrl", monkeypatch)
    trained = _train(t, tr, n=1)
    with pytest.raises(api.XflowError, match=ERR_ARG):
        t.freeze(absent=7)
    m = t.freeze()
    bad = np.array([trained[0], 2 ** 64 - 1], np.uint64)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*reserved"):
        m.predict_host(np.array([0, 2], np.uint32), bad)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*reserved"):
        m.lookup(bad)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*row_ptr"):
        m.predict_host(np.array([0, 2, 1], np.uint32), trained[:2])
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*row_ptr"):
        m.predict_host(np.array([0, 3], np.uint32), trained[:2])
    ft, ftr = _make("fm_ftrl_k8", monkeypatch)
    ftr.ingest_text(b"1\t0:5:1 0:6:1\n0\t0:7:1\n")
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*model"):
        m.predict_ingested(ftr, 0, 2)
    tr.ingest_text(b"1\t0:5:1 0:6:1\n0\t0:7:1\n")
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*range"):
        m.predict_ingested(tr, 0, 3)
    assert m.predict_ingested(tr, 0, 2)[0].size == 2
    for x in (m, ftr, ft, tr, t):
        x.close()


# ---- 9. the CLI ----------------------------------------------------------------------------------------------------
def _cli(tmp, model, **extra):
    os.makedirs(tmp, exist_ok=True)
    env = dict(os.environ, XFLOW_OPTIMIZER="ftrl")
    for k in ("XFLOW_WORLD", "WORLD_SIZE", "XFLOW_EXPORT_MODEL", "XFLOW_EAGER", "XFLOW_ADMIT", "XFLOW_CHECKPOINT",
              "XFLOW_RESUME", "XFLOW_NEG_SAMPLE", "XFLOW_EVICT_MAX_KEYS", "XFLOW_EVICT_IDLE", "XFLOW_EVICT_EVERY"):
        env.pop(k, None)
    env.update(extra)
    return subprocess.run([EXE, TRAIN, TEST, model, "3"], cwd=tmp, env=env, capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("model", ["0", "1"])
def test_cli_exports_the_model_it_predicted_with(model, tmp_path):
    path = str(tmp_path / "model.xfsm")
    plain = _cli(str(tmp_path / "plain"), model)
    exported = _cli(str(tmp_path / "exported"), model, XFLOW_EXPORT_MODEL=path)
    assert plain.returncode == 0 and exported.returncode == 0, plain.stdout + plain.stderr + exported.stdout + exported.stderr
    assert plain.stdout == exported.stdout and "logloss" in plain.stdout
    pred = open(tmp_path / "exported" / "pred_0_0.txt").read()
    assert pred == open(tmp_path / "plain" / "pred_0_0.txt").read()
    lines = [l.split("\t") for l in pred.splitlines()]
    m = api.Model.load(path)
    i = m.info()
    assert i["fm"] == int(model) and i["keys"] > 0 and i["absent"] == api.ABSENT_DEFAULT
    assert i["pruned_keys"] > 0  # at least the keys the CLI's own predict inserted
    got, labels = [], []
    for rp, keys, lab in api.Loader(TEST + "-00000", 64 << 20):
        got.append(m.predict_host(rp, keys))
        labels.append(lab)
    got, labels = np.concatenate(got), np.concatenate(labels)
    assert 0 < len(lines) <= got.size
    assert [l[0] for l in lines] == ["%g" % float(p) for p in got[:len(lines)]]
    assert [int(l[2]) for l in lines] == labels[:len(lines)].tolist()
    m.close()


def test_cli_refuses_export_with_several_ranks(tmp_path):
    r = _cli(str(tmp_path / "w"), "0", XFLOW_EXPORT_MODEL=str(tmp_path / "m"), XFLOW_WORLD="2", XFLOW_RANK="0",
             XFLOW_COMM_FILE=str(tmp_path / "comm.id"))
    assert r.returncode != 0 and "XFLOW_EXPORT_MODEL" in r.stdout + r.stderr, r.stdout + r.stderr
    assert not os.path.exists(tmp_path / "m")

"""Serving models from sharded tables (xf_table_freeze_part, xf_model_merge, the XFSP file; csrc/serve.cu): the merge of
every shard's part is, byte for byte, the model xf_table_freeze makes of one unsharded table holding the same rows.

The shard tables are built on one GPU: an unsharded table is trained, every key's whole state exported, and each key
imported into the shard table xf_shard_of selects and into one more unsharded table U, which the merge is held to."""
import os
import struct
import subprocess
from contextlib import contextmanager

import numpy as np
import pytest

import serving_model as M
import serving_parts_model as P
from common import GOLDEN
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
TRAIN = os.path.join(GOLDEN, "data", "small_train")
TEST = os.path.join(GOLDEN, "data", "small_test")

TABLES = {  # name: (model, optimizer, K, eager LR)
    "lr_ftrl": (api.MODEL_LR, api.OPT_FTRL, 0, False),
    "lr_ftrl_eager": (api.MODEL_LR, api.OPT_FTRL, 0, True),
    "lr_sgd": (api.MODEL_LR, api.OPT_SGD, 0, False),
    "fm_ftrl_k10": (api.MODEL_FM, api.OPT_FTRL, 10, False),
    "fm_ftrl_k16": (api.MODEL_FM, api.OPT_FTRL, 16, False),
    "fm_sgd_k10": (api.MODEL_FM, api.OPT_SGD, 10, False),
    "fm_sgd_k16": (api.MODEL_FM, api.OPT_SGD, 16, False),
}
ALL = sorted(TABLES)
SHARDS = [1, 2, 3, 8]
B, D, SPACE, N = 512, 8, 20000, 3  # rows and tokens per training batch, id space, batches per epoch
CAP = 1 << 16
ERR_ARG, ERR_IO, ERR_STATE = "error -1:", "error -4:", "error -6:"
M64 = (1 << 64) - 1


@contextmanager
def _eager(name):
    old = os.environ.pop("XFLOW_EAGER", None)
    if TABLES[name][3]:
        os.environ["XFLOW_EAGER"] = "1"
    try:
        yield
    finally:
        os.environ.pop("XFLOW_EAGER", None)
        if old is not None:
            os.environ["XFLOW_EAGER"] = old


def _table(name, device=0, seed=11, **kw):
    _, opt, K, _ = TABLES[name]
    with _eager(name):
        # lambda1 well above a once-seen key's |z|, so that FTRL's L1 term leaves exact zeros to prune
        return api.Table(latent_dim=K, optimizer=opt, seed=seed, capacity=CAP, lambda1=2e-3, device=device, **kw)


def _keys_of(ids):
    return api.hash_decimal_ids(np.asarray(ids, np.uint64))


def _unseen():
    return _keys_of(np.arange(9 * SPACE, 9 * SPACE + 400))


_STATES = {}


def _state(name, epochs=1):
    """(keys, export) of a table trained epochs * N Zipf batches, with keys a Pull inserted and no batch trained"""
    if (name, epochs) not in _STATES:
        t = _table(name)
        tr = api.Trainer(t, model=TABLES[name][0], max_rows=B, max_nnz=B * D)
        for i in range(epochs * N):
            rp, ids, _ = datagen.make_ids(1000 + i, B, D, SPACE, dist="zipf")
            lab = (np.random.default_rng(i).random(B) < 0.3).astype(np.uint8)
            tr.step_host(rp, _keys_of(ids), lab, want_loss=False)
        t.pull(_keys_of(np.arange(5 * SPACE, 5 * SPACE + 300)), want_v=False)
        tr.sync()
        keys = np.sort(t.list_keys())
        _STATES[(name, epochs)] = (keys, t.export(keys))
        tr.close()
        t.close()
    return _STATES[(name, epochs)]


def _import(t, ex, sel, K):
    f = dict(w=ex["w"][sel], nw=ex["nw"][sel], zw=ex["zw"][sel])
    if K:
        f.update(v=ex["v"][sel], nv=ex["nv"][sel], zv=ex["zv"][sel])
    t.import_(ex["keys"][sel], **f)


def _tables(name, S, epochs=1, device=0):
    """(shard tables 0 .. S-1, the unsharded table U) holding the trained state"""
    keys, ex = _state(name, epochs)
    K = TABLES[name][2]
    owner = P.shard_of(keys, S)
    shards = []
    for s in range(S):
        t = _table(name, device=device, shard_index=s, num_shards=S)
        _import(t, ex, owner == s, K)
        shards.append(t)
    u = _table(name)
    _import(u, ex, np.ones(keys.size, bool), K)
    return shards, u


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _bytes(m, path):
    m.save(path)
    return open(path, "rb").read()


def _golden_predict(m):
    out = []
    for rp, keys, _ in api.Loader(TEST + "-00000", 64 << 20):
        out.append(m.predict_host(rp, keys))
    return np.concatenate(out)


def _query_predict(m, keys):
    """rows of 0 .. 300 tokens over the trained keys and keys no table holds"""
    rng = np.random.default_rng(3)
    pool = np.concatenate([keys, _unseen()])
    lens = np.array([0, 1, 63, 64, 65, 300] + [8] * 40)
    rp = np.zeros(lens.size + 1, np.uint32)
    rp[1:] = np.cumsum(lens)
    return m.predict_host(rp, pool[rng.integers(0, pool.size, int(rp[-1]))])


def _close(*xs):
    for x in xs:
        if isinstance(x, list):
            _close(*x)
        else:
            x.close()


# ---- 1. the merge is the unsharded freeze ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ALL)
@pytest.mark.parametrize("S", SHARDS)
@pytest.mark.parametrize("prune", [True, False])
def test_merge_is_the_freeze_of_one_table(name, S, prune, tmp_path):
    shards, u = _tables(name, S)
    whole = u.freeze(prune=prune)
    parts = [t.freeze_part(prune=prune) for t in shards]
    assert [p.part_info() for p in parts] == [(s, S) for s in range(S)]
    merged = api.Model.merge(parts)
    want = _bytes(whole, str(tmp_path / "whole"))
    assert _bytes(merged, str(tmp_path / "merged")) == want
    assert merged.info() == whole.info()
    assert sum(p.fingerprint() for p in parts) % (1 << 64) == merged.fingerprint() == whole.fingerprint()
    assert np.array_equal(_bits(_golden_predict(merged)), _bits(_golden_predict(whole)))
    got, ref = _query_predict(merged, _state(name)[0]), _query_predict(whole, _state(name)[0])
    assert np.array_equal(_bits(got), _bits(ref)) and len(set(ref.tolist())) > 10
    # each part holds the whole model's rows of its range and nothing else
    allk = np.concatenate([u.list_keys(), _unseen()])
    lw = whole.lookup(allk)
    owner = P.shard_of(allk, S)
    for s, p in enumerate(parts):
        lp = p.lookup(allk)
        assert np.array_equal(lp["present"], lw["present"] * (owner == s))
        have = lp["present"].astype(bool)
        for f in ("w", "st", "qt"):
            assert np.array_equal(_bits(lp[f][have]), _bits(lw[f][have]))
        i = p.info()
        assert i["keys"] == int(have.sum()) and i["source_keys"] == int((owner[:u.size()] == s).sum())
        assert i["capacity"] == M.capacity_for(i["keys"])
    for f in ("keys", "source_keys", "pruned_keys"):
        assert sum(p.info()[f] for p in parts) == whole.info()[f]
    if not prune:
        assert whole.info()["pruned_keys"] == 0
    _close(parts, merged, whole, shards, u)


# ---- 2. files ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lr_ftrl", "fm_ftrl_k16", "fm_sgd_k10"])
@pytest.mark.parametrize("S", [1, 3, 8])
def test_part_files_round_trip_and_merge_on_the_host(name, S, tmp_path):
    shards, u = _tables(name, S)
    whole = u.freeze()
    want = _bytes(whole, str(tmp_path / "whole"))
    paths = [str(tmp_path / ("p%d.xfsp" % s)) for s in range(S)]
    files = []
    for t, path in zip(shards, paths):
        p = t.freeze_part()
        files.append(_bytes(p, path))
        assert not os.path.exists(path + ".tmp")
        back = api.Model.load(path)
        assert back.part_info() == p.part_info() and back.info() == p.info() and back.fingerprint() == p.fingerprint()
        assert _bytes(back, path + ".again") == files[-1]
        _close(p, back)
    # the documented layout, and the numpy statement of the format
    for s, data in enumerate(files):
        h, rows = P.parse_part(data)
        assert data[:4] == b"XFSP" and struct.unpack_from("<QiiQ", data, 8)[0] == 112
        assert struct.unpack_from("<ii", data, 96) == (s, S)
    loaded = [api.Model.load(path) for path in paths[::-1]]  # any order
    merged = api.Model.merge(loaded)
    assert _bytes(merged, str(tmp_path / "merged")) == want
    assert P.merge(files) == want
    _close(loaded, merged, whole, shards, u)


# ---- 3. deltas -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lr_ftrl", "fm_ftrl_k16"])
def test_merged_models_carry_deltas(name, tmp_path):
    S = 3
    models = []
    for epochs in (1, 2):
        shards, u = _tables(name, S, epochs=epochs)
        parts = [t.freeze_part() for t in shards]
        models.append((api.Model.merge(parts), u.freeze()))
        _close(parts, shards, u)
    (m1, w1), (m2, w2) = models
    d = m1.diff(m2)
    assert d.info()["upserts"] > 0
    m3 = m1.apply(d)
    want = _bytes(w2, str(tmp_path / "w2"))
    assert _bytes(m3, str(tmp_path / "m3")) == want == _bytes(m2, str(tmp_path / "m2"))
    assert np.array_equal(_bits(_query_predict(m3, _state(name, 2)[0])), _bits(_query_predict(w2, _state(name, 2)[0])))
    _close(d, m1, w1, m2, w2, m3)


# ---- 4. nothing changes --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lr_ftrl", "fm_ftrl_k10"])
def test_freeze_part_and_merge_change_no_table_or_part(name, tmp_path):
    S = 3
    shards, u = _tables(name, S)
    before = []
    for s, t in enumerate(shards):
        path = str(tmp_path / ("before%d" % s))
        t.save_state(path, user=1)
        before.append(open(path, "rb").read())
    parts = [t.freeze_part() for t in shards]
    fps = [p.fingerprint() for p in parts]
    infos = [p.info() for p in parts]
    merged = api.Model.merge(parts)
    again = api.Model.merge(parts, device=0)
    assert _bytes(merged, str(tmp_path / "a")) == _bytes(again, str(tmp_path / "b"))
    assert [p.fingerprint() for p in parts] == fps and [p.info() for p in parts] == infos
    for s, t in enumerate(shards):
        path = str(tmp_path / ("after%d" % s))
        t.save_state(path, user=1)
        assert open(path, "rb").read() == before[s]
    _close(parts, merged, again, shards, u)


# ---- 5. refusals ---------------------------------------------------------------------------------------------------------
def test_refusals(tmp_path):
    name, S = "fm_ftrl_k10", 3
    shards, u = _tables(name, S)
    parts = [t.freeze_part() for t in shards]
    whole = u.freeze()
    # tables
    canon = api.Table(latent_dim=8, canonical_fm=1)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*canonical"):
        canon.freeze_part()
    canon.close()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*shard.*xf_table_freeze_part"):
        shards[0].freeze()
    foreign = _table(name, shard_index=0, num_shards=2)
    keys = np.array([5, M64 // 2 + 7, M64 - 1], np.uint64)  # shard 0, 1, 1
    foreign.import_(keys, w=np.ones(3, np.float32))
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*2 keys outside"):
        foreign.freeze_part()
    foreign.close()
    # a part is not a model
    with pytest.raises(api.XflowError, match=ERR_STATE):
        whole.part_info()
    rp, qk = np.array([0, 2], np.uint32), u.list_keys()[:2]
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*xf_model_merge"):
        parts[0].predict_host(rp, qk)
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*xf_model_merge"):
        parts[0].predict_device(1, 1, 0, 0, 1)  # refused before any pointer is read
    tr = api.Trainer(u, model=api.MODEL_FM, max_rows=64, max_nnz=256)
    tr.ingest_text(b"1\t0:5:1 0:6:1\n0\t0:7:1\n")
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*xf_model_merge"):
        parts[0].predict_ingested(tr, 0, 2)
    tr.close()
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*xf_model_merge"):
        parts[0].diff(whole)
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*xf_model_merge"):
        whole.diff(parts[0])
    d = whole.diff(whole)
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*xf_model_merge"):
        parts[0].apply(d)
    d.close()
    # what a merge takes: every shard of one split, once, alike
    for bad, why in ((parts[:2], "3-way split, but 2"), ([parts[0], parts[1], parts[1]], "twice"),
                     ([parts[0], parts[1], whole], "whole model"), ([], "parts")):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*" + why):
            api.Model.merge(bad)
    two = _tables(name, 2)[0]
    p2 = [t.freeze_part() for t in two]
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*2-way split, but 3"):
        api.Model.merge([parts[0], parts[1], p2[1]])
    zero = shards[2].freeze_part(absent=api.ABSENT_ZERO)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*absent"):
        api.Model.merge([parts[0], parts[1], zero])
    seeded = _table(name, seed=12, shard_index=2, num_shards=3)
    sp = seeded.freeze_part()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*seed"):
        api.Model.merge([parts[0], parts[1], sp])
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*device"):
        api.Model.merge(parts, device=api.device_count())
    unpruned = shards[1].freeze_part(prune=False)  # prune may differ
    api.Model.merge([parts[0], unpruned, parts[2]]).close()
    _close(p2, two, zero, sp, seeded, unpruned, parts, whole, shards, u)


def test_damaged_part_files_are_refused(tmp_path):
    shards, u = _tables("lr_ftrl", 3)
    good = str(tmp_path / "good.xfsp")
    p = shards[1].freeze_part()
    data = _bytes(p, good)
    p.close()
    assert len(data) > 112 + 32 + 16 * 10
    bad = str(tmp_path / "bad")

    def refused(content, match=ERR_IO):
        open(bad, "wb").write(content)
        with pytest.raises(api.XflowError, match=match):
            api.Model.load(bad)

    for cut in (3, 50, 104, 111, 112 + 32 + 5, len(data) - 1):
        refused(data[:cut])
    for pos in (5, 20, 97, 101, 106, 112 + 9, len(data) - 3):
        x = bytearray(data)
        x[pos] ^= 0x04
        refused(bytes(x))

    def resummed(x):
        x = bytearray(x)
        struct.pack_into("<Q", x, 104, M.section_sum(bytes(x[:104])))
        body = bytes(x[112 + 32:])
        struct.pack_into("<Q", x, 112 + 16, M.section_sum(body, 0))
        return bytes(x)

    assert resummed(data) == data  # one chunk: the re-summing alone changes nothing
    x = bytearray(data)
    struct.pack_into("<Q", x, len(x) - 16, P.shard_range(2, 3)[0])  # a key of shard 2, last: still ascending
    refused(resummed(x), ERR_IO + ".*outside shard 1 of 3")
    x = bytearray(data)
    x[112 + 32:112 + 48], x[112 + 48:112 + 64] = data[112 + 48:112 + 64], data[112 + 32:112 + 48]
    refused(resummed(x), ERR_IO + ".*ascending")
    x = bytearray(data)
    struct.pack_into("<i", x, 96, 3)
    refused(resummed(x), ERR_IO + ".*shard 3 of 3")
    with pytest.raises(api.XflowError, match=ERR_IO + ".*XFSP"):
        api.Delta.load(good)
    api.Model.load(good).close()
    _close(shards, u)


# ---- 6. the CLI ----------------------------------------------------------------------------------------------------------
def _cli(tmp, model, **extra):
    os.makedirs(tmp, exist_ok=True)
    env = dict(os.environ, XFLOW_OPTIMIZER="ftrl")
    for k in ("XFLOW_WORLD", "WORLD_SIZE", "XFLOW_EXPORT_MODEL", "XFLOW_EXPORT_SHARDED_MODEL", "XFLOW_EXPORT_DELTAS",
              "XFLOW_EAGER", "XFLOW_ADMIT", "XFLOW_CHECKPOINT", "XFLOW_RESUME", "XFLOW_NEG_SAMPLE",
              "XFLOW_EVICT_MAX_KEYS", "XFLOW_EVICT_IDLE", "XFLOW_EVICT_EVERY"):
        env.pop(k, None)
    env.update(extra)
    return subprocess.run([EXE, TRAIN, TEST, model, "3"], cwd=tmp, env=env, capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("model", ["0", "1"])
def test_cli_sharded_export_at_world_one(model, tmp_path):
    out = tmp_path / "out"
    out.mkdir()
    a, b = str(out / "plain.xfsm"), str(out / "sharded.xfsm")
    ra = _cli(str(tmp_path / "a"), model, XFLOW_EXPORT_MODEL=a)
    rb = _cli(str(tmp_path / "b"), model, XFLOW_EXPORT_SHARDED_MODEL=b)
    assert ra.returncode == 0 and rb.returncode == 0, ra.stdout + ra.stderr + rb.stdout + rb.stderr
    assert ra.stdout == rb.stdout
    assert open(a, "rb").read() == open(b, "rb").read()
    assert sorted(os.listdir(out)) == ["plain.xfsm", "sharded.xfsm"]  # no part file is left
    both = _cli(str(tmp_path / "c"), model, XFLOW_EXPORT_MODEL=str(out / "x"), XFLOW_EXPORT_SHARDED_MODEL=str(out / "y"))
    assert both.returncode != 0 and "XFLOW_EXPORT_SHARDED_MODEL" in both.stdout + both.stderr
    assert sorted(os.listdir(out)) == ["plain.xfsm", "sharded.xfsm"]


# ---- 7. two GPUs ---------------------------------------------------------------------------------------------------------
def test_parts_on_another_device_merge_alike(tmp_path):
    if api.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    for name in ("lr_ftrl", "fm_ftrl_k16"):
        shards, u = _tables(name, 3, device=1)
        parts = [t.freeze_part() for t in shards]
        here = api.Model.merge(parts)          # on device 1, in place
        there = api.Model.merge(parts, device=0)  # staged over peer copies
        w = u.freeze()
        want = _bytes(w, str(tmp_path / "w"))
        assert _bytes(here, str(tmp_path / "h")) == want == _bytes(there, str(tmp_path / "t"))
        assert np.array_equal(_bits(_golden_predict(there)), _bits(_golden_predict(here)))
        _close(parts, here, there, w, shards, u)


@pytest.mark.parametrize("model", ["0", "1"])
def test_cli_two_ranks_export_one_model(model, tmp_path):
    if api.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    lines = open(TRAIN + "-00000", "rb").read().splitlines(keepends=True)
    prefix = str(tmp_path / "train")
    open(prefix + "-00000", "wb").write(b"".join(lines[:120]))
    open(prefix + "-00001", "wb").write(b"".join(lines[120:]))
    path = str(tmp_path / "model.xfsm")
    procs = []
    for rank in range(2):
        cwd = tmp_path / ("rank%d" % rank)
        cwd.mkdir()
        env = dict(os.environ, XFLOW_OPTIMIZER="ftrl", XFLOW_RANK=str(rank), XFLOW_WORLD="2", XFLOW_DEVICE=str(rank),
                   XFLOW_COMM_FILE=str(tmp_path / "comm.id"), XFLOW_MG_TIMEOUT_S="60", XFLOW_SEED="0",
                   XFLOW_EXPORT_SHARDED_MODEL=path)
        env.pop("XFLOW_EXPORT_MODEL", None)
        procs.append(subprocess.Popen([EXE, prefix, TEST, model, "5"], cwd=str(cwd), env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    for p in procs:
        out, _ = p.communicate(timeout=600)
        assert p.returncode == 0, out
    assert [f for f in os.listdir(tmp_path) if ".part-" in f] == []
    m = api.Model.load(path)
    assert m.info()["keys"] > 0
    got = _golden_predict(m)
    pred = np.loadtxt(str(tmp_path / "rank0" / "pred_0_0.txt"), ndmin=2)[:, 0]
    assert 0 < pred.size <= got.size
    assert np.all(np.abs(got[:pred.size] - pred) <= 2e-5 * np.abs(pred) + 1.1e-6)
    m.close()

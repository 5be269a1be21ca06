"""Serving model deltas (xf_model_diff / xf_model_apply_delta / xf_delta_*, csrc/delta.cu): applying the delta from A to
B to A gives B, byte for byte in its file and bit for bit in its predictions; the delta holds exactly the keys the two
models' contents say it must; diff and apply change no model; damaged, malformed and mismatched deltas are refused."""
import os
import subprocess

import numpy as np
import pytest

import delta_model as D
import serving_model as SM
from test_gpu_serving import (ALL, EXE, SOME, TABLES, TEST, TRAIN, _bits, _keys_of, _make, _pulled, _query, _train,
                              _unseen)
from xflow_b200 import api

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_FULL, ERR_IO, ERR_STATE = "error -1:", "error -3:", "error -4:", "error -6:"
ABSENT = {"default": api.ABSENT_DEFAULT, "zero": api.ABSENT_ZERO}


def _read(path):
    return open(path, "rb").read()


def _saved(m, path):
    m.save(path)
    return _read(path)


def _new_keys(first, n=500):
    """keys no earlier batch or pull has seen"""
    return _keys_of(np.arange(first, first + n))


def _evolve(name, t, tr, trained, round_):
    """More training after a freeze: batches of the same stream, a batch of new keys, trained keys set to an exact 0
    (FTRL's L1 term writes such zeros; the import writes them deterministically), a Pull that inserts default rows, and
    (lazy LR, FM) an eviction sweep that removes keys.  Returns every key the table has held."""
    K, eager = TABLES[name][2], TABLES[name][3]
    more = _train(t, tr, first=10 * round_, n=2)
    new = _new_keys(20 * 20000 + 1000 * round_)
    rp = (np.arange(new.size // 5 + 1) * 5).astype(np.uint32)
    tr.step_host(rp, new, (np.arange(new.size // 5) % 2).astype(np.uint8), want_loss=False)
    zero = trained[round_ * 7:round_ * 7 + 40]
    t.import_(zero, w=np.zeros(zero.size), nw=np.zeros(zero.size), zw=np.zeros(zero.size),
              v=np.zeros((zero.size, K)) if K else None, nv=np.zeros((zero.size, K)) if K else None,
              zv=np.zeros((zero.size, K)) if K else None)
    pulled = _keys_of(np.arange(6 * 20000 + 300 * round_, 6 * 20000 + 300 * round_ + 200))
    t.pull(pulled, want_v=False)
    if not eager:
        assert t.evict() > 0
    return np.unique(np.concatenate([trained, more, new, pulled, _pulled()]))


def _fresh(name, monkeypatch):
    t, tr = _make(name, monkeypatch)
    if not TABLES[name][3]:
        t.set_eviction(max_idle_batches=3)
    return t, tr


def _snapshot(m, path, rp, keys):
    return m.fingerprint(), _saved(m, path), _bits(m.predict_host(rp, keys)), m.info()


# ---- 1. apply(A, diff(A, B)) is B -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ALL)
@pytest.mark.parametrize("absent", ["default", "zero"])
def test_apply_of_diff_is_the_next_model(name, absent, monkeypatch, tmp_path):
    t, tr = _fresh(name, monkeypatch)
    trained = _train(t, tr)
    a = t.freeze(absent=ABSENT[absent])
    trained = _evolve(name, t, tr, trained, 1)
    b = t.freeze(absent=ABSENT[absent])
    rp, keys = _query(21, trained)
    p = lambda x: str(tmp_path / x)  # noqa: E731
    before = [_snapshot(x, p("before_%d" % i), rp, keys) for i, x in enumerate((a, b))]
    d = a.diff(b)
    r = a.apply(d)
    # the result is B: file, info, fingerprint, predictions (held-out rows with unseen keys)
    want_file = _saved(b, p("b"))
    assert _saved(r, p("r")) == want_file
    assert r.info() == b.info() and r.fingerprint() == b.fingerprint() == d.info()["result_fingerprint"]
    assert np.array_equal(_bits(r.predict_host(rp, keys)), _bits(b.predict_host(rp, keys)))
    # the same through the file
    d.save(p("d"))
    data = _read(p("d"))
    assert len(data) == d.info()["file_bytes"]
    d2 = api.Delta.load(p("d"))
    assert d2.info() == d.info()
    r2 = a.apply(d2)
    assert _saved(r2, p("r2")) == want_file
    assert np.array_equal(_bits(r2.predict_host(rp, keys)), _bits(b.predict_host(rp, keys)))
    d2.save(p("d2"))
    assert _read(p("d2")) == data
    # the delta holds exactly the keys the two models' contents say it must
    allk = np.unique(np.concatenate([np.sort(t.list_keys()), trained, _unseen()]))
    la, lb = a.lookup(allk), b.lookup(allk)
    pa, pb = la["present"].astype(bool), lb["present"].astype(bool)
    differs = np.zeros(allk.size, bool)
    for f in ("w", "st", "qt"):
        differs |= _bits(la[f]) != _bits(lb[f])
    h, up, de = D.parse_file(data)
    assert np.array_equal(up["key"], allk[pb & (~pa | differs)])
    assert np.array_equal(de, allk[pa & ~pb])
    assert up.size > 0 and (de.size > 0 or TABLES[name][3])
    ia, ib = a.info(), b.info()
    assert (h["base_keys"], h["result_keys"], h["source_keys"], h["pruned_keys"]) == \
        (ia["keys"], ib["keys"], ib["source_keys"], ib["pruned_keys"])
    assert h["base_fingerprint"] == a.fingerprint()
    # the numpy statement: the model files' rows, diffed and applied, and its file of that delta is the library's
    _, rows_a = SM.parse_file(before[0][1])
    hb, rows_b = SM.parse_file(want_file)
    assert D.fingerprint(rows_a) == a.fingerprint() and D.fingerprint(rows_b) == b.fingerprint()
    assert D.delta_file(rows_a, rows_b, ib["source_keys"], hb["latent_dim"], hb["optimizer"], hb["absent"], hb["v_init"],
                        hb["v_const"], hb["seed"]) == data
    # neither model changed
    after = [_snapshot(x, p("after_%d" % i), rp, keys) for i, x in enumerate((a, b))]
    for x, y in zip(before, after):
        assert x[0] == y[0] and x[1] == y[1] and np.array_equal(x[2], y[2]) and x[3] == y[3]
    for x in (a, b, r, r2, d, d2, tr, t):
        x.close()


@pytest.mark.parametrize("name", SOME)
def test_a_chain_of_five_deltas_reproduces_the_last_model(name, monkeypatch, tmp_path):
    t, tr = _fresh(name, monkeypatch)
    trained = _train(t, tr)
    models = [t.freeze()]
    for i in range(1, 6):
        trained = _evolve(name, t, tr, trained, i)
        models.append(t.freeze())
    for i in range(5):
        models[i].diff(models[i + 1]).save(str(tmp_path / ("d%d" % i)))
    models[0].save(str(tmp_path / "m0"))
    cur = api.Model.load(str(tmp_path / "m0"))
    for i in range(5):
        d = api.Delta.load(str(tmp_path / ("d%d" % i)))
        nxt = cur.apply(d)
        cur.close()
        d.close()
        cur = nxt
    rp, keys = _query(5, trained)
    assert _saved(cur, str(tmp_path / "got")) == _saved(models[5], str(tmp_path / "want"))
    assert np.array_equal(_bits(cur.predict_host(rp, keys)), _bits(models[5].predict_host(rp, keys)))
    for x in models + [cur, tr, t]:
        x.close()


# ---- 2. edges -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lr_ftrl", "fm_ftrl_k16"])
def test_edges(name, monkeypatch, tmp_path):
    t, tr = _fresh(name, monkeypatch)
    empty = t.freeze()  # a fresh table
    assert empty.info()["keys"] == 0 and empty.fingerprint() == 0
    _train(t, tr)
    extra = _new_keys(30 * 20000, 3000)  # enough kept rows for a model past the smallest capacity
    t.import_(extra, w=np.full(extra.size, 0.5), nw=np.ones(extra.size), zw=np.zeros(extra.size))
    m = t.freeze()
    want = _saved(m, str(tmp_path / "m"))
    # diff(A, A) is empty, and applying it changes nothing
    same = m.diff(m)
    i = same.info()
    assert (i["upserts"], i["deletes"]) == (0, 0) and i["base_fingerprint"] == i["result_fingerprint"] == m.fingerprint()
    assert i["file_bytes"] == 144
    r = m.apply(same)
    assert _saved(r, str(tmp_path / "r")) == want
    # from an empty model: a full model, and the result's capacity grows past the base's
    full = empty.diff(m)
    assert (full.info()["upserts"], full.info()["deletes"]) == (m.info()["keys"], 0)
    grown = empty.apply(full)
    assert grown.info()["capacity"] > empty.info()["capacity"] and grown.info() == m.info()
    assert _saved(grown, str(tmp_path / "g")) == want
    # to an empty model: every key deleted, and the capacity shrinks back
    gone = m.diff(empty)
    assert (gone.info()["upserts"], gone.info()["deletes"]) == (0, m.info()["keys"])
    shrunk = m.apply(gone)
    assert shrunk.info()["capacity"] == 1024 < m.info()["capacity"] and shrunk.fingerprint() == 0
    assert _saved(shrunk, str(tmp_path / "s")) == _saved(empty, str(tmp_path / "e"))
    for x in (same, r, full, grown, gone, shrunk, empty, m, tr, t):
        x.close()


def test_a_delta_of_more_than_one_chunk(monkeypatch, tmp_path):
    """over 4 x 2^20 LR upserts: the 16-byte rows take two 64 MiB chunks"""
    monkeypatch.delenv("XFLOW_EAGER", raising=False)
    n = (4 << 20) + 4321
    t = api.Table(seed=3, capacity=1 << 24)
    empty = t.freeze()
    keys = _keys_of(np.arange(n))
    w = np.random.default_rng(1).standard_normal(n).astype(np.float32)
    t.import_(keys, w=w, nw=np.ones(n), zw=np.zeros(n))
    m = t.freeze()
    assert m.info()["keys"] == n
    d = empty.diff(m)
    path = str(tmp_path / "d")
    d.save(path)
    d.close()
    d = api.Delta.load(path)
    assert d.info()["upserts"] == n and d.info()["file_bytes"] == 144 + 2 * 32 + 16 * n
    r = empty.apply(d)
    assert _saved(r, str(tmp_path / "r")) == _saved(m, str(tmp_path / "m"))
    # and back: n deletes
    back = m.diff(empty)
    back.save(str(tmp_path / "back"))
    back2 = api.Delta.load(str(tmp_path / "back"))
    assert back2.info()["deletes"] == n and m.apply(back2).info()["keys"] == 0
    for x in (d, r, back, back2, m, empty, t):
        x.close()


# ---- 3. refusals ----------------------------------------------------------------------------------------------------
def test_incompatible_models_are_refused(monkeypatch):
    lr, lr_tr = _make("lr_ftrl", monkeypatch)
    _train(lr, lr_tr, n=1)
    fm, fm_tr = _make("fm_ftrl_k8", monkeypatch)
    _train(fm, fm_tr, n=1)
    sgd, sgd_tr = _make("lr_sgd", monkeypatch)
    _train(sgd, sgd_tr, n=1)
    other_seed = api.Table(seed=12, capacity=1 << 12, lambda1=2e-3)
    a = lr.freeze()
    for other, field in ((fm.freeze(), "fm"), (sgd.freeze(), "optimizer"), (lr.freeze(absent=api.ABSENT_ZERO), "absent"),
                         (other_seed.freeze(), "seed")):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*" + field):
            a.diff(other)
        d = other.diff(other)
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*" + field):
            a.apply(d)
        d.close()
        other.close()
    a.close()
    for x in (lr_tr, lr, fm_tr, fm, sgd_tr, sgd, other_seed):
        x.close()


@pytest.mark.skipif(api.device_count() < 2, reason="needs two GPUs")
def test_models_on_two_devices_are_refused(monkeypatch):
    t, tr = _make("lr_ftrl", monkeypatch)
    _train(t, tr, n=1)
    a, b = t.freeze(), t.freeze(device=1)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*device"):
        a.diff(b)
    d = b.diff(b)
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*device"):
        a.apply(d)
    for x in (d, a, b, tr, t):
        x.close()


@pytest.mark.parametrize("name", ["lr_ftrl", "fm_ftrl_k16"])
def test_wrong_base_and_bad_files_are_refused(name, monkeypatch, tmp_path):
    t, tr = _fresh(name, monkeypatch)
    trained = _train(t, tr)
    a = t.freeze()
    trained = _evolve(name, t, tr, trained, 1)
    b = t.freeze()
    d = a.diff(b)
    good = str(tmp_path / "good")
    d.save(good)
    data = _read(good)
    # the wrong base: another key count, or the same key count with other contents
    with pytest.raises(api.XflowError, match=ERR_STATE):
        b.apply(d)
    _, rows_a = SM.parse_file(_saved(a, str(tmp_path / "a")))
    _, rows_b = SM.parse_file(_saved(b, str(tmp_path / "b")))
    hb = SM.parse_file(_read(str(tmp_path / "b")))[0]
    compat = (hb["latent_dim"], hb["optimizer"], hb["absent"], hb["v_init"], hb["v_const"], hb["seed"])
    up, de = D.diff(rows_a, rows_b)
    bad = str(tmp_path / "bad")

    def write(content):
        open(bad, "wb").write(content)
        return bad

    def build(u=up, d_=de, base_fp=None, result_keys=rows_b.size, source_keys=hb["source_keys"], result_fp=None):
        return D.build_file(u, d_, *compat, rows_a.size, D.fingerprint(rows_a) if base_fp is None else base_fp, result_keys,
                            source_keys, D.fingerprint(rows_b) if result_fp is None else result_fp)

    assert build() == data
    other = api.Delta.load(write(build(base_fp=D.fingerprint(rows_a) ^ 1)))
    with pytest.raises(api.XflowError, match=ERR_STATE + ".*not the delta's base"):
        a.apply(other)
    other.close()
    # a result past 2^32 slots
    huge = api.Delta.load(write(build(result_keys=1 << 32, source_keys=1 << 32)))
    with pytest.raises(api.XflowError, match=ERR_FULL):
        a.apply(huge)
    huge.close()

    def refused(content, what=""):
        with pytest.raises(api.XflowError, match=ERR_IO + what):
            api.Delta.load(write(content))

    # damaged, truncated, other formats
    for cut in (0, 3, 100, 144, 144 + 32 + 5, len(data) - 8, len(data) - 1):
        refused(data[:cut])
    refused(data + b"\0" * 8)
    for pos in (5, 17, 30, 41, 60, 75, 99, 107, 115, 121, 137, 144 + 1, 144 + 17, 144 + 32 + 3, len(data) - 5):
        x = bytearray(data)
        x[pos] ^= 0x10
        refused(bytes(x))
    t.save(str(tmp_path / "xftb"))
    t.save_state(str(tmp_path / "xfst"))
    refused(_read(str(tmp_path / "a")), ".*serving model")
    refused(_read(str(tmp_path / "xftb")), ".*checkpoint")
    refused(_read(str(tmp_path / "xfst")), ".*checkpoint")
    with pytest.raises(api.XflowError, match=ERR_IO):
        api.Delta.load(str(tmp_path / "missing"))
    # checksums that pass over contents that break the format
    assert up.size > 3 and de.size > 3
    pad = up.copy()
    if up.dtype == SM.FM_ROW:
        pad["pad"][1, 2] = 7
    else:
        pad["pad"][1] = 1
    dup = up.copy()
    dup["key"][2] = dup["key"][1]
    reserved = up.copy()
    reserved["key"][-1] = D.EMPTY
    reserved_del = de.copy()
    reserved_del[-1] = D.EMPTY
    both = np.sort(np.append(de[1:], up["key"][0]))
    for u, d_, what in ((up[::-1], de, "ascending"), (up, de[::-1], "ascending"), (dup, de, "ascending"),
                        (reserved, de, "ascending"), (up, reserved_del, "ascending"), (pad, de, "padding"),
                        (up, both, "both")):
        refused(build(u=u, d_=d_), ".*" + what)
    api.Delta.load(good).close()
    for x in (d, a, b, tr, t):
        x.close()


# ---- 4. the CLI -----------------------------------------------------------------------------------------------------
def _cli(tmp, model, **extra):
    os.makedirs(tmp, exist_ok=True)
    env = dict(os.environ, XFLOW_OPTIMIZER="ftrl")
    for k in ("XFLOW_WORLD", "WORLD_SIZE", "XFLOW_EXPORT_MODEL", "XFLOW_EXPORT_DELTAS", "XFLOW_EAGER", "XFLOW_ADMIT",
              "XFLOW_CHECKPOINT", "XFLOW_RESUME", "XFLOW_NEG_SAMPLE", "XFLOW_EVICT_MAX_KEYS", "XFLOW_EVICT_IDLE",
              "XFLOW_EVICT_EVERY"):
        env.pop(k, None)
    env.update(extra)
    return subprocess.run([EXE, TRAIN, TEST, model, "3"], cwd=tmp, env=env, capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("model", ["0", "1"])
def test_cli_writes_a_chain_that_ends_at_the_exported_model(model, tmp_path):
    prefix, export = str(tmp_path / "run"), str(tmp_path / "model.xfsm")
    plain = _cli(str(tmp_path / "plain"), model)
    run = _cli(str(tmp_path / "deltas"), model, XFLOW_EXPORT_DELTAS=prefix, XFLOW_EXPORT_MODEL=export)
    assert plain.returncode == 0 and run.returncode == 0, plain.stdout + plain.stderr + run.stdout + run.stderr
    assert plain.stdout == run.stdout and "logloss" in plain.stdout
    assert sorted(os.listdir(tmp_path)) == ["deltas", "model.xfsm", "plain", "run-1.xfsm", "run-2.xfsd", "run-3.xfsd"]
    cur = api.Model.load(prefix + "-1.xfsm")
    for e in (2, 3):
        d = api.Delta.load("%s-%d.xfsd" % (prefix, e))
        assert d.info()["upserts"] > 0
        nxt = cur.apply(d)
        cur.close()
        d.close()
        cur = nxt
    got = _saved(cur, str(tmp_path / "chain.xfsm"))
    want = _read(export)
    hg, rows_g = SM.parse_file(got)
    hw, rows_w = SM.parse_file(want)
    assert rows_g.tobytes() == rows_w.tobytes() and hg["keys"] == hw["keys"] > 0
    assert hg["latent_dim"] == (10 if model == "1" else 0)
    # the export was frozen after the final predict: the keys it inserted are pruned, and nothing else differs
    inserted = hw["source_keys"] - hg["source_keys"]
    assert inserted > 0 and hw["pruned_keys"] - hg["pruned_keys"] == inserted
    assert got[104:] == want[104:]
    cur.close()


def test_cli_refuses_deltas_with_several_ranks(tmp_path):
    r = _cli(str(tmp_path / "w"), "0", XFLOW_EXPORT_DELTAS=str(tmp_path / "d"), XFLOW_WORLD="2", XFLOW_RANK="0",
             XFLOW_COMM_FILE=str(tmp_path / "comm.id"))
    assert r.returncode != 0 and "XFLOW_EXPORT_DELTAS" in r.stdout + r.stderr, r.stdout + r.stderr
    assert not [f for f in os.listdir(tmp_path) if f.startswith("d-")]

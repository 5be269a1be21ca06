"""Half-precision serving models (xf_model_convert, csrc/serve.cu): an F16 model holds the binary16 rounding of the F32
model's latent fields and nothing else changes; every predict entry point returns on it, bit for bit, what it returns on
the F32 model whose latent fields are replaced by their rounding; against the original F32 model the arguments move by
no more than compact_serving_model's bound; files, deltas, merges and the CLI carry the precision."""
import os
import struct
import subprocess

import numpy as np
import pytest

import canonical_serving_model as CM
import compact_serving_model as H
import delta_model as DM
import fm_model as FMM
import serving_model as SM
import test_gpu_canonical_serving as TC
import test_gpu_serving as TS
import test_gpu_serving_parts as TP
from xflow_b200 import api

pytestmark = pytest.mark.gpu

F32, F16 = api.PRECISION_F32, api.PRECISION_F16
ERR_ARG, ERR_IO, ERR_STATE = "error -1:", "error -4:", "error -6:"
FM_NAMES = ["fm_ftrl_k8", "fm_ftrl_k10", "fm_ftrl_k16", "fm_sgd_k8", "fm_sgd_k10", "fm_sgd_k16"]
CANON_KS = [4, 8, 16, 64, 128]
ABSENT = {"default": api.ABSENT_DEFAULT, "zero": api.ABSENT_ZERO}
_bits = TS._bits
F64 = 2.0 ** -29  # a float32 evaluation bound times this bounds the same evaluation in float64 (u = 2^-53)


def _read(m, path):
    m.save(str(path))
    return open(str(path), "rb").read()


def _rows(m, path):
    """the model's rows as its file holds them (sorted by key)"""
    return H.parse_model_file(_read(m, path))


def _device_predict(m, rp, keys, vals=None):
    """xf_model_predict_device(_values) on a non-default stream"""
    import torch
    dev = torch.device("cuda:0")
    d_rp = torch.from_numpy(rp.astype(np.int32)).to(dev)
    d_keys = torch.from_numpy(keys.view(np.int64)).to(dev)
    d_vals = torch.from_numpy(np.ascontiguousarray(vals, np.float32)).to(dev) if vals is not None else None
    d_out = torch.full((rp.size - 1,), -1.0, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    s = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(s):
        m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), rp.size - 1, keys.size, d_out.data_ptr(), stream=s.cuda_stream,
                         d_vals=d_vals.data_ptr() if d_vals is not None else 0)
    s.synchronize()
    return d_out.cpu().numpy()


def _check_pctr(p, arg, bound, what):
    """pctr within the sigmoid of [arg - bound, arg + bound], widened by the float rounding of the sigmoid"""
    lo, hi = FMM.sigmoid_range(arg - bound, arg + bound)
    slack = 2.0 ** -23 * np.maximum(np.abs(lo), np.abs(hi)) + 1e-30
    p = p.astype(np.float64)
    bad = (p < lo - slack) | (p > hi + slack)
    assert not bad.any(), (what, np.flatnonzero(bad)[:5], p[bad][:5], lo[bad][:5], hi[bad][:5])


def _held_query(seed, keys, lens=(1, 2, 8, 31, 64, 100, 300)):
    """rows over keys the model holds only, so that every token's fields are known"""
    rng = np.random.default_rng(seed)
    lens = np.array(list(lens) * 4)
    rp = np.zeros(lens.size + 1, np.int64)
    rp[1:] = np.cumsum(lens)
    return rp.astype(np.uint32), keys[rng.integers(0, keys.size, int(rp[-1]))]


# ---- 1. FM: contents, predictions, bound -----------------------------------------------------------------------------
@pytest.mark.parametrize("name", FM_NAMES)
@pytest.mark.parametrize("absent", sorted(ABSENT))
@pytest.mark.parametrize("prune", [True, False])
def test_fm_f16_is_the_rounded_f32_model(name, absent, prune, monkeypatch, tmp_path):
    t, tr = TS._make(name, monkeypatch)
    trained = TS._train(t, tr)
    K = TS.TABLES[name][2]
    m32 = t.freeze(absent=ABSENT[absent], prune=prune)
    m16 = m32.convert(F16)
    i32, i16 = m32.info(), m16.info()
    for f in ("keys", "source_keys", "pruned_keys", "capacity", "fm", "latent_dim", "optimizer", "absent"):
        assert i16[f] == i32[f], f
    assert i32["precision"] == F32 and i16["precision"] == F16
    assert i16["row_bytes"] == 16 and i16["bytes"] == i16["capacity"] * 16
    # lookup: the binary16 rounding of the F32 fields
    allk = np.concatenate([np.sort(t.list_keys()), TS._unseen()])
    l32, l16 = m32.lookup(allk), m16.lookup(allk)
    assert np.array_equal(l16["present"], l32["present"]) and np.array_equal(_bits(l16["w"]), _bits(l32["w"]))
    for f in ("st", "qt"):
        assert np.array_equal(_bits(l16[f]), _bits(H.rounded(l32[f]))), f
    # the F32 model with rounded fields, built in numpy and loaded (independent of the convert kernel), and F16 -> F32
    h, rows = _rows(m32, tmp_path / "m32")
    ref_rows = H.convert(H.convert(rows, F16), F32)
    ref_path = str(tmp_path / "ref")
    open(ref_path, "wb").write(H.model_file(ref_rows, 1, K, F32, h["optimizer"], h["absent"], h["v_init"], h["v_const"],
                                            h["seed"], h["source_keys"]))
    ref, back = api.Model.load(ref_path), m16.convert(F32)
    assert _read(back, tmp_path / "back") == open(ref_path, "rb").read()
    rp, keys = TS._query(7, trained)
    want = ref.predict_host(rp, keys)
    for m in (m16, back):
        assert np.array_equal(_bits(m.predict_host(rp, keys)), _bits(want))
        assert np.array_equal(_bits(_device_predict(m, rp, keys)), _bits(want))
    assert len(set(want.tolist())) > 10
    # against the original F32 model: the bound, on rows over held keys
    held = allk[l32["present"].astype(bool)]
    hrp, hkeys = _held_query(3, held)
    lk = m32.lookup(hkeys)
    a32, a16, field, ev = H.fm_bound(hrp, lk["w"], lk["st"], lk["qt"])
    assert np.all(np.abs(a16 - a32) <= field + F64 * ev)
    _check_pctr(m16.predict_host(hrp, hkeys), a32, field + ev, "f16")
    _check_pctr(m32.predict_host(hrp, hkeys), a32, ev, "f32")
    ratio = np.max(np.abs(a16 - a32) / np.maximum(field, 1e-300))
    print("%s %s prune=%s: max |darg| / bound = %.3g, max |darg| = %.3g, max |dpctr| = %.3g" % (
        name, absent, prune, ratio, np.max(np.abs(a16 - a32)),
        np.max(np.abs(m16.predict_host(hrp, hkeys).astype(np.float64) - m32.predict_host(hrp, hkeys)))))
    TP._close(ref, back, m16, m32, tr, t)


@pytest.mark.parametrize("name", ["fm_ftrl_k16", "fm_sgd_k10"])
def test_fm_f16_predict_ingested(name, monkeypatch):
    t, tr = TS._make(name, monkeypatch, max_rows=1 << 12, max_nnz=1 << 18)
    rows, _ = tr.ingest_text(open(TS.TRAIN + "-00000", "rb").read())
    tr.step_ingested(0, rows)
    rows, _ = tr.ingest_text(open(TS.TEST + "-00000", "rb").read())
    m16 = t.freeze().convert(F16)
    back = m16.convert(F32)
    got, lab = m16.predict_ingested(tr, 0, rows)
    want, want_lab = back.predict_ingested(tr, 0, rows)
    assert np.array_equal(_bits(got), _bits(want)) and np.array_equal(lab, want_lab) and len(set(want.tolist())) > 10
    TP._close(back, m16, tr, t)


# ---- 2. canonical ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", CANON_KS)
@pytest.mark.parametrize("absent", sorted(ABSENT))
@pytest.mark.parametrize("prune", [True, False])
def test_canonical_f16_is_the_rounded_f32_model(K, absent, prune, tmp_path):
    t, tr = TC._make(K, api.OPT_FTRL)
    trained = TC._train(t, tr)
    m32 = t.freeze_canonical(absent=ABSENT[absent], prune=prune)
    m16 = m32.convert(F16)
    i32, i16 = m32.info(), m16.info()
    for f in ("keys", "source_keys", "pruned_keys", "capacity", "fm", "latent_dim", "optimizer", "absent"):
        assert i16[f] == i32[f], f
    assert i16["precision"] == F16 and i16["row_bytes"] == H.row_bytes(2, K, F16) == (16 + 2 * K + 31) // 32 * 32
    assert i16["bytes"] == i16["capacity"] * i16["row_bytes"]
    allk = np.concatenate([np.sort(t.list_keys()), TC._unseen()])
    l32, l16 = m32.lookup_latent(allk), m16.lookup_latent(allk)
    assert np.array_equal(l16["present"], l32["present"]) and np.array_equal(_bits(l16["w"]), _bits(l32["w"]))
    assert np.array_equal(_bits(l16["v"]), _bits(H.rounded(l32["v"])))
    h, rows = _rows(m32, tmp_path / "m32")
    ref_rows = H.convert(H.convert(rows, F16), F32)
    ref_path = str(tmp_path / "ref")
    open(ref_path, "wb").write(H.model_file(ref_rows, 2, K, F32, h["optimizer"], h["absent"], h["v_init"], h["v_const"],
                                            h["seed"], h["source_keys"]))
    ref, back = api.Model.load(ref_path), m16.convert(F32)
    assert _read(back, tmp_path / "back") == open(ref_path, "rb").read()
    rp, keys, vals = TC._query(K + 5, trained)
    for v in (None, vals):
        want = ref.predict_host(rp, keys, v)
        for m in (m16, back):
            assert np.array_equal(_bits(m.predict_host(rp, keys, v)), _bits(want))
            assert np.array_equal(_bits(_device_predict(m, rp, keys, v)), _bits(want))
        assert len(set(want.tolist())) > 10
    held = allk[l32["present"].astype(bool)]
    hrp, hkeys = _held_query(4, held)
    x = TC._vals(np.random.default_rng(K), hkeys.size)
    lk = m32.lookup_latent(hkeys)
    a32, a16, field, ev = H.canonical_bound(hrp, x, lk["w"], lk["v"])
    assert np.all(np.abs(a16 - a32) <= field + F64 * ev)
    _check_pctr(m16.predict_host(hrp, hkeys, x), a32, field + ev, "f16")
    _check_pctr(m32.predict_host(hrp, hkeys, x), a32, ev, "f32")
    print("canonical K=%d %s prune=%s: max |darg| / bound = %.3g, max |darg| = %.3g" % (
        K, absent, prune, np.max(np.abs(a16 - a32) / np.maximum(field, 1e-300)), np.max(np.abs(a16 - a32))))
    TP._close(ref, back, m16, m32, tr, t)


# ---- 3. files ----------------------------------------------------------------------------------------------------------
def _fm16(monkeypatch, name="fm_ftrl_k16"):
    t, tr = TS._make(name, monkeypatch)
    TS._train(t, tr)
    return t, tr, t.freeze().convert(F16)


def test_fm_file_round_trip(monkeypatch, tmp_path):
    t, tr, m16 = _fm16(monkeypatch)
    data = _read(m16, tmp_path / "a")
    h, rows = H.parse_model_file(data)
    assert h["precision"] == F16 and struct.unpack_from("<II", data, 56)[1] == 1
    allk = np.sort(t.list_keys())
    lk = m16.lookup(allk)
    have = lk["present"].astype(bool)
    mine = np.zeros(int(have.sum()), H.FM_ROW16)
    mine["key"], mine["w"] = allk[have], lk["w"][have]
    mine["st"], mine["qt"] = H.to_half(lk["st"][have]), H.to_half(lk["qt"][have])
    assert mine.tobytes() == rows.tobytes()
    assert H.model_file(mine, 1, 16, F16, h["optimizer"], h["absent"], h["v_init"], h["v_const"], h["seed"],
                        h["source_keys"]) == data
    back = api.Model.load(str(tmp_path / "a"))
    assert back.info() == m16.info() and back.fingerprint() == m16.fingerprint()
    assert _read(back, tmp_path / "b") == data
    TP._close(back, m16, tr, t)


def _resum(x, header=104):
    x = bytearray(x)
    struct.pack_into("<Q", x, header - 8, SM.section_sum(bytes(x[:header - 8])))
    return bytes(x)


def test_damaged_f16_files_are_refused(monkeypatch, tmp_path):
    t, tr, m16 = _fm16(monkeypatch)
    data = _read(m16, tmp_path / "fm")
    bad = str(tmp_path / "bad")

    def refused(content):
        open(bad, "wb").write(content)
        with pytest.raises(api.XflowError, match=ERR_IO):
            api.Model.load(bad)

    refused(_resum(data[:60] + struct.pack("<I", 2) + data[64:]))  # precision word 2
    refused(_resum(data[:32] + struct.pack("<I", 32) + data[36:88] + struct.pack("<Q", (64 << 20) // 32) + data[96:]))
    m32 = t.freeze()
    d32 = _read(m32, tmp_path / "m32")
    refused(_resum(d32[:60] + struct.pack("<I", 1) + d32[64:]))  # F16 precision with F32 row bytes
    TP._close(m32, m16, tr, t)
    # non-zero padding in an F16 canonical row (K = 16: bytes 48 .. 63), with valid checksums
    ct, ctr = TC._make(16, api.OPT_FTRL)
    TC._train(ct, ctr)
    c16 = ct.freeze_canonical().convert(F16)
    cdata = _read(c16, tmp_path / "c")
    rb = struct.unpack_from("<I", cdata, 32)[0]
    assert rb == 64 and len(cdata) == 104 + 32 + struct.unpack_from("<Q", cdata, 16)[0] * rb
    x = bytearray(cdata)
    x[104 + 32 + 2 * rb + 60] = 1
    struct.pack_into("<Q", x, 104 + 16, SM.section_sum(bytes(x[104 + 32:]), 0))
    open(bad, "wb").write(bytes(x))
    with pytest.raises(api.XflowError, match=ERR_IO + ".*padding"):
        api.Model.load(bad)
    api.Model.load(str(tmp_path / "c")).close()
    TP._close(c16, ctr, ct)


# ---- 4. deltas -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["fm", "canonical"])
def test_f16_delta_chain(kind, monkeypatch, tmp_path):
    if kind == "fm":
        t, tr = TS._make("fm_sgd_k16", monkeypatch)
        step = lambda i: TS._train(t, tr, first=10 * i, n=2)
        freeze = t.freeze
    else:
        t, tr = TC._make(64, api.OPT_FTRL)
        step = lambda i: TC._train(t, tr, first=10 * i, n=2, pull=False)
        freeze = t.freeze_canonical
    step(0)
    models = [freeze().convert(F16)]
    for i in range(1, 4):
        step(i)
        models.append(freeze().convert(F16))
    _read(models[0], tmp_path / "m0")
    cur = api.Model.load(str(tmp_path / "m0"))
    for i in range(1, len(models)):
        d = models[i - 1].diff(models[i])
        info = d.info()
        assert info["precision"] == F16 and info["upserts"] > 0
        d.save(str(tmp_path / ("d%d" % i)))
        raw = open(str(tmp_path / ("d%d" % i)), "rb").read()
        hd = dict(zip(DM.FIELDS, DM.HEADER.unpack(raw[:DM.HEADER.size])))
        assert hd["zero"] == F16 and hd["row_bytes"] == models[i].info()["row_bytes"]
        # the numpy statement of the delta between the two models' rows
        ha, ra = H.parse_model_file(_read(models[i - 1], tmp_path / "a"))
        hb, rb = H.parse_model_file(_read(models[i], tmp_path / "b"))
        assert raw == H.delta_file(ra, rb, hb["source_keys"], hb["fm"], hb["latent_dim"], F16, hb["optimizer"],
                                   hb["absent"], hb["v_init"], hb["v_const"], hb["seed"])
        nxt = cur.apply(api.Delta.load(str(tmp_path / ("d%d" % i))))
        assert _read(nxt, tmp_path / "n") == _read(models[i], tmp_path / "b")
        cur.close()
        cur = nxt
    # mixed precisions: refused, naming precision
    m32 = freeze()
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*precision"):
        m32.diff(models[-1])
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*precision"):
        models[-1].diff(m32)
    d32 = m32.diff(freeze())
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*precision"):
        models[-1].apply(d32)
    TP._close(d32, m32, cur, models, tr, t)


# ---- 5. parts --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["fm_ftrl_k16", "fm_sgd_k10"])
@pytest.mark.parametrize("S", TP.SHARDS)
def test_merge_of_converted_parts_is_the_converted_merge(name, S, tmp_path):
    shards, u = TP._tables(name, S)
    parts = [s.freeze_part() for s in shards]
    parts16 = [p.convert(F16) for p in parts]
    assert [p.part_info() for p in parts16] == [(s, S) for s in range(S)]
    assert all(p.info()["precision"] == F16 for p in parts16)
    merged16 = api.Model.merge(parts16)
    want = api.Model.merge(parts).convert(F16)
    assert _read(merged16, tmp_path / "a") == _read(want, tmp_path / "b")
    assert merged16.info() == want.info() and merged16.fingerprint() == want.fingerprint()
    # a part file carries the precision and loads as a part
    parts16[0].save(str(tmp_path / "p0"))
    back = api.Model.load(str(tmp_path / "p0"))
    assert back.part_info() == (0, S) and back.info()["precision"] == F16
    if S > 1:
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*precision"):
            api.Model.merge([parts[0]] + parts16[1:])
    TP._close(back, want, merged16, parts16, parts, shards, u)


# ---- 6. refusals -----------------------------------------------------------------------------------------------------
def _unchanged(m, path):
    return m.fingerprint(), m.info(), _read(m, path)


def test_refusals_leave_the_source_alone(monkeypatch, tmp_path):
    t, tr = TS._make("lr_ftrl", monkeypatch)
    TS._train(t, tr, n=1)
    lr = t.freeze()
    before = _unchanged(lr, tmp_path / "lr")
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*LR"):
        lr.convert(F16)
    assert _unchanged(lr, tmp_path / "lr") == before
    TP._close(lr, tr, t)
    monkeypatch.delenv("XFLOW_EAGER", raising=False)
    ft = api.Table(latent_dim=16, optimizer=api.OPT_FTRL, seed=3, capacity=1 << 14)
    keys = TS._keys_of(np.arange(1000, 1100))
    ft.import_(keys, w=np.full(keys.size, 0.5, np.float32), v=np.full((keys.size, 16), 100.0, np.float32))
    ok = TS._keys_of(np.arange(2000, 2300))
    ft.import_(ok, w=np.ones(ok.size, np.float32), v=np.full((ok.size, 16), 0.25, np.float32))
    m = ft.freeze()
    assert np.all(m.lookup(keys)["qt"] == np.float32(160000.0))
    before = _unchanged(m, tmp_path / "fm")
    for p in (2, -1):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*precision"):
            m.convert(p)
    smallest = int(np.min(keys))
    with pytest.raises(api.XflowError, match=ERR_STATE + ".* %d latent fields.* %d " % (keys.size, smallest)):
        m.convert(F16)
    assert _unchanged(m, tmp_path / "fm") == before
    same = m.convert(F32)  # the model's own precision: a copy
    assert _unchanged(same, tmp_path / "same")[1:] == before[1:] and same.fingerprint() == before[0]
    TP._close(same, m, ft)


# ---- 7. the CLI ------------------------------------------------------------------------------------------------------
def _cli(tmp, model, **extra):
    os.makedirs(tmp, exist_ok=True)
    env = dict(os.environ, XFLOW_OPTIMIZER="ftrl")
    for k in ("XFLOW_WORLD", "WORLD_SIZE", "XFLOW_EXPORT_MODEL", "XFLOW_EXPORT_DELTAS", "XFLOW_EXPORT_SHARDED_MODEL",
              "XFLOW_EXPORT_PRECISION", "XFLOW_EAGER", "XFLOW_ADMIT", "XFLOW_CHECKPOINT", "XFLOW_RESUME",
              "XFLOW_NEG_SAMPLE", "XFLOW_EVICT_MAX_KEYS", "XFLOW_EVICT_IDLE", "XFLOW_EVICT_EVERY"):
        env.pop(k, None)
    env.update(extra)
    return subprocess.run([TS.EXE, TS.TRAIN, TS.TEST, model, "3"], cwd=tmp, env=env, capture_output=True, text=True,
                          timeout=600)


def _same_run(a, b, tmp_path, da, db):
    assert a.returncode == 0 and b.returncode == 0, a.stdout + a.stderr + b.stdout + b.stderr
    assert a.stdout == b.stdout and "logloss" in a.stdout
    assert open(tmp_path / da / "pred_0_0.txt").read() == open(tmp_path / db / "pred_0_0.txt").read()


def test_cli_exports_f16_models(tmp_path):
    p32, p16 = tmp_path / "out32", tmp_path / "out16"
    os.makedirs(p32)
    os.makedirs(p16)
    a = _cli(str(tmp_path / "a"), "1", XFLOW_EXPORT_MODEL=str(p32 / "m"), XFLOW_EXPORT_DELTAS=str(p32 / "d"))
    b = _cli(str(tmp_path / "b"), "1", XFLOW_EXPORT_MODEL=str(p16 / "m"), XFLOW_EXPORT_DELTAS=str(p16 / "d"),
             XFLOW_EXPORT_PRECISION="f16")
    _same_run(a, b, tmp_path, "a", "b")
    m32 = api.Model.load(str(p32 / "m"))
    assert _read(m32.convert(F16), tmp_path / "conv") == open(p16 / "m", "rb").read()
    # the chain: the F32 run's models rebuilt from its chain, converted and diffed, are the F16 run's files
    first = sorted(f for f in os.listdir(p32) if f.endswith(".xfsm"))
    assert first == sorted(f for f in os.listdir(p16) if f.endswith(".xfsm")) and len(first) == 1
    cur = api.Model.load(str(p32 / first[0]))
    assert _read(cur.convert(F16), tmp_path / "c0") == open(p16 / first[0], "rb").read()
    e = int(first[0].split("-")[1].split(".")[0])
    n = 0
    while os.path.exists(p32 / ("d-%d.xfsd" % (e + 1))):
        e += 1
        nxt = cur.apply(api.Delta.load(str(p32 / ("d-%d.xfsd" % e))))
        d = cur.convert(F16).diff(nxt.convert(F16))
        d.save(str(tmp_path / "dd"))
        assert open(tmp_path / "dd", "rb").read() == open(p16 / ("d-%d.xfsd" % e), "rb").read()
        cur = nxt
        n += 1
    assert n >= 1


def test_cli_exports_f16_sharded_model(tmp_path):
    a = _cli(str(tmp_path / "a"), "1", XFLOW_EXPORT_SHARDED_MODEL=str(tmp_path / "m32"))
    b = _cli(str(tmp_path / "b"), "1", XFLOW_EXPORT_SHARDED_MODEL=str(tmp_path / "m16"), XFLOW_EXPORT_PRECISION="f16")
    _same_run(a, b, tmp_path, "a", "b")
    m32 = api.Model.load(str(tmp_path / "m32"))
    assert _read(m32.convert(F16), tmp_path / "conv") == open(tmp_path / "m16", "rb").read()
    assert not [f for f in os.listdir(tmp_path) if f.endswith(".xfsp")]


def test_cli_refuses_f16_for_lr_and_a_malformed_value(tmp_path):
    for model, value in (("0", "f16"), ("1", "half"), ("0", "F16")):
        r = _cli(str(tmp_path / ("w" + model + value)), model, XFLOW_EXPORT_PRECISION=value,
                 XFLOW_EXPORT_MODEL=str(tmp_path / "m"))
        assert r.returncode != 0 and "XFLOW_EXPORT_PRECISION" in r.stdout + r.stderr, r.stdout + r.stderr
        assert "logloss" not in r.stdout and not os.path.exists(tmp_path / "m")
    ok = _cli(str(tmp_path / "ok"), "0", XFLOW_EXPORT_PRECISION="f32")
    assert ok.returncode == 0, ok.stdout + ok.stderr

"""GPU parity on key layouts chosen to drive the device table's rare placement paths (pytest -m gpu).

Uniform keys at load <= 0.5 almost never leave their home bucket, wrap past the last slot, build long chains or race
for one free slot.  The keys here are built (placement_model.py) to do all of that on purpose: clusters homed in the
last bucket (their chains wrap to slot 0 and stay clustered through every growth), clusters homed in bucket 0 that
the wrapped chains run into, single chains of 1000 keys with one probe sequence, and clusters among hashed ordinary
keys.  The oracle's table does not depend on placement, so every result must match it as on ordinary keys:

  A. training steps (lazy LR, eager LR, FM) from a capacity that has to grow twice, LR at every bucket size;
  B. Pull / Push / import / export / list_keys / save-load, with absent keys of the same chains interleaved;
  C. canonical FM and the multi-view machine;
  D. eviction sweeps and Bloom admission;
  E. probe overflow: a chain of XF_MAX_PROBE = 8192 keys fits, one more key is XF_ERR_FULL, and the error is sticky;
  F. the reserved key 2^64 - 1 (the empty-slot marker) is refused by every entry point that takes host keys;
  G. the sharded step on 2 GPUs (skips on one)."""
import os

import numpy as np
import pytest

import placement_model as P
from admission_model import AdmittingTable
from common import MVM64, CanonicalFM64, assert_close, assert_close_noise_aware, bits_equal
from eviction_model import EvictingTable
from oracle import oracle as O
from xflow_b200 import api

pytestmark = pytest.mark.gpu

EMPTY = np.uint64(P.EMPTY_KEY)
ERR_ARG, ERR_FULL = -1, -3
LAYOUTS = ["tail", "tail_head", "one_chain", "mixed"]
FAR = 100000  # builder numbers of keys that no layout uses


def _opt(name):
    return (api.OPT_FTRL, O.OPT_FTRL) if name == "ftrl" else (api.OPT_SGD, O.OPT_SGD)


def _ordinary(n, first):
    return api.hash_decimal_ids(np.arange(first, first + n, dtype=np.uint64))


def layout(name):
    """The keys a test trains on."""
    if name == "tail":
        return P.tail(1500)                                   # start slots 0..3: wrap, mixed in-bucket starts
    if name == "tail_head":
        return np.concatenate([P.tail(900), P.head(600)])     # the wrapped chain runs into the cluster at slot 0
    if name == "one_chain":
        return P.one_chain(1000)                              # one probe sequence for all
    if name == "mixed":
        return np.concatenate([P.tail(700), _ordinary(1500, 7000)])
    raise ValueError(name)


def absent(name, n=120):
    """Keys of the same clusters (same chains) that no step or pull ever inserts."""
    if name == "tail":
        return P.tail(n, start=FAR)
    if name == "tail_head":
        return np.concatenate([P.tail(n // 2, start=FAR), P.head(n // 2, start=FAR)])
    if name == "one_chain":
        return P.one_chain(n, start=FAR)
    return np.concatenate([P.tail(n // 2, start=FAR), _ordinary(n // 2, 90000)])


def _csr(rows):
    rp = np.zeros(len(rows) + 1, np.uint32)
    rp[1:] = np.cumsum([len(r) for r in rows])
    return rp, np.concatenate([np.asarray(r, np.uint64) for r in rows])


def batches(keys, seed, long_lens=(129, 150, 200, 257, 300)):
    """Four batches over `keys` (shuffled): most keys are new in the first, the pool grows step by step, rows repeat
    keys, and the third batch holds rows of 129+ tokens (phase B's re-probe) with a key in chunk 1 and again in chunk 3.
    Token counts grow so that a table created at 1024 slots grows while the clusters are in it."""
    rng = np.random.default_rng(seed)
    u = rng.permutation(keys)
    out = []
    for step, (frac, B, dmax) in enumerate([(0.6, 160, 16), (0.8, 256, 20), (0.9, 96, 16), (1.0, 384, 24)]):
        pool = u[: int(frac * u.size)]
        rows = []
        for r in range(B):
            row = rng.choice(pool, int(rng.integers(1, dmax + 1)))
            if row.size >= 3 and r % 3 == 0:
                row[-1] = row[0]
            rows.append(row)
        if step == 2:
            for n in list(long_lens) * 2:
                row = rng.choice(pool, n)
                row[n - 1] = row[3]
                if n > 130:
                    row[130] = row[3]
                rows.append(row)
        order = rng.permutation(len(rows))
        rp, k = _csr([rows[i] for i in order])
        out.append((rp, k, rng.integers(0, 2, len(rows)).astype(np.uint8)))
    return out


def _raises(code, what=None):
    pat = "error %d:" % code + (".*" + what if what else "")
    return pytest.raises(api.XflowError, match=pat)


# ---------------------------------------------------------------------------------------------------------------------
# A. training steps against the oracle
# ---------------------------------------------------------------------------------------------------------------------
MODELS = {  # name: (model, K, optimizer, eager LR)
    "lr_ftrl": (api.MODEL_LR, 0, "ftrl", False),
    "lr_sgd": (api.MODEL_LR, 0, "sgd", False),
    "lr_ftrl_eager": (api.MODEL_LR, 0, "ftrl", True),
    "fm4_sgd": (api.MODEL_FM, 4, "sgd", False),      # 64-byte rows: buckets of 2, the eager step's first look via L1
    "fm16_ftrl": (api.MODEL_FM, 16, "ftrl", False),  # 256-byte rows: plain linear probing
}
BUCKETS = ["default", "0", "3", "4"]  # XFLOW_BUCKET_LOG2
STEP_CASES = [(lay, m, b) for lay in LAYOUTS for m in MODELS for b in (BUCKETS if MODELS[m][1] == 0 else ["default"])]


def _long_lens(K, opt):
    # FM rows over 128 tokens run with SGD only and stop at 200 (test_gpu_edges.py, section C, says why)
    if K:
        return (129, 160, 200) if opt == "sgd" else ()
    return (129, 150, 200, 257, 300)


def _make(model, monkeypatch, bucket="default", capacity=1024, seed=21):
    gm, K, opt, eager = MODELS[model]
    gopt, oopt = _opt(opt)
    if bucket != "default":
        monkeypatch.setenv("XFLOW_BUCKET_LOG2", bucket)  # for the table's whole life: every growth reads it again
    if eager:
        monkeypatch.setenv("XFLOW_EAGER", "1")
    gt = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=seed, capacity=capacity)
    monkeypatch.delenv("XFLOW_EAGER", raising=False)
    mk = dict(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=seed)
    return gt, gm, K, opt, mk


@pytest.mark.parametrize("lay,model,bucket", STEP_CASES, ids=["-".join(c) for c in STEP_CASES])
def test_clustered_steps_match_oracle(lay, model, bucket, monkeypatch):
    gt, gm, K, opt, mk = _make(model, monkeypatch, bucket)
    ot, xt = O.Table(**mk), O.Table(**mk)
    keys = layout(lay)
    gone = absent(lay)
    bs = batches(keys, 5, _long_lens(K, opt))
    # keys already in the table when it first grows: the rehash has to move the clusters
    pre = np.unique(np.random.default_rng(1).permutation(keys)[:300])
    if K:
        for t in (gt, ot, xt):
            t.pull(pre)
    else:
        w0 = (np.random.default_rng(2).standard_normal(pre.size) * 0.1).astype(np.float32)
        for t in (gt, ot, xt):
            t.import_(pre, w=w0)
    tr = api.Trainer(gt, model=gm, max_rows=max(b[2].size for b in bs), max_nnz=max(b[1].size for b in bs),
                     keep_loss=True)
    fields = ("w", "nw", "zw") + (("v", "nv", "zv") if K else ())
    seen, unique_total = [pre, gone], 0
    for step, (rp, k, lab) in enumerate(bs):
        B = lab.size
        tr.step_host(rp, k, lab)
        _, ol = ot.step(rp.astype(np.int64), k, lab.astype(np.int32))
        with O.exact_sums():
            _, xl = xt.step(rp.astype(np.int64), k, lab.astype(np.int32))
        what = "%s step %d" % (model, step)
        assert_close_noise_aware(tr.get_loss(B), ol, xl, "residuals " + what, abs_floor=1e-6, max_noisy_frac=0.02)
        seen.append(k)
        uk = np.unique(np.concatenate(seen))
        ge, oe, xe = gt.export(uk), ot.export(uk), xt.export(uk)
        assert np.array_equal(ge["present"], oe["present"]), what
        assert not ge["present"][np.isin(uk, gone)].any(), what
        for f in fields:
            assert_close_noise_aware(ge[f], oe[f], xe[f], "%s %s" % (f, what), max_noisy_frac=0.01)
        assert gt.size() == ot.size(), what
        assert gt.size() * 4 <= gt.capacity() * 3, what
        if not K:
            unique_total += np.unique(k).size
            assert tr.stats()["unique_keys"] == unique_total, what
    assert gt.capacity() >= 4096  # grew at least twice from 1024 slots
    # predict over trained keys and absent keys of the same chains (insert-on-pull on both sides)
    rng = np.random.default_rng(9)
    prows = [rng.choice(np.concatenate([keys, gone]), int(rng.integers(1, 20))) for _ in range(128)]
    prp, pk = _csr(prows)
    gp = tr.predict_host(prp, pk)
    op, xp = ot.predict(prp.astype(np.int64), pk), xt.predict(prp.astype(np.int64), pk)
    assert_close_noise_aware(gp, op, xp, "pctr", abs_floor=1e-6, max_noisy_frac=0.02)
    uk = np.unique(np.concatenate(seen + [pk]))
    assert np.array_equal(gt.export(uk)["present"], ot.export(uk)["present"])
    assert gt.size() == ot.size()
    tr.sync()


# ---------------------------------------------------------------------------------------------------------------------
# B. Pull / Push / import / export / list_keys / save-load
# ---------------------------------------------------------------------------------------------------------------------
KV_CASES = [(0, "ftrl"), (0, "sgd"), (4, "sgd"), (16, "ftrl")]


@pytest.mark.parametrize("K,opt", KV_CASES, ids=["k%d_%s" % c for c in KV_CASES])
@pytest.mark.parametrize("lay", LAYOUTS)
def test_clustered_kv_round_trip_bit_exact(lay, K, opt, tmp_path):
    gopt, oopt = _opt(opt)
    gt = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=3, capacity=1024)
    ot = O.Table(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=3)
    keys, gone = layout(lay), absent(lay)
    rng = np.random.default_rng(K + 7)
    inserted = []
    for it in range(4):
        sub = np.unique(rng.choice(keys, int(0.35 * keys.size)))
        order = rng.permutation(sub.size)  # pulls take any order
        gw, gv = gt.pull(sub[order])
        ow, ov = ot.pull(sub[order])
        assert bits_equal(gw, ow), "pull w %d" % it
        if K:
            assert bits_equal(gv, ov), "pull v %d" % it
        g1 = (rng.standard_normal(sub.size) * 0.1).astype(np.float32)
        g1[::7] = 0.0
        g2 = (rng.standard_normal((sub.size, K)) * 0.1).astype(np.float32) if K else None
        gt.push(sub, g1, g2)
        ot.push(sub, g1, g2)
        inserted.append(sub)
    # import over trained and new keys
    imp = np.unique(rng.choice(keys, 300))
    vals = dict(w=(rng.standard_normal(imp.size) * 0.2).astype(np.float32))
    if opt == "ftrl":
        vals.update(nw=np.abs(rng.standard_normal(imp.size)).astype(np.float32),
                    zw=(rng.standard_normal(imp.size) * 0.1).astype(np.float32))
    if K:
        vals["v"] = (rng.standard_normal((imp.size, K)) * 0.1).astype(np.float32)
        if opt == "ftrl":
            vals.update(nv=np.abs(rng.standard_normal((imp.size, K))).astype(np.float32),
                        zv=(rng.standard_normal((imp.size, K)) * 0.1).astype(np.float32))
    gt.import_(imp, **vals)
    ot.import_(imp, **vals)
    inserted.append(imp)
    expect = np.unique(np.concatenate(inserted))
    # export with absent keys of the same chains interleaved: each walks its whole chain and must come back absent
    probe = np.concatenate([keys, gone])[rng.permutation(keys.size + gone.size)]
    e, o = gt.export(probe), ot.export(probe)
    assert np.array_equal(e["present"], o["present"])
    assert not e["present"][np.isin(probe, gone)].any()
    assert int(e["present"].sum()) == expect.size
    names = ("w", "nw", "zw") + (("v", "nv", "zv") if K else ())
    for f in names:
        assert bits_equal(e[f], o[f]), f
    assert gt.size() == ot.size() == expect.size
    assert np.array_equal(np.sort(gt.list_keys()), expect)
    # save / load into a fresh table that grows while loading
    path = str(tmp_path / "clustered.ckpt")
    gt.save(path)
    g2 = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_ZERO, seed=99, capacity=1024)
    g2.load(path)
    e2 = g2.export(probe)
    for f in names + ("present",):
        assert np.array_equal(e[f], e2[f]), f
    assert g2.size() == expect.size
    gt.sync()


# ---------------------------------------------------------------------------------------------------------------------
# C. canonical FM and the multi-view machine
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lay", LAYOUTS)
def test_clustered_canonical_fm_matches_float64_model(lay):
    K = 8
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=4, canonical_fm=1, capacity=1024)
    bs = batches(layout(lay), 13, ())
    tr = api.Trainer(t, model=api.MODEL_FM_CANONICAL, max_rows=max(b[2].size for b in bs),
                     max_nnz=max(b[1].size for b in bs), keep_loss=True)
    model = CanonicalFM64(K, "ftrl", t.pull)
    rng = np.random.default_rng(31)
    for step, (rp, keys, lab) in enumerate(bs):
        x = (rng.random(keys.size) * 1.5 + 0.25).astype(np.float32)
        x[::7] *= -1.0
        loss = model.step(rp, keys, x, lab)
        tr.step_host_values(rp, keys, x, lab)
        assert_close(tr.get_loss(lab.size), loss, "canonical FM residuals, step %d" % step, rel=2e-5, abs_floor=2e-6)
    allk = model.keys()
    e, ref = t.export(allk), model.export(allk)
    assert e["present"].all() and t.size() == allk.size
    assert not t.export(absent(lay))["present"].any()
    for f in ("w", "v", "nw", "zw", "nv", "zv"):
        assert_close(e[f].reshape(allk.size, -1), ref[f], "canonical FM %s" % f, rel=2e-4, abs_floor=2e-7)


@pytest.mark.parametrize("lay", LAYOUTS)
def test_clustered_mvm_matches_float64_model(lay):
    K, F = 8, 5
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=4, canonical_fm=1, capacity=1024)
    bs = batches(layout(lay), 17, ())
    tr = api.Trainer(t, model=api.MODEL_MVM, max_rows=max(b[2].size for b in bs), max_nnz=max(b[1].size for b in bs),
                     keep_loss=True)
    rng = np.random.default_rng(41)
    allk = np.unique(np.concatenate([b[1] for b in bs]))
    V0 = rng.normal(0.0, 0.3, (allk.size, K)).astype(np.float32)
    half = allk.size // 2  # two imports: the second grows the table with the first half's clusters in it
    t.import_(allk[:half], v=V0[:half])
    t.import_(allk[half:], v=V0[half:])
    model = MVM64(V0, "ftrl", 0.0)
    for step, (rp, keys, lab) in enumerate(bs):
        fields = rng.integers(0, F, keys.size).astype(np.uint8)
        x = (rng.random(keys.size) * 1.5 + 0.25).astype(np.float32)
        loss = model.step(np.searchsorted(allk, keys), rp, fields, x, lab)
        tr.step_host_fields(rp, keys, fields, x, lab)
        assert_close(tr.get_loss(lab.size), loss, "MVM residuals, step %d" % step, rel=5e-5, abs_floor=5e-6)
    e = t.export(allk)
    assert e["present"].all() and t.size() == allk.size
    for name, ref in (("v", model.V), ("nv", model.NV), ("zv", model.ZV)):
        assert_close(e[name].reshape(allk.size, -1), ref, "MVM %s" % name, rel=5e-4, abs_floor=5e-7)


# ---------------------------------------------------------------------------------------------------------------------
# D. eviction and admission
# ---------------------------------------------------------------------------------------------------------------------
EVICT_CASES = {"lr_ftrl": dict(max_keys=600), "fm4_sgd": dict(max_idle_batches=1, max_keys=700)}


@pytest.mark.parametrize("model", sorted(EVICT_CASES))
@pytest.mark.parametrize("lay", LAYOUTS)
def test_clustered_eviction_matches_model(lay, model, monkeypatch):
    gt, gm, K, opt, mk = _make(model, monkeypatch, seed=11)
    ot, xt = EvictingTable(**mk), EvictingTable(**mk)
    for t in (gt, ot, xt):
        t.set_eviction(**EVICT_CASES[model])
    bs = batches(layout(lay), 23, _long_lens(K, opt))
    tr = api.Trainer(gt, model=gm, max_rows=max(b[2].size for b in bs), max_nnz=max(b[1].size for b in bs),
                     keep_loss=True)
    fields = ("w", "nw", "zw") + (("v", "nv", "zv") if K else ())
    seen, evicted = [absent(lay)], 0
    for step, (rp, k, lab) in enumerate(bs):
        tr.step_host(rp, k, lab)
        _, ol = ot.step(rp.astype(np.int64), k, lab.astype(np.int32))
        with O.exact_sums():
            _, xl = xt.step(rp.astype(np.int64), k, lab.astype(np.int32))
        assert_close_noise_aware(tr.get_loss(lab.size), ol, xl, "residuals step %d" % step, abs_floor=1e-6,
                                 max_noisy_frac=0.02)
        seen.append(k)
        uk = np.unique(np.concatenate(seen))
        for phase in ("step", "sweep"):
            if phase == "sweep":
                n = gt.evict()
                assert n == ot.evict(), "evicted after step %d" % step
                xt.evict()
                evicted += n
            what = "%s %d" % (phase, step)
            ge, oe, xe = gt.export(uk), ot.export(uk), xt.export(uk)
            assert np.array_equal(ge["present"], oe["present"]), what
            assert gt.size() == ot.size(), what
            assert np.array_equal(gt.last_touch(uk), ot.last_touch(uk)), what
            for f in fields:
                assert_close_noise_aware(ge[f], oe[f], xe[f], "%s %s" % (f, what), max_noisy_frac=0.01)
    assert evicted > 0
    tr.sync()


@pytest.mark.parametrize("lay", LAYOUTS)
def test_clustered_bloom_admission_matches_model(lay):
    pol = dict(mode=api.ADMIT_BLOOM, threshold=2, log2_cells=12, hashes=3, seed=7)
    gt = api.Table(optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=11, capacity=1024)
    ot = AdmittingTable(K=0, opt=O.OPT_FTRL, init_mode=O.INIT_COUNTER, seed=11)
    xt = AdmittingTable(K=0, opt=O.OPT_FTRL, init_mode=O.INIT_COUNTER, seed=11)
    for t in (gt, ot, xt):
        t.set_admission(**pol)
    bs = batches(layout(lay), 29) * 2
    tr = api.Trainer(gt, max_rows=max(b[2].size for b in bs), max_nnz=max(b[1].size for b in bs), keep_loss=True)
    seen = [absent(lay)]
    for step, (rp, k, lab) in enumerate(bs):
        tr.step_host(rp, k, lab)
        _, ol = ot.step(rp.astype(np.int64), k, lab.astype(np.int32))
        with O.exact_sums():
            _, xl = xt.step(rp.astype(np.int64), k, lab.astype(np.int32))
        assert_close_noise_aware(tr.get_loss(lab.size), ol, xl, "residuals step %d" % step, abs_floor=1e-6,
                                 max_noisy_frac=0.02)
        seen.append(k)
        uk = np.unique(np.concatenate(seen))
        ge, oe, xe = gt.export(uk), ot.export(uk), xt.export(uk)
        assert np.array_equal(ge["present"], oe["present"]), step
        assert gt.size() == ot.size(), step
        assert gt.admission_stats() == ot.admission_stats(), step
        for f in ("w", "nw", "zw"):
            assert_close_noise_aware(ge[f], oe[f], xe[f], "%s step %d" % (f, step), max_noisy_frac=0.01)
    assert gt.admission_stats()["rejected_tokens"] > 0
    tr.sync()


# ---------------------------------------------------------------------------------------------------------------------
# E. probe overflow
# ---------------------------------------------------------------------------------------------------------------------
MAX_PROBE = 8192


def test_chain_of_max_probe_keys_fits():
    """8192 keys with one probe sequence: the last one inserted sits at probe depth 8191, the deepest a probe looks.
    This is also the device's check of placement_model: if its restatement of the hash were wrong, the keys would
    spread out and the next test would see no overflow."""
    keys = P.one_chain(MAX_PROBE)
    rng = np.random.default_rng(8)
    w = (rng.standard_normal(keys.size) * 0.1).astype(np.float32)
    nw = np.abs(rng.standard_normal(keys.size)).astype(np.float32)
    zw = (rng.standard_normal(keys.size) * 0.1).astype(np.float32)
    t = api.Table(optimizer=api.OPT_FTRL, capacity=1024)
    t.import_(keys, w=w, nw=nw, zw=zw)
    e = t.export(keys[rng.permutation(keys.size)])
    order = np.argsort(e["keys"])
    ref = np.argsort(keys)
    assert e["present"].all() and t.size() == MAX_PROBE
    for f, a in (("w", w), ("nw", nw), ("zw", zw)):
        assert bits_equal(e[f][order], a[ref]), f
    t.sync()


def _overflow_batch(keys):
    rp = np.arange(0, keys.size + 63, 64, dtype=np.uint32)
    rp[-1] = keys.size
    return rp, keys, (np.arange(rp.size - 1) & 1).astype(np.uint8)


@pytest.mark.parametrize("path", ["import", "push", "pull", "lazy_lr_step", "eager_fm_step", "export_absent"])
def test_chain_past_max_probe_is_table_full_and_sticky(path):
    """One key more than XF_MAX_PROBE on one probe sequence overflows at ANY capacity (the table is nowhere near its
    load limit): the call reports XF_ERR_FULL, and the error is sticky, so every later call on the table fails too.
    A training step reports it at the next synchronising call (xf_trainer_sync or any table call)."""
    keys = P.one_chain(MAX_PROBE + 1)
    msg = "probe sequence overflowed"
    K = 4 if path == "eager_fm_step" else 0
    t = api.Table(latent_dim=K, optimizer=api.OPT_SGD if K else api.OPT_FTRL, capacity=1024)
    if path == "import":
        with _raises(ERR_FULL, msg):
            t.import_(keys, w=np.ones(keys.size, np.float32))
    elif path == "push":
        with _raises(ERR_FULL, msg):
            t.push(keys, gw=np.ones(keys.size, np.float32))
    elif path == "pull":
        with _raises(ERR_FULL, msg):
            t.pull(keys)
    elif path == "export_absent":
        t.import_(keys[:MAX_PROBE], w=np.ones(MAX_PROBE, np.float32))  # full chain: fits
        with _raises(ERR_FULL, msg):
            t.export(keys[MAX_PROBE:])  # an absent key of that chain looks at 8192 occupied slots
    else:
        tr = api.Trainer(t, model=api.MODEL_FM if K else api.MODEL_LR, max_rows=256, max_nnz=keys.size)
        rp, k, lab = _overflow_batch(keys)
        tr.step_host(rp, k, lab)
        with _raises(ERR_FULL, msg):
            tr.sync()
    assert t.capacity() <= 1 << 15  # not a capacity problem
    with _raises(ERR_FULL, msg):
        t.pull(np.array([12345], np.uint64))
    with _raises(ERR_FULL, msg):
        t.sync()


# ---------------------------------------------------------------------------------------------------------------------
# F. the reserved key 2^64 - 1
# ---------------------------------------------------------------------------------------------------------------------
RESERVED_MODELS = {"lr_lazy": (0, False), "lr_eager": (0, True), "fm4": (4, False)}


def _table(name, monkeypatch, **kw):
    K, eager = RESERVED_MODELS[name]
    if eager:
        monkeypatch.setenv("XFLOW_EAGER", "1")
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, capacity=1024, **kw)
    monkeypatch.delenv("XFLOW_EAGER", raising=False)
    return t, K


@pytest.mark.parametrize("name", sorted(RESERVED_MODELS))
def test_reserved_key_push_leaves_its_twin_alone(name, monkeypatch):
    """2^64 - 1 marks an empty slot.  A push of it used to "find" the first free slot of its chain and write its
    state there without claiming the slot; the next key to land there (the twin, same probe sequence) then carried
    that state.  The push is refused, and the twin starts from the default contents."""
    t, K = _table(name, monkeypatch)
    twin = np.array([P.twin_of_empty()], np.uint64)
    with _raises(ERR_ARG, "18446744073709551615"):
        t.push(np.array([EMPTY]), gw=np.ones(1, np.float32), gv=np.ones((1, K), np.float32) if K else None)
    w, _ = t.pull(twin)
    e = t.export(twin)
    assert e["present"].all() and t.size() == 1
    assert w[0] == 0 and e["w"][0] == 0 and e["nw"][0] == 0 and e["zw"][0] == 0
    if K:
        assert not e["nv"].any() and not e["zv"].any()
    t.push(twin, gw=np.full(1, 0.5, np.float32))  # the twin trains normally
    t.sync()


@pytest.mark.parametrize("name", sorted(RESERVED_MODELS))
def test_reserved_key_export_on_empty_table(name, monkeypatch):
    """Export of 2^64 - 1 used to report it present on a table that never saw it; it is refused."""
    t, _ = _table(name, monkeypatch)
    with _raises(ERR_ARG, "18446744073709551615"):
        t.export(np.array([EMPTY]))
    assert t.size() == 0


def test_reserved_key_refused_by_every_host_entry_point():
    """Every entry point that takes keys from host memory refuses a batch holding 2^64 - 1 with XF_ERR_ARG before
    anything is enqueued: nothing is inserted, no step is counted, and the table and trainer go on working."""
    ok = P.tail(5)
    keys = np.concatenate([ok[:2], [EMPTY], ok[2:]]).astype(np.uint64)
    rp = np.array([0, 3, keys.size], np.uint32)
    lab = np.array([1, 0], np.uint8)
    n = keys.size
    t = api.Table(optimizer=api.OPT_FTRL, capacity=1024)
    t.set_eviction()
    tr = api.Trainer(t, max_rows=8, max_nnz=64, keep_loss=True)
    calls = {
        "pull": lambda: t.pull(keys),
        "push": lambda: t.push(keys, gw=np.ones(n, np.float32)),
        "import": lambda: t.import_(keys, w=np.ones(n, np.float32)),
        "export": lambda: t.export(keys),
        "last_touch": lambda: t.last_touch(keys),
        "step_host": lambda: tr.step_host(rp, keys, lab),
        "predict_host": lambda: tr.predict_host(rp, keys),
    }
    ct = api.Table(latent_dim=8, optimizer=api.OPT_FTRL, canonical_fm=1, capacity=1024)
    cf = api.Trainer(ct, model=api.MODEL_FM_CANONICAL, max_rows=8, max_nnz=64, keep_loss=True)
    mt = api.Table(latent_dim=8, optimizer=api.OPT_FTRL, canonical_fm=1, capacity=1024)
    mv = api.Trainer(mt, model=api.MODEL_MVM, max_rows=8, max_nnz=64, keep_loss=True)
    x = np.ones(n, np.float32)
    fields = (np.arange(n) % 3).astype(np.uint8)
    calls.update({
        "step_host_values": lambda: cf.step_host_values(rp, keys, x, lab),
        "predict_host_values": lambda: cf.predict_host_values(rp, keys, x),
        "step_host_fields": lambda: mv.step_host_fields(rp, keys, fields, x, lab),
        "predict_host_fields": lambda: mv.predict_host_fields(rp, keys, fields, x),
    })
    for name, call in calls.items():
        with _raises(ERR_ARG, "18446744073709551615"):
            call()
    for table in (t, ct, mt):
        assert table.size() == 0
    for trainer in (tr, cf, mv):
        assert trainer.stats()["steps"] == 0
    # nothing is left behind: the same batches without the reserved key work
    good = np.delete(keys, 2)
    grp = np.array([0, 2, good.size], np.uint32)
    tr.step_host(grp, good, lab)
    cf.step_host_values(grp, good, x[:-1], lab)
    mv.step_host_fields(grp, good, fields[:-1], x[:-1], lab)
    assert t.size() == ct.size() == mt.size() == good.size
    for trainer in (tr, cf, mv):
        trainer.sync()


# ---------------------------------------------------------------------------------------------------------------------
# G. the sharded step on 2 GPUs
# ---------------------------------------------------------------------------------------------------------------------
def _mg_batches(rank):
    return batches(layout("tail_head"), 60 + rank, (129, 150, 200))


def _mg_worker(rank, world, id_path, ret):
    from xflow_b200 import api as A
    if rank == 0:
        cid = A.Comm.new_id()
        np.save(id_path + ".tmp.npy", cid)
        os.replace(id_path + ".tmp.npy", id_path)
    else:
        import time
        while not os.path.exists(id_path):
            time.sleep(0.05)
        cid = np.load(id_path)
    comm = A.Comm(cid, rank, world, rank)
    table = A.Table(optimizer=A.OPT_FTRL, device=rank, shard_index=rank, num_shards=world, capacity=1024)
    bs = _mg_batches(rank)
    tr = A.Trainer(table, max_rows=512, max_nnz=16384, keep_loss=True, comm=comm)
    losses = []
    for rp, keys, lab in bs:
        tr.step_host(rp, keys, lab)
        losses.append(tr.get_loss(lab.size))
    tr.sync()
    comm.barrier()
    allk = np.concatenate([layout("tail_head"), absent("tail_head")])
    mine = np.array([A.shard_of(int(k), world) == rank for k in allk])
    ret[rank] = dict(keys=allk[mine], e=table.export(allk[mine]), losses=losses, size=table.size())
    comm.barrier()
    tr.close()
    table.close()
    comm.close()


def test_sharded_clustered_steps_match_oracle(tmp_path):
    world = 2
    if api.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_mg_worker, args=(world, str(tmp_path / "ncclid.npy"), ret), nprocs=world, join=True)
    t = O.Table(K=0, opt=O.OPT_FTRL)
    per_rank = [_mg_batches(r) for r in range(world)]
    losses = {r: [] for r in range(world)}
    for step in range(len(per_rank[0])):
        pend = []
        for r in range(world):
            rp, keys, lab = per_rank[r][step]
            uk, gw, _, loss = t.worker_compute(rp.astype(np.int64), keys, lab.astype(np.int32))
            pend.append((uk, gw))
            losses[r].append(loss)
        for uk, gw in pend:
            t.push(uk, gw)
    total = 0
    for r in range(world):
        got = ret[r]
        for a, b in zip(got["losses"], losses[r]):
            assert_close(a, b, "loss rank %d" % r, abs_floor=1e-6)
        ref = t.export(got["keys"])
        assert np.array_equal(got["e"]["present"], ref["present"]), r
        for f in ("w", "nw", "zw"):
            assert_close(got["e"][f], ref[f], "rank %d %s" % (r, f))
        total += got["size"]
    assert total == t.size()

"""Exact training-state checkpoints (xf_table_save_state / xf_table_load_state): a run resumed from an image, and a run
that saved one and went on, both equal the run that never saved, bit for bit; the image is deterministic; damaged
files, mismatched tables and occupied tables are refused and leave the target as it was."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

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
    "fm_sgd_k8": (api.MODEL_FM, api.OPT_SGD, 8, False),
    "fm_ftrl_k16": (api.MODEL_FM, api.OPT_FTRL, 16, False),
    "fmc_ftrl_k8": (api.MODEL_FM_CANONICAL, api.OPT_FTRL, 8, False),
    "mvm_ftrl_k8": (api.MODEL_MVM, api.OPT_FTRL, 8, False),
}
POLICIES = ["none", "bloom", "poisson", "evict", "weights"]
CANONICAL = (api.MODEL_FM_CANONICAL, api.MODEL_MVM)
B, D, SPACE, N = 512, 8, 20000, 5  # rows and tokens per row of a batch, id space, batches before the save
CAP = 1 << 15                      # the tables stay below load 0.5: no growth after the save point


def _batch(seed, canonical):
    """A Zipf batch: row_ptr, keys, labels, values, fields, row weights.  The canonical FM and the MVM add a batch's
    contributions to a key with float atomics, whose order is free: there every key occurs once per batch, so that
    two runs of the same batches are comparable bit for bit at all."""
    rng = np.random.default_rng(seed)
    if canonical:
        _, ids, _ = datagen.make_ids(seed, B * 4, D, SPACE, dist="zipf")
        ids = ids[np.sort(np.unique(ids, return_index=True)[1])]
        ids = np.concatenate([ids, np.setdiff1d(np.arange(SPACE, 3 * SPACE, dtype=ids.dtype), ids)])[:B * D]
    else:
        _, ids, _ = datagen.make_ids(seed, B, D, SPACE, dist="zipf")
    keys = api.hash_decimal_ids(np.asarray(ids, np.uint64))
    rp = np.arange(B + 1, dtype=np.uint32) * D
    lab = (rng.random(B) < 0.3).astype(np.uint8)
    vals = rng.uniform(0.5, 1.5, B * D).astype(np.float32)
    fields = (np.arange(B * D) % 3).astype(np.uint8)
    w = rng.uniform(0.0, 2.0, B).astype(np.float32)
    return rp, keys, lab, vals, fields, w


def _make(name, policy, monkeypatch, capacity=CAP):
    model, opt, K, eager = TABLES[name]
    if eager:
        monkeypatch.setenv("XFLOW_EAGER", "1")
    else:
        monkeypatch.delenv("XFLOW_EAGER", raising=False)
    t = api.Table(latent_dim=K, optimizer=opt, v_init=api.VINIT_COUNTER, seed=11, capacity=capacity,
                  canonical_fm=1 if model in CANONICAL else 0)
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * D, keep_loss=True)
    if policy == "weights":
        tr.set_negative_sampling(0.25, seed=3)
    return t, tr


def _policies(t, policy):
    if policy == "bloom":
        t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=12, hashes=3, decay_batches=3, seed=5)
    elif policy == "poisson":
        t.set_admission(api.ADMIT_POISSON, probability=0.5, seed=5)
    elif policy == "evict":
        t.set_eviction(max_idle_batches=3, max_keys=1500)


def _step(t, tr, name, policy, i):
    """Training batch i; returns (mean_abs_loss, residuals).  Eviction: a sweep after every second batch."""
    model = TABLES[name][0]
    rp, keys, lab, vals, fields, w = _batch(1000 + i, model in CANONICAL)
    if model == api.MODEL_FM_CANONICAL:
        m = tr.step_host_values(rp, keys, vals, lab)
    elif model == api.MODEL_MVM:
        m = tr.step_host_fields(rp, keys, fields, vals, lab)
    elif policy == "weights":
        m = tr.step_host_weighted(rp, keys, lab, w)
    else:
        m = tr.step_host(rp, keys, lab)
    loss = tr.get_loss(B)
    if policy == "evict" and i % 2 == 1:
        t.evict()
    return m, loss


def _predict(tr, name):
    model = TABLES[name][0]
    rp, keys, lab, vals, fields, _ = _batch(99, model in CANONICAL)
    if model == api.MODEL_FM_CANONICAL:
        return tr.predict_host_values(rp, keys, vals)
    if model == api.MODEL_MVM:
        return tr.predict_host_fields(rp, keys, fields, vals)
    return tr.predict_host(rp, keys)


def _state(t, tr, name, policy):
    keys = np.sort(t.list_keys())
    s = dict(keys=keys, export=t.export(keys), size=t.size(), capacity=t.capacity(), stats=t.admission_stats())
    if policy == "evict":
        s["touch"] = t.last_touch(keys)
    s["pred"] = _predict(tr, name)  # last: with a policy, predict inserts nothing; without one it may insert
    return s


def _assert_same(a, b, what):
    assert np.array_equal(a["keys"], b["keys"]), what + ": keys"
    for f in a["export"]:
        x, y = a["export"][f], b["export"][f]
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), "%s: exported %s" % (what, f)
    for f in ("size", "capacity", "stats"):
        assert a[f] == b[f], "%s: %s %r != %r" % (what, f, a[f], b[f])
    if "touch" in a:
        assert np.array_equal(a["touch"], b["touch"]), what + ": last_touch"
    assert np.array_equal(a["pred"].view(np.uint32), b["pred"].view(np.uint32)), what + ": predictions"


def _same_steps(x, y, what):
    """Per step: the residuals bit for bit; the mean |residual|, a float sum the step kernels add up with atomics in
    no fixed order, to its rounding (two uninterrupted runs differ as much)."""
    for i, ((m0, l0), (m1, l1)) in enumerate(zip(x, y)):
        assert np.array_equal(l0.view(np.uint32), l1.view(np.uint32)), "%s: residuals of step %d" % (what, i)
        assert abs(m0 - m1) <= 1e-6 * abs(m0) + 1e-9, "%s: mean_abs_loss of step %d: %r != %r" % (what, i, m0, m1)


def _applicable(name, policy):
    return policy == "none" or TABLES[name][0] not in CANONICAL


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name", sorted(TABLES))
def test_resume_and_save_equal_uninterrupted(name, policy, monkeypatch, tmp_path):
    if not _applicable(name, policy):
        pytest.skip("admission, eviction and weighting do not serve canonical tables")
    path = str(tmp_path / "state.xfst")
    # the run that never saves
    t, tr = _make(name, policy, monkeypatch)
    _policies(t, policy)
    tr.init_push()
    steps_u = [_step(t, tr, name, policy, i) for i in range(2 * N)]
    want = _state(t, tr, name, policy)
    tr.close(); t.close()
    # the run that saves after N batches and goes on
    t, tr = _make(name, policy, monkeypatch)
    _policies(t, policy)
    tr.init_push()
    steps_s = [_step(t, tr, name, policy, i) for i in range(N)]
    t.save_state(path, user=N)
    steps_s += [_step(t, tr, name, policy, i) for i in range(N, 2 * N)]
    _same_steps(steps_s, steps_u, "saved and continued")
    _assert_same(_state(t, tr, name, policy), want, "saved and continued")
    tr.close(); t.close()
    # the run resumed from the image, on a table created at another capacity and without the policies
    t, tr = _make(name, policy, monkeypatch, capacity=1 << 11)
    assert t.load_state(path) == N
    steps_r = [_step(t, tr, name, policy, i) for i in range(N, 2 * N)]
    _same_steps(steps_r, steps_u[N:], "resumed")
    _assert_same(_state(t, tr, name, policy), want, "resumed")
    tr.close(); t.close()


def test_save_is_stream_ordered(monkeypatch, tmp_path):
    """Steps enqueued with step_host_async right before save_state are in the image.  (Two runs compare by state, not
    by file bytes: concurrent inserts race for slots, so where a key lies may differ from run to run.)"""
    name, policy = "lr_ftrl", "bloom"
    L = api.lib()
    bufs = []

    def pinned(a):
        p = C.c_void_p()
        assert L.xf_host_alloc(C.byref(p), max(a.nbytes, 1)) == 0
        C.memmove(p, a.ctypes.data, a.nbytes)
        bufs.append(p)
        return p.value

    t, tr = _make(name, policy, monkeypatch)
    _policies(t, policy)
    steps = [_step(t, tr, name, policy, i) for i in range(N - 2)]
    for i in range(N - 2, N):
        rp, keys, lab, _, _, _ = _batch(1000 + i, False)
        tr.step_host_async(pinned(rp), pinned(keys), pinned(lab), B, B * D)
    t.save_state(str(tmp_path / "a.xfst"))
    tr.sync()
    for p in bufs:
        L.xf_host_free(p)
    tr.close(); t.close()
    t, tr = _make(name, policy, monkeypatch)
    _policies(t, policy)
    steps = [_step(t, tr, name, policy, i) for i in range(N)]
    want = _state(t, tr, name, policy)
    tr.close(); t.close()
    t, tr = _make(name, "none", monkeypatch, capacity=1 << 11)
    t.load_state(str(tmp_path / "a.xfst"))
    _assert_same(_state(t, tr, name, policy), want, "async steps before the save")
    tr.close(); t.close()


@pytest.mark.parametrize("name", ["lr_ftrl", "lr_ftrl_eager", "fm_ftrl_k16"])
def test_image_is_deterministic(name, monkeypatch, tmp_path):
    t, tr = _make(name, "evict", monkeypatch)
    t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=14, hashes=3, decay_batches=3, seed=5)
    t.set_eviction(max_idle_batches=3, max_keys=1500)
    for i in range(N):
        _step(t, tr, name, "evict", i)
    p = [str(tmp_path / ("%d.xfst" % i)) for i in range(3)]
    t.save_state(p[0], user=7)
    t.save_state(p[1], user=7)
    assert not os.path.exists(p[0] + ".tmp")
    t2, tr2 = _make(name, "none", monkeypatch, capacity=1 << 12)
    assert t2.load_state(p[0]) == 7
    t2.save_state(p[2], user=7)
    data = [open(q, "rb").read() for q in p]
    assert data[0] == data[1], "saving the same state twice"
    assert data[0] == data[2], "loading an image and saving it again"


def test_many_chunks_round_trip(monkeypatch, tmp_path):
    """A table of 2^23 slots streams through several chunks of the default size and comes back byte for byte."""
    monkeypatch.delenv("XFLOW_EAGER", raising=False)
    t = api.Table(latent_dim=0, optimizer=api.OPT_FTRL, capacity=1 << 23)
    t.set_eviction()
    t.touch_decimal_ids(0, 3_000_000)
    tr = api.Trainer(t, model=api.MODEL_LR, max_rows=B, max_nnz=B * D, keep_loss=True)
    for i in range(4):
        _step(t, tr, "lr_ftrl", "none", i)
    assert t.capacity() == 1 << 23
    a, b = str(tmp_path / "a.xfst"), str(tmp_path / "b.xfst")
    t.save_state(a)
    hdr = _header(a)
    assert hdr["capacity"] // hdr["chunk_slots"] >= 4
    t2 = api.Table(latent_dim=0, optimizer=api.OPT_FTRL)
    t2.load_state(a)
    t2.save_state(b)
    assert open(a, "rb").read() == open(b, "rb").read()
    k1, k2 = np.sort(t.list_keys()), np.sort(t2.list_keys())
    assert k1.size == t.size() and np.array_equal(k1, k2)
    sample = k1[np.random.default_rng(0).choice(k1.size, 100000, replace=False)]
    e1, e2 = t.export(sample), t2.export(sample)
    for f in e1:
        assert np.array_equal(e1[f].view(np.uint8), e2[f].view(np.uint8)), f
    assert np.array_equal(t.last_touch(sample), t2.last_touch(sample))


# ---- the documented header layout, parsed independently of the library --------------------------------------------
HEADER = [  # (offset, struct format, name)
    (0, "4s", "magic"), (4, "<I", "version"), (8, "<Q", "header_bytes"), (16, "<Q", "capacity"), (24, "<Q", "cap_floor"),
    (32, "<Q", "keys"), (40, "<I", "stride"), (44, "<I", "log2cap"), (48, "<I", "bshift"), (52, "<I", "lazy"),
    (56, "<i", "latent_dim"), (60, "<i", "optimizer"), (64, "<f", "alpha"), (68, "<f", "beta"), (72, "<f", "lambda1"),
    (76, "<f", "lambda2"), (80, "<f", "learning_rate"), (84, "<i", "v_init"), (88, "<Q", "seed"),
    (96, "<i", "shard_index"), (100, "<i", "num_shards"), (104, "<i", "canonical_fm"), (108, "<I", "seq"),
    (112, "<Q", "batches"), (120, "<Q", "rejected"), (128, "<Q", "admitted"), (136, "<i", "admit_mode"),
    (140, "<f", "probability"), (144, "<I", "threshold"), (148, "<I", "log2_cells"), (152, "<I", "hashes"),
    (156, "<I", "tracking"), (160, "<Q", "decay_batches"), (168, "<Q", "admit_seed"), (176, "<Q", "max_idle"),
    (184, "<Q", "max_keys"), (192, "<Q", "user"), (200, "<Q", "chunk_slots"), (208, "<Q", "filter_bytes"),
    (216, "<Q", "ring_entries"), (224, "<Q", "checksum"),
]


def _header(path):
    raw = open(path, "rb").read(232)
    return {name: struct.unpack_from(fmt, raw, off)[0] for off, fmt, name in HEADER}


def _sections(path):
    """Byte offsets of the section boundaries: after the header, after the ring, after each chunk, end of rows."""
    h = _header(path)
    data = open(path, "rb").read()
    pos = 232
    cuts = [pos]
    if h["ring_entries"]:
        pos += 8 * h["ring_entries"] + 8
        cuts.append(pos)
    chunks = []
    for i in range(h["capacity"] // h["chunk_slots"]):
        first, n, _, zero = struct.unpack_from("<4Q", data, pos)
        assert first == i * h["chunk_slots"] and zero == 0
        chunks.append((pos, n))
        pos += 32 + n * (h["stride"] + 8)
        cuts.append(pos)
    assert len(data) == pos + (h["filter_bytes"] + 8 if h["filter_bytes"] else 0)
    return h, cuts, chunks, pos


@pytest.fixture
def image(monkeypatch, tmp_path):
    """A lazy LR FTRL table with Bloom admission and eviction tracking after N batches, and its image."""
    t, tr = _make("lr_ftrl", "none", monkeypatch)
    t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=12, hashes=3, decay_batches=3, seed=5)
    t.set_eviction(max_idle_batches=3, max_keys=1500)
    for i in range(N):
        _step(t, tr, "lr_ftrl", "evict", i)
    path = str(tmp_path / "img.xfst")
    t.save_state(path, user=42)
    yield t, path
    tr.close()
    t.close()


def _refused(t, path, code, *words):
    with pytest.raises(api.XflowError) as e:
        t.load_state(path)
    msg = str(e.value)
    assert ("error %d:" % code) in msg, msg
    for w in words:
        assert w in msg, msg
    # the target is as it was: empty, no batch run, and usable
    assert t.size() == 0 and t.admission_stats()["batches"] == 0
    t.pull(np.arange(1, 5, dtype=np.uint64))
    assert t.size() == 4


def test_header_matches_documented_layout(image):
    t, path = image
    h = _header(path)
    assert h["magic"] == b"XFST" and h["version"] == 1 and h["header_bytes"] == 232
    assert h["capacity"] == t.capacity() == 1 << h["log2cap"] and h["keys"] == t.size()
    assert h["stride"] == t.row_bytes() == 32 and h["lazy"] == 1 and h["latent_dim"] == 0
    assert h["batches"] == N and h["user"] == 42 and h["seq"] == N and h["ring_entries"] == N + 1
    st = t.admission_stats()
    assert (h["rejected"], h["admitted"]) == (st["rejected_tokens"], st["admitted_keys"])
    assert h["admit_mode"] == api.ADMIT_BLOOM and h["threshold"] == 2 and h["log2_cells"] == 12
    assert h["decay_batches"] == 3 and h["admit_seed"] == 5 and h["filter_bytes"] == 1 << 12
    assert h["tracking"] == 1 and h["max_idle"] == 3 and h["max_keys"] == 1500
    assert h["seed"] == 11 and h["num_shards"] == 1 and h["v_init"] == 1
    assert struct.unpack("<f", struct.pack("<f", 5e-2))[0] == h["alpha"]
    _sections(path)


@pytest.mark.parametrize("field,kw,env", [
    ("latent_dim", dict(latent_dim=4), {}),
    ("optimizer", dict(optimizer=api.OPT_SGD), {}),
    ("alpha", dict(alpha=0.1), {}),
    ("beta", dict(beta=2.0), {}),
    ("lambda1", dict(lambda1=1e-4), {}),
    ("lambda2", dict(lambda2=5.0), {}),
    ("learning_rate", dict(learning_rate=1e-2), {}),
    ("v_init", dict(v_init=api.VINIT_ZERO), {}),
    ("seed", dict(seed=12), {}),
    ("num_shards", dict(num_shards=2, shard_index=0), {}),
    ("shard_index", dict(num_shards=1, shard_index=0), "shard"),
    ("row layout", {}, dict(XFLOW_EAGER="1")),
    ("bucket shift", {}, dict(XFLOW_BUCKET_LOG2="0")),
])
def test_mismatched_table_is_refused(image, field, kw, env, monkeypatch):
    _, path = image
    if env == "shard":  # shard_index alone cannot differ from a one-shard image: a shard 1 of 2 image instead
        src = api.Table(latent_dim=0, seed=11, v_init=api.VINIT_COUNTER, num_shards=2, shard_index=1)
        src.save_state(path + ".s")
        path = path + ".s"
        kw = dict(num_shards=2, shard_index=0)
        env = {}
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    args = dict(latent_dim=0, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=11)
    args.update(kw)
    t = api.Table(**args)
    _refused(t, path, -1, field)


def test_canonical_mismatch_is_refused(monkeypatch, tmp_path):
    t, _ = _make("fm_sgd_k8", "none", monkeypatch)
    t.save_state(str(tmp_path / "fm.xfst"))
    c = api.Table(latent_dim=8, optimizer=api.OPT_SGD, v_init=api.VINIT_COUNTER, seed=11, canonical_fm=1)
    _refused(c, str(tmp_path / "fm.xfst"), -1, "canonical_fm")


def test_occupied_target_is_refused(image, monkeypatch):
    _, path = image
    t = api.Table(latent_dim=0, v_init=api.VINIT_COUNTER, seed=11)
    t.pull(np.arange(10, 13, dtype=np.uint64))
    with pytest.raises(api.XflowError, match="error -6:"):
        t.load_state(path)
    assert t.size() == 3
    t2 = api.Table(latent_dim=0, v_init=api.VINIT_COUNTER, seed=11)
    t2.set_admission(api.ADMIT_POISSON, probability=0.0)
    tr = api.Trainer(t2, model=api.MODEL_LR, max_rows=B, max_nnz=B * D)
    rp, keys, lab, _, _, _ = _batch(1, False)
    tr.step_host(rp, keys, lab)
    assert t2.size() == 0 and t2.admission_stats()["batches"] == 1
    with pytest.raises(api.XflowError, match="error -6:"):
        t2.load_state(path)
    assert t2.admission_stats()["batches"] == 1


def test_truncated_and_damaged_images_are_refused(image, tmp_path):
    _, path = image
    h, cuts, chunks, rows_end = _sections(path)
    data = open(path, "rb").read()
    bad = str(tmp_path / "bad.xfst")
    fresh = lambda: api.Table(latent_dim=0, v_init=api.VINIT_COUNTER, seed=11)
    # truncated inside the header, at every section boundary, inside the filter and before its checksum
    for n in [3, 100] + cuts + [rows_end + 100, len(data) - 8, len(data) - 1]:
        if n >= len(data):
            continue
        open(bad, "wb").write(data[:n])
        _refused(fresh(), bad, -4)
    pos, n = next((p, n) for p, n in chunks if n > 0)
    flips = {
        "header": 192,                                        # the user value: the header checksum
        "rows": pos + 32 + 20,                                # a byte of the first row
        "stamps": pos + 32 + n * h["stride"] + 5,             # the stamp of the first row
        "filter": rows_end + 7,
    }
    for what, off in flips.items():
        d = bytearray(data)
        d[off] ^= 0x10
        open(bad, "wb").write(bytes(d))
        _refused(fresh(), bad, -4, "filter" if what == "filter" else ("header" if what == "header" else "rows"))


def test_formats_are_not_interchangeable(image, tmp_path):
    t, path = image
    portable = str(tmp_path / "portable.xftb")
    t.save(portable)
    _refused(api.Table(latent_dim=0, v_init=api.VINIT_COUNTER, seed=11), portable, -4, "xf_table_save")
    t2 = api.Table(latent_dim=0, v_init=api.VINIT_COUNTER, seed=11)
    with pytest.raises(api.XflowError) as e:
        t2.load(path)
    assert "error -4:" in str(e.value) and "xf_table_save_state" in str(e.value)
    assert t2.size() == 0


def test_unwritable_path(image, tmp_path):
    t, _ = image
    path = str(tmp_path / "no_such_dir" / "img.xfst")
    with pytest.raises(api.XflowError, match="error -4:"):
        t.save_state(path)
    assert not os.path.exists(path) and not os.path.exists(path + ".tmp")


# ---- the CLI ---------------------------------------------------------------------------------------------------
CLI_ENV = dict(XFLOW_OPTIMIZER="ftrl", XFLOW_ADMIT="bloom:2", XFLOW_ADMIT_LOG2_CELLS="16", XFLOW_EVICT_MAX_KEYS="300",
               XFLOW_EVICT_EVERY="2", XFLOW_NEG_SAMPLE="0.25")


def _cli(tmp, model, epochs, **extra):
    os.makedirs(tmp, exist_ok=True)
    env = dict(os.environ, **CLI_ENV)
    for k in ("XFLOW_WORLD", "WORLD_SIZE", "XFLOW_CHECKPOINT", "XFLOW_RESUME", "XFLOW_EAGER"):
        env.pop(k, None)
    env.update(extra)
    return subprocess.run([EXE, TRAIN, TEST, model, str(epochs)], cwd=tmp, env=env, capture_output=True, text=True,
                          timeout=600)


@pytest.mark.parametrize("model", ["0", "1"])
def test_cli_resume_equals_uninterrupted(model, tmp_path):
    img = str(tmp_path / "ckpt.xfst")
    runs = {}
    for name, epochs, extra in [("whole", 4, {}), ("first", 2, dict(XFLOW_CHECKPOINT=img)),
                                ("resumed", 4, dict(XFLOW_RESUME=img))]:
        r = _cli(str(tmp_path / name), model, epochs, **extra)
        assert r.returncode == 0, r.stdout + r.stderr
        runs[name] = r
    assert _header(img)["user"] == 2
    metric = lambda r: [l for l in r.stdout.splitlines() if l.startswith("logloss")]
    assert metric(runs["whole"]) and metric(runs["whole"]) == metric(runs["resumed"])
    a = open(tmp_path / "whole" / "pred_0_0.txt", "rb").read()
    assert a and a == open(tmp_path / "resumed" / "pred_0_0.txt", "rb").read()


def test_cli_refuses_policy_change_and_multi_rank(tmp_path):
    img = str(tmp_path / "ckpt.xfst")
    r = _cli(str(tmp_path / "a"), "0", 1, XFLOW_CHECKPOINT=img)
    assert r.returncode == 0, r.stdout + r.stderr
    r = _cli(str(tmp_path / "b"), "0", 2, XFLOW_RESUME=img, XFLOW_ADMIT="bloom:3")
    assert r.returncode != 0 and "XFLOW_ADMIT" in r.stdout + r.stderr, r.stdout + r.stderr
    for var in ("XFLOW_CHECKPOINT", "XFLOW_RESUME"):
        env = {var: img, "XFLOW_WORLD": "2", "XFLOW_RANK": "0", "XFLOW_COMM_FILE": str(tmp_path / "comm.id")}
        for k in ("XFLOW_ADMIT", "XFLOW_EVICT_MAX_KEYS", "XFLOW_EVICT_EVERY", "XFLOW_NEG_SAMPLE"):
            env[k] = ""
        r = _cli(str(tmp_path / "c"), "0", 1, **env)
        assert r.returncode != 0 and var in r.stdout + r.stderr, r.stdout + r.stderr

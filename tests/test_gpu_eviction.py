"""Feature eviction on the device (pytest -m gpu): per-key stamps and sweeps (xf_table_set_eviction / xf_table_evict,
include/xflow_b200.h) against the CPU statement in tests/eviction_model.py, which with the same limits must agree bit
for bit on which keys are present, the stamps, the sweeps' counts, and (within the parity tolerances) the values."""
import os
import re
import subprocess

import numpy as np
import pytest

from common import GOLDEN, assert_close, assert_close_noise_aware
from eviction_model import EvictingTable
from oracle import oracle as O
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN = os.path.join(GOLDEN, "data", "small_train")
TEST = os.path.join(GOLDEN, "data", "small_test")
UNTOUCHED = np.uint64(0xFFFFFFFFFFFFFFFF)

MODELS = {  # name: (model, optimizer, K, eager LR)
    "lr_ftrl": ("lr", "ftrl", 0, False),
    "lr_sgd": ("lr", "sgd", 0, False),
    "lr_ftrl_eager": ("lr", "ftrl", 0, True),
    "fm_sgd_k8": ("fm", "sgd", 8, False),
    "fm_ftrl_k16": ("fm", "ftrl", 16, False),
}
POLICIES = {  # name: (eviction limits, admission policy or None)
    "idle": (dict(max_idle_batches=2), None),
    "budget": (dict(max_keys=3000), None),
    "both": (dict(max_idle_batches=3, max_keys=4000), None),
    "both_bloom": (dict(max_idle_batches=3, max_keys=2500),
                   dict(mode=api.ADMIT_BLOOM, threshold=2, log2_cells=16, hashes=3, seed=7)),
}


def _tables(model, monkeypatch, limits=None, admission=None, capacity=0):
    m, opt, K, eager = MODELS[model]
    if eager:
        monkeypatch.setenv("XFLOW_EAGER", "1")
    gopt = api.OPT_FTRL if opt == "ftrl" else api.OPT_SGD
    oopt = O.OPT_FTRL if opt == "ftrl" else O.OPT_SGD
    gt = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=11, capacity=capacity)
    ot = EvictingTable(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=11)
    xt = EvictingTable(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=11)  # double-accumulating yardstick (Zipf noise)
    if admission is not None:
        for t in (gt, ot, xt):
            t.set_admission(**admission)
    if limits is not None:
        for t in (gt, ot, xt):
            t.set_eviction(**limits)
    return gt, ot, xt, (api.MODEL_LR if m == "lr" else api.MODEL_FM), K


def _agree_keys(gt, ot, uk, what):
    ge, oe = gt.export(uk), ot.export(uk)
    assert np.array_equal(ge["present"], oe["present"]), what
    assert gt.size() == ot.size(), what
    assert np.array_equal(gt.last_touch(uk), ot.last_touch(uk)), what
    return ge, oe


@pytest.mark.parametrize("policy", sorted(POLICIES))
@pytest.mark.parametrize("dist", ["uniform", "zipf"])
@pytest.mark.parametrize("model", sorted(MODELS))
def test_eviction_matches_model(model, dist, policy, monkeypatch):
    B, d, space = 1024, 16, 20000
    limits, admission = POLICIES[policy]
    gt, ot, xt, gm, K = _tables(model, monkeypatch, limits, admission)
    tr = api.Trainer(gt, model=gm, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
    tr.init_push()
    ot.init_push()
    xt.init_push()
    fields = ("w", "nw", "zw") + (("v", "nv", "zv") if K else ())
    all_keys = [np.zeros(1, np.uint64)]
    evicted = 0
    for step in range(8):
        rp, keys, lab = datagen.make_csr_keys(400 + step, B, d, space, api.hash_decimal_ids, dist=dist, zipf_s=1.3,
                                              ragged=(step == 2))
        tr.step_host(rp, keys, lab)
        gl = tr.get_loss(B)
        _, ol = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        with O.exact_sums():
            _, xl = xt.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        all_keys.append(keys)
        if step == 3:  # predict inserts (without admission) are stamped with the batch number
            prp, pkeys, _ = datagen.make_csr_keys(900 + step, B // 4, d, space * 2, api.hash_decimal_ids, dist=dist)
            gp, op = tr.predict_host(prp, pkeys), ot.predict(prp.astype(np.int64), pkeys)
            xp = xt.predict(prp.astype(np.int64), pkeys)
            if dist == "uniform":
                assert_close(gp, op, "pctr", abs_floor=1e-6)
            else:
                assert_close_noise_aware(gp, op, xp, "pctr", abs_floor=1e-6, max_noisy_frac=0.2)
            all_keys.append(pkeys)
        uk = np.unique(np.concatenate(all_keys))
        for phase in ("step", "sweep"):
            if phase == "sweep":
                if step < 2:
                    continue
                n = gt.evict()
                assert n == ot.evict(), "evicted step %d" % step
                xt.evict()
                evicted += n
            what = "%s %d" % (phase, step)
            ge, oe = _agree_keys(gt, ot, uk, what)
            xe = xt.export(uk)
            if dist == "uniform":
                if phase == "step":
                    assert_close(gl, ol, "loss " + what, abs_floor=1e-6)
                for k in fields:
                    assert_close(ge[k], oe[k], "%s %s" % (k, what))
            else:
                if phase == "step":
                    assert_close_noise_aware(gl, ol, xl, "loss " + what, abs_floor=1e-6, max_noisy_frac=0.05)
                for k in fields:
                    assert_close_noise_aware(ge[k], oe[k], xe[k], "%s %s" % (k, what), max_noisy_frac=0.02)
    assert evicted > 0
    assert gt.admission_stats() == ot.admission_stats()
    tr.close()
    gt.close()


def test_stamping_rules(tmp_path):
    t = api.Table(capacity=1 << 12)
    tr = api.Trainer(t, max_rows=64, max_nnz=1024)
    one = np.array([0, 2], np.uint32)

    def step(keys):
        tr.step_host(one, np.asarray(keys, np.uint64), np.array([1], np.uint8), want_loss=False)

    step([1, 2])
    step([3, 4])  # two batches before tracking
    t.set_eviction()
    assert list(t.last_touch([1, 2, 3, 4, 99])) == [2, 2, 2, 2, UNTOUCHED]  # present keys: the current number
    step([1, 5])  # batch 2
    assert list(t.last_touch([1, 2, 5])) == [2, 2, 2]
    # insertions outside a training step: the number of batches run so far (3); existing keys keep their stamps
    t.pull(np.array([10, 1], np.uint64))
    t.push(np.array([11, 2], np.uint64), gw=np.zeros(2, np.float32))
    t.import_(np.array([12, 3], np.uint64), w=np.ones(2, np.float32))
    t.export(np.array([4, 13], np.uint64))  # export never inserts
    tr.predict_host(one, np.array([14, 4], np.uint64))
    tr.init_push()  # key 0
    assert list(t.last_touch([10, 1, 11, 2, 12, 3, 4, 13, 14, 0])) == [3, 2, 3, 2, 3, 2, 2, UNTOUCHED, 3, 3]
    t.touch_decimal_ids(0, 3)
    assert np.all(t.last_touch(api.hash_decimal_ids(np.arange(3))) == 3)
    # an empty batch is not a batch; the next real one is 3
    tr.step_host(np.zeros(1, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.uint8), want_loss=False)
    step([4, 20])
    assert list(t.last_touch([4, 20])) == [3, 3]
    # load: a loaded key is an insertion
    path = str(tmp_path / "ck.bin")
    src = api.Table()
    src.import_(np.array([30, 4], np.uint64), w=np.ones(2, np.float32))
    src.save(path)
    t.load(path)
    assert list(t.last_touch([30, 4])) == [4, 3]
    # tokens that admission rejects stamp nothing
    t.set_admission(api.ADMIT_POISSON, probability=0.0)
    step([40, 20])
    assert list(t.last_touch([40, 20])) == [UNTOUCHED, 4]
    # set_eviction again keeps the stamps; stop_eviction frees them, a restart stamps every key anew
    t.set_eviction(max_keys=100)
    assert t.last_touch([20])[0] == 4
    t.stop_eviction()
    with pytest.raises(api.XflowError, match="tracking"):
        t.last_touch([20])
    t.set_eviction()
    assert np.all(t.last_touch(t.list_keys()) == 5)
    tr.close()
    t.close()


@pytest.mark.parametrize("ring", [None, "5"])
def test_lazy_pending_steps_survive_sweeps(ring, monkeypatch):
    """A lazy and an eager LR table with the same batches and sweeps keep the same keys with the same values; a tiny
    sequence ring makes the lazy table restart its batch numbering on both sides of the sweeps."""
    B, d = 512, 12
    batches = [datagen.make_csr_keys(60 + s, B, d, 6000, api.hash_decimal_ids, dist="zipf", zipf_s=1.2) for s in range(9)]
    out = []
    for eager in (False, True):
        monkeypatch.delenv("XFLOW_SEQ_RING", raising=False)
        monkeypatch.delenv("XFLOW_EAGER", raising=False)
        if ring and not eager:
            monkeypatch.setenv("XFLOW_SEQ_RING", ring)
        if eager:
            monkeypatch.setenv("XFLOW_EAGER", "1")
        t = api.Table()
        t.set_eviction(max_idle_batches=3, max_keys=2000)
        tr = api.Trainer(t, max_rows=B, max_nnz=B * d)
        for i, (rp, keys, lab) in enumerate(batches):
            tr.step_host(rp, keys, lab, want_loss=False)
            if i % 2 == 1:
                t.evict()
        keys = np.sort(t.list_keys())
        out.append((keys, t.last_touch(keys), t.export(keys)))
        tr.close()
        t.close()
    (k0, s0, e0), (k1, s1, e1) = out
    assert np.array_equal(k0, k1) and np.array_equal(s0, s1)
    for f in ("w", "nw", "zw"):
        assert_close(e0[f], e1[f], f)


def test_capacity_floor_noop_and_regrowth():
    t = api.Table(capacity=1 << 12)
    t.set_eviction(max_keys=1000)
    tr = api.Trainer(t, max_rows=4096, max_nnz=4096 * 8)
    rp, keys, lab = datagen.make_csr_keys(1, 4096, 8, 10 ** 7, api.hash_decimal_ids)
    tr.step_host(rp, keys, lab, want_loss=False)
    n0 = t.size()
    assert t.capacity() >= 1 << 16
    assert t.evict() == n0 - 1000
    assert t.size() == 1000 and t.capacity() == 1 << 12  # the creation capacity is the floor
    launches = tr.launches()
    assert t.evict() == 0 and t.capacity() == 1 << 12
    assert tr.launches() - launches <= 1  # the count pass only: no rebuild
    survivors = np.sort(t.list_keys())
    stamps = t.last_touch(survivors)
    # regrowth: many inserts after the shrink, every survivor still found with its stamp
    t.set_eviction()  # no limits: track only
    for s in range(4):
        rp, keys, lab = datagen.make_csr_keys(10 + s, 4096, 8, 10 ** 8, lambda ids: api.hash_decimal_ids(ids + 10 ** 8))
        tr.step_host(rp, keys, lab, want_loss=False)
    assert t.capacity() >= 1 << 17
    assert np.all(t.export(survivors)["present"] == 1)
    assert np.array_equal(t.last_touch(survivors), stamps)
    # a reservation raises the floor
    t.reserve(50000)
    t.set_eviction(max_keys=10)
    t.evict()
    assert t.size() == 10 and t.capacity() == 1 << 17
    tr.close()
    t.close()


@pytest.mark.parametrize("model", ["lr_ftrl", "fm_sgd_k8"])
def test_sweeps_are_bit_reproducible_at_full_size(model, monkeypatch):
    B, d = 65536, 100
    batches = [datagen.make_csr_keys(80 + s, B, d, 10 ** 7, api.hash_decimal_ids, dist="zipf", zipf_s=1.05)
               for s in range(3)]
    out = []
    for _ in range(2):
        t, _, _, gm, _ = _tables(model, monkeypatch, dict(max_idle_batches=1, max_keys=1 << 19), capacity=1 << 22)
        tr = api.Trainer(t, model=gm, max_rows=B, max_nnz=B * d)
        for rp, keys, lab in batches:
            tr.step_host(rp, keys, lab, want_loss=False)
            t.evict()
        keys = np.sort(t.list_keys())
        out.append((keys, t.last_touch(keys), t.export(keys)))
        tr.close()
        t.close()
    (k0, s0, e0), (k1, s1, e1) = out
    assert k0.size == 1 << 19
    assert np.array_equal(k0, k1) and np.array_equal(s0, s1)
    for f in e0:
        assert np.array_equal(e0[f].view(np.uint8), e1[f].view(np.uint8)), f


def test_ingested_slices_stamp_like_step_host():
    tabs = []
    for ingest in (False, True):
        t = api.Table(capacity=1 << 16)
        t.set_eviction(max_keys=300)  # of the bundled shard's 524 keys
        tr = api.Trainer(t, model=api.MODEL_LR, max_rows=1 << 17, max_nnz=1 << 20)
        tr.init_push()
        for _ in range(3):  # epochs
            ld = api.Loader(TRAIN + "-00000", 1 << 16)
            while True:
                if ingest:
                    text = ld.next_raw()
                    if not text:
                        break
                    rows, _ = tr.ingest_text(text)
                    ts = rows // 3
                    for c in range(3):
                        tr.step_ingested(c * ts, (c + 1) * ts)
                else:
                    try:
                        rp, keys, y = next(ld)
                    except StopIteration:
                        break
                    ts = (rp.size - 1) // 3
                    for c in range(3):
                        a, b = c * ts, (c + 1) * ts
                        tr.step_host((rp[a:b + 1] - rp[a]).astype(np.uint32), keys[rp[a]:rp[b]], y[a:b], want_loss=False)
            ld.close()
            t.evict()
        keys = np.sort(t.list_keys())
        tabs.append((keys, t.last_touch(keys), t.export(keys)))
        tr.close()
        t.close()
    (k0, s0, e0), (k1, s1, e1) = tabs
    assert k0.size == 300
    assert np.array_equal(k0, k1) and np.array_equal(s0, s1)
    for name in e0:
        assert np.array_equal(e0[name].view(np.uint8), e1[name].view(np.uint8)), name


@pytest.mark.parametrize("model,K", [("0", 0), ("1", 10)])
def test_cli_with_key_budget_matches_model(model, K, tmp_path):
    exe = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
    env = dict(os.environ, XFLOW_OPTIMIZER="ftrl", XFLOW_EVICT_MAX_KEYS="300", XFLOW_EVICT_EVERY="2")
    for k in ("XFLOW_WORLD", "WORLD_SIZE", "XFLOW_ADMIT"):
        env.pop(k, None)
    r = subprocess.run([exe, TRAIN, TEST, model, "5"], cwd=str(tmp_path), env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    m = re.search(r"logloss: (\S+)\s+auc = (\S+)\s+tp = (\d+) fp = (\d+)", r.stdout)
    assert m, r.stdout
    ll, auc = float(m.group(1)), float(m.group(2))
    t = EvictingTable(K=K)
    t.set_eviction(max_keys=300, every=2)  # of the bundled shard's 524 keys
    O.train_file(t, TRAIN + "-00000", 2 << 20, 5)
    assert t.sweeps == 2 and t.evicted > 0
    lab, p = O.predict_file(t, TEST + "-00000", (4 << 20) if K == 0 else (2 << 20))
    want = O.auc_logloss(lab, p)
    assert abs(ll - want["logloss"]) <= 2e-5 * abs(want["logloss"]) + 1e-6
    assert abs(auc - want["auc"]) <= 2e-5
    pred = np.loadtxt(str(tmp_path / "pred_0_0.txt"), ndmin=2)
    assert np.array_equal(pred[:, 2].astype(np.int32), lab)
    assert np.all(np.abs(pred[:, 0] - p) <= 2e-5 * np.abs(p) + 1.1e-6)


@pytest.mark.parametrize("env,world", [
    (dict(XFLOW_EVICT_MAX_KEYS="100", XFLOW_EVICT_EVERY="2"), "2"),
    (dict(XFLOW_EVICT_MAX_KEYS="x", XFLOW_EVICT_EVERY="2"), "1"),
    (dict(XFLOW_EVICT_IDLE="-3", XFLOW_EVICT_EVERY="2"), "1"),
    (dict(XFLOW_EVICT_IDLE="5"), "1"),
    (dict(XFLOW_EVICT_MAX_KEYS="100", XFLOW_EVICT_EVERY="0"), "1"),
])
def test_cli_refuses_eviction_it_cannot_serve(env, world, tmp_path):
    exe = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
    e = dict(os.environ, XFLOW_WORLD=world, XFLOW_RANK="0", XFLOW_COMM_FILE=str(tmp_path / "comm.id"), **env)
    r = subprocess.run([exe, TRAIN, TEST, "0", "1"], cwd=str(tmp_path), env=e, capture_output=True, text=True,
                       timeout=120)
    assert r.returncode != 0 and "XFLOW_EVICT" in (r.stdout + r.stderr), r.stdout + r.stderr


def test_refusals(monkeypatch):
    t = api.Table()
    for call in (t.evict, lambda: t.last_touch([1])):
        with pytest.raises(api.XflowError, match="tracking"):
            call()
    canon = api.Table(latent_dim=8, canonical_fm=1)
    with pytest.raises(api.XflowError, match="canonical"):
        canon.set_eviction(max_keys=10)
    sharded = api.Table(shard_index=0, num_shards=2)
    with pytest.raises(api.XflowError, match="single-shard"):
        sharded.set_eviction(max_idle_batches=3)
    # a trainer that would run the sharded step (here forced on a one-rank comm)
    import torch  # noqa: F401  (maps PyTorch's NCCL for the comm's bootstrap)
    monkeypatch.setenv("XFLOW_MG_FORCE", "1")
    p = api.Table()
    p.set_eviction(max_keys=10)
    comm = api.Comm(api.Comm.new_id(), 0, 1, 0)
    with pytest.raises(api.XflowError, match="single-GPU"):
        api.Trainer(p, max_rows=4, max_nnz=16, comm=comm)
    # tracking switched on after the sharded trainer exists: its steps refuse
    q = api.Table()
    trq = api.Trainer(q, max_rows=4, max_nnz=16, comm=comm)
    q.set_eviction()
    with pytest.raises(api.XflowError, match="single-GPU"):
        trq.step_host(np.array([0, 1], np.uint32), np.array([5], np.uint64), np.array([1], np.uint8))
    trq.close()
    comm.close()

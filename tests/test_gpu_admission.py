"""Feature admission on the device (pytest -m gpu): xf_table_set_admission with the Bloom-filter and Poisson
policies (include/xflow_b200.h) against the CPU restatement (oracle/), which with the same policy must agree
bit for bit: which keys get a row, the filter's counts and decay, the statistics, and the trained values.  The CPU side
is tests/admission_model.py: the oracle's table, pull, push and worker arithmetic, with the policy stated in numpy."""
import os
import subprocess

import numpy as np
import pytest

from admission_model import ADMIT_BLOOM, AdmittingTable
from common import GOLDEN, assert_close, assert_close_noise_aware
from oracle import oracle as O
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN = os.path.join(GOLDEN, "data", "small_train")
TEST = os.path.join(GOLDEN, "data", "small_test")

MODELS = {  # name: (model, optimizer, K, eager LR)
    "lr_ftrl": ("lr", "ftrl", 0, False),
    "lr_sgd": ("lr", "sgd", 0, False),
    "lr_ftrl_eager": ("lr", "ftrl", 0, True),
    "fm_sgd_k8": ("fm", "sgd", 8, False),
    "fm_ftrl_k16": ("fm", "ftrl", 16, False),
}
POLICIES = {
    # a tiny filter: false positives and the decay decide admissions
    "bloom2_tiny": dict(mode=api.ADMIT_BLOOM, threshold=2, log2_cells=10, hashes=3, decay_batches=2, seed=7),
    "bloom3": dict(mode=api.ADMIT_BLOOM, threshold=3, log2_cells=24, hashes=3, decay_batches=0, seed=1),
    "poisson03": dict(mode=api.ADMIT_POISSON, probability=0.3, seed=3),
}


def _tables(model, policy, monkeypatch, capacity=0):
    m, opt, K, eager = MODELS[model]
    if eager:
        monkeypatch.setenv("XFLOW_EAGER", "1")
    gopt = api.OPT_FTRL if opt == "ftrl" else api.OPT_SGD
    oopt = O.OPT_FTRL if opt == "ftrl" else O.OPT_SGD
    gt = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=11, capacity=capacity)
    ot = AdmittingTable(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=11)
    xt = AdmittingTable(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=11)  # double-accumulating yardstick (Zipf noise)
    if policy is not None:
        gt.set_admission(**policy)
        ot.set_admission(**policy)
        xt.set_admission(**policy)
    return gt, ot, xt, (api.MODEL_LR if m == "lr" else api.MODEL_FM), K


@pytest.mark.parametrize("policy", sorted(POLICIES))
@pytest.mark.parametrize("dist", ["uniform", "zipf"])
@pytest.mark.parametrize("model", sorted(MODELS))
def test_admission_matches_oracle(model, dist, policy, monkeypatch):
    B, d, space = 2048, 24, 30000
    gt, ot, xt, gm, K = _tables(model, POLICIES[policy], monkeypatch)
    tr = api.Trainer(gt, model=gm, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
    tr.init_push()
    ot.init_push()
    xt.init_push()
    fields = ("w", "nw", "zw") + (("v", "nv", "zv") if K else ())
    all_keys = [np.zeros(1, np.uint64)]
    pushed = 0
    for step in range(5):
        rp, keys, lab = datagen.make_csr_keys(300 + step, B, d, space, api.hash_decimal_ids, dist=dist, zipf_s=1.3,
                                              ragged=(step == 2))
        tr.step_host(rp, keys, lab)
        gl = tr.get_loss(B)
        U, ol = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        pushed += U
        with O.exact_sums():
            _, xl = xt.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        all_keys.append(keys)
        uk = np.unique(np.concatenate(all_keys))
        ge, oe, xe = gt.export(uk), ot.export(uk), xt.export(uk)
        assert np.array_equal(ge["present"], oe["present"]), "step %d" % step
        assert gt.size() == ot.size()
        assert gt.admission_stats() == ot.admission_stats()
        if dist == "uniform":
            assert_close(gl, ol, "loss step %d" % step, abs_floor=1e-6)
            for k in fields:
                assert_close(ge[k], oe[k], "%s step %d" % (k, step))
        else:
            assert_close_noise_aware(gl, ol, xl, "loss step %d" % step, abs_floor=1e-6, max_noisy_frac=0.05)
            for k in fields:
                assert_close_noise_aware(ge[k], oe[k], xe[k], "%s step %d" % (k, step), max_noisy_frac=0.02)
    st = gt.admission_stats()
    assert st["batches"] == 5 and st["rejected_tokens"] > 0 and st["admitted_keys"] > 0
    assert tr.stats()["unique_keys"] == pushed  # rejected keys are not counted
    # predict on a fresh batch: absent keys read as 0 and are not inserted
    size = gt.size()
    rp, keys, _ = datagen.make_csr_keys(999, B, d, space, api.hash_decimal_ids, dist=dist, zipf_s=1.3)
    gp, op = tr.predict_host(rp, keys), ot.predict(rp.astype(np.int64), keys)
    if dist == "uniform":
        assert_close(gp, op, "pctr", abs_floor=1e-6)
    else:
        assert_close_noise_aware(gp, op, xt.predict(rp.astype(np.int64), keys), "pctr", abs_floor=1e-6,
                                 max_noisy_frac=0.2)
    assert gt.size() == size == ot.size()


def _train(table, model, batches, B, nnz):
    tr = api.Trainer(table, model=model, max_rows=B, max_nnz=nnz)
    tr.init_push()
    for rp, keys, lab in batches:
        tr.step_host(rp, keys, lab, want_loss=False)
    tr.sync()
    return tr


def _export_all(t):
    keys = np.sort(t.list_keys())
    return keys, t.export(keys)


@pytest.mark.parametrize("model", ["lr_ftrl", "fm_ftrl_k16"])
def test_extreme_policies(model, monkeypatch):
    B, d = 2048, 16
    batches = [datagen.make_csr_keys(50 + s, B, d, 20000, api.hash_decimal_ids, dist="zipf", zipf_s=1.2)
               for s in range(4)]
    # p = 1 admits every key: bit-identical to a table without a policy
    a, _, _, gm, K = _tables(model, None, monkeypatch)
    b, _, _, _, _ = _tables(model, dict(mode=api.ADMIT_POISSON, probability=1.0, seed=5), monkeypatch)
    ta, tb = _train(a, gm, batches, B, B * d), _train(b, gm, batches, B, B * d)
    (ka, ea), (kb, eb) = _export_all(a), _export_all(b)
    assert np.array_equal(ka, kb)
    for k in ea:
        assert np.array_equal(ea[k].view(np.uint8), eb[k].view(np.uint8)), k
    assert b.admission_stats()["rejected_tokens"] == 0
    # p = 0 admits nothing: only the init-push key, and every prediction is sigmoid(0)
    z, _, _, _, _ = _tables(model, dict(mode=api.ADMIT_POISSON, probability=0.0, seed=5), monkeypatch)
    tz = _train(z, gm, batches, B, B * d)
    assert z.size() == 1 and np.array_equal(z.list_keys(), np.zeros(1, np.uint64))
    assert z.admission_stats()["rejected_tokens"] == sum(k.size for _, k, _ in batches)
    rp, keys, _ = batches[0]
    assert np.all(tz.predict_host(rp, keys) == np.float32(O.sigmoid(0.0)))
    # back to ALL after Bloom: absent keys are inserted again
    z.set_admission(api.ADMIT_BLOOM, threshold=200, log2_cells=12)
    tz.step_host(rp, keys, batches[0][2])
    assert z.size() == 1
    z.set_admission(api.ADMIT_ALL)
    tz.step_host(rp, keys, batches[0][2])
    assert z.size() == 1 + np.unique(keys[keys != 0]).size
    for t in (ta, tb, tz):
        t.close()


@pytest.mark.parametrize("model", ["lr_ftrl", "fm_sgd_k8"])
def test_bloom_is_bit_reproducible_at_full_size(model, monkeypatch):
    """B = 65536 rows of 100 Zipf tokens: hot keys make every append, count and insert contended."""
    B, d = 65536, 100
    batches = [datagen.make_csr_keys(70 + s, B, d, 10 ** 7, api.hash_decimal_ids, dist="zipf", zipf_s=1.05)
               for s in range(3)]
    out = []
    for _ in range(2):
        t, _, _, gm, _ = _tables(model, dict(mode=api.ADMIT_BLOOM, threshold=2, log2_cells=24, hashes=3), monkeypatch,
                                 capacity=1 << 22)
        tr = _train(t, gm, batches, B, B * d)
        out.append((_export_all(t), t.admission_stats()))
        tr.close()
        t.close()
    ((k0, e0), s0), ((k1, e1), s1) = out
    assert s0 == s1 and s0["rejected_tokens"] > 0 and s0["admitted_keys"] > 0
    assert np.array_equal(k0, k1)
    for k in e0:
        assert np.array_equal(e0[k].view(np.uint8), e1[k].view(np.uint8)), k


def test_ingested_slices_honour_admission():
    """step_ingested slices of device-parsed blocks == step_host on the same slices, with a Bloom policy."""
    tabs = []
    for ingest in (False, True):
        t = api.Table(capacity=1 << 16)
        t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=16, hashes=3)
        tr = api.Trainer(t, model=api.MODEL_LR, max_rows=1 << 17, max_nnz=1 << 20)
        tr.init_push()
        ld = api.Loader(TRAIN + "-00000", 1 << 16)
        for _ in range(3):  # epochs
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
            ld = api.Loader(TRAIN + "-00000", 1 << 16)
        tr.sync()
        tabs.append((_export_all(t), t.admission_stats()))
        tr.close()
        t.close()
    ((k0, e0), s0), ((k1, e1), s1) = tabs
    assert s0 == s1 and s0["rejected_tokens"] > 0
    assert np.array_equal(k0, k1)
    for name in e0:
        assert np.array_equal(e0[name].view(np.uint8), e1[name].view(np.uint8)), name


@pytest.mark.parametrize("model,K", [("0", 0), ("1", 10)])
def test_cli_with_bloom_admission_matches_oracle(model, K, tmp_path):
    exe = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
    env = dict(os.environ, XFLOW_OPTIMIZER="ftrl", XFLOW_ADMIT="bloom:2", XFLOW_ADMIT_LOG2_CELLS="20")
    env.pop("XFLOW_WORLD", None)
    env.pop("WORLD_SIZE", None)
    r = subprocess.run([exe, TRAIN, TEST, model, "5"], cwd=str(tmp_path), env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    import re
    m = re.search(r"logloss: (\S+)\s+auc = (\S+)\s+tp = (\d+) fp = (\d+)", r.stdout)
    assert m, r.stdout
    ll, auc = float(m.group(1)), float(m.group(2))
    t = AdmittingTable(K=K)
    t.set_admission(ADMIT_BLOOM, threshold=2, log2_cells=20, hashes=3)
    O.train_file(t, TRAIN + "-00000", 2 << 20, 5)
    assert t.admission_stats()["rejected_tokens"] > 0
    lab, p = O.predict_file(t, TEST + "-00000", (4 << 20) if K == 0 else (2 << 20))
    want = O.auc_logloss(lab, p)
    assert abs(ll - want["logloss"]) <= 2e-5 * abs(want["logloss"]) + 1e-6
    assert abs(auc - want["auc"]) <= 2e-5
    pred = np.loadtxt(str(tmp_path / "pred_0_0.txt"), ndmin=2)
    assert np.array_equal(pred[:, 2].astype(np.int32), lab)
    assert np.all(np.abs(pred[:, 0] - p) <= 2e-5 * np.abs(p) + 1.1e-6)


@pytest.mark.parametrize("value,world", [("bloom:2", "2"), ("bloom:x", "1"), ("poisson:1.5", "1"), ("lru:3", "1")])
def test_cli_refuses_admission_it_cannot_serve(value, world, tmp_path):
    exe = os.path.join(ROOT, "xflow_b200", "bin", "xflow_lr")
    env = dict(os.environ, XFLOW_ADMIT=value, XFLOW_WORLD=world, XFLOW_RANK="0",
               XFLOW_COMM_FILE=str(tmp_path / "comm.id"))
    r = subprocess.run([exe, TRAIN, TEST, "0", "1"], cwd=str(tmp_path), env=env, capture_output=True, text=True,
                       timeout=120)
    assert r.returncode != 0 and "XFLOW_ADMIT" in (r.stdout + r.stderr), r.stdout + r.stderr


def test_refusals(monkeypatch):
    t = api.Table()
    bad = [dict(mode=7), dict(mode=api.ADMIT_POISSON, probability=1.5), dict(mode=api.ADMIT_POISSON, probability=-0.1),
           dict(mode=api.ADMIT_BLOOM, threshold=0), dict(mode=api.ADMIT_BLOOM, threshold=256),
           dict(mode=api.ADMIT_BLOOM, log2_cells=9), dict(mode=api.ADMIT_BLOOM, log2_cells=37),
           dict(mode=api.ADMIT_BLOOM, hashes=0), dict(mode=api.ADMIT_BLOOM, hashes=9)]
    for cfg in bad:
        with pytest.raises(api.XflowError, match="admission"):
            t.set_admission(**cfg)
    # a refused config leaves the table as it was: training still inserts every key
    tr = api.Trainer(t, max_rows=4, max_nnz=16)
    tr.step_host(np.array([0, 2], np.uint32), np.array([5, 6], np.uint64), np.array([1], np.uint8))
    assert t.size() == 2 and t.admission_stats()["rejected_tokens"] == 0
    canon = api.Table(latent_dim=8, canonical_fm=1)
    with pytest.raises(api.XflowError, match="canonical"):
        canon.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=12)
    sharded = api.Table(shard_index=0, num_shards=2)
    with pytest.raises(api.XflowError, match="single-shard"):
        sharded.set_admission(api.ADMIT_POISSON, probability=0.5)
    # a trainer that would run the sharded step (here forced on a one-rank comm)
    import torch  # noqa: F401  (maps PyTorch's NCCL for the comm's bootstrap)
    monkeypatch.setenv("XFLOW_MG_FORCE", "1")
    p = api.Table()
    p.set_admission(api.ADMIT_POISSON, probability=0.5)
    comm = api.Comm(api.Comm.new_id(), 0, 1, 0)
    with pytest.raises(api.XflowError, match="single-GPU"):
        api.Trainer(p, max_rows=4, max_nnz=16, comm=comm)
    comm.close()

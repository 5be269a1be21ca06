"""GPU parity at the edges of the kernels' code paths and number ranges (pytest -m gpu), against the oracle (or the
float64 model for the canonical FM):

  A. lazy LR residual sums at and beyond 2^20 tokens of one key (the 48-bit fixed-point field of table.cuh and the
     per-batch unit xf_fix_shift), and the resolution of the sums just below and above that size;
  B. latent widths K = 1 ... 1024: VEC = 1, 2 and 4, the sector path, chunk counts that are not a power of two and
     K / VEC > 32 in xf_k_update, through fused steps and through Pull / Push; canonical FM at K = 32, 64, 128;
  C. rows longer than 128 tokens (phase B's re-probe from chunk 2 on), with and without admission;
  D. the process-wide setting XFLOW_FM_CACHE_LOG2, in a child process (edge_child.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from admission_model import AdmittingTable
from common import CanonicalFM64, assert_close, assert_close_noise_aware, check_fm_first_step
from oracle import oracle as O
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _opt(name):
    return (api.OPT_FTRL, O.OPT_FTRL) if name == "ftrl" else (api.OPT_SGD, O.OPT_SGD)


def _csr(rows):
    rp = np.zeros(len(rows) + 1, np.uint32)
    rp[1:] = np.cumsum([len(r) for r in rows])
    keys = np.concatenate([np.asarray(r, np.uint64) for r in rows]) if rows else np.zeros(0, np.uint64)
    return rp, keys


# ---------------------------------------------------------------------------------------------------------------------
# A. lazy LR: residual sums of one key at and beyond 2^20
# ---------------------------------------------------------------------------------------------------------------------
HEAVY = np.uint64(0x5DEECE66D1234567)
LIGHT = api.hash_decimal_ids(np.arange(3000, dtype=np.uint64))


def _heavy_batch(count, sign, seed, light_rows=2048):
    """`count` tokens of HEAVY in rows of 64 (with w = sign * 1 imported, each such row has wx = 64 sign, beyond the
    sigmoid's clamp: residual 1.0 with label 0, or 1e-6 - 1 with label 1), and rows of 8 uniform light keys."""
    assert count % 64 == 0
    rng = np.random.default_rng(seed)
    heavy = [np.full(64, HEAVY)] * (count // 64)
    light = list(rng.choice(LIGHT, (light_rows, 8)))
    lab = np.concatenate([np.full(len(heavy), 0 if sign > 0 else 1), rng.integers(0, 2, light_rows)]).astype(np.uint8)
    perm = rng.permutation(len(heavy) + light_rows)
    rows = heavy + light
    rp, keys = _csr([rows[i] for i in perm])
    return rp, keys, lab[perm]


@pytest.mark.parametrize("sign", [1, -1], ids=["r+1", "r-1"])
@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("count", [(1 << 20) - 64, 1 << 20, 3 << 20], ids=["2^20-64", "2^20", "3x2^20"])
def test_lazy_lr_residual_sum_beyond_2_20(count, opt, sign, monkeypatch):
    """One key's residual sum over a batch reaches count (|residual| = 1 on every token).  A fixed unit of 2^-27 in the
    48-bit field wraps at 2^20 and flips the sign of the step; the lazy table must agree with the eager table (double
    sums) and the oracle, after the first step (export folds the pending step), in the residuals of the second (they
    pull the folded weight) and after it."""
    gopt, oopt = _opt(opt)
    lazy = api.Table(optimizer=gopt, capacity=1 << 14)
    monkeypatch.setenv("XFLOW_EAGER", "1")
    eager = api.Table(optimizer=gopt, capacity=1 << 14)
    monkeypatch.delenv("XFLOW_EAGER")
    ot = O.Table(K=0, opt=oopt)
    w0 = np.array([float(sign)], np.float32)
    for t in (lazy, eager, ot):
        t.import_(np.array([HEAVY]), w=w0)
    batches = [_heavy_batch(count, sign, 1 + s) for s in range(2)]
    max_nnz = max(b[1].size for b in batches)
    tl = api.Trainer(lazy, max_rows=batches[0][2].size, max_nnz=max_nnz, keep_loss=True)
    te = api.Trainer(eager, max_rows=batches[0][2].size, max_nnz=max_nnz, keep_loss=True)
    uk = np.concatenate([[HEAVY], LIGHT]).astype(np.uint64)
    for step, (rp, keys, lab) in enumerate(batches):
        B = lab.size
        tl.step_host(rp, keys, lab)
        te.step_host(rp, keys, lab)
        with O.exact_sums():
            _, ol = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        assert_close(tl.get_loss(B), ol, "lazy residuals, step %d" % step, abs_floor=1e-6)
        assert_close(te.get_loss(B), ol, "eager residuals, step %d" % step, abs_floor=1e-6)
        la, ea, oa = lazy.export(uk), eager.export(uk), ot.export(uk)
        for k in ("w", "nw", "zw"):
            assert_close(la[k][:1], oa[k][:1], "lazy heavy %s after step %d" % (k, step))
            assert_close(ea[k][:1], oa[k][:1], "eager heavy %s after step %d" % (k, step))
            assert_close(la[k], oa[k], "lazy %s after step %d" % (k, step))
            assert_close(la[k], ea[k], "lazy vs eager %s after step %d" % (k, step), rel=2e-6, abs_floor=1e-9)


@pytest.mark.parametrize("wx", [-9.0, -31.0])
@pytest.mark.parametrize("nnz", [(1 << 20) - 8, 1 << 20], ids=["below", "at"])
def test_lazy_lr_residual_sum_resolution(nnz, wx):
    """Rows of one bias key (imported w = wx: residual sigmoid(-9) ~ 1.2e-4, or the 1e-6 clamp, label 0) and 7 probe keys
    that start at zero.  After one FTRL step a probe key has z = g exactly, and g is its residual sum in units of 2^-s
    (s = 27 below 2^20 tokens, 26 at 2^20): |z - sum_exact / rows| <= count * 2^-s / 2 / rows + 2 ulp(z), where
    sum_exact is the float64 sum of the kernel's own residuals."""
    rows, d = nnz // 8, 8
    rng = np.random.default_rng(5)
    bias = np.uint64(0x0BADC0FFEE)
    probes = api.hash_decimal_ids(np.arange(1000, 3000, dtype=np.uint64))
    tok = rng.choice(probes, (rows, d - 1))
    keys = np.concatenate([np.full((rows, 1), bias), tok], 1).reshape(-1).astype(np.uint64)
    rp = (np.arange(rows + 1) * d).astype(np.uint32)
    lab = np.zeros(rows, np.uint8)
    t = api.Table(optimizer=api.OPT_FTRL, capacity=1 << 14)
    t.import_(np.array([bias]), w=np.array([wx], np.float32))
    tr = api.Trainer(t, max_rows=rows, max_nnz=keys.size, keep_loss=True)
    tr.step_host(rp, keys, lab)
    loss = tr.get_loss(rows).astype(np.float64)
    assert np.all(loss == loss[0]) and 0 < loss[0] < 2e-4
    s = 27 if keys.size < (1 << 20) else 26
    unit = 2.0 ** -s
    uk, inv, cnt = np.unique(tok.reshape(-1), return_inverse=True, return_counts=True)
    exact = np.zeros(uk.size)
    np.add.at(exact, inv, np.repeat(loss, d - 1))
    z = t.export(uk)["zw"].astype(np.float64)
    bound = cnt * unit / 2 / rows + 2 * np.spacing(np.abs(z).astype(np.float32)).astype(np.float64)
    err = np.abs(z - exact / rows)
    assert np.all(err <= bound), "worst %g vs bound %g" % (err.max(), bound[np.argmax(err - bound)])


def _mg_worker(rank, world, id_path, count, ret):
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
    table = A.Table(optimizer=A.OPT_FTRL, device=rank, shard_index=rank, num_shards=world, capacity=1 << 16)
    batches = [_mg_batch(count, r) for r in range(world)]
    tr = A.Trainer(table, max_rows=max(b[2].size for b in batches), max_nnz=max(b[1].size for b in batches) + 8,
                   keep_loss=True, comm=comm)
    if A.shard_of(int(HEAVY), world) == rank:
        table.import_(np.array([HEAVY]), w=np.array([1.0], np.float32))
    comm.barrier()
    losses = []
    for _ in range(2):
        rp, keys, lab = batches[rank]
        tr.step_host(rp, keys, lab)
        losses.append(tr.get_loss(lab.size))
    tr.sync()
    comm.barrier()
    allk = np.concatenate([[HEAVY], LIGHT]).astype(np.uint64)
    mine = np.array([A.shard_of(int(k), world) == rank for k in allk])
    ret[rank] = dict(keys=allk[mine], e=table.export(allk[mine]), losses=losses)
    comm.barrier()
    tr.close()
    table.close()
    comm.close()


def _mg_batch(count, rank):
    # rank 0 carries the heavy key's 2^20 tokens: one source's push holds the whole sum
    return _heavy_batch(count, 1, 40 + rank) if rank == 0 else _heavy_batch(0, 1, 40 + rank)


def test_sharded_lazy_lr_residual_sum_beyond_2_20(tmp_path):
    """The A1 batch through the sharded LR step (the owner's xf_k_push_tokens_lr quantises each (step, source) with its
    own unit) on 2 GPUs, against the oracle's lock-step schedule."""
    world, count = 2, 1 << 20
    if api.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_mg_worker, args=(world, str(tmp_path / "ncclid.npy"), count, ret), nprocs=world, join=True)
    t = O.Table(K=0, opt=O.OPT_FTRL)
    t.import_(np.array([HEAVY]), w=np.array([1.0], np.float32))
    losses = {r: [] for r in range(world)}
    with O.exact_sums():
        for _ in range(2):
            pend = []
            for r in range(world):
                rp, keys, lab = _mg_batch(count, r)
                uk, gw, gv, loss = t.worker_compute(rp.astype(np.int64), keys, lab.astype(np.int32))
                pend.append((uk, gw))
                losses[r].append(loss)
            for uk, gw in pend:
                t.push(uk, gw)
    for r in range(world):
        got = ret[r]
        for a, b in zip(got["losses"], losses[r]):
            assert_close(a, b, "loss rank %d" % r, abs_floor=1e-6)
        ref = t.export(got["keys"])
        for k in ("w", "nw", "zw"):
            assert_close(got["e"][k], ref[k], "rank %d %s" % (r, k))


# ---------------------------------------------------------------------------------------------------------------------
# B. latent widths
# ---------------------------------------------------------------------------------------------------------------------
WIDTHS = [1, 2, 4, 5, 12, 24, 33, 64, 100, 129, 132, 256, 1024]


@pytest.mark.parametrize("dist", ["uniform", "zipf"])
@pytest.mark.parametrize("K", WIDTHS)
def test_fm_latent_widths_match_oracle(K, dist):
    """FTRL widths: the first step against its float64 closed form (common.check_fm_first_step), whose tolerances scale
    with the magnitude of the summed terms.  From K ~ 100 on, the rounding of the K-term float sums (a row's latent
    terms, and the K adds that form a token's w-gradient) moves FTRL's first step by more than 1e-5 relative, and the
    reference's sequential float order is no better an answer than the kernel's, so the float64 model is the yardstick
    there.  SGD widths: three steps against the oracle (the small SGD steps leave that noise below the tolerance)."""
    opt = "ftrl" if WIDTHS.index(K) % 2 == 0 else "sgd"
    gopt, oopt = _opt(opt)
    B, d, space = 512, 12, 2000
    if opt == "ftrl":
        gt = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=13)
        tr = api.Trainer(gt, model=api.MODEL_FM, max_rows=B, max_nnz=B * d, keep_loss=True)
        rp, keys, lab = datagen.make_csr_keys(60, B, d, space, api.hash_decimal_ids, dist=dist, zipf_s=1.3)
        uk = np.unique(keys)
        w0, v0 = gt.pull(uk)
        assert not w0.any()
        tr.step_host(rp, keys, lab)
        check_fm_first_step(rp, keys, lab, K, lambda k: v0, tr.get_loss(B), gt.export, k_fold_w=True)
        return
    gt = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=13)
    ot = O.Table(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=13)
    xt = O.Table(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=13)
    tr = api.Trainer(gt, model=api.MODEL_FM, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
    seen = [np.zeros(1, np.uint64)]
    for step in range(3):
        rp, keys, lab = datagen.make_csr_keys(60 + step, B, d, space, api.hash_decimal_ids, dist=dist, zipf_s=1.3,
                                              ragged=(step == 1))
        tr.step_host(rp, keys, lab)
        gl = tr.get_loss(B)
        _, ol = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        with O.exact_sums():
            _, xl = xt.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        seen.append(keys)
        uk = np.unique(np.concatenate(seen))
        ge, oe, xe = gt.export(uk), ot.export(uk), xt.export(uk)
        assert np.array_equal(ge["present"], oe["present"])
        if dist == "uniform":
            assert_close(gl, ol, "K=%d loss step %d" % (K, step), abs_floor=1e-6)
        else:
            # a hot key's noise shows in every row that holds it: no bound on the noisy fraction of the residuals
            assert_close_noise_aware(gl, ol, xl, "K=%d loss step %d" % (K, step), abs_floor=1e-6, max_noisy_frac=1.0)
        for k in ("w", "v"):
            if dist == "uniform":
                assert_close(ge[k], oe[k], "K=%d %s step %d" % (K, k, step))
            else:
                assert_close_noise_aware(ge[k], oe[k], xe[k], "K=%d %s step %d" % (K, k, step), max_noisy_frac=0.02)


def pull_push_bit_exact(K, opt, seed=3, iters=4, n_keys=1500):
    """Pull / Push against the oracle's handles: same inputs, same op order, bit-exact state."""
    gopt, oopt = _opt(opt)
    gt = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=seed, capacity=1024)
    ot = O.Table(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=seed)
    rng = np.random.default_rng(K)
    universe = rng.integers(0, 2 ** 64 - 1, 6000, dtype=np.uint64)
    for it in range(iters):
        keys = np.unique(rng.choice(universe, n_keys))
        gw, gv = gt.pull(keys)
        ow, ov = ot.pull(keys)
        assert np.array_equal(gw.view(np.uint32), ow.view(np.uint32)), "pull w"
        assert np.array_equal(gv.view(np.uint32), ov.view(np.uint32)), "pull v"
        g1 = (rng.standard_normal(keys.size) * 0.1).astype(np.float32)
        g2 = (rng.standard_normal((keys.size, K)) * 0.1).astype(np.float32)
        g1[::7] = 0.0
        g2[::5] = 0.0
        gt.push(keys, g1, g2)
        ot.push(keys, g1, g2)
    e, o = gt.export(universe), ot.export(universe)
    assert np.array_equal(e["present"], o["present"])
    for k in ("w", "nw", "zw", "v", "nv", "zv"):
        assert np.array_equal(e[k].view(np.uint32), o[k].view(np.uint32)), k
    return gt.size(), ot.size()


@pytest.mark.parametrize("K", WIDTHS)
def test_pull_push_latent_widths_bit_exact(K):
    a, b = pull_push_bit_exact(K, "ftrl" if WIDTHS.index(K) % 2 == 0 else "sgd")
    assert a == b


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("K", [32, 64, 128])
def test_canonical_fm_wide_matches_float64_model(K, opt):
    gopt, _ = _opt(opt)
    B, d, space = 256, 10, 1500
    t = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=4, canonical_fm=1)
    tr = api.Trainer(t, model=api.MODEL_FM_CANONICAL, max_rows=B, max_nnz=B * d * 2, keep_loss=True)
    rng = np.random.default_rng(K)
    model = CanonicalFM64(K, opt, t.pull)
    for step in range(3):
        rp, keys, lab = datagen.make_csr_keys(80 + step, B, d, space, api.hash_decimal_ids, ragged=(step == 1))
        x = (rng.random(keys.size) * 1.5 + 0.25).astype(np.float32)
        x[::7] *= -1.0
        loss = model.step(rp, keys, x, lab)
        tr.step_host_values(rp, keys, x, lab)
        assert_close(tr.get_loss(B), loss, "canonical FM K=%d residuals, step %d" % (K, step), rel=2e-5, abs_floor=2e-6)
    allk = model.keys()
    e, ref = t.export(allk), model.export(allk)
    for k in ("w", "v") + (("nw", "zw", "nv", "zv") if opt == "ftrl" else ()):
        assert_close(e[k].reshape(allk.size, -1), ref[k], "canonical FM K=%d %s" % (K, k), rel=2e-4, abs_floor=2e-7)


# ---------------------------------------------------------------------------------------------------------------------
# C. rows longer than 128 tokens
# ---------------------------------------------------------------------------------------------------------------------
LONG_LENS = [0, 1, 127, 128, 129, 192, 200, 1000, 4097]


def _long_batch(seed, max_len):
    """Rows of every length in LONG_LENS up to max_len (twice, shuffled).  Keys from a small space, so they repeat inside
    rows and across them; every row of 129+ tokens also holds one key in its first chunk and again in chunks 2 and
    later."""
    rng = np.random.default_rng(seed)
    space = api.hash_decimal_ids(np.arange(seed * 1000, seed * 1000 + 400, dtype=np.uint64))
    rows = []
    for n in [n for n in LONG_LENS if n <= max_len] * 2:
        r = rng.choice(space, n)
        if n > 128:
            r[3] = r[n - 1] = space[n % 400]   # token n - 1 sits in chunk 2 or later (64-token chunks)
            if n > 130:
                r[130] = r[3]
        rows.append(r)
    order = rng.permutation(len(rows))
    rp, keys = _csr([rows[i] for i in order])
    return rp, keys, rng.integers(0, 2, len(rows)).astype(np.uint8)


LONG_MODELS = {"fm_k8": (api.MODEL_FM, 8, False), "fm_k10": (api.MODEL_FM, 10, False),
               "lr_eager": (api.MODEL_LR, 0, True), "lr_lazy": (api.MODEL_LR, 0, False)}
LONG_POLICIES = {"none": None,
                 "bloom_tiny": dict(mode=api.ADMIT_BLOOM, threshold=2, log2_cells=10, hashes=3, decay_batches=0, seed=7),
                 "poisson": dict(mode=api.ADMIT_POISSON, probability=0.5, seed=3)}


LONG_RUNS = [(o, m, p) for o in ("ftrl", "sgd") for m in sorted(LONG_MODELS) for p in sorted(LONG_POLICIES)
             if not (LONG_MODELS[m][1] and o == "ftrl")]


@pytest.mark.parametrize("opt,model,policy", LONG_RUNS, ids=["-".join(r) for r in LONG_RUNS])
def test_long_rows_match_oracle(model, opt, policy, monkeypatch):
    """FM rows stop at 200 tokens, and FM runs with SGD only: the reference's forward pass sums a long row's latent
    terms sequentially in float, and with the cancellation in S^2 - Q that noise reaches 1e-4 of the residual, which
    FTRL's first step passes on to z unscaled, so the oracle's order is no yardstick there.  FM + FTRL on rows of up
    to 4097 tokens is held to the float64 model's order-independent bounds instead (test_gpu_fm_step.py,
    test_fm_long_rows_within_bounds).  Phase B's re-probe from chunk 2 on starts at 129 tokens."""
    gm, K, eager = LONG_MODELS[model]
    gopt, oopt = _opt(opt)
    if eager:
        monkeypatch.setenv("XFLOW_EAGER", "1")
    gt = api.Table(latent_dim=K, optimizer=gopt, v_init=api.VINIT_COUNTER, seed=17)
    monkeypatch.delenv("XFLOW_EAGER", raising=False)
    ot = AdmittingTable(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=17)
    xt = AdmittingTable(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=17)
    pol = LONG_POLICIES[policy]
    if pol:
        for t in (gt, ot, xt):
            t.set_admission(**pol)
    batches = [_long_batch(1 + (s % 2), 200 if K else 1 << 30) for s in range(4)]
    tr = api.Trainer(gt, model=gm, max_rows=len(LONG_LENS) * 2, max_nnz=max(b[1].size for b in batches),
                     keep_loss=True)
    seen = [np.zeros(1, np.uint64)]
    fields = ("w", "nw", "zw") + (("v", "nv", "zv") if K else ())
    for step, (rp, keys, lab) in enumerate(batches):
        B = lab.size
        tr.step_host(rp, keys, lab)
        _, ol = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        with O.exact_sums():
            _, xl = xt.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        assert_close_noise_aware(tr.get_loss(B), ol, xl, "loss step %d" % step, abs_floor=1e-6, max_noisy_frac=0.5)
        seen.append(keys)
        uk = np.unique(np.concatenate(seen))
        ge, oe, xe = gt.export(uk), ot.export(uk), xt.export(uk)
        assert np.array_equal(ge["present"], oe["present"]), "step %d" % step
        assert gt.size() == ot.size()
        if pol:
            assert gt.admission_stats() == ot.admission_stats()
        for k in fields:
            assert_close_noise_aware(ge[k], oe[k], xe[k], "%s step %d" % (k, step), max_noisy_frac=0.02)


# ---------------------------------------------------------------------------------------------------------------------
# D. process-wide settings, in a child process
# ---------------------------------------------------------------------------------------------------------------------
def _child(tmp_path, env, what):
    out = str(tmp_path / (what + ".npz"))
    r = subprocess.run([sys.executable, os.path.join(HERE, "edge_child.py"), what, out], env=dict(os.environ, **env),
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    return np.load(out)


@pytest.mark.parametrize("log2", ["0", "10"])
def test_fm_cache_size_setting_matches_oracle(log2, tmp_path):
    got = _child(tmp_path, {"XFLOW_FM_CACHE_LOG2": log2}, "fm_steps")
    _check_fm_steps(got)


def _check_fm_steps(got):
    import edge_child
    for K, opt in edge_child.FM_STEP_CASES:
        oopt = _opt(opt)[1]
        ot = O.Table(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=edge_child.SEED)
        xt = O.Table(K=K, opt=oopt, init_mode=O.INIT_COUNTER, seed=edge_child.SEED)
        for step, (rp, keys, lab) in enumerate(edge_child.fm_batches()):
            _, ol = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
            with O.exact_sums():
                _, xl = xt.step(rp.astype(np.int64), keys, lab.astype(np.int32))
            assert_close_noise_aware(got["loss_%d_%s_%d" % (K, opt, step)], ol, xl, "K=%d loss step %d" % (K, step),
                                     abs_floor=1e-6, max_noisy_frac=0.05)
        uk = got["keys"]
        oe, xe = ot.export(uk), xt.export(uk)
        for k in ("w", "nw", "zw", "v", "nv", "zv"):
            assert_close_noise_aware(got["%s_%d_%s" % (k, K, opt)], oe[k], xe[k], "K=%d %s" % (K, k), max_noisy_frac=0.02)

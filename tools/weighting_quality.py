"""Does importance weighting keep a subsampled model calibrated?  Synthetic click data whose labels depend on the
features (about 3 % positives) and a held-out set from the same distribution; one pass of LR and of FM (k = 8), FTRL,
trained three ways:

  all            every row, weight 1
  sub0.1_w       negatives kept with probability 0.1 (the trainer's negative-sampling policy) and weighted by 10
  sub0.1_unw     the same kept rows, weight 1: the subsample without weights, as a caller without per-row weights
                 would train it (the dropped rows are not passed at all)

Reports, on the held-out set, the mean predicted CTR against the positive rate, and the exact-arithmetic logloss
(natural log) and AUC (ties 1/2).  --backend cpu runs tests/weighting_model.py over the oracle; --backend gpu the
library (needs a CUDA device).  Prints one JSON line per (backend, model, way).

    python tools/weighting_quality.py [--backend cpu|gpu|both] [--rows 400000] [--batch 8192]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from xflow_b200 import datagen  # noqa: E402

RATE, SEED = 0.1, 5


HPARAMS = dict(alpha=0.5, beta=1.0, l1=5e-5, l2=1.0)  # FTRL: faster than the reference's defaults for one pass


def make_data(seed, rows, d=16, space=2000):
    """Uniform ids; each id carries a hidden effect, the label is Bernoulli(sigmoid(-4.2 + sum of effects)).  Every
    row also carries id `space`, a constant feature that lets the linear part learn the base rate."""
    rp, ids, _ = datagen.make_ids(seed, rows, d, space)
    effect = np.random.default_rng(1).normal(0.0, 0.35, space)
    logit = -4.2 + np.add.reduceat(effect[ids.astype(np.int64)], rp[:-1].astype(np.int64))
    u = (datagen.uniform_u64(seed, rows, stream=9) >> np.uint64(11)).astype(np.float64) / float(1 << 53)
    lab = (u < 1.0 / (1.0 + np.exp(-logit))).astype(np.uint8)
    ids = np.insert(ids, rp[:-1].astype(np.int64), np.uint64(space))
    rp = rp.astype(np.int64) + np.arange(rows + 1)
    return rp.astype(np.uint32), ids, lab


def metrics(lab, p):
    p64 = np.clip(p.astype(np.float64), 1e-12, 1 - 1e-12)
    y = lab.astype(np.float64)
    ll = float(-np.mean(y * np.log(p64) + (1 - y) * np.log(1 - p64)))
    order = np.argsort(p, kind="stable")
    ps = p[order]
    ranks = np.empty(p.size, np.float64)
    i = 0
    while i < p.size:  # average ranks over ties
        j = i
        while j + 1 < p.size and ps[j + 1] == ps[i]:
            j += 1
        ranks[order[i:j + 1]] = (i + j) / 2.0 + 1.0
        i = j + 1
    npos = int(y.sum())
    nneg = y.size - npos
    auc = float((ranks[y == 1].sum() - npos * (npos + 1) / 2.0) / (npos * nneg))
    return dict(mean_pctr=float(p64.mean()), pos_rate=float(y.mean()), logloss=ll, auc=auc)


def batches(data, B):
    rp, keys, lab = data
    for s in range(0, lab.size, B):
        e = min(s + B, lab.size)
        yield (rp[s:e + 1] - rp[s]).astype(np.uint32), keys[rp[s]:rp[e]], lab[s:e]


def keep_rows(rp, keys, lab, kept):
    idx = np.flatnonzero(kept)
    lens = np.diff(rp.astype(np.int64))[idx]
    nrp = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    nk = np.concatenate([keys[rp[r]:rp[r + 1]] for r in idx]) if idx.size else keys[:0]
    return nrp, np.ascontiguousarray(nk, np.uint64), lab[idx]


def run_cpu(K, way, train, test, B):
    from oracle import oracle as O
    from weighting_model import WeightingTable, kept_negatives
    t = WeightingTable(K=K, init_mode=O.INIT_COUNTER, seed=3, **HPARAMS)
    if way == "sub0.1_w":
        t.set_negative_sampling(RATE, SEED)
    for rp, keys, lab in batches(train, B):
        if way == "sub0.1_unw":
            kept = (lab != 0) | kept_negatives(rp.astype(np.int64), keys, RATE, SEED)
            rp, keys, lab = keep_rows(rp, keys, lab, kept)
        t.step(rp.astype(np.int64), keys, lab.astype(np.int32))
    ps = [t.predict(rp.astype(np.int64), keys) for rp, keys, _ in batches(test, B)]
    return np.concatenate(ps)


def run_gpu(K, way, train, test, B):
    from weighting_model import kept_negatives
    from xflow_b200 import api
    h = HPARAMS
    t = api.Table(latent_dim=K, v_init=api.VINIT_COUNTER, seed=3, alpha=h["alpha"], beta=h["beta"], lambda1=h["l1"],
                  lambda2=h["l2"])
    tr = api.Trainer(t, model=api.MODEL_FM if K else api.MODEL_LR, max_rows=B, max_nnz=B * 64)
    if way == "sub0.1_w":
        tr.set_negative_sampling(RATE, SEED)
    for rp, keys, lab in batches(train, B):
        if way == "sub0.1_unw":
            kept = (lab != 0) | kept_negatives(rp.astype(np.int64), keys, RATE, SEED)
            rp, keys, lab = keep_rows(rp, keys, lab, kept)
        tr.step_host(rp, keys, lab, want_loss=False)
    ps = [tr.predict_host(rp, keys) for rp, keys, _ in batches(test, B)]
    return np.concatenate(ps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="cpu", choices=["cpu", "gpu", "both"])
    ap.add_argument("--rows", type=int, default=400000)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    from oracle import oracle as O
    rp, ids, lab = make_data(11, args.rows)
    train = (rp, O.hash_decimal_ids(ids), lab)
    rp, ids, lab = make_data(12, args.rows // 4)
    test = (rp, O.hash_decimal_ids(ids), lab)
    backends = ["cpu", "gpu"] if args.backend == "both" else [args.backend]
    for K in (0, 8):
        for way in ("all", "sub0.1_w", "sub0.1_unw"):
            for be in backends:
                p = (run_cpu if be == "cpu" else run_gpu)(K, way, train, test, args.batch)
                out = dict(backend=be, model="lr" if K == 0 else "fm_k8", way=way, train_pos_rate=float(train[2].mean()))
                out.update(metrics(test[2], p))
                print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

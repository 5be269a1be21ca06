"""Wall time of a serving model made from S shard tables (xf_table_freeze_part on each, then xf_model_merge) against
xf_table_freeze of one table that holds the same rows, on one GPU.

    python tools/merge_bench.py [--lr-keys 1e8] [--fm-keys 1e7] [--shards 8] [--repeats 3]

LR FTRL and FM FTRL K = 16 tables get random keys with non-zero imported weights (nothing is pruned).  Both paths are
checked to give the same model (fingerprint and info) before anything is timed.  Prints one line per shape with the
card name and power limit, the median wall time of each path, and its rate in keys/s and GB/s of model rows."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xflow_b200 import api  # noqa: E402

M64 = (1 << 64) - 1


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def fill(tables, S, n, K, seed):
    """n random keys with non-zero weights, each imported into its shard's table and into the last table (whole)"""
    rng = np.random.default_rng(seed)
    step = 1 << 24
    for first in range(0, n, step):
        c = min(step, n - first)
        keys = np.unique(rng.integers(0, M64 - 1, c, dtype=np.uint64))
        w = rng.uniform(0.5, 1.0, keys.size).astype(np.float32)
        f = dict(w=w, nw=w, zw=w)
        if K:
            f.update(v=rng.standard_normal((keys.size, K)).astype(np.float32) * 0.01)
        owner = np.minimum(keys // np.uint64(M64 // S), np.uint64(S - 1)).astype(np.int64)
        for s in range(S):
            sel = owner == s
            tables[s].import_(keys[sel], **{k: v[sel] for k, v in f.items()})
        tables[S].import_(keys, **f)


def run(label, n, K, S, repeats):
    tables = []
    for s in range(S):
        t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, seed=3, shard_index=s, num_shards=S)
        t.reserve(n // S + n // (4 * S))
        tables.append(t)
    whole_t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, seed=3)
    whole_t.reserve(n)
    tables.append(whole_t)
    fill(tables, S, n, K, seed=K + S)

    def sharded():
        parts = [t.freeze_part() for t in tables[:S]]
        m = api.Model.merge(parts)
        for p in parts:
            p.close()
        return m

    def whole():
        return whole_t.freeze()

    a, b = sharded(), whole()
    assert a.fingerprint() == b.fingerprint() and a.info() == b.info(), "the merge is not the whole table's model"
    keys, row_bytes = b.info()["keys"], b.info()["row_bytes"]
    a.close(); b.close()
    times = {"parts+merge": [], "freeze": []}
    for _ in range(repeats):
        for name, fn in (("parts+merge", sharded), ("freeze", whole)):
            t0 = time.perf_counter()
            m = fn()
            times[name].append(time.perf_counter() - t0)
            m.close()
    for name, ts in times.items():
        t = float(np.median(ts))
        print("%s | %s | S = %d | %s: %.1f ms (median of %d) | %.3g keys/s | %.2f GB/s of %d-byte model rows"
              % (card(), label, S, name, t * 1e3, repeats, keys / t, keys * row_bytes / t / 1e9, row_bytes), flush=True)
    for t in tables:
        t.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lr-keys", type=float, default=1e8)
    ap.add_argument("--fm-keys", type=float, default=1e7)
    ap.add_argument("--shards", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if int(args.lr_keys):
        run("LR FTRL %.3g keys" % args.lr_keys, int(args.lr_keys), 0, args.shards, args.repeats)
    if int(args.fm_keys):
        run("FM FTRL K=16 %.3g keys" % args.fm_keys, int(args.fm_keys), 16, args.shards, args.repeats)


if __name__ == "__main__":
    main()

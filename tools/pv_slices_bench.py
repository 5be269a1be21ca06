"""Cost of slicing progressive validation (xf_pv_set_slices) on the headline shape (LR + FTRL, 1e8 ids, 100 tokens per
row, B = 65 536 rows, about 3 % positives), device-resident batches: one trainer trains alternately with an unsliced
pv and a sliced pv attached (xf_trainer_set_validation before each step), so both modes see the same table growth and
the same machine noise.  Two slice maps, 1 000 keys (one slice each) and 100 000 keys (1 000 slices of 100 keys); in
both every row carries one token from the map's keys.  Median ms per step of each mode and their difference, for LR
and for FM K = 16 + FTRL.  Prints the card's name and power limit, then one JSON line per (model, map).

    python tools/pv_slices_bench.py [--steps 40] [--warmup 10] [--ids 100000000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xflow_b200 import api, datagen  # noqa: E402

MAPS = {"1k_keys": (1000, 1000), "100k_keys": (100_000, 1000)}  # name: (keys, slices)
MS = 8


def slice_keys(n):
    """n keys outside the batches' id space (ids >= 2^40)."""
    return api.hash_decimal_ids(np.arange(n, dtype=np.uint64) + np.uint64(1 << 40))


def batch(seed, B, d, ids, map_keys):
    rp, keys, _ = datagen.make_csr_keys(seed, B, d, ids, api.hash_decimal_ids)
    lab = (datagen.uniform_u64(seed, B, stream=7) % np.uint64(100) < np.uint64(3)).astype(np.uint8)
    pick = datagen.uniform_u64(seed, B, stream=9) % np.uint64(map_keys.size)
    keys[rp[:-1] + (rp[1:] - rp[:-1]) // 2] = map_keys[pick.astype(np.int64)]  # one map key per row
    return rp, keys, lab


def run(model, K, map_name, args):
    import torch
    B, d = 65536, 100
    n_keys, n_slices = MAPS[map_name]
    mk = slice_keys(n_keys)
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL)
    t.reserve(int(args.ids * 0.7) if K == 0 else int(args.ids * 0.2))
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * d)
    plain = api.ProgressiveValidation()
    sliced = api.ProgressiveValidation()
    sliced.set_slices(mk, (np.arange(n_keys) % n_slices).astype(np.uint32), n_slices, MS)
    n = 8  # distinct batches, cycled
    dev = []
    for s in range(n):
        rp, keys, lab = batch(1000 + s, B, d, args.ids, mk)
        dev.append([torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda() for a in (rp, keys, lab)])
    torch.cuda.synchronize()
    times = {"pv": [], "sliced_pv": []}
    for i in range(args.warmup + 2 * args.steps):
        mode = "sliced_pv" if i % 2 else "pv"
        tr.set_validation(sliced if mode == "sliced_pv" else plain)
        rp, keys, lab = dev[i % n]
        tr.sync()
        t0 = time.perf_counter()
        tr.step_device(rp.data_ptr(), keys.data_ptr(), lab.data_ptr(), B, B * d)
        tr.sync()
        if i >= args.warmup:
            times[mode].append((time.perf_counter() - t0) * 1e3)
    tr.set_validation(None)
    reps = sliced.report_slices()
    med = {m: float(np.median(ts)) for m, ts in times.items()}
    out = dict(model="lr" if K == 0 else "fm_k16", map=map_name, map_keys=n_keys, slices=n_slices, ms=MS,
               pv_ms_per_step=med["pv"], sliced_ms_per_step=med["sliced_pv"],
               overhead_ms=med["sliced_pv"] - med["pv"], overhead_pct=100.0 * (med["sliced_pv"] / med["pv"] - 1.0),
               pv_min=float(np.min(times["pv"])), sliced_min=float(np.min(times["sliced_pv"])), steps=args.steps,
               slice_rows=int(sum(r["rows"] for r in reps)), global_rows=sliced.report()["rows"])
    tr.close()
    plain.close()
    sliced.close()
    t.close()
    del dev
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--ids", type=int, default=100_000_000)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    for model, K in ((api.MODEL_LR, 0), (api.MODEL_FM, 16)):
        for map_name in MAPS:
            print(json.dumps(run(model, K, map_name, args)), flush=True)


if __name__ == "__main__":
    main()

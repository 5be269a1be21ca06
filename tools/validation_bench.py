"""Cost of progressive validation on the headline shape (LR + FTRL, 1e8 ids, 100 tokens per row, B = 65 536 rows,
labels with about 3 % positives), device-resident batches: one trainer trains alternately with a pv attached and
without one (xf_trainer_set_validation(tr, pv) / NULL before each step), so both modes see the same table growth and
the same machine noise.  Median ms per step of each mode over the timed steps, and the same for FM K = 16 + FTRL.
Prints the card's name and power limit, then one JSON line per (model, mode) and one with the overhead.

    python tools/validation_bench.py [--steps 40] [--warmup 10] [--ids 100000000]
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


def batch(seed, B, d, ids):
    rp, keys, _ = datagen.make_csr_keys(seed, B, d, ids, api.hash_decimal_ids)
    lab = (datagen.uniform_u64(seed, B, stream=7) % np.uint64(100) < np.uint64(3)).astype(np.uint8)
    return rp, keys, lab


def run(model, K, args):
    import torch
    B, d = 65536, 100
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL)
    t.reserve(int(args.ids * 0.7) if K == 0 else int(args.ids * 0.2))
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * d)
    pv = api.ProgressiveValidation()
    n = 8  # distinct batches, cycled
    dev = []
    for s in range(n):
        rp, keys, lab = batch(1000 + s, B, d, args.ids)
        dev.append([torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda() for a in (rp, keys, lab)])
    torch.cuda.synchronize()
    times = {"none": [], "pv": []}
    for i in range(args.warmup + 2 * args.steps):
        mode = "pv" if i % 2 else "none"
        tr.set_validation(pv if mode == "pv" else None)
        rp, keys, lab = dev[i % n]
        tr.sync()
        t0 = time.perf_counter()
        tr.step_device(rp.data_ptr(), keys.data_ptr(), lab.data_ptr(), B, B * d)
        tr.sync()
        if i >= args.warmup:
            times[mode].append((time.perf_counter() - t0) * 1e3)
    tr.set_validation(None)
    name = "lr" if K == 0 else "fm_k16"
    rep = pv.report()
    out = []
    for mode, ts in times.items():
        out.append(dict(model=name, mode=mode, ms_per_step=float(np.median(ts)), ms_min=float(np.min(ts)),
                        ms_max=float(np.max(ts)), steps=len(ts)))
    out.append(dict(model=name, overhead_ms=out[1]["ms_per_step"] - out[0]["ms_per_step"],
                    overhead_pct=100.0 * (out[1]["ms_per_step"] / out[0]["ms_per_step"] - 1.0),
                    pv_rows=rep["rows"], pv_logloss=rep["logloss"], pv_auc=rep["auc"], keys=t.size()))
    tr.close()
    pv.close()
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
        for line in run(model, K, args):
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

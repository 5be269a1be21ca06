"""Device time of a training step and of its optimizer pass for each optimizer (FTRL, SGD, AdaGrad) on bench.py's
shapes: B = 65 536 rows per batch, ids uniform in a 1e8-feature space, 100 tokens per row, keys hashed as the loader
hashes them, for LR (the table pre-populated with all 1e8 ids, as bench.py does) and FM K = 16; and for the canonical
FM at K = 16 and the field-aware FM at L = 32 and 128 on the rows of tools/ffm_bench.py (one token per field).
Two batches are cycled: the warm-up steps insert every key, the timed steps then find them all (LR: the lazy step,
whose optimizer step folds into the next touch of a row, so its optimizer pass is 0).

Each step's device time comes from the trainer's profile events (step kernel + optimizer pass).  Prints the card's
name, power limit and SM clock, then one JSON line per (workload, optimizer).

    python tools/adagrad_bench.py [--steps 20] [--warmup 4] [--workloads lr,fm16,fmc16,ffm32,ffm128]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xflow_b200 import api, datagen  # noqa: E402

B, NNZ, SPACE = 65536, 100, 10 ** 8
OPTS = {"ftrl": api.OPT_FTRL, "sgd": api.OPT_SGD, "adagrad": api.OPT_ADAGRAD}
WORKLOADS = {  # name: (model, K, canonical)
    "lr": (api.MODEL_LR, 0, False),
    "fm16": (api.MODEL_FM, 16, False),
    "fmc16": (api.MODEL_FM_CANONICAL, 16, True),
    "ffm32": (api.MODEL_FFM, 32, True),
    "ffm128": (api.MODEL_FFM, 128, True),
}


def batch(seed, model, K):
    if model == api.MODEL_FFM:
        F = K // 4
        rng = np.random.default_rng(seed)
        ids = rng.integers(0, 1 << 24, (B, F)).astype(np.uint64) + (np.arange(F, dtype=np.uint64) << np.uint64(24))
        keys = api.hash_decimal_ids(ids.reshape(-1))
        fields = np.tile(np.arange(F, dtype=np.uint8), B)
        rp = (np.arange(B + 1) * F).astype(np.uint32)
        return rp, keys, fields, (rng.random(B) < 0.03).astype(np.uint8)
    rp, keys, lab = datagen.make_csr_keys(seed, B, NNZ, SPACE, api.hash_decimal_ids)
    return rp, keys, None, lab


def run(name, opt, args):
    model, K, canonical = WORKLOADS[name]
    t = api.Table(latent_dim=K, optimizer=OPTS[opt], canonical_fm=1 if canonical else 0, v_init=api.VINIT_COUNTER,
                  seed=1)
    if model == api.MODEL_LR:
        t.reserve(SPACE)
        t.touch_decimal_ids(0, SPACE)
    nnz = (K // 4) if model == api.MODEL_FFM else NNZ
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * nnz)
    tr.set_profile(True)
    batches = [batch(100 + 7 * K + s, model, K) for s in range(2)]
    for i in range(args.warmup + args.steps):
        rp, keys, fields, lab = batches[i % 2]
        if model == api.MODEL_FFM:
            tr.step_host_fields(rp, keys, fields, None, lab)
        elif model == api.MODEL_FM_CANONICAL:
            tr.step_host_values(rp, keys, None, lab)
        else:
            tr.step_host(rp, keys, lab)
        if i == args.warmup - 1:
            tr.sync()
            tr.profile()  # drop the warm-up steps' device times
    tr.sync()
    p = tr.profile()
    n = max(p["steps"], 1)
    out = dict(workload=name, optimizer=opt, row_bytes=t.row_bytes(), keys=t.size(), steps=p["steps"],
               device_ms_per_step=(p["step_ms"] + p["update_ms"]) / n, step_kernel_ms=p["step_ms"] / n,
               optimizer_pass_ms=p["update_ms"] / n)
    tr.close()
    t.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("adagrad_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    for name in args.workloads.split(","):
        for opt in OPTS:
            print(json.dumps(run(name, opt, args)), flush=True)


if __name__ == "__main__":
    main()

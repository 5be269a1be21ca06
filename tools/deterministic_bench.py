"""Cost of the deterministic mode (xf_trainer_set_deterministic) of the canonical FM and the multi-view machine:
K = 16 + FTRL, B = 65 536 rows of 39 tokens with feature values (the machine: field ids 0 .. 25 by position), ids
uniform or Zipf (s = 1.05) over 10^7.  Two trainers share one table, one in deterministic mode and one not, and take
alternate steps, so both modes see the same table growth and the same machine noise.  A step is timed on the host
from its call to the end of a device synchronise (the host entry point: upload, step, optimizer pass), and on the
device by the trainer's profile events (step kernel, with the deterministic sort and sums, and optimizer pass).  Prints
the card's name and power limit, then one JSON line per (model, ids, mode) with the median ms per step and the mean
device ms, and one with the overhead.

    python tools/deterministic_bench.py [--steps 30] [--warmup 6]
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

B, D, K, IDS = 65536, 39, 16, 10_000_000


def batch(seed, dist):
    rp, keys, lab = datagen.make_csr_keys(seed, B, D, IDS, api.hash_decimal_ids, dist=dist)
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.1, 1.5, keys.size).astype(np.float32)
    fields = (np.arange(keys.size) % D % 26).astype(np.uint8)
    lab = (rng.random(B) < 0.03).astype(np.uint8)
    return rp, keys, fields, x, lab


def run(mvm, dist, args):
    model = api.MODEL_MVM if mvm else api.MODEL_FM_CANONICAL
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, canonical_fm=1, v_init=api.VINIT_COUNTER, seed=1)
    t.reserve(4_000_000)
    trs = {m: api.Trainer(t, model=model, max_rows=B, max_nnz=B * D) for m in ("default", "deterministic")}
    trs["deterministic"].set_deterministic(True)
    for tr in trs.values():
        tr.set_profile(True)
    batches = [batch(100 + s, dist) for s in range(6)]
    times = {"default": [], "deterministic": []}
    for i in range(args.warmup + 2 * args.steps):
        mode = "deterministic" if i % 2 else "default"
        rp, keys, fields, x, lab = batches[(i // 2) % len(batches)]
        tr = trs[mode]
        tr.sync()
        t0 = time.perf_counter()
        if mvm:
            tr.step_host_fields(rp, keys, fields, x, lab)
        else:
            tr.step_host_values(rp, keys, x, lab)
        tr.sync()
        if i >= args.warmup:
            times[mode].append((time.perf_counter() - t0) * 1e3)
        elif i == args.warmup - 1:
            for tr in trs.values():
                tr.profile()  # drop the warm-up steps' device times
    prof = {m: tr.profile() for m, tr in trs.items()}
    name = "mvm_k16" if mvm else "fmc_k16"
    out = [dict(model=name, ids=dist, mode=m, ms_per_step=float(np.median(ts)), ms_min=float(np.min(ts)),
                ms_max=float(np.max(ts)), steps=len(ts),
                device_step_ms=prof[m]["step_ms"] / max(prof[m]["steps"], 1),
                device_update_ms=prof[m]["update_ms"] / max(prof[m]["steps"], 1)) for m, ts in times.items()]
    out.append(dict(model=name, ids=dist, overhead_ms=out[1]["ms_per_step"] - out[0]["ms_per_step"],
                    overhead_pct=100.0 * (out[1]["ms_per_step"] / out[0]["ms_per_step"] - 1.0), keys=t.size()))
    for tr in trs.values():
        tr.close()
    t.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=6)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    for mvm in (False, True):
        for dist in ("uniform", "zipf"):
            for line in run(mvm, dist, args):
                print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

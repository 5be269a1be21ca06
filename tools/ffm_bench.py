"""Cost of a field-aware FM step (XF_MODEL_FFM, csrc/step_ffm.cu) against the canonical FM at the same latent_dim on
the same keys, and the multi-view machine at latent_dim 32.  FTRL, B = 65 536 rows per batch, one token per field
(F = L / 4 tokens per row, token f in field f), ids uniform over 2^24 per field, hashed as the loader hashes them.
Two batches are cycled: the warm-up steps insert every key, the timed steps then find them all (at L = 128 the
table holds 4.2 M keys in 2^23 rows of 2 112 bytes).

Each step's device time comes from the trainer's profile events (step kernel + optimizer pass); a step is also
timed on the host from its call to the end of a device synchronise (upload included).  Prints the card's name, power
limit and SM clock, then one JSON line per (model, L) with the mean device ms per step, examples/s on that time, and
the median host ms.

    python tools/ffm_bench.py [--steps 20] [--warmup 4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xflow_b200 import api  # noqa: E402

B, SPACE = 65536, 1 << 24


def batch(seed, F):
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, SPACE, (B, F)).astype(np.uint64) + (np.arange(F, dtype=np.uint64) << np.uint64(24))
    keys = api.hash_decimal_ids(ids.reshape(-1))
    fields = np.tile(np.arange(F, dtype=np.uint8), B)
    rp = (np.arange(B + 1) * F).astype(np.uint32)
    lab = (rng.random(B) < 0.03).astype(np.uint8)
    return rp, keys, fields, lab


def run(model, L, args):
    F = L // 4
    t = api.Table(latent_dim=L, optimizer=api.OPT_FTRL, canonical_fm=1, v_init=api.VINIT_COUNTER, seed=1)
    t.reserve(2 * B * F)
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * F)
    tr.set_profile(True)
    batches = [batch(100 + 7 * L + s, F) for s in range(2)]
    host = []
    for i in range(args.warmup + args.steps):
        rp, keys, fields, lab = batches[i % len(batches)]
        tr.sync()
        t0 = time.perf_counter()
        if model == api.MODEL_FM_CANONICAL:
            tr.step_host_values(rp, keys, None, lab)
        else:
            tr.step_host_fields(rp, keys, fields, None, lab)
        tr.sync()
        if i >= args.warmup:
            host.append((time.perf_counter() - t0) * 1e3)
        elif i == args.warmup - 1:
            tr.profile()  # drop the warm-up steps' device times
    p = tr.profile()
    n = max(p["steps"], 1)
    dev = (p["step_ms"] + p["update_ms"]) / n
    name = {api.MODEL_FFM: "ffm", api.MODEL_FM_CANONICAL: "fm_canonical", api.MODEL_MVM: "mvm"}[model]
    out = dict(model=name, L=L, fields=F, rows=B, tokens_per_row=F, device_ms_per_step=dev,
               device_step_kernel_ms=p["step_ms"] / n, device_update_ms=p["update_ms"] / n,
               examples_per_s=B / (dev * 1e-3), host_ms_median=float(np.median(host)), steps=len(host), keys=t.size())
    tr.close()
    t.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    for L in (32, 64, 128):
        for model in (api.MODEL_FFM, api.MODEL_FM_CANONICAL):
            print(json.dumps(run(model, L, args)), flush=True)
    print(json.dumps(run(api.MODEL_MVM, 32, args)), flush=True)


if __name__ == "__main__":
    main()

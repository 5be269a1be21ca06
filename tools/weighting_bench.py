"""Cost of importance weighting on the headline shape (LR + FTRL, 1e8 ids, 100 tokens per row, B = 65 536 rows,
labels with about 3 % positives), device-resident batches, median ms per step over the timed steps:

  none       xf_trainer_step_device: no weights, no policy (the kernels without weighting, no extra launch)
  weights1   xf_trainer_step_device_weighted with every weight 1: the weighting pass plus the WEIGHT step kernel
  sample0.1  xf_trainer_step_device with negative sampling at rate 0.1: about 87 % of the rows skipped

and the same for FM K = 16 + FTRL.  Prints one JSON line per (model, mode).

    python tools/weighting_bench.py [--steps 30] [--warmup 10] [--ids 100000000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xflow_b200 import api, datagen  # noqa: E402


def batch(seed, B, d, ids):
    rp, keys, _ = datagen.make_csr_keys(seed, B, d, ids, api.hash_decimal_ids)
    lab = (datagen.uniform_u64(seed, B, stream=7) % np.uint64(100) < np.uint64(3)).astype(np.uint8)
    return rp, keys, lab


def run(model, K, mode, args):
    import torch
    B, d = 65536, 100
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL)
    t.reserve(int(args.ids * 0.7) if K == 0 else int(args.ids * 0.2))
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * d)
    if mode == "sample0.1":
        tr.set_negative_sampling(0.1, 1)
    n = 8  # distinct batches, cycled
    dev = []
    for s in range(n):
        rp, keys, lab = batch(1000 + s, B, d, args.ids)
        arrs = [torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()
                for a in (rp, keys, lab, np.ones(B, np.float32))]
        dev.append(arrs)
    torch.cuda.synchronize()
    times = []
    for i in range(args.warmup + args.steps):
        rp, keys, lab, w = dev[i % n]
        tr.sync()
        t0 = time.perf_counter()
        if mode == "weights1":
            tr.step_device_weighted(rp.data_ptr(), keys.data_ptr(), lab.data_ptr(), w.data_ptr(), B, B * d)
        else:
            tr.step_device(rp.data_ptr(), keys.data_ptr(), lab.data_ptr(), B, B * d)
        tr.sync()
        if i >= args.warmup:
            times.append((time.perf_counter() - t0) * 1e3)
    out = dict(model="lr" if K == 0 else "fm_k16", mode=mode, ms_per_step=float(np.median(times)),
               ms_min=float(np.min(times)), ms_max=float(np.max(times)), skipped_rows=tr.skipped_rows(),
               rows=(args.warmup + args.steps) * B, launches=tr.launches(), keys=t.size())
    tr.close()
    t.close()
    del dev
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--ids", type=int, default=100_000_000)
    args = ap.parse_args()
    for model, K in ((api.MODEL_LR, 0), (api.MODEL_FM, 16)):
        for mode in ("none", "weights1", "sample0.1"):
            print(json.dumps(run(model, K, mode, args)), flush=True)


if __name__ == "__main__":
    main()

"""Feature eviction on the device (xf_table_set_eviction / xf_table_evict; DESIGN.md section 6): what per-key stamps
cost in the step, and what sweeps save on a drifting stream.

    python tools/eviction_bench.py [--runs 3] [--steps 50] [--warmup 10] [--batches 256] [--skip-cost] [--skip-drift]

Tracking cost: LR+FTRL and FM K = 16 FTRL on the bench's uniform 1e8-id configuration (65 536 rows x 100 nnz, keys
hashed on the device), tracking off vs on, alternated, `--runs` times each: a fresh table, `--warmup` steps over 4
cycled batches, then `--steps` timed steps (CUDA events around every step); median ms per step over the steps, then
over the runs.

Drifting stream: LR+FTRL, 256 batches of 65 536 rows x 100 nnz from an empty table.  Batch b draws Zipf(1.05) ranks r in
[0, 1e8); rank r stands for id r + 1e8 * e, where its epoch e = floor((b + splitmix64(r) % 32) / 32) moves on every 32
batches, staggered over the ranks.  So every batch about 1/32 of the ranks (hot ones included) get a fresh id, and over
the 256 batches the ids slide through a 1e9-id space.  A row's label is 1 iff splitmix64(its first id) % 4 == 0, so the first feature carries the
signal.  Each batch is predicted before it is trained on (progressive validation); the logloss is over all rows of all
batches.  Three runs: no eviction; max_idle_batches = 32 with a sweep every 32 batches; max_keys = 8 M with a sweep
every 32 batches.  Per run: keys, capacity and table + stamp bytes at the end, median step ms, median sweep ms.
Prints one JSON line with the card's name, power limit and SM clocks read in the same run.  Needs a CUDA device.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B_ROWS, NNZ = 65536, 100


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def device_batch(api, torch, stream, rp, ids, lab):
    lib = api.lib()
    nnz = ids.size
    d_ids = torch.from_numpy(ids.astype(np.uint32).view(np.uint8)).cuda()
    d_keys = torch.empty(nnz * 8, dtype=torch.uint8, device="cuda")
    torch.cuda.current_stream().synchronize()
    assert lib.xf_hash_decimal_ids_device(C.c_void_p(d_ids.data_ptr()), nnz, C.c_void_p(d_keys.data_ptr()),
                                          C.c_void_p(stream.cuda_stream)) == 0
    stream.synchronize()
    return torch.from_numpy(rp.view(np.uint8)).cuda(), d_keys, torch.from_numpy(lab.view(np.uint8)).cuda()


def tracking_cost(api, datagen, torch, stream, args):
    nnz = B_ROWS * NNZ
    batches = [device_batch(api, torch, stream, *datagen.make_ids(seed=7000 + i, rows=B_ROWS, nnz_per_row=NNZ,
                                                                   id_space=10 ** 8, dist="uniform"))
               for i in range(4)]
    out = {}
    for name, K, model in (("lr_ftrl", 0, api.MODEL_LR), ("fm_ftrl_k16", 16, api.MODEL_FM)):
        runs = {"off": [], "on": []}
        for _ in range(args.runs):
            for arm in ("off", "on"):
                t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, seed=1, capacity=1 << 27)
                t.set_stream(stream.cuda_stream)
                if arm == "on":
                    t.set_eviction()
                tr = api.Trainer(t, model=model, max_rows=B_ROWS, max_nnz=nnz + 1024)
                for i in range(args.warmup):
                    d = batches[i % 4]
                    tr.step_device(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), B_ROWS, nnz)
                tr.sync()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
                ev[0].record(stream)
                for i in range(args.steps):
                    d = batches[i % 4]
                    tr.step_device(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), B_ROWS, nnz)
                    ev[i + 1].record(stream)
                tr.sync()
                runs[arm].append(float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(args.steps)])))
                tr.close()
                t.close()
                torch.cuda.empty_cache()
        out[name] = {arm: {"ms_per_step": float(np.median(r)), "runs": r} for arm, r in runs.items()}
        out[name]["on_over_off"] = out[name]["on"]["ms_per_step"] / out[name]["off"]["ms_per_step"]
    return out


def drift(api, datagen, torch, stream, args):
    nnz = B_ROWS * NNZ
    base = [datagen.make_ids(seed=9000 + i, rows=B_ROWS, nnz_per_row=NNZ, id_space=10 ** 8, dist="zipf", zipf_s=1.05)
            for i in range(16)]
    arms = {"none": None, "idle32": dict(max_idle_batches=32), "max_keys_8M": dict(max_keys=8 << 20)}
    out = {}
    for arm, limits in arms.items():
        t = api.Table(latent_dim=0, optimizer=api.OPT_FTRL, seed=1)
        t.set_stream(stream.cuda_stream)
        if limits:
            t.set_eviction(**limits)
        tr = api.Trainer(t, model=api.MODEL_LR, max_rows=B_ROWS, max_nnz=nnz + 1024)
        step_ms, sweep_ms, losses = [], [], []
        for b in range(args.batches):
            rp, ranks, _ = base[b % 16]
            epoch = (np.uint64(b) + datagen.splitmix64(ranks) % np.uint64(32)) // np.uint64(32)
            ids = (ranks + np.uint64(10 ** 8) * epoch) % np.uint64(10 ** 9)
            first = ids[rp[:-1].astype(np.int64)]
            lab = ((datagen.splitmix64(first) % np.uint64(4)) == 0).astype(np.uint8)
            d = device_batch(api, torch, stream, rp, ids, lab)
            keys = d[1].cpu().numpy().view(np.uint64)
            p = tr.predict_host(rp, keys)  # progressive validation: before the batch is trained on
            pc = np.clip(p.astype(np.float64), 1e-7, 1 - 1e-7)
            losses.append(-(lab * np.log(pc) + (1 - lab) * np.log(1 - pc)))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            tr.step_device(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), B_ROWS, nnz)
            e1.record(stream)
            tr.sync()
            step_ms.append(e0.elapsed_time(e1))
            if limits and (b + 1) % 32 == 0:
                t0 = time.perf_counter()
                t.evict()
                sweep_ms.append((time.perf_counter() - t0) * 1e3)
        cap = t.capacity()
        out[arm] = {"keys": t.size(), "capacity": cap, "row_bytes": t.row_bytes(),
                    "table_bytes": cap * t.row_bytes(), "stamp_bytes": cap * 4 if limits else 0,
                    "ms_per_step": float(np.median(step_ms)),
                    "ms_per_sweep": float(np.median(sweep_ms)) if sweep_ms else None,
                    "sweeps": len(sweep_ms), "progressive_logloss": float(np.mean(np.concatenate(losses)))}
        tr.close()
        t.close()
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batches", type=int, default=256)
    ap.add_argument("--skip-cost", action="store_true")
    ap.add_argument("--skip-drift", action="store_true")
    args = ap.parse_args()
    import torch
    from xflow_b200 import api, datagen
    if api.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    stream = torch.cuda.Stream()
    res = {"gpu_before": gpu_info()}
    with torch.cuda.stream(stream):
        if not args.skip_cost:
            res["tracking_cost"] = tracking_cost(api, datagen, torch, stream, args)
        if not args.skip_drift:
            res["drift"] = drift(api, datagen, torch, stream, args)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

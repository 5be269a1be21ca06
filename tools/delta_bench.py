"""Serving model deltas on the benchmark's shapes (csrc/delta.cu; DESIGN.md sections 4 and 6).

    python tools/delta_bench.py [--lr-ids 100000000] [--fm-ids 20000000] [--between 1,10,100] [--warm 4]

Shapes: bench.py's headline LR (LR + FTRL, ids uniform in --lr-ids) and its skewed FM (FM K = 16 + FTRL, Zipf(1.05)
ids in --fm-ids), 65 536 rows x 100 tokens per batch.  Every id of the space is in the table
(xf_table_touch_decimal_ids), --warm batches train it, and then for each T of --between: freeze A, train T more batches,
freeze B.  For each T it reports
  - the fraction of B's keys upserted and of A's keys deleted;
  - the delta file's bytes against B's XFSM file;
  - diff, apply and fingerprint: wall time of the (synchronous) call, and the device time of their kernels from one
    torch.profiler session over the three calls (the calls run on the library's own streams, so events on a caller's
    stream cannot bracket them);
  - xf_delta_save / _load against xf_model_save / _load of B (to a temporary directory; the file system bounds them).
Every apply is checked: its result's file is byte-identical to B's.  Prints the card's name and power limit read in the
same run, then one JSON line.  Needs a CUDA device and torch; touches no device setting.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, NNZ = 65536, 100
KERNELS = dict(fingerprint="xf_k_fingerprint", diff_emit="xf_k_delta_emit", apply_base="xf_k_apply_base",
               insert_rows="xf_k_model_insert_rows", gather="xf_k_model_gather", fill="xf_k_model_fill")


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else None


def device_ms(prof):
    """summed device ms and launches of this library's kernels and of cub's sort, by kernel family"""
    out, n = {}, {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        ms = (e.device_time if hasattr(e, "device_time") else e.cuda_time) / 1e3
        fam = next((k for k, v in KERNELS.items() if v in e.name), "sort" if "Radix" in e.name or "cub" in e.name else None)
        if fam:
            out[fam] = out.get(fam, 0.0) + ms
            n[fam] = n.get(fam, 0) + 1
    return out, n


def wall(fn):
    """(result, wall ms) of one synchronous call"""
    t0 = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t0) * 1e3


def run_shape(api, datagen, torch, K, ids, dist, between, warm, tmp):
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL)
    t.reserve(ids)
    t.touch_decimal_ids(0, ids)
    tr = api.Trainer(t, model=api.MODEL_FM if K else api.MODEL_LR, max_rows=B, max_nnz=B * NNZ)
    seed = [0]

    def train(n):
        for _ in range(n):
            seed[0] += 1
            rp, raw, lab = datagen.make_ids(seed=seed[0], rows=B, nnz_per_row=NNZ, id_space=ids, dist=dist, zipf_s=1.05)
            tr.step_host(rp, api.hash_decimal_ids(raw), lab, want_loss=False)
        tr.sync()

    train(warm)
    res = dict(ids=ids, latent_dim=K, id_distribution=dist, rows=B, nnz_per_row=NNZ, warm_batches=warm, runs=[])
    a = t.freeze()
    for T in between:
        train(T)
        b = t.freeze()
        ia, ib = a.info(), b.info()
        # one profiler session over the three calls: the kernels of diff (emit, sort, gather) and of apply (fill,
        # insert, base pass) are their own; every call also runs xf_k_fingerprint, reported per pass
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fp, fp_wall = wall(a.fingerprint)
            d, diff_wall = wall(lambda: a.diff(b))
            r, apply_wall = wall(lambda: a.apply(d))
            torch.cuda.synchronize()
        dev, launches = device_ms(prof)
        di = d.info()
        mpath, dpath, rpath = (os.path.join(tmp, x) for x in ("b.xfsm", "d.xfsd", "r.xfsm"))
        _, msave = wall(lambda: b.save(mpath))
        _, dsave = wall(lambda: d.save(dpath))
        mb, mload = wall(lambda: api.Model.load(mpath))
        dl, dload = wall(lambda: api.Delta.load(dpath))
        r.save(rpath)
        with open(rpath, "rb") as f1, open(mpath, "rb") as f2:
            assert f1.read() == f2.read(), "apply(A, diff(A, B)) is not B"
        xfsm_bytes = os.path.getsize(mpath)
        assert di["file_bytes"] == os.path.getsize(dpath)
        res["runs"].append(dict(
            batches_between=T, base_keys=ia["keys"], next_keys=ib["keys"], upserts=di["upserts"], deletes=di["deletes"],
            upserted_fraction=di["upserts"] / max(ib["keys"], 1), deleted_fraction=di["deletes"] / max(ia["keys"], 1),
            delta_file_bytes=di["file_bytes"], model_file_bytes=xfsm_bytes, delta_over_model=di["file_bytes"] / xfsm_bytes,
            fingerprint_wall_ms=fp_wall, diff_wall_ms=diff_wall, apply_wall_ms=apply_wall, device_ms_by_kernel=dev,
            kernel_launches=launches,
            fingerprint_device_ms_per_pass=dev.get("fingerprint", 0.0) / max(launches.get("fingerprint", 0), 1),
            diff_device_ms=sum(dev.get(k, 0.0) for k in ("diff_emit", "sort", "gather")),
            apply_device_ms=sum(dev.get(k, 0.0) for k in ("fill", "insert_rows", "apply_base")), delta_save_ms=dsave, delta_load_ms=dload,
            model_save_ms=msave, model_load_ms=mload))
        for x in (mb, dl, d, r, a):
            x.close()
        for pth in (mpath, dpath, rpath):
            os.remove(pth)
        a = b
    a.close()
    tr.close()
    t.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lr-ids", type=int, default=10 ** 8)
    ap.add_argument("--fm-ids", type=int, default=2 * 10 ** 7)
    ap.add_argument("--between", default="1,10,100")
    ap.add_argument("--warm", type=int, default=4)
    args = ap.parse_args()
    from xflow_b200 import api, datagen
    if api.device_count() < 1:
        sys.exit("delta_bench needs a CUDA device: there is nothing to measure without one")
    import torch
    between = [int(x) for x in args.between.split(",")]
    res = dict(gpu=gpu_info())
    print("gpu:", res["gpu"], flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        res["lr_ftrl_uniform"] = run_shape(api, datagen, torch, 0, args.lr_ids, "uniform", between, args.warm, tmp)
        res["fm_k16_ftrl_zipf"] = run_shape(api, datagen, torch, 16, args.fm_ids, "zipf", between, args.warm, tmp)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

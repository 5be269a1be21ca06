"""Exact training-state checkpoints (xf_table_save_state / xf_table_load_state; DESIGN.md sections 4 and 6): how long a
save and a load of a large table take, and what bounds them.

    python tools/checkpoint_bench.py [--lr-keys 100000000] [--fm-keys 10000000] [--dir DIR] [--skip-portable]

Tables:
  lr  LR + FTRL (lazy rows), --lr-keys keys, eviction tracking on, Bloom admission with a 2^30-cell filter
  fm  FM K = 16 + FTRL, --fm-keys keys
Keys are made with xf_table_touch_decimal_ids after xf_table_reserve (no growth), then 4 training steps of 65 536 rows
x 16 tokens, so that lazy rows have steps pending and stamps differ.  Per table:
  - save_state and load_state wall time (one unprofiled run each), the file's bytes and GB/s;
  - a second, profiled run of each (torch.profiler, CUDA activities): the summed device time of the pack / unpack
    kernels (xf_k_state_*) against the summed time of the device<->host copies;
  - peak extra device memory (cudaMemGetInfo) and host memory (VmRSS) over the call, sampled every 2 ms by a thread;
  - the same table through the portable xf_table_save / xf_table_load (unless --skip-portable).
The files go to a temporary directory (--dir: its parent) and are deleted after each measurement.  Prints one JSON line
with the card's name and power limit read in the same run.  Needs a CUDA device and torch.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def rss_bytes():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) * 1024
    return 0


class Peak:
    """Peak extra device and host memory while the block runs, sampled by a thread."""

    def __init__(self, torch):
        self.torch = torch

    def __enter__(self):
        self.free0 = self.torch.cuda.mem_get_info()[0]
        self.rss0 = rss_bytes()
        self.dev = self.host = 0
        self.stop = False

        def run():
            while not self.stop:
                self.dev = max(self.dev, self.free0 - self.torch.cuda.mem_get_info()[0])
                self.host = max(self.host, rss_bytes() - self.rss0)
                time.sleep(0.002)

        self.th = threading.Thread(target=run, daemon=True)
        self.th.start()
        return self

    def __exit__(self, *a):
        self.stop = True
        self.th.join()


def profiled(torch, fn):
    """(kernel ms of xf_k_state_*, copy ms of device<->host memcpys) of one call of fn"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kern = copy = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "xf_k_state_" in e.name:
            kern += us
        elif "Memcpy DtoH" in e.name or "Memcpy HtoD" in e.name:
            copy += us
    return kern / 1e3, copy / 1e3


def build_table(api, datagen, kind, keys):
    if kind == "lr":
        t = api.Table(latent_dim=0, optimizer=api.OPT_FTRL)
        t.reserve(keys)
        t.set_eviction()
        t.set_admission(api.ADMIT_BLOOM, threshold=2, log2_cells=30, hashes=3)
        model = api.MODEL_LR
    else:
        t = api.Table(latent_dim=16, optimizer=api.OPT_FTRL)
        t.reserve(keys)
        model = api.MODEL_FM
    t.touch_decimal_ids(0, keys)
    B, d = 65536, 16
    tr = api.Trainer(t, model=model, max_rows=B, max_nnz=B * d)
    for i in range(4):
        rp, k, lab = datagen.make_csr_keys(100 + i, B, d, keys, api.hash_decimal_ids, dist="zipf")
        tr.step_host(rp, k, lab)
    tr.sync()
    return t, tr


def fresh_like(api, kind):
    if kind == "lr":
        return api.Table(latent_dim=0, optimizer=api.OPT_FTRL)
    return api.Table(latent_dim=16, optimizer=api.OPT_FTRL)


def measure(api, torch, kind, t, d, portable):
    out = dict(keys=t.size(), capacity=t.capacity(), row_bytes=t.row_bytes())
    path = os.path.join(d, "state.xfst")
    with Peak(torch) as pk:
        t0 = time.perf_counter()
        t.save_state(path)
        out["save_s"] = time.perf_counter() - t0
    out["save_peak_extra_dev_MB"], out["save_peak_extra_host_MB"] = pk.dev / 2 ** 20, pk.host / 2 ** 20
    out["file_bytes"] = os.path.getsize(path)
    out["save_GBps"] = out["file_bytes"] / out["save_s"] / 1e9
    t2 = fresh_like(api, kind)
    with Peak(torch) as pk:
        t0 = time.perf_counter()
        t2.load_state(path)
        out["load_s"] = time.perf_counter() - t0
    out["load_peak_extra_dev_MB"], out["load_peak_extra_host_MB"] = pk.dev / 2 ** 20, pk.host / 2 ** 20
    out["load_GBps"] = out["file_bytes"] / out["load_s"] / 1e9
    assert t2.size() == t.size()
    t2.close()
    os.remove(path)
    out["save_kernel_ms"], out["save_copy_ms"] = profiled(torch, lambda: t.save_state(path))
    t2 = fresh_like(api, kind)
    out["load_kernel_ms"], out["load_copy_ms"] = profiled(torch, lambda: t2.load_state(path))
    t2.close()
    os.remove(path)
    if portable:
        ppath = os.path.join(d, "portable.xftb")
        t0 = time.perf_counter()
        t.save(ppath)
        out["portable_save_s"] = time.perf_counter() - t0
        out["portable_file_bytes"] = os.path.getsize(ppath)
        t2 = fresh_like(api, kind)
        t0 = time.perf_counter()
        t2.load(ppath)
        out["portable_load_s"] = time.perf_counter() - t0
        t2.close()
        os.remove(ppath)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lr-keys", type=int, default=100_000_000)
    ap.add_argument("--fm-keys", type=int, default=10_000_000)
    ap.add_argument("--dir", default=None)
    ap.add_argument("--skip-portable", action="store_true")
    args = ap.parse_args()
    import torch
    from xflow_b200 import api, datagen
    torch.cuda.init()
    res = dict(gpu=gpu_info())
    d = tempfile.mkdtemp(prefix="xf_ckpt_", dir=args.dir)
    res["tmp_free_GB"] = shutil.disk_usage(d).free / 1e9
    try:
        for kind, keys in (("fm", args.fm_keys), ("lr", args.lr_keys)):
            t, tr = build_table(api, datagen, kind, keys)
            res[kind] = measure(api, torch, kind, t, d, not args.skip_portable)
            tr.close()
            t.close()
            print(kind, json.dumps(res[kind]), file=sys.stderr, flush=True)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Cost of the grouped test metric's finish (xf_group_metric_finish) beside xf_metric_finish on the same rows, in one
process, the two alternated.  Rows 10^6, 10^7 and 10^8 with uniform predictions and labels drawn from them; groups:
1, 10^3 and 10^6 of uniform size (ids spread over 64 bits, as hashed user ids are), and ids drawn from 10^7 with Zipf
(alpha 1.1) popularity.  Both finishes wait for their own result, so each is timed by the host clock around the call
after a device synchronise.  Prints the card's name, power limit and SM clock, then one JSON line per shape: median and
minimum ms of each finish, their ratio, the groups found, and the device memory the group metric's first finish took
(its scratch, which it keeps: the finish's peak).

    python tools/group_metric_bench.py [--rows 1e6,1e7,1e8] [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xflow_b200 import api  # noqa: E402

GOLDEN = -7046029254386353131  # 0x9E3779B97F4A7C15 as int64


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "nvidia-smi unavailable"


def groups_of(torch, n, kind):
    i = torch.arange(n, device="cuda", dtype=torch.int64)
    if kind == "zipf1e7":
        a, K = 1.1, 1e7
        u = torch.rand(n, device="cuda", dtype=torch.float64)
        k = ((K ** (1 - a) - 1) * u + 1) ** (1 / (1 - a))
        return k.floor().to(torch.int64) * GOLDEN
    return (i % int(float(kind))) * GOLDEN


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1e6,1e7,1e8")
    ap.add_argument("--groups", default="1,1e3,1e6,zipf1e7")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    L = api.lib()
    print("card: %s" % card(), flush=True)
    for rows in [int(float(r)) for r in args.rows.split(",")]:
        torch.manual_seed(rows)
        p = torch.rand(rows, device="cuda", dtype=torch.float32)
        y = (torch.rand(rows, device="cuda") < p).to(torch.uint8)
        for kind in args.groups.split(","):
            g = groups_of(torch, rows, kind)
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            gm = api.GroupMetric()
            gm.add_device(p.data_ptr(), y.data_ptr(), g.data_ptr(), rows)
            held = free0 - torch.cuda.mem_get_info()[0]
            free1 = torch.cuda.mem_get_info()[0]
            rep = gm.finish()
            scratch = free1 - torch.cuda.mem_get_info()[0]
            xm = C.c_void_p()
            assert L.xf_metric_create(C.byref(xm), 0) == 0
            assert L.xf_metric_add_device(xm, C.c_void_p(p.data_ptr()), C.c_void_p(y.data_ptr()), rows, None) == 0
            out = (C.c_double * 6)()
            st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

            def xf_metric():
                assert L.xf_metric_finish(xm, st, out) == 0

            t = {"group": [], "metric": []}
            for _ in range(2):  # warm-up
                gm.finish()
                xf_metric()
            for _ in range(args.reps):
                t["group"].append(timed(torch, gm.finish))
                t["metric"].append(timed(torch, xf_metric))
            med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
            print(json.dumps(dict(rows=rows, groups_kind=kind, groups=rep["groups"], scored_groups=rep["scored_groups"],
                                  group_finish_ms=round(med["group"], 3), group_finish_min_ms=round(min(t["group"]), 3),
                                  xf_metric_finish_ms=round(med["metric"], 3),
                                  xf_metric_min_ms=round(min(t["metric"]), 3), ratio=round(med["group"] / med["metric"], 2),
                                  held_mb=round(held / 2 ** 20, 1), finish_scratch_mb=round(scratch / 2 ** 20, 1),
                                  gauc=rep["gauc"], pooled_auc=out[5])), flush=True)
            L.xf_metric_destroy(xm)
            gm.close()
            del g
            torch.cuda.empty_cache()
    print("card: %s" % card(), flush=True)


if __name__ == "__main__":
    main()

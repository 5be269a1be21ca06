"""Cost of the grouped metric's top-k evaluation (xf_group_metric_topk) beside the finish it evaluates, on the shapes of
tools/group_metric_bench.py: rows 10^6, 10^7 and 10^8 with uniform predictions and labels drawn from them; groups 1,
10^3 and 10^6 of uniform size (ids spread over 64 bits) and ids drawn from 10^7 with Zipf (alpha 1.1) popularity.
A topk runs on the rows of the last finish, so each round is a finish, a topk at k = 10 and a topk at k = 1000, in
that order; every call waits for its own result, so each is timed by the host clock around the call after a device
synchronise.  Prints the card's name, power limit and SM clock, then one JSON line per shape: median and minimum ms
of each call, the topk / finish ratios, the groups found and the device memory the first topk added.

    python tools/group_topk_bench.py [--rows 1e6,1e7,1e8] [--reps 5]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from group_metric_bench import card, groups_of, timed  # noqa: E402
from xflow_b200 import api  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1e6,1e7,1e8")
    ap.add_argument("--groups", default="1,1e3,1e6,zipf1e7")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    print("card: %s" % card(), flush=True)
    for rows in [int(float(r)) for r in args.rows.split(",")]:
        torch.manual_seed(rows)
        p = torch.rand(rows, device="cuda", dtype=torch.float32)
        y = (torch.rand(rows, device="cuda") < p).to(torch.uint8)
        for kind in args.groups.split(","):
            g = groups_of(torch, rows, kind)
            gm = api.GroupMetric()
            gm.add_device(p.data_ptr(), y.data_ptr(), g.data_ptr(), rows)
            rep = gm.finish()
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            top = {k: gm.topk(k) for k in (10, 1000)}
            added = free0 - torch.cuda.mem_get_info()[0]
            calls = {"finish": gm.finish, "topk10": lambda: gm.topk(10), "topk1000": lambda: gm.topk(1000)}
            t = {name: [] for name in calls}
            for _ in range(2):  # warm-up
                for fn in calls.values():
                    fn()
            for _ in range(args.reps):
                for name, fn in calls.items():
                    t[name].append(timed(torch, fn))
            med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
            print(json.dumps(dict(rows=rows, groups_kind=kind, groups=rep["groups"], scored_groups=rep["scored_groups"],
                                  finish_ms=round(med["finish"], 3), finish_min_ms=round(min(t["finish"]), 3),
                                  topk10_ms=round(med["topk10"], 3), topk10_min_ms=round(min(t["topk10"]), 3),
                                  topk1000_ms=round(med["topk1000"], 3), topk1000_min_ms=round(min(t["topk1000"]), 3),
                                  ratio10=round(med["topk10"] / med["finish"], 3),
                                  ratio1000=round(med["topk1000"] / med["finish"], 3),
                                  topk_added_mb=round(added / 2 ** 20, 1), ndcg10=top[10]["ndcg"],
                                  precision10=top[10]["precision"], recall1000=top[1000]["recall"])), flush=True)
            gm.close()
            del g
            torch.cuda.empty_cache()
    print("card: %s" % card(), flush=True)


if __name__ == "__main__":
    main()

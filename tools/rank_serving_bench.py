"""Candidate ranking (xf_model_rank_candidates_*) against candidate scoring alone (DESIGN.md sections 4 and 6).

    python tools/rank_serving_bench.py [--calls 30] [--lr-ids 100000000] [--fm-ids 20000000] [--models lr,fm,...]

The models and batches of tools/candidate_serving_bench.py (lr, fm, fm16, canon, mvm; 64 context tokens, 36 per
candidate).  Shapes (R requests x N candidates each): 256 x 256, 4096 x 16, 65 536 x 1, 16 x 4096 and 1 x 65 536, each
ranked with k = 1, 16, 128 and 1024.  For each (model, shape, k), with the batch resident on the device:
  1. the bytes: rank_candidates and rank_candidates_device against the numpy model (tests/rank_model.py) over
     predict_candidates' scores, and d_pctr against them;
  2. device ms, CUDA events, alternating call by call: predict_candidates_device ("score") and rank_candidates_device
     ("rank", which scores and then selects);
  3. kernel ms per call from torch.profiler in a separate run: the scoring kernel and the two rank kernels;
  4. torch.topk on the [R, N] view of the scores, for speed only (its tie order is not the contract's);
  5. host ms: rank_candidates against predict_candidates followed by a numpy per-request selection (a stable argsort
     of each request's scores, the first k kept), which is what a caller does without ranking.
The card's name, power limit and clocks are read in the same run.  One JSON line.  Needs a CUDA device and torch;
touches no device setting.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import candidate_serving_bench as cb  # noqa: E402
from rank_model import rank_model  # noqa: E402

SHAPES = [(256, 256), (4096, 16), (65536, 1), (16, 4096), (1, 65536)]  # (R, N)
KS = [1, 16, 128, 1024]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--lr-ids", type=int, default=100_000_000)
    ap.add_argument("--fm-ids", type=int, default=20_000_000)
    ap.add_argument("--models", default="lr,fm,fm16,canon,mvm")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from xflow_b200 import api

    def dev(x):
        if x is None:
            return None
        if x.dtype == np.uint64:
            x = x.view(np.int64)
        elif x.dtype == np.uint32:
            x = x.view(np.int32)
        return torch.from_numpy(np.ascontiguousarray(x)).cuda()

    def ad(t):
        return 0 if t is None else t.data_ptr()

    def median_ms(fns, st, calls):
        ev = {k: [] for k in fns}
        for _ in range(3):
            for fn in fns.values():
                fn()
        for _ in range(calls):
            for key, fn in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                fn()
                e1.record(st)
                e1.synchronize()
                ev[key].append(e0.elapsed_time(e1))
        return {k: float(np.median(v)) for k, v in ev.items()}

    result = {"gpu": cb.gpu_info(), "n_c": cb.N_C, "n_k": cb.N_K, "models": {}}
    all_equal = True
    for name in a.models.split(","):
        t, m, keys, zipf = cb.build_model(api, name, a)
        rows = {}
        for R, N in SHAPES:
            b, _ = cb.make_batch(name, keys, zipf, R, N, seed=R + N)
            db = {k: dev(v) for k, v in b.items()}
            st = torch.cuda.current_stream()
            scores = m.predict_candidates(b["ctx_ptr"], b["ctx_keys"], b["cand_ptr"], b["row_ptr"], b["keys"],
                                          ctx_vals=b["ctx_vals"], vals=b["vals"], ctx_fields=b["ctx_fields"],
                                          fields=b["fields"])
            out_s = torch.empty(R * N, dtype=torch.float32, device="cuda")
            out_r = torch.empty(R * N, dtype=torch.float32, device="cuda")
            for k in KS:
                top_i = torch.empty(R * k, dtype=torch.int32, device="cuda")
                top_p = torch.empty(R * k, dtype=torch.float32, device="cuda")

                def score():
                    m.predict_candidates_device(R, ad(db["ctx_ptr"]), ad(db["ctx_keys"]), b["ctx_keys"].size,
                                                ad(db["cand_ptr"]), R * N, ad(db["row_ptr"]), ad(db["keys"]),
                                                b["keys"].size, out_s.data_ptr(), stream=st.cuda_stream,
                                                d_ctx_vals=ad(db["ctx_vals"]), d_vals=ad(db["vals"]),
                                                d_ctx_fields=ad(db["ctx_fields"]), d_fields=ad(db["fields"]))

                def rank():
                    m.rank_candidates_device(R, ad(db["ctx_ptr"]), ad(db["ctx_keys"]), b["ctx_keys"].size,
                                             ad(db["cand_ptr"]), R * N, ad(db["row_ptr"]), ad(db["keys"]),
                                             b["keys"].size, k, out_r.data_ptr(), top_i.data_ptr(), top_p.data_ptr(),
                                             stream=st.cuda_stream, d_ctx_vals=ad(db["ctx_vals"]),
                                             d_vals=ad(db["vals"]), d_ctx_fields=ad(db["ctx_fields"]),
                                             d_fields=ad(db["fields"]))

                def topk():
                    out_s.view(R, N).topk(min(k, N), dim=1)

                def rank_host():
                    return m.rank_candidates(b["ctx_ptr"], b["ctx_keys"], b["cand_ptr"], b["row_ptr"], b["keys"], k,
                                             ctx_vals=b["ctx_vals"], vals=b["vals"], ctx_fields=b["ctx_fields"],
                                             fields=b["fields"])

                def select_host():
                    s = m.predict_candidates(b["ctx_ptr"], b["ctx_keys"], b["cand_ptr"], b["row_ptr"], b["keys"],
                                             ctx_vals=b["ctx_vals"], vals=b["vals"], ctx_fields=b["ctx_fields"],
                                             fields=b["fields"])
                    idx = np.argsort(-s.reshape(R, N), axis=1, kind="stable")[:, :k]
                    return idx, np.take_along_axis(s.reshape(R, N), idx, 1)

                # 1. the bytes
                want_i, want_p = rank_model(scores, b["cand_ptr"], k)
                got_i, got_p = rank_host()
                score()
                rank()
                torch.cuda.synchronize()
                dev_i = top_i.cpu().numpy().view(np.uint32).reshape(R, k)
                dev_p = top_p.cpu().numpy().reshape(R, k)
                equal = bool(np.array_equal(got_i, want_i) and np.array_equal(dev_i, want_i)
                             and np.array_equal(got_p.view(np.uint32), want_p.view(np.uint32))
                             and np.array_equal(dev_p.view(np.uint32), want_p.view(np.uint32))
                             and np.array_equal(out_r.cpu().numpy().view(np.uint32), scores.view(np.uint32)))
                all_equal &= equal
                # 2. and 4. device ms
                d_ms = median_ms({"score": score, "rank": rank, "topk": topk}, st, a.calls)
                # 5. host ms
                hs = {"rank": [], "score_select": []}
                for _ in range(max(a.calls // 4, 3)):
                    for key, fn in (("rank", rank_host), ("score_select", select_host)):
                        t0 = time.perf_counter()
                        fn()
                        hs[key].append((time.perf_counter() - t0) * 1e3)
                # 3. kernel ms, in a run of its own
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(10):
                        rank()
                    torch.cuda.synchronize()
                kern = {"score": 0.0, "rank_warp": 0.0, "rank_cta": 0.0}
                for e in prof.events():
                    if e.device_type.name != "CUDA":
                        continue
                    ms = (e.device_time if hasattr(e, "device_time") else e.cuda_time) / 1e3 / 10
                    if "xf_k_serve_cand" in e.name:
                        kern["score"] += ms
                    elif "xf_k_rank_warp" in e.name:
                        kern["rank_warp"] += ms
                    elif "xf_k_rank_cta" in e.name:
                        kern["rank_cta"] += ms
                r = {"bits_equal": equal, "device_ms": d_ms,
                     "host_ms": {key: float(np.median(v)) for key, v in hs.items()}, "kernel_ms": kern,
                     "rank_share_of_score_kernel": (kern["rank_warp"] + kern["rank_cta"]) / max(kern["score"], 1e-9),
                     "d2h_bytes": {"rank": R * k * 8, "score_select": R * N * 4}}
                rows["R%d_N%d_k%d" % (R, N, k)] = r
                print(name, "R=%d N=%d k=%d" % (R, N, k), json.dumps(r), file=sys.stderr, flush=True)
                del top_i, top_p
            del db, out_s, out_r
        result["models"][name] = rows
        m.close()
        t.close()
        torch.cuda.empty_cache()
    result["bits_equal"] = all_equal
    result["gpu_after"] = cb.gpu_info()
    print(json.dumps(result))
    if not all_equal:
        raise SystemExit("a ranking differs from the numpy model")


if __name__ == "__main__":
    main()

"""Candidate scoring (xf_model_predict_candidates_*) against the flat predict of the concatenated rows (DESIGN.md
sections 4 and 6).

    python tools/candidate_serving_bench.py [--calls 40] [--lr-ids 100000000] [--fm-ids 20000000] [--models lr,fm,...]

Models, their rows imported (no training: the scores only have to be real lookups):
  lr       LR + FTRL over --lr-ids keys, every key present in the model
  fm       FM K = 16 over --fm-ids keys, F32, queries Zipf(1.05) over the keys
  fm16     the same model converted to F16
  canon    canonical FM K = 16 over --fm-ids / 4 keys, feature values in [-1, 2)
  mvm      multi-view machine K = 16 over --fm-ids / 4 keys, 8 fields, feature values
Shapes (64 context tokens, 36 per candidate, 65 536 candidates per call): R = 256 requests x N = 256 candidates,
R = 4096 x N = 16, R = 65 536 x N = 1.  For each (model, shape) the batch is made resident on the device; first both
paths must give the same bits; then, alternating call by call:
  flat   Model.predict_device(_values / _fields) on the concatenated rows (65 536 x 100 tokens)
  cand   Model.predict_candidates_device on the request form
with CUDA events around each call; the host entry points (predict_host* on the concatenated rows, predict_candidates)
are timed the same way with perf_counter, uploads included.  Kernel ms per call comes from torch.profiler in a
separate run.  Lookups per candidate and H2D bytes per call are computed from the shape (XF_CAND_RUN = 16).  The card's
name, power limit and clocks are read in the same run.  One JSON line.  Needs a CUDA device and torch; touches no device
setting.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RUN = 16
N_C, N_K, CANDS = 64, 36, 65536
SHAPES = [(256, 256), (4096, 16), (65536, 1)]  # (R, N)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else None


def keys_for(n, salt):
    """n distinct keys below 2^64 - 1 (an odd-multiplier bijection of 1 .. n)"""
    x = (np.arange(1, n + 1, dtype=np.uint64) + np.uint64(salt << 40)) * np.uint64(0x9E3779B97F4A7C15)
    return x ^ (x >> np.uint64(29))


def zipf_index(rng, n, size, s=1.05):
    r = rng.zipf(s + 0.0, size) - 1
    return np.where(r < n, r, rng.integers(0, n, size)).astype(np.int64)


def build_model(api, name, a):
    rng = np.random.default_rng(5)
    if name == "lr":
        n = a.lr_ids
        keys = keys_for(n, 1)
        t = api.Table(optimizer=api.OPT_FTRL, capacity=1 << int(np.ceil(np.log2(2 * n))))
        for i in range(0, n, 1 << 24):
            k = keys[i:i + (1 << 24)]
            t.import_(k, w=rng.normal(0, 0.3, k.size).astype(np.float32))
        return t, t.freeze(prune=False), keys, False
    K = 16
    n = a.fm_ids if name in ("fm", "fm16") else a.fm_ids // 4
    keys = keys_for(n, 2)
    canonical = name in ("canon", "mvm")
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=3,
                  capacity=1 << int(np.ceil(np.log2(2 * n))), canonical_fm=1 if canonical else 0)
    for i in range(0, n, 1 << 22):
        k = keys[i:i + (1 << 22)]
        w = np.zeros(k.size, np.float32) if name == "mvm" else rng.normal(0, 0.3, k.size).astype(np.float32)
        t.import_(k, w=w, v=rng.normal(0, 0.3 if name == "mvm" else 0.1, (k.size, K)).astype(np.float32))
    m = t.freeze_mvm() if name == "mvm" else t.freeze_canonical() if name == "canon" else t.freeze()
    if name == "fm16":
        h = m.convert(api.PRECISION_F16)
        m.close()
        m = h
    return t, m, keys, True


def make_batch(name, keys, zipf, R, N, seed):
    rng = np.random.default_rng(seed)
    pick = (lambda n: zipf_index(rng, keys.size, n)) if zipf else (lambda n: rng.integers(0, keys.size, n))
    b = dict(ctx_ptr=(np.arange(R + 1) * N_C).astype(np.uint32), cand_ptr=(np.arange(R + 1) * N).astype(np.uint32),
             row_ptr=(np.arange(R * N + 1) * N_K).astype(np.uint32))
    b["ctx_keys"] = keys[pick(R * N_C)]
    b["keys"] = keys[pick(R * N * N_K)]
    valued = name in ("canon", "mvm")
    b["ctx_vals"] = rng.uniform(-1, 2, R * N_C).astype(np.float32) if valued else None
    b["vals"] = rng.uniform(-1, 2, R * N * N_K).astype(np.float32) if valued else None
    b["ctx_fields"] = rng.integers(0, 4, R * N_C).astype(np.uint8) if name == "mvm" else None
    b["fields"] = rng.integers(4, 8, R * N * N_K).astype(np.uint8) if name == "mvm" else None
    # the concatenated rows
    req = np.repeat(np.arange(R), N)
    ctx = b["ctx_keys"].reshape(R, N_C)[req]
    own = b["keys"].reshape(R * N, N_K)
    f = dict(row_ptr=(np.arange(R * N + 1) * (N_C + N_K)).astype(np.uint32),
             keys=np.ascontiguousarray(np.concatenate([ctx, own], 1)).ravel())
    f["vals"] = None if not valued else np.concatenate([b["ctx_vals"].reshape(R, N_C)[req],
                                                        b["vals"].reshape(R * N, N_K)], 1).ravel()
    f["fields"] = None if name != "mvm" else np.concatenate([b["ctx_fields"].reshape(R, N_C)[req],
                                                             b["fields"].reshape(R * N, N_K)], 1).ravel()
    return b, f


def h2d_bytes(arrays):
    return int(sum(x.nbytes for x in arrays if x is not None))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
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

    result = {"gpu": gpu_info(), "run": RUN, "n_c": N_C, "n_k": N_K, "candidates_per_call": CANDS, "models": {}}
    for name in a.models.split(","):
        t, m, keys, zipf = build_model(api, name, a)
        rows = {}
        for R, N in SHAPES:
            b, f = make_batch(name, keys, zipf, R, N, seed=R)
            db = {k: dev(v) for k, v in b.items()}
            df = {k: dev(v) for k, v in f.items()}
            out_f = torch.empty(R * N, dtype=torch.float32, device="cuda")
            out_c = torch.empty(R * N, dtype=torch.float32, device="cuda")
            st = torch.cuda.current_stream()

            def flat():
                if name == "mvm":
                    m.predict_device_fields(ad(df["row_ptr"]), ad(df["keys"]), ad(df["fields"]), R * N, f["keys"].size,
                                            out_f.data_ptr(), stream=st.cuda_stream, d_vals=ad(df["vals"]))
                else:
                    m.predict_device(ad(df["row_ptr"]), ad(df["keys"]), R * N, f["keys"].size, out_f.data_ptr(),
                                     stream=st.cuda_stream, d_vals=ad(df["vals"]))

            def cand():
                m.predict_candidates_device(R, ad(db["ctx_ptr"]), ad(db["ctx_keys"]), b["ctx_keys"].size,
                                            ad(db["cand_ptr"]), R * N, ad(db["row_ptr"]), ad(db["keys"]), b["keys"].size,
                                            out_c.data_ptr(), stream=st.cuda_stream, d_ctx_vals=ad(db["ctx_vals"]),
                                            d_vals=ad(db["vals"]), d_ctx_fields=ad(db["ctx_fields"]),
                                            d_fields=ad(db["fields"]))

            def flat_host():
                if name == "mvm":
                    return m.predict_host_fields(f["row_ptr"], f["keys"], f["fields"], f["vals"])
                return m.predict_host(f["row_ptr"], f["keys"], f["vals"])

            def cand_host():
                return m.predict_candidates(b["ctx_ptr"], b["ctx_keys"], b["cand_ptr"], b["row_ptr"], b["keys"],
                                            ctx_vals=b["ctx_vals"], vals=b["vals"], ctx_fields=b["ctx_fields"],
                                            fields=b["fields"])

            flat()
            cand()
            torch.cuda.synchronize()
            same = bool(np.array_equal(out_f.cpu().numpy().view(np.uint32), out_c.cpu().numpy().view(np.uint32)))
            same_host = bool(np.array_equal(flat_host().view(np.uint32), cand_host().view(np.uint32)))
            if not (same and same_host):
                raise SystemExit("%s R=%d N=%d: the candidate path differs from the flat predict" % (name, R, N))
            ev = {"flat": [], "cand": []}
            hs = {"flat": [], "cand": []}
            for _ in range(3):
                flat()
                cand()
            for _ in range(a.calls):
                for key, fn in (("flat", flat), ("cand", cand)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    fn()
                    e1.record(st)
                    e1.synchronize()
                    ev[key].append(e0.elapsed_time(e1))
            for _ in range(max(a.calls // 4, 3)):
                for key, fn in (("flat", flat_host), ("cand", cand_host)):
                    t0 = time.perf_counter()
                    fn()
                    hs[key].append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    flat()
                    cand()
                torch.cuda.synchronize()
            kf = kc = 0.0
            nf = nc = 0
            for e in prof.events():
                if e.device_type.name != "CUDA" or "xf_k_serve" not in e.name:
                    continue
                ms = (e.device_time if hasattr(e, "device_time") else e.cuda_time) / 1e3
                if "_cand" in e.name:
                    kc, nc = kc + ms, nc + 1
                else:
                    kf, nf = kf + ms, nf + 1
            runs = R * -(-N // RUN)
            rows["R%d_N%d" % (R, N)] = {
                "bits_equal": same and same_host,
                "device_ms": {k: float(np.median(v)) for k, v in ev.items()},
                "host_ms": {k: float(np.median(v)) for k, v in hs.items()},
                "kernel_ms": {"flat": kf / max(nf, 1), "cand": kc / max(nc, 1)},
                "lookups_per_candidate": {"flat": N_C + N_K, "cand": (runs * N_C + R * N * N_K) / (R * N)},
                "h2d_bytes": {"flat": h2d_bytes(f.values()), "cand": h2d_bytes(b.values())},
            }
            r = rows["R%d_N%d" % (R, N)]
            r["speedup_device"] = r["device_ms"]["flat"] / r["device_ms"]["cand"]
            r["speedup_kernel"] = r["kernel_ms"]["flat"] / max(r["kernel_ms"]["cand"], 1e-9)
            r["speedup_host"] = r["host_ms"]["flat"] / r["host_ms"]["cand"]
            print(name, "R=%d N=%d" % (R, N), json.dumps(r), file=sys.stderr, flush=True)
            del db, df, out_f, out_c
        result["models"][name] = rows
        m.close()
        t.close()
        torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()

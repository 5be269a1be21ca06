"""Field-aware FM serving model against the FFM table's own predict and a canonical model (DESIGN.md section 6).

    python tools/ffm_serving_bench.py [--dims 16,32,64,128] [--ids 2000000] [--calls 50] [--out ffm_serving.json]

Flat predict.  For each L in --dims: a canonical table (canonical_fm = 1, FTRL) trained by XF_MODEL_FFM on two
batches, whose trained keys then get w and v of N(0, 0.5).  The query batch is 65 536 rows of one token per field
(F = L / 4 tokens), Zipf(1.05) ids in --ids, random values; it is resident on the device.  Timed, alternating call by
call after a warm-up, with CUDA events around each call:
  model     Model.predict_device_fields (xf_k_serve_ffm) of xf_table_freeze_ffm, at F32 and at F16;
  canonical Model.predict_device_values (xf_k_serve_fmc) of xf_table_freeze_canonical of the same table, same keys;
  table     the trainer's FFM predict kernel (xf_k_step_ffm, mode 1) on the same batch: the trainer has no device
            pointer entry point, so its kernel time comes from torch.profiler in the same run.
Candidates.  At each L, 1 024 requests of 64 candidates, 8 context tokens and 8 candidate tokens each: score
(predict_candidates_device), rank top 16 (rank_candidates_device), and the flat predict of the 65 536 concatenated rows
of 16 tokens.  The scores are checked bit for bit against that flat predict, and the F32 model against the table.
Prints one JSON line with ms per call (median over --calls) and the card's name, power limit and SM clock, read in the
same run.  Needs a CUDA device and torch; touches no device setting.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROWS, REQ, CANDS, CTX, CTOK, TOPK = 65536, 1024, 64, 8, 8, 16


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()
    return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")])) if out else None


def timed(torch, fns, calls):
    """Median ms per call of each fn, alternating fn by fn, CUDA events around each call."""
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    ms = {k: [] for k in fns}
    for _ in range(calls):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    return {k: round(float(np.median(v)), 4) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", default="16,32,64,128")
    ap.add_argument("--ids", type=int, default=2000000)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from xflow_b200 import api, datagen
    if api.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(
        {1: np.uint8, 4: np.int32, 8: np.int64}[np.asarray(a).dtype.itemsize])).cuda()
    res = {"rows": ROWS, "requests": REQ, "candidates_per_request": CANDS, "dims": {}}
    for L in [int(x) for x in args.dims.split(",")]:
        F = L // 4
        t = api.Table(latent_dim=L, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=7, capacity=1 << 22,
                      canonical_fm=1)
        tr = api.Trainer(t, model=api.MODEL_FFM, max_rows=ROWS, max_nnz=ROWS * max(F, 16))
        rng = np.random.default_rng(L)
        seen = []
        for s in range(2):
            rp, ids, lab = datagen.make_ids(s, ROWS, F, args.ids, dist="zipf", zipf_s=1.05)
            keys = api.hash_decimal_ids(ids)
            tr.step_host_fields(rp, keys, np.tile(np.arange(F, dtype=np.uint8), ROWS),
                                rng.uniform(-1, 2, keys.size).astype(np.float32), lab)
            seen.append(keys)
        trained = np.unique(np.concatenate(seen))
        t.import_(trained, w=rng.normal(0, 0.5, trained.size).astype(np.float32),
                  v=rng.normal(0, 0.5, (trained.size, L)).astype(np.float32))
        rp, ids, _ = datagen.make_ids(9, ROWS, F, args.ids, dist="zipf", zipf_s=1.05)
        keys = api.hash_decimal_ids(ids)
        f = np.tile(np.arange(F, dtype=np.uint8), ROWS)
        x = rng.uniform(-1, 2, keys.size).astype(np.float32)
        want = tr.predict_host_fields(rp, keys, f, x)  # inserts the unseen keys: every path holds them from here on
        m, mc = t.freeze_ffm(), t.freeze_canonical()
        h16 = m.convert(api.PRECISION_F16)
        d_rp, d_k, d_f, d_x = dev(rp.astype(np.int32)), dev(keys), dev(f), dev(x)
        out = torch.empty(ROWS, dtype=torch.float32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        call = lambda mm: (lambda: mm.predict_device_fields(d_rp.data_ptr(), d_k.data_ptr(), d_f.data_ptr(), ROWS,
                                                            keys.size, out.data_ptr(), stream=st, d_vals=d_x.data_ptr()))
        call(m)()
        torch.cuda.synchronize()
        exact = bool(np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)))
        flat = timed(torch, {"ffm_f32": call(m), "ffm_f16": call(h16),
                             "canonical_f32": lambda: mc.predict_device(
                                 d_rp.data_ptr(), d_k.data_ptr(), ROWS, keys.size, out.data_ptr(), stream=st,
                                 d_vals=d_x.data_ptr())}, args.calls)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                tr.predict_host_fields(rp, keys, f, x)
            torch.cuda.synchronize()
        ks = [e for e in prof.events() if e.device_type.name == "CUDA" and "xf_k_step_ffm" in e.name]
        flat["table_kernel"] = round(sum(getattr(e, "device_time", 0) or e.cuda_time for e in ks) / 1e3 / max(len(ks), 1), 4)
        # candidates: 8 context tokens, 8 per candidate, field ids shared between the sides
        ckeys = np.resize(keys, REQ * CTX + REQ * CANDS * CTOK)  # the query's keys, repeated where they run short
        cvals = np.resize(x, ckeys.size)
        ck, ci = ckeys[:REQ * CTX], ckeys[REQ * CTX:]
        cf, nf = (np.arange(REQ * CTX) % F).astype(np.uint8), ((np.arange(REQ * CANDS * CTOK) * 3) % F).astype(np.uint8)
        cx, nx = cvals[:ck.size], cvals[ck.size:]
        ctx_ptr = (np.arange(REQ + 1) * CTX).astype(np.uint32)
        cand_ptr = (np.arange(REQ + 1) * CANDS).astype(np.uint32)
        row_ptr = (np.arange(REQ * CANDS + 1) * CTOK).astype(np.uint32)
        N = REQ * CANDS
        d = [dev(a) for a in (ctx_ptr, ck, cand_ptr, row_ptr, ci, cx, nx, cf, nf)]
        cat = np.concatenate([np.concatenate([ck[(c // CANDS) * CTX:(c // CANDS + 1) * CTX], ci[c * CTOK:(c + 1) * CTOK]])
                              for c in range(N)])
        catf = np.concatenate([np.concatenate([cf[(c // CANDS) * CTX:(c // CANDS + 1) * CTX], nf[c * CTOK:(c + 1) * CTOK]])
                               for c in range(N)])
        catx = np.concatenate([np.concatenate([cx[(c // CANDS) * CTX:(c // CANDS + 1) * CTX], nx[c * CTOK:(c + 1) * CTOK]])
                               for c in range(N)])
        crp = (np.arange(N + 1) * (CTX + CTOK)).astype(np.uint32)
        dc = [dev(a) for a in (crp.astype(np.int32), cat, catf, catx)]
        sc = torch.empty(N, dtype=torch.float32, device="cuda")
        fo = torch.empty(N, dtype=torch.float32, device="cuda")
        ti = torch.empty(REQ * TOPK, dtype=torch.int32, device="cuda")
        tp = torch.empty(REQ * TOPK, dtype=torch.float32, device="cuda")
        kw = lambda: dict(stream=st, d_ctx_vals=d[5].data_ptr(), d_vals=d[6].data_ptr(), d_ctx_fields=d[7].data_ptr(),
                          d_fields=d[8].data_ptr())
        pos = lambda: (REQ, d[0].data_ptr(), d[1].data_ptr(), ck.size, d[2].data_ptr(), N, d[3].data_ptr(),
                       d[4].data_ptr(), ci.size)
        cands = {}
        for name, mm in (("f32", m), ("f16", h16)):
            score = lambda mm=mm: mm.predict_candidates_device(*pos(), sc.data_ptr(), **kw())
            rank = lambda mm=mm: mm.rank_candidates_device(*pos(), TOPK, sc.data_ptr(), ti.data_ptr(), tp.data_ptr(), **kw())
            flatc = lambda mm=mm: mm.predict_device_fields(dc[0].data_ptr(), dc[1].data_ptr(), dc[2].data_ptr(), N,
                                                           cat.size, fo.data_ptr(), stream=st, d_vals=dc[3].data_ptr())
            score()
            flatc()
            torch.cuda.synchronize()
            same = bool(torch.equal(sc.view(torch.int32), fo.view(torch.int32)))
            tm = timed(torch, {"score": score, "rank_top16": rank, "flat_concatenated": flatc}, args.calls)
            tm["bit_exact_vs_flat"] = same
            cands[name] = tm
        res["dims"][L] = {"flat_ms": flat, "model_equals_table": exact, "candidates_ms": cands,
                          "model_keys": m.info()["keys"], "row_bytes": m.info()["row_bytes"]}
        for o in (m, mc, h16):
            o.close()
        tr.close()
        t.close()
        print(json.dumps({"L": L, **res["dims"][L]}), flush=True)
    res["gpu"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

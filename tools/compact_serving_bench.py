"""F16 against F32 serving models on the same table (xf_model_convert; DESIGN.md sections 4 and 6).

    python tools/compact_serving_bench.py [--fm-ids 20000000] [--canonical-ids 20000000] [--dims 16,64] [--calls 104]
                                          [--train-steps 4]

Shapes: tools/serving_bench.py's FM (FM K = 16 + FTRL, every id of --fm-ids in the table, Zipf(1.05) batches) and
tools/canonical_serving_bench.py's canonical FM (FTRL, K from --dims, Zipf(1.05) ids in --canonical-ids, feature values
in [-1, 2); the table grows with its keys instead of being reserved for every id), each trained on --train-steps batches of 65 536 rows x 100 tokens.  The table is frozen with prune = 0 (every
key kept) and converted to F16.  Then, in one process, alternating the two models call by call over 8 query batches
resident on the device: Model.predict_device on one stream, CUDA events around each call, and torch.profiler's kernel time
of each model's predict kernel in the same run.  Also: model bytes (device) and XFSM file bytes of both models, the
conversion's wall time (median of 3, it ends in a synchronise), the largest |pctr(F16) - pctr(F32)| over the query
batches, and the XFSD file bytes of the deltas between the freeze above and freezes T = 1 and T = 10 training batches
later, at each precision.  Prints the card's name and power limit read in the same run, and one JSON line.  Needs a
CUDA device and torch; touches no device setting; writes only to a temporary directory.
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

B, NNZ, RING = 65536, 100, 8


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else None


def kernel_ms(prof, needle, half):
    """(summed device ms, launches) of the predict kernels named `needle` of one precision (template argument H)"""
    tag = ", true>" if half else ", false>"
    tot, n = 0.0, 0
    for e in prof.events():
        if e.device_type.name == "CUDA" and needle in e.name and tag in e.name:
            tot += (e.device_time if hasattr(e, "device_time") else e.cuda_time) / 1e3
            n += 1
    return tot, n


def batch(api, datagen, seed, ids, canonical):
    rp, raw, lab = datagen.make_ids(seed=seed, rows=B, nnz_per_row=NNZ, id_space=ids, dist="zipf", zipf_s=1.05)
    vals = np.random.default_rng(seed).uniform(-1.0, 2.0, raw.size).astype(np.float32) if canonical else None
    return rp, api.hash_decimal_ids(raw), vals, lab


def run_shape(api, datagen, torch, K, ids, canonical, calls, train_steps, tmp):
    if canonical:
        # no reserve: at K = 64 a table sized for every id (73 GB) leaves no room for the four models measured here;
        # the table's capacity does not enter the models, which are sized by their own keys
        t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, canonical_fm=1, v_init=api.VINIT_COUNTER, seed=3)
        tr = api.Trainer(t, model=api.MODEL_FM_CANONICAL, max_rows=B, max_nnz=B * NNZ)
    else:
        t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL)
        t.reserve(ids)
        t.touch_decimal_ids(0, ids)
        tr = api.Trainer(t, model=api.MODEL_FM, max_rows=B, max_nnz=B * NNZ)

    def train(seed):
        rp, keys, vals, lab = batch(api, datagen, seed, ids, canonical)
        if canonical:
            tr.step_host_values(rp, keys, vals, lab)
        else:
            tr.step_host(rp, keys, lab, want_loss=False)

    for i in range(train_steps):
        train(1 + i)
    tr.sync()
    freeze = (lambda: t.freeze_canonical(prune=False)) if canonical else (lambda: t.freeze(prune=False))
    m32 = freeze()
    conv = []
    for _ in range(3):
        t0 = time.perf_counter()
        m16 = m32.convert(api.PRECISION_F16)
        conv.append(time.perf_counter() - t0)
        if len(conv) < 3:
            m16.close()
    models = {"f32": m32, "f16": m16}
    host, dev = [], []
    for i in range(RING):
        rp, keys, vals, _ = batch(api, datagen, 1000 + i, ids, canonical)
        host.append((rp, keys, vals))
        dev.append(tuple(torch.from_numpy(a.view(np.uint8)).cuda() if a is not None else None for a in (rp, keys, vals)))
    out = torch.empty(B, dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()

    def serve(m, i):
        d_rp, d_keys, d_vals = dev[i % RING]
        m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), B, B * NNZ, out.data_ptr(), stream=stream.cuda_stream,
                         d_vals=d_vals.data_ptr() if d_vals is not None else 0)

    # the F16 model's predictions against the F32 model's, on every query batch (also the warm-up)
    dmax = 0.0
    for i in range(RING):
        got = {}
        for k, m in models.items():
            serve(m, i)
            stream.synchronize()
            got[k] = out.cpu().numpy().astype(np.float64)
        dmax = max(dmax, float(np.max(np.abs(got["f16"] - got["f32"]))))
    ev = {k: 0.0 for k in models}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            for k, m in models.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                serve(m, i)
                b.record(stream)
                b.synchronize()
                ev[k] += a.elapsed_time(b)
        torch.cuda.synchronize()
    needle = "xf_k_serve_fmc" if canonical else "xf_k_serve"
    res = dict(latent_dim=K, kind="canonical" if canonical else "fm", optimizer="ftrl", ids=ids, id_distribution="zipf(1.05)",
               rows=B, nnz_per_row=NNZ, calls=calls, train_steps=train_steps, keys=m32.info()["keys"],
               convert_wall_ms_median_of_3=sorted(conv)[1] * 1e3, max_abs_dpctr_f16_vs_f32=dmax)
    for k, m in models.items():
        kms, kn = kernel_ms(prof, needle, k == "f16")
        assert calls - 2 <= kn <= calls, (k, kn)  # the profiler may miss a launch at the start of its window
        path = os.path.join(tmp, "model_" + k)
        m.save(path)
        i = m.info()
        res[k] = dict(event_ms_per_call=ev[k] / calls, kernel_ms_per_call=kms / kn, kernel_launches_profiled=kn,
                      examples_per_s=B / (ev[k] / calls / 1e3), row_bytes=i["row_bytes"], model_bytes=i["bytes"],
                      xfsm_file_bytes=os.path.getsize(path))
        os.remove(path)
    # deltas: the freeze above against freezes T = 1 and T = 10 training batches later, at each precision
    done = 0
    for T in (1, 10):
        while done < T:
            train(5000 + done)
            done += 1
        tr.sync()
        mb = freeze()
        mb16 = mb.convert(api.PRECISION_F16)
        for k, (a, b) in dict(f32=(m32, mb), f16=(m16, mb16)).items():
            d = a.diff(b)
            res[k]["delta_file_bytes_T%d" % T] = d.info()["file_bytes"]
            res[k]["delta_upserts_T%d" % T] = d.info()["upserts"]
            d.close()
        mb16.close()
        mb.close()
    for m in models.values():
        m.close()
    tr.close()
    t.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fm-ids", type=int, default=2 * 10 ** 7)
    ap.add_argument("--canonical-ids", type=int, default=2 * 10 ** 7)
    ap.add_argument("--dims", default="16,64")
    ap.add_argument("--calls", type=int, default=104)
    ap.add_argument("--train-steps", type=int, default=4)
    args = ap.parse_args()
    from xflow_b200 import api, datagen
    if api.device_count() < 1:
        sys.exit("compact_serving_bench needs a CUDA device: there is nothing to measure without one")
    import torch
    res = dict(gpu=gpu_info())
    with tempfile.TemporaryDirectory() as tmp:
        res["fm_k16_ftrl_zipf"] = run_shape(api, datagen, torch, 16, args.fm_ids, False, args.calls, args.train_steps, tmp)
        for K in (int(k) for k in args.dims.split(",")):
            res["canonical_k%d_ftrl_zipf" % K] = run_shape(api, datagen, torch, K, args.canonical_ids, True, args.calls,
                                                           args.train_steps, tmp)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

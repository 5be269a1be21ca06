"""Canonical serving model against the canonical table's own predict (DESIGN.md sections 4 and 6).

    python tools/canonical_serving_bench.py [--ids 20000000] [--calls 104] [--train-steps 4] [--dims 16,64]

Shape: a canonical FM table (canonical_fm = 1, FTRL, K from --dims) trained on --train-steps batches of 65 536 rows x 100
tokens, Zipf(1.05) ids in --ids, random feature values in [-1, 2).  The table is frozen with xf_table_freeze_canonical
twice: with the defaults (keys no batch trained are pruned) and with prune = 0.  Then 8 query batches of the same shape
are made resident on the device, the table's predict runs once over each (it inserts their unseen keys, so that both
paths hold the same keys from then on) and must equal both models bit for bit.  Then, in one process, alternating the
paths call by call:
  table   Trainer.predict_host_values (xf_k_step_fmc, mode 1).  The table has no predict on device pointers, so the call
          also copies the batch from host memory; the kernel's own time comes from torch.profiler in the same run, and
          the call's wall time is reported beside it as what it is.
  model   Model.predict_device with d_vals (xf_k_serve_fmc), CUDA events around each call, and the same profiler's
          kernel time.
Prints examples/s, algorithmic bytes per token (8 of key, 4 of value, and the row bytes the path reads: the table's
32-byte head sector and 4K of v, the model's 16-byte head and 4K of v) over kernel time against the H100 SXM data-sheet
3.35 TB/s (a data-sheet figure, not a measured peak), model and table bytes, and the card's name and power limit read in
the same run.  One JSON line.  Needs a CUDA device and torch; touches no device setting.
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

B, NNZ, RING = 65536, 100, 8
DATASHEET_BW = 3.35e12  # H100 SXM HBM3, NVIDIA data sheet


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else None


def kernel_ms(prof, needle):
    """(summed device ms, launches) of the kernels whose name contains `needle`"""
    tot, n = 0.0, 0
    for e in prof.events():
        if e.device_type.name == "CUDA" and needle in e.name:
            tot += (e.device_time if hasattr(e, "device_time") else e.cuda_time) / 1e3
            n += 1
    return tot, n


def batch(api, datagen, seed, ids):
    rp, raw, lab = datagen.make_ids(seed=seed, rows=B, nnz_per_row=NNZ, id_space=ids, dist="zipf", zipf_s=1.05)
    vals = np.random.default_rng(seed).uniform(-1.0, 2.0, raw.size).astype(np.float32)
    return rp, api.hash_decimal_ids(raw), vals, lab


def run_shape(api, datagen, torch, K, ids, calls, train_steps):
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, canonical_fm=1, v_init=api.VINIT_COUNTER, seed=3)
    t.reserve(ids)
    tr = api.Trainer(t, model=api.MODEL_FM_CANONICAL, max_rows=B, max_nnz=B * NNZ)
    for i in range(train_steps):
        tr.step_host_values(*batch(api, datagen, 1 + i, ids))
    tr.sync()
    trained_keys = t.size()
    models = dict(pruned=t.freeze_canonical(), full=t.freeze_canonical(prune=False))
    host, dev = [], []
    for i in range(RING):
        rp, keys, vals, _ = batch(api, datagen, 1000 + i, ids)
        host.append((rp, keys, vals))
        dev.append(tuple(torch.from_numpy(a.view(np.uint8)).cuda() for a in (rp, keys, vals)))
    out = torch.empty(B, dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()

    def serve(m, i):
        d_rp, d_keys, d_vals = dev[i % RING]
        m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), B, B * NNZ, out.data_ptr(), stream=stream.cuda_stream,
                         d_vals=d_vals.data_ptr())

    # the two paths agree before anything is timed; the table's first predict of a batch inserts its unseen keys,
    # which read as the model's absent keys do
    for i in range(RING):
        want = tr.predict_host_values(*host[i])
        for m in models.values():
            serve(m, i)
            stream.synchronize()
            assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), "model and table predictions differ"
    res = dict(ids=ids, latent_dim=K, optimizer="ftrl", id_distribution="zipf(1.05)", rows=B, nnz_per_row=NNZ, calls=calls,
               train_steps=train_steps, table_keys_after_training=trained_keys, table_keys_timed=t.size(),
               table_bytes=t.capacity() * t.row_bytes(), table_row_bytes=t.row_bytes())
    ev = {k: [0.0, 0] for k in models}
    wall_table = 0.0
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            t0 = time.perf_counter()
            tr.predict_host_values(*host[i % RING])
            wall_table += time.perf_counter() - t0
            for k, m in models.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                serve(m, i)
                b.record(stream)
                b.synchronize()
                ev[k][0] += a.elapsed_time(b)
                ev[k][1] += 1
        torch.cuda.synchronize()
    step_ms, step_n = kernel_ms(prof, "xf_k_step_fmc")
    serve_ms, serve_n = kernel_ms(prof, "xf_k_serve_fmc")
    tokens = B * NNZ
    table_tok = 8 + 4 + 32 + 4 * K
    model_tok = 8 + 4 + 16 + 4 * K
    res["profiler_launches"] = dict(table=step_n, model=serve_n)
    if step_n:
        res["table"] = dict(kernel_ms_per_call=step_ms / step_n, examples_per_s_kernel=B / (step_ms / step_n / 1e3),
                            wall_ms_per_call_incl_host_copy=wall_table / calls * 1e3, algorithmic_bytes_per_token=table_tok,
                            share_of_datasheet_bw=tokens * table_tok / (step_ms / step_n / 1e3) / DATASHEET_BW)
    if serve_n:
        res["model_kernel_ms_per_call_both_models"] = serve_ms / serve_n
    for k, m in models.items():
        ms = ev[k][0] / ev[k][1]
        i = m.info()
        res["model_" + k] = dict(event_ms_per_call=ms, examples_per_s=B / (ms / 1e3), algorithmic_bytes_per_token=model_tok,
                                 share_of_datasheet_bw=tokens * model_tok / (ms / 1e3) / DATASHEET_BW, model_bytes=i["bytes"],
                                 model_row_bytes=i["row_bytes"], keys=i["keys"],
                                 pruned_fraction=i["pruned_keys"] / max(i["source_keys"], 1))
        m.close()
    tr.close()
    t.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ids", type=int, default=2 * 10 ** 7)
    ap.add_argument("--calls", type=int, default=104)
    ap.add_argument("--train-steps", type=int, default=4)
    ap.add_argument("--dims", default="16,64")
    args = ap.parse_args()
    from xflow_b200 import api, datagen
    if api.device_count() < 1:
        sys.exit("canonical_serving_bench needs a CUDA device: there is nothing to measure without one")
    import torch
    res = dict(gpu=gpu_info(), datasheet_bw_bytes_per_s=DATASHEET_BW)
    for K in (int(k) for k in args.dims.split(",")):
        res["fmc_k%d_ftrl_zipf" % K] = run_shape(api, datagen, torch, K, args.ids, args.calls, args.train_steps)
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Serving model against the training table's own predict (csrc/serve.cu; DESIGN.md sections 4 and 6).

    python tools/serving_bench.py [--lr-ids 100000000] [--fm-ids 50000000] [--calls 104] [--train-steps 4]

Shapes: bench.py's headline LR (LR + FTRL, ids uniform in --lr-ids, 100 tokens per row, 65 536 rows) and its skewed FM
(FM K = 16 + FTRL, Zipf(1.05) ids in --fm-ids).  Every id of the space is in the table (xf_table_touch_decimal_ids), then
--train-steps batches train it, then the table is frozen twice: with the defaults (the untrained keys are pruned) and
with prune = 0 (every key kept: the model's rows are as many as the table's).  Then, in one process, alternating the
paths call by call over 8 distinct query batches resident on the device:
  table   Trainer.predict_host's kernel (xf_k_step* in predict mode).  The table has no predict on device pointers, so
          the call also copies the batch from host memory; the kernel's own time is taken from torch.profiler in the
          same run, the call's wall time is reported beside it as what it is.
  model   Model.predict_device (xf_k_serve), CUDA events around the calls and the same profiler's kernel time.
Prints examples/s, algorithmic bytes per token (8 of key + the row bytes the path reads) over kernel time against the
H100 SXM data-sheet 3.35 TB/s (a data-sheet figure, not a measured peak), model and table bytes, the pruned fraction,
and the card's name and power limit read in the same run.  One JSON line.  Needs a CUDA device and torch; touches no
device setting.
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


def run_shape(api, datagen, torch, name, K, ids, dist, calls, train_steps):
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL)
    t.reserve(ids)
    t.touch_decimal_ids(0, ids)
    tr = api.Trainer(t, model=api.MODEL_FM if K else api.MODEL_LR, max_rows=B, max_nnz=B * NNZ)
    host, dev = [], []
    for i in range(RING + train_steps):
        rp, raw, lab = datagen.make_ids(seed=1 + i, rows=B, nnz_per_row=NNZ, id_space=ids, dist=dist, zipf_s=1.05)
        keys = api.hash_decimal_ids(raw)
        if i < train_steps:
            tr.step_host(rp, keys, lab, want_loss=False)
            continue
        host.append((rp, keys))
        dev.append((torch.from_numpy(rp.view(np.uint8)).cuda(), torch.from_numpy(keys.view(np.uint8)).cuda()))
    tr.sync()
    models = dict(pruned=t.freeze(), full=t.freeze(prune=False))
    out = torch.empty(B, dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()

    def serve(m, i):
        d_rp, d_keys = dev[i % RING]
        m.predict_device(d_rp.data_ptr(), d_keys.data_ptr(), B, B * NNZ, out.data_ptr(), stream=stream.cuda_stream)

    # the two paths agree before anything is timed (the table's predict inserts nothing new: every id is in it)
    for i in range(RING):
        want = tr.predict_host(*host[i])
        for m in models.values():
            serve(m, i)
            stream.synchronize()
            assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), "model and table predictions differ"
    res = dict(ids=ids, latent_dim=K, id_distribution=dist, rows=B, nnz_per_row=NNZ, calls=calls,
               table_bytes=t.capacity() * t.row_bytes(), table_row_bytes=t.row_bytes())
    ev = {k: [0.0, 0] for k in models}
    wall_table = 0.0
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            t0 = time.perf_counter()
            tr.predict_host(*host[i % RING])
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
    step_ms, step_n = kernel_ms(prof, "xf_k_step")
    serve_ms, serve_n = kernel_ms(prof, "xf_k_serve")
    assert step_n == calls and serve_n == calls * len(models), (step_n, serve_n)
    # bytes a token needs: its key and the row sectors its path reads (table: head sector + FM latent row)
    table_tok = 8 + 32 + 4 * K
    model_tok = 8 + (32 if K else 16)
    tokens = B * NNZ
    res["table"] = dict(kernel_ms_per_call=step_ms / calls, examples_per_s_kernel=B / (step_ms / calls / 1e3),
                        wall_ms_per_call_incl_host_copy=wall_table / calls * 1e3, algorithmic_bytes_per_token=table_tok,
                        share_of_datasheet_bw=tokens * table_tok / (step_ms / calls / 1e3) / DATASHEET_BW)
    res["model_kernel_ms_per_call_both_models"] = serve_ms / serve_n
    for k, m in models.items():
        ms = ev[k][0] / ev[k][1]
        i = m.info()
        res["model_" + k] = dict(event_ms_per_call=ms, examples_per_s=B / (ms / 1e3), algorithmic_bytes_per_token=model_tok,
                                 share_of_datasheet_bw=tokens * model_tok / (ms / 1e3) / DATASHEET_BW, model_bytes=i["bytes"],
                                 keys=i["keys"], pruned_fraction=i["pruned_keys"] / max(i["source_keys"], 1))
        m.close()
    tr.close()
    t.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lr-ids", type=int, default=10 ** 8)
    ap.add_argument("--fm-ids", type=int, default=5 * 10 ** 7)
    ap.add_argument("--calls", type=int, default=104)
    ap.add_argument("--train-steps", type=int, default=4)
    args = ap.parse_args()
    from xflow_b200 import api, datagen
    if api.device_count() < 1:
        sys.exit("serving_bench needs a CUDA device: there is nothing to measure without one")
    import torch
    res = dict(gpu=gpu_info(), datasheet_bw_bytes_per_s=DATASHEET_BW)
    res["lr_ftrl_uniform"] = run_shape(api, datagen, torch, "lr", 0, args.lr_ids, "uniform", args.calls, args.train_steps)
    res["fm_k16_ftrl_zipf"] = run_shape(api, datagen, torch, "fm", 16, args.fm_ids, "zipf", args.calls, args.train_steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

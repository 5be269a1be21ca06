"""Multi-view machine serving model against the MVM table's own predict (DESIGN.md sections 4 and 6).

    python tools/mvm_serving_bench.py [--ids 20000000] [--calls 104] [--train-steps 4] [--dims 16,32]

Shape: a canonical table (canonical_fm = 1, FTRL, K from --dims) trained by the multi-view machine on --train-steps
batches of 65 536 rows x 100 tokens, Zipf(1.05) ids in --ids, field ids uniform over 8 views, random feature values in
[-1, 2).  The trained keys then get latent rows of N(0, 0.25), so that
predictions do not all round to sigmoid(0).  The table is frozen with xf_table_freeze_mvm twice, with the defaults (keys no batch trained are pruned) and
with prune = 0, and the pruned model is converted to F16.  Then 8 query batches of the same shape are made resident on
the device, and the table's predict runs once over each (it inserts their unseen keys, so that every path holds the same
keys from then on).  On the batch's collision-free rows (no field with more than two tokens, or no pass of T = 128 / K
tokens holding two tokens of one field) both F32 models must equal it bit for bit; on the other rows its same-field adds
run in an order the hardware picks, so there the F32 models must be within 1e-4 of it, and the share of rows that agree
bit for bit anyway is reported.  Then, in one process, alternating the paths call by call:
  table   Trainer.predict_host_fields (xf_k_step_mvm, mode 1).  The table has no predict on device pointers, so the call
          also copies the batch from host memory; the kernel's own time comes from torch.profiler in the same run, and
          the call's wall time is reported beside it as what it is.
  model   Model.predict_device_fields with d_vals (xf_k_serve_mvm) at F32 (pruned and full) and F16, CUDA events around
          each call, and the same profiler's kernel time.
Prints examples/s, algorithmic bytes per token (8 of key, 1 of field id, 4 of value, and the row bytes the path reads:
the table's 32-byte head sector and 4K of v, the model's 16-byte head and 4K (F32) or 2K (F16) of v) over kernel time
against the H100 SXM data-sheet 3.35 TB/s (a data-sheet figure, not a measured peak), model and table bytes, and the
card's name and power limit read in the same run.  One JSON line.  Needs a CUDA device and torch; touches no device
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

B, NNZ, RING, VIEWS = 65536, 100, 8, 8
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
    rng = np.random.default_rng(seed)
    fields = rng.integers(0, VIEWS, raw.size).astype(np.uint8)
    vals = rng.uniform(-1.0, 2.0, raw.size).astype(np.float32)
    return rp, api.hash_decimal_ids(raw), fields, vals, lab


def collision_free(fields, K):
    """Rows of a fixed-length batch (fields [B, NNZ]) on which the table's predict is reproducible"""
    counts = np.zeros((fields.shape[0], 32), np.int32)
    np.add.at(counts, (np.repeat(np.arange(fields.shape[0]), fields.shape[1]), fields.ravel().astype(np.int64)), 1)
    ok = np.ones(fields.shape[0], bool)
    T = 128 // K
    for p in range(0, fields.shape[1], T):
        s = np.sort(fields[:, p:p + T], axis=1)
        ok &= ~np.any(s[:, 1:] == s[:, :-1], axis=1)
    return ok | (counts.max(axis=1) <= 2)


def run_shape(api, datagen, torch, K, ids, calls, train_steps):
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, canonical_fm=1, v_init=api.VINIT_COUNTER, seed=3)
    t.reserve(ids)
    tr = api.Trainer(t, model=api.MODEL_MVM, max_rows=B, max_nnz=B * NNZ)
    for i in range(train_steps):
        tr.step_host_fields(*batch(api, datagen, 1 + i, ids))
    tr.sync()
    trained_keys = t.size()
    # the initial values (N(0, 0.01)) and a few steps leave products over 8 fields so close to 0 that every prediction
    # would round to sigmoid(0): the trained keys get latent rows of N(0, 0.25) instead, which keep a field's sum of
    # about 12 tokens near 1
    keys = t.list_keys()
    t.import_(keys, w=np.zeros(keys.size, np.float32),
              v=np.random.default_rng(5).normal(0.0, 0.25, (keys.size, K)).astype(np.float32))
    models = dict(f32_pruned=t.freeze_mvm(), f32_full=t.freeze_mvm(prune=False))
    models["f16_pruned"] = models["f32_pruned"].convert(api.PRECISION_F16)
    host, dev = [], []
    for i in range(RING):
        rp, keys, fields, vals, _ = batch(api, datagen, 1000 + i, ids)
        host.append((rp, keys, fields, vals))
        dev.append(tuple(torch.from_numpy(a.view(np.uint8)).cuda() for a in (rp, keys, fields, vals)))
    out = torch.empty(B, dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()

    def serve(m, i):
        d_rp, d_keys, d_fields, d_vals = dev[i % RING]
        m.predict_device_fields(d_rp.data_ptr(), d_keys.data_ptr(), d_fields.data_ptr(), B, B * NNZ, out.data_ptr(),
                                stream=stream.cuda_stream, d_vals=d_vals.data_ptr())

    # the paths agree before anything is timed; the table's first predict of a batch inserts its unseen keys, which
    # read as the model's absent keys do
    cf_rows = bit_equal_rows = 0
    distinct = []
    for i in range(RING):
        want = tr.predict_host_fields(*host[i])
        distinct.append(int(np.unique(want).size))
        cf = collision_free(host[i][2].reshape(B, NNZ), K)
        cf_rows += int(cf.sum())
        for k in ("f32_pruned", "f32_full"):
            serve(models[k], i)
            stream.synchronize()
            got = out.cpu().numpy()
            same = got.view(np.uint32) == want.view(np.uint32)
            assert same[cf].all(), "model and table predictions differ on a collision-free row"
            assert np.all(np.abs(got.astype(np.float64) - want) <= 1e-4 * (1 + np.abs(want))), "model and table differ"
            if k == "f32_pruned":
                bit_equal_rows += int(same.sum())
    res = dict(ids=ids, latent_dim=K, optimizer="ftrl", id_distribution="zipf(1.05)", views=VIEWS, rows=B, nnz_per_row=NNZ,
               calls=calls, train_steps=train_steps, table_keys_after_training=trained_keys, table_keys_timed=t.size(),
               table_bytes=t.capacity() * t.row_bytes(), table_row_bytes=t.row_bytes(),
               checked_rows=RING * B, collision_free_rows=cf_rows, rows_bit_equal_to_table=bit_equal_rows,
               min_distinct_predictions_per_batch=min(distinct))
    ev = {k: [0.0, 0] for k in models}
    wall_table = 0.0
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            t0 = time.perf_counter()
            tr.predict_host_fields(*host[i % RING])
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
    step_ms, step_n = kernel_ms(prof, "xf_k_step_mvm")
    serve_ms, serve_n = kernel_ms(prof, "xf_k_serve_mvm")
    tokens = B * NNZ
    table_tok = 8 + 1 + 4 + 32 + 4 * K
    res["profiler_launches"] = dict(table=step_n, model=serve_n)
    if step_n:
        res["table"] = dict(kernel_ms_per_call=step_ms / step_n, examples_per_s_kernel=B / (step_ms / step_n / 1e3),
                            wall_ms_per_call_incl_host_copy=wall_table / calls * 1e3, algorithmic_bytes_per_token=table_tok,
                            share_of_datasheet_bw=tokens * table_tok / (step_ms / step_n / 1e3) / DATASHEET_BW)
    if serve_n:
        res["model_kernel_ms_per_call_all_models"] = serve_ms / serve_n
    for k, m in models.items():
        ms = ev[k][0] / ev[k][1]
        i = m.info()
        model_tok = 8 + 1 + 4 + 16 + (2 if k.startswith("f16") else 4) * K
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
    ap.add_argument("--dims", default="16,32")
    args = ap.parse_args()
    from xflow_b200 import api, datagen
    if api.device_count() < 1:
        sys.exit("mvm_serving_bench needs a CUDA device: there is nothing to measure without one")
    import torch
    res = dict(gpu=gpu_info(), datasheet_bw_bytes_per_s=DATASHEET_BW)
    for K in (int(k) for k in args.dims.split(",")):
        res["mvm_k%d_ftrl_zipf" % K] = run_shape(api, datagen, torch, K, args.ids, args.calls, args.train_steps)
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

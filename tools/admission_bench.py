"""Feature admission on the device (xf_table_set_admission; DESIGN.md section 6): what a counting Bloom filter saves
and costs on a skewed workload that starts from an EMPTY table.

    python tools/admission_bench.py [--batches 64] [--runs 2] [--log2-cells 30]

LR+FTRL, Zipf(1.05) ids in a 1e8-feature space, 100 nnz/row, 65 536 rows per batch (the cfg5 id distribution on the
headline LR shape); one pass over `--batches` distinct seeded batches (keys hashed on the device, resident before the
timed pass), once without a policy and once with Bloom admission (n = 2, 2^log2_cells one-byte cells, 3 hashes, no
decay), alternating, `--runs` times each.  The table starts at the library's default capacity and grows on demand,
so its capacity at the end reflects the keys it holds.  Prints one JSON line: per arm the median ms per step (CUDA
events around every step, median over the steps, then over the runs), keys, capacity x row bytes, filter bytes and
the share of rejected tokens, with the card's name, power limit and SM clocks.  Needs a CUDA device.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B_ROWS, NNZ, ID_SPACE = 65536, 100, 10 ** 8


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=64)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--log2-cells", type=int, default=30)
    args = ap.parse_args()
    import torch
    from xflow_b200 import api, datagen
    if api.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    stream = torch.cuda.Stream()
    lib = api.lib()
    nnz = B_ROWS * NNZ
    batches = []
    for i in range(args.batches):
        rp, ids, lab = datagen.make_ids(seed=5000 + i, rows=B_ROWS, nnz_per_row=NNZ, id_space=ID_SPACE, dist="zipf",
                                        zipf_s=1.05)
        d_ids = torch.from_numpy(ids.astype(np.uint32).view(np.uint8)).cuda()
        d_keys = torch.empty(nnz * 8, dtype=torch.uint8, device="cuda")
        torch.cuda.current_stream().synchronize()
        assert lib.xf_hash_decimal_ids_device(C.c_void_p(d_ids.data_ptr()), nnz, C.c_void_p(d_keys.data_ptr()),
                                              C.c_void_p(stream.cuda_stream)) == 0
        stream.synchronize()  # d_ids goes back to the allocator only after the hash kernel has read it
        batches.append((torch.from_numpy(rp.view(np.uint8)).cuda(), d_keys, torch.from_numpy(lab.view(np.uint8)).cuda()))
        del d_ids
    arms = {"no_policy": None,
            "bloom_n2": dict(mode=api.ADMIT_BLOOM, threshold=2, log2_cells=args.log2_cells, hashes=3)}
    runs = {a: [] for a in arms}
    info_before = gpu_info()
    with torch.cuda.stream(stream):
        for _ in range(args.runs):
            for arm, policy in arms.items():
                table = api.Table(latent_dim=0, optimizer=api.OPT_FTRL, seed=1)
                table.set_stream(stream.cuda_stream)
                if policy:
                    table.set_admission(**policy)
                tr = api.Trainer(table, model=api.MODEL_LR, max_rows=B_ROWS, max_nnz=nnz + 1024)
                tr.init_push()
                tr.sync()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.batches + 1)]
                ev[0].record(stream)
                for i, d in enumerate(batches):
                    tr.step_device(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), B_ROWS, nnz)
                    ev[i + 1].record(stream)
                tr.sync()
                ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(args.batches)]
                st = table.admission_stats()
                runs[arm].append({
                    "ms_per_step": float(np.median(ms)), "ms_total": float(sum(ms)), "keys": table.size(),
                    "table_slots": table.capacity(), "row_bytes": table.row_bytes(),
                    "table_bytes": table.capacity() * table.row_bytes(),
                    "filter_bytes": (1 << policy["log2_cells"]) if policy else 0,
                    "rejected_token_share": st["rejected_tokens"] / float(args.batches * nnz)})
                tr.close()
                table.close()
                torch.cuda.empty_cache()
    out = {}
    for arm, rs in runs.items():
        r = dict(rs[-1])
        r["ms_per_step"] = float(np.median([x["ms_per_step"] for x in rs]))
        r["ms_per_step_runs"] = [x["ms_per_step"] for x in rs]
        out[arm] = r
    print(json.dumps({"workload": "LR+FTRL, Zipf(1.05) ids in 1e8, 100 nnz/row, batch 65536, one pass over %d batches "
                                  "from an empty table" % args.batches, "arms": out,
                      "gpu_before": info_before, "gpu_after": gpu_info()}))


if __name__ == "__main__":
    main()

"""File -> model throughput of the two ingest paths (SURVEY.md section 8f-1): host parser
(xf_loader_next, one CPU core, like the reference's LoadData) against the device parser
(xf_trainer_ingest_text).  Prints one JSON line; not a bench.py metric."""
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xflow_b200 import api, datagen  # noqa: E402


def main():
    rows = int(os.environ.get("ROWS", 200000))
    block = int(os.environ.get("BLOCK_MB", 8)) << 20
    d = tempfile.mkdtemp()
    path = os.path.join(d, "t-00000")
    row_ptr, ids, labels = datagen.make_ids(3, rows, 40, 1 << 40, dist="zipf")
    datagen.write_text(path, row_ptr, ids, labels)
    size = os.path.getsize(path)
    out = dict(file_bytes=size, rows=rows, block_bytes=block)

    t0 = time.perf_counter()
    n = sum(y.size for _, _, y in api.Loader(path, block))
    out["host_parse_s"] = time.perf_counter() - t0
    assert n == rows

    def train(ingest):
        t = api.Table(latent_dim=0, capacity=1 << 24)
        tr = api.Trainer(t, max_rows=block // 8 + 16, max_nnz=block // 6 + 16)
        tr.init_push()
        for rep in range(2):  # first pass warms the table and the allocations
            ld = api.Loader(path, block)
            tr.sync()
            t0 = time.perf_counter()
            if ingest:
                lib, h = api.lib(), ld.h
                import ctypes as C
                text, ln, r, z = C.c_void_p(), C.c_uint64(), C.c_uint32(), C.c_uint32()
                while True:
                    lib.xf_loader_next_raw(h, C.byref(text), C.byref(ln))
                    if not ln.value:
                        break
                    assert lib.xf_trainer_ingest_text(tr.h, text, ln.value, C.byref(r), C.byref(z)) == 0
                    assert lib.xf_trainer_step_ingested(tr.h, 0, r.value) == 0
            else:
                for rp, k, y in ld:
                    tr.step_host(rp, k, y, want_loss=False)
            tr.sync()
            dt = time.perf_counter() - t0
        tr.close()
        t.close()
        return dt

    out["train_host_parse_s"] = train(False)
    out["train_device_ingest_s"] = train(True)
    for k in ("host_parse_s", "train_host_parse_s", "train_device_ingest_s"):
        out[k.replace("_s", "_MBps")] = round(size / out[k] / 1e6, 1)
        out[k.replace("_s", "_rows_per_s")] = round(rows / out[k])
    print(json.dumps(out))


if __name__ == "__main__":
    main()

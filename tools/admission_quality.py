"""Model quality with and without feature admission (DESIGN.md section 6): logloss and AUC on the bundled shards and
on the synthetic Zipf shard of tests/golden/cases.py, trained by the CPU restatement (oracle/) and by the GPU with the
same policy (the CPU side: tests/admission_model.py over the oracle's table), next to the number of keys each table
holds.  Needs a CUDA device.

    python tools/admission_quality.py [--out FILE.json]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from admission_model import ADMIT_BLOOM, AdmittingTable  # noqa: E402
from cases import SYN, SYN_TEST  # noqa: E402
from oracle import oracle as O  # noqa: E402
from xflow_b200 import api, datagen  # noqa: E402

BLOOM = dict(threshold=2, log2_cells=20, hashes=3, decay_batches=0, seed=0)


def gpu_run(K, train, test, epochs, policy):
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL)
    if policy:
        t.set_admission(api.ADMIT_BLOOM, **BLOOM)
    tr = api.Trainer(t, model=api.MODEL_LR if K == 0 else api.MODEL_FM, max_rows=1 << 17, max_nnz=1 << 22)
    tr.init_push()
    for _ in range(epochs):
        for rp, keys, lab in api.Loader(train, 2 << 20):
            tr.step_host(rp, keys, lab, want_loss=False)
    labs, ps = [], []
    for rp, keys, lab in api.Loader(test, (4 << 20) if K == 0 else (2 << 20)):
        ps.append(tr.predict_host(rp, keys))
        labs.append(lab.astype(np.int32))
    m = O.auc_logloss(np.concatenate(labs), np.concatenate(ps))
    return dict(logloss=m["logloss"], auc=m["auc"], keys=t.size())


def oracle_run(K, train, test, epochs, policy):
    t = AdmittingTable(K=K)
    if policy:
        t.set_admission(ADMIT_BLOOM, **BLOOM)
    O.train_file(t, train, 2 << 20, epochs)
    lab, p = O.predict_file(t, test, (4 << 20) if K == 0 else (2 << 20))
    m = O.auc_logloss(lab, p)
    return dict(logloss=m["logloss"], auc=m["auc"], keys=t.size())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    tmp = tempfile.mkdtemp(prefix="xfadm_")
    syn_tr, syn_te = os.path.join(tmp, "syn_train-00000"), os.path.join(tmp, "syn_test-00000")
    datagen.write_text(syn_tr, *datagen.make_ids(**SYN))
    datagen.write_text(syn_te, *datagen.make_ids(**SYN_TEST))
    small = os.path.join(ROOT, "tests", "golden", "data")
    data = {"bundled": (os.path.join(small, "small_train-00000"), os.path.join(small, "small_test-00000"), 10),
            "syn_zipf": (syn_tr, syn_te, 2)}
    rows = []
    for dname, (train, test, epochs) in data.items():
        for K in (0, 8):
            for policy in (False, True):
                o = oracle_run(K, train, test, epochs, policy)
                g = gpu_run(K, train, test, epochs, policy)
                rows.append(dict(data=dname, model="lr" if K == 0 else "fm_k%d" % K, optimizer="ftrl", epochs=epochs,
                                 admission="bloom n=2, 2^20 cells, 3 hashes" if policy else "none", oracle=o, gpu=g))
                print(json.dumps(rows[-1]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()

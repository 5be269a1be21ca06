"""Child process of tests/test_gpu_edges.py, part D: runs the device side of a case under the process-wide setting
XFLOW_FM_CACHE_LOG2, which the library reads once per process, and writes the results to an npz file for the parent
test to compare.  fm_bounds instead checks its cases itself against tests/fm_model.py (test_gpu_fm_step.py) and exits
non-zero on the first one outside the bounds.

    python tests/edge_child.py fm_steps OUT.npz
    python tests/edge_child.py fm_bounds OUT.npz
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

from xflow_b200 import api, datagen  # noqa: E402

SEED = 23
FM_STEP_CASES = [(8, "ftrl"), (16, "sgd"), (32, "ftrl")]
B, D, SPACE = 2048, 24, 20000


def _gopt(opt):
    return api.OPT_FTRL if opt == "ftrl" else api.OPT_SGD


def fm_batches():
    """Zipf(1.3) batches: hot keys fill the step kernel's hot-key cache and overflow it."""
    return [datagen.make_csr_keys(700 + s, B, D, SPACE, api.hash_decimal_ids, dist="zipf", zipf_s=1.3, ragged=(s == 1))
            for s in range(3)]


def fm_steps(out):
    batches = fm_batches()
    uk = np.unique(np.concatenate([b[1] for b in batches]))
    out["keys"] = uk
    for K, opt in FM_STEP_CASES:
        t = api.Table(latent_dim=K, optimizer=_gopt(opt), v_init=api.VINIT_COUNTER, seed=SEED)
        tr = api.Trainer(t, model=api.MODEL_FM, max_rows=B, max_nnz=B * D * 2, keep_loss=True)
        for step, (rp, keys, lab) in enumerate(batches):
            tr.step_host(rp, keys, lab)
            out["loss_%d_%s_%d" % (K, opt, step)] = tr.get_loss(B)
        e = t.export(uk)
        for k in ("w", "nw", "zw", "v", "nv", "zv"):
            out["%s_%d_%s" % (k, K, opt)] = e[k]
        tr.close()
        t.close()


def main():
    what, path = sys.argv[1], sys.argv[2]
    out = {}
    if what == "fm_steps":
        fm_steps(out)
    elif what == "fm_bounds":
        import test_gpu_fm_step
        test_gpu_fm_step.cache_setting_cases()
    else:
        raise SystemExit("unknown case " + what)
    np.savez(path, **out)


if __name__ == "__main__":
    main()

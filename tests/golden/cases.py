"""Golden case table shared by make_golden.py (generation, needs the reference) and the tests."""

# name -> dict(data, model, opt, epochs, K, block_mb, preinit)
CASES = {
    "small_lr_ftrl_e10": dict(data="small", model="lr", opt="ftrl", epochs=10, K=0),
    "small_lr_ftrl_e60": dict(data="small", model="lr", opt="ftrl", epochs=60, K=0),
    "small_lr_sgd_e60": dict(data="small", model="lr", opt="sgd", epochs=60, K=0),
    "small_fm_sgd_k10_e60": dict(data="small", model="fm", opt="sgd", epochs=60, K=10),
    "small_fm_ftrl_k10_e5": dict(data="small", model="fm", opt="ftrl", epochs=5, K=10, preinit=True),
    "syn_lr_ftrl_e2": dict(data="syn", model="lr", opt="ftrl", epochs=2, K=0, block_mb=1),
    "syn_fm_sgd_k16_e1": dict(data="syn", model="fm", opt="sgd", epochs=1, K=16, block_mb=1),
    "syn_fm_ftrl_k8_e1": dict(data="syn", model="fm", opt="ftrl", epochs=1, K=8, block_mb=1, preinit=True),
}

# runs of the reference on the synthetic shards with its wall-clock seeded FM init (pinned time), stored as
# digests of its final table: (model, opt, K, epochs); block_mb = 1
FRESH_RUNS = [("lr", "ftrl", 0, 3), ("lr", "sgd", 0, 3), ("fm", "sgd", 6, 2), ("fm", "ftrl", 4, 2)]


def fresh_run_name(model, opt, K, epochs):
    return "%s_%s_k%d_e%d" % (model, opt, K, epochs)

SYN = dict(seed=7, rows=3000, nnz_per_row=48, id_space=20000, dist="zipf", zipf_s=1.2)
SYN_TEST = dict(seed=8, rows=500, nnz_per_row=48, id_space=20000, dist="zipf", zipf_s=1.2)

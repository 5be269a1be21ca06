"""Thin ctypes binding of libxflow_b200.so (include/xflow_b200.h) for tests and bench.py.

The product is the C ABI; this module only marshals numpy arrays / raw pointers into it.  It never
computes anything itself and has no fallback: if the shared library (or a CUDA device, for compute
calls) is missing, calls fail loudly.
"""
import ctypes as C
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libxflow_b200.so")

MODEL_LR, MODEL_FM, MODEL_FM_CANONICAL, MODEL_MVM, MODEL_FFM = 0, 1, 2, 3, 4
OPT_FTRL, OPT_SGD, OPT_ADAGRAD = 0, 1, 2
VINIT_DEFAULT, VINIT_COUNTER, VINIT_ZERO = 0, 1, 3
ADMIT_ALL, ADMIT_POISSON, ADMIT_BLOOM = 0, 1, 2
ABSENT_DEFAULT, ABSENT_ZERO = 0, 1
PRECISION_F32, PRECISION_F16 = 0, 1
COMM_ID_BYTES = 128

_lib = None


class XflowError(RuntimeError):
    pass


class TableConfig(C.Structure):
    _fields_ = [("device", C.c_int), ("latent_dim", C.c_int), ("optimizer", C.c_int), ("alpha", C.c_float),
                ("beta", C.c_float), ("lambda1", C.c_float), ("lambda2", C.c_float),
                ("learning_rate", C.c_float), ("v_init", C.c_int), ("seed", C.c_uint64),
                ("capacity", C.c_uint64), ("shard_index", C.c_int), ("num_shards", C.c_int), ("canonical_fm", C.c_int)]


class AdmissionConfig(C.Structure):
    _fields_ = [("mode", C.c_int), ("probability", C.c_float), ("threshold", C.c_uint32), ("log2_cells", C.c_uint32),
                ("hashes", C.c_uint32), ("decay_batches", C.c_uint64), ("seed", C.c_uint64)]


class EvictionConfig(C.Structure):
    _fields_ = [("max_idle_batches", C.c_uint64), ("max_keys", C.c_uint64)]


class FreezeConfig(C.Structure):
    _fields_ = [("absent", C.c_int), ("prune", C.c_int), ("device", C.c_int)]


class ModelInfo(C.Structure):
    _fields_ = [("keys", C.c_uint64), ("capacity", C.c_uint64), ("bytes", C.c_uint64), ("source_keys", C.c_uint64),
                ("pruned_keys", C.c_uint64), ("row_bytes", C.c_uint32), ("latent_dim", C.c_int), ("optimizer", C.c_int),
                ("absent", C.c_int), ("fm", C.c_int), ("precision", C.c_int)]


class CandidateBatch(C.Structure):
    """xf_candidate_batch: R requests, each a context and a run of candidate rows (include/xflow_b200.h)."""
    _fields_ = [("requests", C.c_uint32), ("ctx_ptr", C.c_void_p), ("ctx_keys", C.c_void_p), ("ctx_vals", C.c_void_p),
                ("ctx_fields", C.c_void_p), ("ctx_nnz", C.c_uint32), ("cand_ptr", C.c_void_p), ("candidates", C.c_uint32),
                ("row_ptr", C.c_void_p), ("keys", C.c_void_p), ("vals", C.c_void_p), ("fields", C.c_void_p),
                ("nnz", C.c_uint32)]


class DeltaInfo(C.Structure):
    _fields_ = [("upserts", C.c_uint64), ("deletes", C.c_uint64), ("base_keys", C.c_uint64),
                ("base_fingerprint", C.c_uint64), ("result_keys", C.c_uint64), ("result_fingerprint", C.c_uint64),
                ("source_keys", C.c_uint64), ("pruned_keys", C.c_uint64), ("file_bytes", C.c_uint64),
                ("row_bytes", C.c_uint32), ("latent_dim", C.c_int), ("precision", C.c_int)]


class TrainerConfig(C.Structure):
    _fields_ = [("model", C.c_int), ("max_rows", C.c_uint32), ("max_nnz", C.c_uint32), ("keep_loss", C.c_int)]


class PvReport(C.Structure):
    _fields_ = [("rows", C.c_uint64), ("positives", C.c_uint64), ("negatives", C.c_uint64), ("nan_rows", C.c_uint64),
                ("overflow_rows", C.c_uint64), ("weight_pos", C.c_double), ("weight_neg", C.c_double),
                ("logloss", C.c_double), ("mean_pctr", C.c_double), ("ctr", C.c_double), ("auc", C.c_double),
                ("auc_lo", C.c_double), ("auc_hi", C.c_double)]


class GroupReport(C.Structure):
    _fields_ = [("rows", C.c_uint64), ("positives", C.c_uint64), ("negatives", C.c_uint64), ("nan_rows", C.c_uint64),
                ("groups", C.c_uint64), ("scored_groups", C.c_uint64), ("scored_rows", C.c_uint64),
                ("logloss", C.c_double), ("gauc", C.c_double), ("gauc_mean", C.c_double)]


class GroupTopkReport(C.Structure):
    _fields_ = [("k", C.c_uint32), ("groups", C.c_uint64), ("scored_groups", C.c_uint64), ("scored_rows", C.c_uint64),
                ("ndcg", C.c_double), ("ndcg_mean", C.c_double), ("precision", C.c_double),
                ("precision_mean", C.c_double), ("recall", C.c_double), ("recall_mean", C.c_double)]


# name -> (restype, argtypes); also the list the symbol-export test checks against the header
_vp, _u64, _u32, _i, _f = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_float
SIGNATURES = {
    "xf_last_error": (C.c_char_p, []),
    "xf_version": (_i, []),
    "xf_device_count": (_i, []),
    "xf_table_config_default": (_i, [_vp]),
    "xf_table_create": (_i, [_vp, _vp]),
    "xf_table_destroy": (_i, [_vp]),
    "xf_table_pull": (_i, [_vp, _vp, _u64, _vp, _vp]),
    "xf_table_push": (_i, [_vp, _vp, _u64, _vp, _vp]),
    "xf_table_pull_device": (_i, [_vp, _vp, _u64, _vp, _vp]),
    "xf_table_push_device": (_i, [_vp, _vp, _u64, _vp, _vp]),
    "xf_table_import": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "xf_table_export": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "xf_table_size": (_i, [_vp, _vp]),
    "xf_table_capacity": (_i, [_vp, _vp]),
    "xf_table_row_bytes": (_i, [_vp, _vp]),
    "xf_table_latent_dim": (_i, [_vp, _vp]),
    "xf_table_reserve": (_i, [_vp, _u64]),
    "xf_table_list_keys": (_i, [_vp, _vp, _u64, _vp]),
    "xf_table_touch_decimal_ids": (_i, [_vp, _u64, _u64]),
    "xf_table_save": (_i, [_vp, C.c_char_p]),
    "xf_table_load": (_i, [_vp, C.c_char_p]),
    "xf_table_save_state": (_i, [_vp, C.c_char_p, _u64]),
    "xf_table_load_state": (_i, [_vp, C.c_char_p, _vp]),
    "xf_table_set_stream": (_i, [_vp, _vp]),
    "xf_table_sync": (_i, [_vp]),
    "xf_admission_config_default": (_i, [_vp]),
    "xf_table_set_admission": (_i, [_vp, _vp]),
    "xf_table_admission_stats": (_i, [_vp, _vp, _vp, _vp]),
    "xf_table_set_eviction": (_i, [_vp, _vp]),
    "xf_table_evict": (_i, [_vp, _vp]),
    "xf_table_last_touch": (_i, [_vp, _vp, _u64, _vp]),
    "xf_shard_of": (_i, [_u64, _i]),
    "xf_trainer_create": (_i, [_vp, _vp, _vp, _vp]),
    "xf_trainer_destroy": (_i, [_vp]),
    "xf_trainer_step_host": (_i, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_trainer_step_device": (_i, [_vp, _vp, _vp, _vp, _u32, _u32]),
    "xf_trainer_predict_host": (_i, [_vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_trainer_step_host_values": (_i, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_trainer_step_device_values": (_i, [_vp, _vp, _vp, _vp, _vp, _u32, _u32]),
    "xf_trainer_predict_host_values": (_i, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_trainer_step_host_fields": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_trainer_predict_host_fields": (_i, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_trainer_step_host_weighted": (_i, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_trainer_step_device_weighted": (_i, [_vp, _vp, _vp, _vp, _vp, _u32, _u32]),
    "xf_trainer_set_negative_sampling": (_i, [_vp, _f, _u64]),
    "xf_trainer_skipped_rows": (_i, [_vp, _vp]),
    "xf_trainer_init_push": (_i, [_vp]),
    "xf_trainer_get_loss": (_i, [_vp, _vp, _u32]),
    "xf_trainer_stats": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "xf_trainer_launches": (_i, [_vp, _vp]),
    "xf_trainer_sync": (_i, [_vp]),
    "xf_trainer_wait_uploads": (_i, [_vp]),
    "xf_trainer_step_host_async": (_i, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_trainer_step_host_ids_async": (_i, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_hash_decimal_ids_device": (_i, [_vp, _u64, _vp, _vp]),
    "xf_auc_logloss_exact": (_i, [_vp, _vp, _u64, _vp]),
    "xf_table_dump_text": (_i, [_vp, C.c_char_p, _i, _vp]),
    "xf_trainer_ingest_text": (_i, [_vp, _vp, _u64, _vp, _vp]),
    "xf_trainer_ingest_begin": (_i, [_vp, _vp, _u64]),
    "xf_trainer_ingest_end": (_i, [_vp, _vp, _vp]),
    "xf_trainer_step_ingested": (_i, [_vp, _u32, _u32]),
    "xf_trainer_ingested_export": (_i, [_vp, _vp, _vp, _vp]),
    "xf_trainer_predict_ingested": (_i, [_vp, _u32, _u32, _vp, _vp]),
    "xf_loader_next_raw": (_i, [_vp, _vp, _vp]),
    "xf_trainer_set_profile": (_i, [_vp, _i]),
    "xf_trainer_profile": (_i, [_vp, _vp, _vp]),
    "xf_host_alloc": (_i, [_vp, _u64]),
    "xf_host_free": (_i, [_vp]),
    "xf_auc_logloss": (_i, [_vp, _vp, _u64, _vp]),
    "xf_metric_create": (_i, [_vp, _i]),
    "xf_metric_destroy": (_i, [_vp]),
    "xf_metric_reset": (_i, [_vp]),
    "xf_metric_add_device": (_i, [_vp, _vp, _vp, _u64, _vp]),
    "xf_metric_finish": (_i, [_vp, _vp, _vp]),
    "xf_auc_logloss_device": (_i, [_vp, _vp, _u64, _i, _vp, _vp]),
    "xf_trainer_predict_ingested_metric": (_i, [_vp, _u32, _u32, _vp, _vp, _vp]),
    "xf_hash_bytes": (_u64, [C.c_char_p, _u64]),
    "xf_hash_decimal_ids": (_i, [_vp, _u64, _vp]),
    "xf_loader_open": (_i, [_vp, C.c_char_p, _u64]),
    "xf_loader_close": (_i, [_vp]),
    "xf_loader_rewind": (_i, [_vp]),
    "xf_loader_next": (_i, [_vp, _vp, _vp]),
    "xf_loader_batch": (_i, [_vp, _vp, _vp, _vp]),
    "xf_comm_get_id": (_i, [_vp]),
    "xf_comm_create": (_i, [_vp, _vp, _i, _i, _i]),
    "xf_comm_create_from_file": (_i, [_vp, C.c_char_p, _i, _i, _i]),
    "xf_comm_allreduce_max": (_i, [_vp, _vp]),
    "xf_comm_destroy": (_i, [_vp]),
    "xf_comm_barrier": (_i, [_vp]),
    "xf_freeze_config_default": (_i, [_vp]),
    "xf_table_freeze": (_i, [_vp, _vp, _vp]),
    "xf_table_freeze_canonical": (_i, [_vp, _vp, _vp]),
    "xf_table_freeze_mvm": (_i, [_vp, _vp, _vp]),
    "xf_table_freeze_ffm": (_i, [_vp, _vp, _vp]),
    "xf_table_freeze_part": (_i, [_vp, _vp, _vp]),
    "xf_model_part_info": (_i, [_vp, _vp, _vp]),
    "xf_model_merge": (_i, [_vp, _i, _i, _vp]),
    "xf_model_convert": (_i, [_vp, _i, _vp]),
    "xf_model_destroy": (_i, [_vp]),
    "xf_model_get_info": (_i, [_vp, _vp]),
    "xf_model_save": (_i, [_vp, C.c_char_p]),
    "xf_model_load": (_i, [_vp, C.c_char_p, _i]),
    "xf_model_predict_host": (_i, [_vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_model_predict_device": (_i, [_vp, _vp, _vp, _u32, _u32, _vp, _vp]),
    "xf_model_predict_host_values": (_i, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_model_predict_device_values": (_i, [_vp, _vp, _vp, _vp, _u32, _u32, _vp, _vp]),
    "xf_model_predict_host_fields": (_i, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "xf_model_predict_device_fields": (_i, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp, _vp]),
    "xf_model_predict_candidates_host": (_i, [_vp, _vp, _vp]),
    "xf_model_predict_candidates_device": (_i, [_vp, _vp, _vp, _vp]),
    "xf_model_rank_candidates_host": (_i, [_vp, _vp, _u32, _vp, _vp]),
    "xf_model_rank_candidates_device": (_i, [_vp, _vp, _u32, _vp, _vp, _vp, _vp]),
    "xf_model_lookup": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp]),
    "xf_model_lookup_latent": (_i, [_vp, _vp, _u64, _vp, _vp, _vp]),
    "xf_model_predict_ingested": (_i, [_vp, _vp, _u32, _u32, _vp, _vp]),
    "xf_model_diff": (_i, [_vp, _vp, _vp]),
    "xf_model_apply_delta": (_i, [_vp, _vp, _vp]),
    "xf_model_fingerprint": (_i, [_vp, _vp]),
    "xf_delta_save": (_i, [_vp, C.c_char_p]),
    "xf_delta_load": (_i, [_vp, C.c_char_p, _i]),
    "xf_delta_get_info": (_i, [_vp, _vp]),
    "xf_delta_destroy": (_i, [_vp]),
    "xf_pv_create": (_i, [_vp, _i, _u32]),
    "xf_pv_destroy": (_i, [_vp]),
    "xf_pv_reset": (_i, [_vp]),
    "xf_pv_add_device": (_i, [_vp, _vp, _vp, _vp, _u64, _vp]),
    "xf_pv_report": (_i, [_vp, _vp]),
    "xf_pv_set_slices": (_i, [_vp, _vp, _vp, _u64, _u32, _u32]),
    "xf_pv_add_device_rows": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _u64, _vp]),
    "xf_pv_report_slices": (_i, [_vp, _vp, _u32]),
    "xf_trainer_set_validation": (_i, [_vp, _vp]),
    "xf_group_metric_create": (_i, [_vp, _i]),
    "xf_group_metric_destroy": (_i, [_vp]),
    "xf_group_metric_reset": (_i, [_vp]),
    "xf_group_metric_add_device": (_i, [_vp, _vp, _vp, _vp, _u64, _vp]),
    "xf_group_metric_finish": (_i, [_vp, _vp]),
    "xf_group_metric_groups": (_i, [_vp, _u64, _vp, _vp, _vp, _vp, _vp]),
    "xf_group_metric_topk": (_i, [_vp, _u32, _vp]),
    "xf_group_metric_groups_topk": (_i, [_vp, _u64, _vp, _vp, _vp]),
    "xf_group_metric_discounts": (_i, [_vp, _u32]),
    "xf_trainer_set_deterministic": (_i, [_vp, _i]),
    "XFCreate": (_i, [_vp, C.c_char_p, C.c_char_p]),
    "XFStartTrain": (_i, [_vp]),
    "XFCreateEx": (_i, [_vp, C.c_char_p, C.c_char_p, _i, _i, _i, _i]),
    "XFDestroy": (_i, [_vp]),
}


def lib():
    """Load the shared library (building is __graft_entry__.build()'s job; missing .so is an error)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise XflowError("%s not built: run `python -m xflow_b200.build`" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def _check(rc):
    if rc != 0:
        raise XflowError("xflow_b200 error %d: %s" % (rc, lib().xf_last_error().decode(errors="replace")))


def _p(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(int(a))  # raw address (e.g. torch tensor.data_ptr())


def device_count():
    return lib().xf_device_count()


def hash_bytes(s: bytes) -> int:
    return lib().xf_hash_bytes(s, len(s))


def hash_decimal_ids(ids):
    ids = np.ascontiguousarray(ids, np.uint64)
    out = np.empty_like(ids)
    _check(lib().xf_hash_decimal_ids(_p(ids), ids.size, _p(out)))
    return out


def shard_of(key, num_shards):
    return lib().xf_shard_of(int(key), int(num_shards))


def group_discounts(n=65536):
    """The grouped metric's top-k discounts d(0 .. n-1) = round(2^32 / log2(i + 2)) (uint64), n <= 65536
    (xf_group_metric_discounts; header section 9)."""
    out = np.empty(int(n), np.uint64)
    _check(lib().xf_group_metric_discounts(_p(out), int(n)))
    return out


def auc_logloss(labels, pctr):
    labels = np.ascontiguousarray(labels, np.int32)
    pctr = np.ascontiguousarray(pctr, np.float32)
    out = np.zeros(4, np.float64)
    _check(lib().xf_auc_logloss(_p(labels), _p(pctr), labels.size, _p(out)))
    return dict(logloss=float(out[0]), auc=float(out[1]), tp=int(out[2]), fp=int(out[3]))


def auc_logloss_exact(labels, pctr):
    """Exact-arithmetic test metric: natural-log logloss (negated) and tie-aware AUC."""
    labels = np.ascontiguousarray(labels, np.int32)
    pctr = np.ascontiguousarray(pctr, np.float32)
    out = np.zeros(4, np.float64)
    _check(lib().xf_auc_logloss_exact(_p(labels), _p(pctr), labels.size, _p(out)))
    return dict(logloss=float(out[0]), auc=float(out[1]), positives=int(out[2]), negatives=int(out[3]))


class Loader:
    """xflow::LoadData replacement: iterate CSR blocks of a text shard."""

    def __init__(self, path, block_bytes):
        self.h = C.c_void_p()
        _check(lib().xf_loader_open(C.byref(self.h), path.encode(), block_bytes))

    def close(self):
        if self.h:
            lib().xf_loader_close(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        self.close()

    def __iter__(self):
        return self

    def __next__(self):
        rows, nnz = C.c_uint32(), C.c_uint32()
        _check(lib().xf_loader_next(self.h, C.byref(rows), C.byref(nnz)))
        if rows.value == 0:
            raise StopIteration
        rp, kp, lp = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _check(lib().xf_loader_batch(self.h, C.byref(rp), C.byref(kp), C.byref(lp)))
        B, n = rows.value, nnz.value
        row_ptr = np.ctypeslib.as_array(C.cast(rp, C.POINTER(C.c_uint32)), (B + 1,)).copy()
        keys = np.ctypeslib.as_array(C.cast(kp, C.POINTER(C.c_uint64)), (max(n, 1),))[:n].copy()
        labels = np.ctypeslib.as_array(C.cast(lp, C.POINTER(C.c_uint8)), (B,)).copy()
        return row_ptr, keys, labels


    def next_raw(self):
        """Block formation only: the next block's raw text (b"" at end of file)."""
        text, n = C.c_void_p(), C.c_uint64()
        _check(lib().xf_loader_next_raw(self.h, C.byref(text), C.byref(n)))
        return C.string_at(text, n.value) if n.value else b""


class Table:
    def __init__(self, latent_dim=0, optimizer=OPT_FTRL, device=0, capacity=0, v_init=VINIT_DEFAULT, seed=0,
                 shard_index=0, num_shards=1, **hparams):
        L = lib()
        cfg = TableConfig()
        _check(L.xf_table_config_default(C.byref(cfg)))
        cfg.device, cfg.latent_dim, cfg.optimizer = device, latent_dim, optimizer
        cfg.capacity, cfg.v_init, cfg.seed = capacity, v_init, seed
        cfg.shard_index, cfg.num_shards = shard_index, num_shards
        for k, v in hparams.items():
            if not hasattr(cfg, k):
                raise TypeError("unknown hyper-parameter %s" % k)
            setattr(cfg, k, v)
        self.K = latent_dim
        self.cfg = cfg
        self.h = C.c_void_p()
        _check(L.xf_table_create(C.byref(self.h), C.byref(cfg)))

    def close(self):
        if getattr(self, "h", None):
            lib().xf_table_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def pull(self, keys, want_w=True, want_v=True):
        keys = np.ascontiguousarray(keys, np.uint64)
        w = np.empty(keys.size, np.float32) if want_w else None
        v = np.empty((keys.size, self.K), np.float32) if (want_v and self.K) else None
        _check(lib().xf_table_pull(self.h, _p(keys), keys.size, _p(w), _p(v)))
        return w, v

    def push(self, keys, gw=None, gv=None):
        keys = np.ascontiguousarray(keys, np.uint64)
        gw = None if gw is None else np.ascontiguousarray(gw, np.float32)
        gv = None if gv is None else np.ascontiguousarray(gv, np.float32)
        _check(lib().xf_table_push(self.h, _p(keys), keys.size, _p(gw), _p(gv)))

    def import_(self, keys, w=None, nw=None, zw=None, v=None, nv=None, zv=None):
        keys = np.ascontiguousarray(keys, np.uint64)
        arrs = [None if a is None else np.ascontiguousarray(a, np.float32) for a in (w, nw, zw, v, nv, zv)]
        _check(lib().xf_table_import(self.h, _p(keys), keys.size, *[_p(a) for a in arrs]))

    def export(self, keys):
        keys = np.ascontiguousarray(keys, np.uint64)
        n, K = keys.size, self.K
        out = dict(keys=keys, w=np.zeros(n, np.float32), nw=np.zeros(n, np.float32), zw=np.zeros(n, np.float32),
                   v=np.zeros((n, K), np.float32), nv=np.zeros((n, K), np.float32),
                   zv=np.zeros((n, K), np.float32), present=np.zeros(n, np.uint8))
        _check(lib().xf_table_export(self.h, _p(keys), n, _p(out["w"]), _p(out["nw"]), _p(out["zw"]),
                                     _p(out["v"]) if K else None, _p(out["nv"]) if K else None,
                                     _p(out["zv"]) if K else None, _p(out["present"])))
        return out

    def size(self):
        n = C.c_uint64()
        _check(lib().xf_table_size(self.h, C.byref(n)))
        return n.value

    def capacity(self):
        n = C.c_uint64()
        _check(lib().xf_table_capacity(self.h, C.byref(n)))
        return n.value

    def row_bytes(self):
        n = C.c_uint32()
        _check(lib().xf_table_row_bytes(self.h, C.byref(n)))
        return n.value

    def reserve(self, n_keys):
        _check(lib().xf_table_reserve(self.h, int(n_keys)))

    def touch_decimal_ids(self, first_id, count):
        _check(lib().xf_table_touch_decimal_ids(self.h, int(first_id), int(count)))

    def list_keys(self):
        n = self.size()
        keys = np.empty(max(n, 1), np.uint64)
        got = C.c_uint64()
        _check(lib().xf_table_list_keys(self.h, _p(keys), n, C.byref(got)))
        return keys[:min(n, got.value)]

    def save(self, path):
        _check(lib().xf_table_save(self.h, path.encode()))

    def dump_text(self, path, nonzero_only=False):
        n = C.c_uint64()
        _check(lib().xf_table_dump_text(self.h, path.encode(), int(nonzero_only), C.byref(n)))
        return n.value

    def load(self, path):
        _check(lib().xf_table_load(self.h, path.encode()))

    def save_state(self, path, user=0):
        """Exact training-state image of the table (xf_table_save_state); `user` is stored with it."""
        _check(lib().xf_table_save_state(self.h, path.encode(), int(user)))

    def load_state(self, path):
        """Load an image written by save_state into this table, which must never have held state; returns `user`."""
        user = C.c_uint64()
        _check(lib().xf_table_load_state(self.h, path.encode(), C.byref(user)))
        return user.value

    def set_stream(self, cuda_stream):
        _check(lib().xf_table_set_stream(self.h, C.c_void_p(int(cuda_stream)) if cuda_stream else None))

    def sync(self):
        _check(lib().xf_table_sync(self.h))

    def set_admission(self, mode, probability=None, threshold=None, log2_cells=None, hashes=None, decay_batches=None,
                      seed=None):
        """Feature admission of the keys training steps insert (ADMIT_ALL / ADMIT_POISSON / ADMIT_BLOOM); replaces
        the policy and clears the filter.  Unset fields keep xf_admission_config_default's values."""
        cfg = AdmissionConfig()
        _check(lib().xf_admission_config_default(C.byref(cfg)))
        cfg.mode = mode
        for k, v in dict(probability=probability, threshold=threshold, log2_cells=log2_cells, hashes=hashes,
                         decay_batches=decay_batches, seed=seed).items():
            if v is not None:
                setattr(cfg, k, v)
        _check(lib().xf_table_set_admission(self.h, C.byref(cfg)))

    def admission_stats(self):
        """Training batches, rejected tokens and keys admitted since the table was created."""
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        _check(lib().xf_table_admission_stats(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(batches=a.value, rejected_tokens=b.value, admitted_keys=c.value)

    def set_eviction(self, max_idle_batches=0, max_keys=0):
        """Feature eviction: start (or keep) per-key stamps of the last training batch and set the limits a sweep
        (evict) applies: drop keys no training batch touched among the last max_idle_batches, then keep only the
        max_keys most recently touched.  0 = no such limit; calling again replaces the limits and keeps the stamps."""
        cfg = EvictionConfig(max_idle_batches, max_keys)
        _check(lib().xf_table_set_eviction(self.h, C.byref(cfg)))

    def stop_eviction(self):
        """Stop tracking and free the stamps."""
        _check(lib().xf_table_set_eviction(self.h, None))

    def evict(self):
        """One sweep now (waits for the table's stream); returns the number of keys removed."""
        n = C.c_uint64()
        _check(lib().xf_table_evict(self.h, C.byref(n)))
        return n.value

    def last_touch(self, keys):
        """The batch number that last touched each key (np.uint64), UINT64_MAX for an absent key; never inserts."""
        keys = np.ascontiguousarray(keys, np.uint64)
        out = np.empty(keys.size, np.uint64)
        _check(lib().xf_table_last_touch(self.h, _p(keys), keys.size, _p(out)))
        return out


    def freeze(self, absent=None, prune=True, device=None):
        """A serving Model of the table as it is now (xf_table_freeze); the table is not changed.  absent: ABSENT_DEFAULT
        / ABSENT_ZERO, None = what the table's own predict does; device: None = the table's."""
        cfg = FreezeConfig(-1 if absent is None else absent, 1 if prune else 0, -1 if device is None else device)
        h = C.c_void_p()
        _check(lib().xf_table_freeze(self.h, C.byref(cfg), C.byref(h)))
        return Model(h)

    def freeze_canonical(self, absent=None, prune=True, device=None):
        """A canonical serving Model of a canonical_fm table (xf_table_freeze_canonical): rows {key, w, v[K]} served
        with the canonical FM's forward on feature values; arguments as for freeze."""
        cfg = FreezeConfig(-1 if absent is None else absent, 1 if prune else 0, -1 if device is None else device)
        h = C.c_void_p()
        _check(lib().xf_table_freeze_canonical(self.h, C.byref(cfg), C.byref(h)))
        return Model(h)

    def freeze_mvm(self, absent=None, prune=True, device=None):
        """A multi-view machine's serving Model of a canonical_fm table (xf_table_freeze_mvm): rows {key, 0, v[K]}
        served with the machine's forward on field ids and feature values (Model.predict_*_fields); arguments as for
        freeze."""
        cfg = FreezeConfig(-1 if absent is None else absent, 1 if prune else 0, -1 if device is None else device)
        h = C.c_void_p()
        _check(lib().xf_table_freeze_mvm(self.h, C.byref(cfg), C.byref(h)))
        return Model(h)

    def freeze_ffm(self, absent=None, prune=True, device=None):
        """A field-aware FM's serving Model of a canonical_fm table (xf_table_freeze_ffm): rows {key, w, v[L]} served
        with XF_MODEL_FFM's forward on field ids (< L / 4) and feature values (Model.predict_*_fields, the candidate
        and rank methods); arguments as for freeze.  The table does not record which model trained it: freeze a table
        trained with MODEL_FFM with this method, not freeze_canonical or freeze_mvm."""
        cfg = FreezeConfig(-1 if absent is None else absent, 1 if prune else 0, -1 if device is None else device)
        h = C.c_void_p()
        _check(lib().xf_table_freeze_ffm(self.h, C.byref(cfg), C.byref(h)))
        return Model(h)

    def freeze_part(self, absent=None, prune=True, device=None):
        """The part of a shard table (xf_table_freeze_part): the rows freeze would make of it, tagged with its shard;
        Model.merge of every shard's part is the whole model.  Arguments as for freeze."""
        cfg = FreezeConfig(-1 if absent is None else absent, 1 if prune else 0, -1 if device is None else device)
        h = C.c_void_p()
        _check(lib().xf_table_freeze_part(self.h, C.byref(cfg), C.byref(h)))
        return Model(h)


class Model:
    """A frozen, read-only serving model (xf_model_*): made by Table.freeze, Model.merge or Model.load; or a part of
    one (Table.freeze_part, Model.load of an XFSP file)."""

    def __init__(self, handle):
        self.h = handle

    @classmethod
    def load(cls, path, device=0):
        """The model (XFSM file) or part (XFSP file) at `path`."""
        h = C.c_void_p()
        _check(lib().xf_model_load(C.byref(h), path.encode(), device))
        return cls(h)

    @classmethod
    def merge(cls, parts, device=-1):
        """The whole model of the parts of shards 0 .. n-1 (xf_model_merge), on `device` (-1: parts[0]'s)."""
        arr = (C.c_void_p * max(len(parts), 1))(*[p.h.value for p in parts])
        h = C.c_void_p()
        _check(lib().xf_model_merge(arr, len(parts), device, C.byref(h)))
        return cls(h)

    def convert(self, precision):
        """A new Model (or part): this one with its latent fields at `precision`, PRECISION_F32 or PRECISION_F16
        (xf_model_convert); this one is not changed."""
        h = C.c_void_p()
        _check(lib().xf_model_convert(self.h, precision, C.byref(h)))
        return Model(h)

    def part_info(self):
        """(shard_index, num_shards) of a part; XflowError for a whole model."""
        s, n = C.c_int(), C.c_int()
        _check(lib().xf_model_part_info(self.h, C.byref(s), C.byref(n)))
        return s.value, n.value

    def close(self):
        if getattr(self, "h", None):
            lib().xf_model_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def info(self):
        i = ModelInfo()
        _check(lib().xf_model_get_info(self.h, C.byref(i)))
        return {k: getattr(i, k) for k, _ in ModelInfo._fields_}

    def save(self, path):
        _check(lib().xf_model_save(self.h, path.encode()))

    def predict_host(self, row_ptr, keys, vals=None):
        """Forward pass on host CSR arrays; vals: the tokens' feature values (canonical models only; None: all 1)."""
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        rows = row_ptr.size - 1
        out = np.empty(rows, np.float32)
        if vals is None:
            _check(lib().xf_model_predict_host(self.h, _p(row_ptr), _p(keys), rows, keys.size, _p(out)))
        else:
            vals = np.ascontiguousarray(vals, np.float32)
            if vals.size != keys.size:
                raise ValueError("one value per token: %d values for %d keys" % (vals.size, keys.size))
            _check(lib().xf_model_predict_host_values(self.h, _p(row_ptr), _p(keys), _p(vals), rows, keys.size, _p(out)))
        return out

    def predict_device(self, d_row_ptr, d_keys, rows, nnz, d_out, stream=0, d_vals=0):
        """Asynchronous forward pass on device pointers (raw addresses) on the CUDA stream `stream`; d_vals: the tokens'
        feature values on the device (canonical models only; 0: all 1)."""
        st = C.c_void_p(int(stream)) if stream else None
        if d_vals:
            _check(lib().xf_model_predict_device_values(self.h, _p(d_row_ptr), _p(d_keys), _p(d_vals), rows, nnz, _p(d_out), st))
        else:
            _check(lib().xf_model_predict_device(self.h, _p(d_row_ptr), _p(d_keys), rows, nnz, _p(d_out), st))

    def predict_host_fields(self, row_ptr, keys, fields, vals=None):
        """Forward pass of a multi-view machine's model (field ids < 32) or a field-aware FM's model (field ids
        < latent_dim / 4) on host CSR arrays with the tokens' field ids and feature values (None: all 1)."""
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        fields = np.ascontiguousarray(fields, np.uint8)
        if fields.size != keys.size:
            raise ValueError("one field id per token: %d field ids for %d keys" % (fields.size, keys.size))
        if vals is not None:
            vals = np.ascontiguousarray(vals, np.float32)
            if vals.size != keys.size:
                raise ValueError("one value per token: %d values for %d keys" % (vals.size, keys.size))
        rows = row_ptr.size - 1
        out = np.empty(rows, np.float32)
        _check(lib().xf_model_predict_host_fields(self.h, _p(row_ptr), _p(keys), _p(fields), _p(vals), rows, keys.size,
                                                  _p(out)))
        return out

    def predict_device_fields(self, d_row_ptr, d_keys, d_fields, rows, nnz, d_out, stream=0, d_vals=0):
        """Asynchronous forward pass of a multi-view machine's or a field-aware FM's model on device pointers (raw
        addresses) on the CUDA stream `stream`: d_fields the tokens' u8 field ids, d_vals their feature values (0: all
        1)."""
        st = C.c_void_p(int(stream)) if stream else None
        _check(lib().xf_model_predict_device_fields(self.h, _p(d_row_ptr), _p(d_keys), _p(d_fields),
                                                    _p(d_vals) if d_vals else None, rows, nnz, _p(d_out), st))

    @staticmethod
    def _candidate_batch(ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals, vals, ctx_fields, fields):
        """(CandidateBatch, the arrays it points into) for host arrays, their sizes checked."""
        ctx_ptr = np.ascontiguousarray(ctx_ptr, np.uint32)
        cand_ptr = np.ascontiguousarray(cand_ptr, np.uint32)
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        ctx_keys = np.ascontiguousarray(ctx_keys, np.uint64)
        keys = np.ascontiguousarray(keys, np.uint64)
        if ctx_ptr.size != cand_ptr.size or cand_ptr.size < 1:
            raise ValueError("one context per request: ctx_ptr has %d entries, cand_ptr %d" % (ctx_ptr.size, cand_ptr.size))

        def side(a, dtype, n, what):
            if a is None:
                return None
            a = np.ascontiguousarray(a, dtype)
            if a.size != n:
                raise ValueError("one %s per token: %d for %d keys" % (what, a.size, n))
            return a

        ctx_vals, vals = side(ctx_vals, np.float32, ctx_keys.size, "value"), side(vals, np.float32, keys.size, "value")
        ctx_fields = side(ctx_fields, np.uint8, ctx_keys.size, "field id")
        fields = side(fields, np.uint8, keys.size, "field id")
        n = row_ptr.size - 1
        b = CandidateBatch(cand_ptr.size - 1, ctx_ptr.ctypes.data, ctx_keys.ctypes.data,
                           None if ctx_vals is None else ctx_vals.ctypes.data,
                           None if ctx_fields is None else ctx_fields.ctypes.data, ctx_keys.size, cand_ptr.ctypes.data, n,
                           row_ptr.ctypes.data, keys.ctypes.data, None if vals is None else vals.ctypes.data,
                           None if fields is None else fields.ctypes.data, keys.size)
        return b, (ctx_ptr, cand_ptr, row_ptr, ctx_keys, keys, ctx_vals, vals, ctx_fields, fields)

    @staticmethod
    def _device_batch(requests, d_ctx_ptr, d_ctx_keys, ctx_nnz, d_cand_ptr, candidates, d_row_ptr, d_keys, nnz,
                      d_ctx_vals, d_vals, d_ctx_fields, d_fields):
        a = lambda x: int(x) or None
        return CandidateBatch(requests, a(d_ctx_ptr), a(d_ctx_keys), a(d_ctx_vals), a(d_ctx_fields), ctx_nnz,
                              a(d_cand_ptr), candidates, a(d_row_ptr), a(d_keys), a(d_vals), a(d_fields), nnz)

    def predict_candidates(self, ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals=None, vals=None, ctx_fields=None,
                           fields=None):
        """Score each request's candidates against its context (xf_model_predict_candidates_host): request q's context
        is ctx_keys[ctx_ptr[q] .. ctx_ptr[q+1]), its candidates rows cand_ptr[q] .. cand_ptr[q+1] - 1 of the CSR
        (row_ptr, keys).  Returns float32 [candidates]: for each candidate, the flat predict of its request's context
        followed by its own tokens, bit for bit.  Values (None: all 1) for canonical, multi-view machine and
        field-aware FM models, field ids for multi-view machine and field-aware FM models, on either side."""
        b, arrays = self._candidate_batch(ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals, vals, ctx_fields, fields)
        out = np.empty(max(arrays[2].size - 1, 0), np.float32)
        _check(lib().xf_model_predict_candidates_host(self.h, C.byref(b), _p(out)))
        return out

    def predict_candidates_device(self, requests, d_ctx_ptr, d_ctx_keys, ctx_nnz, d_cand_ptr, candidates, d_row_ptr,
                                  d_keys, nnz, d_out, stream=0, d_ctx_vals=0, d_vals=0, d_ctx_fields=0, d_fields=0):
        """Asynchronous predict_candidates on device pointers (raw addresses) on the CUDA stream `stream`; d_out
        [candidates].  A 0 address for values reads every value as 1; field ids as for predict_candidates."""
        st = C.c_void_p(int(stream)) if stream else None
        b = self._device_batch(requests, d_ctx_ptr, d_ctx_keys, ctx_nnz, d_cand_ptr, candidates, d_row_ptr, d_keys, nnz,
                               d_ctx_vals, d_vals, d_ctx_fields, d_fields)
        _check(lib().xf_model_predict_candidates_device(self.h, C.byref(b), _p(d_out), st))

    def rank_candidates(self, ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, k, ctx_vals=None, vals=None, ctx_fields=None,
                        fields=None):
        """Each request's top k candidates by pctr (xf_model_rank_candidates_host), selected on the device from the
        scores predict_candidates returns.  Returns (index uint32 [R, k], pctr float32 [R, k]): row q holds request
        q's local candidate indices (0 .. n_q - 1), highest pctr first, equal pctr by smaller index, NaN last, and
        their scores; slots past n_q hold index 0xFFFFFFFF and a NaN.  Values and field ids as for predict_candidates
        (field ids: multi-view machine and field-aware FM models)."""
        b, arrays = self._candidate_batch(ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals, vals, ctx_fields, fields)
        index = np.empty((b.requests, k), np.uint32)
        pctr = np.empty((b.requests, k), np.float32)
        _check(lib().xf_model_rank_candidates_host(self.h, C.byref(b), k, _p(index), _p(pctr)))
        return index, pctr

    def rank_candidates_device(self, requests, d_ctx_ptr, d_ctx_keys, ctx_nnz, d_cand_ptr, candidates, d_row_ptr,
                               d_keys, nnz, k, d_pctr, d_top_index, d_top_pctr=0, stream=0, d_ctx_vals=0, d_vals=0,
                               d_ctx_fields=0, d_fields=0):
        """Asynchronous rank_candidates on device pointers (raw addresses) on the CUDA stream `stream`: d_pctr
        [candidates] receives every score, d_top_index [R * k] and d_top_pctr [R * k] (0: not written) the ranking."""
        st = C.c_void_p(int(stream)) if stream else None
        b = self._device_batch(requests, d_ctx_ptr, d_ctx_keys, ctx_nnz, d_cand_ptr, candidates, d_row_ptr, d_keys, nnz,
                               d_ctx_vals, d_vals, d_ctx_fields, d_fields)
        _check(lib().xf_model_rank_candidates_device(self.h, C.byref(b), k, _p(d_pctr) if d_pctr else None,
                                                     _p(d_top_index) if d_top_index else None,
                                                     _p(d_top_pctr) if d_top_pctr else None, st))

    def lookup(self, keys):
        """What the model holds for `keys`: dict of w, st, qt (0 for LR) and present."""
        keys = np.ascontiguousarray(keys, np.uint64)
        n = keys.size
        out = dict(keys=keys, w=np.zeros(n, np.float32), st=np.zeros(n, np.float32), qt=np.zeros(n, np.float32),
                   present=np.zeros(n, np.uint8))
        _check(lib().xf_model_lookup(self.h, _p(keys), n, _p(out["w"]), _p(out["st"]), _p(out["qt"]), _p(out["present"])))
        return out

    def lookup_latent(self, keys):
        """What a canonical, multi-view machine's or field-aware FM's model holds for `keys`: dict of w (0 for a
        multi-view machine), v [n, K] and present."""
        keys = np.ascontiguousarray(keys, np.uint64)
        n, K = keys.size, self.info()["latent_dim"]
        out = dict(keys=keys, w=np.zeros(n, np.float32), v=np.zeros((n, K), np.float32), present=np.zeros(n, np.uint8))
        _check(lib().xf_model_lookup_latent(self.h, _p(keys), n, _p(out["w"]), _p(out["v"]), _p(out["present"])))
        return out

    def predict_ingested(self, trainer, row_start, row_end):
        """Trainer.predict_ingested on the trainer's current ingested block, read from this model."""
        n = row_end - row_start
        p = np.empty(n, np.float32)
        lab = np.empty(n, np.uint8)
        _check(lib().xf_model_predict_ingested(self.h, trainer.h, row_start, row_end, _p(p), _p(lab)))
        return p, lab

    def fingerprint(self):
        """The order-free u64 of the model's contents (xf_model_fingerprint)."""
        f = C.c_uint64()
        _check(lib().xf_model_fingerprint(self.h, C.byref(f)))
        return f.value

    def diff(self, next_model):
        """The Delta that carries this model to `next_model` (xf_model_diff); neither model changes."""
        h = C.c_void_p()
        _check(lib().xf_model_diff(self.h, next_model.h, C.byref(h)))
        return Delta(h)

    def apply(self, delta):
        """A new Model: this one with `delta` applied (xf_model_apply_delta); this one is not changed."""
        h = C.c_void_p()
        _check(lib().xf_model_apply_delta(self.h, delta.h, C.byref(h)))
        return Model(h)


class Delta:
    """The difference between two serving models (xf_delta_*): made by Model.diff or Delta.load."""

    def __init__(self, handle):
        self.h = handle

    @classmethod
    def load(cls, path, device=0):
        h = C.c_void_p()
        _check(lib().xf_delta_load(C.byref(h), path.encode(), device))
        return cls(h)

    def close(self):
        if getattr(self, "h", None):
            lib().xf_delta_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def info(self):
        i = DeltaInfo()
        _check(lib().xf_delta_get_info(self.h, C.byref(i)))
        return {k: getattr(i, k) for k, _ in DeltaInfo._fields_}

    def save(self, path):
        _check(lib().xf_delta_save(self.h, path.encode()))


class Comm:
    @staticmethod
    def new_id():
        buf = np.zeros(COMM_ID_BYTES, np.uint8)
        _check(lib().xf_comm_get_id(_p(buf)))
        return buf

    def __init__(self, comm_id, rank, nranks, device):
        comm_id = np.ascontiguousarray(comm_id, np.uint8)
        self.rank, self.nranks = rank, nranks
        self.h = C.c_void_p()
        _check(lib().xf_comm_create(C.byref(self.h), _p(comm_id), rank, nranks, device))

    def barrier(self):
        _check(lib().xf_comm_barrier(self.h))

    def close(self):
        if getattr(self, "h", None):
            lib().xf_comm_destroy(self.h)
            self.h = None


class ProgressiveValidation:
    """A streaming, binned metric on the device (xf_pv_*): 20 * 2^mantissa_bits + 1 bins of the prediction, exact
    integer sums, a report that depends only on the rows added.  Fed by add_device or by Trainer.set_validation."""

    def __init__(self, device=0, mantissa_bits=10):
        self.device = device
        self.num_slices = 0
        self.h = C.c_void_p()
        _check(lib().xf_pv_create(C.byref(self.h), int(device), int(mantissa_bits)))

    def close(self):
        if getattr(self, "h", None):
            _check(lib().xf_pv_destroy(self.h))
            self.h = None

    def __del__(self):
        if getattr(self, "h", None):
            lib().xf_pv_destroy(self.h)
            self.h = None

    def add_device(self, d_pctr, d_labels, n, d_weights=None, stream=0):
        """n predictions (float32), labels (uint8) and weights (float32 or None: all 1) at device addresses."""
        _check(lib().xf_pv_add_device(self.h, _p(d_pctr), _p(d_labels), _p(d_weights) if d_weights else None, int(n),
                                      _p(stream) if stream else None))

    def report_bytes(self):
        """The raw struct xf_pv_report, for byte comparisons."""
        r = PvReport()
        _check(lib().xf_pv_report(self.h, C.byref(r)))
        return bytes(r)

    def report(self):
        r = PvReport.from_buffer_copy(self.report_bytes())
        return {name: getattr(r, name) for name, _ in PvReport._fields_}

    def reset(self):
        _check(lib().xf_pv_reset(self.h))

    def set_slices(self, keys, slice_of, num_slices, mantissa_bits=8):
        """The slice map: keys[i] (uint64) names slice slice_of[i] (< num_slices).  Clears every sum; num_slices = 0
        with no keys removes slicing."""
        keys = np.ascontiguousarray(keys, np.uint64)
        slice_of = np.ascontiguousarray(slice_of, np.uint32)
        if keys.size != slice_of.size:
            raise ValueError("keys and slice_of differ in length")
        _check(lib().xf_pv_set_slices(self.h, _p(keys), _p(slice_of), keys.size, int(num_slices), int(mantissa_bits)))
        self.num_slices = int(num_slices)

    def add_device_rows(self, d_pctr, d_labels, d_row_ptr, d_keys, rows, d_weights=None, stream=0):
        """add_device plus each row's tokens: keys d_keys[row_ptr[r] .. row_ptr[r + 1]) (uint32 row_ptr, uint64 keys at
        device addresses), which name its slices."""
        _check(lib().xf_pv_add_device_rows(self.h, _p(d_pctr), _p(d_labels), _p(d_weights) if d_weights else None,
                                           _p(d_row_ptr), _p(d_keys), int(rows), _p(stream) if stream else None))

    def report_slices_bytes(self, n=None):
        """The raw struct xf_pv_report of each slice, in slice order, for byte comparisons."""
        n = self.num_slices if n is None else int(n)
        arr = (PvReport * max(n, 1))()
        _check(lib().xf_pv_report_slices(self.h, arr, n))
        return [bytes(arr[s]) for s in range(n)]

    def report_slices(self):
        out = []
        for raw in self.report_slices_bytes():
            r = PvReport.from_buffer_copy(raw)
            out.append({name: getattr(r, name) for name, _ in PvReport._fields_})
        return out


class GroupMetric:
    """Exact per-group AUC and logloss of held-out predictions on the device (xf_group_metric_*), keyed by one uint64
    group id per row, and their row-weighted mean (GAUC).  The report depends only on the rows added."""

    def __init__(self, device=0):
        self.device = device
        self.last_groups = 0  # the group count of the last finish
        self.h = C.c_void_p()
        _check(lib().xf_group_metric_create(C.byref(self.h), int(device)))

    def close(self):
        if getattr(self, "h", None):
            _check(lib().xf_group_metric_destroy(self.h))
            self.h = None

    def __del__(self):
        self.close()

    def add_device(self, d_pctr, d_labels, d_groups, n, stream=0):
        """n predictions (float32), labels (uint8, != 0 positive) and group ids (uint64) at device addresses."""
        _check(lib().xf_group_metric_add_device(self.h, _p(d_pctr), _p(d_labels), _p(d_groups), int(n),
                                                _p(stream) if stream else None))

    def finish_bytes(self):
        """The raw struct xf_group_report, for byte comparisons."""
        r = GroupReport()
        _check(lib().xf_group_metric_finish(self.h, C.byref(r)))
        self.last_groups = r.groups
        return bytes(r)

    def finish(self):
        r = GroupReport.from_buffer_copy(self.finish_bytes())
        return {name: getattr(r, name) for name, _ in GroupReport._fields_}

    def groups(self, n=None):
        """The last finish's groups in ascending id order: ids, rows, positives, auc, logloss (numpy arrays).  n
        defaults to that finish's group count."""
        n = self.last_groups if n is None else int(n)
        out = dict(ids=np.empty(n, np.uint64), rows=np.empty(n, np.uint64), positives=np.empty(n, np.uint64),
                   auc=np.empty(n, np.float64), logloss=np.empty(n, np.float64))
        _check(lib().xf_group_metric_groups(self.h, n, _p(out["ids"]), _p(out["rows"]), _p(out["positives"]),
                                            _p(out["auc"]), _p(out["logloss"])))
        return out

    def topk_bytes(self, k):
        """The raw struct xf_group_topk_report of topk(k), for byte comparisons."""
        r = GroupTopkReport()
        _check(lib().xf_group_metric_topk(self.h, int(k), C.byref(r)))
        return bytes(r)

    def topk(self, k):
        """Ranking quality at cutoff k of the last finish's rows (xf_group_metric_topk): k, groups, scored_groups,
        scored_rows and ndcg, precision, recall with their unweighted _mean, over the groups finish scores."""
        r = GroupTopkReport.from_buffer_copy(self.topk_bytes(k))
        return {name: getattr(r, name) for name, _ in GroupTopkReport._fields_}

    def groups_topk(self, n=None):
        """The last topk's per-group ndcg, precision and recall (numpy float64, NaN for a group without positives), in
        the order of groups().  n defaults to the last finish's group count."""
        n = self.last_groups if n is None else int(n)
        out = dict(ndcg=np.empty(n, np.float64), precision=np.empty(n, np.float64), recall=np.empty(n, np.float64))
        _check(lib().xf_group_metric_groups_topk(self.h, n, _p(out["ndcg"]), _p(out["precision"]),
                                                 _p(out["recall"])))
        return out

    def reset(self):
        _check(lib().xf_group_metric_reset(self.h))


class Trainer:
    def __init__(self, table, model=MODEL_LR, max_rows=65536, max_nnz=65536 * 64, keep_loss=False, comm=None):
        cfg = TrainerConfig(model, max_rows, max_nnz, 1 if keep_loss else 0)
        self.table = table
        self.comm = comm
        self.h = C.c_void_p()
        _check(lib().xf_trainer_create(C.byref(self.h), table.h, comm.h if comm else None, C.byref(cfg)))

    def close(self):
        if getattr(self, "h", None):
            lib().xf_trainer_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def init_push(self):
        _check(lib().xf_trainer_init_push(self.h))

    def step_host(self, row_ptr, keys, labels, want_loss=True):
        """One update() on host CSR arrays (numpy or raw pinned addresses with explicit sizes)."""
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        labels = np.ascontiguousarray(labels, np.uint8)
        loss = C.c_float()
        _check(lib().xf_trainer_step_host(self.h, _p(row_ptr), _p(keys), _p(labels), labels.size, keys.size,
                                          C.byref(loss) if want_loss else None))
        return loss.value if want_loss else None

    def step_host_weighted(self, row_ptr, keys, labels, weights, want_loss=True):
        """One step on host CSR arrays with a weight per row (see xf_trainer_step_host_weighted)."""
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        labels = np.ascontiguousarray(labels, np.uint8)
        weights = np.ascontiguousarray(weights, np.float32)
        if weights.size != labels.size:
            raise ValueError("one weight per row: %d weights for %d rows" % (weights.size, labels.size))
        loss = C.c_float()
        _check(lib().xf_trainer_step_host_weighted(self.h, _p(row_ptr), _p(keys), _p(labels), _p(weights), labels.size,
                                                   keys.size, C.byref(loss) if want_loss else None))
        return loss.value if want_loss else None

    def step_device_weighted(self, d_row_ptr, d_keys, d_labels, d_weights, rows, nnz):
        _check(lib().xf_trainer_step_device_weighted(self.h, _p(d_row_ptr), _p(d_keys), _p(d_labels), _p(d_weights),
                                                     rows, nnz))

    def set_negative_sampling(self, rate, seed=0):
        """Keep each negative row of every later training step with probability `rate`, weighted 1 / rate (1: off)."""
        _check(lib().xf_trainer_set_negative_sampling(self.h, float(rate), int(seed)))

    def set_validation(self, pv):
        """Every later training step adds its rows' pre-update predictions to `pv` (a ProgressiveValidation); None
        detaches.  The trainer keeps a reference so that the pv outlives the attachment."""
        _check(lib().xf_trainer_set_validation(self.h, pv.h if pv is not None else None))
        self.pv = pv

    def set_deterministic(self, on=True):
        """Canonical FM / multi-view machine trainers: sum each key's gradient in token order (xf_trainer_set_deterministic),
        so that runs on the same batches give the same bits; False restores the default atomic kernels."""
        _check(lib().xf_trainer_set_deterministic(self.h, 1 if on else 0))

    def skipped_rows(self):
        """Rows trained with effective weight 0 since the trainer was created."""
        n = C.c_uint64()
        _check(lib().xf_trainer_skipped_rows(self.h, C.byref(n)))
        return n.value

    def step_host_values(self, row_ptr, keys, vals, labels):
        """One step of the canonical FM (XF_MODEL_FM_CANONICAL) on host CSR arrays with feature values."""
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        vals = None if vals is None else np.ascontiguousarray(vals, np.float32)
        labels = np.ascontiguousarray(labels, np.uint8)
        loss = C.c_float()
        _check(lib().xf_trainer_step_host_values(self.h, _p(row_ptr), _p(keys), _p(vals), _p(labels), labels.size, keys.size,
                                                 C.byref(loss)))
        return loss.value

    def predict_host_values(self, row_ptr, keys, vals):
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        vals = None if vals is None else np.ascontiguousarray(vals, np.float32)
        rows = row_ptr.size - 1
        out = np.empty(rows, np.float32)
        _check(lib().xf_trainer_predict_host_values(self.h, _p(row_ptr), _p(keys), _p(vals), rows, keys.size, _p(out)))
        return out

    def step_host_fields(self, row_ptr, keys, fields, vals, labels):
        """One step of the defined multi-view machine (XF_MODEL_MVM, field ids < 32) or the field-aware FM
        (XF_MODEL_FFM, field ids < latent_dim / 4): host CSR arrays + the tokens' field ids; vals may be None (all 1)."""
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        fields = np.ascontiguousarray(fields, np.uint8)
        vals = None if vals is None else np.ascontiguousarray(vals, np.float32)
        labels = np.ascontiguousarray(labels, np.uint8)
        loss = C.c_float()
        _check(lib().xf_trainer_step_host_fields(self.h, _p(row_ptr), _p(keys), _p(fields), _p(vals), _p(labels), labels.size,
                                                 keys.size, C.byref(loss)))
        return loss.value

    def predict_host_fields(self, row_ptr, keys, fields, vals):
        """Forward only of an XF_MODEL_MVM or XF_MODEL_FFM trainer on host CSR arrays + field ids; returns pctr[rows]."""
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        fields = np.ascontiguousarray(fields, np.uint8)
        vals = None if vals is None else np.ascontiguousarray(vals, np.float32)
        rows = row_ptr.size - 1
        out = np.empty(rows, np.float32)
        _check(lib().xf_trainer_predict_host_fields(self.h, _p(row_ptr), _p(keys), _p(fields), _p(vals), rows, keys.size, _p(out)))
        return out

    def step_host_raw(self, row_ptr_addr, keys_addr, labels_addr, rows, nnz, want_loss=True):
        loss = C.c_float()
        _check(lib().xf_trainer_step_host(self.h, _p(row_ptr_addr), _p(keys_addr), _p(labels_addr), rows, nnz,
                                          C.byref(loss) if want_loss else None))
        return loss.value if want_loss else None

    def step_host_async(self, row_ptr_addr, keys_addr, labels_addr, rows, nnz, out_addr=None):
        """Pipelined step on page-locked buffers given by address; never blocks on the device."""
        _check(lib().xf_trainer_step_host_async(self.h, _p(row_ptr_addr), _p(keys_addr), _p(labels_addr), rows, nnz,
                                                _p(out_addr) if out_addr else None))

    def step_host_ids_async(self, row_ptr_addr, ids_addr, labels_addr, rows, nnz, out_addr=None):
        """Like step_host_async but with u32 feature ids (hashed to keys on the device)."""
        _check(lib().xf_trainer_step_host_ids_async(self.h, _p(row_ptr_addr), _p(ids_addr), _p(labels_addr), rows,
                                                    nnz, _p(out_addr) if out_addr else None))

    def ingest_text(self, text: bytes):
        """Parse one text block on the device; returns (rows, nnz) of the CSR now resident there."""
        rows, nnz = C.c_uint32(), C.c_uint32()
        buf = C.create_string_buffer(text, len(text))
        _check(lib().xf_trainer_ingest_text(self.h, C.cast(buf, C.c_void_p), len(text), C.byref(rows), C.byref(nnz)))
        return rows.value, nnz.value

    def ingested_export(self, rows, nnz):
        rp = np.empty(rows + 1, np.uint32)
        keys = np.empty(nnz, np.uint64)
        lab = np.empty(rows, np.uint8)
        _check(lib().xf_trainer_ingested_export(self.h, _p(rp), _p(keys), _p(lab)))
        return rp, keys, lab

    def step_ingested(self, row_start, row_end):
        _check(lib().xf_trainer_step_ingested(self.h, row_start, row_end))

    def predict_ingested(self, row_start, row_end):
        n = row_end - row_start
        p = np.empty(n, np.float32)
        lab = np.empty(n, np.uint8)
        _check(lib().xf_trainer_predict_ingested(self.h, row_start, row_end, _p(p), _p(lab)))
        return p, lab

    def wait_uploads(self):
        _check(lib().xf_trainer_wait_uploads(self.h))

    def set_profile(self, on):
        _check(lib().xf_trainer_set_profile(self.h, 1 if on else 0))

    def profile(self):
        ms = (C.c_double * 2)()
        steps = C.c_uint64()
        _check(lib().xf_trainer_profile(self.h, ms, C.byref(steps)))
        return dict(step_ms=ms[0], update_ms=ms[1], steps=steps.value)

    def step_device(self, d_row_ptr, d_keys, d_labels, rows, nnz):
        _check(lib().xf_trainer_step_device(self.h, _p(d_row_ptr), _p(d_keys), _p(d_labels), rows, nnz))

    def predict_host(self, row_ptr, keys):
        row_ptr = np.ascontiguousarray(row_ptr, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        rows = row_ptr.size - 1
        out = np.empty(rows, np.float32)
        _check(lib().xf_trainer_predict_host(self.h, _p(row_ptr), _p(keys), rows, keys.size, _p(out)))
        return out

    def get_loss(self, rows):
        out = np.empty(rows, np.float32)
        _check(lib().xf_trainer_get_loss(self.h, _p(out), rows))
        return out

    def stats(self):
        a, b, c, d = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
        _check(lib().xf_trainer_stats(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return dict(steps=a.value, rows=b.value, nnz=c.value, unique_keys=d.value)

    def launches(self):
        n = C.c_uint64()
        _check(lib().xf_trainer_launches(self.h, C.byref(n)))
        return n.value

    def sync(self):
        _check(lib().xf_trainer_sync(self.h))

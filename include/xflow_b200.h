/*
 * xflow_b200 — C ABI of the H100-native drop-in for xflow's data-parallel hot path.
 *
 * Plain C: pointers, sizes and POD structs only (no torch / STL types).  Every entry point below is
 * what the reference's FFI for this path binds; the comment on each names the reference interface it
 * replaces (paths relative to the xswang/xflow tree).  All functions return 0 on success and a
 * negative code on failure (never throw across the ABI); xf_last_error() describes the last failure
 * of the calling thread.  There is NO CPU fallback: without a CUDA device every compute entry point
 * fails with XF_ERR_CUDA.
 *
 * Layers
 *   1. reference C API        XFCreate / XFStartTrain                    (src/c_api/c_api.h:26-29)
 *   2. parameter table        xf_table_*   = KVServer + FTRL/SGD handle  (src/model/server.h:20-35,
 *                                            src/optimizer/ftrl.h, sgd.h ; ps-lite kv_app.h:110-165)
 *   3. fused worker step      xf_trainer_* = LRWorker/FMWorker::update + predict
 *                                            (src/model/lr/lr_worker.cc:25-177, fm/fm_worker.cc:25-245)
 *   4. host ingest            xf_loader_*, xf_hash_* = LoadData::load_minibatch_hash_data_fread
 *                                            (src/io/load_data_from_disk.cc:103-210)
 *   5. multi-GPU exchange     xf_comm_*    = KVWorker slicing + Van transport
 *                                            (ps-lite kv_app.h:405-460, postoffice.cc:134-143)
 *   6. serving model          xf_model_*   = a trained table frozen for prediction only (no reference counterpart:
 *                                            the reference predicts on its training servers, lr_worker.cc:25-77)
 *   7. serving model deltas   xf_model_diff / _apply_delta, xf_delta_* = one model carried to the next
 *   8. progressive validation xf_pv_*      = each training row scored before its step learns from it
 */
#ifndef XFLOW_B200_H_
#define XFLOW_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
#define XF_DLL extern "C" __attribute__((visibility("default")))
#else
#define XF_DLL __attribute__((visibility("default")))
#endif

enum {
  XF_OK = 0,
  XF_ERR_ARG = -1,       /* bad argument */
  XF_ERR_CUDA = -2,      /* CUDA runtime error (incl. "no device") */
  XF_ERR_FULL = -3,      /* no room: capacity past 2^31 slots, or a probe sequence overflowed (sticky, see
                            "Probe overflow" above xf_table_pull) */
  XF_ERR_IO = -4,        /* file open / read failure (reference: exit(1), io.h:33-36) */
  XF_ERR_COMM = -5,      /* NCCL failure */
  XF_ERR_STATE = -6
};

enum { XF_MODEL_LR = 0, XF_MODEL_FM = 1,              /* main.cc:26-39: '0' = LR, '1' = FM */
       XF_MODEL_FM_CANONICAL = 2,                     /* NOT the reference's model: the textbook FM, see below */
       XF_MODEL_MVM = 3,                              /* a DEFINED multi-view machine (mvm_worker.cc is not), see below */
       XF_MODEL_FFM = 4 };                            /* the field-aware FM (libffm's model), see below */
enum { XF_OPTIMIZER_FTRL = 0, XF_OPTIMIZER_SGD = 1, /* server.h:24-29 (comment toggle in the reference) */
       XF_OPTIMIZER_ADAGRAD = 2 };                    /* NOT the reference's: per-coordinate AdaGrad, see section 2 */
enum {
  XF_VINIT_DEFAULT = 0,  /* FTRL: N(0,1)*1e-2 (ftrl.h:114-120, counter-based here); SGD: 0.001 (sgd.h:68-70) */
  XF_VINIT_COUNTER = 1,  /* counter-based N(0,1)*1e-2 keyed by (key,k,seed) for either optimizer */
  XF_VINIT_ZERO = 3      /* zeros (used before xf_table_import of a replayed table) */
};

XF_DLL const char* xf_last_error(void);
XF_DLL int xf_version(void);
/* number of CUDA devices visible (0 without a GPU; never fails) */
XF_DLL int xf_device_count(void);

/* ------------------------------------------------------------------------------------------------
 * 2. Parameter table
 * ---------------------------------------------------------------------------------------------- */
typedef struct xf_table xf_table;

typedef struct xf_table_config {
  int device;            /* CUDA ordinal */
  int latent_dim;        /* K: 0 = LR (app 0 only); >0 = FM (apps 0 and 1).  ftrl.h:16 / fm_worker.h:92 default 10 */
  int optimizer;         /* XF_OPTIMIZER_* */
  float alpha;           /* ftrl.h:17  default 5e-2 */
  float beta;            /* ftrl.h:18  default 1.0  */
  float lambda1;         /* ftrl.h:19  default 5e-5 */
  float lambda2;         /* ftrl.h:20  default 10.0 */
  float learning_rate;   /* sgd.h:16   default 1e-3 */
  int v_init;            /* XF_VINIT_* */
  uint64_t seed;
  uint64_t capacity;     /* initial slot count (rounded up to a power of two); 0 = 1<<20.  Grows on demand. */
  int shard_index;       /* this table owns keys of shard_index out of num_shards (postoffice.cc:134-143) */
  int num_shards;        /* 1 = whole key space */
  int canonical_fm;      /* 1: rows carry the accumulators of XF_MODEL_FM_CANONICAL / XF_MODEL_MVM / XF_MODEL_FFM
                            (latent_dim in {4,8,16,32,64,128}) */
} xf_table_config;

/* XF_OPTIMIZER_ADAGRAD (not the reference's; libffm's optimizer).  Per coordinate (w, and each v_k of a latent
 * table), with g the float the FTRL or SGD step would receive (after the division by rows), eta = learning_rate and
 * beta = beta, every operation float32 rounded to nearest, no FMA:
 *     n' = fl(n + fl(g * g))
 *     w' = fl(w - fl( fl(eta * g) / fl(sqrt_rn(fl(beta + n'))) ))
 * beta plays the accumulator's start (beta = 1 is libffm's start in exact arithmetic); alpha, lambda1 and lambda2 are
 * unused (no regularisation).  xf_table_create refuses, with XF_ERR_ARG naming the field, beta that is not a finite
 * number above 0 and eta that is not finite.  A fresh row has n = 0; XF_VINIT_DEFAULT resolves to the counter-based
 * N(0,1)*1e-2, as for FTRL.  A zero gradient leaves w and n unchanged.  Row layout: n in the head's n field with z = 0;
 * latent block v[K], its accumulators, then nv[K] and no zv (FM K = 16: 192 bytes against FTRL's 256); a lazy LR row's
 * state word holds (w, n).  xf_table_export reports nw = n, zw = 0, nv = n, zv = 0; xf_table_import takes nw and nv and
 * ignores zw and zv; xf_table_save writes has_nz = 1 with zero z fields.  State images load only into a table with
 * the same optimizer; serving models record optimizer 2. */

/* fills *cfg with the reference's compile-time defaults (ftrl.h:15-20, sgd.h:16) */
XF_DLL int xf_table_config_default(xf_table_config* cfg);

/* replaces: new ps::KVServer<float>(0/1) + set_request_handle(FTRL/SGD handle)  (server.h:22-31) */
XF_DLL int xf_table_create(xf_table** out, const xf_table_config* cfg);
XF_DLL int xf_table_destroy(xf_table* t);

/* Keys.  Any u64 but 2^64 - 1, which marks an empty slot of the table (the reference has no server range that holds
 * it either).  The entry points that take keys from HOST memory refuse it with XF_ERR_ARG, naming it, before anything
 * is enqueued: xf_table_pull, _push, _import, _export, _last_touch, and xf_trainer_step_host / _predict_host with
 * their _values and _fields forms.  The device-pointer entry points (xf_table_pull_device / _push_device,
 * xf_trainer_step_device*), the _async steps, the id and text-ingest paths do not look: that would be one more pass
 * over every batch on the paths that carry the bulk of the training data, and a key hashed on the device is 2^64 - 1
 * with probability 2^-64 per id.  There the key is the caller's contract.
 *
 * Probe overflow.  A lookup visits at most 8192 slots (XF_MAX_PROBE) of its key's probe sequence.  Growth keeps the
 * load at or below 0.75, so hashed keys never come near that; but keys that share one probe sequence form a single
 * chain whatever the capacity, and once 8192 of them are present, inserting or even looking up another key of that
 * sequence overflows, at any capacity.  The call reports XF_ERR_FULL ("table probe sequence overflowed"); a training
 * step reports it at the next call that checks the table: xf_trainer_sync, xf_table_sync, a predict, or a table call
 * below that returns data to the host.  The key or token that overflowed is skipped.  The error is sticky: nothing
 * clears it, and every later such call on the table returns XF_ERR_FULL. */

/* replaces: KVWorker<float>::Pull + Wait (kv_app.h:147-165) served by KVServerFTRLHandle_w/_v pull
 * branch (ftrl.h:49-52,75-77,108-111,142-144 ; sgd.h).  keys: n host u64 (any order, duplicates allowed
 * for pulls).  w_out: n floats or NULL.  v_out: n*K floats (row-major) or NULL.  Missing keys are
 * inserted with the optimizer's default contents, as `store[key]` does. */
XF_DLL int xf_table_pull(xf_table* t, const uint64_t* keys, uint64_t n, float* w_out, float* v_out);

/* replaces: KVWorker<float>::Push + Wait (kv_app.h:110-118) served by the handles' push branch
 * (ftrl.h:54-74,112-141 ; sgd.h:46-52,90-96).  keys must be unique, in any order (KVWorker::Push takes them
 * sorted and unique; a repeated key is refused with XF_ERR_ARG before anything is applied).  gw: n floats or
 * NULL (app 0); gv: n*K floats or NULL (app 1). */
XF_DLL int xf_table_push(xf_table* t, const uint64_t* keys, uint64_t n, const float* gw, const float* gv);

/* same two operations on DEVICE pointers, asynchronous on the table's stream (no host sync).  The device push
 * does not look for repeated keys (that would take a sort): unique keys are the caller's contract there. */
XF_DLL int xf_table_pull_device(xf_table* t, const uint64_t* d_keys, uint64_t n, float* d_w_out, float* d_v_out);
XF_DLL int xf_table_push_device(xf_table* t, const uint64_t* d_keys, uint64_t n, const float* d_gw, const float* d_gv);

/* Overwrite / read full optimizer state of given keys (host arrays; any pointer but keys may be NULL).
 * The reference has no checkpoint (SURVEY §5); these exist for parity replay and save/restore.
 * export does NOT insert: present[i] = 0 and zeros for unknown keys. */
XF_DLL int xf_table_import(xf_table* t, const uint64_t* keys, uint64_t n, const float* w, const float* nw,
                           const float* zw, const float* v, const float* nv, const float* zv);
XF_DLL int xf_table_export(xf_table* t, const uint64_t* keys, uint64_t n, float* w, float* nw, float* zw,
                           float* v, float* nv, float* zv, uint8_t* present);

XF_DLL int xf_table_size(xf_table* t, uint64_t* n_keys);        /* = store.size() */
XF_DLL int xf_table_capacity(xf_table* t, uint64_t* n_slots);
XF_DLL int xf_table_row_bytes(xf_table* t, uint32_t* bytes);
XF_DLL int xf_table_latent_dim(xf_table* t, int* latent_dim);   /* K of the table (0 = LR) */
/* make room for at least n_keys keys at load factor <= 0.5 (rehashes on device if needed) */
XF_DLL int xf_table_reserve(xf_table* t, uint64_t n_keys);
/* Pre-populate: make the keys of the integer feature ids [first_id, first_id + count) exist with default
 * contents, as a Pull of them would (store[key], ftrl.h:56,114-120); ids are hashed on the device as their
 * decimal strings (load_data_from_disk.cc:151).  A sharded table keeps only the keys of its own range.
 * Asynchronous on the table's stream. */
XF_DLL int xf_table_touch_decimal_ids(xf_table* t, uint64_t first_id, uint64_t count);
/* copy up to max_keys live keys to host; *n_out = number of live keys */
XF_DLL int xf_table_list_keys(xf_table* t, uint64_t* keys_out, uint64_t max_keys, uint64_t* n_out);
/* binary checkpoint of the whole shard (keys + full optimizer state) */
XF_DLL int xf_table_save(xf_table* t, const char* path);
XF_DLL int xf_table_load(xf_table* t, const char* path);
/* text model dump, one "<key>\t<w>[\t<v_0> ... <v_K-1>]" line per key in key order (weights only, %.9g);
 * nonzero_only skips keys whose weights are all exactly 0 (FTRL's L1 zeros).  *written = lines (may be NULL) */
XF_DLL int xf_table_dump_text(xf_table* t, const char* path, int nonzero_only, uint64_t* written);
/* use an external CUDA stream (cudaStream_t passed as void*) for all table work; NULL = own stream */
XF_DLL int xf_table_set_stream(xf_table* t, void* cuda_stream);
XF_DLL int xf_table_sync(xf_table* t);

/* Feature admission (McMahan et al., "Ad Click Prediction: a View from the Trenches", section 5.1).  A per-table
 * policy for the keys that TRAINING STEPS insert; explicit pull / push / import / load, xf_table_touch_decimal_ids,
 * xf_trainer_init_push and the ps-lite functors still insert as `store[key]` does.  The table numbers its training
 * batches b = 0, 1, 2, ...; in batch b a token whose key is absent from the table is
 *   XF_ADMIT_ALL      inserted (the default: today's behaviour);
 *   XF_ADMIT_POISSON  inserted iff u24(key, b) < floor(probability * 2^24), u24 = the top 24 bits of
 *                     splitmix64(key ^ splitmix64(seed + b)) (all tokens of one key in one batch decide alike);
 *   XF_ADMIT_BLOOM    inserted iff min_j cell[c_j] >= threshold, over the key's cells
 *                     c_j = top log2_cells bits of splitmix64(key ^ splitmix64(seed + (j+1) * 0x9E3779B97F4A7C15)),
 *                     j < hashes, in 2^log2_cells one-byte counters as they stood BEFORE batch b.  After the step
 *                     every rejected token adds 1 to each of its cells (once per j), saturating at 255; then, if
 *                     decay_batches > 0 and (b+1) % decay_batches == 0, every cell is halved.
 * A rejected token reads as a row of zeros that nobody updates: w = 0 (FM: v = 0), no gradient, no optimizer step,
 * not counted in unique_keys.  An admitted key starts as an inserted key always does.  With a policy other than
 * XF_ADMIT_ALL, predict never inserts: an absent key contributes 0.
 * Single-GPU tables only: refused on canonical tables (canonical_fm = 1), on tables with num_shards > 1, and by
 * xf_trainer_create with a multi-rank comm.  The filter lives in device memory owned by the table (2^log2_cells
 * bytes).  It is part of the state image (xf_table_save_state), not of the portable xf_table_save format. */
enum { XF_ADMIT_ALL = 0, XF_ADMIT_POISSON = 1, XF_ADMIT_BLOOM = 2 };
typedef struct xf_admission_config {
  int mode;                /* XF_ADMIT_* */
  float probability;       /* POISSON: 0..1 */
  uint32_t threshold;      /* BLOOM: 1..255 occurrences before a key is admitted */
  uint32_t log2_cells;     /* BLOOM: 10..36 (2^log2_cells bytes of filter) */
  uint32_t hashes;         /* BLOOM: 1..8 */
  uint64_t decay_batches;  /* BLOOM: halve the filter every decay_batches training batches; 0 = never */
  uint64_t seed;
} xf_admission_config;
/* mode XF_ADMIT_ALL, probability 1, threshold 2, log2_cells 30, hashes 3, decay_batches 0, seed 0 */
XF_DLL int xf_admission_config_default(xf_admission_config* cfg);
/* replaces the table's policy and clears the filter (XF_ADMIT_ALL frees it); on failure the table is unchanged */
XF_DLL int xf_table_set_admission(xf_table* t, const xf_admission_config* cfg);
/* since the table was created: training batches, rejected tokens, keys inserted by admission (any pointer may be
 * NULL; reads device counters, waits for the table's stream) */
XF_DLL int xf_table_admission_stats(xf_table* t, uint64_t* batches, uint64_t* rejected_tokens, uint64_t* admitted_keys);

/* Feature eviction: per-key stamps of the last training batch, and sweeps that drop idle keys or keep a key budget.
 * Batch numbers b are admission's: 0, 1, 2, ... per non-empty training step on the table (an empty batch is not one).
 * With tracking on, every present key k carries a stamp last(k), a 32-bit batch number:
 *   - a training step of batch b sets last(k) = b for every key one of its tokens reads from a row, including the
 *     keys the step inserts or admits; a token that admission rejects stamps nothing (its key has no row);
 *   - any other insertion (predict's insert-on-pull, xf_table_pull / _push / _import / _load,
 *     xf_table_touch_decimal_ids, xf_trainer_init_push, the ps-lite functors) sets last(k) = the number of training
 *     batches run so far;
 *   - reading or updating an existing key outside a training step (predict, pull, push, import, export) leaves its
 *     stamp alone;
 *   - when tracking starts, every key already present gets the number of training batches run so far.
 * A sweep (xf_table_evict) runs at the current batch number B, stream-ordered after everything enqueued on the
 * table's stream.  It removes
 *   1. with max_idle_batches = T > 0: every key with last(k) < B - T (no training batch among the last T touched
 *      it; nothing when B <= T);
 *   2. with max_keys = N > 0: of the keys left, all but the N most recently touched, where a larger stamp is more
 *      recent and, between equal stamps, the smaller 64-bit key is.  Exactly min(N, keys left) keys survive.
 * An evicted key is absent, as if never inserted: its optimizer state (a lazy row's pending step included) goes with
 * it, its next training touch asks the admission policy again, and its next insertion starts from default contents.
 * Surviving rows are copied as they are.  The sweep rebuilds the table at the smallest power-of-two capacity >= the
 * floor (the larger of the creation capacity and the largest xf_table_reserve) that holds the survivors at load
 * <= 0.5, never above the current capacity; the old and the new table are both allocated while it runs, as in
 * growth.  A sweep that would remove nothing and keep the capacity does nothing.
 * The stamps are one uint32_t per slot of device memory beside the rows (+12.5 % for LR rows, +1.6 % for FM K = 16
 * FTRL rows); they are part of the state image (xf_table_save_state) but not of xf_table_save (a key xf_table_load
 * loads is an insertion).  A table that has run 2^32 - 1
 * training batches refuses further tracked training steps.  Single-GPU tables only: refused on canonical tables
 * (canonical_fm = 1), on tables with num_shards > 1, and by xf_trainer_create / the step with a multi-rank comm. */
typedef struct xf_eviction_config {
  uint64_t max_idle_batches;  /* > 0: a sweep drops keys no training batch touched among the last max_idle_batches */
  uint64_t max_keys;          /* > 0: a sweep then keeps only the max_keys most recently touched keys */
} xf_eviction_config;
/* starts (or keeps) per-key stamps and sets the sweep's limits; both 0 = track only; cfg = NULL stops tracking and
 * frees them.  Calling it again replaces the limits and keeps the stamps.  On failure the table is unchanged. */
XF_DLL int xf_table_set_eviction(xf_table* t, const xf_eviction_config* cfg);
/* one sweep now (waits for the table's stream); *evicted = keys removed (may be NULL).  XF_ERR_STATE without
 * tracking.  On failure (allocation included) the table is unchanged. */
XF_DLL int xf_table_evict(xf_table* t, uint64_t* evicted);
/* out[i] = last(keys[i]), or UINT64_MAX for an absent key; never inserts.  XF_ERR_STATE without tracking. */
XF_DLL int xf_table_last_touch(xf_table* t, const uint64_t* keys, uint64_t n, uint64_t* out);

/* Exact training-state checkpoint of one table (not the portable xf_table_save format).
 * xf_table_save_state writes an image of everything that decides the table's future: every live row's raw bytes in
 * its slot, the capacity, the capacity floor and the probing layout, the key count, the training-batch number, the
 * admission policy, its counters and Bloom filter, the eviction limits and every live key's stamp, the lazy LR
 * tables' pending-step ring, the config fields that define the rows and their arithmetic, and the caller's `user`
 * value (the CLI stores the epochs done there).  A table loaded from it is byte-identical to the saved one and trains
 * on bit for bit as the saved table would have: a run that saves and continues, and a run resumed from the image,
 * both equal the run that never saved.  For XF_MODEL_FM_CANONICAL and XF_MODEL_MVM that holds on batches with repeated
 * keys in deterministic mode (xf_trainer_set_deterministic); their default steps sum a repeated key's terms in atomic
 * order.  XF_MODEL_FFM has no deterministic mode: it holds on batches in which no key repeats.  Not in the image: the trainers' state (xf_trainer_stats counters, the
 * negative-sampling policy, which is caller config) and xf_table_set_stream's choice.
 * Save runs stream-ordered after everything enqueued on the table's stream, waits for it, and changes nothing in the
 * table.  It writes <path>.tmp and renames it to <path>; on failure no .tmp is left.  Saving the same state twice
 * gives identical files.
 * Load needs a table that has never held state: no keys and no training batch (XF_ERR_STATE otherwise).  Its config
 * must equal the image's field by field (floats bitwise; device and capacity excepted), and so must its row stride,
 * its lazy or eager row layout (XFLOW_EAGER) and its bucket shift at the image's capacity: XF_ERR_ARG names the first
 * field that differs.  The table then takes the image's capacity and every row goes back into its saved slot; the
 * policies, stamps, filter, counters, batch number and capacity floor are the image's (a policy set on the target is
 * replaced).  A damaged or truncated file, or a file of the other format, is XF_ERR_IO.  On any failure the table
 * is unchanged.  *user (may be NULL) receives the saved value.
 * Memory: besides the table, a save or load takes two device and two page-locked staging chunks of at most 64 MiB
 * each, whatever the table's size; a load holds the old and the new table at once, as growth does.
 *
 * File format (little-endian), version 1:
 *   header, 232 bytes
 *     0 "XFST"   4 u32 version   8 u64 header bytes (232)   16 u64 capacity   24 u64 capacity floor   32 u64 keys
 *     40 u32 row stride   44 u32 log2 capacity   48 u32 bucket shift   52 u32 lazy (1) or eager (0) rows
 *     56 i32 latent_dim   60 i32 optimizer   64 f32 alpha   68 f32 beta   72 f32 lambda1   76 f32 lambda2
 *     80 f32 learning_rate   84 i32 resolved v_init (0 constant, 1 counter-based normal, 3 zero)   88 u64 seed
 *     96 i32 shard_index   100 i32 num_shards   104 i32 canonical_fm   108 u32 seq (lazy: the ring's last batch)
 *     112 u64 training batches   120 u64 rejected tokens   128 u64 admitted keys
 *     136 i32 admission mode   140 f32 probability   144 u32 threshold   148 u32 log2_cells   152 u32 hashes
 *     156 u32 eviction tracking (0/1)   160 u64 decay_batches   168 u64 admission seed
 *     176 u64 max_idle_batches   184 u64 max_keys   192 u64 user   200 u64 chunk slots C
 *     208 u64 filter bytes F (Bloom: 2^log2_cells, else 0)   216 u64 ring entries R (lazy: seq + 1, else 0)
 *     224 u64 checksum of bytes [0, 224)
 *   ring section (R > 0): R u64 (the pending steps' divisors by batch number), u64 checksum
 *   rows section: capacity / C chunks, chunk i covering slots [i C, (i + 1) C):
 *     u64 first slot (= i C), u64 live rows n, u64 checksum, u64 0; then n rows of `stride` raw bytes in slot order,
 *     then n u64 slot | stamp << 32 (stamp 0 without tracking)
 *   filter section (F > 0): F bytes of cells, u64 checksum
 * A section's checksum is the sum mod 2^64 of splitmix64(w ^ o) over its 8-byte words w, o = the word's byte offset
 * in the section's payload; in the rows section o = i << 40 | the offset in chunk i's payload (after its 32 bytes). */
XF_DLL int xf_table_save_state(xf_table* t, const char* path, uint64_t user);
XF_DLL int xf_table_load_state(xf_table* t, const char* path, uint64_t* user /* may be NULL */);

/* bucketing rule of ps::Postoffice::GetServerKeyRanges (postoffice.cc:134-143) + DefaultSlicer
 * (kv_app.h:405-460): shard = min(key / floor((2^64-1)/S), S-1).  Pure host function. */
XF_DLL int xf_shard_of(uint64_t key, int num_shards);

/* ------------------------------------------------------------------------------------------------
 * 3. Fused worker step
 * ---------------------------------------------------------------------------------------------- */
typedef struct xf_trainer xf_trainer;
typedef struct xf_comm xf_comm;

typedef struct xf_trainer_config {
  int model;             /* XF_MODEL_* ; FM requires table latent_dim > 0 */
  uint32_t max_rows;     /* largest batch (rows) the trainer will be given */
  uint32_t max_nnz;      /* largest batch (tokens) */
  int keep_loss;         /* 1: keep the per-row residual (pctr - label) of the last batch for xf_trainer_get_loss */
} xf_trainer_config;

/* replaces: new xflow::LRWorker / FMWorker (lr_worker.h:34-42, fm_worker.h:33-42) bound to the table.
 * comm may be NULL (single GPU).  With a comm of N ranks the table must be shard `rank` of N. */
XF_DLL int xf_trainer_create(xf_trainer** out, xf_table* table, xf_comm* comm, const xf_trainer_config* cfg);
XF_DLL int xf_trainer_destroy(xf_trainer* tr);

/* replaces: LRWorker::update / FMWorker::update on one slice (lr_worker.cc:145-177, fm_worker.cc:204-245)
 * INCLUDING the server-side optimizer step the Push triggers.  CSR batch in HOST memory:
 *   row_ptr[rows+1] (u32 offsets into keys), keys[nnz] (u64 feature hashes), labels[rows] (0/1).
 * Copies the batch to the device (pinned staging, async), runs the step, and returns
 * *mean_abs_loss = mean |pctr - label| of the batch (one float read back; pass NULL to skip the
 * read-back and stay asynchronous). */
XF_DLL int xf_trainer_step_host(xf_trainer* tr, const uint32_t* row_ptr, const uint64_t* keys,
                                const uint8_t* labels, uint32_t rows, uint32_t nnz, float* mean_abs_loss);
/* same step on a batch already resident in device memory; asynchronous on the table's stream */
XF_DLL int xf_trainer_step_device(xf_trainer* tr, const uint32_t* d_row_ptr, const uint64_t* d_keys,
                                  const uint8_t* d_labels, uint32_t rows, uint32_t nnz);
/* replaces: calculate_pctr (lr_worker.cc:25-71, fm_worker.cc:25-96): forward only, pctr_out[rows] host */
XF_DLL int xf_trainer_predict_host(xf_trainer* tr, const uint32_t* row_ptr, const uint64_t* keys, uint32_t rows,
                                   uint32_t nnz, float* pctr_out);
/* The textbook factorisation machine with feature VALUES (SURVEY 8f-4; the reference ignores `val` and collapses
 * the interaction over k, fm_worker.cc:177-196 — parity mode = XF_MODEL_FM):
 *     y = sum_i w_i x_i + 1/2 sum_k [ (sum_i v_ik x_i)^2 - sum_i (v_ik x_i)^2 ],   p = sigmoid(y)
 *     dL/dw_i = (p - label) x_i ,  dL/dv_ik = (p - label) x_i (S_k - v_ik x_i) ,  gradients / rows, one FTRL / SGD step
 * vals[nnz] are the tokens' values (NULL: all 1).  Needs a table created with canonical_fm = 1; single GPU. */
XF_DLL int xf_trainer_step_host_values(xf_trainer* tr, const uint32_t* row_ptr, const uint64_t* keys, const float* vals,
                                       const uint8_t* labels, uint32_t rows, uint32_t nnz, float* mean_abs_loss);
XF_DLL int xf_trainer_step_device_values(xf_trainer* tr, const uint32_t* d_row_ptr, const uint64_t* d_keys,
                                         const float* d_vals, const uint8_t* d_labels, uint32_t rows, uint32_t nnz);
XF_DLL int xf_trainer_predict_host_values(xf_trainer* tr, const uint32_t* row_ptr, const uint64_t* keys, const float* vals,
                                          uint32_t rows, uint32_t nnz, float* pctr_out);
/* A DEFINED multi-view machine (SURVEY 8f-4).  src/model/mvm/mvm_worker.cc indexes its per-row field sums one past
 * their end and multiplies in the sums of fields a row does not have (:43,57,75,86-92,262): its output is not a
 * function of its input.  This is the model that code is reaching for, over the same table:
 *     s[f][k] = sum over the row's tokens of field f of v_ik x_i ,   y = sum_k prod_{f present in the row} s[f][k]
 *     p = sigmoid(y) ,  dL/dv_ik = (p - label) x_i prod_{f' present, f' != field(i)} s[f'][k] ,  gradients / rows, one
 *     FTRL / SGD step per touched key on v only (no linear term: mvm_worker.cc pulls and pushes v alone).
 * fields[nnz]: the tokens' field ids (libffm's fgid), each < 32.  vals[nnz] or NULL (all 1).  A row without
 * tokens predicts sigmoid(0).  Needs XF_MODEL_MVM on a table with canonical_fm = 1 and latent_dim in {4,8,16,32};
 * single GPU. */
XF_DLL int xf_trainer_step_host_fields(xf_trainer* tr, const uint32_t* row_ptr, const uint64_t* keys,
                                       const uint8_t* fields, const float* vals, const uint8_t* labels, uint32_t rows,
                                       uint32_t nnz, float* mean_abs_loss);
XF_DLL int xf_trainer_predict_host_fields(xf_trainer* tr, const uint32_t* row_ptr, const uint64_t* keys,
                                          const uint8_t* fields, const float* vals, uint32_t rows, uint32_t nnz,
                                          float* pctr_out);
/* The field-aware factorisation machine, XF_MODEL_FFM (Juan, Zhuang, Chin, Lin, RecSys 2016; libffm's model;
 * csrc/step_ffm.cu), through the same two entry points.  Needs a table created with canonical_fm = 1 (any latent_dim
 * L in {4,8,16,32,64,128}) and no comm.
 *   Layout: the per-field latent dimension is 4 (libffm's default -k 4), so the table holds F = L / 4 fields.  A key's
 *   latent row v[L] is F pieces of 4 floats: piece b (coordinates 4b .. 4b+3) is v_{i,b}, the key's vector for
 *   interacting with field b.  Rows, optimizer state, xf_table_export / _import and the state image are the canonical
 *   tables' own.  Field ids must be < F (18 fields need L = 128, of whose 32 pieces 14 are then never used: the rows
 *   cost what 32 fields would).
 *   Definition, row r with tokens i (key k_i, field f_i, value x_i; vals NULL = all 1):
 *     y = sum_i w_i x_i + sum_{i<j} <v_{i,f_j}, v_{j,f_i}> x_i x_j      (pairs of token positions, same field included)
 *     p = sigmoid(y) ,  r = p - label                                    (a row without tokens: y = 0; no global bias)
 *     dL/dw_i = r x_i ,  dL/dv_{i,b} = r x_i ( T[b][f_i] - [b = f_i] x_i v_{i,f_i} ) ,  T[a][b] = sum_{f_i = a} x_i v_{i,b}
 *   gradients / rows and one FTRL or SGD step per touched key on w and all L coordinates, as XF_MODEL_FM_CANONICAL.
 *   Absent keys are inserted on pull, in training and in predict.
 *   Fixed-order forward: T[a][b], sum w x and Q = sum x^2 |v_{i,f_i}|^2 are added in ascending token position from +0,
 *   the pair sum over the present fields a ascending, the warp reduction by the xor 16 .. 1 tree.  So a row's
 *   prediction depends only on its tokens and on the table, not on its batch, its place in it or the grid, and
 *   xf_trainer_predict_host_fields returns, bit for bit, what a training step on that table state computes (and
 *   feeds an attached pv).  Per-key gradient sums are float atomics: a key repeated within a batch gets bits that
 *   depend on the order they land in (see xf_table_save_state).
 *   Refused with XF_ERR_ARG: every entry point without field ids when nnz > 0 (xf_trainer_step_host, _device,
 *   _values, _async, the ingested steps and their predicts), field ids >= F (naming the token and the bound),
 *   xf_trainer_set_deterministic, importance weighting and negative sampling.
 *   Kernels per step (xf_trainer_launches): training, the step kernel and the optimizer pass (+1 with a pv); predict,
 *   one.  Serving: xf_table_freeze_ffm (section 6, "Field-aware FM models").  The table does not record which model
 *   trained it, so xf_table_freeze_canonical / _mvm of an FFM-trained table are not refused: they give those models'
 *   forwards, not this one's. */
/* Deterministic mode for XF_MODEL_FM_CANONICAL and XF_MODEL_MVM trainers (csrc/step_det.cu).  The default steps of
 * these two models add each token's gradient terms into its key's accumulators with float atomics (and the machine's
 * forward adds a row's same-field terms with shared-memory atomics), so a key with several tokens in a batch gets bits
 * that depend on the order the atomics land in.  on != 0: every later step of tr, training and predict, sums in one
 * fixed order instead; on = 0 restores the default kernels.  LR and FM trainers are refused (XF_ERR_ARG): their
 * per-key sums are fixed point or f64 already and this mode does not change them.  Turning the mode on allocates its
 * scratch for the trainer's max_rows / max_nnz: canonical FM 4K + 4 bytes per row and 20 bytes per token, the machine
 * 4 bytes per row and 4K + 16 bytes per token; both about K / 4 + 5 more bytes per token for the run sums of keys with
 * more than 32 tokens, and the sort's temporary storage.  If that fails the call returns XF_ERR_CUDA and the trainer is
 * unchanged.  The switch waits for the table's stream.
 *   1. Per-token terms, today's op for op.  Canonical FM, token j of row r (residual r, value x): A term
 *      fl(fl(r x) S_k), G term (double)r (double)x, L2 term (double)r (double)x (double)x.  The machine: A term
 *      fl(fl(r x) o_k), o_k the product of the other present fields' sums in ascending field order from 1; g term +0.0.
 *   2. Association.  Each key's tokens in ascending position in the batch's token array, cut into consecutive runs of
 *      32.  A run is summed by a butterfly: term i in lane i, -0.0 (the exact additive identity) in the lanes past the
 *      run; for o = 16, 8, 4, 2, 1: a_i = a_i + a_(i^o); the run's sum is a_0.  The run sums are then added in order
 *      onto the row's accumulator as it stood (g from -0.0, A and L2 from +0).  Every add rounds to nearest, no FMA,
 *      no flush; A in float, G and L2 in double.  So the result depends only on the table before the step and on the
 *      batch, not on grid, scheduling, streams or the other keys; a key with one token in the batch gets exactly the
 *      bits of the default step.
 *   3. The machine's forward, training and predict, is the frozen model's (section 6, "Forward, row r"): field sums as
 *      a left fold in token order from +0, P_k over the present fields ascending, y by the xor 16 .. 1 tree.  With the
 *      mode on, xf_trainer_predict_host_fields returns on every row, bit for bit, what xf_model_predict_host_fields
 *      returns on a model frozen from the table at that moment.  The canonical FM's forward has a fixed order already
 *      (lane-sequential passes, then a shuffle tree) and is unchanged.
 *   4. mean_abs_loss and the _async abs-loss sum: thread t of 256 adds the rows' |r| for rows t, t + 256, ... in row
 *      order from +0, then the 256 partial sums are added as s_i = s_i + s_(i+o) for o = 128, 64, .., 1; s_0 is the
 *      sum.  The order depends only on the row count.
 *   5. Reproducible, per key: xf_table_export of every key, the set of keys, xf_trainer_get_loss, predictions,
 *      xf_trainer_stats and pv reports; two runs on the same batches freeze to byte-identical xf_model_save files.  Not
 *      per slot: a key's slot depends on insertion races between keys.
 *   6. Kernels per training step with tokens (xf_trainer_launches): the step kernel, the radix sort's (1 up to 4864
 *      tokens, else 2 + ceil((log2(capacity) + 1) / 8)), three for the per-key sums, the optimizer pass, and one more
 *      for the abs-loss sum on the host-batch entry points (_host_values, _host_fields, the _async ones, which report
 *      it); a pv adds its one.  Predict
 *      launches one kernel, as without the mode. */
XF_DLL int xf_trainer_set_deterministic(xf_trainer* tr, int on);
/* Importance-weighted training (McMahan et al., "Ad Click Prediction: a View from the Trenches", section 6.1):
 * per-row weights and negative subsampling for XF_MODEL_LR / XF_MODEL_FM.  Each row r of a training step has an
 * effective weight e_r = c_r * s_r (float product, rounded to nearest):
 *   c_r  the caller's weight (xf_trainer_step_host_weighted / _device_weighted); 1 for every other entry point;
 *   s_r  the trainer's negative-sampling policy (xf_trainer_set_negative_sampling): 1 for a positive row (label != 0)
 *        or without a policy; for a negative row inv = (float)(1.0 / rate) if the row is kept and 0 if it is dropped.
 *        A negative row is kept iff the top 24 bits of splitmix64(seed ^ F_r) < floor(rate * 2^24), where
 *        F_r = sum over the row's tokens of splitmix64(key) mod 2^64 (0 for a row without tokens).  The decision is a
 *        function of the row alone, computed on the device: the same whatever the entry point, block cut or slice.
 *        Since F_r ignores token order, rows with equal key multisets decide alike.
 * The step then uses the weighted residual loss_r = e_r * (pctr_r - label_r) wherever it used pctr_r - label_r:
 *   - the gradients are sum over the tokens of key i of loss_r (FM: and loss_r * (S_r - v_ik)), divided by the batch's
 *     row count B as before.  B counts every row, skipped ones included, so that under subsampling the gradient stays
 *     an unbiased estimate of the full batch's.  Weights of 1 give the unweighted step bit for bit.
 *   - a row with e_r = 0 is skipped: its tokens do not probe, insert or ask the admission policy (the Bloom filter
 *     does not count them), nothing is stamped, deposited or counted in unique_keys for it, and keep_loss reports 0
 *     for it.  The batch is still a training batch (admission's and eviction's batch number moves on).
 *   - lazy LR tables sum each batch's residuals per key in a fixed-point unit 2^-s; weighted, s = the same function of
 *     W = sum over the trained rows of ceil(e_r) * tokens_r (instead of the token count), so every key's sum stays in
 *     its field.  Sums stay exact while W < 2^47.  xf_trainer_step_host_weighted refuses a batch whose W could
 *     reach 2^47 (XF_ERR_ARG, bounded with the policy's largest factor); device weights that do are outside the
 *     step's range.
 *   - *mean_abs_loss = sum_r e_r * |pctr_r - label_r| / B; xf_trainer_get_loss keeps reporting the UNWEIGHTED
 *     pctr_r - label_r of the trained rows.
 * Predict is unweighted.  A step with caller weights or a policy runs one more kernel (weight.cu) before the step
 * kernel: xf_trainer_launches counts +1 per such step.  Refused (XF_ERR_ARG): canonical FM / MVM trainers, trainers
 * that run the sharded step (a comm of more than one rank, or XFLOW_MG_FORCE=1), and host weights that are NaN,
 * negative or infinite.  Weights in device memory are the caller's contract, as device keys are. */
/* one step with row weights weights[rows] (host memory); otherwise xf_trainer_step_host */
XF_DLL int xf_trainer_step_host_weighted(xf_trainer* tr, const uint32_t* row_ptr, const uint64_t* keys,
                                         const uint8_t* labels, const float* weights, uint32_t rows, uint32_t nnz,
                                         float* mean_abs_loss);
/* the same on a batch and weights in device memory; asynchronous on the table's stream, like xf_trainer_step_device */
XF_DLL int xf_trainer_step_device_weighted(xf_trainer* tr, const uint32_t* d_row_ptr, const uint64_t* d_keys,
                                           const uint8_t* d_labels, const float* d_weights, uint32_t rows,
                                           uint32_t nnz);
/* Negative sampling for every later training step of the trainer, on every entry point (host, device, _async,
 * _ids_async, _ingested and the _weighted pair): keep each negative row with probability `rate` (decided as above,
 * with this policy's own seed) and weight it by 1 / rate.  rate = 1 turns the policy off; a rate outside
 * [2^-24, 1] (NaN included) is refused. */
XF_DLL int xf_trainer_set_negative_sampling(xf_trainer* tr, float rate, uint64_t seed);
/* rows trained with e_r = 0 since the trainer was created (device counter; waits for the table's stream) */
XF_DLL int xf_trainer_skipped_rows(xf_trainer* tr, uint64_t* skipped);
/* the one-off "init push" of key 0 with zero gradient (lr_worker.cc:180-182, fm_worker.cc:248-252) */
XF_DLL int xf_trainer_init_push(xf_trainer* tr);
/* residuals (pctr - label) of the last step; needs keep_loss = 1 */
XF_DLL int xf_trainer_get_loss(xf_trainer* tr, float* loss_out, uint32_t rows);
/* counters since creation: steps, rows, tokens and unique keys summed over steps (device counter) */
XF_DLL int xf_trainer_stats(xf_trainer* tr, uint64_t* steps, uint64_t* rows, uint64_t* nnz, uint64_t* unique_keys);
/* number of kernels this library launched on behalf of the trainer/table since creation */
XF_DLL int xf_trainer_launches(xf_trainer* tr, uint64_t* launches);
XF_DLL int xf_trainer_sync(xf_trainer* tr);
/* block until every host->device batch copy issued so far has finished (the caller may then
 * overwrite host buffers it passed to xf_trainer_step_host with mean_abs_loss == NULL) */
XF_DLL int xf_trainer_wait_uploads(xf_trainer* tr);
/* Asynchronous variant of xf_trainer_step_host for pipelined callers: the batch arrays and
 * `pinned_abs_loss_sum` (one float, receives sum |pctr - label| of this batch by an asynchronous
 * device->host copy) must be page-locked host memory and stay untouched until xf_trainer_sync /
 * xf_trainer_wait_uploads.  Never blocks on the device. */
XF_DLL int xf_trainer_step_host_async(xf_trainer* tr, const uint32_t* row_ptr, const uint64_t* keys,
                                      const uint8_t* labels, uint32_t rows, uint32_t nnz,
                                      float* pinned_abs_loss_sum);
/* Same as xf_trainer_step_host_async for callers that hold integer feature ids instead of hashed keys:
 * ids[nnz] are u32 ids whose DECIMAL STRING is what the reference's loader would hash
 * (load_data_from_disk.cc:151); the device computes keys = std::hash(decimal string) itself (ingest.cu),
 * so only 4 bytes per token cross PCIe.  Buffers must be page-locked. */
XF_DLL int xf_trainer_step_host_ids_async(xf_trainer* tr, const uint32_t* row_ptr, const uint32_t* ids,
                                          const uint8_t* labels, uint32_t rows, uint32_t nnz,
                                          float* pinned_abs_loss_sum);
/* keys[i] = std::hash<std::string>(decimal string of ids[i]) on DEVICE arrays (stream: cudaStream_t or NULL) */
XF_DLL int xf_hash_decimal_ids_device(const uint32_t* d_ids, uint64_t n, uint64_t* d_keys, void* cuda_stream);
/* Device-side ingest of one text block (load_data_from_disk.cc:126-209 on the GPU, ingest.cu): uploads
 * `len` bytes of "<label>\t<fgid>:<fid>:<val> ...\n" rows, parses them into a CSR batch that stays on
 * the device, and reports its size.  xf_trainer_step_ingested / _predict_ingested then run the step on a
 * row range [row_start, row_end) of that block (the reference's per-thread slices, lr_worker.cc:190-196). */
XF_DLL int xf_trainer_ingest_text(xf_trainer* tr, const char* text, uint64_t len, uint32_t* rows, uint32_t* nnz);
/* The same in two phases, for pipelined callers: _begin enqueues the copy and the parse of the NEXT block on
 * the trainer's ingest stream (two device-side block buffers) and returns at once; `text` must stay untouched
 * until _end returns (page-locked memory is copied by DMA, pageable memory is staged first).  _end waits for
 * that parse only — not for training steps still running on the previous block — and makes the block
 * current.  Up to TWO blocks may be outstanding: the second _begin copies its text at once (into the buffer of
 * the block being trained on, whose text is no longer needed) and its parse is launched by the _end that
 * retires that block, so that with  begin(i+2); step(i); end(i+1)  the H2D of one block runs beside the parse
 * of the previous one and the training step of the one before.  _end always completes the OLDEST outstanding
 * block.  If _end fails (malformed or oversized block) every outstanding block is dropped. */
XF_DLL int xf_trainer_ingest_begin(xf_trainer* tr, const char* text, uint64_t len);
XF_DLL int xf_trainer_ingest_end(xf_trainer* tr, uint32_t* rows, uint32_t* nnz);
XF_DLL int xf_trainer_step_ingested(xf_trainer* tr, uint32_t row_start, uint32_t row_end);
/* copy the ingested block's CSR back to host arrays of rows+1 / nnz / rows elements (any may be NULL) */
XF_DLL int xf_trainer_ingested_export(xf_trainer* tr, uint32_t* row_ptr_out, uint64_t* keys_out, uint8_t* labels_out);
XF_DLL int xf_trainer_predict_ingested(xf_trainer* tr, uint32_t row_start, uint32_t row_end, float* pctr_out,
                                       uint8_t* labels_out);
/* Per-kernel device timing for roofline reporting.  on != 0: record CUDA events around the kernels
 * of every following step (on the table's stream).  xf_trainer_profile syncs and returns, summed
 * over the profiled steps since the last call: ms[0] = fused step kernel, ms[1] = optimizer kernel
 * (+ batch bookkeeping), and the number of steps. */
XF_DLL int xf_trainer_set_profile(xf_trainer* tr, int on);
XF_DLL int xf_trainer_profile(xf_trainer* tr, double ms[2], uint64_t* steps);
/* page-locked host memory for callers without a CUDA runtime of their own */
XF_DLL int xf_host_alloc(void** out, uint64_t bytes);
XF_DLL int xf_host_free(void* p);

/* Base::calculate_auc (base.h:84-110), host: out[0]=logloss (base-2, not negated, float accumulator)
 * out[1]=auc (float `area`; NaN when single-class) out[2]=tp out[3]=fp */
XF_DLL int xf_auc_logloss(const int32_t* labels, const float* pctr, uint64_t n, double out[4]);
/* the same metric in exact arithmetic (not the reference's numbers): out[0] = mean negative natural-log
 * likelihood, out[1] = AUC with ties counted 1/2, out[2]=positives out[3]=negatives */
XF_DLL int xf_auc_logloss_exact(const int32_t* labels, const float* pctr, uint64_t n, double out[4]);

/* The metric on the DEVICE (csrc/metric.cu): predictions and labels of every forward block are appended to a
 * device buffer, xf_metric_finish sorts them there (radix sort, stable) and reduces:
 *   out[0] the reference's logloss (base 2, not negated; double accumulator)   out[1] the reference's AUC (64-bit
 *   integer rank sum instead of the float `area` that stops counting at 2^24)  out[2] positives  out[3] negatives
 *   out[4] mean negative natural-log likelihood   out[5] AUC with ties counted 1/2          (base.h:84-110) */
typedef struct xf_metric xf_metric;
XF_DLL int xf_metric_create(xf_metric** out, int device);
XF_DLL int xf_metric_destroy(xf_metric* m);
XF_DLL int xf_metric_reset(xf_metric* m);
/* append n predictions / 0-1 labels living in device memory (copies run on `cuda_stream`, no sync) */
XF_DLL int xf_metric_add_device(xf_metric* m, const float* d_pctr, const uint8_t* d_labels, uint64_t n, void* cuda_stream);
XF_DLL int xf_metric_finish(xf_metric* m, void* cuda_stream, double out[6]);
XF_DLL int xf_auc_logloss_device(const float* d_pctr, const uint8_t* d_labels, uint64_t n, int device, void* cuda_stream,
                                 double out[6]);
/* forward pass over rows [row_start, row_end) of the current ingested block, appended to `m` without leaving the
 * device (asynchronous).  pctr_out / labels_out (optional host arrays of rows elements): the same values for a
 * caller that also writes them out; the call then waits for them. */
XF_DLL int xf_trainer_predict_ingested_metric(xf_trainer* tr, uint32_t row_start, uint32_t row_end, xf_metric* m,
                                              float* pctr_out, uint8_t* labels_out);

/* ------------------------------------------------------------------------------------------------
 * 4. Host ingest
 * ---------------------------------------------------------------------------------------------- */
/* std::hash<std::string> of libstdc++ (MurmurHash64A, seed 0xc70f6907) as used at
 * load_data_from_disk.cc:151,173,194 */
XF_DLL uint64_t xf_hash_bytes(const char* s, uint64_t len);
/* hashes of the decimal strings of ids[] ("%llu"): what the loader produces for numeric feature ids */
XF_DLL int xf_hash_decimal_ids(const uint64_t* ids, uint64_t n, uint64_t* out);

typedef struct xf_loader xf_loader;
/* replaces: xflow::LoadData(path, block_bytes) (load_data_from_disk.h:19-21) */
XF_DLL int xf_loader_open(xf_loader** out, const char* path, uint64_t block_bytes);
XF_DLL int xf_loader_close(xf_loader* l);
/* restart at the first byte (what re-opening the file at the top of every epoch does, lr_worker.cc:184) */
XF_DLL int xf_loader_rewind(xf_loader* l);
/* replaces: load_minibatch_hash_data_fread (load_data_from_disk.cc:103-210): parse the next block.
 * *rows = 0 at end of file.  The CSR arrays stay valid until the next call. */
XF_DLL int xf_loader_next(xf_loader* l, uint32_t* rows, uint32_t* nnz);
XF_DLL int xf_loader_batch(xf_loader* l, const uint32_t** row_ptr, const uint64_t** keys, const uint8_t** labels);
/* block formation only (load_data_from_disk.cc:108-124): the next block's raw text, for the device parser
 * (xf_trainer_ingest_text / _begin).  *len = 0 at end of file.  The loader alternates two (page-locked) text
 * buffers: a block's text stays valid until the call AFTER the next one.  Tab-less rows ("0\n") count as rows
 * without features on the device parser; the host parser (xf_loader_next), like the reference, scans on to the
 * next tab and merges them into the following row. */
XF_DLL int xf_loader_next_raw(xf_loader* l, const char** text, uint64_t* len);

/* ------------------------------------------------------------------------------------------------
 * 5. Multi-GPU exchange (one process per GPU over NVLink / NVSwitch).  A trainer created with a comm of
 *    N ranks runs the sharded step (csrc/comm.cu): every rank must create its trainer with the same
 *    max_rows / max_nnz / model and call the step / predict entry points the same number of times, in the
 *    same order (an empty batch is a valid step).  NCCL serves bootstrap only (exchange of cudaIpc handles);
 *    inside a step kernels store into the peers' memory directly.
 * ---------------------------------------------------------------------------------------------- */
#define XF_COMM_ID_BYTES 128
/* rank 0 creates the id and distributes it out of band (file, MPI, torch.distributed ...) */
XF_DLL int xf_comm_get_id(uint8_t id[XF_COMM_ID_BYTES]);
XF_DLL int xf_comm_create(xf_comm** out, const uint8_t id[XF_COMM_ID_BYTES], int rank, int nranks, int device);
/* the same with the id passed through a file: rank 0 writes it, the others wait for it (launchers that have no
 * other channel, e.g. the reference's CLI started once per GPU with XFLOW_RANK / XFLOW_WORLD) */
XF_DLL int xf_comm_create_from_file(xf_comm** out, const char* path, int rank, int nranks, int device);
/* max over the ranks of one host value (blocking; to agree on the number of collective steps) */
XF_DLL int xf_comm_allreduce_max(xf_comm* c, uint64_t* inout);
XF_DLL int xf_comm_destroy(xf_comm* c);
XF_DLL int xf_comm_barrier(xf_comm* c);
/* ------------------------------------------------------------------------------------------------
 * 6. Serving model (csrc/serve.cu).  xf_table_freeze makes an xf_model from a trained table: an immutable, compact,
 *    device-resident hash table that holds, per key, only what the forward pass reads, with a forward-only predict
 *    kernel and a file format of its own.  The model shares nothing with the table: the table may train on, be saved
 *    or destroyed, and a predict on the model never inserts a key.
 *
 *    Rows.  LR: {u64 key, f32 w, u32 0} = 16 bytes.  FM of any K: {u64 key, f32 w, f32 st, f32 qt, 12 zero bytes} =
 *    32 bytes, one aligned sector, with st = sum_k v_k and qt = sum_k v_k^2: the reference's FM forward
 *    (fm_worker.cc:177-196) reads nothing else of a latent row, and in a frozen model both are constants.  Open
 *    addressing with the table's hash and bucketised probe sequence; empty slots hold key 2^64 - 1; capacity = the
 *    smallest power of two >= 2 x keys (load <= 0.5), at least 1024.
 *
 *    Freeze waits for everything enqueued on the table's stream and changes nothing in the table (no row, stamp,
 *    filter cell, batch number or pending step).  It resolves each row as a reader does: a lazy LR row's pending step is
 *    folded in, an imported weight is honoured, an FM row whose latent block is not materialised gets st, qt of its
 *    initial values.  The frozen w of a key is, bit for bit, what xf_table_export returns for it, and st, qt are what
 *    the step kernels' forward pass computes for it; xf_model_predict_* therefore returns, bit for bit, what
 *    xf_trainer_predict_* returns on the table at the moment of the freeze (with the matching `absent` policy).
 *
 *    Absent keys.  XF_ABSENT_DEFAULT: a key the model does not hold reads as the row the table would insert for it
 *    (w = 0; FM: st, qt of the table's initial latent values, evaluated on the fly: K evaluations per absent token).
 *    XF_ABSENT_ZERO: it contributes nothing, which is what predict does on a table with an admission policy.
 *    prune = 1 leaves out every row that reads exactly as an absent key would: w == 0 and (LR, or, under DEFAULT, the
 *    latent block is not materialised; under ZERO, st == 0 and qt == 0).  Pruning never changes a prediction, and
 *    keys + pruned_keys == source_keys.  FTRL's L1 term writes exact zeros (ftrl.h:66-74): those are the rows pruned.
 *
 *    Refused with XF_ERR_ARG: tables with canonical_fm = 1 (the per-k sums of the canonical FM and the multi-view
 *    machine do not collapse to st, qt: xf_table_freeze_canonical and xf_table_freeze_mvm serve them) and tables with num_shards > 1 (one
 *    shard's rows are not a model: xf_table_freeze_part and xf_model_merge, below, serve them).
 *
 *    Canonical models.  xf_table_freeze_canonical freezes a table created with canonical_fm = 1 for the textbook FM
 *    with feature values (XF_MODEL_FM_CANONICAL): its predict is the canonical FM's forward, whichever trainer trained
 *    the table (the caller states it by calling this function).
 *      Row: {u64 key, f32 w, u32 0, f32 v[K], zero padding}, 16 + 4K bytes rounded up to 32: K = 4 -> 32, 8 -> 64,
 *      16 -> 96, 32 -> 160, 64 -> 288, 128 -> 544.  Every row starts on a sector and v starts 16 bytes in, so a
 *      token's 16-byte piece c of v is one aligned load.  xf_model_info reports fm = 2 and these row bytes.
 *      Freeze resolves each row as the step kernel reads it: w, and v = the latent block if it is materialised, else
 *      the initial values of (key, k), evaluated at the freeze.  w and v equal xf_table_export's bit for bit.
 *      Absent keys: XF_ABSENT_DEFAULT reads an absent key as the row the table would insert (w = 0, v its initial
 *      values, evaluated on the fly: K per absent token); a canonical table has no admission policy, so absent = -1
 *      is DEFAULT.  XF_ABSENT_ZERO: an absent key contributes nothing.
 *      prune = 1 leaves out rows with w == 0 and, under DEFAULT, a latent block that is not materialised; under ZERO,
 *      every resolved v_k == 0.  Adding +-0 to a float sum that starts at +0 never changes it, so for finite feature
 *      values pruning never changes a prediction; a NaN or Inf value on a pruned key makes the table's term NaN where
 *      the model adds nothing.
 *      xf_model_predict_host_values / _device_values on a canonical model return, bit for bit, what
 *      xf_trainer_predict_host_values returns on the table at the moment of the freeze (under ZERO: on that table with
 *      zero rows imported for the query's absent keys).  xf_model_predict_host / _device read every value as 1.
 *      The XFSM and XFSD files keep version 1 and record fm = 2, latent_dim and these row bytes; a load refuses
 *      non-zero padding in a canonical row.  Not served: shards.
 *
 *    Multi-view machine models.  xf_table_freeze_mvm freezes a table created with canonical_fm = 1 for the multi-view
 *    machine (XF_MODEL_MVM, which trains such tables): its predict is the machine's forward on the tokens' field ids
 *    and feature values, served by xf_model_predict_host_fields / _device_fields only.
 *      Row: {u64 key, u64 0, f32 v[K], zero padding}: the canonical row with w = 0, the same bytes (K = 4 -> 32, 8 -> 64,
 *      16 -> 96, 32 -> 160; F16 as the canonical table below), piece c of v at the same place.  The machine has no
 *      linear term, so the row holds no w: bytes 8 .. 15 are zero.  K is 4, 8, 16 or 32, the latent dimensions the
 *      machine trains.  xf_model_info reports fm = 3 and these row bytes.
 *      Freeze resolves v as xf_table_freeze_canonical does (v equals xf_table_export's bit for bit) and ignores w;
 *      absent = -1 is DEFAULT.  Refused with XF_ERR_ARG: tables with canonical_fm = 0, a latent_dim outside
 *      {4, 8, 16, 32}, num_shards > 1.
 *      Absent keys: XF_ABSENT_DEFAULT reads an absent key as the row the table would insert (v its initial values,
 *      evaluated on the fly), which is what the table's own predict sees after inserting it.  XF_ABSENT_ZERO reads it
 *      as a row of zeros: its field is present and it adds 0 x, as the table does with zero rows imported for the
 *      query's absent keys.  ZERO does not skip the token: in a product over fields, a skipped token would remove its
 *      field from the product, a different model, and pruning would then change predictions.
 *      prune = 1 leaves out the rows that read exactly as an absent key does: under DEFAULT a latent block that is
 *      not materialised, under ZERO every resolved v_k == +-0; w plays no part.  A field's sum starts at +0 and
 *      round-to-nearest adds never make it -0, so a term of +0 and one of -0 leave it alike, and 0 x is the same NaN
 *      for either sign when x is NaN or Inf: pruning never changes a prediction, NaN and Inf values included.
 *      Forward, row r with tokens j = row_ptr[r] .. row_ptr[r+1] - 1 in that order, f_j = fields[j] & 31,
 *      x_j = vals[j] (1 when vals is NULL) and v_j the token's row as the absent policy reads it:
 *          S[f][k] = +0;  for j in order: S[f_j][k] = S[f_j][k] + (v_jk * x_j)   (round to nearest, no FMA, no flush)
 *          P_k = 1;  for the fields f present in the row, ascending: P_k = P_k * S[f][k]   (k < K; no tokens: P_k = 0)
 *          y = the sum of P_0 .. P_K-1 and zeros for k >= K over 32 lanes by xor 16, 8, 4, 2, 1;  pctr = sigmoid(y)
 *      This is xf_trainer_predict_host_fields's forward (step_mvm.cu) with its same-field adds in token order.  That
 *      kernel adds a pass's same-field terms with shared-memory atomics (a pass: T = 128 / K consecutive tokens from
 *      the row's first), whose order among contending lanes the hardware picks, and token order is one of those
 *      orders.  So the model returns, bit for bit, what the table's predict returns at the moment of the freeze (under
 *      ZERO: with zero rows imported for the absent keys) on every row where no field has more than two tokens (0 + a
 *      + b is commutative) or no pass holds two tokens of one field.  On other rows the table's own default result is not
 *      reproducible, and the model's is the order above, the same bits on every call and every entry point; in
 *      deterministic mode (xf_trainer_set_deterministic) the table's predict is this order on every row.
 *      The XFSM and XFSD files keep version 1 and record fm = 3, latent_dim and these row bytes; a load refuses a
 *      non-zero byte 8 .. 15 or padding byte.  Diff, apply and convert serve these models as canonical ones (a
 *      canonical model and a multi-view machine's differ in fm and are never diffed or applied to one another);
 *      merge does not apply (canonical tables are never sharded).
 *
 *    Field-aware FM models.  xf_table_freeze_ffm freezes a table created with canonical_fm = 1 for the field-aware FM
 *    (XF_MODEL_FFM, which trains such tables): its predict is the FFM's forward on the tokens' field ids and feature
 *    values, served by xf_model_predict_host_fields / _device_fields and the candidate and rank entry points only.
 *      Row: the canonical row {u64 key, f32 w, u32 0, f32 v[L], zero padding}, the same bytes at F32 and F16; piece b
 *      of v (coordinates 4b .. 4b+3) is the key's vector for field b, so the model serves F = L / 4 fields, L in
 *      {4, 8, 16, 32, 64, 128}.  xf_model_info reports fm = 4 and these row bytes.
 *      Freeze resolves w and v as xf_table_freeze_canonical does (both equal xf_table_export's bit for bit); absent =
 *      -1 is DEFAULT.  Refused with XF_ERR_ARG: tables with canonical_fm = 0, a latent_dim outside {4, ..., 128},
 *      num_shards > 1.  The table does not change.
 *      Absent keys: XF_ABSENT_DEFAULT reads an absent key as the row the table would insert (w = 0, v its initial
 *      values, evaluated on the fly).  XF_ABSENT_ZERO reads it as a row of zeros whose field is present: the token
 *      adds 0 x to its field sums and w x = 0 x, as the table does with zero rows imported for the query's absent keys.
 *      prune = 1 leaves out rows with w == +-0 and, under DEFAULT, a latent block that is not materialised; under ZERO,
 *      every resolved v_k == +-0.  That never changes a prediction, NaN and Inf values included: every sum (Σwx, each
 *      T[a][b], Q) starts at +0 and a round-to-nearest sum is never -0, so adding +-0 leaves it unchanged whatever the
 *      sign, and 0 x is the same NaN for either sign of zero when x is NaN or Inf.
 *      Forward, row r with tokens j = row_ptr[r] .. row_ptr[r+1] - 1 in that order, f_j = fields[j] & (F - 1) (the
 *      host entry points refuse ids >= F), x_j = vals[j] (1 when vals is NULL), (w_j, v_j) the token's row as the
 *      absent policy reads it, a_j = v_j x_j (L products), every sum a left fold from +0 in j's order:
 *          T[f_j][b] += a_j[4b .. 4b+3]  (b < F);  Q += fma(a3, a3, fma(a2, a2, fma(a1, a1, a0 a0))) over piece f_j;
 *          Σwx += w_j x_j;  lane b < F: P_b = sum over the present fields a ascending of
 *          fma(u3, s3, fma(u2, s2, fma(u0, s0, u1 s1))), u = T[a][b], s = T[b][a];  y = fma(0.5, (the xor 16 .. 1 sum
 *          of P over 32 lanes) - Q, Σwx);  pctr = sigmoid(y)   (round to nearest, no other contraction, no flush)
 *      This is xf_k_step_ffm's pass 1, pair sum and sigmoid, whose order is fixed, with its fused multiply-adds.  So on
 *      every row xf_model_predict_*_fields of a DEFAULT model returns, bit for bit, what xf_trainer_predict_host_fields
 *      returns on the table at the moment of the freeze, and a ZERO model what it returns on that table with zero rows
 *      imported for the query's absent keys.  A candidate's score is the flat predict of its request's context
 *      followed by its tokens, bit for bit.
 *      The XFSM and XFSD files keep version 1 and record fm = 4, latent_dim and these row bytes; a load refuses
 *      non-zero padding as for canonical rows.  Diff, apply and convert serve these models as canonical ones (a
 *      canonical model and a field-aware FM's differ in fm and are never diffed or applied to one another); merge
 *      does not apply.
 *
 *    Sharded tables: parts and merge.  A run sharded over S GPUs holds shard s of the key space in table s
 *    (num_shards = S; shard s owns [s width, (s + 1) width) with width = floor((2^64 - 1) / S), the last shard up to
 *    2^64 - 2, as xf_shard_of).  xf_table_freeze_part freezes one LR or FM table of any num_shards (1 included) into
 *    a part: an xf_model whose rows are exactly those xf_table_freeze would make of the same table (the same
 *    resolution, prune rule and absent policy; the table does not change) and which records shard_index and
 *    num_shards.  xf_model_merge(parts of shards 0 .. S-1) builds the whole model: its contents, info and file are
 *    those of xf_table_freeze applied to one unsharded table that holds the union of the shards' rows, so its
 *    xf_model_save file is byte-identical to that freeze's, its predictions equal that model's bit for bit, and its
 *    fingerprint is the sum mod 2^64 of the parts' fingerprints.  A part serves xf_model_get_info (its shard's keys,
 *    source_keys, pruned_keys), xf_model_lookup, xf_model_fingerprint and xf_model_save (an XFSP file, below); it is
 *    not a model: xf_model_predict_* (every variant), xf_model_diff and xf_model_apply_delta refuse it with
 *    XF_ERR_STATE.  Memory of a merge: the parts, the result, and on the result's device one staging buffer of at
 *    most 64 MiB for the slots of parts on other devices (peer copies, a chunk at a time).  The merge only reads the
 *    parts.  Not provided: a model served sharded across GPUs, a merge over the comm's peer mappings without files
 *    or staging, and deltas made from parts without merging them.
 *
 *    Precision.  Every model has a precision for its latent fields.  XF_PRECISION_F32 is what freeze, merge, load and
 *    apply make of F32 inputs.  xf_model_convert makes an XF_PRECISION_F16 model of an FM, canonical or multi-view
 *    machine's one: w stays float32, and only the latent fields (FM st and qt; canonical and multi-view machine every
 *    v_k) become IEEE binary16, rounded to nearest
 *    even (subnormals included).  Every row still starts with its u64 key, and padding stays zero:
 *      kind        F32                                                   F16
 *      LR          {key, f32 w, u32 0} 16 bytes                          refused: nothing to narrow
 *      FM          {key, f32 w, f32 st, f32 qt, 12 zero bytes} 32        {key, f32 w, f16 st, f16 qt} 16, no padding
 *      canonical   {key, f32 w, u32 0, f32 v[K], 0...} 16 + 4K           {key, f32 w, u32 0, f16 v[K], 0...} 16 + 2K
 *                  rounded up to 32                                      rounded up to 32: K = 4 -> 32, 8 -> 32,
 *                                                                        16 -> 64, 32 -> 96, 64 -> 160, 128 -> 288
 *    In an F16 canonical row a token's piece c of v (v[4c .. 4c+3]) is one aligned 8-byte load at byte 16 + 8c.  Every
 *    xf_model_predict_* on an F16 model returns, bit for bit, what it returns on the F32 model whose latent fields are
 *    replaced by their binary16 values: the kernels widen each field after the load and then run the F32 model's
 *    arithmetic in its order.  Absent keys under XF_ABSENT_DEFAULT read as before, evaluated in float32 on the fly:
 *    only stored rows are narrowed.  xf_model_lookup (st, qt) and xf_model_lookup_latent (v) return the widened
 *    binary16 values.  The files, deltas and merges of F16 models work as for F32 ones; two models of different
 *    precisions cannot be diffed, applied or merged.
 * ---------------------------------------------------------------------------------------------- */
typedef struct xf_model xf_model;
enum { XF_ABSENT_DEFAULT = 0, XF_ABSENT_ZERO = 1 };
enum { XF_PRECISION_F32 = 0, XF_PRECISION_F16 = 1 };  /* of a model's latent fields (above) */
typedef struct xf_freeze_config {
  int absent;            /* XF_ABSENT_*, or -1 = what the table's own predict does: DEFAULT if its admission policy is
                            XF_ADMIT_ALL, else ZERO */
  int prune;             /* 1: leave out the rows that read as absent keys (above); 0: keep every key of the table */
  int device;            /* CUDA ordinal the model lives on; -1 = the table's (another device: built on the table's,
                            then copied there) */
} xf_freeze_config;
/* absent = -1, prune = 1, device = -1 */
XF_DLL int xf_freeze_config_default(xf_freeze_config* cfg);
/* cfg == NULL: the defaults.  On failure *out is NULL. */
XF_DLL int xf_table_freeze(xf_table* t, const xf_freeze_config* cfg, xf_model** out);
/* A canonical model of a table with canonical_fm = 1 (above); the same config and defaults.  XF_ERR_ARG for tables with
 * canonical_fm = 0 and tables with num_shards > 1. */
XF_DLL int xf_table_freeze_canonical(xf_table* t, const xf_freeze_config* cfg, xf_model** out);
/* A multi-view machine's model of a table with canonical_fm = 1 (above); the same config and defaults.  XF_ERR_ARG,
 * naming the reason, for tables with canonical_fm = 0, a latent_dim outside {4, 8, 16, 32} and num_shards > 1. */
XF_DLL int xf_table_freeze_mvm(xf_table* t, const xf_freeze_config* cfg, xf_model** out);
/* A field-aware FM's model of a table with canonical_fm = 1 (above); the same config and defaults.  XF_ERR_ARG,
 * naming the reason, for tables with canonical_fm = 0, a latent_dim outside {4, 8, 16, 32, 64, 128} and
 * num_shards > 1.  The table does not change. */
XF_DLL int xf_table_freeze_ffm(xf_table* t, const xf_freeze_config* cfg, xf_model** out);
/* A part of a table of any num_shards (above); the same config and defaults.  XF_ERR_ARG for canonical tables (they
 * are never sharded); XF_ERR_STATE, naming their count, if the table holds keys outside its shard's range (a Pull,
 * Push or import can put them there). */
XF_DLL int xf_table_freeze_part(xf_table* t, const xf_freeze_config* cfg, xf_model** out);
/* the shard a part holds; XF_ERR_STATE for a whole model */
XF_DLL int xf_model_part_info(xf_model* m, int* shard_index, int* num_shards);
/* The whole model of parts[0 .. n) on `device` (-1: parts[0]'s).  The parts must be shards 0 .. n-1 of one n-way
 * split, each once, and agree on fm, latent_dim, precision, optimizer, absent, the resolved v_init, v_const and seed
 * (prune may differ): else XF_ERR_ARG, naming what is wrong.  XF_ERR_FULL past 2^32 slots or on a probe overflow.  No part
 * changes; on failure *out is NULL. */
XF_DLL int xf_model_merge(xf_model* const* parts, int n, int device, xf_model** out);
/* A new model on m's device, m with its latent fields at `precision` (XF_PRECISION_*); m is unchanged.  F32 -> F16
 * rounds each latent field to nearest even, F16 -> F32 widens it exactly, and converting to m's own precision copies
 * m.  The result holds exactly m's keys (conversion never prunes), and its keys, source_keys, pruned_keys, absent,
 * optimizer, v_init and seed are m's; a part converts to a part of the same shard.  Runs on a stream of its own and
 * reads m only.  Refused, with *out NULL and m unchanged: XF_ERR_ARG for an LR model or an unknown precision;
 * XF_ERR_STATE if a field is finite in float32 and not in binary16 (|x| >= 65520), naming how many such fields there
 * are and the smallest key that holds one (conversion never saturates).  A NaN field stays NaN. */
XF_DLL int xf_model_convert(xf_model* m, int precision, xf_model** out);
XF_DLL int xf_model_destroy(xf_model* m);
typedef struct xf_model_info {
  uint64_t keys;         /* keys the model holds */
  uint64_t capacity;     /* slots */
  uint64_t bytes;        /* capacity x row_bytes: the model's device memory */
  uint64_t source_keys;  /* keys of the table when it was frozen */
  uint64_t pruned_keys;  /* source_keys - keys */
  uint32_t row_bytes;    /* F32: 16 (LR), 32 (FM), 16 + 4K rounded up to 32 (canonical, multi-view machine,
                            field-aware FM); F16: 16 (FM), 16 + 2K rounded up to 32 (the others but LR) */
  int latent_dim, optimizer, absent, fm;  /* fm: 0 LR, 1 FM, 2 canonical FM, 3 multi-view machine, 4 field-aware FM */
  int precision;         /* XF_PRECISION_* of the latent fields */
} xf_model_info;
XF_DLL int xf_model_get_info(xf_model* m, xf_model_info* out);
/* Model file "XFSM" (little-endian): a 104-byte header
 *     0 "XFSM"   4 u32 version (1)   8 u64 header bytes (104)   16 u64 keys   24 u64 capacity   32 u32 row bytes
 *    36 i32 fm (0 LR, 1 FM, 2 canonical, 3 multi-view machine, 4 field-aware FM)   40 i32 latent_dim   44 i32 optimizer   48 i32 absent
 *    52 i32 resolved v_init (0 constant, 1 counter-based normal, 3 zero)   56 f32 the constant
 *    60 u32 precision (0 F32, 1 F16; the word was reserved as 0, so every F32 file is unchanged)   64 u64 seed
 *    72 u64 source keys   80 u64 pruned keys
 *    88 u64 rows per chunk (64 MiB / row bytes)   96 u64 checksum of bytes [0, 96)
 *  then the rows SORTED BY KEY in ceil(keys / rows per chunk) chunks, each {u64 index of its first row, u64 rows,
 *  u64 checksum, u64 0} followed by its rows.  Checksums are those of the state image above (sum of
 *  splitmix64(word ^ offset), a chunk's offsets being chunk << 40 | byte offset in its rows).  The file is a function
 *  of the model's contents, not of where its keys lie: two freezes of one table, and load then save, give identical
 *  bytes.  Written to <path>.tmp and renamed; the staging is bounded by the chunk size.  xf_model_load rebuilds the
 *  device table from the rows; a truncated, damaged or other-format file is XF_ERR_IO and leaves *out NULL, and so is
 *  a file whose checksums pass but whose keys do not ascend strictly below 2^64 - 1 or whose rows have a non-zero
 *  padding byte (LR bytes 12 .. 15, FM 20 .. 31 at F32 and none at F16, canonical 12 .. 15 and 16 + 4K .. row bytes at
 *  F32 or 16 + 2K .. row bytes at F16, multi-view machine as canonical and 8 .. 11 too), and a header whose precision is not 0 or 1 or whose row bytes are not those of
 *  its fm, latent_dim and precision (an F16 LR model included).
 * Part file "XFSP" (xf_model_save of a part): XFSM's layout with a 112-byte header
 *     0 "XFSP"   4 u32 version (1)   8 u64 header bytes (112)   16 .. 95 as XFSM's (the part's keys, capacity,
 *    source and pruned keys; fm 0 or 1)   96 i32 shard_index   100 i32 num_shards   104 u64 checksum of bytes [0, 104)
 *  then the part's rows sorted by key in XFSM's chunks.  xf_model_load reads either magic and returns a part for
 *  XFSP; it also refuses (XF_ERR_IO) a part file whose keys do not ascend strictly, whose keys leave the shard's range,
 *  or whose shard_index is not below num_shards.  xf_delta_load refuses both. */
XF_DLL int xf_model_save(xf_model* m, const char* path);
XF_DLL int xf_model_load(xf_model** out, const char* path, int device);
/* Forward pass over a CSR batch (row r = keys[row_ptr[r] .. row_ptr[r+1]), row_ptr non-decreasing and <= nnz);
 * pctr_out[rows].  Rows of any length (none: sigmoid(0)) and rows == 0 are valid; there is no max_rows: the model's
 * staging grows on demand.  _host refuses key 2^64 - 1 and a malformed row_ptr with XF_ERR_ARG, runs on the model's
 * own stream and returns when pctr_out is filled; calls on one model are serialised.  _device takes device pointers
 * on the model's device, is asynchronous on `cuda_stream` (cudaStream_t or NULL), reads nothing on the host and uses
 * no state of the model but its rows, so any number may be in flight. */
XF_DLL int xf_model_predict_host(xf_model* m, const uint32_t* row_ptr, const uint64_t* keys, uint32_t rows,
                                 uint32_t nnz, float* pctr_out);
XF_DLL int xf_model_predict_device(xf_model* m, const uint32_t* d_row_ptr, const uint64_t* d_keys, uint32_t rows,
                                   uint32_t nnz, float* d_pctr_out, void* cuda_stream);
/* The same with the tokens' feature values vals[nnz] (NULL: all 1; device memory for _device_values), for canonical
 * models; the contracts are those of _host / _device.  Non-NULL vals on an LR or FM model are XF_ERR_ARG: that model
 * ignores values.  These four and xf_model_predict_ingested refuse a multi-view machine's or a field-aware FM's model
 * (XF_ERR_ARG): they read field ids. */
XF_DLL int xf_model_predict_host_values(xf_model* m, const uint32_t* row_ptr, const uint64_t* keys, const float* vals,
                                        uint32_t rows, uint32_t nnz, float* pctr_out);
XF_DLL int xf_model_predict_device_values(xf_model* m, const uint32_t* d_row_ptr, const uint64_t* d_keys,
                                          const float* d_vals, uint32_t rows, uint32_t nnz, float* d_pctr_out,
                                          void* cuda_stream);
/* The forward of a multi-view machine's or a field-aware FM's model (above) with the tokens' field ids fields[nnz] and
 * feature values vals[nnz] (NULL: all 1); the contracts are those of _host_values / _device_values.  _host refuses a
 * field id of 32 or more (multi-view machine) or of F = L / 4 or more (field-aware FM) with XF_ERR_ARG, naming the
 * token, the id and, for the field-aware FM, the bound; on the device the ids are the caller's contract, and the kernel
 * reads fields[j] & 31 or & (F - 1) as the step kernels do.  NULL fields with nnz > 0 are XF_ERR_ARG.  XF_ERR_ARG on an
 * LR, FM or canonical model: they read no field ids. */
XF_DLL int xf_model_predict_host_fields(xf_model* m, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* fields,
                                        const float* vals, uint32_t rows, uint32_t nnz, float* pctr_out);
XF_DLL int xf_model_predict_device_fields(xf_model* m, const uint32_t* d_row_ptr, const uint64_t* d_keys,
                                          const uint8_t* d_fields, const float* d_vals, uint32_t rows, uint32_t nnz,
                                          float* d_pctr_out, void* cuda_stream);
/* Candidate scoring.  A ranking request scores one context (the user, page and device features) against N candidates,
 * each with features of its own.  A batch of R requests gives each its context once:
 *   request q's context is tokens ctx_ptr[q] .. ctx_ptr[q+1] - 1 of ctx_keys (ctx_vals, ctx_fields);
 *   its candidates are rows cand_ptr[q] .. cand_ptr[q+1] - 1, candidate c being tokens row_ptr[c] .. row_ptr[c+1] - 1
 *   of keys (vals, fields), with cand_ptr[0] = 0 and cand_ptr[R] = candidates.
 * Candidate c of request q is scored as the concatenated row "request q's context tokens in order, then row c's
 * tokens", values and field ids concatenated alike (a NULL vals side reads as every value 1): pctr_out[c] is, bit for
 * bit, what the model's flat predict returns for that row (xf_model_predict_host / _host_values for LR, FM and
 * canonical models, _host_fields for multi-view machines; F32 and F16 models, either absent policy, pruned or not).
 * A request without candidates produces nothing; an empty context gives the flat predict of the candidate rows, an
 * empty candidate row that of the context.  Values are read by canonical and multi-view machine models only (non-NULL
 * vals on an LR or FM model: XF_ERR_ARG); field ids are required by multi-view machine models (NULL with tokens: XF_ERR_ARG)
 * and refused by every other model.
 * The device folds each context once per run of up to 16 candidates of its request and starts every candidate's forward
 * from that state, so a context's rows are looked up about N / 16 times rather than N times. */
typedef struct xf_candidate_batch {
  uint32_t requests;            /* R */
  const uint32_t* ctx_ptr;      /* [R + 1] */
  const uint64_t* ctx_keys;     /* [ctx_nnz] */
  const float* ctx_vals;        /* [ctx_nnz] or NULL (every value 1); canonical and multi-view machine models only */
  const uint8_t* ctx_fields;    /* [ctx_nnz]; multi-view machine and field-aware FM models only, and required by them */
  uint32_t ctx_nnz;
  const uint32_t* cand_ptr;     /* [R + 1]: cand_ptr[0] = 0, cand_ptr[R] = candidates */
  uint32_t candidates;
  const uint32_t* row_ptr;      /* [candidates + 1] into keys / vals / fields, as a flat predict's row_ptr */
  const uint64_t* keys;         /* [nnz] */
  const float* vals;            /* as ctx_vals */
  const uint8_t* fields;        /* as ctx_fields */
  uint32_t nnz;
} xf_candidate_batch;
/* _host: host arrays.  Refused with XF_ERR_ARG, naming the cause: null arguments, a decreasing ctx_ptr, cand_ptr or
 * row_ptr, cand_ptr[0] != 0 or cand_ptr[R] != candidates, ctx_ptr[R] > ctx_nnz or row_ptr[candidates] > nnz, the key
 * 2^64 - 1 on either side, a field id of 32 or more on either side; a part with XF_ERR_STATE.  Stages the batch through
 * the model's buffers in one upload (each context once), runs on the model's stream and returns when pctr_out
 * [candidates] is filled; calls on one model are serialised. */
XF_DLL int xf_model_predict_candidates_host(xf_model* m, const xf_candidate_batch* b, float* pctr_out);
/* _device: the struct on the host, its arrays in device memory on the model's device.  The contract of
 * xf_model_predict_device: asynchronous on `cuda_stream`, reads nothing on the host, uses no state of the model but its
 * rows, any number in flight.  The arrays are the caller's contract (the _host checks are not made; field ids are read
 * & 31). */
XF_DLL int xf_model_predict_candidates_device(xf_model* m, const xf_candidate_batch* b, float* d_pctr_out,
                                              void* cuda_stream);
/* Candidate ranking: each request's top k candidates by pctr, selected on the device.  Candidate i of request q
 * (0 <= i < n_q = cand_ptr[q+1] - cand_ptr[q], its local index) has the score p_i that xf_model_predict_candidates_*
 * returns for candidate cand_ptr[q] + i, bit for bit, and the key
 *   r_i = ord(p_i) << 32 | (2^32 - 1 - i),  ord(NaN) = 0,  ord(p) = bits(p) ^ 0x80000000 (sign clear), ~bits(p) (set);
 * a candidate ranks before another iff its key is larger.  So a higher pctr ranks first, equal pctr bits rank by
 * smaller index, and NaN ranks after every number.  Ties are common at the ends: xf_sigmoid returns exactly 1.0f for
 * y > 30 and rounds to 1.0f above about y = 17, and returns 1e-6 for y < -30; such candidates rank by index.
 * For j < m_q = min(k, n_q), top_index[q k + j] is the local index of request q's j-th ranked candidate and
 * top_pctr[q k + j] its score, bit for bit; every slot j >= m_q holds index 0xFFFFFFFF and pctr bits 0x7FC00000.  All
 * R k slots are written, also when candidates == 0.
 * _host: every check of xf_model_predict_candidates_host, with its codes; XF_ERR_ARG for k = 0, k > XF_RANK_MAX_K and
 * a NULL top_index with R > 0.  Uploads the batch as xf_model_predict_candidates_host does and scores into the model's
 * buffers; downloads the R k indices (and the R k scores when top_pctr is not NULL), never the candidates' scores.
 * Runs on the model's stream; calls on one model are serialised.
 * _device: the contract of xf_model_predict_candidates_device.  d_pctr [candidates] receives every candidate's score,
 * the bytes xf_model_predict_candidates_device writes, and the selection reads them; d_top_pctr may be NULL.  Uses no
 * device memory but its arguments. */
enum { XF_RANK_MAX_K = 1024 };
XF_DLL int xf_model_rank_candidates_host(xf_model* m, const xf_candidate_batch* b, uint32_t k,
                                         uint32_t* top_index /* [R * k] */, float* top_pctr /* [R * k] or NULL */);
XF_DLL int xf_model_rank_candidates_device(xf_model* m, const xf_candidate_batch* b, uint32_t k,
                                           float* d_pctr /* [candidates] */, uint32_t* d_top_index /* [R * k] */,
                                           float* d_top_pctr /* [R * k] or NULL */, void* cuda_stream);
/* what the model holds for n host keys: w[n], st[n], qt[n] (0 for LR), present[n]; any output may be NULL.  On a
 * canonical or multi-view machine's model st and qt must be NULL (XF_ERR_ARG): its rows are read with
 * xf_model_lookup_latent. */
XF_DLL int xf_model_lookup(xf_model* m, const uint64_t* keys, uint64_t n, float* w, float* st, float* qt,
                           uint8_t* present);
/* what a canonical model holds for n host keys: w[n], v[n * K], present[n] (0 for an absent key); any output may be
 * NULL.  On a multi-view machine's model w is 0: its row holds no linear term.  XF_ERR_ARG on an LR or FM model. */
XF_DLL int xf_model_lookup_latent(xf_model* m, const uint64_t* keys, uint64_t n, float* w, float* v, uint8_t* present);
/* forward pass over rows [row_start, row_end) of a trainer's current ingested block, read from `m` instead of the
 * trainer's table (same outputs as xf_trainer_predict_ingested; runs on the table's stream).  XF_ERR_ARG if the
 * trainer's model is not LR / FM as the model is, if the two live on different devices, or for a canonical model
 * (an ingested text block carries no feature values). */
XF_DLL int xf_model_predict_ingested(xf_model* m, xf_trainer* tr, uint32_t row_start, uint32_t row_end,
                                     float* pctr_out, uint8_t* labels_out);

/* ------------------------------------------------------------------------------------------------
 * 7. Serving model deltas (csrc/delta.cu).  A training run that keeps learning exports models one after another; a
 *    delta carries one model to the next without shipping and reloading the whole of it.
 *
 *    The delta from model A to model B:
 *      upserts  the rows of B whose key A does not hold, or whose row differs from A's in any byte (a row is 16
 *               bytes for LR, 32 for FM and 16 + 4K rounded up to 32 for a canonical or multi-view machine's
 *               model, padding included),
 *               sorted by key;
 *      deletes  the keys of A that B does not hold, sorted by key;
 *      header   what XFSM records of B: keys, source_keys and pruned_keys.
 *    Applying it to A builds a new model whose contents and info are B's, so that xf_model_save of the result is
 *    byte-identical to xf_model_save(B) and every xf_model_predict_* returns on it, bit for bit, what it returns on B.
 *
 *    Fingerprint.  An order-free u64 of a model's contents: the sum mod 2^64 over its rows of h(row), where for the
 *    row's 8-byte little-endian words w_0 .. w_{n-1} (n = 2 for LR, 4 for FM, row bytes / 8 for a canonical or multi-view machine's model)
 *    h_0 = 0, h_{i+1} = splitmix64(h_i ^ w_i)
 *    and h(row) = h_n.  The empty model's fingerprint is 0.  A delta records the fingerprint and key count of its base
 *    and of its result; apply refuses a base whose fingerprint or key count is not the delta's (XF_ERR_STATE), so a
 *    delta applied to the wrong model never makes a wrong model, and checks the result's after building it.
 *
 *    Compatibility.  A and B must agree on what defines how an absent key reads: fm, latent_dim, optimizer, absent,
 *    the resolved v_init, v_const and seed, and on their rows' precision (else XF_ERR_ARG, naming the field).  Prune
 *    may differ: a delta compares contents only.  A delta between F16 models carries F16 rows and records the
 *    precision; convert both models first to carry an F32 chain to F16.
 *
 *    A delta lives on a device: that of the models it was diffed from, or the one xf_delta_load names.  Diff and
 *    apply run on streams of their own and read their models only: neither changes a model, and apply does not use
 *    the base's host staging or lock it, so the base keeps serving while the next model is built beside it.  The
 *    caller swaps its pointer to the result and destroys the base afterwards.  Memory: diff takes 24 bytes of scratch
 *    per key of the larger model (what xf_model_save takes, without its 64 MiB row chunk) besides the delta itself;
 *    apply holds the base, the delta and the result at once.  On every failure *out is NULL and no model changes.
 * ---------------------------------------------------------------------------------------------- */
typedef struct xf_delta xf_delta;
typedef struct xf_delta_info {
  uint64_t upserts;             /* rows set in the result */
  uint64_t deletes;             /* keys of the base dropped from the result */
  uint64_t base_keys, base_fingerprint;
  uint64_t result_keys, result_fingerprint;
  uint64_t source_keys, pruned_keys;  /* the result's, as xf_model_info has them */
  uint64_t file_bytes;          /* the size of the file xf_delta_save writes */
  uint32_t row_bytes;           /* as xf_model_info has them */
  int latent_dim;
  int precision;                /* XF_PRECISION_* of the models it carries */
} xf_delta_info;
/* The delta from `base` to `next` (same device, compatible); neither model changes. */
XF_DLL int xf_model_diff(xf_model* base, xf_model* next, xf_delta** out);
/* A new model: `base` with the delta applied, on base's device; base is unchanged.  XF_ERR_ARG: the delta is not
 * compatible with base (the field is named) or lives on another device; XF_ERR_STATE: base's key count or
 * fingerprint is not the delta's base's; XF_ERR_FULL: the result would exceed 2^32 slots. */
XF_DLL int xf_model_apply_delta(xf_model* base, const xf_delta* d, xf_model** out);
XF_DLL int xf_model_fingerprint(xf_model* m, uint64_t* out);
/* Delta file "XFSD" (little-endian): a 144-byte header
 *     0 "XFSD"   4 u32 version (1)   8 u64 header bytes (144)   16 i32 fm (as XFSM's: 0 .. 4)   20 i32 latent_dim
 *    24 i32 optimizer   28 i32 absent   32 i32 resolved v_init   36 f32 the constant   40 u64 seed   48 u32 row bytes
 *    52 u32 precision (as XFSM's; reserved as 0 before, so every F32 file is unchanged)
 *    56 u64 base keys   64 u64 base fingerprint   72 u64 result keys   80 u64 result source keys
 *    88 u64 result pruned keys   96 u64 result fingerprint   104 u64 upserts U   112 u64 deletes D
 *   120 u64 rows per chunk (64 MiB / row bytes)   128 u64 keys per delete chunk (64 MiB / 8)
 *   136 u64 checksum of bytes [0, 136)
 *  then the U upsert rows sorted by key in ceil(U / rows per chunk) chunks, then the D delete keys sorted by key in
 *  ceil(D / keys per chunk) chunks.  Every chunk is {u64 index of its first entry in its section, u64 entries,
 *  u64 checksum, u64 0} followed by its entries; chunks are numbered through both sections (the first delete chunk
 *  follows the last upsert chunk) and chunk c's checksum is XFSM's (sum of splitmix64(word ^ (c << 40 | byte offset
 *  in its entries))).  The file is a function of the two models' contents.  Written to <path>.tmp and renamed; the
 *  staging is bounded by the chunk size.  xf_delta_load refuses with XF_ERR_IO a truncated or damaged file, another
 *  format (an XFSM model, an XFST or XFTB checkpoint), and a file whose checksums pass but whose contents break the
 *  format: keys not strictly ascending in a section, a key both upserted and deleted, key 2^64 - 1, non-zero padding,
 *  or counts that cannot hold (more upserts than result keys, more deletes than base keys). */
XF_DLL int xf_delta_save(xf_delta* d, const char* path);
XF_DLL int xf_delta_load(xf_delta** out, const char* path, int device);
XF_DLL int xf_delta_get_info(xf_delta* d, xf_delta_info* out);
XF_DLL int xf_delta_destroy(xf_delta* d);

/* ------------------------------------------------------------------------------------------------
 * 8. Progressive validation (csrc/validate.cu).  Each training row is scored by the model as it stood just before
 *    the step that trains on it; the weighted mean over the stream estimates hold-out quality without setting data
 *    aside (Blum, Kalai and Langford 1999; McMahan et al. 2013).  An xf_pv is a streaming, binned metric in constant
 *    device memory whose report depends only on the multiset of (p, label, e) added to it: not on call boundaries,
 *    streams, grid shape or atomic order.  Every accumulator is an integer.
 *
 *    Rows.  A row (p, label, e), label != 0 positive, e its weight (1 when no weights are given):
 *      - e == 0 (either sign): adds nothing;
 *      - e NaN, infinite, negative or >= 2^31: counted in overflow_rows, adds nothing else;
 *      - p NaN: counted in nan_rows, adds nothing else;
 *      - otherwise the row is scored: rows, positives or negatives count it.
 *    Binning, with m = mantissa_bits and pc = p clamped to [2^-20, 1] (float; xf_sigmoid already returns values in
 *    [1e-6, 1], so the clamp never changes a step's prediction):
 *      bin(pc) = (bits(pc) >> (23 - m)) - (bits(2^-20) >> (23 - m)),  20 * 2^m + 1 bins, in the order of p.
 *    Fixed-point sums, unit 2^-32, each row's term rounded to nearest even after exact scaling:
 *      per bin and class   the row count (u64) and the weight mass sum e (128 bits);
 *      globally            sum e * l (192 bits) and sum e * pc (128 bits), where l = -ln(q) for a positive row and
 *                          -ln(1 - q) for a negative one, q = p clamped to [1e-15, 1 - 1e-15] in double (the clamp of
 *                          xf_metric's out[4]), e * l rounded once in double; e * pc is exact in double.
 *    No sum can wrap before 2^64 rows.  Memory: 48 bytes per bin (about 1 MB at m = 10, 63 MB at m = 16).  An add
 *    aggregates the rows of a warp that share a bin and class before its atomics (__match_any_sync).
 *
 *    Report.  With W+ and W- the exact weight masses and W = W+ + W-:
 *      weight_pos, weight_neg   W+, W- correctly rounded to double;
 *      logloss = sum e l / W,  mean_pctr = sum e pc / W,  ctr = W+ / W   (exact ratios, correctly rounded; NaN if W = 0);
 *      auc_lo = sum_b W-_b W+_{>b} / (W+ W-),  auc_hi = auc_lo + sum_b W-_b W+_b / (W+ W-),  auc = their midpoint,
 *      over the bins in ascending order, in double on the device (a scan over the bins, then one reduction in a fixed
 *      order); NaN if W+ or W- is 0.  The exact weighted AUC of the raw floats with ties counted 1/2 lies in
 *      [auc_lo, auc_hi]: the bin width m chooses is the error bar.  Equal inputs give identical report bytes.
 *
 *    Training.  xf_trainer_set_validation attaches a pv to a trainer: every later TRAINING step (every entry point:
 *    _host, _device, _host_async, _host_ids_async, _ingested, the _weighted pair, _values, _fields; LR lazy or eager,
 *    FM, canonical FM, MVM) adds, for each of its rows, the pctr it computed from the table before its update, the
 *    row's label and its effective weight e_r (importance weighting, section 3; 1 without weighting).  Rows that
 *    weighting skips (e_r = 0) add nothing.  Predict never adds.  The step kernels store their predictions and one more
 *    kernel scores them on the table's stream: xf_trainer_launches counts +1 per step while a pv is attached.
 *    Attaching changes no bit of training: tables, state images and every other output are those of a run without.
 *    Not in the state image: a resumed run starts its pv afresh.
 *
 *    Slices.  xf_pv_set_slices gives a pv a slice map: a set of (key, slice) pairs, slice < n_slices.  Many keys may
 *    name one slice; a key names at most one.  A row belongs to slice s when at least one of its tokens has a key that
 *    the map sends to s: a row belongs to every slice its keys name, and counts once per slice however many of its
 *    tokens name it and wherever they sit in the row.  A row whose keys name no slice is in no slice (the global sums
 *    still count it).  Membership depends only on the batch's keys, not on the table, admission or eviction.  Each
 *    slice has the pv's accumulators with the same row classification (e == 0 adds nothing; overflow and NaN rows are
 *    counted per slice), fixed-point units and sums, binned with the slice mantissa bits ms chosen at set time:
 *      slice s's report is, byte for byte, the xf_pv_report of an unsliced pv with mantissa_bits = ms fed exactly the
 *      rows of slice s, and the sliced pv's own xf_pv_report is that of an unsliced pv with its m fed every row;
 *    so the slice reports too depend only on the rows added, not on batch cuts, streams, grid or atomic order.  A
 *    sliced pv needs each row's tokens: xf_pv_add_device_rows (xf_pv_add_device refuses it).  A trainer feeding a
 *    sliced pv passes its batch's row_ptr and keys, and xf_trainer_launches counts +2 per step instead of +1; the
 *    training itself changes no bit.  Memory: n_slices * (20 * 2^ms + 1) * 48 bytes for the bins, and a map of 12
 *    bytes per slot with at least 2 slots per key.  One table lookup per token (one 32-byte sector for a key that
 *    names no slice, almost always); a row's (row, slice) pairs add with the same multi-word atomics as the bins.
 *    Made for up to about 10^4 segments (ms = 8: 246 KB of bins per slice), not one slice per user.
 * ---------------------------------------------------------------------------------------------- */
typedef struct xf_pv xf_pv;
/* the report of xf_pv_report; a struct tag only (like POSIX's struct stat), the function has the name */
struct xf_pv_report {
  uint64_t rows;            /* scored rows = positives + negatives */
  uint64_t positives, negatives, nan_rows, overflow_rows;
  double weight_pos, weight_neg;
  double logloss, mean_pctr, ctr;
  double auc, auc_lo, auc_hi;
};
/* a pv on `device` with 20 * 2^mantissa_bits + 1 bins; mantissa_bits 4 .. 16, else XF_ERR_ARG */
XF_DLL int xf_pv_create(xf_pv** out, int device, uint32_t mantissa_bits);
/* XF_ERR_STATE while a trainer has it attached */
XF_DLL int xf_pv_destroy(xf_pv* pv);
/* clears every sum, stream-ordered after every add enqueued so far; later adds come after it */
XF_DLL int xf_pv_reset(xf_pv* pv);
/* n predictions, labels (!= 0 positive) and weights (NULL: all 1) in device memory on pv's device; asynchronous on
 * cuda_stream (cudaStream_t or NULL): the arrays must stay untouched until that stream has run the add.  XF_ERR_STATE
 * on a pv with slices (xf_pv_add_device_rows) */
XF_DLL int xf_pv_add_device(xf_pv* pv, const float* d_pctr, const uint8_t* d_labels, const float* d_weights,
                            uint64_t n, void* cuda_stream);
/* waits for every add enqueued so far, on any stream; does not reset */
XF_DLL int xf_pv_report(xf_pv* pv, struct xf_pv_report* out);
/* Replace pv's slice map and clear every sum (global and per slice), like xf_pv_reset.  n_slices = 0 (with
 * n_keys = 0) removes slicing; slice_mantissa_bits is then ignored.  XF_ERR_STATE while a trainer feeds pv.
 * XF_ERR_ARG, naming the reason, leaving pv as it was, for: slice_of[i] >= n_slices, a key listed twice, the reserved
 * key 2^64-1, n_slices > 65536, n_keys > 2^24, slice_mantissa_bits outside 4..16, and slice accumulators over 1 GiB
 * (n_slices * ((20 << ms) + 1) * 48 bytes + 56 bytes of sums per slice).  Waits for every add enqueued so far. */
XF_DLL int xf_pv_set_slices(xf_pv* pv, const uint64_t* keys, const uint32_t* slice_of, uint64_t n_keys,
                            uint32_t n_slices, uint32_t slice_mantissa_bits);
/* rows predictions/labels/weights as xf_pv_add_device, plus each row's tokens: d_keys[d_row_ptr[r] .. d_row_ptr[r+1]).
 * d_row_ptr[0] need not be 0 (the ingested path passes absolute offsets).  On a pv without slices it equals
 * xf_pv_add_device (d_row_ptr and d_keys are then not read).  Asynchronous on cuda_stream, like xf_pv_add_device. */
XF_DLL int xf_pv_add_device_rows(xf_pv* pv, const float* d_pctr, const uint8_t* d_labels, const float* d_weights,
                                 const uint32_t* d_row_ptr, const uint64_t* d_keys, uint64_t rows, void* cuda_stream);
/* out[n_slices], slice s at out[s]; XF_ERR_ARG unless n equals the pv's n_slices (> 0); waits like xf_pv_report;
 * does not reset */
XF_DLL int xf_pv_report_slices(xf_pv* pv, struct xf_pv_report* out, uint32_t n);
/* every later training step of tr feeds pv (above); NULL detaches.  With a sliced pv the steps add their rows' keys
 * too (xf_pv_add_device_rows).  XF_ERR_ARG, naming the reason, for a trainer that
 * runs the sharded step (a comm of more than one rank, or XFLOW_MG_FORCE=1) and for a pv on another device than the
 * table.  A pv may feed several trainers; the caller resets it (for windows, epochs). */
XF_DLL int xf_trainer_set_validation(xf_trainer* tr, xf_pv* pv);

/* ------------------------------------------------------------------------------------------------
 * 9. Grouped test metric (csrc/group_metric.cu).  The exact AUC and logloss inside each group of a held-out set,
 *    where a group is whatever one uint64 id per row names (a user, a request), and their mean over the groups
 *    weighted by rows: group AUC, GAUC (Zhou et al., "Deep Interest Network for Click-Through Rate Prediction", KDD
 *    2018).  A ranker orders candidates within a request, which a pooled AUC (xf_metric) does not judge.  The metric
 *    sorts on the device, like xf_metric; with one id per segment it is a sliced xf_metric.
 *
 *    Rows.  A row (p, y, g): p the float prediction, y != 0 positive, g any uint64 (0 and 2^64 - 1 included).  A row
 *    with p NaN counts in nan_rows and nothing else; it is in no group, and a group of NaN rows only does not exist.
 *    Predictions tie when equal as floats (-0.0 ties with +0.0; +-Inf allowed, equal infinities tie).
 *    Per group g, over its other rows: n_g rows, P_g positives, N_g negatives, and
 *      U2_g      = sum over its negatives j of (2 #{positives i of g: p_i > p_j} + #{positives i of g: p_i == p_j}),
 *                  twice the tie-aware Mann-Whitney U, an integer;
 *      auc_g     = (double)U2_g / ((2.0 * (double)P_g) * (double)N_g) in IEEE double, NaN when P_g or N_g is 0 (the
 *                  expression of xf_metric_finish's out[5]: rows that form one group report out[5] bit for bit);
 *      L_i       = a row's logloss term in units of 2^-32: the pv's with weight 1 (section 8), l * 2^32 rounded to the
 *                  nearest integer, l = -ln q (positive) or -ln(1 - q) (negative), q = p clamped to [1e-15, 1 - 1e-15];
 *      S_g       = sum of L_i over the group, exact (128 bits);
 *      logloss_g = (double)S_g / ((double)n_g * 2^32): S_g rounded to the nearest double, then one division.
 *    Report, with "correctly rounded" the exact ratio rounded to nearest even, and NaN for a zero denominator:
 *      rows = sum n_g, positives, negatives, nan_rows, groups;  scored_groups: groups with P_g > 0 and N_g > 0,
 *      scored_rows: their sum of n_g;
 *      logloss   = sum S_g / (2^32 rows), correctly rounded: byte for byte the logloss of an unweighted xf_pv fed the
 *                  same rows;
 *      gauc      = sum over scored groups of T_g / (2^32 scored_rows), correctly rounded,
 *                  T_g = __double2ull_rn(((double)n_g * auc_g) * 2^32);
 *      gauc_mean = sum over scored groups of M_g / (2^32 scored_groups), correctly rounded, M_g = __double2ull_rn(auc_g
 *                  * 2^32).
 *    Bounds: a metric holds fewer than 2^31 rows (xf_metric's limit), so sum T_g and sum M_g stay below 2^64, sum S_g
 *    below 2^70 and U2_g, 2 P_g N_g below 2^63.  Every accumulator is an integer and every double a fixed function of
 *    integers: the report and the per-group arrays depend only on the multiset of rows, not on how they were cut into
 *    adds, their order, the streams, the grid or the order of atomics.
 *    Memory: 13 bytes per held row; a finish adds 76 bytes of scratch per held row (two 16-byte sort keys, a 12-byte
 *    scan, 32 bytes of per-group sums) and CUB's temporary storage, and keeps them for later calls.
 *
 *    Ranking quality at a cutoff k (xf_group_metric_topk): NDCG@k, precision@k and recall@k of every group, over the
 *    rows of the last finish.  The rows, the sort, NaN handling and the tie rule are the finish's.  Within group g, the
 *    non-NaN rows are ordered by descending p, and equal floats tie (-0 ties with +0).  Positions are counted from 0.
 *    Tie run r of g starts at position a_r; has c_r rows, of which m_r are positive (y != 0); and overlaps the top k
 *    in o_r = min(max(k - a_r, 0), c_r) positions.  n_g is the group's rows, P_g its positives and N_g its negatives.
 *      Discounts: d(i) = 2^32 / log2(i + 2), rounded to the nearest integer, for i = 0 .. 65535 (the table of
 *                  xf_group_metric_discounts); D(i) = sum of d(j), j < i.  d(0) = 2^32 and D(65536) < 2^44.2.
 *                  rn(x) is the exact rational x rounded to the nearest integer, ties to even, computed in 128-bit
 *                  integers (m_r (D(a) - D(b)) reaches about 2^75).
 *      Per-group integers, in units of 2^-32:
 *        H_g = sum over runs of rn(m_r o_r 2^32 / c_r): the hits in the top k (only a run that straddles position k
 *              rounds);
 *        G_g = sum over runs of rn(m_r (D(a_r + o_r) - D(a_r)) / c_r): the DCG at k;
 *        I_g = D(min(P_g, k)): the ideal DCG.
 *      Per-group doubles, each one division of exactly representable values, all three NaN when P_g = 0:
 *        ndcg_g      = (double)G_g / (double)I_g;
 *        precision_g = (double)H_g / ((double)min(k, n_g) * 2^32): a request with fewer than k candidates can reach 1;
 *        recall_g    = (double)H_g / ((double)P_g * 2^32).
 *      These are the expectations over a uniformly random order inside each tie run, up to the units' rounding: a
 *      run's positives are spread evenly over its positions, the top-k counterpart of the AUC's tied pair counting 1/2,
 *      so a model that outputs many equal scores is not credited with a lucky order.
 *      Report: the scored groups are the finish's (P_g > 0 and N_g > 0, so the numbers sit beside gauc; an
 *      all-positive group scores 1 at every k and would inflate the mean).  For X in {ndcg, precision, recall}, built
 *      as gauc and gauc_mean:
 *        X      = sum over scored groups of __double2ull_rn(((double)n_g * X_g) * 2^32) / (2^32 scored_rows),
 *        X_mean = sum over scored groups of __double2ull_rn(X_g * 2^32) / (2^32 scored_groups),
 *      both correctly rounded, NaN for a zero denominator; every sum stays below 2^63 since rows < 2^31.  The same
 *      bytes under any permutation, cut or stream of the adds, as the finish's.
 *    Memory: a topk keeps 24 bytes per group for groups_topk and the metric keeps D (512 KB) once it has run one.
 * ---------------------------------------------------------------------------------------------- */
typedef struct xf_group_metric xf_group_metric;
/* the report of xf_group_metric_finish (a struct tag only, like xf_pv_report) */
struct xf_group_report {
  uint64_t rows, positives, negatives, nan_rows, groups, scored_groups, scored_rows;
  double logloss, gauc, gauc_mean;
};
XF_DLL int xf_group_metric_create(xf_group_metric** out, int device);
XF_DLL int xf_group_metric_destroy(xf_group_metric* m);
/* drops every row; stream-ordered after every add enqueued so far, and before every later one */
XF_DLL int xf_group_metric_reset(xf_group_metric* m);
/* n predictions, labels (!= 0 positive) and group ids in device memory on m's device, copied into m on cuda_stream
 * (cudaStream_t or NULL) without a synchronisation: the arrays must stay untouched until that stream has run the add.
 * XF_ERR_ARG, naming the reason, leaving m unchanged, for a NULL array with n > 0 and for an add that would bring m to
 * 2^31 rows or more. */
XF_DLL int xf_group_metric_add_device(xf_group_metric* m, const float* d_pctr, const uint8_t* d_labels,
                                      const uint64_t* d_groups, uint64_t n, void* cuda_stream);
/* waits for every add enqueued so far, on any stream; does not reset.  An empty metric reports zero counts and NaN
 * ratios. */
XF_DLL int xf_group_metric_finish(xf_group_metric* m, struct xf_group_report* out);
/* the groups of the last finish in ascending id order into host arrays of n elements, any of them NULL: id, n_g, P_g,
 * auc_g, logloss_g.  XF_ERR_ARG unless n is that finish's `groups`; XF_ERR_STATE if no finish came after the last
 * reset or add. */
XF_DLL int xf_group_metric_groups(xf_group_metric* m, uint64_t n, uint64_t* ids, uint64_t* rows, uint64_t* positives,
                                  double* auc, double* logloss);
enum { XF_GROUP_TOPK_MAX_K = 65536 };
/* the report of xf_group_metric_topk: k, the finish's groups, scored_groups and scored_rows, and the means above */
struct xf_group_topk_report {
  uint32_t k;
  uint64_t groups, scored_groups, scored_rows;
  double ndcg, ndcg_mean, precision, precision_mean, recall, recall_mean;
};
/* evaluates the rows of the last finish at cutoff k, on m's stream; does not change what xf_group_metric_groups
 * returns.  XF_ERR_STATE if no finish came after the last reset or add; XF_ERR_ARG, naming k, for k = 0 or
 * k > XF_GROUP_TOPK_MAX_K.  A refused call leaves m unchanged.  An empty finish gives zero counts and NaN ratios. */
XF_DLL int xf_group_metric_topk(xf_group_metric* m, uint32_t k, struct xf_group_topk_report* out);
/* the last topk's ndcg_g, precision_g and recall_g in the order of xf_group_metric_groups (ascending id) into host
 * arrays of n elements, any of them NULL.  XF_ERR_ARG unless n is the last finish's `groups`; XF_ERR_STATE if no topk
 * came after the last finish, reset or add. */
XF_DLL int xf_group_metric_groups_topk(xf_group_metric* m, uint64_t n, double* ndcg, double* precision,
                                       double* recall);
/* the discounts d(0 .. n-1) of the definition above, n <= XF_GROUP_TOPK_MAX_K (XF_ERR_ARG otherwise, or for d NULL
 * with n > 0); host only, needs no device */
XF_DLL int xf_group_metric_discounts(uint64_t* d, uint32_t n);

/* ------------------------------------------------------------------------------------------------
 * 1. Reference C API (src/c_api/c_api.h:26-29), unchanged signatures.
 *    XFCreate builds an LR worker on <train_path>-%05d / <test_path>-%05d (rank from XFLOW_RANK,
 *    default 0); paths are copied.  XFStartTrain trains `epochs` (default 60, lr_worker.h:63; env
 *    XFLOW_EPOCHS) and, on rank 0, predicts and prints logloss/auc like lr_worker.cc:207-217.
 *    Extensions: XFCreateEx picks model/optimizer/K; XFDestroy frees the handle.
 * ---------------------------------------------------------------------------------------------- */
XF_DLL int XFCreate(void** h, const char* train_path, const char* test_path);
XF_DLL int XFStartTrain(void** h);
XF_DLL int XFCreateEx(void** h, const char* train_path, const char* test_path, int model, int optimizer,
                      int latent_dim, int epochs);
XF_DLL int XFDestroy(void** h);

#endif /* XFLOW_B200_H_ */

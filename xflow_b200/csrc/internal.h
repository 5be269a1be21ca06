// Internal host-side structures shared by capi.cu / comm.cu / worker.cc.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <functional>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/xflow_b200.h"
#include "kernels.h"
#include "table.cuh"

void xf_set_error(const char* fmt, ...);
// XF_ERR_ARG, naming the key, if any of the n host keys is the reserved empty-slot marker 2^64 - 1 (capi.cu)
int xf_check_host_keys(const uint64_t* keys, uint64_t n, const char* fn);
// XF_ERR_ARG, naming the row, if any of the n host row weights is NaN, negative or infinite (capi.cu)
int xf_check_host_weights(const float* weights, uint64_t n, const char* fn);
// log2 of the slots per probing bucket of a table of 2^log2cap rows of `stride` bytes (capi.cu)
uint32_t xf_bucket_shift(uint32_t stride, uint32_t log2cap);

#define XF_CUDA_TRY(expr)                                                              \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      xf_set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, \
                   cudaGetErrorString(_e));                                            \
      return XF_ERR_CUDA;                                                              \
    }                                                                                  \
  } while (0)

#define XF_TRY(expr)            \
  do {                          \
    int _r = (expr);            \
    if (_r != XF_OK) return _r; \
  } while (0)

// growable device buffer
struct XfDevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes);
  void release();
  template <typename T> T* as() { return reinterpret_cast<T*>(p); }
};

// growable pinned host buffer
struct XfPinBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes);
  void release();
  template <typename T> T* as() { return reinterpret_cast<T*>(p); }
};

struct xf_table {
  xf_table_config cfg;
  XfTableView view;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  unsigned long long* d_size = nullptr;
  int* d_error = nullptr;
  uint64_t size_bound = 0;   // host-side upper bound on the number of live keys (sync path)
  // asynchronous size read-back (no host sync in steady state): the device counter is copied to a
  // pinned ring after every step; bound = last completed reading + keys submitted since it was issued
  unsigned long long* h_size_ring = nullptr;
  cudaEvent_t size_ev[4] = {nullptr, nullptr, nullptr, nullptr};
  uint64_t size_issued_at[4] = {0, 0, 0, 0};
  bool size_inflight[4] = {false, false, false, false};
  int size_next = 0;
  uint64_t cum_incoming = 0, known_size = 0, known_at = 0;
  uint64_t launches = 0;
  int refs = 1;              // the creator + every trainer bound to the table (destroy order is free)
  // lazy ("update on next touch") tables: batch sequence number and the per-batch row counts and fixed-point units
  uint32_t seq = 0;
  uint64_t* d_rows_by_seq = nullptr;
  size_t rows_cap = 0;
  int next_seq();            // advances seq; flushes all pending steps and restarts when the ring is used up
  int reserve_seqs(int n);   // makes sure the next n numbers come without a restart (flushes now if they would not)
  // scratch for the host-pointer API (pull/push/import/export on host arrays); like KVWorker::Push/Pull
  // (kv_app.h:110-165) those entry points may be called from several threads: serialised by this mutex
  std::mutex host_mu;
  XfDevBuf s_keys, s_slots, s_w, s_v, s_nw, s_zw, s_nv, s_zv, s_present;
  // feature admission (xf_table_set_admission, admit.cu): the policy, the Bloom filter, the training-batch number b
  xf_admission_config admit{};                // mode XF_ADMIT_ALL
  uint8_t* d_filter = nullptr;                // 2^log2_cells one-byte counters (XF_ADMIT_BLOOM only)
  unsigned long long* d_admit = nullptr;      // {rejected tokens, admitted keys, rejected-list length of even / odd b}
  uint64_t admit_batches = 0;
  // feature eviction (xf_table_set_eviction, evict.cu): the sweep's limits and the stamps, one uint32_t per slot beside
  // the rows (nullptr = tracking off); kernels that may stamp get stamps(): the array and the current batch number
  xf_eviction_config evict{};
  uint32_t* d_stamp = nullptr;
  XfStampView stamps() const { return XfStampView{d_stamp, (uint32_t)(admit_batches < 0xFFFFFFFFull ? admit_batches : 0xFFFFFFFFull)}; }
  uint64_t cap_floor = 0;     // no sweep shrinks the table below this: the creation capacity, the largest reserve
  XfDevBuf s_hist;            // the sweep's 2^16-bin histogram

  int alloc_table(uint64_t capacity);  // a fresh table (with a stamp array if tracking is on); on failure view is kept
  int ensure_room(uint64_t incoming_keys);
  int grow(uint64_t new_capacity);
  // rebuild at new_capacity with the rows `keep` keeps (grow keeps all): old + new are allocated at the peak
  int rebuild(uint64_t new_capacity, const XfKeep& keep);
  int check_error();
};

// deterministic training steps (xf_trainer_set_deterministic, step_det.cu): the scratch of one step, allocated for the
// trainer's max_rows / max_nnz when the mode is turned on
struct XfDetBufs {
  XfDevBuf keys_in, keys_out, toks_in, toks_out;  // the (slot, token position) pairs before and after the sort
  XfDevBuf tok_row, row_s;                        // canonical FM: each token's row, each row's S[K]
  XfDevBuf terms;                                 // multi-view machine: each token's K terms
  XfDevBuf res;                                   // each row's residual
  XfDevBuf run_a, run_d, rdesc, longs, cnt;       // segments of more than 32 tokens: their runs' sums
  XfDevBuf tmp;                                   // the sort's temporary storage
  int alloc(bool mvm, int K, uint32_t max_rows, uint32_t max_nnz);  // on failure some buffers may be held: release()
  void release();
};
// one deterministic step (mode 0 train, 1 predict: the multi-view machine only); touched[] gets nnz entries
int xf_det_step(const XfTableView& t, XfDetBufs& b, bool mvm, const uint32_t* row_ptr, const uint64_t* keys,
                const float* vals, const uint8_t* fields, const uint8_t* labels, uint32_t rows, uint32_t nnz, int mode,
                uint32_t* touched, float* loss_out, float* pctr_out, float* abs_loss_sum, cudaStream_t st);
// kernels a deterministic training step launches besides its step kernel and the optimizer pass: the sort's, the
// three of the per-key sums (none without tokens) and the abs-loss sum's (abs_sum)
uint64_t xf_det_extra_launches(uint32_t nnz, uint32_t log2cap, bool abs_sum);

struct XfBatchBuf {
  XfDevBuf row_ptr, keys, labels, ids, vals, fields, weights;
  XfPinBuf h_row_ptr, h_keys, h_labels;
  cudaEvent_t copied = nullptr;   // H2D of this buffer finished (copy stream)
  cudaEvent_t consumed = nullptr; // kernels reading this buffer finished (compute stream)
  cudaEvent_t staged = nullptr;   // H2D out of the pinned staging finished
};

struct xf_trainer {
  xf_table* table = nullptr;
  xf_comm* comm = nullptr;
  xf_trainer_config cfg;
  cudaStream_t copy_stream = nullptr;
  XfBatchBuf buf[2];
  uint64_t step_index = 0;
  XfDevBuf touched, loss, pctr;
  XfDevBuf rejected;                    // keys of the rejected tokens of the current step (max_nnz; Bloom admission only)
  unsigned long long* d_unique_total = nullptr;
  float* d_abs_loss = nullptr;          // 2 slots
  float* h_abs_loss = nullptr;          // pinned, 2 slots
  uint64_t n_steps = 0, n_rows = 0, n_nnz = 0;
  uint32_t last_rows = 0;
  uint64_t launches = 0;
  // importance weighting (xf_trainer_set_negative_sampling, the _weighted steps; weight.cu): the negative-sampling
  // policy (rate 1: none), the rows' effective weights of the current step (max_rows floats, allocated on first use)
  // and {W of the current step, rows skipped since creation}
  float neg_rate = 1.f;
  uint64_t neg_seed = 0;
  XfDevBuf row_w;
  unsigned long long* d_wstat = nullptr;
  // progressive validation (xf_trainer_set_validation, validate.cu): the pv every training step feeds, or nullptr
  xf_pv* pv = nullptr;
  // deterministic mode (xf_trainer_set_deterministic, step_det.cu): its scratch, or nullptr when the mode is off
  XfDetBufs* det = nullptr;
  // device-side ingest (xf_trainer_ingest_begin / _end): two sets of {raw text, the block's CSR}, so that
  // block i+1 is copied and parsed on the ingest stream while block i is being trained on the table stream
  struct IngestSet {
    XfDevBuf text, row_ptr, keys, labels, totals;
    XfPinBuf stage;                 // page-locked copy of a pageable source
    uint32_t* h_totals = nullptr;   // pinned {rows, tokens, parse error}
    cudaEvent_t parsed = nullptr;   // H2D + parse of this set finished (ingest stream)
    cudaEvent_t copied = nullptr;   // the block's text has arrived in `text` (ingest copy stream)
    uint64_t len = 0;               // bytes of the block whose text is in `text`
    cudaEvent_t consumed = nullptr; // the last step that reads this set finished (table stream)
    uint32_t rows = 0, nnz = 0, max_rows = 0, max_tok = 0;
  };
  IngestSet ing[2];
  XfDevBuf ing_scratch;
  cudaStream_t ing_stream = nullptr;       // parses
  cudaStream_t ing_copy_stream = nullptr;  // H2D of the blocks' text: the copy of block i+2 runs beside the parse of i+1
  int ing_cur = 0;                  // the set xf_trainer_step_ingested works on
  int ing_pending = 0;              // xf_trainer_ingest_begin calls not yet matched by _end (0..2); the second one
                                    // targets the set being trained: its text is copied at once, its parse is
                                    // launched by the _end that frees the set
  uint32_t ing_rows = 0, ing_nnz = 0;
  void* mg = nullptr;                   // multi-GPU exchange state (comm.cu)
  cudaEvent_t input_ready = nullptr;    // set by the host-batch paths: H2D of the batch about to be stepped
  // optional per-kernel timing (xf_trainer_set_profile): events around the kernels of each step
  bool profile = false;
  std::vector<cudaEvent_t> prof_events;  // 4 marks per step: step kernel [0,1], optimizer kernel(s) [2,3]
  size_t prof_used = 0;
};

// checkpoint.cu: the section checksum of the file formats (XFST state images, XFSM serving models) = the integer sum,
// mod 2^64, of xf_st_hash(word, offset) over a section's 8-byte words; xf_st_host_sum sums `bytes` of host memory whose
// first word has offset off0
#define XF_ST_CHUNK_BYTES (64ull << 20)     // staging bytes per chunk of a file's rows section
__host__ __device__ __forceinline__ uint64_t xf_st_hash(uint64_t word, uint64_t off) { return xf_splitmix64(word ^ off); }
// offsets of a chunk's words: the chunk index above bit 40, the byte offset in the chunk's payload below
__host__ __device__ __forceinline__ uint64_t xf_st_tag(uint64_t chunk) { return chunk << 40; }
uint64_t xf_st_host_sum(const void* p, uint64_t bytes, uint64_t off0);
// Write a file so that a reader never sees it half written: body(f, name) writes `path`.tmp (named `name` in its
// errors), which is then closed and renamed to `path`.  On any failure the temporary file is removed and the error
// returned; a short write or a failed close or rename is XF_ERR_IO.
int xf_save_atomic(const char* path, const std::function<int(FILE* f, const char* name)>& body);
// XF_ERR_IO, naming the format and the call that loads it, if the `got` bytes at `head` begin with the magic of one of
// the project's file formats (XFTB, XFST, XFSM, XFSP, XFSD) that is not among `own`, the caller's magics (4 characters
// each, the first naming what the caller loads); XF_OK otherwise
int xf_refuse_foreign(const void* head, size_t got, const char* path, const char* own);

// ingest.cu
int xf_launch_parse(const char* d_text, uint64_t len, XfDevBuf& scratch, uint32_t* d_row_ptr, uint64_t* d_keys,
                    uint8_t* d_labels, uint32_t max_rows, uint32_t max_tok, uint32_t* d_totals, int* d_error,
                    cudaStream_t st);
int xf_launch_hash_ids(const uint32_t* d_ids, uint32_t n, uint64_t* d_keys, cudaStream_t st);

// capi.cu: XF_ERR_ARG unless [row_start, row_end) lies in the current ingested block (sharded: is all of it)
int xf_ingested_range(xf_trainer* tr, uint32_t row_start, uint32_t row_end);
int xf_trainer_forward_ingested(xf_trainer* tr, uint32_t row_start, uint32_t row_end);

// validate.cu: a trainer whose table lives on `device` starts (XF_ERR_ARG, naming both devices, if pv lives on
// another) or stops feeding pv; xf_pv_destroy refuses a pv that trainers feed
int xf_pv_attach(xf_pv* pv, int device);
void xf_pv_detach(xf_pv* pv);
// does pv have slices (xf_pv_set_slices)?  Its adds then launch two kernels, not one
bool xf_pv_sliced(xf_pv* pv);

// multi-GPU pieces implemented in comm.cu
int xf_mg_create(xf_trainer* tr);
void xf_mg_destroy(xf_trainer* tr);
int xf_mg_step(xf_trainer* tr, const uint32_t* d_row_ptr, const uint64_t* d_keys, const uint8_t* d_labels,
               uint32_t rows, uint32_t nnz, int mode, float* d_abs_loss, cudaEvent_t* prof_marks);
int xf_mg_unique(xf_trainer* tr, unsigned long long* out);
int xf_comm_nranks(xf_comm* c);
int xf_comm_rank(xf_comm* c);

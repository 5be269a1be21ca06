// Host-callable launchers of kernels.cu (internal; the public surface is include/xflow_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "table.cuh"
#include "mg.cuh"

int xf_vec_for(int K);
int xf_tps_for(int K);

void xf_launch_fill(const XfTableView& t, cudaStream_t st);
void xf_launch_step(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* labels,
                    int B, int mode, uint32_t* touched, uint32_t nnz, float* loss_out, float* pctr_out,
                    float* abs_loss_sum, const XfAdmitView* adm, const XfStampView& sv, const XfWeightView& wv,
                    cudaStream_t st);
// importance weighting (weight.cu): e_out[r] = the effective weight of row r of a training batch; *W += the lazy
// step's fixed-point bound, *skipped += the rows with e = 0.  caller_w may be NULL (all 1); sample: the negative-
// sampling policy (keep a negative row iff top24(splitmix64(seed ^ F_r)) < p24, with weight inv)
void xf_launch_row_weights(const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* labels, const float* caller_w,
                           int B, bool sample, uint32_t p24, float inv, uint64_t seed, float* e_out,
                           unsigned long long* W, unsigned long long* skipped, cudaStream_t st);
// feature admission (admit.cu): after a step on the table's stream, count the batch's rejected tokens into the
// Bloom filter (n = *rej_n of them in rej_keys, at most nnz), add n to *rejected_total and zero *next_rej_n
void xf_launch_admit_count(const XfAdmitView& a, uint8_t* cells, const uint64_t* rej_keys, const unsigned long long* rej_n,
                           uint32_t nnz, unsigned long long* rejected_total, unsigned long long* next_rej_n, cudaStream_t st);
// halve every counter of the Bloom filter (2^log2_cells bytes)
void xf_launch_admit_decay(uint8_t* cells, uint32_t log2_cells, cudaStream_t st);
// FM step: shared-memory hot-key cache; its flush uses touched[nnz .. nnz + xf_step_touched_extra)
uint32_t xf_step_touched_extra(int K, int B);
// touched[j] (one entry per token position) = slot of the key first touched by token j, else 0xFFFFFFFF;
// sv.stamp != nullptr (feature eviction): the rows updated get stamp[slot] = sv.now
void xf_launch_update_touched(const XfTableView& t, const uint32_t* touched, uint64_t nnz, double rows,
                              unsigned long long* unique_total, const XfStampView& sv, cudaStream_t st);
void xf_launch_update_pushed(const XfTableView& t, const uint32_t* slots, uint64_t n, const float* gw,
                             const float* gv, cudaStream_t st);
// a key it inserts gets stamp = sv.now when sv.stamp != nullptr (feature eviction)
void xf_launch_probe(const XfTableView& t, const uint64_t* keys, uint64_t n, bool insert, uint32_t* slots,
                     float* w_out, cudaStream_t st, const XfStampView& sv = XfStampView{nullptr, 0u});
void xf_launch_gather_v(const XfTableView& t, const uint32_t* slots, const uint64_t* keys, uint64_t n,
                        float* v_out, cudaStream_t st);
void xf_launch_import(const XfTableView& t, const uint32_t* slots, uint64_t n, const float* w, const float* nw,
                      const float* zw, const float* v, const float* nv, const float* zv, cudaStream_t st);
void xf_launch_export(const XfTableView& t, const uint32_t* slots, const uint64_t* keys, uint64_t n, float* w,
                      float* nw, float* zw, float* v, float* nv, float* zv, uint8_t* present, cudaStream_t st);
// re-insert the rows of `src` that `keep` keeps into `dst` (growth: all of them), with their stamps
void xf_launch_rehash(const XfTableView& src, const XfTableView& dst, const XfKeep& keep, const uint32_t* src_stamp,
                      uint32_t* dst_stamp, cudaStream_t st);
// feature eviction (evict.cu): stamp every slot with `value` (tracking starts); out[i] = stamp of slots[i], or
// UINT64_MAX for 0xFFFFFFFF; the histogram passes of the sweep's radix select
void xf_launch_stamp_fill(uint32_t* stamp, uint64_t n, uint32_t value, cudaStream_t st);
void xf_launch_gather_stamps(const uint32_t* stamp, const uint32_t* slots, uint64_t n, uint64_t* out, cudaStream_t st);
struct XfEvictPass {
  int what;          // 0: high 16 bits of the stamp; 1: its low 16 bits, among stamps with high bits `hi`;
                     // 2: the 16-bit key digit at `shift`, among keys of stamp `s_star` whose bits above it are `prefix`
  uint32_t cutoff;   // only stamps >= cutoff count
  uint32_t hi, s_star;
  uint64_t prefix;
  int shift;
};
void xf_launch_evict_hist(const XfTableView& t, const uint32_t* stamp, const XfEvictPass& p, unsigned int* hist,
                          cudaStream_t st);
void xf_launch_list_keys(const XfTableView& t, uint64_t* keys_out, unsigned long long* count, uint64_t max_out,
                         cudaStream_t st);
int xf_grid_for(uint64_t work_items, int block, int blocks_per_sm);
// xf_grid_for for a kernel whose CTAs of `block` threads take `smem` bytes of dynamic shared memory each: as many CTAs
// per SM as its 227 KB hold (1 KB of it reserved per CTA), at most 8.  Past the 48 KB a launch gets without opting in,
// `kernel` is opted in to `smem` first, once per device and kernel, under a lock.
int xf_grid_smem(const void* kernel, uint64_t work_items, int block, size_t smem);
void xf_launch_step_lr_lazy(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys,
                            const uint8_t* labels, int B, uint64_t nnz, int mode, uint32_t seq, uint64_t* rows_by_seq,
                            float* loss_out, float* pctr_out, float* abs_loss_sum, unsigned long long* unique_total,
                            const XfAdmitView* adm, const XfStampView& sv, const XfWeightView& wv, cudaStream_t st);

// lazy tables: fold all pending steps (sequence numbers restart afterwards)
void xf_launch_flush_pending(const XfTableView& t, cudaStream_t st);
void xf_launch_update_touched_dev(const XfTableView& t, const uint32_t* touched, uint64_t work_bound,
                                  const uint32_t* n_dev, const uint32_t* rows_dev, uint32_t extra_base,
                                  uint32_t extra_n, const float* v0_side, unsigned long long* unique_total,
                                  cudaStream_t st);
// sharded step (mg_kernels.cu)
void xf_launch_signal(const XfPeers& peers, const XfSlabLayout& L, int S, int me, int flag, uint64_t step, int parity,
                      const uint32_t* bucket_cnt, uint32_t rows, cudaStream_t st);
void xf_launch_wait(const uint64_t* flags, int S, uint64_t step, int* error, unsigned long long timeout_ns,
                    cudaStream_t st);
void xf_launch_route(const uint32_t* row_ptr, const uint64_t* keys, uint32_t rows, uint32_t nnz_bound, uint64_t width,
                     int S, int me, uint32_t cap, const XfPeers& peers, uint64_t off_keys, uint64_t off_rows,
                     uint32_t* bucket_cnt, uint32_t* tok_pos, cudaStream_t st);
void xf_launch_pull_tokens(const XfTableView& t, const uint64_t* in_keys, const uint32_t* meta, int S, int me,
                           uint32_t cap, uint64_t work_bound, const XfPeers& peers, uint64_t off_vals,
                           uint32_t* slots, float* side_v, void* stash, cudaStream_t st);
void xf_launch_rows(bool fm, const uint32_t* row_ptr, const uint8_t* labels, int B, int mode, const uint32_t* tok_pos,
                    const void* vals, float* rowv, float* loss_out, float* pctr_out, float* abs_loss_sum,
                    cudaStream_t st);
void xf_launch_bcast_rowv(const float* src, uint32_t n_words, int S, const XfPeers& peers, uint64_t off_rowv,
                          uint64_t dst_word_off, cudaStream_t st);
void xf_launch_push_tokens_lr(const XfTableView& t, const uint32_t* slots, const uint32_t* in_rows, const float* rowv,
                              const uint32_t* meta_s, uint32_t cap, uint64_t work_bound, uint32_t seq,
                              uint64_t* rows_by_seq, unsigned long long* uniq_remote, const void* stash,
                              cudaStream_t st);
uint32_t xf_acc_touched_extra(int K, uint64_t work_bound);
void xf_launch_acc_tokens(const XfTableView& t, const uint32_t* slots, const uint32_t* in_rows, const void* rowv,
                          const uint32_t* meta_s, uint32_t cap, uint64_t work_bound, uint32_t* touched,
                          cudaStream_t st);

// a defined multi-view machine on canonical tables (step_mvm.cu); field ids < XF_MVM_FIELDS, K <= 32
#define XF_MVM_FIELDS 32
void xf_launch_step_mvm(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* fields,
                        const float* vals, const uint8_t* labels, int B, int mode, uint32_t* touched, float* loss_out,
                        float* pctr_out, float* abs_loss_sum, cudaStream_t st);

// the field-aware FM on canonical tables (step_ffm.cu); field ids < K / 4
void xf_launch_step_ffm(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys, const uint8_t* fields,
                        const float* vals, const uint8_t* labels, int B, int mode, uint32_t* touched, float* loss_out,
                        float* pctr_out, float* abs_loss_sum, cudaStream_t st);

// canonical per-k FM with feature values (step_fmc.cu)
void xf_launch_step_fmc(const XfTableView& t, const uint32_t* row_ptr, const uint64_t* keys, const float* vals,
                        const uint8_t* labels, int B, int mode, uint32_t* touched, float* loss_out, float* pctr_out,
                        float* abs_loss_sum, cudaStream_t st);

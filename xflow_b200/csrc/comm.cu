// C ABI layer 5: the multi-GPU exchange that replaces ps-lite's KVWorker slicing + ZeroMQ Van
// (ps-lite/include/ps/kv_app.h:405-460, ps-lite/src/zmq_van.h).  One process per GPU over NVLink /
// NVSwitch.  NCCL is used for bootstrap only (exchange of the cudaIpc handles, barriers at creation and
// destruction); the communicator id is created by rank 0 and distributed out of band by the launcher.
//
// A step never calls NCCL, never synchronises with the host and never moves a count through the host:
// kernels store into the peers' memory (mg.cuh: one IPC-mapped slab per rank) and order themselves with
// step counters.  Every rank is at once a WORKER (its own CSR batch) and the OWNER of one key range.
// Streams of rank r at step t (parity p = t & 1):
//
//   stream 2 (runs one step ahead)            table stream
//   --------------------------------          ------------------------------------------------------------
//   wait  DONE >= t-2 from all owners
//   xf_k_route  batch t -> owners' in_keys[p]  wait  KEYS >= t from all sources   (+ ROWV >= t-1: vals[] free)
//   signal KEYS = t (+ bucket sizes, rows)     xf_k_pull_tokens  -> sources' vals[]        (Pull handler)
//                                              signal VALS = t
//                                              wait  VALS >= t from all owners
//                                              xf_k_rows (+ broadcast of the per-row residuals)
//                                              signal ROWV = t
//                                              wait  ROWV >= t from all sources
//                                              for s in 0..S-1:  push kernel(s) of source s  (Push handler,
//                                                   one optimizer step per (source, key), rank order)
//   side stream (after the pushes): token-count readback for the growth checks, then signal DONE = t
//
// Semantics = one legal schedule of the reference's asynchronous run: every worker pulls before any push
// of the round, pushes land in rank order (tests/test_gpu_multi.py against the oracle's lock-step run).
// Buffer reuse needs no further signalling: in_keys/in_rows are double-buffered and re-written only
// after DONE of the step that used them; vals[] of step t+1 is written by pull(t+1), which every owner
// issues after it has seen ROWV = t from everybody (all row kernels of step t have finished);
// in_rowv of step t+1 is written after VALS = t+1 from every owner, i.e. after every push of step t.
#include <dlfcn.h>
#include <nccl.h>  // types and prototypes only: the library itself is bound at run time, see XfNccl
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <string>
#include <vector>

#include "internal.h"

// NCCL is bound with dlopen at the first xf_comm_* call instead of at link time.  A process that also
// hosts PyTorch already has PyTorch's own (newer) libnccl.so.2 mapped; linking ours against the system
// copy made whichever library loaded second fail on missing symbols.  RTLD_NOLOAD first reuses an
// already-mapped libnccl.so.2, otherwise the system one is loaded (plain C++ hosts).
struct XfNccl {
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclAllReduce) AllReduce = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  decltype(&ncclSend) Send = nullptr;
  decltype(&ncclRecv) Recv = nullptr;
  decltype(&ncclGroupStart) GroupStart = nullptr;
  decltype(&ncclGroupEnd) GroupEnd = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  bool ok = false;
};
static XfNccl g_nccl;

static int xf_nccl_bind() {
  if (g_nccl.ok) return XF_OK;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) {
    xf_set_error("cannot load libnccl.so.2: %s", dlerror());
    return XF_ERR_COMM;
  }
#define XF_BIND(name)                                                         \
  g_nccl.name = reinterpret_cast<decltype(g_nccl.name)>(dlsym(h, "nccl" #name)); \
  if (!g_nccl.name) {                                                         \
    xf_set_error("libnccl lacks nccl" #name);                                 \
    return XF_ERR_COMM;                                                       \
  }
  XF_BIND(GetUniqueId) XF_BIND(CommInitRank) XF_BIND(CommDestroy) XF_BIND(AllReduce) XF_BIND(AllGather)
  XF_BIND(Send) XF_BIND(Recv) XF_BIND(GroupStart) XF_BIND(GroupEnd) XF_BIND(GetErrorString)
#undef XF_BIND
  g_nccl.ok = true;
  return XF_OK;
}

#define XF_NCCL_TRY(expr)                                                                        \
  do {                                                                                           \
    ncclResult_t _r = (expr);                                                                    \
    if (_r != ncclSuccess) {                                                                     \
      xf_set_error("NCCL error at %s:%d: %s", __FILE__, __LINE__, g_nccl.GetErrorString(_r));       \
      return XF_ERR_COMM;                                                                        \
    }                                                                                            \
  } while (0)

struct xf_comm {
  ncclComm_t nccl = nullptr;
  int rank = 0, nranks = 1, device = 0;
};

static_assert(sizeof(ncclUniqueId) <= XF_COMM_ID_BYTES, "ncclUniqueId does not fit XF_COMM_ID_BYTES");

XF_DLL int xf_comm_get_id(uint8_t id[XF_COMM_ID_BYTES]) {
  if (!id) return XF_ERR_ARG;
  XF_TRY(xf_nccl_bind());
  ncclUniqueId uid;
  XF_NCCL_TRY(g_nccl.GetUniqueId(&uid));
  memset(id, 0, XF_COMM_ID_BYTES);
  memcpy(id, &uid, sizeof(uid));
  return XF_OK;
}

XF_DLL int xf_comm_create(xf_comm** out, const uint8_t id[XF_COMM_ID_BYTES], int rank, int nranks, int device) {
  if (!out || !id || nranks < 1 || rank < 0 || rank >= nranks) return XF_ERR_ARG;
  XF_TRY(xf_nccl_bind());
  XF_CUDA_TRY(cudaSetDevice(device));
  xf_comm* c = new xf_comm;
  c->rank = rank;
  c->nranks = nranks;
  c->device = device;
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  ncclResult_t r = g_nccl.CommInitRank(&c->nccl, nranks, uid, rank);
  if (r != ncclSuccess) {
    xf_set_error("ncclCommInitRank failed: %s", g_nccl.GetErrorString(r));
    delete c;
    return XF_ERR_COMM;
  }
  *out = c;
  return XF_OK;
}

XF_DLL int xf_comm_destroy(xf_comm* c) {
  if (!c) return XF_OK;
  if (c->nccl) g_nccl.CommDestroy(c->nccl);
  delete c;
  return XF_OK;
}

// Rendezvous through a file for launchers that have no other channel (the reference's CLI / c_api under
// XFLOW_RANK / XFLOW_WORLD, worker.cc): rank 0 writes the id (temporary name + rename), the others wait
// for it; rank 0 removes the file once its communicator exists, i.e. once every rank has read it.
XF_DLL int xf_comm_create_from_file(xf_comm** out, const char* path, int rank, int nranks, int device) {
  if (!out || !path || nranks < 1 || rank < 0 || rank >= nranks) return XF_ERR_ARG;
  uint8_t id[XF_COMM_ID_BYTES];
  if (rank == 0) {
    XF_TRY(xf_comm_get_id(id));
    std::string tmp = std::string(path) + ".tmp";
    FILE* f = fopen(tmp.c_str(), "wb");
    if (!f || fwrite(id, 1, XF_COMM_ID_BYTES, f) != XF_COMM_ID_BYTES || fclose(f) != 0 || rename(tmp.c_str(), path) != 0) {
      xf_set_error("cannot write the communicator id to %s", path);
      return XF_ERR_IO;
    }
  } else {
    const char* to = getenv("XFLOW_RENDEZVOUS_TIMEOUT_S");
    const int limit_ms = ((to && atoi(to) > 0) ? atoi(to) : 300) * 1000;
    int waited = 0;
    for (;;) {
      FILE* f = fopen(path, "rb");
      if (f) {
        const size_t got = fread(id, 1, XF_COMM_ID_BYTES, f);
        fclose(f);
        if (got == XF_COMM_ID_BYTES) break;
      }
      if (waited >= limit_ms) { xf_set_error("timed out waiting for rank 0's communicator id in %s", path); return XF_ERR_COMM; }
      usleep(20000);
      waited += 20;
    }
  }
  int rc = xf_comm_create(out, id, rank, nranks, device);
  if (rank == 0) remove(path);
  return rc;
}

// max over ranks of one host value (used to agree on the number of collective steps of an epoch)
XF_DLL int xf_comm_allreduce_max(xf_comm* c, uint64_t* inout) {
  if (!c || !inout) return XF_ERR_ARG;
  XF_CUDA_TRY(cudaSetDevice(c->device));
  unsigned long long* d = nullptr;
  XF_CUDA_TRY(cudaMalloc(&d, sizeof(*d)));
  XF_CUDA_TRY(cudaMemcpy(d, inout, sizeof(*d), cudaMemcpyHostToDevice));
  ncclResult_t r = g_nccl.AllReduce(d, d, 1, ncclUint64, ncclMax, c->nccl, 0);
  if (r != ncclSuccess) { cudaFree(d); xf_set_error("ncclAllReduce failed: %s", g_nccl.GetErrorString(r)); return XF_ERR_COMM; }
  XF_CUDA_TRY(cudaStreamSynchronize(0));
  XF_CUDA_TRY(cudaMemcpy(inout, d, sizeof(*d), cudaMemcpyDeviceToHost));
  cudaFree(d);
  return XF_OK;
}

int xf_comm_nranks(xf_comm* c) { return c ? c->nranks : 1; }
int xf_comm_rank(xf_comm* c) { return c ? c->rank : 0; }

XF_DLL int xf_comm_barrier(xf_comm* c) {
  if (!c) return XF_ERR_ARG;
  XF_CUDA_TRY(cudaSetDevice(c->device));
  int* d = nullptr;
  XF_CUDA_TRY(cudaMalloc(&d, sizeof(int)));
  XF_CUDA_TRY(cudaMemset(d, 0, sizeof(int)));
  XF_NCCL_TRY(g_nccl.AllReduce(d, d, 1, ncclInt, ncclSum, c->nccl, 0));
  XF_CUDA_TRY(cudaStreamSynchronize(0));
  cudaFree(d);
  return XF_OK;
}


// -------------------------------------------------------------------------------------------------
// sharded step: host orchestration
// -------------------------------------------------------------------------------------------------
struct XfMg {
  int S = 1, rank = 0, K = 0;
  bool fm = false;
  uint64_t width = 0;
  uint32_t cap = 0, max_rows = 0;
  XfSlabLayout L;
  uint8_t* slab = nullptr;  // this rank's slab (cudaMalloc, exported with cudaIpc)
  XfPeers peers;            // every rank's slab as mapped here (peers.slab[rank] == slab)
  XfDevBuf slots, tok_pos[2], bucket_cnt[2], rowv_local, touched;
  XfDevBuf side_v;  // FM, S > 1: latent rows as pulled by the tokens of sources >= 1 (see xf_k_pull_tokens)
  XfDevBuf stash;   // LR, lazy table: the state words (16 B) of every routed token's row as the Pull found them, for the Push
  uint32_t touched_extra = 0;
  cudaStream_t st2 = nullptr;
  cudaStream_t st3 = nullptr;   // token-count readbacks (a copy engine switch costs the table stream ~40 us)
  cudaEvent_t ev_meta = nullptr;
  cudaEvent_t ev_rows_done[2] = {nullptr, nullptr};  // tok_pos[p] no longer read by the table stream
  uint64_t step_no = 0;
  unsigned long long timeout_ns = 120ull * 1000000000ull;
  // received-token counts of recent steps, read back asynchronously: sizes the next steps' growth checks
  uint32_t* h_meta = nullptr;  // pinned [4][XF_MG_MAX_SHARDS * 4]
  cudaEvent_t meta_ev[4] = {nullptr, nullptr, nullptr, nullptr};
  bool meta_inflight[4] = {false, false, false, false};
  uint64_t last_recv = 0;
  bool have_recv = false;
  // XFLOW_MG_TRACE=1: CUDA events at the phase boundaries of every step, averages printed at destroy
  bool trace = false;
  std::vector<cudaEvent_t> tev;
  uint64_t tsteps = 0;
};
enum { XF_TR_NMARK = 8 };
static const char* kMgPhase[] = {"wait KEYS (route of this batch ran on stream 2)", "owner: pull tokens", "wait VALS",
                                 "worker: rows + residual broadcast", "wait ROWV", "owner: push (S sources)", "signal DONE"};
#define XF_MG_TRACE_STEPS 512
#define XF_MG_MARK(i) do { if (mg->trace && mg->tsteps < XF_MG_TRACE_STEPS) cudaEventRecord(mg->tev[mg->tsteps * XF_TR_NMARK + (i)], st); } while (0)

static int xf_mg_nccl_barrier(xf_comm* c, int* d_word, cudaStream_t st) {
  XF_NCCL_TRY(g_nccl.AllReduce(d_word, d_word, 1, ncclInt, ncclSum, c->nccl, st));
  return XF_OK;
}

// Export this rank's slab, map everybody else's.  A rank that cannot (no IPC, no peer access) makes the
// whole creation fail on every rank: there is no slower fallback path.
static int xf_mg_map_peers(xf_trainer* tr, XfMg* mg) {
  xf_comm* c = tr->comm;
  const int S = mg->S;
  cudaStream_t st = tr->table->stream;
  struct Pack { cudaIpcMemHandle_t h; uint64_t total; uint32_t cap, max_rows; int K, ok; };
  Pack mine;
  memset(&mine, 0, sizeof(mine));
  mine.ok = cudaIpcGetMemHandle(&mine.h, mg->slab) == cudaSuccess ? 1 : 0;
  if (!mine.ok) cudaGetLastError();
  mine.total = mg->L.total; mine.cap = mg->cap; mine.max_rows = mg->max_rows; mine.K = mg->K;
  std::vector<Pack> all((size_t)S);
  XfDevBuf d_all;
  XF_TRY(d_all.ensure(sizeof(Pack) * (size_t)S + 16));
  XF_CUDA_TRY(cudaMemcpyAsync((char*)d_all.p + sizeof(Pack) * (size_t)mg->rank, &mine, sizeof(Pack), cudaMemcpyHostToDevice, st));
  XF_NCCL_TRY(g_nccl.AllGather((char*)d_all.p + sizeof(Pack) * (size_t)mg->rank, d_all.p, sizeof(Pack), ncclChar, c->nccl, st));
  XF_CUDA_TRY(cudaMemcpyAsync(all.data(), d_all.p, sizeof(Pack) * (size_t)S, cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  int ok = 1;
  for (int q = 0; q < S; ++q) {
    ok &= all[q].ok;
    if (all[q].total != mine.total || all[q].cap != mine.cap || all[q].max_rows != mine.max_rows || all[q].K != mine.K) ok = 0;
  }
  memset(&mg->peers, 0, sizeof(mg->peers));
  mg->peers.slab[mg->rank] = mg->slab;
  for (int q = 0; q < S && ok; ++q) {
    if (q == mg->rank) continue;
    void* p = nullptr;
    if (cudaIpcOpenMemHandle(&p, all[q].h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
      cudaGetLastError();
      ok = 0;
    }
    mg->peers.slab[q] = (uint8_t*)p;
  }
  // agree on the outcome (sum of failures)
  int* d_word = (int*)d_all.p;
  int flag = ok ? 0 : 1;
  XF_CUDA_TRY(cudaMemcpyAsync(d_word, &flag, sizeof(int), cudaMemcpyHostToDevice, st));
  XF_TRY(xf_mg_nccl_barrier(c, d_word, st));
  XF_CUDA_TRY(cudaMemcpyAsync(&flag, d_word, sizeof(int), cudaMemcpyDeviceToHost, st));
  XF_CUDA_TRY(cudaStreamSynchronize(st));
  d_all.release();
  if (flag != 0) {
    xf_set_error("sharded trainer: cudaIpc peer mapping failed or trainer configurations differ between ranks "
                 "(%d rank(s) reported a problem; all ranks need the same max_rows / max_nnz / model)", flag);
    return XF_ERR_COMM;
  }
  return XF_OK;
}

int xf_mg_create(xf_trainer* tr) {
  xf_comm* c = tr->comm;
  XfMg* mg = new XfMg;
  tr->mg = mg;
  mg->S = c->nranks;
  mg->rank = c->rank;
  if (mg->S > XF_MG_MAX_SHARDS) {
    xf_set_error("at most %d shards supported", XF_MG_MAX_SHARDS);
    delete mg; tr->mg = nullptr;
    return XF_ERR_ARG;
  }
  const int S = mg->S;
  mg->width = 0xFFFFFFFFFFFFFFFFull / (uint64_t)S;  // postoffice.cc:138-140
  mg->cap = tr->cfg.max_nnz;                        // a (source, owner) segment can hold a whole batch
  mg->max_rows = tr->cfg.max_rows;
  mg->K = tr->table->view.K;
  mg->fm = mg->K > 0;
  mg->L = xf_slab_layout(S, mg->cap, mg->max_rows, mg->fm);
  const char* to = getenv("XFLOW_MG_TIMEOUT_S");
  if (to && atoi(to) > 0) mg->timeout_ns = (unsigned long long)atoi(to) * 1000000000ull;
  cudaStream_t st = tr->table->stream;
  int rc = XF_OK;
  do {
    if (cudaMalloc(&mg->slab, mg->L.total) != cudaSuccess) { cudaGetLastError(); xf_set_error("cannot allocate the %llu-byte exchange slab", (unsigned long long)mg->L.total); rc = XF_ERR_CUDA; break; }
    // flags, meta and counters start at zero; the rest is written before it is read
    if (cudaMemsetAsync(mg->slab, 0, mg->L.off_in_keys, st) != cudaSuccess) { rc = XF_ERR_CUDA; break; }
    // Routing and the DONE signal are what the OTHER ranks wait for; a high priority for their streams did not
    // make the 2-GPU step faster, so they run at the default priority.
    if (cudaStreamCreateWithFlags(&mg->st2, cudaStreamNonBlocking) != cudaSuccess) { rc = XF_ERR_CUDA; break; }
    if (cudaStreamCreateWithFlags(&mg->st3, cudaStreamNonBlocking) != cudaSuccess) { rc = XF_ERR_CUDA; break; }
    if (cudaEventCreateWithFlags(&mg->ev_meta, cudaEventDisableTiming) != cudaSuccess) { rc = XF_ERR_CUDA; break; }
    if ((rc = mg->slots.ensure((size_t)S * mg->cap * 4)) != XF_OK) break;
    if ((rc = mg->rowv_local.ensure((size_t)mg->max_rows * 8 + 16)) != XF_OK) break;
    const bool lazy = tr->table->view.lazy != 0;
    if (lazy && (rc = mg->stash.ensure((size_t)S * mg->cap * 16)) != XF_OK) break;
    if (!lazy) {
      mg->touched_extra = xf_acc_touched_extra(mg->K, (uint64_t)mg->cap);
      if ((rc = mg->touched.ensure(((size_t)mg->cap + 2 * (size_t)mg->touched_extra) * 4)) != XF_OK) break;
      if (mg->fm && S > 1 && (rc = mg->side_v.ensure((size_t)S * mg->cap * (size_t)mg->K * 4)) != XF_OK) break;
    }
    for (int b = 0; b < 2 && rc == XF_OK; ++b) {
      if ((rc = mg->tok_pos[b].ensure((size_t)mg->cap * 4 + 16)) != XF_OK) break;
      if ((rc = mg->bucket_cnt[b].ensure(XF_MG_MAX_SHARDS * 4)) != XF_OK) break;
      if (cudaEventCreateWithFlags(&mg->ev_rows_done[b], cudaEventDisableTiming) != cudaSuccess) rc = XF_ERR_CUDA;
    }
    if (rc != XF_OK) break;
    if (cudaHostAlloc(&mg->h_meta, 4 * XF_MG_MAX_SHARDS * 4 * sizeof(uint32_t), cudaHostAllocDefault) != cudaSuccess) { rc = XF_ERR_CUDA; break; }
    for (int i = 0; i < 4; ++i)
      if (cudaEventCreateWithFlags(&mg->meta_ev[i], cudaEventDisableTiming) != cudaSuccess) rc = XF_ERR_CUDA;
    if (rc != XF_OK) break;
    if (cudaStreamSynchronize(st) != cudaSuccess) { rc = XF_ERR_CUDA; break; }
    const char* tenv = getenv("XFLOW_MG_TRACE");
    mg->trace = tenv && *tenv == '1';
    if (mg->trace) {
      mg->tev.resize((size_t)XF_TR_NMARK * XF_MG_TRACE_STEPS);
      for (auto& e : mg->tev) cudaEventCreate(&e);
    }
    rc = xf_mg_map_peers(tr, mg);
  } while (0);
  if (rc != XF_OK) {
    if (rc == XF_ERR_CUDA) xf_set_error("CUDA error while creating the sharded trainer: %s", cudaGetErrorString(cudaGetLastError()));
    xf_mg_destroy(tr);
    return rc;
  }
  return XF_OK;
}

void xf_mg_destroy(xf_trainer* tr) {
  XfMg* mg = (XfMg*)tr->mg;
  if (!mg) return;
  cudaStream_t st = tr->table->stream;
  if (mg->st2) cudaStreamSynchronize(mg->st2);
  if (mg->st3) cudaStreamSynchronize(mg->st3);
  cudaStreamSynchronize(st);
  if (mg->trace && mg->tsteps) {
    // skip the first steps (population / allocation); events were recorded without any extra sync
    const uint64_t skip = mg->tsteps > 40 ? 30 : 0;
    double tsum[XF_TR_NMARK] = {0};
    for (uint64_t t = skip; t < mg->tsteps; ++t)
      for (int i = 0; i + 1 < XF_TR_NMARK; ++i) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, mg->tev[t * XF_TR_NMARK + i], mg->tev[t * XF_TR_NMARK + i + 1]);
        tsum[i] += ms;
      }
    const double n = (double)(mg->tsteps - skip);
    fprintf(stderr, "[xflow mg trace] rank %d of %d, steps %llu..%llu, mean ms per phase on the table stream:\n", mg->rank,
            mg->S, (unsigned long long)skip, (unsigned long long)mg->tsteps);
    double tot = 0;
    for (int i = 0; i + 1 < XF_TR_NMARK; ++i) { fprintf(stderr, "    %-52s %8.4f\n", kMgPhase[i], tsum[i] / n); tot += tsum[i] / n; }
    fprintf(stderr, "    %-52s %8.4f\n", "total", tot);
  }
  // nobody may still be storing into a slab that is about to be unmapped / freed
  bool mapped = false;
  for (int q = 0; q < mg->S; ++q) mapped |= (q != mg->rank && mg->peers.slab[q] != nullptr);
  if (mapped) {
    int* d_word = nullptr;
    if (cudaMalloc(&d_word, sizeof(int)) == cudaSuccess) {
      cudaMemsetAsync(d_word, 0, sizeof(int), st);
      if (xf_mg_nccl_barrier(tr->comm, d_word, st) == XF_OK) cudaStreamSynchronize(st);
      for (int q = 0; q < mg->S; ++q)
        if (q != mg->rank && mg->peers.slab[q]) cudaIpcCloseMemHandle(mg->peers.slab[q]);
      if (xf_mg_nccl_barrier(tr->comm, d_word, st) == XF_OK) cudaStreamSynchronize(st);
      cudaFree(d_word);
    }
  }
  if (mg->slab) cudaFree(mg->slab);
  mg->slots.release(); mg->rowv_local.release(); mg->touched.release(); mg->side_v.release(); mg->stash.release();
  for (int b = 0; b < 2; ++b) {
    mg->tok_pos[b].release(); mg->bucket_cnt[b].release();
    if (mg->ev_rows_done[b]) cudaEventDestroy(mg->ev_rows_done[b]);
  }
  for (int i = 0; i < 4; ++i) if (mg->meta_ev[i]) cudaEventDestroy(mg->meta_ev[i]);
  if (mg->h_meta) cudaFreeHost(mg->h_meta);
  if (mg->st2) cudaStreamDestroy(mg->st2);
  if (mg->st3) cudaStreamDestroy(mg->st3);
  if (mg->ev_meta) cudaEventDestroy(mg->ev_meta);
  for (auto& e : mg->tev) cudaEventDestroy(e);
  delete mg;
  tr->mg = nullptr;
}

// unique keys of this rank's batches, as counted by the owners (remote atomics into our slab)
int xf_mg_unique(xf_trainer* tr, unsigned long long* out) {
  XfMg* mg = (XfMg*)tr->mg;
  XF_CUDA_TRY(cudaMemcpyAsync(out, mg->slab + mg->L.off_uniq, sizeof(*out), cudaMemcpyDeviceToHost, tr->table->stream));
  XF_CUDA_TRY(cudaStreamSynchronize(tr->table->stream));
  return XF_OK;
}

// How many tokens this owner should expect in the coming step: the last total it has seen arrive (read
// back asynchronously, 1-2 steps old) with a margin, never less than twice its own batch.  Only the
// growth check uses it; a shard that receives far more than that in a single step while nearly full
// reports XF_ERR_FULL instead of growing (murmur-hashed keys spread evenly over the ranges).
static uint64_t xf_mg_expected_tokens(XfMg* mg, uint32_t nnz_local) {
  for (int i = 0; i < 4; ++i)
    if (mg->meta_inflight[i] && cudaEventQuery(mg->meta_ev[i]) == cudaSuccess) {
      mg->meta_inflight[i] = false;
      uint64_t tot = 0;
      for (int s = 0; s < mg->S; ++s) tot += mg->h_meta[(size_t)i * XF_MG_MAX_SHARDS * 4 + (size_t)s * 4];
      mg->last_recv = tot;
      mg->have_recv = true;
    }
  cudaGetLastError();  // cudaErrorNotReady from the queries is not an error
  uint64_t est = 2ull * nnz_local + 65536;
  if (mg->have_recv && mg->last_recv + mg->last_recv / 4 + 65536 > est) est = mg->last_recv + mg->last_recv / 4 + 65536;
  return est;
}

int xf_mg_step(xf_trainer* tr, const uint32_t* d_row_ptr, const uint64_t* d_keys, const uint8_t* d_labels,
               uint32_t rows, uint32_t nnz, int mode, float* d_abs, cudaEvent_t* pm) {
  XfMg* mg = (XfMg*)tr->mg;
  xf_table* t = tr->table;
  cudaStream_t st = t->stream, sd = mg->st2;
  const int S = mg->S, me = mg->rank;
  const XfSlabLayout& L = mg->L;
  const uint64_t step = ++mg->step_no;
  const int p = (int)(step & 1);
  const uint32_t cap = mg->cap;
  uint64_t* flags = reinterpret_cast<uint64_t*>(mg->slab + L.off_flags);
  uint32_t* meta_p = reinterpret_cast<uint32_t*>(mg->slab + L.off_meta) + (size_t)p * XF_MG_MAX_SHARDS * 4;
  const uint64_t off_keys_p = L.off_in_keys + (uint64_t)p * S * cap * 8;
  const uint64_t off_rows_p = L.off_in_rows + (uint64_t)p * S * cap * 4;
  uint32_t* bucket = mg->bucket_cnt[p].as<uint32_t>();
  uint32_t* tok_pos = mg->tok_pos[p].as<uint32_t>();

  // ---- stream 2: route this batch's tokens to their owners (overlaps the previous step's tail)
  XF_CUDA_TRY(cudaStreamWaitEvent(sd, mg->ev_rows_done[p], 0));           // tok_pos[p] free (rows of step t-2)
  if (tr->input_ready) XF_CUDA_TRY(cudaStreamWaitEvent(sd, tr->input_ready, 0));  // host path: H2D of this batch
  tr->input_ready = nullptr;
  if (step > 2) xf_launch_wait(flags + (size_t)XF_F_DONE * XF_MG_MAX_SHARDS, S, step - 2, t->d_error, mg->timeout_ns, sd);
  XF_CUDA_TRY(cudaMemsetAsync(bucket, 0, XF_MG_MAX_SHARDS * 4, sd));
  xf_launch_route(d_row_ptr, d_keys, rows, nnz, mg->width, S, me, cap, mg->peers, off_keys_p, off_rows_p, bucket, tok_pos, sd);
  xf_launch_signal(mg->peers, L, S, me, XF_F_KEYS, step, p, bucket, rows, sd);
  tr->launches += 3;

  // ---- table stream, owner: Pull handler over everything routed here
  XF_TRY(t->ensure_room(xf_mg_expected_tokens(mg, nnz)));
  XF_MG_MARK(0);
  xf_launch_wait(flags + (size_t)XF_F_KEYS * XF_MG_MAX_SHARDS, S, step, t->d_error, mg->timeout_ns, st);
  if (step > 1) xf_launch_wait(flags + (size_t)XF_F_ROWV * XF_MG_MAX_SHARDS, S, step - 1, t->d_error, mg->timeout_ns, st);
  XF_MG_MARK(1);
  if (mode == 0) XF_TRY(t->reserve_seqs(S));  // no restart of the batch numbering between this Pull and its pushes
  if (pm) XF_CUDA_TRY(cudaEventRecord(pm[0], st));
  xf_launch_pull_tokens(t->view, reinterpret_cast<const uint64_t*>(mg->slab + off_keys_p), meta_p, S, me, cap,
                        (uint64_t)nnz + 1, mg->peers, L.off_vals, mg->slots.as<uint32_t>(),
                        (mode == 0 && mg->side_v.p) ? mg->side_v.as<float>() : nullptr,
                        mode == 0 ? mg->stash.p : nullptr, st);
  if (pm) XF_CUDA_TRY(cudaEventRecord(pm[1], st));
  {
    // how many tokens arrived, for the next steps' growth checks: read back on a side stream (the counts are
    // final once the KEYS wait has passed; DONE is signalled from the same side stream, behind the copy, because
    // the sources may overwrite the counts after that)
    const int slot = (int)(step & 3);
    if (!mg->meta_inflight[slot]) {
      XF_CUDA_TRY(cudaEventRecord(mg->ev_meta, st));
      XF_CUDA_TRY(cudaStreamWaitEvent(mg->st3, mg->ev_meta, 0));
      XF_CUDA_TRY(cudaMemcpyAsync(mg->h_meta + (size_t)slot * XF_MG_MAX_SHARDS * 4, meta_p, XF_MG_MAX_SHARDS * 4 * sizeof(uint32_t),
                                  cudaMemcpyDeviceToHost, mg->st3));
      XF_CUDA_TRY(cudaEventRecord(mg->meta_ev[slot], mg->st3));
      mg->meta_inflight[slot] = true;
    }
  }
  xf_launch_signal(mg->peers, L, S, me, XF_F_VALS, step, p, nullptr, 0, st);
  tr->launches += 4;

  // ---- worker: per-row sums, sigmoid, residual against the answers in vals[]
  XF_MG_MARK(2);
  xf_launch_wait(flags + (size_t)XF_F_VALS * XF_MG_MAX_SHARDS, S, step, t->d_error, mg->timeout_ns, st);
  XF_MG_MARK(3);
  xf_launch_rows(mg->fm, d_row_ptr, d_labels, (int)rows, mode, tok_pos, mg->slab + L.off_vals, mg->rowv_local.as<float>(),
                 (mode == 0 && tr->cfg.keep_loss) ? tr->loss.as<float>() : nullptr,
                 mode == 1 ? tr->pctr.as<float>() : nullptr, d_abs, st);
  XF_CUDA_TRY(cudaEventRecord(mg->ev_rows_done[p], st));
  const uint32_t rowv_words = mg->fm ? 2 : 1;
  if (mode == 0)
    xf_launch_bcast_rowv(mg->rowv_local.as<float>(), rows * rowv_words, S, mg->peers, L.off_in_rowv,
                         (uint64_t)me * mg->max_rows * rowv_words, st);
  xf_launch_signal(mg->peers, L, S, me, XF_F_ROWV, step, p, nullptr, 0, st);
  tr->launches += 4;
  XF_MG_MARK(4);
  if (mode != 0) {
    // forward only: nothing to push; the routed tokens are no longer needed
    XF_MG_MARK(5);
    XF_MG_MARK(6);
    XF_CUDA_TRY(cudaEventRecord(mg->ev_meta, st));
    XF_CUDA_TRY(cudaStreamWaitEvent(mg->st3, mg->ev_meta, 0));
    xf_launch_signal(mg->peers, L, S, me, XF_F_DONE, step, p, nullptr, 0, mg->st3);
    ++tr->launches;
    if (mg->trace && mg->tsteps < XF_MG_TRACE_STEPS) { cudaEventRecord(mg->tev[mg->tsteps * XF_TR_NMARK + 7], st); ++mg->tsteps; }
    XF_CUDA_TRY(cudaGetLastError());
    return XF_OK;
  }

  // ---- owner: Push handler, one optimizer step per (source, key), sources in rank order
  xf_launch_wait(flags + (size_t)XF_F_ROWV * XF_MG_MAX_SHARDS, S, step, t->d_error, mg->timeout_ns, st);
  XF_MG_MARK(5);
  if (pm) XF_CUDA_TRY(cudaEventRecord(pm[2], st));
  const uint8_t* in_rowv = mg->slab + L.off_in_rowv;
  for (int s = 0; s < S; ++s) {
    const uint32_t* slots_s = mg->slots.as<uint32_t>() + (size_t)s * cap;
    const uint32_t* rows_s = reinterpret_cast<const uint32_t*>(mg->slab + off_rows_p) + (size_t)s * cap;
    const uint8_t* rowv_s = in_rowv + (size_t)s * mg->max_rows * rowv_words * 4;
    const uint32_t* meta_s = meta_p + (size_t)s * 4;
    unsigned long long* uniq_s = reinterpret_cast<unsigned long long*>(mg->peers.slab[s] + L.off_uniq);
    // every source sends about nnz / S tokens here; the kernels loop, so the bound only sizes the grid
    const uint64_t work = (uint64_t)nnz / (uint64_t)S + 1024;
    if (t->view.lazy) {
      XF_TRY(t->next_seq());
      xf_launch_push_tokens_lr(t->view, slots_s, rows_s, reinterpret_cast<const float*>(rowv_s), meta_s, cap, work, t->seq,
                               t->d_rows_by_seq, uniq_s, (const uint8_t*)mg->stash.p + (size_t)s * cap * 16, st);
      ++tr->launches;
    } else {
      xf_launch_acc_tokens(t->view, slots_s, rows_s, rowv_s, meta_s, cap, work, mg->touched.as<uint32_t>(), st);
      xf_launch_update_touched_dev(t->view, mg->touched.as<uint32_t>(), work, meta_s, meta_s + 1, cap,
                                   xf_acc_touched_extra(mg->K, work),
                                   (s > 0 && mg->side_v.p) ? mg->side_v.as<float>() + (size_t)s * cap * (size_t)mg->K : nullptr,
                                   uniq_s, st);
      tr->launches += 2;
    }
  }
  if (pm) XF_CUDA_TRY(cudaEventRecord(pm[3], st));
  XF_MG_MARK(6);
  // DONE is consumed two steps later (the sources' routing): signalled from the side stream, behind the count
  // readback (which must precede it, see above), so that its system-scope release does not sit on the table stream
  XF_CUDA_TRY(cudaEventRecord(mg->ev_meta, st));
  XF_CUDA_TRY(cudaStreamWaitEvent(mg->st3, mg->ev_meta, 0));
  xf_launch_signal(mg->peers, L, S, me, XF_F_DONE, step, p, nullptr, 0, mg->st3);
  ++tr->launches;
  if (mg->trace && mg->tsteps < XF_MG_TRACE_STEPS) { cudaEventRecord(mg->tev[mg->tsteps * XF_TR_NMARK + 7], st); ++mg->tsteps; }
  XF_CUDA_TRY(cudaGetLastError());
  return XF_OK;
}

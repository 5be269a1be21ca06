// C++ surface of the drop-in: the reference's model / optimizer / server classes for the
// data-parallel hot path, backed by the GPU-resident table and fused step of include/xflow_b200.h.
//
// Same names, constructor arguments and call order as the reference:
//   xflow::Server           src/model/server.h:20-35
//   xflow::LRWorker         src/model/lr/lr_worker.h:32-86
//   xflow::FMWorker         src/model/fm/fm_worker.h:31-95
//   xflow::w_dim, v_dim, alpha, beta, lambda1, lambda2   src/optimizer/ftrl.h:15-20
//   xflow::learning_rate                                  src/optimizer/sgd.h:16
//   xflow::FTRL::KVServerFTRLHandle_w/_v, xflow::SGD::KVServerSGDHandle_w/_v and the ps::KVServer /
//   ps::KVWorker surface they plug into live in ps_compat.h  (src/optimizer/ftrl.h:38,98 ; sgd.h:30,74)
// so that src/model/main.cc compiles against this header unchanged in shape:
//     if (server role) new xflow::Server();  ...  xflow::LRWorker w(train, test); w.epochs = N; w.train();
//
// What is intentionally different (see INTEGRATION.md):
//   * the optimizer is chosen at run time (Server(Optimizer)) instead of by commenting lines in
//     server.h:24-29; default FTRL like the reference;
//   * update(start,end) runs the fused device step (pull + loss + gradient + push + optimizer) for
//     rows [start,end) of the current block; the merge-join helpers calculate_loss /
//     calculate_gradient have no host-side equivalent;
//   * slices of a block are processed sequentially (the deterministic schedule core_num workers
//     would follow one after another); core_num defaults to 1, not hardware_concurrency().
#ifndef XFLOW_XFLOW_H_
#define XFLOW_XFLOW_H_

#include <stdint.h>

#include <fstream>
#include <functional>
#include <string>
#include <vector>

#include "../xflow_b200.h"

#define XF_CXX_API __attribute__((visibility("default")))

namespace xflow {

// global hyper-parameters, same names and defaults as the reference
extern XF_CXX_API int w_dim;            // ftrl.h:15
extern XF_CXX_API int v_dim;            // ftrl.h:16  (10)
extern XF_CXX_API float alpha;          // ftrl.h:17  (5e-2)
extern XF_CXX_API float beta;           // ftrl.h:18  (1.0)
extern XF_CXX_API float lambda1;        // ftrl.h:19  (5e-5)
extern XF_CXX_API float lambda2;        // ftrl.h:20  (10.0)
extern XF_CXX_API float learning_rate;  // sgd.h:16   (1e-3)

enum class Optimizer { FTRL = 0, SGD = 1 };

// Owns the device-resident parameter table(s) of this process (one shard per GPU).
class XF_CXX_API Server {
 public:
  // latent_dim < 0: size the table for FM with xflow::v_dim (the reference server always
  // installs both the w and the v handle, server.h:23-28)
  explicit Server(Optimizer opt = Optimizer::FTRL, int latent_dim = -1, int device = -1);
  ~Server();
  xf_table* table_lr();   // K = 0 table (created on first use)
  xf_table* table_fm();   // K = v_dim table (created on first use)
  Optimizer optimizer() const { return opt_; }
  int device() const { return device_; }
  // XFLOW_WORLD / WORLD_SIZE > 1: this process is worker `rank()` of `world()` and owns key range `rank()`
  // (postoffice.cc:134-143); comm() is the exchange the sharded trainers use (nullptr when alone)
  int rank() const { return rank_; }
  int world() const { return world_; }
  xf_comm* comm() const { return comm_; }
  // the process-wide server the workers attach to (created with defaults if none exists)
  static Server* Get();

 private:
  Optimizer opt_;
  int latent_dim_;
  int device_;
  int rank_ = 0, world_ = 1;
  xf_comm* comm_ = nullptr;
  xf_table* lr_ = nullptr;
  xf_table* fm_ = nullptr;
};

struct auc_key {  // Base::auc_key base.h:79-82
  int label;
  float pctr;
};

class XF_CXX_API WorkerBase {
 public:
  virtual ~WorkerBase();
  void train();                              // lr_worker.cc:207-217 / fm_worker.cc:277-287
  void batch_training();                     // lr_worker.cc:179-205 / fm_worker.cc:247-275
  void update(int start, int end);           // lr_worker.cc:145-177 / fm_worker.cc:204-245
  void calculate_pctr(int start, int end);   // lr_worker.cc:25-71   / fm_worker.cc:25-96
  void predict(int rank, int block);         // lr_worker.cc:73-98   / fm_worker.cc:98-124

 public:
  int epochs = 60;          // lr_worker.h:63
  int core_num = 1;         // slices per block (reference: hardware_concurrency(), lr_worker.h:40)
  int block_size = 2;       // MiB of text per training block (lr_worker.h:68)
  int test_block_size = 4;  // MiB per prediction block: 4 for LR (lr_worker.cc:80), 2 for FM (fm_worker.cc:106)
  int rank = 0;
  // metric of the last predict(): base-2 un-negated logloss and AUC as base.h:84-110 prints them
  double last_logloss = 0.0, last_auc = 0.0;
  uint64_t rows_trained = 0;

 protected:
  WorkerBase(const char* train_file, const char* test_file, int model);
  const char* model_name() const { return model_ == XF_MODEL_LR ? "LR" : "FM"; }
  void ensure_trainer(uint32_t rows, uint32_t nnz);
  void ensure_trainer_for_block(uint64_t bytes);
  void ingest_block(const char* text, uint64_t len, uint32_t* rows, uint32_t* nnz);
  void open_loader(const char* path, uint64_t block_bytes);
  uint64_t count_blocks(const char* path, uint64_t block_bytes);
  void run_blocks(uint64_t collective_blocks, const std::function<void(uint32_t rows)>& on_block);

  int model_;
  std::string train_file_path, test_file_path;
  char train_data_path[1024];
  char test_data_path[1024];
  xf_table* table_ = nullptr;
  xf_comm* comm_ = nullptr;       // non-null: the sharded (multi-GPU) step; core_num is then 1
  xf_loader* loader_ = nullptr;   // one loader for every epoch of a file
  std::string loader_path_;
  uint64_t loader_block_ = 0;
  xf_trainer* trainer_ = nullptr;
  uint32_t trainer_rows_ = 0, trainer_nnz_ = 0;
  xf_pv* pv_ = nullptr;           // XFLOW_PROGRESSIVE = 1: the training steps' progressive validation
  uint32_t pv_slices_ = 0;        // XFLOW_PV_SLICES: the slices pv_ reports
  // current block (valid inside batch_training / predict)
  const uint32_t* cur_row_ptr_ = nullptr;
  const uint64_t* cur_keys_ = nullptr;
  const uint8_t* cur_labels_ = nullptr;
  std::vector<uint32_t> slice_row_ptr_;
  std::vector<auc_key> test_auc_vec;
  std::ofstream md;
};

class XF_CXX_API LRWorker : public WorkerBase {
 public:
  LRWorker(const char* train_file, const char* test_file);
};

class XF_CXX_API FMWorker : public WorkerBase {
 public:
  FMWorker(const char* train_file, const char* test_file);
};

// what a ps-lite process would ask its environment (ps.h): single-box, one process per GPU.
// XFLOW_RANK (or RANK) and XFLOW_WORLD (or WORLD_SIZE); XFLOW_DEVICE / LOCAL_RANK pick the GPU.
XF_CXX_API int MyRank();
XF_CXX_API int NumWorkers();

}  // namespace xflow

#endif  // XFLOW_XFLOW_H_

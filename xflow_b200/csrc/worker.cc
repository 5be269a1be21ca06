// C ABI layer 1 and the C++ model/optimizer surface (include/xflow/xflow.h): the reference's
// LRWorker / FMWorker / Server call flow, re-hosted on the device table and the fused step.
// Host orchestration only; all arithmetic of the hot path runs in kernels.cu.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <fstream>
#include <functional>
#include <iostream>
#include <memory>
#include <mutex>
#include <sstream>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/xflow/xflow.h"

void xf_set_error(const char* fmt, ...);
int xf_table_policies(xf_table* t, xf_admission_config* admit, xf_eviction_config* evict, int* tracking);  // checkpoint.cu

namespace xflow {

int w_dim = 1;                // ftrl.h:15
int v_dim = 10;               // ftrl.h:16
float alpha = 5e-2;           // ftrl.h:17
float beta = 1.0;             // ftrl.h:18
float lambda1 = 5e-5;         // ftrl.h:19
float lambda2 = 10.0;         // ftrl.h:20
float learning_rate = 0.001;  // sgd.h:16

namespace {
std::mutex g_mu;
Server* g_server = nullptr;

int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}

// errors from the C ABI surface as exceptions inside the C++ façade (the reference's CHECK ->
// LOG(FATAL) -> throw dmlc::Error convention, dmlc/logging.h:183-209); XF* entry points catch them.
void must(int rc, const char* what) {
  if (rc != XF_OK) throw std::runtime_error(std::string(what) + ": " + xf_last_error());
}
}  // namespace

// Feature admission of the tables' training steps (xf_table_set_admission): XFLOW_ADMIT = bloom:<n> (a key gets a row
// once it has occurred n times, counted in a counting Bloom filter of 2^XFLOW_ADMIT_LOG2_CELLS bytes, default 30,
// 3 hashes, halved every XFLOW_ADMIT_DECAY batches, default 0 = never) or poisson:<p> (inserted with probability p).
// Unset: every key is inserted.  Single GPU only.
static xf_admission_config AdmissionFromEnv(int world) {
  xf_admission_config c;
  xf_admission_config_default(&c);
  const char* e = getenv("XFLOW_ADMIT");
  if (!e || !*e) return c;
  const std::string s(e);
  const size_t colon = s.find(':');
  const std::string kind = s.substr(0, colon), arg = colon == std::string::npos ? "" : s.substr(colon + 1);
  char* end = nullptr;
  if (kind == "bloom") {
    const long n = strtol(arg.c_str(), &end, 10);
    if (arg.empty() || *end || n < 1 || n > 255) throw std::runtime_error("XFLOW_ADMIT=bloom:<n> needs 1 <= n <= 255, got '" + s + "'");
    c.mode = XF_ADMIT_BLOOM;
    c.threshold = (uint32_t)n;
    const char* lg = getenv("XFLOW_ADMIT_LOG2_CELLS");
    if (lg && *lg) {
      const long v = strtol(lg, &end, 10);
      if (*end || v < 10 || v > 36) throw std::runtime_error(std::string("XFLOW_ADMIT_LOG2_CELLS must be 10..36, got '") + lg + "'");
      c.log2_cells = (uint32_t)v;
    }
    const char* d = getenv("XFLOW_ADMIT_DECAY");
    if (d && *d) {
      const long long v = strtoll(d, &end, 10);
      if (*end || v < 0) throw std::runtime_error(std::string("XFLOW_ADMIT_DECAY must be a batch count >= 0, got '") + d + "'");
      c.decay_batches = (uint64_t)v;
    }
  } else if (kind == "poisson") {
    const double p = strtod(arg.c_str(), &end);
    if (arg.empty() || *end || !(p >= 0.0 && p <= 1.0)) throw std::runtime_error("XFLOW_ADMIT=poisson:<p> needs 0 <= p <= 1, got '" + s + "'");
    c.mode = XF_ADMIT_POISSON;
    c.probability = (float)p;
  } else {
    throw std::runtime_error("XFLOW_ADMIT must be bloom:<n> or poisson:<p>, got '" + s + "'");
  }
  c.seed = (uint64_t)env_int("XFLOW_SEED", 0);
  if (world > 1) throw std::runtime_error("XFLOW_ADMIT is single-GPU only: unset it or run with XFLOW_WORLD = 1");
  return c;
}

// Feature eviction (xf_table_set_eviction): XFLOW_EVICT_IDLE = T drops keys no training batch touched among the last
// T, XFLOW_EVICT_MAX_KEYS = N keeps the N most recently touched; the worker sweeps after every training step that makes
// the table's batch number a multiple of XFLOW_EVICT_EVERY = E (required with a limit).  Unset: no tracking.  Single
// GPU only.  *every = E (0: eviction off).
static uint64_t env_count(const char* name, bool positive) {
  const char* v = getenv(name);
  if (!v || !*v) return 0;
  char* end = nullptr;
  const unsigned long long n = strtoull(v, &end, 10);
  if (*end || *v == '-' || (positive && n == 0))
    throw std::runtime_error(std::string(name) + " must be a count " + (positive ? "> 0" : ">= 0") + ", got '" + v + "'");
  return (uint64_t)n;
}
static xf_eviction_config EvictionFromEnv(int world, uint64_t* every) {
  xf_eviction_config c;
  c.max_idle_batches = env_count("XFLOW_EVICT_IDLE", false);
  c.max_keys = env_count("XFLOW_EVICT_MAX_KEYS", false);
  *every = env_count("XFLOW_EVICT_EVERY", true);
  const bool limit = c.max_idle_batches > 0 || c.max_keys > 0;
  if (limit && *every == 0)
    throw std::runtime_error("XFLOW_EVICT_IDLE / XFLOW_EVICT_MAX_KEYS need XFLOW_EVICT_EVERY = <batches between sweeps>");
  if (!limit && *every > 0) throw std::runtime_error("XFLOW_EVICT_EVERY needs XFLOW_EVICT_IDLE or XFLOW_EVICT_MAX_KEYS");
  if (limit && world > 1) throw std::runtime_error("XFLOW_EVICT_* is single-GPU only: unset it or run with XFLOW_WORLD = 1");
  return c;
}

// Negative sampling of the trainers' steps (xf_trainer_set_negative_sampling): XFLOW_NEG_SAMPLE = r keeps each negative
// row with probability r and weights it by 1 / r, decided per row from its keys and XFLOW_SEED.  Unset or 1: every row
// is trained with weight 1.  Single GPU only.
static float NegSampleFromEnv(int world) {
  const char* e = getenv("XFLOW_NEG_SAMPLE");
  if (!e || !*e) return 1.f;
  char* end = nullptr;
  const double r = strtod(e, &end);
  if (*end || !(r > 0.0 && r <= 1.0) || (float)r < 1.0f / 16777216.0f)
    throw std::runtime_error(std::string("XFLOW_NEG_SAMPLE must be a rate in [2^-24, 1], got '") + e + "'");
  if (world > 1)
    throw std::runtime_error("XFLOW_NEG_SAMPLE is single-GPU only: unset it or run with XFLOW_WORLD = 1");
  return (float)r;
}

// Progressive validation (xf_pv_*, xf_trainer_set_validation): XFLOW_PROGRESSIVE = 1 scores every training row with
// the model as it stood before the step that trains on it, and prints one line per epoch, then starts afresh.  Single
// GPU only.
static bool ProgressiveFromEnv(int world) {
  const char* e = getenv("XFLOW_PROGRESSIVE");
  if (!e || !*e || strcmp(e, "0") == 0) return false;
  if (strcmp(e, "1") != 0) throw std::runtime_error(std::string("XFLOW_PROGRESSIVE must be 0 or 1, got '") + e + "'");
  if (world > 1)
    throw std::runtime_error("XFLOW_PROGRESSIVE is single-GPU only: unset it or run with XFLOW_WORLD = 1");
  return true;
}

// Sliced progressive validation (xf_pv_set_slices): XFLOW_PV_SLICES = <path> reports the progressive metric per
// segment too.  The file holds one "<feature id> <slice>" pair per line; the id is hashed as the loader hashes the
// text's ids, so a row belongs to every slice its ids name.  n_slices is the largest slice + 1, binned with 8 mantissa
// bits.  Needs XFLOW_PROGRESSIVE = 1; single GPU only.  A malformed file or an id listed twice fails here.
struct PvSlices {
  std::vector<uint64_t> keys;
  std::vector<uint32_t> slice_of;
  uint32_t n = 0;  // 0: no slices
};
static PvSlices PvSlicesFromEnv(int world) {
  PvSlices ps;
  const char* path = getenv("XFLOW_PV_SLICES");
  if (!path || !*path) return ps;
  if (world > 1) throw std::runtime_error("XFLOW_PV_SLICES is single-GPU only: unset it or run with XFLOW_WORLD = 1");
  if (!ProgressiveFromEnv(1)) throw std::runtime_error("XFLOW_PV_SLICES needs XFLOW_PROGRESSIVE = 1");
  std::ifstream in(path);
  if (!in) throw std::runtime_error(std::string("XFLOW_PV_SLICES: cannot open '") + path + "'");
  std::unordered_map<uint64_t, uint64_t> line_of;  // key -> the line that named it
  std::string text, id, slice, extra;
  for (uint64_t line = 1; std::getline(in, text); ++line) {
    const std::string where = std::string("XFLOW_PV_SLICES: ") + path + " line " + std::to_string(line);
    std::istringstream ss(text);
    id.clear();
    slice.clear();
    if (!(ss >> id >> slice) || (ss >> extra) || slice.size() > 5 ||
        slice.find_first_not_of("0123456789") != std::string::npos)
      throw std::runtime_error(where + " is not '<feature id> <slice>'");
    const unsigned long s = strtoul(slice.c_str(), nullptr, 10);
    if (s >= 65536) throw std::runtime_error(where + ": slice " + slice + " is over 65535");
    const uint64_t key = xf_hash_bytes(id.data(), id.size());
    const auto ins = line_of.emplace(key, line);
    if (!ins.second)
      throw std::runtime_error(where + ": id '" + id + "' was named on line " + std::to_string(ins.first->second));
    ps.keys.push_back(key);
    ps.slice_of.push_back((uint32_t)s);
    ps.n = std::max(ps.n, (uint32_t)s + 1);
  }
  if (ps.n == 0) throw std::runtime_error(std::string("XFLOW_PV_SLICES: ") + path + " names no slice");
  return ps;
}

// the table's training-batch number (host state, no device sync)
static uint64_t TableBatches(xf_table* t) {
  uint64_t b = 0;
  if (xf_table_admission_stats(t, &b, nullptr, nullptr) != XF_OK) throw std::runtime_error(std::string("xf_table_admission_stats: ") + xf_last_error());
  return b;
}
// after a training step that started at batch number `before`: sweep if the step made the number a multiple of E
static void SweepIfDue(xf_table* t, uint64_t before) {
  static const uint64_t every = [] { uint64_t e = 0; EvictionFromEnv(1, &e); return e; }();
  if (!every) return;
  const uint64_t b = TableBatches(t);
  if (b != before && b % every == 0 && xf_table_evict(t, nullptr) != XF_OK)
    throw std::runtime_error(std::string("xf_table_evict: ") + xf_last_error());
}

// Checkpoints and exact resume (xf_table_save_state / _load_state): XFLOW_CHECKPOINT = <path> writes a state image of the
// worker's table after every epoch, with user = the epochs completed; XFLOW_RESUME = <path> loads one into the fresh
// table before training and trains the epochs [user, XFLOW_EPOCHS).  Single GPU only.
static std::string env_path(const char* name, int world) {
  const char* v = getenv(name);
  if (!v || !*v) return std::string();
  if (world > 1) throw std::runtime_error(std::string(name) + " is single-GPU only: unset it or run with XFLOW_WORLD = 1");
  return v;
}

// A resumed run keeps the policies it was saved with: the environment must describe the image's, or the run stops,
// naming the variable that differs.
static void CheckResumedPolicies(xf_table* t) {
  xf_admission_config img;
  xf_eviction_config img_ev;
  int tracking = 0;
  xf_table_policies(t, &img, &img_ev, &tracking);
  const xf_admission_config env = AdmissionFromEnv(1);
  uint64_t every = 0;
  const xf_eviction_config env_ev = EvictionFromEnv(1, &every);
  const char* var = nullptr;
  if (env.mode != img.mode) var = "XFLOW_ADMIT";
  else if (env.mode == XF_ADMIT_BLOOM && (env.threshold != img.threshold || env.hashes != img.hashes)) var = "XFLOW_ADMIT";
  else if (env.mode == XF_ADMIT_BLOOM && env.log2_cells != img.log2_cells) var = "XFLOW_ADMIT_LOG2_CELLS";
  else if (env.mode == XF_ADMIT_BLOOM && env.decay_batches != img.decay_batches) var = "XFLOW_ADMIT_DECAY";
  else if (env.mode == XF_ADMIT_POISSON && memcmp(&env.probability, &img.probability, sizeof(float)) != 0) var = "XFLOW_ADMIT";
  else if (env.mode != XF_ADMIT_ALL && env.seed != img.seed) var = "XFLOW_SEED";
  else if (env_ev.max_idle_batches != img_ev.max_idle_batches) var = "XFLOW_EVICT_IDLE";
  else if (env_ev.max_keys != img_ev.max_keys) var = "XFLOW_EVICT_MAX_KEYS";
  else if ((every != 0) != (tracking != 0)) var = "XFLOW_EVICT_EVERY";
  if (var)
    throw std::runtime_error(std::string("XFLOW_RESUME: ") + var + " describes another policy than the one the image was "
                             "saved with; a resumed run keeps its policies");
}

// XFLOW_EXPORT_PRECISION = f32 | f16 (default f32): the precision of the latent fields of every model the run exports
// (XFLOW_EXPORT_MODEL, XFLOW_EXPORT_DELTAS, XFLOW_EXPORT_SHARDED_MODEL).  With f16 each frozen model or part is
// converted (xf_model_convert) before it is written or diffed.  An LR model has no latent fields: f16 is refused.
static int ExportPrecision() {
  const char* v = getenv("XFLOW_EXPORT_PRECISION");
  if (!v || !*v || strcmp(v, "f32") == 0) return XF_PRECISION_F32;
  if (strcmp(v, "f16") == 0) return XF_PRECISION_F16;
  throw std::runtime_error(std::string("XFLOW_EXPORT_PRECISION = '") + v + "' is not f32 or f16");
}
// the frozen model m at the export precision (m itself at f32; else m is destroyed and its conversion returned)
static xf_model* AtExportPrecision(xf_model* m) {
  const int precision = ExportPrecision();
  if (precision == XF_PRECISION_F32) return m;
  xf_model* c = nullptr;
  const int rc = xf_model_convert(m, precision, &c);
  xf_model_destroy(m);
  must(rc, "xf_model_convert");
  return c;
}

// XFLOW_EXPORT_DELTAS = <prefix>: after every epoch the table frozen with the defaults.  The first epoch this process
// trains writes the whole model, <prefix>-<epochs done>.xfsm; every later epoch writes the delta from the previous
// epoch's model, <prefix>-<epochs done>.xfsd, and that model is then dropped for the new one.  A server follows the run
// by loading the first file and applying the others in order.  Single GPU only.
struct ModelDeleter {
  void operator()(xf_model* m) const { xf_model_destroy(m); }
};
using ModelPtr = std::unique_ptr<xf_model, ModelDeleter>;
static void ExportEpoch(xf_table* t, const std::string& prefix, uint64_t epochs_done, ModelPtr& prev) {
  xf_model* m = nullptr;
  must(xf_table_freeze(t, nullptr, &m), "xf_table_freeze");
  m = AtExportPrecision(m);
  ModelPtr next(m);
  const std::string path = prefix + "-" + std::to_string(epochs_done);
  if (!prev) {
    must(xf_model_save(m, (path + ".xfsm").c_str()), "xf_model_save");
  } else {
    xf_delta* d = nullptr;
    must(xf_model_diff(prev.get(), m, &d), "xf_model_diff");
    const int rc = xf_delta_save(d, (path + ".xfsd").c_str());
    xf_delta_destroy(d);
    must(rc, "xf_delta_save");
  }
  prev = std::move(next);
}

// XFLOW_EXPORT_SHARDED_MODEL = <path>: the serving model of a run of any world size.  Every rank freezes its shard of
// the table into a part (xf_table_freeze_part, the defaults) and writes <path>.part-<rank>-of-<world>.xfsp; after a
// barrier rank 0 loads the parts onto its device, merges them (xf_model_merge) and writes <path>, the file
// XFLOW_EXPORT_MODEL would write for the same rows in one table.  Rank 0 removes the part files once <path> is in
// place; on a failure they stay and the run fails.  The ranks share a filesystem, as for XFLOW_COMM_FILE.
static std::string PartPath(const std::string& path, int rank, int world) {
  return path + ".part-" + std::to_string(rank) + "-of-" + std::to_string(world) + ".xfsp";
}
static void ExportShardedModel(xf_table* t, xf_comm* comm, const std::string& path, int rank, int world, int device) {
  xf_model* part = nullptr;
  must(xf_table_freeze_part(t, nullptr, &part), "xf_table_freeze_part");
  part = AtExportPrecision(part);
  const int rc = xf_model_save(part, PartPath(path, rank, world).c_str());
  xf_model_destroy(part);
  must(rc, "xf_model_save");
  if (comm) must(xf_comm_barrier(comm), "xf_comm_barrier");
  if (rank != 0) return;
  std::vector<ModelPtr> parts;
  std::vector<xf_model*> raw;
  for (int r = 0; r < world; ++r) {
    xf_model* m = nullptr;
    must(xf_model_load(&m, PartPath(path, r, world).c_str(), device), "xf_model_load");
    parts.emplace_back(m);
    raw.push_back(m);
  }
  xf_model* whole = nullptr;
  must(xf_model_merge(raw.data(), world, device, &whole), "xf_model_merge");
  ModelPtr merged(whole);
  must(xf_model_save(whole, path.c_str()), "xf_model_save");
  for (int r = 0; r < world; ++r) remove(PartPath(path, r, world).c_str());
}

int MyRank() { return env_int("XFLOW_RANK", env_int("RANK", 0)); }
int NumWorkers() { return env_int("XFLOW_WORLD", env_int("WORLD_SIZE", 1)); }

// One process per GPU (the reference: one ps-lite worker + one server process each, local.sh).  With
// XFLOW_WORLD / WORLD_SIZE = N > 1 this process is worker `rank` of N AND the server of key range `rank`
// (postoffice.cc:134-143); the N processes find each other through a file (XFLOW_COMM_FILE).
static int LocalDevice() {
  const int d = env_int("XFLOW_DEVICE", env_int("LOCAL_RANK", -1));
  if (d >= 0) return d;
  const int n = xf_device_count();
  return n > 0 ? MyRank() % n : 0;
}
static std::string CommFile() {
  const char* f = getenv("XFLOW_COMM_FILE");
  if (f && *f) return f;
  const char* port = getenv("MASTER_PORT");
  return std::string("/tmp/xflow_b200_comm_") + (port && *port ? port : "default") + ".id";
}

// ------------------------------------------------------------------------------------------------
// Server  (src/model/server.h:20-35)
// ------------------------------------------------------------------------------------------------
Server::Server(Optimizer opt, int latent_dim, int device)
    : opt_(opt), latent_dim_(latent_dim), device_(device < 0 ? LocalDevice() : device) {
  rank_ = MyRank();
  world_ = NumWorkers();
  if (world_ < 1) world_ = 1;
  if (rank_ < 0 || rank_ >= world_)
    throw std::runtime_error("rank " + std::to_string(rank_) + " needs XFLOW_WORLD / WORLD_SIZE > rank: a worker with rank > 0 "
                             "has no servers to talk to on its own");
  AdmissionFromEnv(world_);  // a malformed XFLOW_ADMIT, or one with XFLOW_WORLD > 1, fails here
  uint64_t every = 0;
  EvictionFromEnv(world_, &every);  // likewise XFLOW_EVICT_*
  NegSampleFromEnv(world_);         // and XFLOW_NEG_SAMPLE
  PvSlicesFromEnv(world_);          // and XFLOW_PV_SLICES (its file too)
  ProgressiveFromEnv(world_);       // and XFLOW_PROGRESSIVE
  env_path("XFLOW_CHECKPOINT", world_);
  env_path("XFLOW_RESUME", world_);
  env_path("XFLOW_EXPORT_MODEL", world_);
  env_path("XFLOW_EXPORT_DELTAS", world_);
  ExportPrecision();  // a malformed XFLOW_EXPORT_PRECISION fails here
  if (!env_path("XFLOW_EXPORT_MODEL", 1).empty() && !env_path("XFLOW_EXPORT_SHARDED_MODEL", 1).empty())
    throw std::runtime_error("XFLOW_EXPORT_MODEL and XFLOW_EXPORT_SHARDED_MODEL write the same model: set one of them");
  if (world_ > 1) must(xf_comm_create_from_file(&comm_, CommFile().c_str(), rank_, world_, device_), "xf_comm_create_from_file");
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_server) g_server = this;
  std::cout << "init server success " << std::endl;  // server.h:30
}

Server::~Server() {
  {
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_server == this) g_server = nullptr;
  }
  if (lr_) xf_table_destroy(lr_);
  if (fm_) xf_table_destroy(fm_);
  if (comm_) xf_comm_destroy(comm_);
}

Server* Server::Get() {
  {
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_server) return g_server;
  }
  Optimizer opt = Optimizer::FTRL;
  const char* o = getenv("XFLOW_OPTIMIZER");
  if (o && (strcmp(o, "sgd") == 0 || strcmp(o, "SGD") == 0 || strcmp(o, "1") == 0)) opt = Optimizer::SGD;
  return new Server(opt);
}

static xf_table* make_table(Optimizer opt, int K, int device, int rank, int world) {
  xf_table_config cfg;
  xf_table_config_default(&cfg);
  cfg.device = device;
  cfg.shard_index = rank;
  cfg.num_shards = world;
  cfg.latent_dim = K;
  cfg.optimizer = (opt == Optimizer::FTRL) ? XF_OPTIMIZER_FTRL : XF_OPTIMIZER_SGD;
  cfg.alpha = alpha; cfg.beta = beta; cfg.lambda1 = lambda1; cfg.lambda2 = lambda2;
  cfg.learning_rate = learning_rate;
  cfg.seed = (uint64_t)env_int("XFLOW_SEED", 0);
  cfg.capacity = (uint64_t)1 << env_int("XFLOW_TABLE_LOG2", 20);
  xf_table* t = nullptr;
  must(xf_table_create(&t, &cfg), "xf_table_create");
  const xf_admission_config adm = AdmissionFromEnv(world);
  if (adm.mode != XF_ADMIT_ALL) {
    const int rc = xf_table_set_admission(t, &adm);
    if (rc != XF_OK) {
      const std::string err = xf_last_error();
      xf_table_destroy(t);
      throw std::runtime_error("xf_table_set_admission: " + err);
    }
  }
  uint64_t every = 0;
  const xf_eviction_config ev = EvictionFromEnv(world, &every);
  if (every) {
    const int rc = xf_table_set_eviction(t, &ev);
    if (rc != XF_OK) {
      const std::string err = xf_last_error();
      xf_table_destroy(t);
      throw std::runtime_error("xf_table_set_eviction: " + err);
    }
  }
  return t;
}

xf_table* Server::table_lr() {
  if (!lr_) lr_ = make_table(opt_, 0, device_, rank_, world_);
  return lr_;
}
xf_table* Server::table_fm() {
  if (!fm_) fm_ = make_table(opt_, latent_dim_ > 0 ? latent_dim_ : v_dim, device_, rank_, world_);
  return fm_;
}

// ------------------------------------------------------------------------------------------------
// workers
// ------------------------------------------------------------------------------------------------
WorkerBase::WorkerBase(const char* train_file, const char* test_file, int model)
    : model_(model), train_file_path(train_file ? train_file : ""), test_file_path(test_file ? test_file : "") {
  // the reference keeps the caller's pointers (lr_worker.h:81-82); we copy the strings
  core_num = env_int("XFLOW_CORE_NUM", 1);
  if (core_num < 1) core_num = 1;
  block_size = env_int("XFLOW_BLOCK_MB", 2);
  test_block_size = (model == XF_MODEL_LR) ? 4 : 2;
  if (model == XF_MODEL_LR && ExportPrecision() != XF_PRECISION_F32)
    throw std::runtime_error("XFLOW_EXPORT_PRECISION = f16: an LR model has no latent fields to narrow (its rows stay "
                             "16 bytes); unset it or set it to f32");
  Server* s = Server::Get();
  table_ = (model == XF_MODEL_LR) ? s->table_lr() : s->table_fm();
  comm_ = s->comm();
  if (comm_) core_num = 1;  // a sharded step is collective: one slice per block on every rank
  train_data_path[0] = test_data_path[0] = '\0';
}

WorkerBase::~WorkerBase() {
  if (trainer_) xf_trainer_destroy(trainer_);
  if (pv_) xf_pv_destroy(pv_);
  if (loader_) xf_loader_close(loader_);
}

LRWorker::LRWorker(const char* train_file, const char* test_file) : WorkerBase(train_file, test_file, XF_MODEL_LR) {}
FMWorker::FMWorker(const char* train_file, const char* test_file) : WorkerBase(train_file, test_file, XF_MODEL_FM) {}

void WorkerBase::ensure_trainer(uint32_t rows, uint32_t nnz) {
  if (trainer_ && rows <= trainer_rows_ && nnz <= trainer_nnz_) return;
  if (trainer_ && comm_)
    throw std::runtime_error("sharded worker: a block exceeds the trainer's limits (all ranks size their trainer from the "
                             "block size; rows without features can break that bound)");
  if (trainer_) {
    must(xf_trainer_sync(trainer_), "xf_trainer_sync");
    xf_trainer_destroy(trainer_);
    trainer_ = nullptr;
  }
  xf_trainer_config cfg;
  cfg.model = model_;
  cfg.max_rows = rows + rows / 4 + 16;
  cfg.max_nnz = nnz + nnz / 4 + 16;
  cfg.keep_loss = 0;
  must(xf_trainer_create(&trainer_, table_, comm_, &cfg), "xf_trainer_create");
  const float neg_rate = NegSampleFromEnv(1);  // XFLOW_WORLD > 1 was refused at Server creation
  if (neg_rate < 1.f)
    must(xf_trainer_set_negative_sampling(trainer_, neg_rate, (uint64_t)env_int("XFLOW_SEED", 0)),
         "xf_trainer_set_negative_sampling");
  if (pv_) must(xf_trainer_set_validation(trainer_, pv_), "xf_trainer_set_validation");
  trainer_rows_ = cfg.max_rows;
  trainer_nnz_ = cfg.max_nnz;
}

// rows [start,end) of the current block, as one fused device step
void WorkerBase::update(int start, int end) {
  if (end <= start) return;
  const uint32_t base = cur_row_ptr_[start];
  const uint32_t rows = (uint32_t)(end - start);
  const uint32_t nnz = cur_row_ptr_[end] - base;
  const uint32_t* rp = cur_row_ptr_ + start;
  if (base != 0) {
    // slice offsets must start at 0 for the step's CSR view
    slice_row_ptr_.resize(rows + 1);
    for (uint32_t i = 0; i <= rows; ++i) slice_row_ptr_[i] = cur_row_ptr_[start + i] - base;
    rp = slice_row_ptr_.data();
  }
  ensure_trainer(rows, nnz);
  const uint64_t before = TableBatches(table_);
  must(xf_trainer_step_host(trainer_, rp, cur_keys_ + base, cur_labels_ + start, rows, nnz, nullptr),
       "xf_trainer_step_host");
  SweepIfDue(table_, before);
  rows_trained += rows;
}

// a well-formed text block of `bytes` bytes holds at most bytes/8 rows ("0\ta:b:c\n") and bytes/6 tokens
// ("a:b:c ")
void WorkerBase::ensure_trainer_for_block(uint64_t bytes) {
  // sharded: one trainer for the whole run (its exchange buffers are mapped by the peers): big enough for the
  // training blocks AND the prediction blocks
  if (comm_) bytes = std::max<uint64_t>(bytes, (uint64_t)std::max(block_size, test_block_size) << 20);
  ensure_trainer((uint32_t)(bytes / 8 + 2), (uint32_t)(bytes / 6 + 2));
}

// parse one raw block on the device; a block with rows that carry no features ("0\n") can hold more rows
// than ensure_trainer_for_block assumed: size the trainer for the absolute worst case and try once more
void WorkerBase::ingest_block(const char* text, uint64_t len, uint32_t* rows, uint32_t* nnz) {
  int rc = xf_trainer_ingest_text(trainer_, text, len, rows, nnz);
  if (rc == XF_ERR_ARG && !comm_ && (trainer_rows_ < len / 2 + 2 || trainer_nnz_ < len / 4 + 2)) {
    ensure_trainer((uint32_t)(len / 2 + 2), (uint32_t)(len / 4 + 2));
    rc = xf_trainer_ingest_text(trainer_, text, len, rows, nnz);
  }
  must(rc, "xf_trainer_ingest_text");
}

// open (or rewind) the loader of `path`; one loader serves every epoch
void WorkerBase::open_loader(const char* path, uint64_t block_bytes) {
  if (loader_ && loader_path_ == path && loader_block_ == block_bytes && xf_loader_rewind(loader_) == XF_OK) return;
  if (loader_) { xf_loader_close(loader_); loader_ = nullptr; }
  must(xf_loader_open(&loader_, path, block_bytes), "xf_loader_open");
  loader_path_ = path;
  loader_block_ = block_bytes;
}

// number of blocks the loader will form from `path` (one pass over the file, no parsing)
uint64_t WorkerBase::count_blocks(const char* path, uint64_t block_bytes) {
  open_loader(path, block_bytes);
  uint64_t n = 0;
  for (;;) {
    const char* text = nullptr;
    uint64_t len = 0;
    must(xf_loader_next_raw(loader_, &text, &len), "xf_loader_next_raw");
    if (len == 0) break;
    ++n;
  }
  return n;
}

// The device-parser loop shared by training and prediction.  Pipeline per block i:
//   host   read block i+1 from the file            (xf_loader_next_raw, second text buffer)
//   device H2D + parse of block i+1                (xf_trainer_ingest_begin, ingest stream)
//   device step / forward pass of block i          (table stream)
// all three overlap; the host only waits for a parse (xf_trainer_ingest_end), never for a step.
// Sharded: every rank runs `collective_blocks` iterations (the maximum over the ranks); a rank whose file
// has ended keeps taking part with empty blocks.
void WorkerBase::run_blocks(uint64_t collective_blocks, const std::function<void(uint32_t rows)>& on_block) {
  const char* text = nullptr;
  uint64_t len = 0;
  must(xf_loader_next_raw(loader_, &text, &len), "xf_loader_next_raw");
  bool pending = false;
  if (len) { must(xf_trainer_ingest_begin(trainer_, text, len), "xf_trainer_ingest_begin"); pending = true; }
  for (uint64_t blk = 0; comm_ ? blk < collective_blocks : pending; ++blk) {
    // read the following block while the device parses this one
    const char* next_text = nullptr;
    uint64_t next_len = 0;
    if (pending) must(xf_loader_next_raw(loader_, &next_text, &next_len), "xf_loader_next_raw");
    uint32_t rows = 0, nnz = 0;
    if (pending) {
      int rc = xf_trainer_ingest_end(trainer_, &rows, &nnz);
      if (rc == XF_ERR_ARG && !comm_ && (trainer_rows_ < len / 2 + 2 || trainer_nnz_ < len / 4 + 2)) {
        // rows without features: more rows than a well-formed block can hold; re-size and parse again
        must(xf_trainer_sync(trainer_), "xf_trainer_sync");
        ensure_trainer((uint32_t)(len / 2 + 2), (uint32_t)(len / 4 + 2));
        rc = xf_trainer_ingest_text(trainer_, text, len, &rows, &nnz);
      }
      must(rc, "xf_trainer_ingest_end");
    } else {
      // sharded, file exhausted: an empty block keeps this rank in the collective step
      must(xf_trainer_ingest_text(trainer_, "", 0, &rows, &nnz), "xf_trainer_ingest_text");
    }
    if (rows == 0 && !comm_) break;  // lr_worker.cc:189
    on_block(rows);
    text = next_text;
    len = next_len;
    pending = next_len != 0;
    if (pending) must(xf_trainer_ingest_begin(trainer_, text, len), "xf_trainer_ingest_begin");
  }
}

// one line per epoch: the progressive metric of that epoch's training rows (%.17g: the report's doubles exactly),
// then one per slice (XFLOW_PV_SLICES)
static void PrintProgressive(xf_pv* pv, int epoch, uint32_t n_slices) {
  struct xf_pv_report r;
  must(xf_pv_report(pv, &r), "xf_pv_report");
  printf("progressive epoch %d : logloss = %.17g  auc = %.17g [%.17g, %.17g]  mean_pctr = %.17g  ctr = %.17g  "
         "rows = %llu\n", epoch, r.logloss, r.auc, r.auc_lo, r.auc_hi, r.mean_pctr, r.ctr, (unsigned long long)r.rows);
  if (n_slices) {
    std::vector<struct xf_pv_report> rs(n_slices);
    must(xf_pv_report_slices(pv, rs.data(), n_slices), "xf_pv_report_slices");
    for (uint32_t s = 0; s < n_slices; ++s)
      printf("progressive epoch %d slice %u : logloss = %.17g  auc = %.17g [%.17g, %.17g]  mean_pctr = %.17g  "
             "ctr = %.17g  rows = %llu\n", epoch, s, rs[s].logloss, rs[s].auc, rs[s].auc_lo, rs[s].auc_hi,
             rs[s].mean_pctr, rs[s].ctr, (unsigned long long)rs[s].rows);
  }
  fflush(stdout);
  must(xf_pv_reset(pv), "xf_pv_reset");
}

void WorkerBase::batch_training() {
  const bool host_parse = env_int("XFLOW_HOST_PARSE", 0) != 0 && !comm_;
  const uint64_t block_bytes = (uint64_t)block_size << 20;
  if (host_parse) ensure_trainer(1024, 65536);
  else ensure_trainer_for_block(block_bytes);
  const std::string checkpoint = env_path("XFLOW_CHECKPOINT", 1), resume = env_path("XFLOW_RESUME", 1);
  const std::string deltas = env_path("XFLOW_EXPORT_DELTAS", 1);
  ModelPtr exported;  // the model of the last epoch XFLOW_EXPORT_DELTAS wrote
  uint64_t first_epoch = 0;
  if (!resume.empty()) {
    // the image holds the init push's effect: the uninterrupted run made it once, before its first epoch
    must(xf_table_load_state(table_, resume.c_str(), &first_epoch), "xf_table_load_state");
    CheckResumedPolicies(table_);
  } else {
    must(xf_trainer_init_push(trainer_), "xf_trainer_init_push");  // lr_worker.cc:180-182
  }
  if (!pv_ && ProgressiveFromEnv(1)) {  // XFLOW_WORLD > 1 was refused at Server creation
    must(xf_pv_create(&pv_, Server::Get()->device(), 10), "xf_pv_create");
    const PvSlices ps = PvSlicesFromEnv(1);
    if (ps.n)
      must(xf_pv_set_slices(pv_, ps.keys.data(), ps.slice_of.data(), ps.keys.size(), ps.n, 8), "xf_pv_set_slices");
    pv_slices_ = ps.n;
    must(xf_trainer_set_validation(trainer_, pv_), "xf_trainer_set_validation");
  }
  uint64_t collective_blocks = 0;
  if (comm_) {
    collective_blocks = count_blocks(train_data_path, block_bytes);
    must(xf_comm_allreduce_max(comm_, &collective_blocks), "xf_comm_allreduce_max");
  }
  for (int epoch = (int)std::min<uint64_t>(first_epoch, (uint64_t)std::max(epochs, 0)); epoch < epochs; ++epoch) {
    open_loader(train_data_path, block_bytes);  // :184 (the reference re-opens the file every epoch)
    if (!host_parse) {
      // default path: the host only forms the block; parsing, hashing and the step run on the device
      run_blocks(collective_blocks, [&](uint32_t rows) {
        const uint32_t thread_size = rows / (uint32_t)core_num;  // :190 — remainder rows are dropped, as in the reference
        for (uint32_t i = 0; i < (uint32_t)core_num; ++i) {      // :192-196
          const uint64_t before = TableBatches(table_);
          must(xf_trainer_step_ingested(trainer_, i * thread_size, (i + 1) * thread_size), "xf_trainer_step_ingested");
          SweepIfDue(table_, before);
          rows_trained += thread_size;
        }
      });
    }
    while (host_parse) {
      // the loader alternates two output sets; before it overwrites one, the copies that read it
      // must have drained
      if (trainer_) must(xf_trainer_wait_uploads(trainer_), "xf_trainer_wait_uploads");
      uint32_t rows = 0, nnz = 0;
      must(xf_loader_next(loader_, &rows, &nnz), "xf_loader_next");
      if (rows == 0) break;  // :189
      must(xf_loader_batch(loader_, &cur_row_ptr_, &cur_keys_, &cur_labels_), "xf_loader_batch");
      const int thread_size = (int)rows / core_num;  // :190 — remainder rows are dropped, as in the reference
      for (int i = 0; i < core_num; ++i) update(i * thread_size, (i + 1) * thread_size);  // :192-196
    }
    must(xf_trainer_sync(trainer_), "xf_trainer_sync");
    if (pv_) PrintProgressive(pv_, epoch, pv_slices_);
    if (!checkpoint.empty())
      must(xf_table_save_state(table_, checkpoint.c_str(), (uint64_t)epoch + 1), "xf_table_save_state");
    if (!deltas.empty()) ExportEpoch(table_, deltas, (uint64_t)epoch + 1, exported);
    if ((epoch + 1) % 30 == 0) std::cout << "epoch : " << epoch << std::endl;  // :202
  }
  cur_row_ptr_ = nullptr;
  cur_keys_ = nullptr;
  cur_labels_ = nullptr;
}

void WorkerBase::calculate_pctr(int start, int end) {
  if (end <= start) return;
  const uint32_t base = cur_row_ptr_[start];
  const uint32_t rows = (uint32_t)(end - start);
  const uint32_t nnz = cur_row_ptr_[end] - base;
  const uint32_t* rp = cur_row_ptr_ + start;
  if (base != 0) {
    slice_row_ptr_.resize(rows + 1);
    for (uint32_t i = 0; i <= rows; ++i) slice_row_ptr_[i] = cur_row_ptr_[start + i] - base;
    rp = slice_row_ptr_.data();
  }
  ensure_trainer(rows, nnz);
  std::vector<float> pctr(rows);
  must(xf_trainer_predict_host(trainer_, rp, cur_keys_ + base, rows, nnz, pctr.data()), "xf_trainer_predict_host");
  for (uint32_t i = 0; i < rows; ++i) {
    auc_key ak;
    ak.label = cur_labels_[start + i];
    ak.pctr = pctr[i];
    test_auc_vec.push_back(ak);
    md << pctr[i] << "\t" << 1 - ak.label << "\t" << ak.label << std::endl;  // lr_worker.cc:67
  }
}

// rank 0 predicts on <test>-00000 (lr_worker.cc:213-216).  Sharded: the forward pass needs the owners of
// the keys, so every rank runs the same number of collective forward steps; ranks > 0 feed empty blocks and
// write nothing.
void WorkerBase::predict(int rank_arg, int block) {
  const bool feeding = (rank_arg == 0);
  char buffer[1024];
  snprintf(buffer, 1024, "%d_%d", rank_arg, block);
  std::string filename = buffer;
  if (feeding) {
    md.open("pred_" + filename + ".txt");  // lr_worker.cc:77
    if (!md.is_open()) std::cout << "open pred file failure!" << std::endl;
  }
  snprintf(test_data_path, 1024, "%s-%05d", test_file_path.c_str(), rank_arg);
  const uint64_t block_bytes = (uint64_t)test_block_size << 20;
  test_auc_vec.clear();
  const bool host_parse = env_int("XFLOW_HOST_PARSE", 0) != 0 && !comm_;
  uint64_t collective_blocks = 0;
  if (comm_) {
    collective_blocks = feeding ? count_blocks(test_data_path, block_bytes) : 0;
    must(xf_comm_allreduce_max(comm_, &collective_blocks), "xf_comm_allreduce_max");
  }
  if (!host_parse) ensure_trainer_for_block(block_bytes);
  std::vector<float> pctr_buf;
  std::vector<uint8_t> label_buf;
  // XFLOW_DEVICE_METRIC=1: the metric is computed on the device (radix sort + integer rank sums, metric.cu) and the
  // printed numbers come from there.  Default: the host restatement of Base::calculate_auc, whose float
  // accumulators and std::sort tie order are what the reference's own printout (and the golden fixtures) contain;
  // the predictions come back to the host either way, the reference writes every one to pred_<rank>_<block>.txt.
  xf_metric* metric = nullptr;
  if (!host_parse && env_int("XFLOW_DEVICE_METRIC", 0) != 0)
    must(xf_metric_create(&metric, Server::Get()->device()), "xf_metric_create");
  if (!host_parse) {
    if (feeding) open_loader(test_data_path, block_bytes);
    else open_loader("/dev/null", block_bytes);  // nothing to feed: every block is empty
    run_blocks(collective_blocks, [&](uint32_t rows) {
      const uint32_t thread_size = rows / (uint32_t)core_num;
      pctr_buf.resize(thread_size + 1);
      label_buf.resize(thread_size + 1);
      for (uint32_t i = 0; i < (uint32_t)core_num; ++i) {
        if (metric)
          must(xf_trainer_predict_ingested_metric(trainer_, i * thread_size, (i + 1) * thread_size, metric,
                                                  feeding ? pctr_buf.data() : nullptr, feeding ? label_buf.data() : nullptr),
               "xf_trainer_predict_ingested_metric");
        else
          must(xf_trainer_predict_ingested(trainer_, i * thread_size, (i + 1) * thread_size, pctr_buf.data(), label_buf.data()),
               "xf_trainer_predict_ingested");
        if (!feeding) continue;
        for (uint32_t r = 0; r < thread_size; ++r) {
          auc_key ak;
          ak.label = label_buf[r];
          ak.pctr = pctr_buf[r];
          test_auc_vec.push_back(ak);
          md << pctr_buf[r] << "\t" << 1 - ak.label << "\t" << ak.label << "\n";  // lr_worker.cc:67
        }
      }
    });
  }
  if (host_parse) open_loader(test_data_path, block_bytes);
  while (host_parse) {
    uint32_t rows = 0, nnz = 0;
    must(xf_loader_next(loader_, &rows, &nnz), "xf_loader_next");
    if (rows == 0) break;
    must(xf_loader_batch(loader_, &cur_row_ptr_, &cur_keys_, &cur_labels_), "xf_loader_batch");
    const int thread_size = (int)rows / core_num;
    for (int i = 0; i < core_num; ++i) calculate_pctr(i * thread_size, (i + 1) * thread_size);
  }
  if (md.is_open()) md.close();
  cur_row_ptr_ = nullptr;
  cur_keys_ = nullptr;
  cur_labels_ = nullptr;
  double dm[6] = {0, 0, 0, 0, 0, 0};
  if (metric) {
    if (feeding) must(xf_metric_finish(metric, nullptr, dm), "xf_metric_finish");
    xf_metric_destroy(metric);
  }
  if (!feeding) return;
  if (metric) {
    // Base::calculate_auc's printout (base.h:101-109) from the device-side metric
    last_logloss = dm[0];
    last_auc = dm[1];
    std::cout << "logloss: " << (float)dm[0] << "\t";
    if (dm[2] == 0 || dm[3] == 0) {
      std::cout << "tp_n = " << (int)dm[2] << std::endl;
    } else {
      std::cout << "auc = " << (float)dm[1] << "\ttp = " << (int)dm[2] << " fp = " << (size_t)dm[3] << std::endl;
    }
    if (env_int("XFLOW_EXACT_METRIC", 0))
      std::cout << "exact: logloss(ln) = " << dm[4] << "\tauc = " << dm[5] << std::endl;
    return;
  }

  // Base::calculate_auc (base.h:84-110), same printout
  std::vector<int32_t> labels(test_auc_vec.size());
  std::vector<float> pctr(test_auc_vec.size());
  for (size_t i = 0; i < test_auc_vec.size(); ++i) {
    labels[i] = test_auc_vec[i].label;
    pctr[i] = test_auc_vec[i].pctr;
  }
  double m[4] = {0, 0, 0, 0};
  xf_auc_logloss(labels.data(), pctr.data(), labels.size(), m);
  last_logloss = m[0];
  last_auc = m[1];
  std::cout << "logloss: " << (float)m[0] << "\t";
  if (m[2] == 0 || m[3] == 0) {
    std::cout << "tp_n = " << (int)m[2] << std::endl;
  } else {
    std::cout << "auc = " << (float)m[1] << "\ttp = " << (int)m[2] << " fp = " << (size_t)m[3] << std::endl;
  }
  if (env_int("XFLOW_EXACT_METRIC", 0)) {
    // the same test set in exact arithmetic (natural-log logloss, tie-aware AUC); off by default so that
    // stdout stays the reference's
    double x[4] = {0, 0, 0, 0};
    xf_auc_logloss_exact(labels.data(), pctr.data(), labels.size(), x);
    std::cout << "exact: logloss(ln) = " << x[0] << "\tauc = " << x[1] << std::endl;
  }
}

void WorkerBase::train() {
  rank = MyRank();
  std::cout << "my rank is = " << rank << std::endl;
  snprintf(train_data_path, 1024, "%s-%05d", train_file_path.c_str(), rank);
  batch_training();
  if (rank == 0) {
    std::cout << model_name() << " AUC: " << std::endl;
    predict(rank, 0);
    // XFLOW_EXPORT_MODEL = <path>: the trained table frozen into a serving model (xf_table_freeze, the defaults) and
    // written there; the keys the predict above inserted read as absent keys and are pruned
    const std::string export_model = env_path("XFLOW_EXPORT_MODEL", 1);
    if (!export_model.empty()) {
      xf_model* m = nullptr;
      must(xf_table_freeze(table_, nullptr, &m), "xf_table_freeze");
      m = AtExportPrecision(m);
      const int rc = xf_model_save(m, export_model.c_str());
      xf_model_destroy(m);
      must(rc, "xf_model_save");
    }
  } else if (comm_) {
    predict(rank, 0);  // takes part in rank 0's collective forward steps; feeds and prints nothing
  }
  const std::string sharded = env_path("XFLOW_EXPORT_SHARDED_MODEL", 1);
  if (!sharded.empty()) {
    Server* s = Server::Get();
    ExportShardedModel(table_, comm_, sharded, rank, s->world(), s->device());
  }
  std::cout << "train end......" << std::endl;
}

}  // namespace xflow

// ------------------------------------------------------------------------------------------------
// reference C API  (src/c_api/c_api.h:26-41, c_api.cc:10-20)
// ------------------------------------------------------------------------------------------------
namespace {
struct XFlowHandle {  // the reference's `class XFlow { LRWorker* lr_worker_; }`
  xflow::WorkerBase* worker = nullptr;
};

int xf_guard(const char* what, const std::function<void()>& fn) {
  try {
    fn();
    return XF_OK;
  } catch (const std::exception& e) {
    xf_set_error("%s: %s", what, e.what());
    return XF_ERR_STATE;
  } catch (...) {
    xf_set_error("%s: unknown exception", what);
    return XF_ERR_STATE;
  }
}
}  // namespace

XF_DLL int XFCreateEx(void** h, const char* train_path, const char* test_path, int model, int optimizer,
                      int latent_dim, int epochs) {
  if (!h || !train_path || !test_path) { xf_set_error("null argument"); return XF_ERR_ARG; }
  return xf_guard("XFCreate", [&]() {
    if (latent_dim > 0) xflow::v_dim = latent_dim;
    if (optimizer >= 0) {
      // make sure a server with the requested optimizer exists before the worker attaches
      bool need;
      {
        std::lock_guard<std::mutex> lk(xflow::g_mu);
        need = (xflow::g_server == nullptr);
      }
      if (need) new xflow::Server(optimizer == XF_OPTIMIZER_SGD ? xflow::Optimizer::SGD : xflow::Optimizer::FTRL);
    }
    XFlowHandle* xf = new XFlowHandle;
    if (model == XF_MODEL_FM) xf->worker = new xflow::FMWorker(train_path, test_path);
    else xf->worker = new xflow::LRWorker(train_path, test_path);
    if (epochs > 0) xf->worker->epochs = epochs;
    *h = xf;
  });
}

XF_DLL int XFCreate(void** h, const char* train_path, const char* test_path) {
  const char* e = getenv("XFLOW_EPOCHS");
  return XFCreateEx(h, train_path, test_path, XF_MODEL_LR, -1, 0, (e && *e) ? atoi(e) : 0);
}

XF_DLL int XFStartTrain(void** h) {
  if (!h || !*h) { xf_set_error("null handle"); return XF_ERR_ARG; }
  XFlowHandle* xf = reinterpret_cast<XFlowHandle*>(*h);
  return xf_guard("XFStartTrain", [&]() { xf->worker->train(); });
}

XF_DLL int XFDestroy(void** h) {
  if (!h || !*h) return XF_OK;
  XFlowHandle* xf = reinterpret_cast<XFlowHandle*>(*h);
  delete xf->worker;
  delete xf;
  *h = nullptr;
  return XF_OK;
}

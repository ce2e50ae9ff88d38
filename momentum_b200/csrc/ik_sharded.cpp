// Single-process multi-GPU (SURVEY 8e): one batch of IK instances cut into contiguous blocks, one per device, every block an
// ordinary batched solver (mb2_solver) on its own device. A host component above the C-ABI, like ik_mixed_batch.cpp.
//
// The reference runs a batch element by element on the host's threads (pymomentum/tensor_ik/tensor_ik.cpp:127-177,
// dispenso::parallel_for(0, nBatch)): the instances never exchange anything, so the device version needs no collective either —
// each shard gets its slice of the parameters / targets over PCIe, solves, and returns its slice. One host thread per shard keeps
// the copies and the (rare) convergence polls of the shards independent of each other; the only cross-shard quantity is the
// aggregate {sum of errors, iterations, instances ok}, summed here from the per-instance results.
#include "../../include/momentum_b200.h"

#include <memory>
#include <string>
#include <thread>
#include <vector>

namespace {

thread_local std::string g_shardedError;
int shardedFail(int code, const std::string& msg) {
  g_shardedError = msg;
  return code;
}

struct Shard {
  int device{0};
  int first{0}, count{0};
  mb2_character* ch{nullptr};
  mb2_solver_function* fn{nullptr};
  mb2_solver* solver{nullptr};
  ~Shard() {
    if (solver) mb2_solver_destroy(solver);
    if (fn) mb2_solver_function_destroy(fn);
    if (ch) mb2_character_destroy(ch);
  }
};

// runs work(k) for every shard on its own thread; first failure (code + message of that thread) wins
template <class F>
int forEachShard(std::vector<std::unique_ptr<Shard>>& shards, F work) {
  const size_t n = shards.size();
  std::vector<int> rc(n, MB2_OK);
  std::vector<std::string> msg(n);
  auto body = [&](size_t k) {
    rc[k] = work(*shards[k]);
    if (rc[k] != MB2_OK) msg[k] = mb2_last_error(); // thread-local in the library: read it on the thread that failed
  };
  if (n == 1) body(0);
  else {
    std::vector<std::thread> threads;
    for (size_t k = 0; k < n; ++k) threads.emplace_back(body, k);
    for (auto& t : threads) t.join();
  }
  for (size_t k = 0; k < n; ++k)
    if (rc[k] != MB2_OK) return shardedFail(rc[k], "shard " + std::to_string(k) + " (device " + std::to_string(shards[k]->device) + "): " + msg[k]);
  return MB2_OK;
}

} // namespace

struct mb2_sharded_solver {
  int totalBatch{0}, numParams{0};
  std::vector<std::unique_ptr<Shard>> shards;
  std::vector<int32_t> targetSize; // floats per instance of every error-function block
  double aggregate[3]{0, 0, 0};
};

extern "C" {

const char* mb2_sharded_last_error(void) { return g_shardedError.c_str(); }

int mb2_sharded_solver_create(const mb2_solver_function* prototype, int32_t totalBatch, int32_t numDevices, const int32_t* devices,
                              const mb2_gauss_newton_options* opt, mb2_sharded_solver** out) {
  if (!prototype || !devices || !opt || !out) return shardedFail(MB2_ERR_INVALID_ARGUMENT, "null argument");
  if (numDevices < 1 || totalBatch < numDevices) return shardedFail(MB2_ERR_INVALID_ARGUMENT, "need at least one device and one instance per device");
  const int available = mb2_device_count();
  for (int k = 0; k < numDevices; ++k)
    if (devices[k] < 0 || devices[k] >= available)
      return shardedFail(MB2_ERR_CUDA, "device " + std::to_string(devices[k]) + " is not a usable sm_90 device (" + std::to_string(available) + " found)");
  auto s = std::make_unique<mb2_sharded_solver>();
  s->totalBatch = totalBatch;
  s->numParams = mb2_solver_function_num_parameters(prototype);
  for (int i = 0; i < mb2_solver_function_num_error_functions(prototype); ++i) s->targetSize.push_back(mb2_solver_function_target_size(prototype, i));
  int first = 0;
  for (int k = 0; k < numDevices; ++k) {
    auto sh = std::make_unique<Shard>();
    sh->device = devices[k];
    sh->first = first;
    sh->count = totalBatch / numDevices + (k < totalBatch % numDevices ? 1 : 0);
    first += sh->count;
    s->shards.push_back(std::move(sh));
  }
  const mb2_character* protoCh = mb2_solver_function_character(prototype);
  const int rc = forEachShard(s->shards, [&](Shard& sh) {
    int r = mb2_character_clone(protoCh, sh.device, &sh.ch);
    if (r != MB2_OK) return r;
    if ((r = mb2_solver_function_clone(prototype, sh.ch, sh.count, &sh.fn)) != MB2_OK) return r;
    return mb2_solver_create(sh.fn, opt, &sh.solver);
  });
  if (rc != MB2_OK) return rc;
  *out = s.release();
  return MB2_OK;
}

void mb2_sharded_solver_destroy(mb2_sharded_solver* s) { delete s; }

int32_t mb2_sharded_solver_num_shards(const mb2_sharded_solver* s) { return s ? int32_t(s->shards.size()) : 0; }

int mb2_sharded_solver_shard_info(const mb2_sharded_solver* s, int32_t shard, int32_t info[3]) {
  if (!s || !info || shard < 0 || shard >= int32_t(s->shards.size())) return shardedFail(MB2_ERR_INVALID_ARGUMENT, "shard index out of range");
  const Shard& sh = *s->shards[shard];
  info[0] = sh.device; info[1] = sh.first; info[2] = sh.count;
  return MB2_OK;
}

int mb2_sharded_solver_set_options(mb2_sharded_solver* s, const mb2_gauss_newton_options* opt) {
  if (!s || !opt) return shardedFail(MB2_ERR_INVALID_ARGUMENT, "null argument");
  for (auto& sh : s->shards) {
    const int rc = mb2_solver_set_options(sh->solver, opt);
    if (rc != MB2_OK) return shardedFail(rc, mb2_last_error());
  }
  return MB2_OK;
}

int mb2_sharded_solver_set_targets(mb2_sharded_solver* s, int32_t index, const float* targets) {
  if (!s || !targets) return shardedFail(MB2_ERR_INVALID_ARGUMENT, "null argument");
  if (index < 0 || index >= int32_t(s->targetSize.size())) return shardedFail(MB2_ERR_INVALID_ARGUMENT, "error function index out of range");
  const size_t size = size_t(s->targetSize[index]);
  return forEachShard(s->shards, [&](Shard& sh) { return mb2_set_targets(sh.fn, index, targets + size_t(sh.first) * size); });
}

int mb2_sharded_solver_solve(mb2_sharded_solver* s, float* parameters, double* errors, int32_t* iterations, int32_t* status) {
  if (!s || !parameters) return shardedFail(MB2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<double> err(errors ? 0 : size_t(s->totalBatch));
  std::vector<int32_t> its(iterations ? 0 : size_t(s->totalBatch)), st(status ? 0 : size_t(s->totalBatch));
  double* e = errors ? errors : err.data();
  int32_t* it = iterations ? iterations : its.data();
  int32_t* stp = status ? status : st.data();
  const size_t n = size_t(s->numParams);
  const int rc = forEachShard(s->shards, [&](Shard& sh) { return mb2_solver_solve(sh.solver, parameters + size_t(sh.first) * n, e + sh.first, it + sh.first, stp + sh.first); });
  if (rc != MB2_OK) return rc;
  // the one "collective" of the path (SURVEY 8e), in instance order so that the sum does not depend on the number of shards
  double sumErr = 0.0, total = 0.0, ok = 0.0;
  for (int b = 0; b < s->totalBatch; ++b) { sumErr += e[b]; total += double(it[b]); ok += stp[b] == MB2_INSTANCE_OK ? 1.0 : 0.0; }
  s->aggregate[0] = sumErr; s->aggregate[1] = total; s->aggregate[2] = ok;
  return MB2_OK;
}

int mb2_sharded_solver_get_aggregate(const mb2_sharded_solver* s, double aggregate[3]) {
  if (!s || !aggregate) return shardedFail(MB2_ERR_INVALID_ARGUMENT, "null argument");
  for (int k = 0; k < 3; ++k) aggregate[k] = s->aggregate[k];
  return MB2_OK;
}

} // extern "C"

// comm.cu -- the ONE exchange step of the path, inside the library: NCCL all-reduce of the [L][D'] consensus buffer.
//
//   mlease_comm   : one NCCL communicator rank (one process per GPU: mlease_comm_create with a shared unique id; several
//                   GPUs in one process: mlease_world below).  A session with a communicator attached runs the whole
//                   RegressionAdmmTrain loop in C (mlease_admm_run) -- local x-updates, ncclAllReduce(sum, fp64) of
//                   sum_p float(x_p)+u_p on the session stream, z/u update -- with no host language in the loop.
//   mlease_world  : N sessions on N GPUs of THIS process (one worker thread per GPU, ncclCommInitAll), behind the same
//                   calls as a single session.  It is what a single-JVM RegressionAdmmTrain.run() (or the C++ job layer
//                   in host/) binds to drive the 8-GPU box; partitions go to GPU  pid % N  (SURVEY 8e).
//
// Replaces the reference's per-iteration Hadoop job + HDFS model files + driver-side mean
// (jobs/RegressionAdmmTrain.java:355-364, cons/MeanLinearModelConsumer.java:44-70) by one all-reduce.
// NCCL is resolved at run time (dlopen "libnccl.so.2"): a host process that already holds an NCCL (e.g. torch's bundled
// copy) shares it, a plain C++/JNI host gets the system library, and single-GPU use needs no NCCL at all.
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "host.cuh"

using mlease::fail;

namespace {

struct NcclApi {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  std::string err;
};

NcclApi* nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.h) break;
    }
    if (!api.h) { api.err = std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : "?"); return; }
    auto sym = [&](const char* s) { void* p = dlsym(api.h, s); if (!p) api.err = std::string("NCCL symbol missing: ") + s; return p; };
    api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
    api.CommInitAll = (decltype(api.CommInitAll))sym("ncclCommInitAll");
    api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
    api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
    api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
    api.GetVersion = (decltype(api.GetVersion))sym("ncclGetVersion");
  });
  return &api;
}

int nccl_ready() {
  NcclApi* a = nccl();
  if (!a->err.empty()) return fail(MLEASE_ERR_CUDA, a->err);
  return 0;
}

}  // namespace

struct mlease_comm {
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1, device = 0;
};

extern "C" {

int mlease_comm_unique_id(void* id128) {
  if (!id128) return fail(MLEASE_ERR_INVALID, "null id buffer");
  if (int rc = nccl_ready()) return rc;
  static_assert(sizeof(ncclUniqueId) == MLEASE_COMM_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  ncclResult_t r = nccl()->GetUniqueId(&id);
  if (r != ncclSuccess) return fail(MLEASE_ERR_CUDA, std::string("ncclGetUniqueId: ") + nccl()->GetErrorString(r));
  std::memcpy(id128, &id, sizeof(id));
  return 0;
}

int mlease_comm_create(const void* id128, int32_t rank, int32_t nranks, int32_t device, mlease_comm** out) {
  if (!id128 || !out || nranks < 1 || rank < 0 || rank >= nranks) return fail(MLEASE_ERR_INVALID, "bad communicator arguments");
  if (int rc = nccl_ready()) return rc;
  if (cudaSetDevice(device) != cudaSuccess) return fail(MLEASE_ERR_CUDA, "cudaSetDevice failed");
  ncclUniqueId id;
  std::memcpy(&id, id128, sizeof(id));
  mlease_comm* c = new mlease_comm();
  c->rank = rank; c->nranks = nranks; c->device = device;
  ncclResult_t r = nccl()->CommInitRank(&c->comm, nranks, id, rank);
  if (r != ncclSuccess) { delete c; return fail(MLEASE_ERR_CUDA, std::string("ncclCommInitRank: ") + nccl()->GetErrorString(r)); }
  *out = c;
  return 0;
}

int mlease_comm_destroy(mlease_comm* c) {
  if (!c) return 0;
  if (c->comm) { cudaSetDevice(c->device); nccl()->CommDestroy(c->comm); }
  delete c;
  return 0;
}

int mlease_comm_info(const mlease_comm* c, int32_t* rank, int32_t* nranks, int32_t* nccl_version) {
  if (!c) return fail(MLEASE_ERR_INVALID, "null communicator");
  if (rank) *rank = c->rank;
  if (nranks) *nranks = c->nranks;
  if (nccl_version) { int v = 0; nccl()->GetVersion(&v); *nccl_version = v; }
  return 0;
}

}  // extern "C"

int mlease::comm_allreduce(mlease_comm* c, double* buf, size_t count, cudaStream_t st) {
  if (!c || !c->comm) return fail(MLEASE_ERR_STATE, "no communicator attached");
  ncclResult_t r = nccl()->AllReduce(buf, buf, count, ncclDouble, ncclSum, c->comm, st);
  if (r != ncclSuccess) return fail(MLEASE_ERR_CUDA, std::string("ncclAllReduce: ") + nccl()->GetErrorString(r));
  return 0;
}

// ============================================================================================ mlease_world
struct mlease_world {
  int ndev = 0, P = 0, L = 0, Dt = 0;
  std::vector<int> devices;
  std::vector<mlease_session*> sess;
  std::vector<mlease_comm*> comms;
  std::vector<int> nparts;        // partitions resident per device
};

namespace {

// Run fn(d) for every device on its own thread (every library call sets the CUDA device itself); first error wins.
int on_all(mlease_world* w, const std::function<int(int)>& fn) {
  if (w->ndev == 1) return fn(0);
  std::vector<int> rc(w->ndev, 0);
  std::vector<std::string> msg(w->ndev);
  std::vector<std::thread> th;
  for (int d = 0; d < w->ndev; d++)
    th.emplace_back([&, d] {
      rc[d] = fn(d);
      if (rc[d]) msg[d] = mlease_last_error();   // the error string is thread-local
    });
  for (auto& t : th) t.join();
  for (int d = 0; d < w->ndev; d++)
    if (rc[d]) return fail(rc[d], "device " + std::to_string(w->devices[d]) + ": " + msg[d]);
  return 0;
}
int owner(const mlease_world* w, int pid) { return pid % w->ndev; }

}  // namespace

extern "C" {

int mlease_world_create(const mlease_admm_config* cfg, const int32_t* devices, int32_t ndev, mlease_world** out) {
  if (!cfg || !out || ndev < 1) return fail(MLEASE_ERR_INVALID, "bad world arguments");
  mlease_world* w = new mlease_world();
  w->ndev = ndev; w->P = cfg->num_blocks; w->L = cfg->num_lambdas; w->Dt = cfg->num_features + 1;
  for (int d = 0; d < ndev; d++) w->devices.push_back(devices ? devices[d] : d);
  w->sess.assign(ndev, nullptr); w->comms.assign(ndev, nullptr); w->nparts.assign(ndev, 0);
  for (int d = 0; d < ndev; d++) {
    mlease_admm_config c = *cfg;
    c.device = w->devices[d];
    c.stream = nullptr;
    if (int rc = mlease_session_create(&c, &w->sess[d])) { mlease_world_destroy(w); return rc; }
  }
  if (ndev > 1) {
    if (int rc = nccl_ready()) { mlease_world_destroy(w); return rc; }
    std::vector<ncclComm_t> cs(ndev);
    ncclResult_t r = nccl()->CommInitAll(cs.data(), ndev, w->devices.data());
    if (r != ncclSuccess) { mlease_world_destroy(w); return fail(MLEASE_ERR_CUDA, std::string("ncclCommInitAll: ") + nccl()->GetErrorString(r)); }
    for (int d = 0; d < ndev; d++) {
      w->comms[d] = new mlease_comm();
      w->comms[d]->comm = cs[d]; w->comms[d]->rank = d; w->comms[d]->nranks = ndev; w->comms[d]->device = w->devices[d];
      if (int rc = mlease_session_set_comm(w->sess[d], w->comms[d])) { mlease_world_destroy(w); return rc; }
    }
  }
  *out = w;
  return 0;
}

int mlease_world_destroy(mlease_world* w) {
  if (!w) return 0;
  for (auto* s : w->sess) if (s) mlease_session_destroy(s);
  for (auto* c : w->comms) if (c) mlease_comm_destroy(c);
  delete w;
  return 0;
}

int mlease_world_num_devices(const mlease_world* w) { return w ? w->ndev : 0; }

int mlease_world_add_partition_dense(mlease_world* w, int32_t pid, int64_t nrows, const float* X, int64_t ldx, const int32_t* response,
                                     const float* weight, const float* offset) {
  if (!w) return fail(MLEASE_ERR_INVALID, "null world");
  if (pid < 0 || pid >= w->P) return fail(MLEASE_ERR_INVALID, "Map key is wrong! key has to be in the range of [0,numPartitions-1].");
  const int d = owner(w, pid);
  if (int rc = mlease_add_partition_dense(w->sess[d], pid, nrows, X, ldx, response, weight, offset)) return rc;
  w->nparts[d]++;
  return 0;
}

int mlease_world_add_partition_csr(mlease_world* w, int32_t pid, int64_t nrows, const int64_t* rowptr, const int32_t* colidx, const float* vals,
                                   const int32_t* response, const float* weight, const float* offset) {
  if (!w) return fail(MLEASE_ERR_INVALID, "null world");
  if (pid < 0 || pid >= w->P) return fail(MLEASE_ERR_INVALID, "Map key is wrong! key has to be in the range of [0,numPartitions-1].");
  const int d = owner(w, pid);
  if (int rc = mlease_add_partition_csr(w->sess[d], pid, nrows, rowptr, colidx, vals, response, weight, offset)) return rc;
  w->nparts[d]++;
  return 0;
}

static int world_check_complete(mlease_world* w) {
  int tot = 0;
  for (int d = 0; d < w->ndev; d++) {
    tot += w->nparts[d];
    if (w->nparts[d] == 0)
      return fail(MLEASE_ERR_STATE, "device " + std::to_string(w->devices[d]) + " owns no partition (num.blocks must be >= the number of GPUs)");
  }
  if (tot != w->P) return fail(MLEASE_ERR_STATE, "Some models failed! (" + std::to_string(tot) + " of " + std::to_string(w->P) + " partitions present)");
  return 0;
}

int mlease_world_begin(mlease_world* w) {
  if (!w) return fail(MLEASE_ERR_INVALID, "null world");
  if (int rc = world_check_complete(w)) return rc;
  return on_all(w, [&](int d) { return mlease_admm_begin(w->sess[d]); });
}

int mlease_world_begin_initialized(mlease_world* w, const double* z0, float boost_rate) {
  if (!w) return fail(MLEASE_ERR_INVALID, "null world");
  if (int rc = world_check_complete(w)) return rc;
  return on_all(w, [&](int d) { return mlease_admm_begin_initialized(w->sess[d], z0, boost_rate); });
}

int mlease_world_iterate(mlease_world* w, double* maxdiff, int32_t* stop) {
  if (!w) return fail(MLEASE_ERR_INVALID, "null world");
  std::vector<double> md(w->ndev, 0.0);
  std::vector<int32_t> st(w->ndev, 0);
  if (int rc = on_all(w, [&](int d) { return mlease_admm_iterate(w->sess[d], &md[d], &st[d]); })) return rc;
  if (maxdiff) *maxdiff = md[0];   // every rank applies the z-update to the same reduced buffer: identical on all devices
  if (stop) *stop = st[0];
  return 0;
}

int mlease_world_run(mlease_world* w, int32_t num_iters, int32_t* iters_done) {
  if (!w) return fail(MLEASE_ERR_INVALID, "null world");
  if (int rc = world_check_complete(w)) return rc;
  std::vector<int32_t> done(w->ndev, 0);
  if (int rc = on_all(w, [&](int d) { return mlease_admm_run(w->sess[d], num_iters, nullptr, nullptr, &done[d]); })) return rc;
  if (iters_done) *iters_done = done[0];
  return 0;
}

int mlease_world_get_z(mlease_world* w, int32_t l, double* out) { return w ? mlease_get_z(w->sess[0], l, out) : fail(MLEASE_ERR_INVALID, "null world"); }
int mlease_world_get_final_model(mlease_world* w, int32_t l, float* out) {
  return w ? mlease_get_final_model(w->sess[0], l, out) : fail(MLEASE_ERR_INVALID, "null world");
}
int mlease_world_get_x(mlease_world* w, int32_t pid, int32_t l, double* out) {
  return (w && pid >= 0) ? mlease_get_x(w->sess[owner(w, pid)], pid, l, out) : fail(MLEASE_ERR_INVALID, "bad argument");
}
int mlease_world_get_u(mlease_world* w, int32_t pid, int32_t l, float* out) {
  return (w && pid >= 0) ? mlease_get_u(w->sess[owner(w, pid)], pid, l, out) : fail(MLEASE_ERR_INVALID, "bad argument");
}
int mlease_world_get_uplusx(mlease_world* w, int32_t pid, int32_t l, float* out) {
  return (w && pid >= 0) ? mlease_get_uplusx(w->sess[owner(w, pid)], pid, l, out) : fail(MLEASE_ERR_INVALID, "bad argument");
}
int mlease_world_fit_partition(mlease_world* w, int32_t pid, double* x, const double* m, const double* q, int32_t* newton_steps) {
  return (w && pid >= 0) ? mlease_fit_partition(w->sess[owner(w, pid)], pid, x, m, q, newton_steps) : fail(MLEASE_ERR_INVALID, "bad argument");
}
// every device sums its own partitions, the all-reduce inside mlease_admm_posterior sums the devices, and every device factorises
// the same sum; device 0's result is returned
int mlease_world_admm_posterior(mlease_world* w, int32_t lambda_index, const double* z, int32_t full, double* var, double* cov) {
  if (!w || !var) return fail(MLEASE_ERR_INVALID, "null argument");
  if (int rc = world_check_complete(w)) return rc;
  std::vector<std::vector<double>> vd(w->ndev), cd(w->ndev);
  return on_all(w, [&](int d) {
    double* v = var;
    double* c = cov;
    if (d > 0) {
      vd[d].resize(w->Dt);
      v = vd[d].data();
      if (cov) { cd[d].resize((size_t)w->Dt * w->Dt); c = cd[d].data(); }
    }
    return mlease_admm_posterior(w->sess[d], lambda_index, z, full, v, c);
  });
}

int mlease_world_get_stats(mlease_world* w, mlease_stats* out) {
  if (!w || !out) return fail(MLEASE_ERR_INVALID, "null argument");
  std::memset(out, 0, sizeof(*out));
  for (int d = 0; d < w->ndev; d++) {
    mlease_stats s;
    if (int rc = mlease_get_stats(w->sess[d], &s)) return rc;
    out->k1_passes += s.k1_passes; out->gram_builds += s.gram_builds; out->newton_steps += s.newton_steps;
    out->rejected_steps += s.rejected_steps; out->kernel_launches += s.kernel_launches; out->not_converged += s.not_converged;
    out->k1_shared_bytes += s.k1_shared_bytes; out->k1_fused = s.k1_fused;
    if (d == 0) { out->last_iter_slots = s.last_iter_slots; out->last_maxdiff = s.last_maxdiff; out->liblinear_epsilon = s.liblinear_epsilon; }
  }
  return 0;
}

}  // extern "C"

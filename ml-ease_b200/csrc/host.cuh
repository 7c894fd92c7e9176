// host.cuh -- private to the host files of libmlease_b200.so (not installed, not part of the C ABI): error reporting, device
// memory ownership, the device checks, the partition / batch / session state and the batch and ingest functions they share.
// No CPU fallback anywhere: every compute entry point needs a CUDA device and fails loudly without one.
#pragma once
#include <cuda.h>

#include <cstring>
#include <string>
#include <vector>

#include "../../include/mlease_b200.h"
#include "kernels.cuh"

// nothing declared here is exported from the library
#pragma GCC visibility push(hidden)

namespace mlease {

// sets the thread-local error string that mlease_last_error returns; returns code
int fail(int code, const std::string& msg);

#define CK(call)                                                                                                  \
  do {                                                                                                            \
    cudaError_t e__ = (call);                                                                                     \
    if (e__ != cudaSuccess)                                                                                       \
      return fail(MLEASE_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__) + " (" + __FILE__ + ":" + \
                                       std::to_string(__LINE__) + ")");                                           \
  } while (0)

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// Device (cudaMalloc) or pinned host (cudaMallocHost) allocations, freed with their owner.  get: count elements of T (16 B when
// count is 0), zero-filled on request; adopt: device memory another function allocated.
template <bool Pinned>
class MemOwner {
 public:
  MemOwner() = default;
  MemOwner(const MemOwner&) = delete;
  MemOwner& operator=(const MemOwner&) = delete;
  ~MemOwner() { for (void* p : ptrs_) Pinned ? cudaFreeHost(p) : cudaFree(p); }
  template <class T> int get(T** p, size_t count, bool zero) {
    const size_t bytes = count * sizeof(T) ? count * sizeof(T) : 16;
    CK(Pinned ? cudaMallocHost((void**)p, bytes) : cudaMalloc((void**)p, bytes));
    ptrs_.push_back(*p);
    if (zero && Pinned) std::memset(*p, 0, bytes);
    if (zero && !Pinned) CK(cudaMemset(*p, 0, bytes));
    return 0;
  }
  void adopt(void* p) { ptrs_.push_back(p); }

 private:
  std::vector<void*> ptrs_;
};
using DevMem = MemOwner<false>;
using PinnedMem = MemOwner<true>;

bool is_device_ptr(const void* p);
// the device for a compute call: present (no CPU fallback), ordinal valid, made current, sm_90; *num_sms if not NULL
int open_device(int device, int* num_sms);

// returns a device pointer for host-or-device input (copies when the pointer is not device memory)
template <class T> int to_device(DevMem& mem, const T* in, size_t count, const T** out, cudaStream_t st) {
  if (!in || is_device_ptr(in)) { *out = in; return 0; }
  T* d;
  if (int rc = mem.get(&d, count, false)) return rc;
  CK(cudaMemcpyAsync(d, in, count * sizeof(T), cudaMemcpyDefault, st));
  *out = d;
  return 0;
}

// One uploaded partition: its data fields of Problem (X or the CSR arrays, labels, the derived lists and scalars)
struct PartData {
  int pid = -1;
  bool csr = false;
  Problem data{};
};

// A batch of problems with identical shape that advance in lockstep through the Newton slots.
struct Batch {
  int nprob = 0, Dt = 0, ldx = 0, Dp = 0, ldh = 0;
  bool csr = false;
  int has_bias = 1;
  int k1_grid = 1, gram_slices = 1, ntiles = 0;
  int gram_from_csr = 0;          // every problem of the batch assembles its Gram tiles from CSR (no dense bf16 operand)
  int csr_gram = 0;               // the CSR Gram kernel of the batch (CSR_GRAM_WGMMA / CSR_GRAM_SPARSE, set in batch_alloc), else 0
  int csr_fx = 0;                 // CSR rows sorted and unique: the deterministic K1 kernels (fixed point / segment lists) and their Hv
                                  // modes run, sqrt(d) goes to sdvec.  The Gram path has it with its block-major lists; a matrix-free
                                  // session (policy 2) builds no lists and has it from the rows alone
  int group_L = 1;                // problems b = g * group_L + l share the data of partition g (the lambdas of one partition)
  int k1_fused = 0;               // the fused multi-lambda CSR K1 runs (segment lists present): one launch, grid (sg_S, nprob / group_L)
  int k1f_LP = 1;                 // lambdas padded to 1 / 2 / 4 in the interleaved shared-memory vectors
  size_t k1f_smem = 0;
  int k1_dyn = 0;                 // > 0: K1 CTAs are dealt to the running problems at run time (value = nprob, <= 32); k1_grid = whole grid
  int rebuild_is_expensive = 0;   // cost model: Gram + Cholesky + inverse vs one K1 pass (set in batch_alloc)
  int matfree = 0;                // Newton-CG directions from Hv passes: no Gram, factor or inverse is allocated (set in batch_alloc)
  bool has_factor = false;        // batch_factor has run on this batch: Hinv / Ysym hold a factorisation
  bool ysym_shared = false;       // a wide batch whose followers were pointed at their leader's Ysym (chol_share_end_kernel)
  std::vector<Problem> h;
  Problem* d = nullptr;
  Problem* d_compact = nullptr;   // large batches: Problem structs of the problems that may rebuild in the next slot
  Ctrl* d_ctrl = nullptr;
  CUtensorMap* d_tmaps = nullptr;
  short* d_tiles = nullptr;
  std::vector<Ctrl> mirror;   // host copy of the control blocks as of the last read-back
  Ctrl* h_ctrl[2] = {nullptr, nullptr};   // pinned read-back buffers of the slot pipeline (small batches)
  cudaEvent_t slot_ev[2] = {nullptr, nullptr};
  DevMem mem;
  PinnedMem pinned;
  ~Batch() {
    for (int i = 0; i < 2; i++) if (slot_ev[i]) cudaEventDestroy(slot_ev[i]);
  }
};

struct Counters {
  long long k1_passes = 0, gram_builds = 0, newton_steps = 0, rejected = 0, launches = 0;
  int not_converged = 0, last_slots = 0;
  double k1_bytes = 0;     // algorithmic bytes of all K1 passes (SURVEY 8d): dense n*(4*ldx+9), CSR 8*nnz+8*n+9*n
  double k1_emit_bytes = 0;// extra bytes written by passes that emitted the scaled bf16 copy (n*Dp*2)
  double gram_flops = 0;   // flops of all Gram builds as run: n*Dt*(Dt+1) (wgmma, lower triangle, 2 flop/MAC), or 2 per product
                           // the sparse CSR kernel forms
  double k1_shared_bytes = 0;  // CSR: bytes of the K1 passes when the lambdas of a partition are counted as ONE read of its rows:
                               // per (partition, slot) with A active lambdas 8*nnz + 9*n + 8*n*A (rows once, r/d out per lambda)
};

// Optional per-kernel device timing (CUDA events on the launching stream) for bench.py's roofline.
struct Profiler {
  bool on = false;
  struct Rec { int cat; cudaEvent_t a, b; };
  std::vector<Rec> recs;
  std::vector<cudaEvent_t> pool;
  double ms[4] = {0, 0, 0, 0};
  long long n[4] = {0, 0, 0, 0};
  cudaEvent_t get() {
    if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
  }
  void begin(int cat, cudaStream_t st) {
    if (!on) return;
    Rec r; r.cat = cat; r.a = get(); r.b = get();
    cudaEventRecord(r.a, st);
    recs.push_back(r);
  }
  void end(cudaStream_t st) {
    if (!on) return;
    cudaEventRecord(recs.back().b, st);
  }
  void resolve() {   // call after a stream synchronize
    for (auto& r : recs) {
      float t = 0;
      if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) { ms[r.cat] += t; n[r.cat]++; }
      pool.push_back(r.a); pool.push_back(r.b);
    }
    recs.clear();
  }
  ~Profiler() { for (auto& r : recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); } for (auto e : pool) cudaEventDestroy(e); }
};

// batch.cu
int batch_alloc(Batch& B, int num_sms, int hessian_policy, int csr_gram_force = 0);
cudaError_t batch_gram(const Batch& B, const Problem* d_probs, int n, int force, cudaStream_t st, int* launches, int share = 0);
cudaError_t batch_k1(Batch& B, int force_emit, cudaStream_t st, int* launches, int mode = K1_GRAD);
int batch_factor(Batch& B, const Problem* d_hess, int n_hess, int share, bool share_fact, int skip_prep, cudaStream_t st, int* launches);
// what one slot of an x-update runs with: the stream, profiler and launch counter, the problems its rebuild launches run over,
// the cold-start sharing of slot 0 (with the flops it saved), the flag words, and whether the end-of-slot poll kernel runs
struct SlotCtx {
  cudaStream_t st; Profiler* pf; int* launches;
  const Problem* d_hess; int n_hess;
  int share_first_gram, share_first_factor;
  double* shared_flops;
  int* h_flag; int* d_flag;
  bool poll;
};
int batch_slot(Batch& B, const SlotCtx& x, int slot_idx, bool with_hess, bool spec);
int batch_xupdate(Batch& B, cudaStream_t st, double xtol, int max_newton, int policy, int invalidate, int* h_flag, int* d_flag,
                  Counters& cnt, Profiler* prof = nullptr, int share_first_gram = 0, int share_first_factor = 0);

// ingest.cu.  Each reads back through d_flag / h_flag (device / pinned, two ints at least) where it reads back.
// Labels of n rows from host or device input: response {1,0,-1} -> int8 y, weight (>= 0, 1 if NULL) -> w, offset (0 if NULL) -> o;
// *wmax (if not NULL): the largest weight, from the same read-back.
int ingest_labels(cudaStream_t st, long long n, const int32_t* response, const float* weight, const float* offset, signed char* y, float* w,
                  float* o, int* d_flag, int* h_flag, float* wmax);
// Enqueues the checks of device CSR arrays: a column id outside [0, Dg) sets d_flag[0], a row whose column ids are not strictly
// increasing sets d_flag[1] (both must be 0 before); binary rewrites every stored value to 1.  The caller reads the flags back.
void check_csr(cudaStream_t st, long long n, long long nnz, const long long* rowptr, const int* colidx, float* vals, int Dg, int binary,
               int* d_flag);
// n rows of Dg floats, ld_in apart, from host or device into dst with ldx floats a row; column Dg is 1 (has_bias) or 0, like the
// rest of the padding.
int upload_dense_rows(float* dst, int ldx, const float* src, long long ld_in, long long n, int Dg, int has_bias, cudaStream_t st);
// dst[i] = src[i] - base for i in [0, n]: the row pointers of a row range copied out of a larger CSR, made range-local
void rebase_rowptr(cudaStream_t st, long long n, const long long* src, long long base, long long* dst);

// Keyed calls (keyed_fit.cu, k5_score.cu).  keyed_budget: the device bytes the mode decision and the chunk plan of a keyed call may
// use, min(free, the test cap of mlease_internal_set_keyed_budget).  keyed_record: the key boundaries of the chunks the call ran and
// whether it streamed, with the host time the streamed rows took to stage and the time the solve waited for them.
size_t keyed_budget(size_t free_b);
void keyed_record(const std::vector<long long>& bounds, bool streamed, double stage_ms, double wait_ms);
// host copies of rowptr[idx[i]] (host or device rowptr)
int gather_rowptr(const int64_t* rowptr, const std::vector<long long>& idx, std::vector<long long>& out);
// whether the CUDA copy engines can read p directly (device, managed or pinned host memory)
bool is_dma_ptr(const void* p);

}  // namespace mlease

struct mlease_session {
  mlease_admm_config cfg;
  std::vector<float> lambdas, rhos, lambda_map;
  int Dg = 0, Dt = 0, ldx = 0, L = 0, P = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;   // H2D of a CSR partition's arrays, overlapped with the previous partition's layout build
  cudaEvent_t copy_ev = nullptr;        // orders copy_stream after what the caller queued on `stream` (e.g. kernels that produce device inputs)
  int pending_csr = -1;                 // index into parts of the CSR partition whose checks and lists are not built yet
  int num_sms = 132;
  std::vector<mlease::PartData> parts;
  mlease::DevMem mem;
  mlease::PinnedMem pinned;
  bool any_csr = false, any_dense = false;
  mlease::Batch* batch = nullptr;    // ADMM problems, b = local_part * L + l
  mlease::Batch* scratch = nullptr;  // 1 problem for mlease_objective / mlease_fit_partition / timing
  int scratch_part = -1;
  double* d_z = nullptr;
  double* d_wz = nullptr;
  double* d_rho = nullptr;   // [L] rho_eff of the coming iteration
  double* d_diff = nullptr;
  double* d_l1thr = nullptr; // [L] soft-threshold of the L1 z-update (regularizer = 1), else NULL
  double* d_exch = nullptr;  // [L][Dt] (+1: failed-fit count of this rank) for mlease_admm_run / mlease_admm_iterate
  mlease_comm* comm = nullptr;   // NCCL communicator of a multi-GPU job (not owned), or NULL
  int* d_flag = nullptr;
  int* h_flag = nullptr;     // pinned
  double* h_small = nullptr; // pinned, >= 4*L doubles
  std::vector<double> rho_fact;  // rho_eff the current Cholesky factors were built with
  int iter = 0;
  float liblinear_eps = 0.01f;
  double mindiff = 99999999;
  double last_maxdiff = 0;
  bool begun = false;
  float boost_rate = 0.f;    // initialize.boost.rate of the current run (0: cold start from z = {})
  mlease::Counters cnt;
  mlease::Profiler prof;
  double xtol = 1e-8;
  int max_newton = 50;
  int csr_gram_force = 0;    // 0: batch_alloc picks the CSR Gram kernel; CSR_GRAM_WGMMA / CSR_GRAM_SPARSE (mlease_internal_set_csr_gram)
  ~mlease_session() {
    delete batch;
    delete scratch;
    if (copy_stream) cudaStreamDestroy(copy_stream);
    if (copy_ev) cudaEventDestroy(copy_ev);
  }
};

namespace mlease {

// session.cu: the one-problem scratch batch of partition pid (device made current, pending CSR lists built), the Hv vector v
// (Dt entries) of problem b, and the cleared control block after a one-off factorisation
int scratch_for(mlease_session* s, int pid, Batch** B);
int load_hv(Batch& B, int b, const double* v, cudaStream_t st);
int reset_ctrl(Batch& B);
// session.cu: the reducers' rho of iteration `iter` for lambda l (the boost at iteration 1, then rho.adapt.coefficient), and the z/u
// update of an iteration around the caller's one stream synchronisation: consensus_enqueue (rho of the next iteration to d_rho, K4 on
// the summed exchange, read-back of the per-lambda diff), consensus_finish (maxdiff, mindiff, the stop rule)
double rho_eff_for_iter(mlease_session* s, int l, int iter);
int consensus_enqueue(mlease_session* s, const double* exchange_sum_dev);
void consensus_finish(mlease_session* s, double* maxdiff, int32_t* stop);
// ingest.cu: checks and derived lists of one uploaded CSR partition
int csr_build_layout(mlease_session* s, PartData& pd);
// comm.cu: in-place sum of `count` doubles over the communicator's ranks on `st`
int comm_allreduce(mlease_comm* c, double* buf, size_t count, cudaStream_t st);

}  // namespace mlease

#pragma GCC visibility pop

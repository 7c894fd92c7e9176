// common.cuh -- shared device structures and sm_90a PTX wrappers (mbarrier, bulk-copy TMA,
// tensor-map TMA, wgmma).  H100 only: compile with -gencode arch=compute_90a,code=sm_90a.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mlease {

// Secant pairs kept on top of the (possibly stale) explicit inverse Hessian.  Measured at 1M x 10k x 1 %: 12 / 16 pairs save
// 2-4 % of the K1 passes and cost 45-60 % more two-loop time.
constexpr int BFGS_M = 6;
constexpr int CG_MAX_STEPS = 64;  // CG steps per matrix-free Newton direction (newton.cu, where the choice is explained)

// ------------------------------------------------------------------------------------------
// Per-problem control block, device resident.  A "problem" is one (local partition, lambda)
// x-update = one AdmmReducer.reduce call (jobs/RegressionAdmmTrain.java:642-718).
// Every kernel of the Newton slot reads these flags and exits early when it has nothing to
// do, so the host launches a fixed kernel sequence per slot and never branches on device data.
// ------------------------------------------------------------------------------------------
struct Ctrl {
  int done;          // x-update finished (converged or gave up)
  int have_dir;      // a Newton direction exists for the accepted point
  int need_solve;    // accepted a point this slot -> compute a new direction
  int need_hess;     // ... and rebuild Gram + Cholesky first
  int emit;          // K1 must write the sqrt(d)-scaled bf16 copy (a Hessian rebuild may follow)
  int hess_valid;    // a Cholesky factor exists (possibly stale -> chord Newton)
  int fail;          // 1 = not SPD, 2 = line search gave up, 3 = max_newton hit
  int newton_steps;  // accepted steps in this x-update
  int evals;         // K1 passes in this x-update
  int rejects;       // rejected trial points in this x-update
  int hess_builds;   // Gram+Cholesky rebuilds in this x-update
  int stall;         // consecutive poor contractions
  int bfgs_count;    // secant pairs stored so far (ring of BFGS_M), reset when the Hessian is rebuilt
  double h0_scale;   // self-scaling factor applied to the explicit inverse inside the L-BFGS two-loop (wide systems only; 1 after a rebuild)
  int k1_chunks;     // number of per-CTA partials the last K1 pass wrote for this problem (gpart / fpart rows)
  int refresh_next;  // rebuild the Hessian at the first point of the NEXT x-update (chord steps contracted slowly)
  int skip_eval;     // 1: the gradient at the start point of this x-update is already in g_t (data term) -- see admm_consensus_kernel:
                     //    slot 0 runs no K1 pass for this problem, the decide kernel accepts the start point on that gradient
  int warm_used;     // this x-update started from the estimated gradient (skip_eval was consumed): its first exact evaluation is accepted
                     // unconditionally (the estimate is not good enough to police a line search; the secant pair of that step is
                     // kept whenever s.y > 0: it carries most of the curvature information of the update)
  int build_step;    // newton_steps at the last rebuild of this x-update (0 if none yet): steps taken on the current factor = newton_steps - build_step
  double worst_ratio;// largest |g_new|/|g_old| seen over the chord steps of this x-update
  double alpha;      // current step length along dir
  double phi0;       // g_acc . dir  (< 0)
  double f_acc, f_t; // objective at accepted / trial point
  double gnorm;      // |g_acc|_inf
  double gnorm_prev;
  double dirnorm;    // |dir|_inf
  double dirnorm_prev;
  double xtol;
  int max_newton;
  int hess_policy;   // 0 adaptive chord, 1 every step
  int rebuild_is_expensive;  // a Gram+Cholesky rebuild costs more than ~8 passes over X: never rebuild mid-update, lean on L-BFGS
                             // and adapt h0_scale from the secant pairs
  // cumulative counters (never reset by begin-of-iteration)
  long long tot_evals, tot_newton, tot_rejects, tot_hess;
  // factored inverse the direction kernels read: this problem's own Ysym after its own factorisation, the group leader's after a
  // shared cold-start factorisation (the lambdas of a partition then stream ONE copy of Y for all their directions)
  const void* ysym_use;
  // matrix-free batches (hess_policy 2): preconditioned CG for the Newton direction (newton.cu cg_*_kernel)
  int cg_active;     // this problem's CG runs: the Hv / diagonal K1 modes and the CG kernels work on it
  int cg_iter;       // CG steps taken for the current direction
  double cg_rz;      // r.z of the current CG step
  double cg_g2;      // |g|_2^2 at the accepted point (forcing rule |r| <= eta |g|)
  float hv_vinf;     // max |hv_vf[k]|, written with hv_vf: the fixed-point scale of the next Hv pass
};

// K1 modes: the gradient pass, and the two passes of the matrix-free solver over the same rows (fixed d = w p (1-p) of the last
// gradient pass, read back from sdvec as sqrt(d)^2):  Hv:  column sums of t_i x_i with t_i = d_i (x_i . v) (v = hv_vf, fp32);
// diagonal:  column sums of d_i x_ic^2 (the Jacobi preconditioner).
enum { K1_GRAD = 0, K1_HV = 1, K1_DIAG = 2 };
// CSR Gram kernels (k2_gram.cu): e4m3 wgmma on operand blocks assembled in shared memory, or the exact sparse kernel that forms
// only the nonzero products of each row.  batch_alloc picks one per batch from the data.
enum { CSR_GRAM_WGMMA = 1, CSR_GRAM_SPARSE = 2 };

// One problem's device pointers.  Vectors have length ldv (= ldx, multiple of 4, >= Dt) and are
// zero in [Dt, ldv).  The bias column is PHYSICAL: column Dt-1 of X is 1.0f for every row when the
// problem has an intercept (llf/LibLinearDataset.java:592-614), so no kernel special-cases it.
struct Problem {
  // data (shared by the L problems of one partition)
  const float* X;          // dense [n][ldx] fp32, or nullptr for CSR
  long long n;             // rows
  int ldx;                 // leading dim in floats (multiple of 4)
  int Dt;                  // columns incl. bias
  const signed char* y;    // +1 / -1
  const float* w;          // weight
  const float* o;          // offset
  const long long* rowptr; // CSR (bias NOT stored; handled by the kernels)
  const int* colidx;
  const float* vals;
  long long nnz_hint;      // CSR nnz (host-side accounting only)
  int csr_unique;          // every CSR row has strictly increasing column ids (parallel bf16 emit is exact)
  const long long* bm_offs;       // block-major entry list for the CSR Gram: run offsets [nblk128][bm_groups] (+1 total)
  const unsigned short* bm_keys;  // per entry: byte offset inside the swizzled [128 cols][32 rows] operand block
  const float* bm_vals;           // per entry: the stored value (1 for the bias column, which the list holds explicitly)
  long long bm_groups;            // number of 32-row groups
  long long bm_entries;           // entries of the list: nnz + n (one bias entry per row)
  unsigned char* bm_e4m3;         // [bm_entries] this problem's Gram operand, e4m3(value * sqrt(d_row) * gram_scale), written by
                                  // gram_csr_operand_kernel before every CSR Gram build (per problem: the list is shared, sdvec is not)
  uint32_t* bm_word;              // [bm_entries] the same operand values for the sparse CSR Gram in ROW order (row r at
                                  // [rowptr[r] + r, rowptr[r + 1] + r], its intercept entry last), pre-decoded (k2_gram.cu
                                  // gram_word); a batch has one of the two forms (bm_e4m3 for CSR_GRAM_WGMMA, bm_word for CSR_GRAM_SPARSE)
  const uint32_t* gc_offs;        // [Dt + 1] column index of the sparse CSR Gram: column c's entries are at the positions
  const uint32_t* gc_pos;         // gc_pos[gc_offs[c] .. gc_offs[c + 1]) of bm_word, ascending (NULL where that kernel cannot run)
  float vmax, wmax;               // max |stored value| and max record weight of the partition (fixed-point scale of the CSR K1)
  int nblk128;             // number of 128-column blocks (Dp / 128)
  // fused multi-lambda CSR K1 (k1_csr_fused.cu): the partition's rows cut into sg_S segments of sg_rows rows; per segment the
  // stored values regrouped by column: 32 columns (lanes) per group, groups of columns of similar length, entries [k][lane]
  int sg_S, sg_rows, sg_ngrp;
  const int* sg_perm;               // [sg_S][sg_ngrp*32] column id of each lane slot, -1 = unused slot
  const int* sg_depth;              // [sg_S][sg_ngrp] entries per lane of the group
  const long long* sg_goff;         // [sg_S][sg_ngrp] first 32-lane row of the group in sg_row16 / sg_val
  const unsigned short* sg_row16;   // [..][32] row inside the segment
  const float* sg_val;              // [..][32] value (0 in padding slots)
  const unsigned short* sg_col16;   // [nnz] colidx as 16-bit ids (the fused kernel's phase A reads these: 6 instead of 8 B per value)
  float* gpart_f;                   // [sg_S][ldx] per-segment partial gradients when the fused K1 runs (else NULL; gpart is used)
  float* sdvec;            // [n] sqrt(d_i) written by K1 when the Gram is assembled straight from CSR (no Xt)
  float* rvec;             // [n] row residuals r_i, only for CSR partitions wider than one K1 column window (else NULL)
  int gram_from_csr;       // 1: the Gram is built from the block-major entry list (no dense bf16 operand)
  int csr_gram;            // which kernel builds it then: CSR_GRAM_WGMMA or CSR_GRAM_SPARSE (0 otherwise)
  double gram_pairs;       // products of one sparse build, sum over rows of (k_i + 1)(k_i + 2) / 2 (host-side accounting only)
  float gram_scale;        // CSR Gram operands are e4m3: sqrt(d) x is multiplied by this power of two before rounding ...
  float gram_unscale;      // ... and the Gram sums by 1 / gram_scale^2 in chol_prep (1 for the bf16 dense-operand path)
  __nv_bfloat16* Xt;       // [n][Dp] bf16 = sqrt(d_i) * x_ij  (Gram operand), zero in [ldx, Dp)
  int Dp;                  // multiple of 128
  // solver state
  double* beta;            // accepted iterate
  double* beta_t;          // trial iterate
  float* beta_tf;          // float copy of the trial iterate (what K1 reads)
  double* m;               // prior mean  (z - u)
  double* q;               // prior precision 1/priorVar (rho for ADMM)
  double* g_t;             // gradient at trial
  double* g_acc;           // gradient at accepted
  double* dir;             // Newton direction
  double* gpart;           // [k1_ctas][ldx] per-CTA partial X^T r
  double* fpart;           // [k1_ctas] per-CTA partial loss
  int k1_ctas;
  float* Hpart;            // [gram_slices][Dp][Dp] split-K partial Gram (lower tiles)
  int gram_slices;
  double* Lc;              // [ldh][ldh] Cholesky factor (lower), ldh multiple of 32
  double* Ldiag;           // [ldh][32] factorised diagonal blocks (side buffer, see k3_cholesky.cu)
  double* Ldinv;           // [ldh][32] inverses of the diagonal blocks (lower triangular)
  double* Yinv;            // [ldh][ldh] L^-1 (lower)
  double* Hinv;            // [ldh][ldh] (L L^T)^-1, full symmetric: a Newton direction is one GEMV
  __nv_bfloat16* Ysym;    // wide systems (ldh > 2048; NULL otherwise): operand of the direction product.  It holds Y = L^-1 as bf16 in
                          // symmetric storage M[i][j] = Y[max(i,j)][min(i,j)] (k3_cholesky.cu ysym_kernel): H^-1 q ~ Y^T (Y q) is two
                          // row-wise triangular GEMVs over it, HBM-bound on D'^2 2-byte entries in total.  The product form is
                          // symmetric positive definite for ANY rounding of Y, so the low precision can never turn the preconditioner
                          // indefinite (a rounded explicit H^-1 could)
  float* qf;              // [ldx] fp32 copy of the two-loop vector q (written by the decide kernel when Ysym is in use)
  float* tf;              // [ldx] t = Y q in fp32 (between the two phases)
  int ldh;
  Ctrl* ctrl;
  // ADMM per-problem vectors (float, as the reference's avro files hold them)
  float* u_f;              // u used by this iteration
  float* uplusx_f;         // float(u + x)
  float* x_f;              // float(x)
  double* bfgs_S;          // [BFGS_M][ldx] steps  s_k = beta_{k+1} - beta_k
  double* bfgs_Y;          // [BFGS_M][ldx] gradient differences y_k
  double* bfgs_rho;        // [BFGS_M] 1/(s.y)
  double* bfgs_alpha;      // [BFGS_M] two-loop scratch
  double* x_d;             // x of the last x-update (the ADMM consensus overwrites beta with the next init)
  int lambda_idx;
  int self_idx;            // index of this problem in its batch (tensor-map slot), valid also in compacted copies
  int part_local;
  // Hessian-vector products (K1 modes K1_HV / K1_DIAG) and the matrix-free Newton-CG direction
  float rowl1;             // max over rows of sum_j |x_ij| (stored values): bounds |x_i . v| for the fixed-point CSR scatter
  float* hv_vf;            // [ldx] fp32 vector the Hv pass multiplies (aliases qf: the factored-inverse GEMV is not used then)
  double* cg_r;            // [ldx] CG residual (matrix-free batches only, else NULL)
  double* cg_p;            // [ldx] CG search direction
  double* cg_z;            // [ldx] preconditioned residual
  double* cg_Hp;           // [ldx] H p
  double* cg_diag;         // [ldx] Jacobi preconditioner diag(H)
};

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// The same on a 32-bit shared-space address (see sts_u8): loops that hold barrier addresses in registers need no conversion.
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}

// Byte store to a 32-bit shared-space address.  A pointer derived from the dynamic shared array by integer alignment loses its
// address space: the compiler then emits GENERIC stores and rebuilds the 64-bit window base (S2UR CgaCtaId / SWINHI, ~10
// instructions) at every store -- the Gram producers' scatter stores spent more instructions on that than on the data.
__device__ __forceinline__ void sts_u8(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(saddr), "r"(v) : "memory"); }
// 1-D bulk copy global -> shared (TMA engine, no tensor map): SASS UBLKCP.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// 2-D tensor-map TMA load: SASS UTMALDG.
__device__ __forceinline__ void tma_load_2d(void* dst_smem, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst_smem)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// wgmma (warpgroup MMA, sm_90a).  Shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor layout):
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset (0: atoms 1024-B aligned) | [62,64) layout
//   (0 = no swizzle, 1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B)
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)(layout & 3) << 62;
  return d;
}
// orders register accesses to the accumulators before the wgmma that follows (needed before the first one of a warpgroup)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// d[64 x 256] += A[64 x 16] * B[16 x 256], bf16 in, fp32 accumulate; both operands MN-major (transposed) in shared memory.
__device__ __forceinline__ void wgmma_bf16_m64n256k16_tt(float (&d)[128], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}
// d[64 x 128] (+)= A[64 x 32] * B[32 x 128], e4m3 in; both operands K-major in shared memory (the only layout wgmma takes for
// 8-bit types).  accumulate = 0 overwrites d.  The tensor core keeps an fp8 product's running sum at less than fp32 precision,
// so callers add short chains of these into fp32 registers themselves.
__device__ __forceinline__ void wgmma_e4m3_m64n128k32(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// Hands registers between the warpgroups of a CTA (every thread of a warpgroup executes it with the same count).
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// warp / block reductions
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace mlease

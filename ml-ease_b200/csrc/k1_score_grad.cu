// k1_score_grad.cu -- K1: fused score + sigmoid/IRLS reweight + gradient (+ objective, + the
// sqrt(d)-scaled bf16 operand of the Gram kernel) in ONE pass over X.
//
// Replaces LogisticRegressionL2.fun + grad (llf/LogisticRegressionL2.java:156-225), i.e. the
// two sparse passes Xv (:115-129) and XTv (:131-150), and the score recomputation inside
// hessian() (:261-269).  HBM-bound: algorithmic bytes per row = 4*ldx (X once) + 9 (y,w,o).
//
// Dense layout: X row-major [n][ldx] fp32, ldx % 4 == 0, bias column physical.  A CTA streams
// row tiles of R rows (R*ldx*4 contiguous bytes) through an S-stage shared-memory ring with
// 1-D bulk TMA copies (cp.async.bulk, mbarrier complete_tx), then
//   phase A: s_i = x_i.beta + o_i, p = sigmoid(y s), r_i = w (p-1) y, d_i = w p (1-p), loss_i      (row dots)
//   phase B: g += r_i * x_i over the tile's rows, and (optionally) Xt[i][:] = bf16(sqrt(d_i) * x_i[:])
// so every element of X is read from HBM exactly once and from shared memory exactly once (into registers).
// Per-CTA partial gradients are accumulated in fp64 registers and written to gpart; a fixed
// order reduction (k1_reduce_decide in newton.cu) makes the result run-to-run deterministic.
#include <algorithm>

#include "kernels.cuh"

namespace mlease {

constexpr int K1_THREADS = 256;
constexpr int K1_WARPS = K1_THREADS / 32;


// tile -> registers + partial dots (FULL: every row of the tile exists, no guards)
template <int G, int RT, bool FULL>
__device__ __forceinline__ void k1_phase_a(float4 (&x)[G][RT], float (&p)[RT], const float4* __restrict__ tile4, const float4 (&b4)[G],
                                           int ncg, int cg0, int myrows0, int rows) {
#pragma unroll
  for (int j = 0; j < RT; j++) {
    const bool ok = FULL || (myrows0 + j < rows);
    float pj = 0.f;
#pragma unroll
    for (int g = 0; g < G; g++) {
      const bool okc = ok && (G == 1 || cg0 + g * K1_THREADS < ncg);
      x[g][j] = okc ? tile4[(uint32_t)(j * ncg + g * K1_THREADS)] : make_float4(0.f, 0.f, 0.f, 0.f);
      pj = fmaf(x[g][j].x, b4[g].x, pj); pj = fmaf(x[g][j].y, b4[g].y, pj);
      pj = fmaf(x[g][j].z, b4[g].z, pj); pj = fmaf(x[g][j].w, b4[g].w, pj);
    }
    p[j] = pj;
  }
}

// Warp-level transposed reduction of RT per-lane values: after log2(RT) halving exchanges every lane holds ONE value,
// the sum over its 32/RT-lane-strided group, for row r = lane / (32/RT); the remaining butterfly sums the group.
// Returns the warp total of row (lane / (32/RT)) in every lane of that group.  ~RT + log2(32) shuffles instead of 5*RT.
template <int RT>
__device__ __forceinline__ float k1_warp_rows_reduce(float (&p)[RT], int lane) {
  int c = RT;
#pragma unroll
  for (int m = 16; m >= 32 / RT; m >>= 1) {   // halving steps: xor 16, 8, ... while more than one value is held
    c >>= 1;
    const bool up = (lane & m) != 0;
#pragma unroll
    for (int i = 0; i < RT / 2; i++) {
      if (i < c) {
        const float send = up ? p[i] : p[i + c];
        const float keep = up ? p[i + c] : p[i];
        p[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
      }
    }
  }
  float v = p[0];
#pragma unroll
  for (int m = 16 / RT; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}

// CTA -> (problem, chunk of the problem's rows).  Static: blockIdx.y is the problem, blockIdx.x the chunk.  Dynamic
// (nprob_dyn = number of problems, <= 32, one-dimensional grid): the CTAs are dealt round-robin to the problems that are
// still running, so a slot in which only some problems need a pass still uses every SM.  The chunk count a problem got is
// published in Ctrl::k1_chunks for the reduction kernels; partial sums are combined in chunk order (deterministic).
// In the Hv / diagonal modes the running problems are those whose CG runs (Ctrl::cg_active), so that the whole grid serves them.
struct K1Map { int prob, chunk, nchunks; };
template <int MODE = K1_GRAD>
__device__ __forceinline__ K1Map k1_map(const Problem* __restrict__ probs, int nprob_dyn) {
  K1Map m;
  if (nprob_dyn == 0) { m.prob = blockIdx.y; m.chunk = blockIdx.x; m.nchunks = gridDim.x; return m; }
  __shared__ int s_act[34];
  if (threadIdx.x < 32) {
    const bool a = (int)threadIdx.x < nprob_dyn && (MODE != K1_GRAD ? probs[threadIdx.x].ctrl->cg_active != 0 : probs[threadIdx.x].ctrl->done == 0);
    const unsigned mask = __ballot_sync(0xffffffffu, a);
    if (a) s_act[2 + __popc(mask & ((1u << threadIdx.x) - 1u))] = threadIdx.x;
    if (threadIdx.x == 0) s_act[0] = __popc(mask);
  }
  __syncthreads();
  const int na = s_act[0];
  if (na == 0) { m.prob = -1; m.chunk = 0; m.nchunks = 1; return m; }
  const int idx = (int)blockIdx.x % na;
  m.prob = s_act[2 + idx];
  m.chunk = (int)blockIdx.x / na;
  m.nchunks = ((int)gridDim.x - idx + na - 1) / na;
  return m;
}

// Thread t owns float4 column group(s) cg = t (+256 g) and RT rows of every tile (rows sl*RT .. sl*RT+RT-1 when
// several row slices share the 256 threads for narrow matrices).  The tile is read from shared memory ONCE, into
// registers, and serves both the row dots (phase A) and the column sums / bf16 emit (phase B):
//   A  : x[j] <- tile, p[j] = x[j].beta (beta float4 lives in registers for the whole kernel), p -> smem pd[row][t]
//   -- barrier 1 (all of the stage is in registers: the producer thread refills it immediately) --
//   A' : warp w sums pd rows w, w+8, ..; lanes 0..k do the sigmoid / loss / IRLS weight of those rows in parallel
//   -- barrier 2 --
//   B  : g += r[row] * x[j];  optionally Xt[row] = bf16(sqrt(d[row]) * x[j])
// pd / r / sqrt(d) are double buffered by tile parity, so two barriers per tile are enough.
template <int G, int RT>
__global__ void __launch_bounds__(K1_THREADS, (G == 1 ? 2 : 1))
k1_dense_kernel(const Problem* __restrict__ probs, int S, int nsl, int force_emit, int nprob_dyn) {
  const K1Map km = k1_map(probs, nprob_dyn);
  if (km.prob < 0) return;
  const Problem& pb = probs[km.prob];
  Ctrl* ctrl = pb.ctrl;
  if (ctrl->done) return;
  if (km.chunk == 0 && threadIdx.x == 0) ctrl->k1_chunks = km.nchunks;
  const bool emit = force_emit >= 0 ? (force_emit != 0) : (ctrl->emit != 0);

  const int ldx = pb.ldx;
  const int ncg = ldx >> 2;  // float4 column groups
  const long long n = pb.n;
  const int Rt = RT * nsl;   // rows per tile
  const int pdw = (G == 1) ? ncg : K1_THREADS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* __restrict__ Xg = pb.X;
  const signed char* __restrict__ yg = pb.y;
  const float* __restrict__ wg = pb.w;
  const float* __restrict__ og = pb.o;
  __nv_bfloat16* __restrict__ Xt = pb.Xt;
  const int Dp = pb.Dp;

  extern __shared__ __align__(128) unsigned char smem_raw[];
  const size_t stage_bytes = (size_t)Rt * ldx * sizeof(float);
  float* pd_s = reinterpret_cast<float*>(smem_raw + (size_t)S * stage_bytes);   // [2][Rt][pdw]
  float* r_s = pd_s + 2 * (size_t)Rt * pdw;                                     // [2][Rt]
  float* sd_s = r_s + 2 * Rt;                                                   // [2][Rt]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(sd_s + 3 * Rt) + 15) & ~uintptr_t(15));
  double* red_s = reinterpret_cast<double*>(full_bar + 8);

  const int ntiles = (int)((n + Rt - 1) / Rt);
  const int my_tiles = ntiles > km.chunk ? (ntiles - km.chunk + km.nchunks - 1) / km.nchunks : 0;

  if (tid == 0) {
    for (int s = 0; s < S; s++) mbar_init(&full_bar[s], 1);
    fence_mbar_init();
  }
  __syncthreads();

  // producer (thread 0): bulk-copy tile number `t` of the matrix into stage `stg`
  auto issue = [&](int t, int stg) {
    const long long row0 = (long long)t * Rt;
    const int rows = (int)min((long long)Rt, n - row0);
    const uint32_t bytes = (uint32_t)rows * (uint32_t)ldx * 4u;
    uint64_t* bar = &full_bar[stg];
    mbar_arrive_expect_tx(bar, bytes);
    bulk_g2s(smem_raw + (size_t)stg * stage_bytes, Xg + row0 * ldx, bytes, bar);
  };
  if (tid == 0) {
    for (int k = 0; k < S && k < my_tiles; k++) issue(km.chunk + k * km.nchunks, k);
  }

  // column / row-slice ownership
  int sl = 0, cg0 = tid;
  if (G == 1) { sl = tid / ncg; cg0 = tid - sl * ncg; }
  const bool act = (G == 1) ? (sl < nsl) : true;
  float4 b4[G];
#pragma unroll
  for (int g = 0; g < G; g++) {
    const int cg = cg0 + g * K1_THREADS;
    b4[g] = (act && cg < ncg) ? reinterpret_cast<const float4*>(pb.beta_tf)[cg] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  double acc64[G][4];
#pragma unroll
  for (int g = 0; g < G; g++) acc64[g][0] = acc64[g][1] = acc64[g][2] = acc64[g][3] = 0.0;
  double loss64 = 0.0;
  float* s_s = sd_s + 2 * Rt;                       // [Rt] row scores (x_i . beta)
  const uint32_t xoff = (uint32_t)(sl * RT * ncg + cg0);   // float4 index of this thread's first element in a tile
  const uint32_t poff = (uint32_t)(sl * RT * pdw + ((G == 1) ? cg0 : tid));
  const int myrows0 = sl * RT;

  int st = 0;
  uint32_t par = 0;
  int tile_no = km.chunk;
  const int tile_step = km.nchunks;
  for (int k = 0; k < my_tiles; k++, tile_no += tile_step) {
    const int buf = k & 1;
    const long long row0 = (long long)tile_no * Rt;
    const int rows = (int)min((long long)Rt, n - row0);
    const bool full = rows == Rt;
    // per-row scalars (thread t < rows owns row t): issued before the wait so their latency is hidden
    float yy = 0.f, ww = 0.f, oo = 0.f;
    const bool has = tid < rows;
    if (has) { const long long i = row0 + tid; yy = (float)yg[i]; ww = wg[i]; oo = og[i]; }

    mbar_wait(&full_bar[st], par);
    const float4* tile4 = reinterpret_cast<const float4*>(smem_raw + (size_t)st * stage_bytes) + xoff;
    float* pd = pd_s + (size_t)buf * Rt * pdw;

    // ---- phase A: tile -> registers, partial dots ---------------------------------------------------------
    float4 x[G][RT];
    float p[RT];
    if (act) {
      if (full) k1_phase_a<G, RT, true>(x, p, tile4, b4, ncg, cg0, myrows0, rows);
      else k1_phase_a<G, RT, false>(x, p, tile4, b4, ncg, cg0, myrows0, rows);
    } else {
#pragma unroll
      for (int j = 0; j < RT; j++) p[j] = 0.f;
    }
    float score = 0.f;
    if (nsl == 1) {
      // all 256 threads share the tile's RT rows: reduce in registers with shuffles, 1 smem word per (warp,row)
      const float v = k1_warp_rows_reduce<RT>(p, lane);
      if ((lane & (32 / RT - 1)) == 0) pd[warp * RT + lane / (32 / RT)] = v;
      __syncthreads();   // barrier 1: the stage is fully in registers
      if (tid == 0 && k + S < my_tiles) issue(tile_no + S * tile_step, st);
      if (has) {
#pragma unroll
        for (int w = 0; w < K1_WARPS; w++) score += pd[w * RT + tid];
      }
    } else {
      if (act) {
        float* pw = pd + poff;
#pragma unroll
        for (int j = 0; j < RT; j++) pw[(uint32_t)(j * pdw)] = p[j];   // rows beyond `rows` get 0: harmless
      }
      __syncthreads();   // barrier 1: the stage is fully in registers
      if (tid == 0 && k + S < my_tiles) issue(tile_no + S * tile_step, st);
      // row sums (warp w: rows w, w+8, ...) -> s_s
      for (int row = warp; row < rows; row += K1_WARPS) {
        const float* pr = pd + (uint32_t)(row * pdw);
        float a = 0.f;
        for (int c = lane; c < pdw; c += 32) a += pr[c];
        a = warp_sum(a);
        if (lane == 0) s_s[row] = a;
      }
      __syncthreads();   // barrier 1b
      if (has) score = s_s[tid];
    }
    if (++st == S) { st = 0; par ^= 1u; }
    // ---- per-row scalar math, one thread per row (only the first warps of the CTA take this branch) -------
    if (has) {
      const float t = yy * (score + oo);
      const float e = __expf(-fabsf(t));                 // in (0,1]
      const float inv = __frcp_rn(1.f + e);
      const float pp = t >= 0.f ? inv : e * inv;         // sigmoid(y s)
      const float qq = t >= 0.f ? e * inv : inv;         // 1 - p, no cancellation
      // log1p(e) = -log(1/(1+e)); absolute error ~1e-7 per row, the objective only steers the line search
      loss64 += (double)(ww * ((t >= 0.f ? 0.f : -t) - __logf(inv)));
      r_s[buf * Rt + tid] = -ww * yy * qq;               // w (p-1) y
      sd_s[buf * Rt + tid] = sqrtf(ww * pp * qq);        // sqrt(d_i)
    }
    __syncthreads();   // barrier 2

    // ---- phase B: column sums from registers (+ bf16 emit) ------------------------------------------------
    if (act) {
      float rr[RT];
      {
        const float4* rb4 = reinterpret_cast<const float4*>(r_s + buf * Rt + myrows0);
#pragma unroll
        for (int j4 = 0; j4 < RT / 4; j4++) {
          const float4 v = rb4[j4];
          rr[4 * j4] = v.x; rr[4 * j4 + 1] = v.y; rr[4 * j4 + 2] = v.z; rr[4 * j4 + 3] = v.w;
        }
      }
      if (!full) {
#pragma unroll
        for (int j = 0; j < RT; j++) if (myrows0 + j >= rows) rr[j] = 0.f;   // x is 0 there too; avoid 0*NaN from stale smem
      }
#pragma unroll
      for (int g = 0; g < G; g++) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < RT; j++) {
          a.x = fmaf(x[g][j].x, rr[j], a.x); a.y = fmaf(x[g][j].y, rr[j], a.y);
          a.z = fmaf(x[g][j].z, rr[j], a.z); a.w = fmaf(x[g][j].w, rr[j], a.w);
        }
        acc64[g][0] += (double)a.x; acc64[g][1] += (double)a.y; acc64[g][2] += (double)a.z; acc64[g][3] += (double)a.w;
      }
      if (emit) {
        const float* sb = sd_s + buf * Rt + myrows0;
#pragma unroll
        for (int g = 0; g < G; g++) {
          const int cg = cg0 + g * K1_THREADS;
          if (G == 1 || cg < ncg) {
            __nv_bfloat16* xt = Xt + (size_t)(row0 + myrows0) * Dp + 4 * cg;
#pragma unroll
            for (int j = 0; j < RT; j++) {
              if (full || myrows0 + j < rows) {
                const float sd = sb[j];
                __nv_bfloat162 lo = __floats2bfloat162_rn(x[g][j].x * sd, x[g][j].y * sd);
                __nv_bfloat162 hi = __floats2bfloat162_rn(x[g][j].z * sd, x[g][j].w * sd);
                uint2 pk;
                pk.x = *reinterpret_cast<uint32_t*>(&lo);
                pk.y = *reinterpret_cast<uint32_t*>(&hi);
                *reinterpret_cast<uint2*>(xt + (size_t)j * Dp) = pk;
              }
            }
          }
        }
      }
    }
  }

  // ---- CTA epilogue: reduce row slices, write partials ---------------------------------------------------
  __syncthreads();
  double* gp = pb.gpart + (size_t)km.chunk * ldx;
  if (G == 1 && nsl > 1) {
    double* sc = reinterpret_cast<double*>(smem_raw);  // every bulk copy has completed and been consumed
    if (act) {
      double* d = sc + ((size_t)sl * ncg + cg0) * 4;
      d[0] = acc64[0][0]; d[1] = acc64[0][1]; d[2] = acc64[0][2]; d[3] = acc64[0][3];
    }
    __syncthreads();
    for (int c = tid; c < ldx; c += K1_THREADS) {
      double sacc = 0.0;
      for (int q = 0; q < nsl; q++) sacc += sc[(size_t)q * ldx + c];
      gp[c] = sacc;
    }
  } else {
#pragma unroll
    for (int g = 0; g < G; g++) {
      const int cg = cg0 + g * K1_THREADS;
      if (act && cg < ncg) {
        gp[4 * cg + 0] = acc64[g][0]; gp[4 * cg + 1] = acc64[g][1];
        gp[4 * cg + 2] = acc64[g][2]; gp[4 * cg + 3] = acc64[g][3];
      }
    }
  }
  loss64 = warp_sum(loss64);
  if (lane == 0) red_s[warp] = loss64;
  __syncthreads();
  if (tid == 0) {
    double sacc = 0.0;
    for (int wq = 0; wq < K1_WARPS; wq++) sacc += red_s[wq];
    pb.fpart[km.chunk] = sacc;
  }
}

// ------------------------------------------------------------------------------------------
// CSR variant (configs 3/4: ~1 % dense rows).  One warp per row, rows dealt to CTAs in contiguous chunks:
//   gather : s_i = sum_j v_ij * beta[c_ij] (+ beta[bias]), beta staged in shared memory
//   scatter: g[c_ij] += r_i * v_ij into a per-CTA shared-memory gradient (float atomics, spread addresses), flushed once per
//            CTA as an fp64 partial row of gpart -> the same fixed-order cross-CTA reduction as the dense path
//   emit   : Xt[i][c_ij] = bf16(sqrt(d_i) v_ij): the dense bf16 Gram operand is assembled from the sparse row (positions
//            outside the row's pattern stay 0 from the one-time memset; rows with repeated columns take a serial path
//            because duplicates add in the reference's Xv)
// HBM-bound on 8 B per stored value (+ 17 B per row).
// ------------------------------------------------------------------------------------------
// 1024 threads per CTA: the row loop is a chain of dependent global loads (rowptr -> colidx/vals -> gather), so the kernel
// lives on occupancy (up to 64 warps per SM with two CTAs).
// CSR K1 for partitions whose rows hold each column at most once (the normal case; checked at upload).
// Same pass as k1_csr_kernel below, but the per-CTA gradient is accumulated in shared memory as two-word fixed point
// with native 32-bit integer atomics (ATOMS.ADD) instead of float atomics, which compile to compare-and-swap loops.
// Integer addition commutes, so the result does not depend on the order in which warps retire: the pass is
// deterministic, like the dense one.  With B >= sum over the CTA's rows of |contribution| to any one column
// (rows x max weight x max |value|), S = 2^(29 - ceil(log2 B)) and k = 30 - ceil(log2 rows):
//   hi = rint(c S), lo = rint((c S - hi) 2^k), gradient = (sum hi + sum lo / 2^k) / S,
// i.e. a resolution of B 2^-(29+k) per contribution (k = 16 at 16k rows per CTA), below fp32 rounding of the
// contribution itself.  The first 128 entries of a row stay in registers between the margin and the gradient half.
constexpr int K1_FX_THREADS = 768;   // 24 warps: 80 registers per thread, which holds 7 chunks of two rows per warp without spilling
// BSM: beta staged in shared memory (LDS gathers) / read through L1 from global memory.
// WIN: the accumulators do not fit shared memory for all ldx columns (more than ~28k features): this launch accumulates the
// columns [0, col_w) only and stores the row residuals r_i in rvec; k1_csr_fx_window_kernel adds the other column windows.
// MODE K1_HV / K1_DIAG (common.cuh): the row weight is t_i = d_i (x_i . v + v_bias) / d_i instead of the residual, with the
// fixed-point bound of k1_fx_mode_bound; problems take part when Ctrl::cg_active is set.
// Fixed-point bound of the Hv / diagonal modes: |t_i| <= (w_i / 4) (rowl1 + 1) |v|_inf resp. w_i / 4, times max(|x|max, 1) per
// contribution (max(|x|max^2, 1) for the diagonal).  |v|_inf is Ctrl::hv_vinf, written with hv_vf.
template <int MODE>
__device__ __forceinline__ float k1_fx_mode_bound(const Problem& pb, long long per) {
  if constexpr (MODE == K1_HV) return (float)per * 0.25f * pb.wmax * (pb.rowl1 + 1.f) * pb.ctrl->hv_vinf * fmaxf(pb.vmax, 1.f);
  return (float)per * 0.25f * pb.wmax * fmaxf(pb.vmax * pb.vmax, 1.f);
}

template <bool BSM, bool WIN, int MODE = K1_GRAD>
__global__ void __launch_bounds__(K1_FX_THREADS, 1) k1_csr_fx_kernel(const Problem* __restrict__ probs, int has_bias, int force_emit, int nprob_dyn, int col_w) {
  const K1Map km = k1_map<MODE>(probs, nprob_dyn);
  if (km.prob < 0) return;
  const Problem& pb = probs[km.prob];
  Ctrl* ctrl = pb.ctrl;
  if (MODE != K1_GRAD ? !ctrl->cg_active : ctrl->done) return;
  if (km.chunk == 0 && threadIdx.x == 0) ctrl->k1_chunks = km.nchunks;
  const bool emit = force_emit >= 0 ? (force_emit != 0) : (ctrl->emit != 0);
  extern __shared__ __align__(16) float csr_sm[];
  const int ldx = pb.ldx, Dt = pb.Dt;
  // layout: g_hi[W + 32] | g_lo[W + 32] | beta[ldx] (W = ldx unless WIN); the 32 extra words are per-lane dummy slots for
  // lanes past the end of a row or outside the column window (they add 0 there): no divergent branches in the gradient half
  const int W = WIN ? col_w : ldx;
  const int gs = W + 32;
  int* g_hi = reinterpret_cast<int*>(csr_sm);
  int* g_lo = g_hi + gs;
  float* b_s = csr_sm + 2 * (size_t)gs;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int k = tid; k < gs; k += blockDim.x) { g_hi[k] = 0; g_lo[k] = 0; }
  const float* __restrict__ bg = MODE == K1_GRAD ? pb.beta_tf : pb.hv_vf;
  if (BSM)
    for (int k = tid; k < ldx; k += blockDim.x) b_s[k] = bg[k];
  __syncthreads();
  const long long n = pb.n;
  const long long per = (n + km.nchunks - 1) / km.nchunks;
  const long long rb = (long long)km.chunk * per, re = min(n, rb + per);
  // fixed-point scales (powers of two: scaling is exact)
  float bound = MODE != K1_GRAD ? k1_fx_mode_bound<MODE>(pb, per) : (float)per * pb.wmax * fmaxf(pb.vmax, has_bias ? 1.f : 0.f);
  if (!(bound > 0.f) || !(bound < 3.0e38f)) bound = 1.f;
  const int e_hi = 29 - (ilogbf(bound) + 1);
  int kbits = 30 - (64 - __clzll((unsigned long long)max(per, 1LL)));
  kbits = max(0, min(kbits, 24));
  const float s_hi = ldexpf(1.f, e_hi), s_k = ldexpf(1.f, kbits);
  const long long* __restrict__ rp = pb.rowptr;
  const signed char* __restrict__ yv = pb.y;
  const float* __restrict__ wv = pb.w;
  const float* __restrict__ ov = pb.o;
  // Two rows per warp: each half-warp (16 lanes) owns a row, so the per-row work (row header, reduction, sigmoid, loss)
  // is shared by two rows per instruction and a 100-entry row wastes 12 of 112 lane slots instead of 28 of 128.
  constexpr int HW = 16, NCH = 7;          // lanes per row, register-resident chunks per row (NCH*HW = 112 entries)
  const int sub = lane >> 4, sl = lane & 15;
  const int dummy = W + lane;
  const float bias_b = has_bias ? (BSM ? b_s[Dt - 1] : __ldg(bg + Dt - 1)) : 0.f;
  double loss = 0.0;
  const long long rstep = 2LL * nw;
  long long i = rb + 2 * warp + sub;       // this half-warp's row; the loop runs while either half has one
  long long j0 = 0;
  int len = 0;
  if (i < re) { j0 = __ldg(rp + i); len = (int)(__ldg(rp + i + 1) - j0); }
  for (long long ib = rb + 2 * warp; ib < re; ib += rstep) {
    const bool has_row = i < re;
    const float* __restrict__ vr = pb.vals + j0;
    const int* __restrict__ cr = pb.colidx + j0;
    float v[NCH];
    int c[NCH];
#pragma unroll
    for (int q = 0; q < NCH; q++) {
      const bool ok = sl + HW * q < len;
      v[q] = ok ? __ldg(vr + sl + HW * q) : 0.f;
      c[q] = ok ? __ldg(cr + sl + HW * q) : dummy;
    }
    // this row's scalars and the next row's extent while the entries are in flight
    float yy = 0.f, ww = 0.f, oo = 0.f;
    if (has_row) { yy = (float)__ldg(yv + i); ww = __ldg(wv + i); oo = __ldg(ov + i); }
    const long long in = i + rstep;
    long long j0n = 0;
    int lenn = 0;
    if (in < re) { j0n = __ldg(rp + in); lenn = (int)(__ldg(rp + in + 1) - j0n); }
    float a = 0.f;
#pragma unroll
    for (int q = 0; q < NCH; q++) a = fmaf(v[q], BSM ? b_s[min(c[q], ldx - 1)] : __ldg(bg + min(c[q], ldx - 1)), a);   // v = 0 on dummy lanes
    for (int j = NCH * HW + sl; j < len; j += HW) a = fmaf(__ldg(vr + j), BSM ? b_s[__ldg(cr + j)] : __ldg(bg + __ldg(cr + j)), a);
#pragma unroll
    for (int m = HW / 2; m >= 1; m >>= 1) a += __shfl_xor_sync(0xffffffffu, a, m);   // stays inside the half-warp
    a += bias_b;
    float rs, rrow = 0.f, p = 0.f, qq = 0.f;
    if constexpr (MODE != K1_GRAD) {
      const float sd = has_row ? __ldg(pb.sdvec + i) : 0.f;
      rrow = MODE == K1_HV ? sd * sd * a : sd * sd;
      rs = rrow * s_hi;
    } else {
      const float t = yy * (a + oo);
      const float e = __expf(-fabsf(t));
      const float inv = __frcp_rn(1.f + e);
      p = t >= 0.f ? inv : e * inv;
      qq = t >= 0.f ? e * inv : inv;
      if (sl == 0 && has_row) loss += (double)(ww * ((t >= 0.f ? 0.f : -t) - __logf(inv)));
      rs = has_row ? -ww * yy * qq * s_hi : 0.f;     // contribution scale: c S = value * rs
    }
#pragma unroll
    for (int q = 0; q < NCH; q++) {
      const float ts = (MODE == K1_DIAG ? v[q] * v[q] : v[q]) * rs, h = rintf(ts);
      const int cc = (!WIN || c[q] < W) ? c[q] : dummy;
      atomicAdd(&g_hi[cc], (int)h);
      atomicAdd(&g_lo[cc], __float2int_rn((ts - h) * s_k));
    }
    for (int j = NCH * HW + sl; j < len; j += HW) {
      const float xj = __ldg(vr + j);
      const float ts = (MODE == K1_DIAG ? xj * xj : xj) * rs, h = rintf(ts);
      int cc = __ldg(cr + j);
      if (WIN && cc >= W) cc = dummy;
      atomicAdd(&g_hi[cc], (int)h);
      atomicAdd(&g_lo[cc], __float2int_rn((ts - h) * s_k));
    }
    if (has_bias && sl == 0 && has_row && (!WIN || Dt - 1 < W)) {
      const float h = rintf(rs);
      atomicAdd(&g_hi[Dt - 1], (int)h);
      atomicAdd(&g_lo[Dt - 1], __float2int_rn((rs - h) * s_k));
    }
    if (MODE == K1_GRAD && emit && sl == 0 && has_row) pb.sdvec[i] = sqrtf(ww * p * qq);   // the Gram kernel assembles the scaled rows itself
    if (WIN && sl == 0 && has_row) pb.rvec[i] = MODE == K1_GRAD ? -ww * yy * qq : rrow;   // row weight for the other column windows
    i = in; j0 = j0n; len = lenn;
  }
  loss += __shfl_down_sync(0xffffffffu, loss, 16);   // lane 0 += lane 16
  __syncthreads();
  double* gp = pb.gpart + (size_t)km.chunk * ldx;
  const double inv_hi = (double)ldexpf(1.f, -e_hi), inv_k = (double)ldexpf(1.f, -kbits);
  for (int k = tid; k < min(W, ldx); k += blockDim.x) gp[k] = ((double)g_hi[k] + (double)g_lo[k] * inv_k) * inv_hi;
  if (MODE != K1_GRAD) return;
  __shared__ double red[32];
  if (lane == 0) red[warp] = loss;
  __syncthreads();
  if (tid == 0) {
    double sacc = 0.0;
    for (int wq = 0; wq < nw; wq++) sacc += red[wq];
    pb.fpart[km.chunk] = sacc;
  }
}

// Columns [col_lo, col_lo + col_w) of the gradient for partitions too wide for one shared-memory window: same CTA -> rows
// mapping and the same fixed-point scales as k1_csr_fx_kernel<.., true>, which ran first in this slot and left r_i in rvec.
template <int MODE = K1_GRAD>
__global__ void __launch_bounds__(K1_FX_THREADS, 1) k1_csr_fx_window_kernel(const Problem* __restrict__ probs, int has_bias, int nprob_dyn,
                                                                            int col_lo, int col_w) {
  const K1Map km = k1_map<MODE>(probs, nprob_dyn);
  if (km.prob < 0) return;
  const Problem& pb = probs[km.prob];
  if (MODE != K1_GRAD ? !pb.ctrl->cg_active : pb.ctrl->done) return;
  extern __shared__ __align__(16) float csr_sm[];
  const int ldx = pb.ldx, Dt = pb.Dt;
  const int gs = col_w + 32;
  int* g_hi = reinterpret_cast<int*>(csr_sm);
  int* g_lo = g_hi + gs;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int k = tid; k < gs; k += blockDim.x) { g_hi[k] = 0; g_lo[k] = 0; }
  __syncthreads();
  const long long n = pb.n;
  const long long per = (n + km.nchunks - 1) / km.nchunks;
  const long long rb = (long long)km.chunk * per, re = min(n, rb + per);
  float bound = MODE != K1_GRAD ? k1_fx_mode_bound<MODE>(pb, per) : (float)per * pb.wmax * fmaxf(pb.vmax, has_bias ? 1.f : 0.f);
  if (!(bound > 0.f) || !(bound < 3.0e38f)) bound = 1.f;
  const int e_hi = 29 - (ilogbf(bound) + 1);
  int kbits = 30 - (64 - __clzll((unsigned long long)max(per, 1LL)));
  kbits = max(0, min(kbits, 24));
  const float s_hi = ldexpf(1.f, e_hi), s_k = ldexpf(1.f, kbits);
  const long long* __restrict__ rp = pb.rowptr;
  const int sub = lane >> 4, sl = lane & 15;
  const int dummy = col_w + lane;
  const int bias_idx = Dt - 1 - col_lo;
  for (long long i = rb + 2 * warp + sub; i < re; i += 2LL * nw) {
    const long long j0 = __ldg(rp + i);
    const int len = (int)(__ldg(rp + i + 1) - j0);
    const float rs = __ldg(pb.rvec + i) * s_hi;
    const float* __restrict__ vr = pb.vals + j0;
    const int* __restrict__ cr = pb.colidx + j0;
    for (int j = sl; j < len; j += 16) {
      const float xj = __ldg(vr + j);
      const float ts = (MODE == K1_DIAG ? xj * xj : xj) * rs, h = rintf(ts);
      const int idx = __ldg(cr + j) - col_lo;
      const int cc = (unsigned)idx < (unsigned)col_w ? idx : dummy;
      const bool in = (unsigned)idx < (unsigned)col_w;
      atomicAdd(&g_hi[cc], in ? (int)h : 0);
      atomicAdd(&g_lo[cc], in ? __float2int_rn((ts - h) * s_k) : 0);
    }
    if (has_bias && sl == 0 && (unsigned)bias_idx < (unsigned)col_w) {
      const float h = rintf(rs);
      atomicAdd(&g_hi[bias_idx], (int)h);
      atomicAdd(&g_lo[bias_idx], __float2int_rn((rs - h) * s_k));
    }
  }
  __syncthreads();
  double* gp = pb.gpart + (size_t)km.chunk * ldx + col_lo;
  const double inv_hi = (double)ldexpf(1.f, -e_hi), inv_k = (double)ldexpf(1.f, -kbits);
  for (int k = tid; k < min(col_w, ldx - col_lo); k += blockDim.x) gp[k] = ((double)g_hi[k] + (double)g_lo[k] * inv_k) * inv_hi;
}

__global__ void __launch_bounds__(1024) k1_csr_kernel(const Problem* __restrict__ probs, int has_bias, int force_emit, int beta_in_smem, int nprob_dyn) {
  const K1Map km = k1_map(probs, nprob_dyn);
  if (km.prob < 0) return;
  const Problem& pb = probs[km.prob];
  Ctrl* ctrl = pb.ctrl;
  if (ctrl->done) return;
  if (km.chunk == 0 && threadIdx.x == 0) ctrl->k1_chunks = km.nchunks;
  const bool emit = force_emit >= 0 ? (force_emit != 0) : (ctrl->emit != 0);
  extern __shared__ __align__(16) float csr_sm[];
  const int ldx = pb.ldx, Dt = pb.Dt;
  float* g_s = csr_sm;
  float* b_s = csr_sm + ldx;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int k = tid; k < ldx; k += blockDim.x) { g_s[k] = 0.f; if (beta_in_smem) b_s[k] = pb.beta_tf[k]; }
  __syncthreads();
  const float* __restrict__ bt = beta_in_smem ? b_s : pb.beta_tf;
  const long long n = pb.n;
  const long long per = (n + km.nchunks - 1) / km.nchunks;
  const long long rb = (long long)km.chunk * per, re = min(n, rb + per);
  const long long* __restrict__ rp = pb.rowptr;
  const int* __restrict__ ci = pb.colidx;
  const float* __restrict__ vv = pb.vals;
  const bool uniq = pb.csr_unique != 0;
  double loss = 0.0;
  for (long long i = rb + warp; i < re; i += nw) {
    const long long j0 = rp[i], j1 = rp[i + 1];
    const float yy = (float)pb.y[i], ww = pb.w[i], oo = pb.o[i];
    float a = 0.f;
    for (long long j = j0 + lane; j < j1; j += 32) a = fmaf(vv[j], bt[ci[j]], a);
    a = warp_sum(a);
    if (has_bias) a += bt[Dt - 1];
    const float t = yy * (a + oo);
    const float e = __expf(-fabsf(t));
    const float inv = __frcp_rn(1.f + e);
    const float p = t >= 0.f ? inv : e * inv;
    const float qq = t >= 0.f ? e * inv : inv;
    if (lane == 0) loss += (double)(ww * ((t >= 0.f ? 0.f : -t) - __logf(inv)));
    const float rr = -ww * yy * qq;
    for (long long j = j0 + lane; j < j1; j += 32) atomicAdd(&g_s[ci[j]], vv[j] * rr);
    if (has_bias && lane == 0) atomicAdd(&g_s[Dt - 1], rr);
    if (emit) {
      const float sd = sqrtf(ww * p * qq);
      __nv_bfloat16* xt = pb.Xt + (size_t)i * pb.Dp;
      if (uniq) {
        for (long long j = j0 + lane; j < j1; j += 32) xt[ci[j]] = __float2bfloat16_rn(vv[j] * sd);
      } else {
        for (long long j = j0 + lane; j < j1; j += 32) xt[ci[j]] = __float2bfloat16_rn(0.f);
        __syncwarp();
        if (lane == 0)
          for (long long j = j0; j < j1; j++) xt[ci[j]] = __float2bfloat16_rn(__bfloat162float(xt[ci[j]]) + vv[j] * sd);
      }
      if (has_bias && lane == 0) xt[Dt - 1] = __float2bfloat16_rn(sd);
    }
  }
  __syncthreads();
  double* gp = pb.gpart + (size_t)km.chunk * ldx;
  for (int k = tid; k < ldx; k += blockDim.x) gp[k] = (double)g_s[k];
  __shared__ double red[32];
  if (lane == 0) red[warp] = loss;
  __syncthreads();
  if (tid == 0) {
    double sacc = 0.0;
    for (int wq = 0; wq < nw; wq++) sacc += red[wq];
    pb.fpart[km.chunk] = sacc;
  }
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
struct K1Plan { int G, RT, nsl, S, rows_per_tile, ctas_per_sm; size_t smem; };

static size_t k1_smem_bytes(int ldx, int Rt, int S, int pdw) {
  return (size_t)S * Rt * ldx * 4 + (size_t)2 * Rt * pdw * 4 + (size_t)5 * Rt * 4 + 16 + 8 * 8 + 8 * 8 + 64;
}

// Tile shape for a given ldx.  G==1 (ldx <= 1024): RT=8 rows in registers, nsl row slices share the 256 threads,
// two CTAs per SM; wider matrices: G column groups per thread, one CTA per SM.
static bool k1_plan(int ldx, K1Plan* p) {
  const int ncg = ldx / 4;
  p->G = (ncg + K1_THREADS - 1) / K1_THREADS;
  if (p->G > 4) return false;
  if (p->G == 3) p->G = 4;
  p->RT = p->G == 4 ? 4 : 8;
  p->nsl = 1;
  if (p->G == 1) {
    p->nsl = K1_THREADS / ncg;
    if (p->nsl < 1) p->nsl = 1;
    if (p->nsl > 16) p->nsl = 16;   // rows per tile <= 128 keeps the per-warp row loop short
  }
  p->rows_per_tile = p->RT * p->nsl;
  const int pdw = p->G == 1 ? ncg : K1_THREADS;
  p->ctas_per_sm = p->G == 1 ? 2 : 1;
  const size_t budget = p->ctas_per_sm == 2 ? (size_t)113 * 1024 : (size_t)225 * 1024;
  for (int S = 4; S >= 2; S--) {
    const size_t b = k1_smem_bytes(ldx, p->rows_per_tile, S, pdw);
    if (b <= budget) { p->S = S; p->smem = b; return true; }
  }
  return false;
}

bool k1_dense_plan(int ldx, int* R_out, int* S_out, int* G_out, size_t* smem_out, int* ctas_per_sm) {
  K1Plan p;
  if (!k1_plan(ldx, &p)) return false;
  *R_out = p.rows_per_tile; *S_out = p.S; *G_out = p.G; *smem_out = p.smem;
  if (ctas_per_sm) *ctas_per_sm = p.ctas_per_sm;
  return true;
}

// Column-window width of the CSR K1 when ldx exceeds one shared-memory window (0: everything fits in one launch).
int k1_csr_window(int ldx) {
  const size_t cap = 220 * 1024;
  if ((size_t)2 * (ldx + 32) * 4 <= cap) return 0;
  return (int)((cap / 8 - 32) & ~(size_t)31);
}

// The CSR fixed-point K1 in mode MODE: one launch when the accumulators of every column fit shared memory, else the row pass with
// columns [0, W) (it leaves the row weights in rvec) and one window launch per further W columns.
template <int MODE>
static cudaError_t k1_csr_fx_launch(const Problem* d_probs, dim3 grid_all, int ldx, int has_bias, int force_emit, cudaStream_t stream, int* launches,
                                    int nprob_dyn) {
  const size_t cap = 220 * 1024;
  const size_t g_bytes = (size_t)2 * (ldx + 32) * 4;
  cudaError_t e;
  if (g_bytes <= cap) {
    const bool bsm = g_bytes + (size_t)ldx * 4 <= cap;
    const size_t smem = g_bytes + (bsm ? (size_t)ldx * 4 : 0);
    e = bsm ? cudaFuncSetAttribute(k1_csr_fx_kernel<true, false, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
            : cudaFuncSetAttribute(k1_csr_fx_kernel<false, false, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (bsm) k1_csr_fx_kernel<true, false, MODE><<<grid_all, K1_FX_THREADS, smem, stream>>>(d_probs, has_bias, force_emit, nprob_dyn, ldx);
    else k1_csr_fx_kernel<false, false, MODE><<<grid_all, K1_FX_THREADS, smem, stream>>>(d_probs, has_bias, force_emit, nprob_dyn, ldx);
    if (launches) *launches += 1;
    return cudaGetLastError();
  }
  // wider than one shared-memory window: the first launch does the margins and columns [0, W), one more launch per window
  const int W = k1_csr_window(ldx);
  const size_t smem = (size_t)2 * (W + 32) * 4;
  if ((e = cudaFuncSetAttribute(k1_csr_fx_kernel<false, true, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k1_csr_fx_window_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
  k1_csr_fx_kernel<false, true, MODE><<<grid_all, K1_FX_THREADS, smem, stream>>>(d_probs, has_bias, force_emit, nprob_dyn, W);
  if (launches) *launches += 1;
  for (int lo = W; lo < ldx; lo += W) {
    k1_csr_fx_window_kernel<MODE><<<grid_all, K1_FX_THREADS, smem, stream>>>(d_probs, has_bias, nprob_dyn, lo, W);
    if (launches) *launches += 1;
  }
  return cudaGetLastError();
}

cudaError_t k1_launch(const Problem* d_probs, int nprob, bool csr, int ldx, int has_bias, int ctas_per_problem,
                      int force_emit, cudaStream_t stream, int* launches, int csr_fx, int nprob_dyn, int mode) {
  // dynamic mapping: ctas_per_problem is then the size of the whole one-dimensional grid
  const dim3 grid_all = nprob_dyn ? dim3(ctas_per_problem, 1) : dim3(ctas_per_problem, nprob);
  if (mode != K1_GRAD && !(csr && csr_fx)) return cudaErrorInvalidValue;   // the Hv / diagonal modes exist for sorted unique CSR rows only
  if (csr && csr_fx) {
    if (mode == K1_HV) return k1_csr_fx_launch<K1_HV>(d_probs, grid_all, ldx, has_bias, 0, stream, launches, nprob_dyn);
    if (mode == K1_DIAG) return k1_csr_fx_launch<K1_DIAG>(d_probs, grid_all, ldx, has_bias, 0, stream, launches, nprob_dyn);
    return k1_csr_fx_launch<K1_GRAD>(d_probs, grid_all, ldx, has_bias, force_emit, stream, launches, nprob_dyn);
  }
  if (csr) {
    const int beta_in_smem = (size_t)2 * ldx * 4 <= 200 * 1024 ? 1 : 0;
    const size_t smem = (size_t)(beta_in_smem ? 2 : 1) * ldx * 4;
    if (smem > 220 * 1024) return cudaErrorInvalidValue;   // > 56k features: needs a column-blocked gradient (not built yet)
    cudaError_t e = cudaFuncSetAttribute(k1_csr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k1_csr_kernel<<<grid_all, 1024, smem, stream>>>(d_probs, has_bias, force_emit, beta_in_smem, nprob_dyn);
    if (launches) *launches += 1;
    return cudaGetLastError();
  }
  K1Plan p;
  if (!k1_plan(ldx, &p)) return cudaErrorInvalidValue;
  const dim3 grid = grid_all;
  cudaError_t e;
#define K1_LAUNCH(GG, RR)                                                                                          \
  e = cudaFuncSetAttribute(k1_dense_kernel<GG, RR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem);      \
  if (e != cudaSuccess) return e;                                                                                   \
  k1_dense_kernel<GG, RR><<<grid, K1_THREADS, p.smem, stream>>>(d_probs, p.S, p.nsl, force_emit, nprob_dyn);
  if (p.G == 1) { K1_LAUNCH(1, 8) } else if (p.G == 2) { K1_LAUNCH(2, 8) } else { K1_LAUNCH(4, 4) }
#undef K1_LAUNCH
  if (launches) *launches += 1;
  return cudaGetLastError();
}

// max over rows of sum_j |v_ij|: warp per row; fp32 sums of non-negative terms, atomicMax on the bits (upload, once per partition)
__global__ void csr_row_l1_kernel(long long n, const long long* __restrict__ rowptr, const float* __restrict__ vals, unsigned* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  float m = 0.f;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nw) {
    float a = 0.f;
    for (long long j = rowptr[i] + lane; j < rowptr[i + 1]; j += 32) a += fabsf(vals[j]);
    m = fmaxf(m, warp_sum(a));
  }
  if (lane == 0) atomicMax(out, __float_as_uint(m));
}
cudaError_t csr_row_l1_max(long long n, const long long* rowptr, const float* vals, unsigned* out, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  csr_row_l1_kernel<<<(int)std::min<long long>((n + 7) / 8, 2048), 256, 0, st>>>(n, rowptr, vals, out);
  return cudaGetLastError();
}

}  // namespace mlease

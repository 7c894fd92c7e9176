// k2_gram.cu -- K2: weighted Gram  G = Xt^T Xt  (Xt = diag(sqrt d) X in bf16, written by K1), the
// data term of LogisticRegressionL2.hessian (llf/LogisticRegressionL2.java:258-297):
//     H[m][n] = (m==n ? 1/priorVar[m] : 0) + sum_i D_ii x_im x_in ,  D_ii = w_i p_i (1-p_i).
// It genuinely is a dense GEMM (K = rows, M = N = features), so it runs on the Hopper tensor
// cores: TMA (tensor map, 128B swizzle) -> shared memory -> wgmma (bf16 x bf16 -> fp32 in
// registers).  Both operands are tiles of the SAME row-major matrix, i.e. they are MN-major
// ("transposed") wgmma operands: no transpose pass over X is ever made.
//
// Work decomposition: output tiles of 128 (M) x 256 (N) restricted to the lower block triangle,
// split-K over row slices; each CTA owns one (tile, slice), accumulates it in registers and
// stores the fp32 partial to Hpart[slice] (plain stores, deterministic).  chol_prep_kernel
// (k3_cholesky.cu) sums the slices in fixed order and adds diag(q).
//
// Warpgroup roles (384 threads): warpgroup 0 = TMA producer (one lane), warpgroups 1-2 = consumers,
// each issuing m64n256k16 wgmma for its 64 rows of the tile (128 fp32 accumulators a thread).
//
// CSR partitions have two kernels on the same e4m3 operand values: gram_csr_wgmma_kernel (operand blocks assembled in shared
// memory, wgmma; one byte an entry) and gram_csr_sparse_kernel (only the nonzero products of each row, exact int64 sums; one
// pre-decoded 32-bit word an entry).  session.cu batch_alloc
// picks one per batch from the data: the sparse one wins below about 3 % density at 10k features.
//
// A fp32 SIMT kernel computing the same partials from the same bf16 operand is kept ONLY as a
// debug cross-check reachable through mlease_objective(tensor=0); the product path never uses it.
#include <cuda.h>
#include <cuda_fp8.h>

#include <algorithm>
#include <cub/device/device_scan.cuh>

#include "kernels.cuh"

namespace mlease {

// ------------------------------------------------------------------------------------------
// bf16 wgmma kernel
// ------------------------------------------------------------------------------------------
constexpr int GM = 128;          // tile rows
constexpr int GN = 256;          // tile cols (wgmma N)
constexpr int GK = 64;           // K (data rows) per pipeline stage
constexpr int UK = 16;           // K per wgmma (bf16)
constexpr int GSTAGES = 4;
constexpr int G_A_BYTES = GK * GM * 2;   // 16 KB : 2 boxes of [64 k][64 feat]
constexpr int G_B_BYTES = GK * GN * 2;   // 32 KB : 4 boxes
constexpr int G_STAGE_BYTES = G_A_BYTES + G_B_BYTES;
constexpr int G_BOX_BYTES = GK * 64 * 2; // 8 KB, one TMA box = 64 k-rows x 128 B
constexpr int G_THREADS = 384;
constexpr size_t G_SMEM = (size_t)GSTAGES * G_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
// canonical MN-major SWIZZLE_128B layout (bf16) of a TMA box: ((64 elems,m),(8,k)) : ((1,LBO),(128B,SBO)), i.e.
// SBO = 1024 B between 8-row K groups, LBO = one box (GK*128 B) between 64-element MN groups.
constexpr uint32_t DESC_SW128 = 1, DESC_SW32 = 3;

struct GramTile { short bi, bj; };   // 128-row block index, column block index (256 or 128 wide)

// Stores a consumer warpgroup's m64nN accumulator into rows row0 .. row0+63 of the Dp x Dp partial.  wgmma D fragment: warp w
// of the group holds rows 16w .. 16w+15; lane l holds rows 16w + l/4 and 16w + l/4 + 8, columns 8j + 2(l%4) + {0,1}, in
// d[4j .. 4j+3].  Dp is a multiple of 128, so a column pair is either wholly inside or wholly outside.
template <int N>
__device__ __forceinline__ void store_acc(float* out, int Dp, int row0, int col0, const float (&d)[N / 2]) {
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int r = row0 + w * 16 + (lane >> 2);
  if (r + 8 >= Dp) return;
#pragma unroll
  for (int j = 0; j < N / 8; j++) {
    const int c = col0 + 8 * j + 2 * (lane & 3);
    if (c < Dp) {
      *reinterpret_cast<float2*>(out + (size_t)r * Dp + c) = make_float2(d[4 * j], d[4 * j + 1]);
      *reinterpret_cast<float2*>(out + (size_t)(r + 8) * Dp + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
  }
}

__global__ void __launch_bounds__(G_THREADS, 1)
gram_wgmma_kernel(const Problem* __restrict__ probs, const CUtensorMap* __restrict__ tmaps, const GramTile* __restrict__ tiles,
                  int ntiles, int force, int share) {
  // share = L > 1: the L problems of one partition are at the same iterate (cold start), so their Grams are identical;
  // only the first of each group is built and chol_prep_kernel reads it for the whole group
  if (share > 1 && blockIdx.z % share != 0) return;
  const int pidx = blockIdx.z;
  const Problem& pb = probs[pidx];
  Ctrl* ctrl = pb.ctrl;
  if (!force && (ctrl->done || !ctrl->need_hess)) return;
  const CUtensorMap* tmap = &tmaps[pb.self_idx];   // not blockIdx.z: large batches launch over a compacted copy of the problem array
  const GramTile tile = tiles[blockIdx.x];
  const int slice = blockIdx.y, nslices = gridDim.y;
  const int Dp = pb.Dp;
  const long long ksteps_total = (pb.n + GK - 1) / GK;
  const long long per = (ksteps_total + nslices - 1) / nslices;
  const long long ks0 = slice * per;
  const long long ks1 = min(ksteps_total, ks0 + per);
  const int nk = (int)max(0LL, ks1 - ks0);

  extern __shared__ unsigned char g_smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(g_smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)GSTAGES * G_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + GSTAGES;

  const int lane = threadIdx.x & 31, wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(tmap);
    for (int s = 0; s < GSTAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }   // 8 = the consumer warps
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      for (int k = 0; k < nk; k++) {
        const int st = k % GSTAGES;
        if (k >= GSTAGES) mbar_wait(&empty_bar[st], (uint32_t)(((k / GSTAGES) - 1) & 1));
        unsigned char* a_dst = smem + (size_t)st * G_STAGE_BYTES;
        unsigned char* b_dst = a_dst + G_A_BYTES;
        mbar_arrive_expect_tx(&full_bar[st], G_STAGE_BYTES);
        const int krow = (int)((ks0 + k) * GK);
#pragma unroll
        for (int b = 0; b < GM / 64; b++) tma_load_2d(a_dst + b * G_BOX_BYTES, tmap, tile.bi * GM + b * 64, krow, &full_bar[st]);
#pragma unroll
        for (int b = 0; b < GN / 64; b++) tma_load_2d(b_dst + b * G_BOX_BYTES, tmap, tile.bj * GN + b * 64, krow, &full_bar[st]);
      }
    }
  } else {
    // ===== consumer warpgroup wg: the tile's rows (wg - 1) * 64 .. +63 = box wg - 1 of the A block =====
    float acc[GN / 2];
#pragma unroll
    for (int j = 0; j < GN / 2; j++) acc[j] = 0.f;
    const uint32_t smem_base = smem_u32(smem);
    for (int k = 0; k < nk; k++) {
      const int st = k % GSTAGES;
      mbar_wait(&full_bar[st], (uint32_t)((k / GSTAGES) & 1));
      const uint32_t a_addr = smem_base + (uint32_t)(st * G_STAGE_BYTES + (wg - 1) * G_BOX_BYTES);
      const uint32_t b_addr = smem_base + (uint32_t)(st * G_STAGE_BYTES + G_A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < GK / UK; kk++)   // 16 k-rows = 2 swizzle atoms of 1024 B along K
        wgmma_bf16_m64n256k16_tt(acc, wgmma_desc(a_addr + kk * (UK * 128), G_BOX_BYTES, 1024, DESC_SW128),
                                 wgmma_desc(b_addr + kk * (UK * 128), G_BOX_BYTES, 1024, DESC_SW128));
      wgmma_commit();
      wgmma_wait<1>();   // the previous stage's products have retired: hand its buffer back to the producer
      if (k > 0 && lane == 0) mbar_arrive(&empty_bar[(k - 1) % GSTAGES]);
    }
    wgmma_wait<0>();
    store_acc<GN>(pb.Hpart + (size_t)slice * Dp * Dp, Dp, tile.bi * GM + (wg - 1) * 64, tile.bj * GN, acc);
  }
}

// ------------------------------------------------------------------------------------------
// Sparse variant: the same split-K Gram, but the operand tiles are ASSEMBLED IN SHARED MEMORY, as e4m3, from the partition's
// block-major entry list (no dense Xt in HBM: at 1 % density that copy is 100x the input and makes the dense kernel
// HBM-bound).  One K-step = one 32-row group = one m64n128k32 wgmma per consumer warpgroup; its entries for a 128-column block
// are one contiguous run of (key, byte), the key being the byte offset of the element inside the K-major SWIZZLE_32B operand
// block the wgmma descriptors expect (kmaj_off; wgmma takes 8-bit operands K-major only), the byte the finished e4m3 operand
// element that gram_csr_operand_kernel wrote just before the build.  Producer warps, one per operand block of a stage: load
// the run coalesced and store each byte at its key.  Positions outside the sparsity pattern are zero: the ring is cleared
// once, and a producer re-clears exactly the entries it wrote when it gets its stage back.  Generic-proxy stores are
// published to the tensor core's async proxy with fence.proxy.async before the mbarrier arrive.
// A CTA owns a 128 x 128 lower tile, two consumer warpgroups of 64 rows.  The tensor core keeps the running sum of an fp8
// product at less than fp32 precision, so a consumer runs chains of S_CHAIN wgmma (K = 128 rows) into one set of 64
// registers and adds each finished chain into a second, fp32, set; setmaxnreg moves the registers this takes from the
// producer warpgroups to the consumers.
// The build is bound by instruction issue, not by the tensor pipe (one K-step is 128 tensor cycles of an SM for 8 consumer and
// 2 producer warps): both loops are unrolled over the ring so that stage addresses, descriptors and barrier parities are
// immediates or loop-carried registers, and the producers move ready-made bytes instead of scaling and rounding values.
// Warp roles (16 warps): 0..7 = consumers, 8..15 = producers (4 groups of an A-block and a B-block warp).
// ------------------------------------------------------------------------------------------
constexpr int SK = 32;                       // data rows (K) per stage
constexpr int SN = 128;                      // tile cols
constexpr int S_BOX_BYTES = SK * 128;        // 4 KB = one [128 cols][32 k] e4m3 operand block
constexpr int SPW = 2;                       // producer warps per stage: one per operand block (A, B)
constexpr int NGRP = 4;                      // producer groups: K-step k belongs to group k % NGRP
constexpr int SST = 2 * NGRP;                // ring stages: K-step k lives in stage k % SST, so a group alternates between two
                                             // stages (the refill round trip is several MMA periods long)
constexpr int S_STAGE_BYTES = SPW * S_BOX_BYTES;
constexpr int S_CONSUMER_WARPS = 8;
constexpr int S_THREADS = (S_CONSUMER_WARPS + SPW * NGRP) * 32;   // 512: 128 registers a thread at launch
constexpr int S_CHAIN = 4;                   // wgmma per fp32 promotion
static_assert(SST == 2 * S_CHAIN, "the consumer loop runs two chains per pass over the ring");
constexpr int S_REG_PRODUCER = 72, S_REG_CONSUMER = 184;          // 256 x 72 + 256 x 184 = 65536
constexpr size_t S_SMEM = (size_t)SST * S_STAGE_BYTES + 1024 /*align*/ + 512 /*barriers*/;

// byte offset of element (K-row k < 32, column col < 128) inside one operand block of 1-byte elements in the canonical K-major
// SWIZZLE_32B layout: 32 B (= the 32 K values) per column, 8 columns per 256-B swizzle atom, and the 16-byte chunk index
// XOR-ed with bit 2 of the column (address bit 7)
__device__ __forceinline__ uint32_t kmaj_off(int k, int col) {
  return (uint32_t)(col * 32 + ((((k >> 4) ^ (col >> 2)) & 1) << 4) + (k & 15));
}
// the K-row (row inside the 32-row group) of a key
__device__ __forceinline__ int kmaj_row(uint32_t key) { return (int)(((((key >> 4) ^ (key >> 7)) & 1) << 4) | (key & 15)); }

__global__ void __launch_bounds__(S_THREADS, 1)
gram_csr_wgmma_kernel(const Problem* __restrict__ probs, const GramTile* __restrict__ tiles, int ntiles, int force, int share) {
  if (share > 1 && blockIdx.z % share != 0) return;   // see gram_wgmma_kernel
  const Problem& pb = probs[blockIdx.z];
  Ctrl* ctrl = pb.ctrl;
  if (!force && (ctrl->done || !ctrl->need_hess)) return;
  const GramTile tile = tiles[blockIdx.x];
  const int slice = blockIdx.y, nslices = gridDim.y;
  const int Dp = pb.Dp;
  const long long ksteps_total = (pb.n + SK - 1) / SK;
  const long long per = (ksteps_total + nslices - 1) / nslices;
  const long long ks0 = slice * per;
  const long long ks1 = min(ksteps_total, ks0 + per);
  const int nk = (int)max(0LL, ks1 - ks0);

  extern __shared__ unsigned char g_smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(g_smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)SST * S_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + SST;
  // shared-space addresses: the ring, and the barriers of stage s at full_u32 + 8 s / empty_u32 + 8 s
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t full_u32 = smem_base + (uint32_t)SST * S_STAGE_BYTES, empty_u32 = full_u32 + 8 * SST;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // clear the whole ring once
  for (int e = threadIdx.x; e < SST * S_STAGE_BYTES / 16; e += S_THREADS) reinterpret_cast<uint4*>(smem)[e] = make_uint4(0u, 0u, 0u, 0u);
  if (threadIdx.x == 0) {
    // full: one arrival per producer warp of the stage; empty: one per consumer warp
    for (int s = 0; s < SST; s++) { mbar_init(&full_bar[s], SPW); mbar_init(&empty_bar[s], S_CONSUMER_WARPS); }
    fence_mbar_init();
  }
  fence_proxy_async_smem();   // the zero fill must be visible to the async proxy too
  __syncthreads();

  if (warp < S_CONSUMER_WARPS) {
    // ===== consumer warpgroup wg: the tile's rows wg * 64 .. +63 = columns wg * 64 .. of the A block =====
    setmaxnreg_inc<S_REG_CONSUMER>();
    const int wg = warp >> 2;
    float acc[SN / 2], chain[SN / 2];
#pragma unroll
    for (int j = 0; j < SN / 2; j++) acc[j] = 0.f;
    // Descriptors of stage 0 (K = 32 = the stage's 32-row group = one swizzle atom along K: LBO unused, SBO = 256 B between
    // 8-column groups); stage st's differ by st * S_STAGE_BYTES / 16 in the start-address field, which cannot carry out of it
    // (shared addresses are < 2^18).  Built once: left to itself the compiler re-derives every descriptor from the shared
    // window base at every K-step.
    const uint64_t desc_a0 = wgmma_desc(smem_base + (uint32_t)(wg * 64 * SK), 16, 256, DESC_SW32);
    const uint64_t desc_b0 = wgmma_desc(smem_base + (uint32_t)S_BOX_BYTES, 16, 256, DESC_SW32);
    const uint32_t desc_hi = (uint32_t)(desc_a0 >> 32);   // same SBO and layout for both operands
    uint32_t a_lo = (uint32_t)desc_a0, b_lo = (uint32_t)desc_b0;
    asm volatile("" : "+r"(a_lo), "+r"(b_lo));   // opaque: kept in registers, not recomputed
    auto desc_a = [&](int st) { return ((uint64_t)desc_hi << 32) | (a_lo + (uint32_t)(st * S_STAGE_BYTES / 16)); };
    auto desc_b = [&](int st) { return ((uint64_t)desc_hi << 32) | (b_lo + (uint32_t)(st * S_STAGE_BYTES / 16)); };
    // stage st: wait for its operands (fill parity ph), issue its product into the chain registers (accumulate = 0 starts a chain)
    auto issue = [&](int st, uint32_t ph, uint64_t a, uint64_t b, uint32_t accumulate) {
      mbar_wait(full_u32 + 8 * st, ph);
      wgmma_fence();
      wgmma_e4m3_m64n128k32(chain, a, b, accumulate);
      wgmma_commit();
    };
    // stage st's product has retired: hand its buffer back to the producers
    auto release = [&](int st) { if (lane == 0) mbar_arrive(empty_u32 + 8 * st); };
    auto promote = [&]() {
#pragma unroll
      for (int j = 0; j < SN / 2; j++) acc[j] += chain[j];
    };
    // one whole chain in the stages s0 .. s0 + S_CHAIN - 1.  Straight-line code: a data-dependent branch between a wgmma and the
    // next makes the compiler wait for every product in flight at the join
    auto run_chain = [&](int s0, uint32_t ph) {
#pragma unroll
      for (int c = 0; c < S_CHAIN; c++) {
        issue(s0 + c, ph, desc_a(s0 + c), desc_b(s0 + c), c != 0 ? 1u : 0u);
        if (c > 0) { wgmma_wait<1>(); release(s0 + c - 1); }
      }
      wgmma_wait<0>();
      release(s0 + S_CHAIN - 1);
      promote();
    };
    // K-step k lives in stage k % SST and is that stage's fill k / SST: a pass over the ring is two chains at one parity
    const int nring = nk - nk % SST, nfull = nk - nk % S_CHAIN;
    uint32_t ph = 0;
    int k = 0;
    for (; k < nring; k += SST) {
      run_chain(0, ph);
      run_chain(S_CHAIN, ph);
      ph ^= 1u;
    }
    if (k < nfull) { run_chain(0, ph); k += S_CHAIN; }   // a last whole chain in stages 0 .. S_CHAIN - 1
    for (; k < nk; k++) {   // the last nk % S_CHAIN stages, a chain each
      const int st = k % SST;
      issue(st, (uint32_t)(k / SST) & 1u, desc_a(st), desc_b(st), 0u);
      wgmma_wait<0>();
      release(st);
      promote();
    }
    store_acc<SN>(pb.Hpart + (size_t)slice * Dp * Dp, Dp, tile.bi * 128 + wg * 64, tile.bj * SN, acc);
  } else {
    // ===== producers: SPW warps per stage, one per 128-column operand block (the A block, the B block).
    // One K-step = one 32-row group, whose entries for a 128-column block are one contiguous run of the block-major list.
    // Offsets are fetched three uses ahead and the first 64 entries of a run two uses ahead, so the loads of a use are in flight
    // during the whole previous uses.  Group t owns the K-steps k = t, t + NGRP, ...; K-step k lives in ring stage k % SST, so a
    // group alternates between the stages t (stage 0 of the group) and t + NGRP (stage 1), and the loop handles one of each per
    // pass: each stage keeps its own registers, and the run loaded after a hand-over is the stage's next one.
    setmaxnreg_dec<S_REG_PRODUCER>();
    const int pw = warp - S_CONSUMER_WARPS;
    const int grp = pw / SPW, strm = pw % SPW;
    const int blk = strm == 0 ? tile.bi : tile.bj;
    const bool valid = blk < pb.nblk128;
    const long long* __restrict__ my_offs = pb.bm_offs + (size_t)(valid ? blk : 0) * pb.bm_groups + ks0 + (lane & 1);
    const unsigned short* __restrict__ keys = pb.bm_keys;
    const unsigned char* __restrict__ bytes = pb.bm_e4m3;
    constexpr uint32_t NOKEY = 0xFFFFFFFFu;
    const bool fetch = valid && lane < 2;
    // the list holds < 2^32 entries (checked at upload): entry numbers are 32-bit
    auto ld_offs = [&](int k) -> uint32_t { return (fetch && k < nk) ? (uint32_t)__ldg(my_offs + k) : 0u; };

    struct Run { uint32_t lo, hi, key[2], byte[2]; };   // a use's run [lo, hi) and its first 64 entries (lane, lane + 32)
    struct Written { uint32_t lo, hi, key[2]; };        // the run a stage holds, to be cleared before its next fill
    auto take_offs = [&](Run& r, uint32_t o) { r.lo = __shfl_sync(0xffffffffu, o, 0); r.hi = __shfl_sync(0xffffffffu, o, 1); };
    auto ld_entries = [&](Run& r) {
#pragma unroll
      for (int q = 0; q < 2; q++) {
        const uint32_t e = r.lo + lane + 32 * q;
        r.key[q] = e < r.hi ? (uint32_t)__ldg(keys + e) : NOKEY;
        r.byte[q] = e < r.hi ? (uint32_t)__ldg(bytes + e) : 0u;
      }
    };
    Run r0, r1;
    Written w0 = {0u, 0u, {NOKEY, NOKEY}}, w1 = {0u, 0u, {NOKEY, NOKEY}};
    take_offs(r0, ld_offs(grp));
    take_offs(r1, ld_offs(grp + NGRP));
    uint32_t o_c = ld_offs(grp + 2 * NGRP);
    ld_entries(r0);
    ld_entries(r1);
    const uint32_t sbase0 = smem_base + (uint32_t)(grp * S_STAGE_BYTES + strm * S_BOX_BYTES), sbase1 = sbase0 + NGRP * S_STAGE_BYTES;
    const uint32_t full0 = full_u32 + 8 * grp, empty0 = empty_u32 + 8 * grp;
    // one use: K-step k in the stage at sbase (barriers full / empty), r = its run, w = what the stage's previous fill stored
    auto use = [&](int k, uint32_t sbase, uint32_t full, uint32_t empty, bool refill, uint32_t ph, Run& r, Written& w) {
      // ---- un-write what the previous fill of this stage stored (same addresses, zero)
      if (refill) {
        mbar_wait(empty, ph);
#pragma unroll
        for (int q = 0; q < 2; q++)
          if (w.key[q] != NOKEY) sts_u8(sbase + w.key[q], 0u);
        for (uint32_t e0 = w.lo + 64; e0 < w.hi; e0 += 32) {
          const uint32_t e = e0 + lane;
          if (e < w.hi) sts_u8(sbase + (uint32_t)__ldg(keys + e), 0u);
        }
      }
      // ---- write this use
#pragma unroll
      for (int q = 0; q < 2; q++)
        if (r.key[q] != NOKEY) sts_u8(sbase + r.key[q], r.byte[q]);
      for (uint32_t e0 = r.lo + 64; e0 < r.hi; e0 += 32) {
        const uint32_t e = e0 + lane;
        if (e < r.hi) sts_u8(sbase + (uint32_t)__ldg(keys + e), (uint32_t)__ldg(bytes + e));
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(full);
      w.lo = r.lo; w.hi = r.hi; w.key[0] = r.key[0]; w.key[1] = r.key[1];
      // ---- issue the loads of this stage's next use (K-step k + SST).  AFTER the hand-over, not before this use's stores: the
      // fence above compiles to a memory barrier that waits for every load this thread still has in flight -- issued at the top
      // of the use they would make each hand-over wait out a DRAM round trip; issued here they have the whole next use to arrive.
      take_offs(r, o_c);
      o_c = ld_offs(k + 3 * NGRP);
      ld_entries(r);
    };
    // fill f >= 1 of a stage waits for the consumers' release of fill f - 1: empty-barrier phase parity (f - 1) & 1
    uint32_t ph = 1u;
    for (int k = grp; k < nk; k += SST) {
      use(k, sbase0, full0, empty0, k >= SST, ph, r0, w0);
      if (k + NGRP >= nk) break;
      use(k + NGRP, sbase1, full0 + 8 * NGRP, empty0 + 8 * NGRP, k >= SST, ph, r1, w1);
      ph ^= 1u;
    }
  }
}

// e4m3 byte -> signed integer number of units of 2^-9 (subnormal m: m units; normal (e, m): (8 + m) << (e - 1)).  0x7F / 0xFF
// (NaN) never occur: the operand pass converts with __NV_SATFINITE.
__device__ __forceinline__ int e4m3_units(uint32_t b) {
  const int e = (int)((b >> 3) & 15u), m = (int)(b & 7u);
  const int mag = e ? (8 | m) << (e - 1) : m;
  return (b & 0x80u) ? -mag : mag;
}

// The sparse kernel's operand word of an entry: everything it needs, decoded once per build instead of once per tile reading it.
// The e4m3 value in units of 2^-9 is an integer of at most 4 significant bits below 2^18, so as an fp32 its low 20 mantissa bits
// are zero; the low 15 carry the entry's row in its span (8 bits: 32 (group mod span) + row in group) and column in its 128-block
// (7 bits).  Bits 15 .. 19 stay zero.  Decoding is a mask and one float-to-int conversion, a shift and two masks.
constexpr uint32_t SW_VALUE_MASK = 0xFFFF8000u;
__device__ __forceinline__ uint32_t sparse_word(uint32_t byte, int row_in_span, int col) {
  return __float_as_uint((float)e4m3_units(byte)) | ((uint32_t)row_in_span << 7) | (uint32_t)col;
}
__device__ __forceinline__ int sw_units(uint32_t w) { return __float2int_rz(__uint_as_float(w & SW_VALUE_MASK)); }
__device__ __forceinline__ int sw_row(uint32_t w) { return (int)((w >> 7) & 255u); }
__device__ __forceinline__ int sw_col(uint32_t w) { return (int)(w & 127u); }

// Gram operand of the CSR kernels, once per build: for every entry of the block-major list, the e4m3 byte
// e4m3(value * (sqrt(d_row) * gram_scale)), or for a sparse-kernel batch (csr_gram == CSR_GRAM_SPARSE) the same value as
// sparse_word.  gram_scale is a power of two that keeps sqrt(d) x in e4m3's normal range (chol_prep undoes it exactly).  sdvec
// is rewritten by K1 between builds, so this runs immediately before each build, gated like it.
// One warp per 32-row group: lane l holds sqrt(d) of row 32 g + l, and the group's runs of every column block follow.
__global__ void __launch_bounds__(256) gram_csr_operand_kernel(const Problem* __restrict__ probs, int force, int share) {
  if (share > 1 && blockIdx.y % share != 0) return;   // see gram_wgmma_kernel
  const Problem& pb = probs[blockIdx.y];
  const Ctrl* ctrl = pb.ctrl;
  if (!force && (ctrl->done || !ctrl->need_hess)) return;
  const int lane = threadIdx.x & 31;
  const long long n = pb.n, ngroups = pb.bm_groups;
  const int nblk = pb.nblk128;
  const long long* __restrict__ offs = pb.bm_offs;
  const unsigned short* __restrict__ keys = pb.bm_keys;
  const float* __restrict__ vals = pb.bm_vals;
  unsigned char* __restrict__ out = pb.bm_e4m3;
  uint32_t* __restrict__ out_w = pb.bm_word;
  const bool word = pb.csr_gram == CSR_GRAM_SPARSE;
  const int span = gram_sparse_span(pb.bm_entries, nblk, ngroups);   // as gram_csr_sparse_kernel computes it
  const float gscale = pb.gram_scale;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long g = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < ngroups; g += nw) {
    const long long r = g * SK + lane;
    const float sd = r < n ? pb.sdvec[r] * gscale : 0.f;
    const int row0 = 32 * (int)(g % span);   // the group's first row in its span
    for (int b = 0; b < nblk; b++) {
      const uint32_t lo = (uint32_t)offs[(size_t)b * ngroups + g], hi = (uint32_t)offs[(size_t)b * ngroups + g + 1];
      for (uint32_t e0 = lo; e0 < hi; e0 += 32) {
        const uint32_t e = e0 + lane;
        const bool v = e < hi;
        const uint32_t key = v ? (uint32_t)keys[e] : 0u;
        const float val = v ? vals[e] : 0.f;
        const int k = kmaj_row(key);
        const float sdk = __shfl_sync(0xffffffffu, sd, k);
        const uint32_t byte = __nv_cvt_float_to_fp8(val * sdk, __NV_SATFINITE, __NV_E4M3);
        if (!v) continue;
        if (word) out_w[e] = sparse_word(byte, row0 + k, (int)(key >> 5));
        else out[e] = (unsigned char)byte;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Sparse CSR Gram: the same partial from the same e4m3 operand values, but only the nonzero products of each row are formed.  At
// 1 % density a 32-row x 128-column operand block holds ~1 % nonzeros, so the wgmma kernel above spends ~10^4 multiply-adds per
// nonzero product; here each product is one integer multiply and (mostly) one native shared-memory atomic add.
// Exact and deterministic: an e4m3 value is an integer number of units of 2^-9 (|v| <= 448 = 229376 units < 2^18), so a product
// is an integer number of units of 2^-18 below 2^35.6, and the tile accumulates them as int64 (integer addition is associative:
// the sum does not depend on the warp schedule).  A 64-bit shared atomic add is a compare-and-swap loop on sm_90a, so each cell
// is a pair of 32-bit words: the product's low word goes in with a native ATOMS.ADD that returns the old word, and its high word
// plus the carry out of the low add (old + lo < old) goes into the high word -- skipped when that is 0, which is the usual case
// for |product| < 2^32 of either sign.  The pair holds the two's complement int64 sum exactly.  The epilogue rounds each cell
// once to fp32.  The sum cannot overflow below
// 2^27.4 rows (every row adds at most one product to a cell: rows have unique columns); gram_sparse_max_rows() states the limit
// the batch rule applies.
// One CTA per (128 x 128 lower tile (bi, bj), problem), one slice.  A warp's unit of work is a span of consecutive 32-row groups:
// SP_SPAN (256 rows), fewer on denser data (gram_sparse_span: the mean range of a span must fit 3/4 of a stage chunk, since each
// further chunk re-reads the bi range); warp w takes the spans w, w + SP_WARPS, ...  The list is block-major with ascending
// groups, so a block's entries for a span are one contiguous range [offs[b][g0], offs[b][g0 + span]), in row order (group, then
// row in group: csr_bm_fill_kernel writes lane 0's entries, then lane 1's, ...).  The operand pass, which visits every entry once
// per build anyway, writes each entry as one sparse_word holding its value in units, its row in the span
// (32 (group - g0) + row in group) and its column, so that the 80-odd tiles reading an entry each decode it with a few masks and
// one conversion (before: a key and a byte load, the e4m3 decode, the swizzle decode and a walk over the span's group bounds).  Per
// span the warp stages the bj range's nonzero entries in shared memory with each row's [start, end), then enumerates the
// (bi entry, staged partner of its row) pairs in a flat index space: per 32 bi entries an inclusive warp scan of the partner
// counts, then steps of 32 pairs, one per lane, each lane finding its owner entry from one OR-reduction of the owners' end
// positions in the step (owners are compacted to a per-warp table first).  So lanes stay busy however the partners are spread
// over the rows, and a row with 128 entries in both blocks (128^2 pairs) is as many full steps.  A bj range longer than SP_STAGE
// entries is staged in chunks (boundaries may fall inside a row: each chunk pairs with its own part of the row), the bi range
// re-read for each.
// What bounds it (1M x 10k x 1 %, H100 80GB HBM3 at 700 W, 36.5 ms a build): the per-entry work, not the products.  Each batch
// of 32 entries is 50 warp instructions to stage (load, decode, ballot, row table) and 76 to scan on the bi side up to the pair
// steps (row-table lookup, partner-count scan, owner table), for ~1.3 products per entry; with the byte operand they were 89 and
// 114, plus ~12 for every group bound a batch crossed.
// Diagonal tiles keep the pairs with c2 <= c1 only (predicated) and mirror them in the epilogue.  Zero operand values (w = 0
// rows, the end of a range) are skipped.
// Same-cell contention: every row's intercept entry pairs with itself in the intercept's diagonal tile, so consecutive rows'
// (intercept, intercept) products would be one step of 32 same-address atomics.  A lane sums that cell's products in an int64
// register instead, and the warp adds its total once at the end (the sum is exact, so the order does not matter).  In the other
// intercept tiles (bi = the intercept's block) the intercept row's products spread over the 128 cells of bj: at ~1 partner per
// row, a step's 32 lanes meet ~4 same-cell pairs, no worse than a bank conflict, so those are left to the atomics.
// ------------------------------------------------------------------------------------------
constexpr int SP_THREADS = 1024;
constexpr int SP_WARPS = SP_THREADS / 32;
constexpr int SP_SPAN = 8;                                         // 32-row groups per span
constexpr int SP_ROWS = SP_SPAN * 32;                              // rows per span: the row table's length
constexpr int SP_AHEAD = 1;                                        // batches of 32 entries loaded ahead of use (2: slower)
constexpr int SP_STAGE = 448;                                      // staged bj entries per warp and chunk (< 2^16: u16 row table)
constexpr size_t SP_ACC_BYTES = (size_t)SN * SN * 2 * sizeof(uint32_t);   // 128 KB: low words, then high words
// per warp: the stage (int), the row table (u32: start | end << 16) and the owner table (int2), 3 KB
constexpr size_t SP_WARP_BYTES = (size_t)SP_STAGE * 4 + (size_t)SP_ROWS * 4 + 32 * 8;
constexpr size_t SP_SMEM = SP_ACC_BYTES + (size_t)SP_WARPS * SP_WARP_BYTES;
static_assert(SP_SMEM <= 227 * 1024, "sparse Gram shared memory");
static_assert(SP_STAGE % 16 == 0, "layout of the stage");
static_assert(SP_SPAN == 8 && SP_STAGE == 448, "gram_sparse_span (kernels.cuh) assumes these");
static_assert(SP_ROWS <= 256, "sparse_word holds the row in the span in 8 bits");

__global__ void __launch_bounds__(SP_THREADS, 1)
gram_csr_sparse_kernel(const Problem* __restrict__ probs, const GramTile* __restrict__ tiles, int force, int share) {
  if (share > 1 && blockIdx.z % share != 0) return;   // see gram_wgmma_kernel
  const Problem& pb = probs[blockIdx.z];
  Ctrl* ctrl = pb.ctrl;
  if (!force && (ctrl->done || !ctrl->need_hess)) return;
  const GramTile tile = tiles[blockIdx.x];
  const int bi = tile.bi, bj = tile.bj;
  const bool diag = bi == bj;
  const int Dp = pb.Dp;
  const long long ngroups = pb.bm_groups;
  const int span = gram_sparse_span(pb.bm_entries, pb.nblk128, ngroups);   // groups per span, <= SP_SPAN
  const long long nspans = (ngroups + span - 1) / span;
  // the intercept's cell (column Dt - 1, the last entry of every row) when this is its diagonal tile, else -1 (matches no column)
  const int hot = diag && (pb.Dt - 1) / SN == bi ? (pb.Dt - 1) % SN : -1;

  extern __shared__ __align__(16) unsigned char g_smem_raw[];
  uint32_t* acc_lo = reinterpret_cast<uint32_t*>(g_smem_raw);   // [c1][c2]: low and high 32-bit words of an int64 sum
  int* acc_hi = reinterpret_cast<int*>(g_smem_raw) + SN * SN;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* wsm = g_smem_raw + SP_ACC_BYTES + (size_t)warp * SP_WARP_BYTES;
  int* stage = reinterpret_cast<int*>(wsm);                                // (units << 7) | c2
  uint32_t* rtab = reinterpret_cast<uint32_t*>(wsm + SP_STAGE * 4);        // a row's staged entries [start, end): start | end << 16
  unsigned short* rtab16 = reinterpret_cast<unsigned short*>(rtab);        // start of row r at 2 r, end at 2 r + 1
  int2* own = reinterpret_cast<int2*>(wsm + SP_STAGE * 4 + SP_ROWS * 4);  // owners of a batch: ((units << 7) | c1, start - first pair)

  for (int e = threadIdx.x; e < SN * SN; e += SP_THREADS) { acc_lo[e] = 0u; acc_hi[e] = 0; }
  __syncthreads();

  const bool valid = bi < pb.nblk128 && bj < pb.nblk128;
  const long long* __restrict__ offs_i = pb.bm_offs + (size_t)bi * ngroups;
  const long long* __restrict__ offs_j = pb.bm_offs + (size_t)bj * ngroups;
  const uint32_t* __restrict__ words = pb.bm_word;
  const uint32_t lt = (1u << lane) - 1u;
  // a cell gets the product p (units of 2^-18, int64): the low word with a native atomic add that returns the old word, the high
  // word plus the carry out of the low add when that is not 0
  auto add_cell = [&](int cell, long long p) {
    const uint32_t lo = (uint32_t)p;
    const uint32_t old = atomicAdd(acc_lo + cell, lo);
    const int hi = (int)(p >> 32) + (old + lo < old ? 1 : 0);
    if (hi != 0) atomicAdd(acc_hi + cell, hi);
  };
  // the list holds < 2^32 entries (checked at upload): entry numbers are 32-bit.  A span's ranges, lane-distributed: lanes 0, 1
  // hold offs_i[g0], offs_i[g0 + span], lanes 2, 3 the same of offs_j, clamped to the last group (a short last span's missing
  // groups are empty).  Fetched two spans ahead, and the first SP_AHEAD batches of 32 entries of both ranges one span ahead: a
  // warp has one span in flight.  Inside a range the entries are loaded SP_AHEAD batches ahead: most bj ranges are not in L2 (a
  // wave's tiles read ~80 different bj blocks), so a batch's loads need the time of several batches' work to arrive.
  auto ld_bounds = [&](long long s) -> uint32_t {
    if (!valid || s >= nspans || lane >= 4) return 0u;
    return (uint32_t)__ldg((lane < 2 ? offs_i : offs_j) + min(s * span + (lane & 1) * span, ngroups));
  };
  // an entry's operand word, 0 past the end of its range (a zero value: skipped like any zero operand)
  auto ld_entry = [&](uint32_t e, uint32_t hi) -> uint32_t { return e < hi ? __ldg(words + e) : 0u; };
  struct Span { uint32_t ilo, ihi, jlo, jhi, i[SP_AHEAD], j[SP_AHEAD]; };
  auto take = [&](Span& q, uint32_t b) {
    q.ilo = __shfl_sync(0xffffffffu, b, 0); q.ihi = __shfl_sync(0xffffffffu, b, 1);
    q.jlo = __shfl_sync(0xffffffffu, b, 2); q.jhi = __shfl_sync(0xffffffffu, b, 3);
#pragma unroll
    for (int k = 0; k < SP_AHEAD; k++) { q.i[k] = ld_entry(q.ilo + lane + 32 * k, q.ihi); q.j[k] = ld_entry(q.jlo + lane + 32 * k, q.jhi); }
  };
  long long hot_sum = 0;   // this lane's products of the intercept's cell
  auto run = [&](const Span& q) {
    const uint32_t ilo = q.ilo, ihi = q.ihi, jlo = q.jlo, jhi = q.jhi;
    if (ilo == ihi || jlo == jhi) return;
    for (uint32_t c0 = jlo; c0 < jhi; c0 += SP_STAGE) {
      const uint32_t c1 = min(jhi, c0 + SP_STAGE);   // >= jlo + 32 * SP_AHEAD or = jhi: the prefetched batches lie in the first chunk
      __syncwarp();   // the previous chunk's readers are done
#pragma unroll
      for (int k = 0; k < SP_ROWS / 128; k++) reinterpret_cast<uint4*>(rtab)[lane + 32 * k] = make_uint4(0u, 0u, 0u, 0u);
      __syncwarp();
      // ---- stage the chunk's nonzero entries; a kept entry whose row differs from the previous kept one starts its row
      int nst = 0, prev_row = -1;
      uint32_t x[SP_AHEAD + 1];   // the batches base, base + 32, ...
#pragma unroll
      for (int k = 0; k < SP_AHEAD; k++) x[k] = c0 == jlo ? q.j[k] : ld_entry(c0 + 32 * k + lane, c1);
      for (uint32_t base = c0; base < c1; base += 32) {
        x[SP_AHEAD] = ld_entry(base + 32 * SP_AHEAD + lane, c1);
        const uint32_t w = x[0];
        const int v = sw_units(w);
        const int r = sw_row(w);
        const bool keep = v != 0;
        const uint32_t m = __ballot_sync(0xffffffffu, keep);
        const uint32_t below = m & lt;
        const int up = __shfl_sync(0xffffffffu, r, below ? 31 - __clz(below) : 0);
        const int pr = below ? up : prev_row;
        const int s = nst + __popc(below);
        if (keep) {
          stage[s] = v * 128 + sw_col(w);
          if (r != pr) { rtab16[2 * r] = (unsigned short)s; if (pr >= 0) rtab16[2 * pr + 1] = (unsigned short)s; }
        }
        if (m) prev_row = __shfl_sync(0xffffffffu, r, 31 - __clz(m));
        nst += __popc(m);
#pragma unroll
        for (int k = 0; k < SP_AHEAD; k++) x[k] = x[k + 1];
      }
      if (nst == 0) continue;
      if (lane == 0) rtab16[2 * prev_row + 1] = (unsigned short)nst;
      __syncwarp();
      // ---- the (bi entry, staged partner) pairs, 32 bi entries at a time
#pragma unroll
      for (int k = 0; k < SP_AHEAD; k++) x[k] = q.i[k];
      for (uint32_t base = ilo; base < ihi; base += 32) {
        x[SP_AHEAD] = ld_entry(base + 32 * SP_AHEAD + lane, ihi);
        const uint32_t w = x[0];
        const int a = sw_units(w);
        const uint32_t t = a != 0 ? rtab[sw_row(w)] : 0u;
        const int s0 = (int)(t & 0xFFFFu), cnt = (int)(t >> 16) - s0;
        int incl = cnt;   // inclusive warp scan of the partner counts
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int u = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= d) incl += u;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
#pragma unroll
        for (int k = 0; k < SP_AHEAD; k++) x[k] = x[k + 1];
        if (total == 0) continue;
        // owners (entries with partners) in lane order: pair p belongs to the owner of rank #{owners whose pairs end at or before p}
        const uint32_t owners = __ballot_sync(0xffffffffu, cnt > 0);
        __syncwarp();   // the previous batch's readers of own[] are done
        if (cnt > 0) own[__popc(owners & lt)] = make_int2(a * 128 + sw_col(w), s0 - (incl - cnt));
        __syncwarp();
        int before = 0;   // owners whose pairs end before this step
        for (int p0 = 0; p0 < total; p0 += 32) {
          const int end = incl - p0;
          const uint32_t ends = __reduce_or_sync(0xffffffffu, cnt > 0 && end >= 0 && end < 32 ? 1u << end : 0u);
          const int p = p0 + lane;
          if (p < total) {
            const int2 o = own[before + __popc(ends & (0xFFFFFFFFu >> (31 - lane)))];
            const int pv = stage[p + o.y];
            const int c1 = o.x & 127, c2 = pv & 127;
            if (!diag || c2 <= c1) {
              const long long prod = (long long)(o.x >> 7) * (long long)(pv >> 7);
              if (c2 == hot && c1 == hot) hot_sum += prod;
              else add_cell(c1 * SN + c2, prod);
            }
          }
          before += __popc(ends);
        }
      }
    }
  };
  Span cur, nxt;
  take(cur, ld_bounds(warp));
  uint32_t nb = ld_bounds(warp + SP_WARPS);
  for (long long s = warp; s < nspans; s += SP_WARPS) {
    take(nxt, nb);   // the next span's loads are in flight while this one runs
    nb = ld_bounds(s + 2 * SP_WARPS);
    run(cur);
    cur = nxt;
  }
  if (hot >= 0) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) hot_sum += __shfl_down_sync(0xffffffffu, hot_sum, d);
    if (lane == 0 && hot_sum != 0) add_cell(hot * SN + hot, hot_sum);
  }
  __syncthreads();
  // ---- one rounding per cell: units of 2^-18 -> fp32
  float* out = pb.Hpart + (size_t)bi * SN * Dp + (size_t)bj * SN;
  for (int e = threadIdx.x; e < SN * SN; e += SP_THREADS) {
    const int c1 = e >> 7, c2 = e & 127;
    const int idx = diag && c2 > c1 ? c2 * SN + c1 : e;
    const long long v = (long long)(((unsigned long long)(uint32_t)acc_hi[idx] << 32) | acc_lo[idx]);
    out[(size_t)c1 * Dp + c2] = __ll2float_rn(v) * 0x1p-18f;
  }
}

// Largest partition (rows) the sparse kernel's int64 tile sums are safe for: every row adds at most one product of magnitude
// <= 229376^2 < 2^35.62 units to a cell, and 2^27 * 2^35.62 < 2^63
long long gram_sparse_max_rows() { return 1LL << 27; }

// Block-major entry list for the CSR Gram.  For every 128-column block b and every 32-row group g the entries
// (row in group, column in block, value) are stored contiguously at [offs[b*ngroups+g], offs[b*ngroups+g+1]); the key is
// the byte offset of the element inside a swizzled [128 col][32 k] operand block (kmaj_off), the value the stored float.
// Every row also gets an entry of value 1 for the bias column bias_col (llf/LibLinearDataset.java:592-614), which the CSR
// rows do not store; bias_col is larger than every stored column, so it is the row's last entry in its block.
// Rows must be sorted by column (strictly increasing), which the upload checks.
__device__ __forceinline__ bool bias_in_block(long long r, long long n, int bias_col, int b) {
  return r < n && bias_col >= b * 128 && bias_col < b * 128 + 128;
}

__global__ void __launch_bounds__(256) csr_bm_count_kernel(long long n, const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                           int bias_col, int nblk, long long ngroups, long long* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long g = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < ngroups; g += nw) {
    const long long r = g * 32 + lane;
    long long j = r < n ? rowptr[r] : 0;
    const long long j1 = r < n ? rowptr[r + 1] : 0;
    for (int b = 0; b < nblk; b++) {
      const long long s = j;
      while (j < j1 && colidx[j] < (b + 1) * 128) j++;
      int c = (int)(j - s) + (bias_in_block(r, n, bias_col, b) ? 1 : 0);
      c = __reduce_add_sync(0xffffffffu, c);
      if (lane == 0) counts[(size_t)b * ngroups + g] = c;
    }
  }
}

__global__ void __launch_bounds__(256) csr_bm_fill_kernel(long long n, const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                          const float* __restrict__ vals, int bias_col, int nblk, long long ngroups,
                                                          const long long* __restrict__ offs, unsigned short* __restrict__ keys,
                                                          float* __restrict__ bvals) {
  const int lane = threadIdx.x & 31;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long g = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < ngroups; g += nw) {
    const long long r = g * 32 + lane;
    long long j = r < n ? rowptr[r] : 0;
    const long long j1 = r < n ? rowptr[r + 1] : 0;
    for (int b = 0; b < nblk; b++) {
      const long long s = j;
      while (j < j1 && colidx[j] < (b + 1) * 128) j++;
      const bool bias = bias_in_block(r, n, bias_col, b);
      const int c = (int)(j - s) + (bias ? 1 : 0);
      int incl = c;   // inclusive warp scan
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
      }
      long long pos = offs[(size_t)b * ngroups + g] + (incl - c);
      for (long long e = s; e < j; e++, pos++) {
        keys[pos] = (unsigned short)kmaj_off(lane, colidx[e] - b * 128);
        bvals[pos] = vals[e];
      }
      if (bias) {
        keys[pos] = (unsigned short)kmaj_off(lane, bias_col - b * 128);
        bvals[pos] = 1.f;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// fp32 SIMT debug kernel: same operand (bf16 Xt), same output format (slice 0; other slices zeroed).
// 64x64 lower tiles, 256 threads x (4x4).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gram_simt_kernel(const Problem* __restrict__ probs, int force) {
  const Problem& pb = probs[blockIdx.z];
  Ctrl* ctrl = pb.ctrl;
  if (!force && (ctrl->done || !ctrl->need_hess)) return;
  if (blockIdx.x > blockIdx.y) return;
  const int Dp = pb.Dp;
  const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
  __shared__ float Ai[16][64 + 1];
  __shared__ float Aj[16][64 + 1];
  const int tid = threadIdx.x;
  const int ti = (tid / 16) * 4, tj = (tid % 16) * 4;
  float acc[4][4] = {};
  for (long long r0 = 0; r0 < pb.n; r0 += 16) {
    for (int e = tid; e < 16 * 64; e += 256) {
      const int r = e / 64, c = e % 64;
      const long long rr = r0 + r;
      Ai[r][c] = rr < pb.n ? __bfloat162float(pb.Xt[(size_t)rr * Dp + i0 + c]) : 0.f;
      Aj[r][c] = rr < pb.n ? __bfloat162float(pb.Xt[(size_t)rr * Dp + j0 + c]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 16; r++) {
      float x[4], y[4];
#pragma unroll
      for (int a = 0; a < 4; a++) { x[a] = Ai[r][ti + a]; y[a] = Aj[r][tj + a]; }
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b] = fmaf(x[a], y[b], acc[a][b]);
    }
    __syncthreads();
  }
  for (int s = 0; s < pb.gram_slices; s++) {
    float* out = pb.Hpart + (size_t)s * Dp * Dp;
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
      for (int b = 0; b < 4; b++) out[(size_t)(i0 + ti + a) * Dp + j0 + tj + b] = (s == 0) ? acc[a][b] : 0.f;
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Tensor map over Xt [n][Dp] bf16 row-major: dim0 = feature (contiguous), dim1 = row; box 64 x GK, 128B swizzle.
int gram_make_tensor_map(void* out_map_host /*CUtensorMap, 128 B*/, const void* xt, long long n, int Dp) {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || !p) return 1;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  cuuint64_t dims[2] = {(cuuint64_t)Dp, (cuuint64_t)n};
  cuuint64_t strides[1] = {(cuuint64_t)Dp * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)GK};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(reinterpret_cast<CUtensorMap*>(out_map_host), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(xt), dims,
                  strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 2;
}

// Lower block-triangle tile list for a Dp x Dp output (Dp multiple of 128): 128 x 256 tiles (bi, bj) for the bf16 kernel, or
// 128 x 128 tiles for the CSR kernels (csr_tiles != 0).  The tiles of one bi are consecutive, so CTAs resident at the same time
// share the bi run of the entry list in L2; the sparse kernel (csr_tiles == 2) takes the bi in descending order, which puts the
// tile of the intercept column (every row's last entry: the most contended cell) into the first wave.
int gram_tile_list(int Dp, short* bi_bj_pairs /*[2*max]*/, int max_tiles, int csr_tiles) {
  int n = 0;
  const int cols = csr_tiles ? SN : GN;
  const int nbi = (Dp + GM - 1) / GM, nbj = (Dp + cols - 1) / cols;
  for (int k = 0; k < nbi; k++) {
    const int bi = csr_tiles == 2 ? nbi - 1 - k : k;
    for (int bj = 0; bj < nbj; bj++)
      if (bj * cols <= bi * GM + GM - 1) {
        if (n >= max_tiles) return -1;
        bi_bj_pairs[2 * n] = (short)bi; bi_bj_pairs[2 * n + 1] = (short)bj; n++;
      }
  }
  return n;
}

// the attribute is per device: set it once for every device this process launches on
template <typename K>
static cudaError_t set_smem_once(K kernel, size_t bytes, bool (&configured)[64]) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  return cudaSuccess;
}

cudaError_t gram_launch_wgmma(const Problem* d_probs, int nprob, const void* d_tmaps, const void* d_tiles, int ntiles,
                              int nslices, int force, cudaStream_t st, int* launches, int share) {
  static bool configured[64] = {};
  cudaError_t e = set_smem_once(gram_wgmma_kernel, G_SMEM, configured);
  if (e != cudaSuccess) return e;
  gram_wgmma_kernel<<<dim3(ntiles, nslices, nprob), G_THREADS, G_SMEM, st>>>(
      d_probs, reinterpret_cast<const CUtensorMap*>(d_tmaps), reinterpret_cast<const GramTile*>(d_tiles), ntiles, force, share);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

// One CSR Gram build: the operand pass, then the Gram, on the same stream and gated the same way.  d_tiles holds the
// 128 x 128 tiles of gram_tile_list(..., 1)
cudaError_t gram_launch_csr_wgmma(const Problem* d_probs, int nprob, const void* d_tiles, int ntiles, int nslices, int force,
                                  cudaStream_t st, int* launches, int share) {
  static bool configured[64] = {};
  cudaError_t e = set_smem_once(gram_csr_wgmma_kernel, S_SMEM, configured);
  if (e != cudaSuccess) return e;
  gram_csr_operand_kernel<<<dim3(1024, nprob), 256, 0, st>>>(d_probs, force, share);   // ~8 warps an SM per problem
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  gram_csr_wgmma_kernel<<<dim3(ntiles, nslices, nprob), S_THREADS, S_SMEM, st>>>(
      d_probs, reinterpret_cast<const GramTile*>(d_tiles), ntiles, force, share);
  if (launches) *launches += 2;
  return cudaGetLastError();
}

// One sparse CSR Gram build: the operand pass, then the sparse Gram into slice 0.  d_tiles holds the tiles of
// gram_tile_list(..., 2)
cudaError_t gram_launch_csr_sparse(const Problem* d_probs, int nprob, const void* d_tiles, int ntiles, int force, cudaStream_t st,
                                   int* launches, int share) {
  static bool configured[64] = {};
  cudaError_t e = set_smem_once(gram_csr_sparse_kernel, SP_SMEM, configured);
  if (e != cudaSuccess) return e;
  gram_csr_operand_kernel<<<dim3(1024, nprob), 256, 0, st>>>(d_probs, force, share);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  gram_csr_sparse_kernel<<<dim3(ntiles, 1, nprob), SP_THREADS, SP_SMEM, st>>>(d_probs, reinterpret_cast<const GramTile*>(d_tiles), force, share);
  if (launches) *launches += 2;
  return cudaGetLastError();
}

// counts -> exclusive offsets in place: offs has nblk*ngroups+1 entries (the last one = total entries)
cudaError_t csr_bm_offsets(long long n, const long long* rowptr, const int* colidx, int bias_col, int nblk, long long ngroups,
                           long long* offs, cudaStream_t st) {
  const long long m = (long long)nblk * ngroups;
  cudaError_t e = cudaMemsetAsync(offs, 0, (size_t)(m + 1) * sizeof(long long), st);
  if (e != cudaSuccess) return e;
  const int grid = (int)std::min<long long>((ngroups + 7) / 8, 132 * 32);
  csr_bm_count_kernel<<<std::max(grid, 1), 256, 0, st>>>(n, rowptr, colidx, bias_col, nblk, ngroups, offs);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  size_t tmp_bytes = 0;
  if ((e = cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, offs, offs, (long long)(m + 1), st)) != cudaSuccess) return e;
  void* tmp = nullptr;
  if ((e = cudaMallocAsync(&tmp, tmp_bytes ? tmp_bytes : 16, st)) != cudaSuccess) return e;   // stream-ordered: no device-wide wait
  e = cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, offs, offs, (long long)(m + 1), st);
  cudaError_t e2 = cudaFreeAsync(tmp, st);
  return e != cudaSuccess ? e : e2;
}

cudaError_t csr_bm_fill(long long n, const long long* rowptr, const int* colidx, const float* vals, int bias_col, int nblk,
                        long long ngroups, const long long* offs, unsigned short* keys, float* bvals, cudaStream_t st) {
  const int grid = (int)std::min<long long>((ngroups + 7) / 8, 132 * 32);
  csr_bm_fill_kernel<<<std::max(grid, 1), 256, 0, st>>>(n, rowptr, colidx, vals, bias_col, nblk, ngroups, offs, keys, bvals);
  return cudaGetLastError();
}

cudaError_t gram_launch_simt(const Problem* d_probs, int nprob, int Dp, int force, cudaStream_t st, int* launches) {
  const int T = Dp / 64;
  gram_simt_kernel<<<dim3(T, T, nprob), 256, 0, st>>>(d_probs, force);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

}  // namespace mlease

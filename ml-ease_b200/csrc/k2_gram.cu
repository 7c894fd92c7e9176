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
// memory, wgmma; one byte an entry) and gram_csr_column_kernel (only the nonzero products of each row, column by column, exact
// int64 sums; one pre-decoded 32-bit word an entry, in row order).  batch.cu batch_alloc picks one per batch from the data.
//
// A fp32 SIMT kernel computing the same partials from the same bf16 operand is kept ONLY as a
// debug cross-check reachable through mlease_objective(tensor=0); the product path never uses it.
#include <cuda.h>
#include <cuda_fp8.h>

#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
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

// The sparse kernel's operand word of an entry of the row-order operand: the e4m3 value in units of 2^-9 is an integer of at most
// 4 significant bits below 2^18, so as an fp32 its low 20 mantissa bits are zero; they carry the entry's column (D' <= 2^20, which
// the batch rule checks).  Decoding is a mask and one float-to-int conversion, and a mask.
constexpr uint32_t GW_VALUE_MASK = 0xFFF00000u, GW_COL_MASK = 0x000FFFFFu;
__device__ __forceinline__ uint32_t gram_word(uint32_t byte, int col) { return __float_as_uint((float)e4m3_units(byte)) | (uint32_t)col; }
__device__ __forceinline__ int gw_units(uint32_t w) { return __float2int_rz(__uint_as_float(w & GW_VALUE_MASK)); }
__device__ __forceinline__ int gw_col(uint32_t w) { return (int)(w & GW_COL_MASK); }

// Gram operand of the CSR kernels, once per build: e4m3(value * (sqrt(d_row) * gram_scale)).  gram_scale is a power of two that
// keeps sqrt(d) x in e4m3's normal range (chol_prep undoes it exactly).  sdvec is rewritten by K1 between builds, so this runs
// immediately before each build, gated like it.
// wgmma batches: the byte of every entry of the block-major list, one warp per 32-row group (lane l holds sqrt(d) of row 32 g + l,
// and the group's runs of every column block follow).  Sparse batches (csr_gram == CSR_GRAM_SPARSE): the gram_word of every entry
// in row order, one warp per row: row r's entries at [rowptr[r] + r, rowptr[r + 1] + r), then its intercept entry (value 1,
// column Dt - 1), so every row ends with the word of the intercept.
__global__ void __launch_bounds__(256) gram_csr_operand_kernel(const Problem* __restrict__ probs, int force, int share) {
  if (share > 1 && blockIdx.y % share != 0) return;   // see gram_wgmma_kernel
  const Problem& pb = probs[blockIdx.y];
  const Ctrl* ctrl = pb.ctrl;
  if (!force && (ctrl->done || !ctrl->need_hess)) return;
  const int lane = threadIdx.x & 31;
  const long long n = pb.n;
  const float gscale = pb.gram_scale;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (pb.csr_gram == CSR_GRAM_SPARSE) {
    const long long* __restrict__ rowptr = pb.rowptr;
    const int* __restrict__ colidx = pb.colidx;
    const float* __restrict__ vals = pb.vals;
    uint32_t* __restrict__ out_w = pb.bm_word;
    const int bias_col = pb.Dt - 1;
    for (long long r = w0; r < n; r += nw) {
      const float sd = pb.sdvec[r] * gscale;
      const long long j0 = rowptr[r], j1 = rowptr[r + 1];
      for (long long j = j0 + lane; j <= j1; j += 32) {
        const bool bias = j == j1;
        const uint32_t byte = __nv_cvt_float_to_fp8((bias ? 1.f : vals[j]) * sd, __NV_SATFINITE, __NV_E4M3);
        out_w[j + r] = gram_word(byte, bias ? bias_col : colidx[j]);
      }
    }
    return;
  }
  const long long ngroups = pb.bm_groups;
  const int nblk = pb.nblk128;
  const long long* __restrict__ offs = pb.bm_offs;
  const unsigned short* __restrict__ keys = pb.bm_keys;
  const float* __restrict__ vals = pb.bm_vals;
  unsigned char* __restrict__ out = pb.bm_e4m3;
  for (long long g = w0; g < ngroups; g += nw) {
    const long long r = g * SK + lane;
    const float sd = r < n ? pb.sdvec[r] * gscale : 0.f;
    for (int b = 0; b < nblk; b++) {
      const uint32_t lo = (uint32_t)offs[(size_t)b * ngroups + g], hi = (uint32_t)offs[(size_t)b * ngroups + g + 1];
      for (uint32_t e0 = lo; e0 < hi; e0 += 32) {
        const uint32_t e = e0 + lane;
        const bool v = e < hi;
        const uint32_t key = v ? (uint32_t)keys[e] : 0u;
        const float val = v ? vals[e] : 0.f;
        const float sdk = __shfl_sync(0xffffffffu, sd, kmaj_row(key));
        const uint32_t byte = __nv_cvt_float_to_fp8(val * sdk, __NV_SATFINITE, __NV_E4M3);
        if (v) out[e] = (unsigned char)byte;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Sparse CSR Gram, column by column (Gustavson): the lower triangle's column c1 is
//     G[c2][c1] = sum over the rows r holding c1 of x_{r,c1} x_{r,c2},   c2 >= c1,
// and since a row's entries are in ascending column order with the intercept last, the partners of the entry (r, c1) are exactly
// the row's suffix from that entry up to and including its intercept entry.  So a column is a walk over its positions in the
// row-order operand (the column index gc_offs / gc_pos, built once at upload), each reading a contiguous run of words in which
// every word read is one product: no tile re-reads a block's entries, and nothing is staged or scanned.  At 1M x 10k x 1 % a
// build forms 5.2e9 products from 5.2e9 suffix words (21 GB, mostly from HBM: the operand is 404 MB), where the 128 x 128 tile
// kernel this replaces read 8.1e9 entries and spent most of its time staging and scanning them.
// Exact and deterministic: an e4m3 value is an integer number of units of 2^-9 (|v| <= 448 = 229376 units < 2^18), so a product
// is an integer number of units of 2^-18 below 2^35.6, and the column accumulates them as int64 (integer addition is associative:
// the sum does not depend on the warp schedule).  A 64-bit shared atomic add is a compare-and-swap loop on sm_90a, so each cell
// is a pair of 32-bit words: the product's low word goes in with a native ATOMS.ADD that returns the old word, and its high word
// plus the carry out of the low add (old + lo < old) goes into the high word -- skipped when that is 0, which is the usual case
// for |product| < 2^32 of either sign.  The pair holds the two's complement int64 sum exactly.  The epilogue rounds each cell
// once to fp32.  The sum cannot overflow below 2^27.4 rows (every row adds at most one product to a cell: rows have unique
// columns); gram_sparse_max_rows() states the limit the batch rule applies.
// A CTA takes the columns k = blockIdx.x, + gridDim.x, ... of one problem in the order bias column first (n positions of one
// product each), then 0, 1, ...: low columns have the longest suffixes, so each CTA starts with its heaviest.  Its accumulator
// holds the cells [c1, c1 + GC_CELLS) (a column of a wider system is walked once per window of GC_CELLS cells).  A warp takes 32
// positions of the column at a time and walks them GC_GROUP at a time: the first 32 words of the next group's suffixes are
// loaded while the current group's are multiplied, and a suffix longer than 32 words loads its next 32 before multiplying these,
// so a warp has GC_GROUP to 2 GC_GROUP runs in flight (~16 KB an SM).  Lane 0's word is the multiplier; the intercept word ends
// the walk (the ballot of its column).  Zero operands (w = 0 rows, underflow to 0) are skipped.
// What bounds it (1M x 10k x 1 %, H100 80GB HBM3 at 700 W, 26.1 ms a build with the 1.2 ms operand pass): the walk's suffix reads
// and their per-step instructions, ~19 ms; a walk step of 32 lanes reads 4 - 5 sectors whatever its suffix's length.  Loads in
// flight do not bound it (GC_GROUP 2, 4 and 8 build in 25.2, 26.1 and 25.9 ms).  Timed without them, the shared atomics take ~4.1
// ms and the epilogue's strided stores ~2.1 ms.
// The intercept's cell (Dt - 1, c1) gets one product per row of the column: a lane sums it in an int64 register and the warp adds
// its total once per column, instead of a stream of same-address atomics; the bias column's own positions are one product each
// (the intercept squared), summed by lanes in parallel.
// Epilogue: every cell of the column is rounded once and stored to Hpart[c2 Dp + c1], c2 >= c1 (and the cells above the diagonal
// of c1's 128 x 128 diagonal tile, which chol_prep reads whole, as their mirror Hpart[c1 Dp + c2]), zeros included, so every build
// writes the whole lower block triangle; reading a cell clears it for the next column.
// ------------------------------------------------------------------------------------------
constexpr int GC_THREADS = 512;
constexpr int GC_WARPS = GC_THREADS / 32;
constexpr int GC_GROUP = 4;           // positions a warp walks together (their first runs loaded one group ahead)
constexpr int GC_CELLS = 112 * 128;   // int64 cells of the accumulator: 112 KB, two CTAs an SM
constexpr int GC_BIAS_UNROLL = 8;     // positions of the bias column a thread has in flight

__global__ void __launch_bounds__(GC_THREADS, 2)
gram_csr_column_kernel(const Problem* __restrict__ probs, int force, int share) {
  if (share > 1 && blockIdx.z % share != 0) return;   // see gram_wgmma_kernel
  const Problem& pb = probs[blockIdx.z];
  Ctrl* ctrl = pb.ctrl;
  if (!force && (ctrl->done || !ctrl->need_hess)) return;
  const int Dp = pb.Dp, Dt = pb.Dt;
  const int hot = Dt - 1;   // the intercept's column: every row's last entry
  const int W = min(Dp, GC_CELLS);
  const uint32_t nent = (uint32_t)pb.bm_entries;
  const uint32_t* __restrict__ words = pb.bm_word;
  const uint32_t* __restrict__ offs = pb.gc_offs;
  const uint32_t* __restrict__ cpos = pb.gc_pos;
  float* __restrict__ out = pb.Hpart;

  extern __shared__ __align__(16) unsigned char g_smem_raw[];
  uint32_t* acc_lo = reinterpret_cast<uint32_t*>(g_smem_raw);   // [cell]: low and high 32-bit words of an int64 sum
  int* acc_hi = reinterpret_cast<int*>(g_smem_raw) + W;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = threadIdx.x; e < W; e += GC_THREADS) { acc_lo[e] = 0u; acc_hi[e] = 0; }
  __syncthreads();

  // a cell gets the product p (units of 2^-18, int64): the low word with a native atomic add that returns the old word, the high
  // word plus the carry out of the low add when that is not 0
  auto add_cell = [&](int cell, long long p) {
    const uint32_t lo = (uint32_t)p;
    const uint32_t old = atomicAdd(acc_lo + cell, lo);
    const int hi = (int)(p >> 32) + (old + lo < old ? 1 : 0);
    if (hi != 0) atomicAdd(acc_hi + cell, hi);
  };
  // the operand holds < 2^32 - 64 words (checked at upload): positions are 32-bit; past its end a word is 0
  auto word_at = [&](uint32_t q) -> uint32_t { return q < nent ? __ldg(words + q) : 0u; };

  for (int k = blockIdx.x; k < Dp; k += gridDim.x) {
    const int c1 = k == 0 ? hot : (k <= hot ? k - 1 : k);
    const uint32_t p0 = c1 < Dt ? __ldg(offs + c1) : 0u, p1 = c1 < Dt ? __ldg(offs + c1 + 1) : 0u;
    for (int w0 = c1; w0 < Dp; w0 += W) {
      const int w1 = min(Dp, w0 + W);
      long long hot_sum = 0;   // this lane's products of the intercept's cell (hot, c1)
      if (c1 == hot) {
        // every position is a row's intercept word, its only partner itself
        for (uint32_t i0 = p0 + threadIdx.x; i0 < p1; i0 += GC_THREADS * GC_BIAS_UNROLL) {
          uint32_t x[GC_BIAS_UNROLL];
#pragma unroll
          for (int u = 0; u < GC_BIAS_UNROLL; u++) {
            const uint32_t i = i0 + u * GC_THREADS;
            x[u] = i < p1 ? __ldg(cpos + i) : 0xFFFFFFFFu;
          }
#pragma unroll
          for (int u = 0; u < GC_BIAS_UNROLL; u++) x[u] = word_at(x[u]);
#pragma unroll
          for (int u = 0; u < GC_BIAS_UNROLL; u++) { const long long v = gw_units(x[u]); hot_sum += v * v; }
        }
      } else {
        // one position q (warp-uniform) with the first 32 words of its suffix in x (lane l: word q + l)
        auto walk = [&](uint32_t q, uint32_t x) {
          const int a = gw_units(__shfl_sync(0xffffffffu, x, 0));
          if (a == 0) return;
          while (true) {
            const int c2 = gw_col(x);
            const uint32_t ends = __ballot_sync(0xffffffffu, c2 == hot);
            uint32_t nx = 0u;
            if (!ends) nx = word_at(q + 32 + lane);   // the next 32 words are in flight while these are multiplied
            const int v = gw_units(x);
            if ((!ends || lane < __ffs(ends)) && v != 0) {
              const long long prod = (long long)a * (long long)v;
              if (c2 == hot) hot_sum += prod;
              else if (c2 >= w0 && c2 < w1) add_cell(c2 - w0, prod);
            }
            if (ends) return;
            x = nx;
            q += 32;
          }
        };
        for (uint32_t cb = p0 + 32u * warp; cb < p1; cb += 32u * GC_WARPS) {
          const int cnt = (int)min(32u, p1 - cb);
          const uint32_t mine = lane < cnt ? __ldg(cpos + cb + lane) : 0u;   // the chunk's positions, one a lane
          uint32_t cur[GC_GROUP];
#pragma unroll
          for (int g = 0; g < GC_GROUP; g++) {
            const uint32_t q = __shfl_sync(0xffffffffu, mine, g);
            cur[g] = g < cnt ? word_at(q + lane) : 0u;
          }
          for (int j = 0; j < cnt; j += GC_GROUP) {
            uint32_t nxt[GC_GROUP];
#pragma unroll
            for (int g = 0; g < GC_GROUP; g++) {
              const int jj = j + GC_GROUP + g;
              const uint32_t q = __shfl_sync(0xffffffffu, mine, jj & 31);
              nxt[g] = jj < cnt ? word_at(q + lane) : 0u;
            }
#pragma unroll
            for (int g = 0; g < GC_GROUP; g++) {
              const uint32_t q = __shfl_sync(0xffffffffu, mine, j + g);
              if (j + g < cnt) walk(q, cur[g]);
            }
#pragma unroll
            for (int g = 0; g < GC_GROUP; g++) cur[g] = nxt[g];
          }
        }
      }
      if (hot >= w0 && hot < w1) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) hot_sum += __shfl_down_sync(0xffffffffu, hot_sum, d);
        if (lane == 0 && hot_sum != 0) add_cell(hot - w0, hot_sum);
      }
      __syncthreads();
      // ---- one rounding per cell: units of 2^-18 -> fp32; the cell is cleared for the next column
      const int dend = (c1 / 128 + 1) * 128;   // end of c1's diagonal tile
      for (int e = threadIdx.x; e < w1 - w0; e += GC_THREADS) {
        const int c2 = w0 + e;
        const long long v = (long long)(((unsigned long long)(uint32_t)acc_hi[e] << 32) | acc_lo[e]);
        acc_lo[e] = 0u; acc_hi[e] = 0;
        const float f = __ll2float_rn(v) * 0x1p-18f;
        out[(size_t)c2 * Dp + c1] = f;
        if (c2 > c1 && c2 < dend) out[(size_t)c1 * Dp + c2] = f;
      }
      __syncthreads();
    }
  }
}

// Largest partition (rows) the sparse kernel's int64 column sums are safe for: every row adds at most one product of magnitude
// <= 229376^2 < 2^35.62 units to a cell, and 2^27 * 2^35.62 < 2^63
long long gram_sparse_max_rows() { return 1LL << 27; }
// Widest system (D', the intercept included) the sparse kernel takes: its operand word holds the column in 20 bits
int gram_sparse_max_cols() { return 1 << 20; }

// Column index of the sparse CSR Gram: for every column c < D' the positions, in the row-order operand, of its entries, ascending
// (so in row order): pos[offs[c] .. offs[c + 1]).  Row r's entries sit at [rowptr[r] + r, rowptr[r + 1] + r] with its intercept
// (column bias_col = D' - 1) last.  Built by a stable radix sort of the entries' columns in row order.
__global__ void __launch_bounds__(256) csr_col_keys_kernel(long long n, const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                           int bias_col, uint32_t* __restrict__ keys, uint32_t* __restrict__ idx) {
  const int lane = threadIdx.x & 31;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += nw) {
    const long long j0 = rowptr[r], j1 = rowptr[r + 1];
    for (long long j = j0 + lane; j <= j1; j += 32) {
      keys[j + r] = j == j1 ? (uint32_t)bias_col : (uint32_t)colidx[j];
      idx[j + r] = (uint32_t)(j + r);
    }
  }
}
// offs[c] = the first sorted entry of column >= c, for c in [0, ncols]
__global__ void __launch_bounds__(256) csr_col_offsets_kernel(long long entries, const uint32_t* __restrict__ sorted, int ncols,
                                                              uint32_t* __restrict__ offs) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= entries; i += (long long)gridDim.x * blockDim.x) {
    const long long lo = i == 0 ? -1 : (long long)sorted[i - 1];
    const long long hi = i == entries ? (long long)ncols : (long long)sorted[i];
    for (long long c = lo + 1; c <= hi; c++) offs[c] = (uint32_t)i;
  }
}

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
// 128 x 128 tiles for the CSR wgmma kernel (csr_tiles != 0).  The tiles of one bi are consecutive, so CTAs resident at the same
// time share the bi run of the entry list in L2.
int gram_tile_list(int Dp, short* bi_bj_pairs /*[2*max]*/, int max_tiles, int csr_tiles) {
  int n = 0;
  const int cols = csr_tiles ? SN : GN;
  const int nbi = (Dp + GM - 1) / GM, nbj = (Dp + cols - 1) / cols;
  for (int bi = 0; bi < nbi; bi++) {
    for (int bj = 0; bj < nbj; bj++)
      if (bj * cols <= bi * GM + GM - 1) {
        if (n >= max_tiles) return -1;
        bi_bj_pairs[2 * n] = (short)bi; bi_bj_pairs[2 * n + 1] = (short)bj; n++;
      }
  }
  return n;
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

// One sparse CSR Gram build of Dp x Dp problems: the operand pass, then the column kernel into slice 0, two CTAs an SM for every
// problem (a gated-off one returns at once)
cudaError_t gram_launch_csr_sparse(const Problem* d_probs, int nprob, int Dp, int force, cudaStream_t st, int* launches, int share) {
  static bool configured[64] = {};
  static int sms[64] = {};
  cudaError_t e = set_smem_once(gram_csr_column_kernel, (size_t)GC_CELLS * 8, configured);
  if (e != cudaSuccess) return e;
  int dev = 0, nsm = 0;
  if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
  if (dev >= 0 && dev < 64 && sms[dev]) nsm = sms[dev];
  else {
    if ((e = cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) sms[dev] = nsm;
  }
  gram_csr_operand_kernel<<<dim3(1024, nprob), 256, 0, st>>>(d_probs, force, share);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  const size_t smem = (size_t)std::min(Dp, GC_CELLS) * 8;
  gram_csr_column_kernel<<<dim3(std::min(Dp, 2 * nsm), 1, nprob), GC_THREADS, smem, st>>>(d_probs, force, share);
  if (launches) *launches += 2;
  return cudaGetLastError();
}

// The column index of the sparse CSR Gram (csr_col_keys_kernel): offs [bias_col + 2], pos [entries = nnz + n]
cudaError_t csr_col_index(long long n, const long long* rowptr, const int* colidx, int bias_col, long long entries, uint32_t* offs,
                          uint32_t* pos, cudaStream_t st) {
  cudaError_t e = cudaSuccess;
  uint32_t *keys = nullptr, *sorted = nullptr, *idx = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
  int bits = 1;
  while ((1LL << bits) <= bias_col) bits++;
  auto run = [&]() -> cudaError_t {
    cudaError_t r;
    // stream-ordered temporaries: no device-wide wait
    if ((r = cudaMallocAsync(&keys, (size_t)entries * 4, st)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync(&sorted, (size_t)entries * 4, st)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync(&idx, (size_t)entries * 4, st)) != cudaSuccess) return r;
    const int grid = (int)std::min<long long>((n + 7) / 8, 132 * 32);
    csr_col_keys_kernel<<<std::max(grid, 1), 256, 0, st>>>(n, rowptr, colidx, bias_col, keys, idx);
    if ((r = cudaGetLastError()) != cudaSuccess) return r;
    if ((r = cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, sorted, idx, pos, entries, 0, bits, st)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync(&tmp, tmp_bytes ? tmp_bytes : 16, st)) != cudaSuccess) return r;
    if ((r = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, sorted, idx, pos, entries, 0, bits, st)) != cudaSuccess) return r;
    csr_col_offsets_kernel<<<(int)std::min<long long>((entries + 256) / 256, 132 * 32), 256, 0, st>>>(entries, sorted, bias_col + 1, offs);
    return cudaGetLastError();
  };
  e = run();
  for (void* p : {(void*)keys, (void*)sorted, (void*)idx, tmp})
    if (p) { cudaError_t e2 = cudaFreeAsync(p, st); if (e == cudaSuccess) e = e2; }
  return e;
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

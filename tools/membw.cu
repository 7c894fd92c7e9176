// membw.cu -- microbenchmark: how fast can one pass over a 8 GB fp32 matrix be streamed into an SM by
//   (a) 1-D bulk TMA copies (cp.async.bulk, UBLKCP) into a shared-memory ring
//   (b) plain ld.global.nc.v4 into registers
//   (c) cp.async 16 B (LDGSTS) into a shared-memory ring
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o membw tools/membw.cu ; run on the H100.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c)); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ bool mbar_try(uint64_t* b, uint32_t par) { uint32_t ok; asm volatile("{.reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0,1,0,p;}" : "=r"(ok) : "r"(s32(b)), "r"(par) : "memory"); return ok; }
__device__ __forceinline__ void bulk(void* d, const void* s, uint32_t bytes, uint64_t* b) { asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(d)), "l"(s), "r"(bytes), "r"(s32(b)) : "memory"); }

// (a) bulk: tile_bytes per stage, S stages; consumers just read one float4 per thread per 4 KB to keep it honest
__global__ void __launch_bounds__(256) k_bulk(const float* x, size_t nbytes, int tile_bytes, int S, float* out) {
  extern __shared__ __align__(128) unsigned char sm[];
  uint64_t* bar = (uint64_t*)(sm + (size_t)S * tile_bytes);
  size_t ntiles = nbytes / tile_bytes;
  size_t my = ntiles > blockIdx.x ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  if (threadIdx.x == 0) { for (int s = 0; s < S; s++) mbar_init(&bar[s], 1); asm volatile("fence.mbarrier_init.release.cluster;"); }
  __syncthreads();
  auto issue = [&](size_t k) { size_t t = blockIdx.x + k * gridDim.x; mbar_expect(&bar[k % S], tile_bytes); bulk(sm + (k % S) * (size_t)tile_bytes, (const char*)x + t * tile_bytes, tile_bytes, &bar[k % S]); };
  if (threadIdx.x == 0) for (size_t k = 0; k < (size_t)S && k < my; k++) issue(k);
  float acc = 0;
  for (size_t k = 0; k < my; k++) {
    while (!mbar_try(&bar[k % S], (k / S) & 1)) {}
    const float4* t4 = (const float4*)(sm + (k % S) * (size_t)tile_bytes);
    for (int i = threadIdx.x; i < tile_bytes / 16; i += 256) { float4 v = t4[i]; acc += v.x + v.y + v.z + v.w; }
    __syncthreads();
    if (threadIdx.x == 0 && k + S < my) issue(k + S);
  }
  if (acc == 12345.f) out[0] = acc;
}
// (b) LDG: each thread loads U float4 per iteration (coalesced), grid-stride
template <int U> __global__ void __launch_bounds__(256) k_ldg(const float4* x, size_t n4, float* out) {
  float acc = 0;
  size_t stride = (size_t)gridDim.x * 256 * U;
  for (size_t base = (size_t)blockIdx.x * 256 * U + threadIdx.x; base < n4; base += stride) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; u++) { size_t i = base + (size_t)u * 256; if (i < n4) asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[u].x), "=f"(v[u].y), "=f"(v[u].z), "=f"(v[u].w) : "l"(x + i)); else v[u] = make_float4(0, 0, 0, 0); }
#pragma unroll
    for (int u = 0; u < U; u++) acc += v[u].x + v[u].y + v[u].z + v[u].w;
  }
  if (acc == 12345.f) out[0] = acc;
}
// (c) cp.async 16B ring
__global__ void __launch_bounds__(256) k_cpasync(const float4* x, size_t n4, int tile4, int S, float* out) {
  extern __shared__ __align__(128) unsigned char sm[];
  float4* ring = (float4*)sm;
  size_t ntiles = n4 / tile4;
  size_t my = ntiles > blockIdx.x ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  auto issue = [&](size_t k) { size_t t = blockIdx.x + k * gridDim.x; const float4* src = x + t * tile4; float4* dst = ring + (k % S) * (size_t)tile4;
    for (int i = threadIdx.x; i < tile4; i += 256) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s32(dst + i)), "l"(src + i));
    asm volatile("cp.async.commit_group;"); };
  for (size_t k = 0; k < (size_t)(S - 1); k++) { if (k < my) issue(k); else asm volatile("cp.async.commit_group;"); }
  float acc = 0;
  for (size_t k = 0; k < my; k++) {
    if (k + S - 1 < my) issue(k + S - 1); else asm volatile("cp.async.commit_group;");
    asm volatile("cp.async.wait_group %0;" ::"n"(2));   // S-1 = 2 groups may stay in flight (S must be 3)
    __syncthreads();
    const float4* t4 = ring + (k % S) * (size_t)tile4;
    for (int i = threadIdx.x; i < tile4; i += 256) { float4 v = t4[i]; acc += v.x + v.y + v.z + v.w; }
    __syncthreads();
  }
  if (acc == 12345.f) out[0] = acc;
}
int main() {
  size_t nbytes = (size_t)8 << 30;
  float* x; float* out;
  cudaMalloc(&x, nbytes); cudaMalloc(&out, 64); cudaMemset(x, 0, nbytes);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  auto time = [&](const char* name, auto launch) { launch(); cudaDeviceSynchronize(); cudaEventRecord(a); for (int r = 0; r < 5; r++) launch(); cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); ms /= 5;
    printf("%-44s %7.3f ms  %7.1f GB/s  %s\n", name, ms, nbytes / 1e6 / ms, cudaGetErrorString(cudaGetLastError())); };
  for (int tile : {8192, 16384, 32768, 65536}) for (int S : {2, 3, 4}) for (int cps : {1, 2, 3}) {
    size_t smem = (size_t)S * tile + 64; if (smem * cps > 225 * 1024) continue;
    cudaFuncSetAttribute(k_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    char nm[96]; snprintf(nm, 96, "bulk tile=%dKB S=%d ctas/sm=%d", tile / 1024, S, cps);
    time(nm, [&] { k_bulk<<<132 * cps, 256, smem>>>(x, nbytes, tile, S, out); });
  }
  for (int cps : {2, 4, 8}) {
    char nm[96];
    snprintf(nm, 96, "ldg U=4 ctas/sm=%d", cps); time(nm, [&] { k_ldg<4><<<132 * cps, 256>>>((const float4*)x, nbytes / 16, out); });
    snprintf(nm, 96, "ldg U=8 ctas/sm=%d", cps); time(nm, [&] { k_ldg<8><<<132 * cps, 256>>>((const float4*)x, nbytes / 16, out); });
    snprintf(nm, 96, "ldg U=16 ctas/sm=%d", cps); time(nm, [&] { k_ldg<16><<<132 * cps, 256>>>((const float4*)x, nbytes / 16, out); });
  }
  for (int tile : {16384, 32768}) for (int cps : {1, 2}) {
    size_t smem = (size_t)3 * tile; cudaFuncSetAttribute(k_cpasync, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    char nm[96]; snprintf(nm, 96, "cp.async16 tile=%dKB S=3 ctas/sm=%d", tile / 1024, cps);
    time(nm, [&] { k_cpasync<<<132 * cps, 256, smem>>>((const float4*)x, nbytes / 16, tile / 16, 3, out); });
  }
  return 0;
}

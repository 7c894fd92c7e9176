// dmma_rate.cu -- microbenchmark: issue-bound throughput of the fp64 tensor-core instructions on the card, operands in
// registers (no shared memory, no global traffic in the timed loop):
//   (a) mma.m8n8k4  (SASS DMMA.8x8x4,  256 FMA per instruction), what dgemm_kernel (csrc/k3_cholesky.cu) issues
//   (b) mma.m16n8k4 (SASS DMMA.16x8x4, 512 FMA per instruction)
// Each warp keeps ACC independent accumulator sets so that the loop is bound by issue, not by the DMMA latency.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dmma_rate tools/dmma_rate.cu ; run on the H100.
#include <cstdio>
#include <cuda_runtime.h>

constexpr int ACC = 8, ITERS = 4096;

__global__ void __launch_bounds__(256) k_884(double* out, double seed) {
  double c[ACC][2];
  const double a = seed + threadIdx.x, b = seed - threadIdx.x;
#pragma unroll
  for (int q = 0; q < ACC; q++) c[q][0] = c[q][1] = 0.0;
  for (int i = 0; i < ITERS; i++)
#pragma unroll
    for (int q = 0; q < ACC; q++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[q][0]), "+d"(c[q][1]) : "d"(a), "d"(b));
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < ACC; q++) s += c[q][0] + c[q][1];
  if (s == 1.2345) out[0] = s;
}

__global__ void __launch_bounds__(256) k_1684(double* out, double seed) {
  double c[ACC][4];
  const double a0 = seed + threadIdx.x, a1 = seed * 2 + threadIdx.x, b = seed - threadIdx.x;
#pragma unroll
  for (int q = 0; q < ACC; q++) c[q][0] = c[q][1] = c[q][2] = c[q][3] = 0.0;
  for (int i = 0; i < ITERS; i++)
#pragma unroll
    for (int q = 0; q < ACC; q++)
      asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                   : "+d"(c[q][0]), "+d"(c[q][1]), "+d"(c[q][2]), "+d"(c[q][3]) : "d"(a0), "d"(a1), "d"(b));
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < ACC; q++) s += c[q][0] + c[q][1] + c[q][2] + c[q][3];
  if (s == 1.2345) out[0] = s;
}

int main() {
  int dev = 0, sms = 0, clk = 0;
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, dev);
  printf("%s, %d SMs, max SM clock %.0f MHz\n", prop.name, sms, clk / 1e3);
  double* out;
  cudaMalloc(&out, 64);
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  auto time = [&](const char* name, double fma_per_instr, auto launch, int ctas) {
    launch(ctas); cudaDeviceSynchronize();
    cudaEventRecord(a);
    for (int r = 0; r < 5; r++) launch(ctas);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b); ms /= 5;
    const double flop = 2.0 * fma_per_instr * ACC * ITERS * (ctas * 8.0);   // 8 warps per CTA
    printf("%-18s ctas/sm=%d  %8.3f ms  %6.2f TFLOP/s  %s\n", name, ctas / sms, ms, flop / ms / 1e9, cudaGetErrorString(cudaGetLastError()));
  };
  for (int cps : {1, 2, 4}) {
    time("DMMA.8x8x4", 256.0, [&](int n) { k_884<<<n, 256>>>(out, 1.0); }, sms * cps);
    time("DMMA.16x8x4", 512.0, [&](int n) { k_1684<<<n, 256>>>(out, 1.0); }, sms * cps);
  }
  return 0;
}

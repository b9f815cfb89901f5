// ifetch.cu — microbenchmark: cycles per instruction of a straight-line FP32 loop body as a function of its code size,
// with 1 or 2 warps per SM sub-partition.  Diagnostic for DESIGN.md §5 (the step kernel's substep body is 57 KB).
#include <cstdio>
#include <cuda_runtime.h>
template <int BODY>
__global__ void __launch_bounds__(32) k(float* out, int iters, float x, float y, long long* cyc) {
  float a0 = threadIdx.x, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < BODY / 8; i++) {
      a0 = fmaf(a0, x, y); a1 = fmaf(a1, x, a0 * 0.f + y); a2 = fmaf(a2, x, y); a3 = fmaf(a3, y, x);
      a4 = fmaf(a4, x, y); a5 = fmaf(a5, y, x); a6 = fmaf(a6, x, y); a7 = fmaf(a7, y, x);
    }
  }
  long long t1 = clock64();
  out[blockIdx.x * 32 + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
template <int BODY>
void run(int grid) {
  float* out; long long* cyc; cudaMalloc(&out, grid * 32 * 4); cudaMalloc(&cyc, grid * 8);
  int iters = 200000 / BODY + 4;
  k<BODY><<<grid, 32>>>(out, iters, 1.0001f, 0.5f, cyc);
  k<BODY><<<grid, 32>>>(out, iters, 1.0001f, 0.5f, cyc);
  cudaDeviceSynchronize();
  long long* h = new long long[grid]; cudaMemcpy(h, cyc, grid * 8, cudaMemcpyDeviceToHost);
  double s = 0, mx = 0; for (int i = 0; i < grid; i++) { s += h[i]; if (h[i] > mx) mx = h[i]; }
  cudaFuncAttributes fa; cudaFuncGetAttributes(&fa, k<BODY>);
  printf("{\"body_instr\": %d, \"grid\": %d, \"cpi_mean\": %.3f, \"cpi_max\": %.3f}\n", BODY, grid, s / grid / ((double)BODY * 1.125 * iters), mx / ((double)BODY * 1.125 * iters));
  cudaFree(out); cudaFree(cyc); delete[] h;
}
int main() {
  for (int grid : {132, 528, 1056, 2112}) {
    run<256>(grid); run<1024>(grid); run<1792>(grid); run<2304>(grid); run<3584>(grid); run<7168>(grid);
  }
  return 0;
}

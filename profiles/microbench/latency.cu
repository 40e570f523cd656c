// Dependent-issue latencies on the box (cycles per operation in a serial chain, one warp):
// DADD, DMUL, DFMA, double division, sqrt, rsqrt, SHFL, shared load, L1-hit global load.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o latency latency.cu ; run: ./latency
#include <cstdio>
#include <cuda_runtime.h>

template <int OP>
__global__ void chain(double* out, long long* cyc, double seed, const double* tbl, int n) {
  __shared__ double sh[64];
  sh[threadIdx.x & 63] = seed;
  __syncthreads();
  double x = seed + threadIdx.x * 1e-9, y = 1.0000001;
  long long idx = 0;
  const long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < n; ++i) {
    if (OP == 0) x = __dadd_rn(x, y);
    if (OP == 1) x = __dmul_rn(x, y);
    if (OP == 2) x = __fma_rn(x, y, y);
    if (OP == 3) x = y / x + 1.5;            // division (+1 add so the value stays bounded)
    if (OP == 4) x = sqrt(x) + 1.5;
    if (OP == 5) x = rsqrt(x) + 1.5;
    if (OP == 6) x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31);
    if (OP == 7) { x = sh[(int)(x) & 63]; }
    if (OP == 8) { idx = (long long)tbl[idx]; }
  }
  const long long t1 = clock64();
  out[threadIdx.x] = x + (double)idx;
  if (threadIdx.x == 0) *cyc = t1 - t0;
}

int main() {
  double* out; long long* cyc; double* tbl;
  cudaMalloc(&out, 64 * sizeof(double)); cudaMalloc(&cyc, sizeof(long long));
  const int T = 1024;
  double h[T];
  for (int i = 0; i < T; ++i) h[i] = (double)((i * 37 + 11) % T);
  cudaMalloc(&tbl, T * sizeof(double)); cudaMemcpy(tbl, h, sizeof(h), cudaMemcpyHostToDevice);
  const char* names[] = {"dadd", "dmul", "dfma", "ddiv+dadd", "dsqrt+dadd", "drsqrt+dadd", "shfl(64b)", "lds(64b)+cvt", "ldg L1 hit(64b)+cvt"};
  const int n = 4096;
  for (int op = 0; op < 9; ++op) {
    long long c = 0;
    for (int rep = 0; rep < 2; ++rep) {
      switch (op) {
        case 0: chain<0><<<1, 32>>>(out, cyc, 1.0, tbl, n); break;
        case 1: chain<1><<<1, 32>>>(out, cyc, 1.0, tbl, n); break;
        case 2: chain<2><<<1, 32>>>(out, cyc, 1.0, tbl, n); break;
        case 3: chain<3><<<1, 32>>>(out, cyc, 1.0, tbl, n); break;
        case 4: chain<4><<<1, 32>>>(out, cyc, 1.0, tbl, n); break;
        case 5: chain<5><<<1, 32>>>(out, cyc, 1.0, tbl, n); break;
        case 6: chain<6><<<1, 32>>>(out, cyc, 1.0, tbl, n); break;
        case 7: chain<7><<<1, 32>>>(out, cyc, 1.0, tbl, n); break;
        case 8: chain<8><<<1, 32>>>(out, cyc, 0.0, tbl, n); break;
      }
      cudaDeviceSynchronize();
      cudaMemcpy(&c, cyc, sizeof(c), cudaMemcpyDeviceToHost);
    }
    printf("%-22s %7.1f cycles/op\n", names[op], (double)c / n);
  }
  return 0;
}

// Latency calibration (diagnostics only): dependent-chain cycles per op for one warp.
#include <cstdio>
#include <cuda_runtime.h>
#define N 512
__global__ void k(double *out, long long *cyc, double a, double b, float fa, float fb) {
  __shared__ double sm[1024];
  __shared__ int si[1024];
  int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) { sm[i] = a + i; si[i] = (i * 7 + 1) & 1023; }
  __syncthreads();
  double x = a + lane; float fx = fa + lane; int ix = lane; long long t0, t1;
  // 0: DFMA chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) x = __fma_rn(x, b, a);
  t1 = clock64(); if (threadIdx.x == 0) cyc[0] = t1 - t0;
  // 1: DADD chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) x = __dadd_rn(x, b);
  t1 = clock64(); if (threadIdx.x == 0) cyc[1] = t1 - t0;
  // 2: DMUL chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) x = __dmul_rn(x, b);
  t1 = clock64(); if (threadIdx.x == 0) cyc[2] = t1 - t0;
  // 3: ddiv chain
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; i++) x = __ddiv_rn(x, b);
  t1 = clock64(); if (threadIdx.x == 0) cyc[3] = t1 - t0;
  // 4: FFMA chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) fx = __fmaf_rn(fx, fb, fa);
  t1 = clock64(); if (threadIdx.x == 0) cyc[4] = t1 - t0;
  // 5: IMAD chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) ix = ix * 3 + lane;
  t1 = clock64(); if (threadIdx.x == 0) cyc[5] = t1 - t0;
  // 6: LDS pointer chase
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) ix = si[ix & 1023];
  t1 = clock64(); if (threadIdx.x == 0) cyc[6] = t1 - t0;
  // 7: shfl chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) ix = __shfl_sync(0xffffffffu, ix, (lane + 1) & 31);
  t1 = clock64(); if (threadIdx.x == 0) cyc[7] = t1 - t0;
  // 8: ballot+ffs chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) ix = __ffs(__ballot_sync(0xffffffffu, ix & 1)) + ix;
  t1 = clock64(); if (threadIdx.x == 0) cyc[8] = t1 - t0;
  // 9: __syncthreads chain
  t0 = clock64();
  for (int i = 0; i < N; i++) __syncthreads();
  t1 = clock64(); if (threadIdx.x == 0) cyc[9] = t1 - t0;
  // 10: 64-bit integer multiply chain (key hash)
  unsigned long long h = ix;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) { h *= 0x9E3779B97F4A7C15ull; h ^= h >> 32; }
  t1 = clock64(); if (threadIdx.x == 0) cyc[10] = t1 - t0;
  // 11: double->int round trip (trunc + cvt)
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) x = (double)__double2int_rz(x) + 0.25;
  t1 = clock64(); if (threadIdx.x == 0) cyc[11] = t1 - t0;
  // 12: 3 independent DFMA chains (ILP)
  double y = x + 1, z = x + 2;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++) { x = __fma_rn(x, b, a); y = __fma_rn(y, b, a); z = __fma_rn(z, b, a); }
  t1 = clock64(); if (threadIdx.x == 0) cyc[12] = t1 - t0;
  out[threadIdx.x] = x + y + z + fx + ix + (double)h;
}
int main() {
  double *out; long long *cyc; cudaMalloc(&out, 1024 * 8); cudaMalloc(&cyc, 16 * 8);
  const char *nm[] = {"DFMA", "DADD", "DMUL", "DDIV_RN", "FFMA", "IMAD", "LDS chase", "SHFL", "BALLOT+FFS", "BAR.SYNC", "IMUL64+XORSHIFT", "D2I+I2D+DADD", "3xDFMA ILP (per triple)"};
  for (int nt : {32, 128}) {
    k<<<1, nt>>>(out, cyc, 1.0000001, 0.9999999, 1.0001f, 0.9999f); cudaDeviceSynchronize();
    k<<<1, nt>>>(out, cyc, 1.0000001, 0.9999999, 1.0001f, 0.9999f); cudaDeviceSynchronize();
    long long h[16]; cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    printf("threads=%d\n", nt);
    for (int i = 0; i < 13; i++) printf("  %-24s %7.1f cycles/op\n", nm[i], (double)h[i] / N);
  }
  printf("err=%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}

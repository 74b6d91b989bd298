// Single-warp latency probes for sor_lane_kernel's design (a warp alone on its scheduler):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probe/warp_latency_probe tools/probe/warp_latency_probe.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void probe(float* out, long long* cyc, int n) {
  __shared__ float sm[1024];
  const int l = threadIdx.x;
  for (int i = l; i < 1024; i += 32) sm[i] = 1.0f;
  __syncwarp();
  float x = l * 0.5f, y = 1.0f, z = 2.0f, w4 = 3.0f;
  long long t0, t1;
  // 1: dependent shuffle + add
  t0 = clock64();
  for (int i = 0; i < n; ++i) x = __shfl_up_sync(0xffffffffu, x, 1) + 1.0f;
  t1 = clock64();
  if (l == 0) cyc[0] = t1 - t0;
  // 2: four shuffles then four adds (one dependent round)
  t0 = clock64();
  for (int i = 0; i < n; ++i) {
    float a = __shfl_up_sync(0xffffffffu, x, 1), b = __shfl_up_sync(0xffffffffu, y, 1), c = __shfl_up_sync(0xffffffffu, z, 1), d = __shfl_up_sync(0xffffffffu, w4, 1);
    x = a + 1.0f; y = b + 1.0f; z = c + 1.0f; w4 = d + 1.0f;
  }
  t1 = clock64();
  if (l == 0) cyc[1] = t1 - t0;
  // 3: dependent shared-memory round trip (store, then load the neighbour's slot)
  t0 = clock64();
  for (int i = 0; i < n; ++i) {
    sm[l] = x;
    __syncwarp();
    x = sm[(l + 31) & 31] + 1.0f;
    __syncwarp();
  }
  t1 = clock64();
  if (l == 0) cyc[2] = t1 - t0;
  // 4: dependent chain of 16 FADD/FMUL (no FMA)
  t0 = clock64();
  for (int i = 0; i < n; ++i) {
#pragma unroll
    for (int k = 0; k < 8; ++k) x = __fadd_rn(__fmul_rn(x, 0.999f), 0.001f);
  }
  t1 = clock64();
  if (l == 0) cyc[3] = t1 - t0;
  // 5: dependent LDS (pointer chase in shared memory)
  int idx = l;
  t0 = clock64();
  for (int i = 0; i < n; ++i) idx = __float_as_int(sm[idx & 1023]) & 1023;
  t1 = clock64();
  if (l == 0) cyc[4] = t1 - t0;
  // 6: uniform branch on a freshly computed predicate
  int acc = 0;
  t0 = clock64();
  for (int i = 0; i < n; ++i) {
    if (__float_as_int(x) + i > 0x7f000000) acc += __popc(i) * 3;
    x = __fadd_rn(x, 1.0f);
  }
  t1 = clock64();
  if (l == 0) cyc[5] = t1 - t0;
  out[l] = x + y + z + w4 + idx + acc;
}
int main() {
  float* out; long long* cyc;
  cudaMalloc(&out, 128); cudaMalloc(&cyc, 64);
  const int n = 4096;
  for (int r = 0; r < 2; ++r) probe<<<1, 32>>>(out, cyc, n);
  long long h[6];
  cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
  const char* names[6] = {"shfl_up + fadd, dependent", "4 independent shfl_up + 4 fadd per round", "sts + syncwarp + lds neighbour + fadd + syncwarp", "16 dependent fmul/fadd", "dependent lds", "uniform branch on fresh predicate + fadd"};
  for (int i = 0; i < 6; ++i) printf("%-52s %7.1f cycles per iteration\n", names[i], (double)h[i] / n);
  return 0;
}

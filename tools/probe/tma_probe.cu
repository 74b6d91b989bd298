// Probe of the TMA tensor-tile load variants the P=12 patch kernel could use (tools only).
//   tma_probe <variant>   0: 2-D map, one thread issues   1: 3-D map, one thread   2: 3-D, 4 divergent lanes of a warp
//                         3: like 2 but descriptor read from global memory instead of a __grid_constant__ parameter
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define W 104
#define H 72
#define NF 2
#ifndef XOFF
#define XOFF 4  // box start along the inner dimension: must be a multiple of 4 floats (16 bytes), see DESIGN.md 5.2
#endif
static_assert(XOFF % 4 == 0, "an unaligned box start faults (illegal instruction)");
#ifndef BW
#define BW 20
#endif
#ifndef BH
#define BH 13
#endif
#ifndef PROMO
#define PROMO CU_TENSOR_MAP_L2_PROMOTION_L2_128B
#endif

__device__ __forceinline__ void mbar_init(unsigned a) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(a) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned a, unsigned ph) {
  asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}" ::"r"(a), "r"(ph) : "memory");
}

template <int RANK>
__global__ void probe(const __grid_constant__ CUtensorMap tmap, const CUtensorMap* gmap, int use_g, int lanes, float* out) {
  extern __shared__ __align__(128) float smem[];
  const int tid = threadIdx.x;
  const int q = tid >> 3, l8 = tid & 7;
  constexpr int WIN = (BW * BH * 4 + 127) / 128 * 32;
  float* win = smem + q * WIN;
  const unsigned mbar = (unsigned)__cvta_generic_to_shared(smem + 4 * WIN) + 8u * q;
  if (l8 == 0) { mbar_init(mbar); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncwarp();
  const bool issue = (l8 == 0) && (q < lanes);
  if (issue) {
    const unsigned dst = (unsigned)__cvta_generic_to_shared(win);
    const CUtensorMap* d = use_g ? gmap : &tmap;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"((unsigned)(BW * BH * 4)) : "memory");
    const int x = XOFF + 4 * q, y = 5 + 2 * q, z = q & 1;
    if (RANK == 2)
      asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                   ::"r"(dst), "l"(d), "r"(mbar), "r"(x), "r"(y) : "memory");
    else
      asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                   ::"r"(dst), "l"(d), "r"(mbar), "r"(x), "r"(y), "r"(z) : "memory");
  }
  if (q < lanes) mbar_wait(mbar, 0);
  __syncwarp();
  if (q < lanes && l8 == 0) { out[q * 2] = win[0]; out[q * 2 + 1] = win[BW * (BH - 1) + BW - 1]; }
}

int main(int argc, char** argv) {
  const int variant = argc > 1 ? atoi(argv[1]) : 0;
  std::vector<float> h((size_t)NF * H * W);
  for (size_t i = 0; i < h.size(); ++i) h[i] = (float)i;
  float *d, *out;
  cudaMalloc(&d, h.size() * 4);
  cudaMalloc(&out, 64);
  cudaMemcpy(d, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess) { printf("no entry point\n"); return 2; }
  EncodeFn encode = (EncodeFn)fn;
  const int rank = variant == 0 ? 2 : 3;
  CUtensorMap tm;
  const cuuint64_t dims[3] = {W, H, NF};
  const cuuint64_t strides[2] = {W * 4, (cuuint64_t)W * H * 4};
  const cuuint32_t box[3] = {BW, BH, 1}, estr[3] = {1, 1, 1};
  CUresult r = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, d, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_NONE, PROMO, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  printf("encode rc=%d\n", (int)r);
  CUtensorMap* gmap;
  cudaMalloc(&gmap, sizeof(tm));
  cudaMemcpy(gmap, &tm, sizeof(tm), cudaMemcpyHostToDevice);
  const int lanes = variant >= 2 ? 4 : 1;
  constexpr int WIN = (BW * BH * 4 + 127) / 128 * 32;
  const size_t sm = 4 * WIN * 4 + 64;
  if (rank == 2) probe<2><<<1, 32, sm>>>(tm, gmap, variant == 3, lanes, out);
  else probe<3><<<1, 32, sm>>>(tm, gmap, variant == 3, lanes, out);
  cudaError_t e = cudaDeviceSynchronize();
  float ho[8] = {0};
  cudaMemcpy(ho, out, 32, cudaMemcpyDeviceToHost);
  printf("variant %d: %s", variant, cudaGetErrorString(e));
  for (int q = 0; q < lanes; ++q) {
    const int x = XOFF + 4 * q, y = 5 + 2 * q, z = (rank == 3) ? (q & 1) : 0;
    printf(" | q%d got %.0f %.0f want %.0f %.0f", q, ho[q * 2], ho[q * 2 + 1], h[((size_t)z * H + y) * W + x], h[((size_t)z * H + y + BH - 1) * W + x + BW - 1]);
  }
  printf("\n");
  return e != cudaSuccess;
}

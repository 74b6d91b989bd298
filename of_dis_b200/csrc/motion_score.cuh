// The RANSAC scoring kernel of global motion (motion_kernels.cu) and relative pose (relpose_kernels.cu): a pair's
// float4 correspondences stream through shared memory in 64 KB tiles (cp.async.bulk + mbarrier, two buffers); each
// warp keeps 4 hypotheses' 9 floats (MotionHyp::g) in registers, tests them against every correspondence it reads with
// Test::inlier(g, c, mg.t) and takes one 64-bit atomicMax per solvable hypothesis: the best (count << 32) |
// (0xFFFFFFFF - h).  A pair of fewer than mg.n_min correspondences solved no hypothesis and is skipped.
#pragma once
#include <cuda_runtime.h>

#include "bulk_tile.cuh"
#include "ofdis_internal.cuh"

namespace ofdis {
namespace {

constexpr int kScoreWarps = 16, kScoreHpw = 4, kScoreHpb = kScoreWarps * kScoreHpw;  // hypotheses per warp / CTA
constexpr int kTile = 4096;                                                          // float4 per 64 KB tile
constexpr size_t kScoreSmem = 2 * kTile * sizeof(float4) + 16;                       // two tiles, two mbarriers

template <class Test>
__global__ void __launch_bounds__(kScoreWarps * 32, 1) motion_score_kernel(MotionGeom mg, MotionWork ws) {
  using namespace tiles;
  extern __shared__ __align__(16) float4 tiles[];  // [2][kTile], then two mbarriers
  const int k = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int m = ws.m[k];
  if (m < mg.n_min) return;  // no solvable hypothesis (uniform over the CTA)
  const int h0 = blockIdx.x * kScoreHpb + warp * kScoreHpw;
  float g[kScoreHpw][9];
  bool ok[kScoreHpw];
#pragma unroll
  for (int i = 0; i < kScoreHpw; ++i) {
    const int h = h0 + i;
    ok[i] = false;
    for (int e = 0; e < 9; ++e) g[i][e] = 0.f;
    if (h < mg.nh) {
      const MotionHyp& r = ws.hg[(size_t)k * mg.hyp_cap + h];
      ok[i] = r.ok != 0;
#pragma unroll
      for (int e = 0; e < 9; ++e) g[i][e] = r.g[e];
    }
  }
  const unsigned buf0 = smem_u32(tiles), mbar0 = buf0 + 2u * kTile * sizeof(float4);
  const float4* src = ws.corr + (size_t)k * mg.cell_cap;
  const int ntiles = (m + kTile - 1) / kTile;
  auto issue = [&](int t) {
    const int cnt = min(kTile, m - t * kTile);
    bulk_tile(buf0 + (unsigned)(t & 1) * kTile * sizeof(float4), src + (size_t)t * kTile, (unsigned)cnt * 16u,
              mbar0 + 8u * (t & 1));
  };
  if (threadIdx.x == 0) {
    mbar_init(mbar0, 1);
    mbar_init(mbar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    issue(0);
    if (ntiles > 1) issue(1);
  }
  int cnt[kScoreHpw];
#pragma unroll
  for (int i = 0; i < kScoreHpw; ++i) cnt[i] = 0;
  const float t = mg.t;
  for (int tt = 0; tt < ntiles; ++tt) {
    const int b = tt & 1;
    mbar_wait(mbar0 + 8u * b, (unsigned)(tt >> 1) & 1u);
    const float4* tile = tiles + b * kTile;
    const int n_in = min(kTile, m - tt * kTile);
#pragma unroll 4
    for (int e = lane; e < n_in; e += 32) {
      const float4 c = tile[e];
#pragma unroll
      for (int i = 0; i < kScoreHpw; ++i) cnt[i] += Test::inlier(g[i], c, t);
    }
    __syncthreads();  // every warp is done with buffer b
    if (threadIdx.x == 0 && tt + 2 < ntiles) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      issue(tt + 2);
    }
  }
#pragma unroll
  for (int i = 0; i < kScoreHpw; ++i) {
    const unsigned total = __reduce_add_sync(0xffffffffu, (unsigned)cnt[i]);
    if (lane == 0 && ok[i])
      atomicMax(ws.key + k, ((unsigned long long)total << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)(h0 + i)));
  }
}

// one launch of the scoring kernel for n pairs: 0, or -1 on a launch error
template <class Test>
int launch_motion_score(const MotionGeom& mg, const MotionWork& ws, int n, cudaStream_t st) {
  if (smem_optin((const void*)motion_score_kernel<Test>, kScoreSmem, false) != cudaSuccess) return -1;
  motion_score_kernel<Test><<<dim3((mg.nh + kScoreHpb - 1) / kScoreHpb, n), kScoreWarps * 32, kScoreSmem, st>>>(mg, ws);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

}  // namespace
}  // namespace ofdis

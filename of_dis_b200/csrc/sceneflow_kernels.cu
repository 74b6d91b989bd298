// Scene flow from flows and disparities (ofdis_scene_flow_fullres; the header states the contract,
// preprocess.scene_flow restates it bit for bit).  One kernel, one thread per pixel, every pair of a call in one grid
// dimension: the flow through upsample_at, the second disparity gathered at the flow's target, both points
// triangulated, the outputs and, with stats, the per-(pair, class) counts.  A CTA is 32 x 32 pixels of one pair, a
// warp one row of it: the warp adds its counts per class into the CTA's shared counters, and the CTA adds those to
// the pair's with one global atomicAdd per class and count.  All of a pair's counts land on its 8 x nclasses
// counters, so one global atomic per warp and count would bound a call with stats.  Float32 without contraction.
#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int SF_ROWS = 32;  // rows of a CTA (32 x SF_ROWS threads)

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }
__device__ __forceinline__ float canon(float v) { return isnan(v) ? qnan() : v; }
// KITTI's outlier rule of ofdis_flow_error_fullres
__device__ __forceinline__ bool outlier(float e, float g) { return e > 3.0f && e > 0.05f * g; }

// count bits of one pixel: bit i (0..3) counts it for D1, D2, Fl, SF, bit 4 + i marks it an outlier there
__global__ void __launch_bounds__(32 * SF_ROWS) sceneflow_kernel(LevelGeom g, int fa, SfArgs a, int w_org, int h_org,
                                                        int crop_x, int crop_y) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  const int k = blockIdx.z;
  const bool in_px = X < w_org && Y < h_org;
  const size_t pix = (size_t)w_org * h_org;
  const size_t o = (size_t)k * pix + (size_t)Y * w_org + X;
  int cls = -1;
  unsigned flags = 0;
  if (in_px) {
    const float* F = g.flow + (size_t)frame_of(g, fa, k) * g.flow_frame_stride;
    float f[2];
    upsample_at<2>(g, F, X, Y, crop_x, crop_y, [&f](int c, float v) { f[c] = v; });
    const float* D0 = a.disp0 + (size_t)k * a.stride;
    const float* D1 = a.disp1 + (size_t)k * a.stride;
    const float d0 = D0[(size_t)Y * w_org + X];
    const float xs = (float)X + f[0], ys = (float)Y + f[1];
    const bool in = in_frame_f(xs, ys, w_org, h_org);
    float d1 = qnan();
    if (in) d1 = sf_d1_at(D1, xs, ys, w_org, h_org, a.edge_diff);
    const bool k0 = known_d(d0), k1 = in && known_d(d1);
    const unsigned char st = (unsigned char)((k0 ? 0 : 1) | (in ? 0 : 2) | (in && !k1 ? 4 : 0));
    const float d1w = k1 ? d1 : qnan();
    if (a.status) a.status[o] = st;
    if (a.disp1w) a.disp1w[o] = d1w;
    if (a.motion) {
      const DispCamera& c = a.cam;
      const float s0 = d0 + c.doffs, s1 = d1 + c.doffs;
      float m[3] = {qnan(), qnan(), qnan()};
      if (st == 0 && s0 > 0.0f && s1 > 0.0f) {
        const float Z0 = c.fb / s0, X0 = (((float)X - c.cx) * Z0) / c.fx, Y0 = (((float)Y - c.cy) * Z0) / c.fy;
        const float Z1 = c.fb / s1, X1 = ((xs - c.cx) * Z1) / c.fx, Y1 = ((ys - c.cy) * Z1) / c.fy;
        m[0] = canon(X1 - X0);
        m[1] = canon(Y1 - Y0);
        m[2] = canon(Z1 - Z0);
      }
      float* q = a.motion + o * 3;
      q[0] = m[0];
      q[1] = m[1];
      q[2] = m[2];
    }
    if (a.stats) {
      const int c = a.classes ? (int)a.classes[o] : 0;
      const float G0 = a.gt_d0[o], G1 = a.gt_d1[o], Gu = a.gt_flow[2 * o], Gv = a.gt_flow[2 * o + 1];
      const bool kg0 = known_d(G0), kg1 = known_d(G1), kgf = fabsf(Gu) <= 1e9f && fabsf(Gv) <= 1e9f;
      const float inf = __int_as_float(0x7f800000);
      const float e0 = k0 ? fabsf(d0 - G0) : inf, e1 = k1 ? fabsf(d1w - G1) : inf;
      const float du = f[0] - Gu, dv = f[1] - Gv;
      const bool kf = fabsf(f[0]) <= 1e9f && fabsf(f[1]) <= 1e9f;
      const float ef = kf ? sqrtf(du * du + dv * dv) : inf, gf = sqrtf(Gu * Gu + Gv * Gv);
      const bool o0 = outlier(e0, fabsf(G0)), o1 = outlier(e1, fabsf(G1)), of = outlier(ef, gf);
      const bool ksf = kg0 && kg1 && kgf;
      flags = (kg0 ? 1u : 0u) | (kg1 ? 2u : 0u) | (kgf ? 4u : 0u) | (ksf ? 8u : 0u) | (kg0 && o0 ? 16u : 0u) |
              (kg1 && o1 ? 32u : 0u) | (kgf && of ? 64u : 0u) | (ksf && (o0 || o1 || of) ? 128u : 0u);
      if (c < a.nclasses && flags) cls = c;
    }
  }
  if (a.stats) {  // uniform over the grid, so every thread of the CTA takes part
    __shared__ unsigned int sc[16 * 8];
    const int t = threadIdx.y * 32 + threadIdx.x;
    if (t < 16 * 8) sc[t] = 0;
    __syncthreads();
    const unsigned same = __match_any_sync(FULL, cls);
    const bool leader = threadIdx.x == __ffs(same) - 1;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const unsigned cnt = __popc(__ballot_sync(FULL, (flags >> b) & 1u) & same);
      if (leader && cls >= 0 && cnt) atomicAdd(sc + cls * 8 + b, cnt);
    }
    __syncthreads();
    if (t < a.nclasses * 8 && sc[t])
      atomicAdd(reinterpret_cast<unsigned long long*>(a.stats + (size_t)k * a.nclasses) + t, (unsigned long long)sc[t]);
  }
}

}  // namespace

int launch_scene_flow(const LevelGeom& g, int fa, int n, const SfArgs& a, int w_org, int h_org, int crop_x, int crop_y,
                      cudaStream_t st) {
  const dim3 block(32, SF_ROWS), grid((w_org + 31) / 32, (h_org + SF_ROWS - 1) / SF_ROWS, n);
  sceneflow_kernel<<<grid, block, 0, st>>>(g, fa, a, w_org, h_org, crop_x, crop_y);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ofdis

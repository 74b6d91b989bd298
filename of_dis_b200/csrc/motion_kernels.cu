// Global camera motion from dense flows (ofdis_global_motion_fullres; the header states the contract,
// preprocess.global_motion restates it bit for bit).  A fixed number of launches per call, whatever the number of
// pairs:
//   motion_corr_kernel     one thread per (cell, pair): the validity flag and the normalized correspondence;
//   motion_compact_kernel  one CTA per pair: a block scan over the cells in tiles, compacting in place in cell order;
//   motion_hyp_kernel      one thread per (hypothesis, pair): the draws and the float64 elimination;
//   motion_score_kernel    the hot path (motion_score.cuh, shared with relative pose): the pair's correspondences
//                          stream through shared memory in 64 KB tiles; each warp tests 4 hypotheses per shared read
//                          and takes one 64-bit atomicMax per hypothesis;
//   motion_refit_kernel    one CTA per pair: every refit round (inlier test, chunk sums, tree, solve) and the model;
//   motion_apply_kernel    one thread per pixel: residual, mask and registered bytes (only when asked for).
// The flows are read through upsample_at / consistency_at; no full-resolution copy is stored.  float32 and float64
// without contraction (-fmad=false), IEEE division.
#include <cuda_runtime.h>

#include "motion_score.cuh"

namespace ofdis {

namespace {

constexpr int kCorrThreads = 256;
constexpr int kCompactThreads = 1024;
constexpr int kHypThreads = 128;
constexpr int kRefitThreads = 256;
constexpr int kChunk = 32;

// the two rows r1 | b1, r2 | b2 of correspondence c (float64 of its float32 values)
template <int MODEL>
__device__ __forceinline__ void motion_rows(const float4 c, double* r1, double* r2, double& b1, double& b2) {
  const double x = c.x, y = c.y, p = c.z, q = c.w;
  b1 = p;
  b2 = q;
  if (MODEL == OFDIS_MOTION_SIMILARITY) {
    r1[0] = x, r1[1] = -y, r1[2] = 1.0, r1[3] = 0.0;
    r2[0] = y, r2[1] = x, r2[2] = 0.0, r2[3] = 1.0;
  } else {
    r1[0] = x, r1[1] = y, r1[2] = 1.0, r1[3] = 0.0, r1[4] = 0.0, r1[5] = 0.0;
    r2[0] = 0.0, r2[1] = 0.0, r2[2] = 0.0, r2[3] = x, r2[4] = y, r2[5] = 1.0;
    if (MODEL == OFDIS_MOTION_HOMOGRAPHY) {
      r1[6] = -(x * p), r1[7] = -(y * p);
      r2[6] = -(x * q), r2[7] = -(y * q);
    }
  }
}

// H^ (row-major 3 x 3) of the parameters x
template <int MODEL>
__device__ __forceinline__ void motion_hmat(const double* x, double* H) {
  if (MODEL == OFDIS_MOTION_SIMILARITY) {
    H[0] = x[0], H[1] = -x[1], H[2] = x[2], H[3] = x[1], H[4] = x[0], H[5] = x[3], H[6] = 0.0, H[7] = 0.0;
  } else {
    for (int i = 0; i < 6; ++i) H[i] = x[i];
    H[6] = MODEL == OFDIS_MOTION_HOMOGRAPHY ? x[6] : 0.0;
    H[7] = MODEL == OFDIS_MOTION_HOMOGRAPHY ? x[7] : 0.0;
  }
  H[8] = 1.0;
}

// ---- 1. correspondences ------------------------------------------------------------------------------------------
template <bool FB>
__global__ void __launch_bounds__(kCorrThreads) motion_corr_kernel(LevelGeom g, int fa, int fb, MotionGeom mg,
                                                                   MotionWork ws) {
  const int c = blockIdx.x * kCorrThreads + threadIdx.x, k = blockIdx.y;
  if (c >= mg.cells) return;
  const int cx = min((c % mg.ncx) * mg.s + mg.s / 2, mg.w - 1), cy = min((c / mg.ncx) * mg.s + mg.s / 2, mg.h - 1);
  const float* F = g.flow + (size_t)frame_of(g, fa, k) * g.flow_frame_stride;
  float f[2] = {0.f, 0.f};
  upsample_at<2>(g, F, cx, cy, mg.crop_x, mg.crop_y, [&f](int ch, float v) { f[ch] = v; });
  const float xs = (float)cx + f[0], ys = (float)cy + f[1];
  bool ok = fabsf(f[0]) <= 1e9f && fabsf(f[1]) <= 1e9f && in_frame_f(xs, ys, mg.w, mg.h);
  if (FB && ok) {
    const float* B = g.flow + (size_t)frame_of(g, fb, k) * g.flow_frame_stride;
    consistency_at<2>(g, B, f, cx, cy, mg.w, mg.h, mg.crop_x, mg.crop_y, mg.alpha, mg.beta,
                      [&ok](unsigned char mask, float) { ok = mask == 0; });
  }
  const size_t o = (size_t)k * mg.cell_cap + c;
  ws.flag[o] = ok ? 1 : 0;
  if (ok)
    ws.corr[o] = make_float4(((float)cx - mg.cx) * mg.sigma, ((float)cy - mg.cy) * mg.sigma, (xs - mg.cx) * mg.sigma,
                             (ys - mg.cy) * mg.sigma);
}

// ---- 2. compaction (integer offsets only, so the order is the cell order) ------------------------------------------
__global__ void __launch_bounds__(kCompactThreads) motion_compact_kernel(MotionGeom mg, MotionWork ws) {
  __shared__ int warp_off[kCompactThreads / 32], tile_total;
  const int k = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float4* corr = ws.corr + (size_t)k * mg.cell_cap;
  const unsigned char* flag = ws.flag + (size_t)k * mg.cell_cap;
  int base = 0;
  for (int t0 = 0; t0 < mg.cells; t0 += kCompactThreads) {
    const int c = t0 + threadIdx.x;
    const bool f = c < mg.cells && flag[c];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (f) v = corr[c];
    const unsigned ball = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_off[warp] = __popc(ball);
    __syncthreads();  // every read of this tile is done before any write below (the writes go to indices <= c)
    if (warp == 0) {
      const int cnt = warp_off[lane];
      int incl = cnt;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
      }
      warp_off[lane] = incl - cnt;
      if (lane == 31) tile_total = incl;
    }
    __syncthreads();
    if (f) corr[base + warp_off[warp] + __popc(ball & ((1u << lane) - 1u))] = v;
    base += tile_total;
    __syncthreads();  // the next tile rewrites warp_off and tile_total
  }
  if (threadIdx.x == 0) {
    ws.m[k] = base;
    ws.key[k] = 0ull;
  }
}

// ---- 3. hypotheses ---------------------------------------------------------------------------------------------------
template <int MODEL>
__global__ void __launch_bounds__(kHypThreads) motion_hyp_kernel(MotionGeom mg, MotionWork ws) {
  constexpr int N = MODEL + 1, K = 2 * N;
  const int h = blockIdx.x * kHypThreads + threadIdx.x, k = blockIdx.y;
  if (h >= mg.nh) return;
  const int m = ws.m[k];
  MotionHyp rec{};
  double x[K];
  bool ok = false;
  if (m >= N) {
    const float4* corr = ws.corr + (size_t)k * mg.cell_cap;
    double A[K][K], b[K];
#pragma unroll
    for (int d = 0; d < N; ++d) {
      const unsigned idx = motion_draw(mg.seed, h, d, m);
      motion_rows<MODEL>(corr[idx], A[2 * d], A[2 * d + 1], b[2 * d], b[2 * d + 1]);
    }
    ok = motion_solve<K>(A, b, x);
  }
  double* hp = ws.hp + ((size_t)k * mg.hyp_cap + h) * 8;
  if (ok) {
    double H[9];
    motion_hmat<MODEL>(x, H);
#pragma unroll
    for (int i = 0; i < K; ++i) hp[i] = x[i];
#pragma unroll
    for (int i = 0; i < 9; ++i) rec.g[i] = (float)H[i];
  }
  rec.ok = ok ? 1 : 0;
  ws.hg[(size_t)k * mg.hyp_cap + h] = rec;
}

// ---- 4. scoring (the hot path) ----------------------------------------------------------------------------------------
// the inlier test of the header; without a perspective row W' is exactly 1, so the test reduces to its float32 value
template <bool PERSP>
__device__ __forceinline__ int motion_inlier(const float* g, float4 c, float t) {
  const float X = (g[0] * c.x + g[1] * c.y) + g[2], Y = (g[3] * c.x + g[4] * c.y) + g[5];
  if (PERSP) {
    const float W = (g[6] * c.x + g[7] * c.y) + g[8];
    const float ex = X - c.z * W, ey = Y - c.w * W, tw = t * W;
    return (W > 0.f && ex * ex + ey * ey <= tw * tw) ? 1 : 0;
  }
  const float ex = X - c.z, ey = Y - c.w;
  return (ex * ex + ey * ey <= t * t) ? 1 : 0;
}

// the scoring kernel's inlier tests of the similarity and affine map (PERSP false) and the homography (true)
template <bool PERSP>
struct MotionTest {
  static __device__ __forceinline__ int inlier(const float* g, float4 c, float t) { return motion_inlier<PERSP>(g, c, t); }
};

// ---- 5. refits and the model -------------------------------------------------------------------------------------------
template <int MODEL>
__global__ void __launch_bounds__(kRefitThreads) motion_refit_kernel(MotionGeom mg, MotionWork ws) {
  constexpr int N = MODEL + 1, K = 2 * N, NE = K * (K + 1) / 2 + K;
  __shared__ double model[K];
  __shared__ float gs[9];
  __shared__ int count, stop, refits;
  const int k = blockIdx.x;
  const int m = ws.m[k];
  const unsigned long long key = ws.key[k];
  MotionOut* out = ws.out + k;
  const int status = m < N ? 1 : key == 0ull ? 2 : 0;
  if (status) {
    if (threadIdx.x == 0) {
      for (int i = 0; i < 9; ++i) out->M[i] = __longlong_as_double(0x7ff8000000000000ll);
      out->st = ofdis_motion_stats{status, m, -1, 0, 0, 0};
    }
    return;
  }
  const int best = (int)(0xFFFFFFFFu - (unsigned)key);
  if (threadIdx.x == 0) {
    const double* hp = ws.hp + ((size_t)k * mg.hyp_cap + best) * 8;
    for (int i = 0; i < K; ++i) model[i] = hp[i];
    refits = 0;
  }
  const float4* corr = ws.corr + (size_t)k * mg.cell_cap;
  double* chunk = ws.chunk + (size_t)k * mg.chunk_cap * MOTION_NE;
  const int nc = (m + kChunk - 1) / kChunk;
  int P = 1;
  while (P < nc) P <<= 1;
  for (int r = 0;; ++r) {
    if (threadIdx.x == 0) {
      double H[9];
      motion_hmat<MODEL>(model, H);
      for (int i = 0; i < 9; ++i) gs[i] = (float)H[i];
      count = 0;
      stop = 0;
    }
    __syncthreads();
    float g[9];
    for (int i = 0; i < 9; ++i) g[i] = gs[i];
    const bool acc = r < mg.refine;
    int local = 0;
    for (int ch = threadIdx.x; ch < nc; ch += kRefitThreads) {
      double s[NE];
#pragma unroll
      for (int e = 0; e < NE; ++e) s[e] = 0.0;
      const int end = min(m, (ch + 1) * kChunk);
      for (int i = ch * kChunk; i < end; ++i) {
        const float4 c = corr[i];
        if (!motion_inlier<MODEL == OFDIS_MOTION_HOMOGRAPHY>(g, c, mg.t)) continue;  // adds +0.0: no change
        ++local;
        if (!acc) continue;
        double r1[K], r2[K], b1, b2;
        motion_rows<MODEL>(c, r1, r2, b1, b2);
        int e = 0;
#pragma unroll
        for (int a = 0; a < K; ++a)
#pragma unroll
          for (int bb = a; bb < K; ++bb) s[e] = s[e] + ((r1[a] * r1[bb]) + (r2[a] * r2[bb])), ++e;
#pragma unroll
        for (int a = 0; a < K; ++a) s[e] = s[e] + ((r1[a] * b1) + (r2[a] * b2)), ++e;
      }
      if (acc) {
#pragma unroll
        for (int e = 0; e < NE; ++e) chunk[(size_t)ch * MOTION_NE + e] = s[e];
      }
    }
    atomicAdd(&count, local);
    __syncthreads();
    if (!acc || count < N) break;  // uniform: every thread reads the same shared values
    // the pairwise tree over the chunk sums, padded with +0.0 to P leaves, in place: v_j += v_(j + stride)
    for (int stride = 1; stride < P; stride <<= 1) {
      for (int j = threadIdx.x * 2 * stride; j < nc; j += kRefitThreads * 2 * stride) {
        const int o = j + stride;
        for (int e = 0; e < NE; ++e)
          chunk[(size_t)j * MOTION_NE + e] = chunk[(size_t)j * MOTION_NE + e] + (o < nc ? chunk[(size_t)o * MOTION_NE + e] : 0.0);
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      double A[K][K], b[K], x[K];
      int e = 0;
      for (int a = 0; a < K; ++a)
        for (int bb = a; bb < K; ++bb) A[a][bb] = A[bb][a] = chunk[e++];
      for (int a = 0; a < K; ++a) b[a] = chunk[e++];
      if (motion_solve<K>(A, b, x)) {
        for (int a = 0; a < K; ++a) model[a] = x[a];
        ++refits;
      } else {
        stop = 1;
      }
    }
    __syncthreads();
    if (stop) break;
  }
  if (threadIdx.x == 0) {
    double H[9], A[9], M[9];
    motion_hmat<MODEL>(model, H);
    const double S = (double)mg.sigma, Cx = (double)mg.cx, Cy = (double)mg.cy;
    for (int rr = 0; rr < 3; ++rr) {
      A[3 * rr] = H[3 * rr] * S;
      A[3 * rr + 1] = H[3 * rr + 1] * S;
      A[3 * rr + 2] = H[3 * rr + 2] - (A[3 * rr] * Cx + A[3 * rr + 1] * Cy);
    }
    for (int c = 0; c < 3; ++c) {
      M[c] = A[c] / S + Cx * A[6 + c];
      M[3 + c] = A[3 + c] / S + Cy * A[6 + c];
      M[6 + c] = A[6 + c];
    }
    if (MODEL == OFDIS_MOTION_HOMOGRAPHY) {
      const double d = M[8];
      for (int i = 0; i < 9; ++i) M[i] = M[i] / d;
    }
    for (int i = 0; i < 9; ++i) out->M[i] = isnan(M[i]) ? __longlong_as_double(0x7ff8000000000000ll) : M[i];
    out->st = ofdis_motion_stats{0, m, best, (int)(key >> 32), refits, count};
  }
}

// ---- 6. per-pixel outputs -----------------------------------------------------------------------------------------------
template <int NOC>
__global__ void __launch_bounds__(256) motion_apply_kernel(LevelGeom g, int fa, int fb, MotionGeom mg, MotionWork ws,
                                                           MotionOutputs o) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y, k = blockIdx.z;
  const int w = mg.w, h = mg.h;
  if (X >= w || Y >= h) return;
  const size_t px = (size_t)k * w * h + (size_t)Y * w + X;
  const MotionOut& mo = ws.out[k];
  float rx = __int_as_float(0x7fc00000), ry = rx;
  unsigned char mask = 2, reg[NOC];
  for (int c = 0; c < NOC; ++c) reg[c] = 0;
  if (mo.st.status == 0) {
    float m[9];
    for (int i = 0; i < 9; ++i) m[i] = (float)mo.M[i];
    const float fX = (float)X, fY = (float)Y;
    const float mx = (m[0] * fX + m[1] * fY) + m[2], my = (m[3] * fX + m[4] * fY) + m[5];
    const float wq = (m[6] * fX + m[7] * fY) + m[8];
    const float xw = mx / wq, yw = my / wq;
    const float* F = g.flow + (size_t)frame_of(g, fa, k) * g.flow_frame_stride;
    float f[2] = {0.f, 0.f};
    upsample_at<2>(g, F, X, Y, mg.crop_x, mg.crop_y, [&f](int ch, float v) { f[ch] = v; });
    rx = f[0] - (xw - fX);
    ry = f[1] - (yw - fY);
    rx = isnan(rx) ? __int_as_float(0x7fc00000) : rx;  // every NaN written is the qNaN
    ry = isnan(ry) ? __int_as_float(0x7fc00000) : ry;
    bool known = fabsf(f[0]) <= 1e9f && fabsf(f[1]) <= 1e9f && in_frame_f(fX + f[0], fY + f[1], w, h);
    if (known && mg.fb_check) {
      const float* B = g.flow + (size_t)frame_of(g, fb, k) * g.flow_frame_stride;
      consistency_at<2>(g, B, f, X, Y, w, h, mg.crop_x, mg.crop_y, mg.alpha, mg.beta,
                        [&known](unsigned char cm, float) { known = cm == 0; });
    }
    mask = !known ? 2 : (rx * rx + ry * ry <= mg.thr * mg.thr) ? 0 : 1;
    if (o.registered && wq > 0.f && in_frame_f(xw, yw, w, h)) {
      float v[NOC];
      bil_u8<NOC>(o.i1 + k * o.stride, w, h, xw, yw, v);
      for (int c = 0; c < NOC; ++c) reg[c] = round_u8(v[c]);
    }
  }
  if (o.residual) {
    o.residual[2 * px] = rx;
    o.residual[2 * px + 1] = ry;
  }
  if (o.mask) o.mask[px] = mask;
  if (o.registered)
    for (int c = 0; c < NOC; ++c) o.registered[px * NOC + c] = reg[c];
}

template <int MODEL>
int launch_model(const MotionGeom& mg, const MotionWork& ws, int n, cudaStream_t st) {
  motion_hyp_kernel<MODEL><<<dim3((mg.nh + kHypThreads - 1) / kHypThreads, n), kHypThreads, 0, st>>>(mg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  if (launch_motion_score<MotionTest<MODEL == OFDIS_MOTION_HOMOGRAPHY>>(mg, ws, n, st) < 0) return -1;
  motion_refit_kernel<MODEL><<<n, kRefitThreads, 0, st>>>(mg, ws);
  return cudaGetLastError() == cudaSuccess ? 3 : -1;
}

}  // namespace

int launch_motion_corr(const LevelGeom& g, int fa, int fb, int n, const MotionGeom& mg, const MotionWork& ws,
                       cudaStream_t st) {
  const dim3 cgrid((mg.cells + kCorrThreads - 1) / kCorrThreads, n);
  if (mg.fb_check) motion_corr_kernel<true><<<cgrid, kCorrThreads, 0, st>>>(g, fa, fb, mg, ws);
  else motion_corr_kernel<false><<<cgrid, kCorrThreads, 0, st>>>(g, fa, fb, mg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  motion_compact_kernel<<<n, kCompactThreads, 0, st>>>(mg, ws);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_global_motion(const LevelGeom& g, int fa, int fb, int n, const MotionGeom& mg, const MotionWork& ws,
                         const MotionOutputs& o, cudaStream_t st) {
  if (g.nop != 2 || (mg.noc != 1 && mg.noc != 3)) return -1;
  if (launch_motion_corr(g, fa, fb, n, mg, ws, st) < 0) return -1;
  const int l = mg.model == OFDIS_MOTION_SIMILARITY ? launch_model<OFDIS_MOTION_SIMILARITY>(mg, ws, n, st)
                : mg.model == OFDIS_MOTION_AFFINE   ? launch_model<OFDIS_MOTION_AFFINE>(mg, ws, n, st)
                                                    : launch_model<OFDIS_MOTION_HOMOGRAPHY>(mg, ws, n, st);
  if (l < 0) return -1;
  if (!o.mask && !o.residual && !o.registered) return 2 + l;
  const dim3 block(32, 8), grid((mg.w + 31) / 32, (mg.h + 7) / 8, n);
  if (mg.noc == 3) motion_apply_kernel<3><<<grid, block, 0, st>>>(g, fa, fb, mg, ws, o);
  else motion_apply_kernel<1><<<grid, block, 0, st>>>(g, fa, fb, mg, ws, o);
  return cudaGetLastError() == cudaSuccess ? 3 + l : -1;
}

}  // namespace ofdis

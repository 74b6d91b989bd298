// Stereo ego-motion from flows and disparities (ofdis_egomotion_fullres; the header states the contract,
// preprocess.egomotion restates it bit for bit).  A fixed number of launches per call, whatever the number of pairs:
//   ego_corr_kernel     one thread per (cell, pair): validity, P (scene flow's xyz) and the observation (xs, ys, d1);
//   ego_compact_kernel  one CTA per pair: a block scan over the cells in tiles, compacting in place in cell order;
//   ego_hyp_kernel      one thread per (hypothesis, pair): three draws, the closed-form triad fit in float64;
//   ego_score_kernel    the hot path: the pair's 32-byte correspondences stream through shared memory in 64 KB tiles
//                       (cp.async.bulk + mbarrier, two buffers); each warp keeps 4 hypotheses' 12 floats in registers,
//                       tests them against every correspondence it reads and takes one 64-bit atomicMax per hypothesis;
//   ego_refit_kernel    one CTA per pair: every Gauss-Newton round (inlier test, chunk sums, tree, solve, update);
//   ego_apply_kernel    one thread per pixel: mask, residual flow and object motion (only when asked for).
// The flows are read through upsample_at / consistency_at; no full-resolution copy is stored.  float32 and float64
// without contraction (-fmad=false), IEEE division and square root.
#include <cuda_runtime.h>

#include "bulk_tile.cuh"
#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

using namespace tiles;

constexpr int kCorrThreads = 256;
constexpr int kCompactThreads = 1024;
constexpr int kHypThreads = 128;
constexpr int kScoreWarps = 16, kScoreHpw = 4, kScoreHpb = kScoreWarps * kScoreHpw;  // hypotheses per warp / CTA
constexpr int kTile = 2048;                                                          // EgoCorr per 64 KB tile
constexpr size_t kScoreSmem = 2 * kTile * sizeof(EgoCorr) + 16;                      // two tiles, two mbarriers
constexpr int kRefitThreads = 256;
constexpr int kChunk = 32;

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }
__device__ __forceinline__ float canon(float v) { return isnan(v) ? qnan() : v; }

// Step 1 of the header at pixel (px, py) of pair k: returns whether it is a valid correspondence; fills P, the target,
// d0, d1 and s1 (s0 > 0 tells whether P is usable).
struct EgoPixel {
  float f[2], xs, ys, d0, d1, s0, s1, X, Y, Z;
  bool usable0;  // d0 known and s0 > 0: P is defined
};
template <bool FB>
__device__ __forceinline__ bool ego_pixel(const LevelGeom& g, int fa, int fb, int k, const EgoGeom& eg, int px, int py,
                                          EgoPixel& e) {
  const float* F = g.flow + (size_t)frame_of(g, fa, k) * g.flow_frame_stride;
  upsample_at<2>(g, F, px, py, eg.crop_x, eg.crop_y, [&e](int ch, float v) { e.f[ch] = v; });
  const float* D0 = eg.disp0 + (size_t)k * eg.stride;
  const float* D1 = eg.disp1 + (size_t)k * eg.stride;
  e.d0 = D0[(size_t)py * eg.w + px];
  e.xs = (float)px + e.f[0];
  e.ys = (float)py + e.f[1];
  const bool in = in_frame_f(e.xs, e.ys, eg.w, eg.h);
  e.d1 = in ? sf_d1_at(D1, e.xs, e.ys, eg.w, eg.h, eg.edge_diff) : qnan();
  const DispCamera& c = eg.cam;
  e.s0 = e.d0 + c.doffs;
  e.s1 = e.d1 + c.doffs;
  e.usable0 = known_d(e.d0) && e.s0 > 0.0f;
  e.Z = c.fb / e.s0;
  e.X = (((float)px - c.cx) * e.Z) / c.fx;
  e.Y = (((float)py - c.cy) * e.Z) / c.fy;
  bool ok = e.usable0 && in && known_d(e.d1) && e.s1 > 0.0f;
  if (FB && ok) {
    const float* B = g.flow + (size_t)frame_of(g, fb, k) * g.flow_frame_stride;
    consistency_at<2>(g, B, e.f, px, py, eg.w, eg.h, eg.crop_x, eg.crop_y, eg.alpha, eg.beta,
                      [&ok](unsigned char mask, float) { ok = mask == 0; });
  }
  return ok;
}

// the t+1 point Q of an observation (scene flow's X1, Y1, Z1)
__device__ __forceinline__ void ego_q(const DispCamera& c, float xs, float ys, float s1, float& X1, float& Y1,
                                      float& Z1) {
  Z1 = c.fb / s1;
  X1 = ((xs - c.cx) * Z1) / c.fx;
  Y1 = ((ys - c.cy) * Z1) / c.fy;
}

// P' = g P (float32) and the inlier test of the header
__device__ __forceinline__ void ego_transform(const float* g, float X, float Y, float Z, float& Xp, float& Yp,
                                              float& Zp) {
  Xp = ((g[0] * X + g[1] * Y) + g[2] * Z) + g[3];
  Yp = ((g[4] * X + g[5] * Y) + g[6] * Z) + g[7];
  Zp = ((g[8] * X + g[9] * Y) + g[10] * Z) + g[11];
}
__device__ __forceinline__ int ego_inlier(const float* g, const EgoCorr& c, const DispCamera& cam, float thr) {
  float Xp, Yp, Zp;
  ego_transform(g, c.a.x, c.a.y, c.a.z, Xp, Yp, Zp);
  const float ex = (cam.fx * Xp + cam.cx * Zp) - c.a.w * Zp;
  const float ey = (cam.fy * Yp + cam.cy * Zp) - c.b.x * Zp;
  const float ed = cam.fb - c.b.z * Zp;
  const float tz = thr * Zp;
  return (Zp > 0.f && (ex * ex + ey * ey) + ed * ed <= tz * tz) ? 1 : 0;
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
// the orthonormal triad (e1, e2, n) of three points; false when a length is not > 0
__device__ __forceinline__ bool ego_triad(const double (&A)[3], const double (&B)[3], const double (&C)[3],
                                          double (&T)[3][3]) {
  double u[3], v[3], n[3];
  for (int i = 0; i < 3; ++i) u[i] = B[i] - A[i], v[i] = C[i] - A[i];
  const double L = sqrt((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]);
  for (int i = 0; i < 3; ++i) T[0][i] = u[i] / L;
  cross3(T[0], v, n);
  const double Ln = sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
  for (int i = 0; i < 3; ++i) T[2][i] = n[i] / Ln;
  cross3(T[2], T[0], T[1]);
  return L > 0.0 && Ln > 0.0;
}

// ---- 1. correspondences ------------------------------------------------------------------------------------------
template <bool FB>
__global__ void __launch_bounds__(kCorrThreads) ego_corr_kernel(LevelGeom g, int fa, int fb, EgoGeom eg, EgoWork ws) {
  const int c = blockIdx.x * kCorrThreads + threadIdx.x, k = blockIdx.y;
  if (c >= eg.cells) return;
  const int px = min((c % eg.ncx) * eg.s + eg.s / 2, eg.w - 1), py = min((c / eg.ncx) * eg.s + eg.s / 2, eg.h - 1);
  EgoPixel e;
  const bool ok = ego_pixel<FB>(g, fa, fb, k, eg, px, py, e);
  const size_t o = (size_t)k * eg.cell_cap + c;
  ws.flag[o] = ok ? 1 : 0;
  if (ok) {
    ws.corr[o].a = make_float4(e.X, e.Y, e.Z, e.xs);
    ws.corr[o].b = make_float4(e.ys, e.d1, e.s1, 0.f);
  }
}

// ---- 2. compaction (integer offsets only, so the order is the cell order) ------------------------------------------
__global__ void __launch_bounds__(kCompactThreads) ego_compact_kernel(EgoGeom eg, EgoWork ws) {
  __shared__ int warp_off[kCompactThreads / 32], tile_total;
  const int k = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  EgoCorr* corr = ws.corr + (size_t)k * eg.cell_cap;
  const unsigned char* flag = ws.flag + (size_t)k * eg.cell_cap;
  int base = 0;
  for (int t0 = 0; t0 < eg.cells; t0 += kCompactThreads) {
    const int c = t0 + threadIdx.x;
    const bool f = c < eg.cells && flag[c];
    EgoCorr v{};
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
__global__ void __launch_bounds__(kHypThreads) ego_hyp_kernel(EgoGeom eg, EgoWork ws) {
  const int h = blockIdx.x * kHypThreads + threadIdx.x, k = blockIdx.y;
  if (h >= eg.nh) return;
  const int m = ws.m[k];
  EgoHyp rec{};
  double M[12];
  bool ok = false;
  if (m >= 3) {
    const EgoCorr* corr = ws.corr + (size_t)k * eg.cell_cap;
    double P[3][3], Q[3][3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const unsigned idx = motion_draw(eg.seed, h, d, m);
      const EgoCorr c = corr[idx];
      float X1, Y1, Z1;
      ego_q(eg.cam, c.a.w, c.b.x, c.b.z, X1, Y1, Z1);
      P[d][0] = c.a.x, P[d][1] = c.a.y, P[d][2] = c.a.z;
      Q[d][0] = X1, Q[d][1] = Y1, Q[d][2] = Z1;
    }
    double E[3][3], G[3][3];
    ok = ego_triad(P[0], P[1], P[2], E);
    ok = ego_triad(Q[0], Q[1], Q[2], G) && ok;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) M[4 * i + j] = ((G[0][i] * E[0][j]) + (G[1][i] * E[1][j])) + (G[2][i] * E[2][j]);
    double cP[3], cQ[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      cP[i] = ((P[0][i] + P[1][i]) + P[2][i]) / 3.0;
      cQ[i] = ((Q[0][i] + Q[1][i]) + Q[2][i]) / 3.0;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
      M[4 * i + 3] = cQ[i] - (((M[4 * i] * cP[0]) + (M[4 * i + 1] * cP[1])) + (M[4 * i + 2] * cP[2]));
#pragma unroll
    for (int i = 0; i < 12; ++i) ok = ok && isfinite(M[i]);
  }
  double* hp = ws.hp + ((size_t)k * eg.hyp_cap + h) * 12;
  if (ok) {
#pragma unroll
    for (int i = 0; i < 12; ++i) {
      hp[i] = M[i];
      rec.g[i] = (float)M[i];
    }
  }
  rec.ok = ok ? 1 : 0;
  ws.hg[(size_t)k * eg.hyp_cap + h] = rec;
}

// ---- 4. scoring (the hot path) ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kScoreWarps * 32, 1) ego_score_kernel(EgoGeom eg, EgoWork ws) {
  extern __shared__ __align__(16) EgoCorr etiles[];  // [2][kTile], then two mbarriers
  const int k = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int m = ws.m[k];
  if (m < 3) return;  // no hypothesis was solved (uniform over the CTA)
  const int h0 = blockIdx.x * kScoreHpb + warp * kScoreHpw;
  float g[kScoreHpw][12];
  bool ok[kScoreHpw];
#pragma unroll
  for (int i = 0; i < kScoreHpw; ++i) {
    const int h = h0 + i;
    ok[i] = false;
#pragma unroll
    for (int e = 0; e < 12; ++e) g[i][e] = 0.f;
    if (h < eg.nh) {
      const EgoHyp& r = ws.hg[(size_t)k * eg.hyp_cap + h];
      ok[i] = r.ok != 0;
#pragma unroll
      for (int e = 0; e < 12; ++e) g[i][e] = r.g[e];
    }
  }
  const unsigned buf0 = smem_u32(etiles), mbar0 = buf0 + 2u * kTile * sizeof(EgoCorr);
  const EgoCorr* src = ws.corr + (size_t)k * eg.cell_cap;
  const int ntiles = (m + kTile - 1) / kTile;
  auto issue = [&](int t) {
    const int cnt = min(kTile, m - t * kTile);
    bulk_tile(buf0 + (unsigned)(t & 1) * kTile * sizeof(EgoCorr), src + (size_t)t * kTile,
              (unsigned)cnt * (unsigned)sizeof(EgoCorr), mbar0 + 8u * (t & 1));
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
  const DispCamera cam = eg.cam;
  const float thr = eg.thr;
  for (int tt = 0; tt < ntiles; ++tt) {
    const int b = tt & 1;
    mbar_wait(mbar0 + 8u * b, (unsigned)(tt >> 1) & 1u);
    const EgoCorr* tile = etiles + b * kTile;
    const int n_in = min(kTile, m - tt * kTile);
#pragma unroll 2
    for (int e = lane; e < n_in; e += 32) {
      const EgoCorr c = tile[e];
#pragma unroll
      for (int i = 0; i < kScoreHpw; ++i) cnt[i] += ego_inlier(g[i], c, cam, thr);
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

// ---- 5. Gauss-Newton refits and the pose --------------------------------------------------------------------------------
// the three residuals of one inlier and their Jacobian rows (omega, tau) at P' = R P + t (float64)
__device__ __forceinline__ void ego_rows(const double* M, const EgoCorr& c, const DispCamera& cam, double (&J)[3][6],
                                         double (&r)[3]) {
  const double X = c.a.x, Y = c.a.y, Z = c.a.z;
  double Pp[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) Pp[i] = (((M[4 * i] * X) + (M[4 * i + 1] * Y)) + (M[4 * i + 2] * Z)) + M[4 * i + 3];
  const double fx = cam.fx, fy = cam.fy, cx = cam.cx, cy = cam.cy, fb = cam.fb, doffs = cam.doffs;
  const double iz = 1.0 / Pp[2], u = Pp[0] * iz, v = Pp[1] * iz;
  const double ax[3] = {fx * iz, 0.0, -((fx * iz) * u)};
  const double ay[3] = {0.0, fy * iz, -((fy * iz) * v)};
  const double ad[3] = {0.0, 0.0, -((fb * iz) * iz)};
  r[0] = ((fx * u) + cx) - (double)c.a.w;
  r[1] = ((fy * v) + cy) - (double)c.b.x;
  r[2] = ((fb * iz) - doffs) - (double)c.b.y;
  const double w0 = 2.0 * Pp[0], w1 = 2.0 * Pp[1], w2 = 2.0 * Pp[2];
  const double* a[3] = {ax, ay, ad};
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    J[q][0] = (a[q][1] * -w2) + (a[q][2] * w1);
    J[q][1] = (a[q][0] * w2) + (a[q][2] * -w0);
    J[q][2] = (a[q][0] * -w1) + (a[q][1] * w0);
    J[q][3] = a[q][0];
    J[q][4] = a[q][1];
    J[q][5] = a[q][2];
  }
}

__global__ void __launch_bounds__(kRefitThreads) ego_refit_kernel(EgoGeom eg, EgoWork ws) {
  __shared__ double model[12];
  __shared__ float gs[12];
  __shared__ int count, stop, refits;
  const int k = blockIdx.x;
  const int m = ws.m[k];
  const unsigned long long key = ws.key[k];
  EgoOut* out = ws.out + k;
  const int status = m < 3 ? 1 : key == 0ull ? 2 : 0;
  if (status) {
    if (threadIdx.x == 0) {
      for (int i = 0; i < 12; ++i) out->pose[i] = __longlong_as_double(0x7ff8000000000000ll);
      out->st = ofdis_motion_stats{status, m, -1, 0, 0, 0};
    }
    return;
  }
  const int best = (int)(0xFFFFFFFFu - (unsigned)key);
  if (threadIdx.x == 0) {
    const double* hp = ws.hp + ((size_t)k * eg.hyp_cap + best) * 12;
    for (int i = 0; i < 12; ++i) model[i] = hp[i];
    refits = 0;
  }
  const EgoCorr* corr = ws.corr + (size_t)k * eg.cell_cap;
  double* chunk = ws.chunk + (size_t)k * eg.chunk_cap * EGO_NE;
  const int nc = (m + kChunk - 1) / kChunk;
  int P = 1;
  while (P < nc) P <<= 1;
  const DispCamera cam = eg.cam;
  for (int r = 0;; ++r) {
    if (threadIdx.x == 0) {
      for (int i = 0; i < 12; ++i) gs[i] = (float)model[i];
      count = 0;
      stop = 0;
    }
    __syncthreads();
    float g[12];
    double M[12];
    for (int i = 0; i < 12; ++i) g[i] = gs[i], M[i] = model[i];
    const bool acc = r < eg.refine;
    int local = 0;
    for (int ch = threadIdx.x; ch < nc; ch += kRefitThreads) {
      double s[EGO_NE];
#pragma unroll
      for (int e = 0; e < EGO_NE; ++e) s[e] = 0.0;
      const int end = min(m, (ch + 1) * kChunk);
      for (int i = ch * kChunk; i < end; ++i) {
        const EgoCorr c = corr[i];
        if (!ego_inlier(g, c, cam, eg.thr)) continue;  // adds +0.0: no change
        ++local;
        if (!acc) continue;
        double J[3][6], rr[3];
        ego_rows(M, c, cam, J, rr);
        int e = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
          for (int bb = a; bb < 6; ++bb)
            s[e] = s[e] + (((J[0][a] * J[0][bb]) + (J[1][a] * J[1][bb])) + (J[2][a] * J[2][bb])), ++e;
#pragma unroll
        for (int a = 0; a < 6; ++a) s[e] = s[e] + -(((J[0][a] * rr[0]) + (J[1][a] * rr[1])) + (J[2][a] * rr[2])), ++e;
      }
      if (acc) {
#pragma unroll
        for (int e = 0; e < EGO_NE; ++e) chunk[(size_t)ch * EGO_NE + e] = s[e];
      }
    }
    atomicAdd(&count, local);
    __syncthreads();
    if (!acc || count < 3) break;  // uniform: every thread reads the same shared values
    refit_tree<EGO_NE>(chunk, nc, P, kRefitThreads);
    if (threadIdx.x == 0) {
      double A[6][6], b[6], x[6];
      int e = 0;
      for (int a = 0; a < 6; ++a)
        for (int bb = a; bb < 6; ++bb) A[a][bb] = A[bb][a] = chunk[e++];
      for (int a = 0; a < 6; ++a) b[a] = chunk[e++];
      if (motion_solve<6>(A, b, x)) {
        // the Cayley rotation C(omega) = ((1 - |w|^2) I + 2 w w^T + 2 [w]x) / (1 + |w|^2), then R <- C R, t <- C t + tau
        const double q = (x[0] * x[0] + x[1] * x[1]) + x[2] * x[2], dg = 1.0 - q, dn = 1.0 + q;
        const double K[3][3] = {{0.0, -x[2], x[1]}, {x[2], 0.0, -x[0]}, {-x[1], x[0], 0.0}};
        double C[3][3], Mn[12];
        for (int i = 0; i < 3; ++i)
          for (int j = 0; j < 3; ++j) C[i][j] = (((i == j ? dg : 0.0) + (2.0 * (x[i] * x[j]))) + (2.0 * K[i][j])) / dn;
        for (int i = 0; i < 3; ++i) {
          for (int j = 0; j < 4; ++j)
            Mn[4 * i + j] = ((C[i][0] * model[j]) + (C[i][1] * model[4 + j])) + (C[i][2] * model[8 + j]);
          Mn[4 * i + 3] = Mn[4 * i + 3] + x[3 + i];
        }
        for (int i = 0; i < 12; ++i) model[i] = Mn[i];
        ++refits;
      } else {
        stop = 1;
      }
    }
    __syncthreads();
    if (stop) break;
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < 12; ++i)
      out->pose[i] = isnan(model[i]) ? __longlong_as_double(0x7ff8000000000000ll) : model[i];
    out->st = ofdis_motion_stats{0, m, best, (int)(key >> 32), refits, count};
  }
}

// ---- 6. per-pixel outputs -----------------------------------------------------------------------------------------------
template <bool FB>
__global__ void __launch_bounds__(256) ego_apply_kernel(LevelGeom g, int fa, int fb, EgoGeom eg, EgoWork ws,
                                                        EgoOutputs o) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y, k = blockIdx.z;
  if (X >= eg.w || Y >= eg.h) return;
  const size_t px = (size_t)k * eg.w * eg.h + (size_t)Y * eg.w + X;
  const EgoOut& eo = ws.out[k];
  float rx = qnan(), ry = qnan(), om[3] = {qnan(), qnan(), qnan()};
  unsigned char mask = 2;
  if (eo.st.status == 0) {
    float gp[12];
    for (int i = 0; i < 12; ++i) gp[i] = (float)eo.pose[i];
    EgoPixel e;
    const bool valid = ego_pixel<FB>(g, fa, fb, k, eg, X, Y, e);
    float Xp, Yp, Zp;
    ego_transform(gp, e.X, e.Y, e.Z, Xp, Yp, Zp);
    const DispCamera& c = eg.cam;
    if (e.usable0) {
      const float xi = (c.fx * Xp) / Zp + c.cx, yi = (c.fy * Yp) / Zp + c.cy;
      rx = canon(e.f[0] - (xi - (float)X));
      ry = canon(e.f[1] - (yi - (float)Y));
    }
    if (valid && Zp > 0.f) {
      EgoCorr cc;
      cc.a = make_float4(e.X, e.Y, e.Z, e.xs);
      cc.b = make_float4(e.ys, e.d1, e.s1, 0.f);
      mask = ego_inlier(gp, cc, c, eg.thr) ? 0 : 1;
      float X1, Y1, Z1;
      ego_q(c, e.xs, e.ys, e.s1, X1, Y1, Z1);
      om[0] = canon(X1 - Xp);
      om[1] = canon(Y1 - Yp);
      om[2] = canon(Z1 - Zp);
    }
  }
  if (o.mask) o.mask[px] = mask;
  if (o.residual) {
    o.residual[2 * px] = rx;
    o.residual[2 * px + 1] = ry;
  }
  if (o.object_motion) {
    o.object_motion[3 * px] = om[0];
    o.object_motion[3 * px + 1] = om[1];
    o.object_motion[3 * px + 2] = om[2];
  }
}

}  // namespace

int launch_egomotion(const LevelGeom& g, int fa, int fb, int n, const EgoGeom& eg, const EgoWork& ws,
                     const EgoOutputs& o, cudaStream_t st) {
  if (g.nop != 2) return -1;
  const dim3 cgrid((eg.cells + kCorrThreads - 1) / kCorrThreads, n);
  if (eg.fb_check) ego_corr_kernel<true><<<cgrid, kCorrThreads, 0, st>>>(g, fa, fb, eg, ws);
  else ego_corr_kernel<false><<<cgrid, kCorrThreads, 0, st>>>(g, fa, fb, eg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  ego_compact_kernel<<<n, kCompactThreads, 0, st>>>(eg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  ego_hyp_kernel<<<dim3((eg.nh + kHypThreads - 1) / kHypThreads, n), kHypThreads, 0, st>>>(eg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  if (smem_optin((const void*)ego_score_kernel, kScoreSmem, false) != cudaSuccess) return -1;
  ego_score_kernel<<<dim3((eg.nh + kScoreHpb - 1) / kScoreHpb, n), kScoreWarps * 32, kScoreSmem, st>>>(eg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  ego_refit_kernel<<<n, kRefitThreads, 0, st>>>(eg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  if (!o.mask && !o.residual && !o.object_motion) return 5;
  const dim3 block(32, 8), grid((eg.w + 31) / 32, (eg.h + 7) / 8, n);
  if (eg.fb_check) ego_apply_kernel<true><<<grid, block, 0, st>>>(g, fa, fb, eg, ws, o);
  else ego_apply_kernel<false><<<grid, block, 0, st>>>(g, fa, fb, eg, ws, o);
  return cudaGetLastError() == cudaSuccess ? 6 : -1;
}

}  // namespace ofdis

// Monocular relative pose from dense flows (ofdis_relpose_fullres; the header states the contract, preprocess.relpose
// restates it bit for bit).  A fixed number of launches per call, whatever the number of pairs:
//   motion_corr_kernel, motion_compact_kernel  global motion's, in pixel coordinates (launch_motion_corr);
//   relpose_hyp_kernel     one thread per (hypothesis, pair): eight draws, the 8 x 9 full-pivot elimination in float64,
//                          F = K^-T E K^-1 rounded to float32 as the hypothesis record;
//   motion_score_kernel    the hot path (motion_score.cuh) with the Sampson test;
//   relpose_refit_kernel   one CTA per pair: E's four (R, t), the cheirality vote, every Gauss-Newton round and the
//                          parallax guard;
//   relpose_apply_kernel   one thread per pixel: mask, Sampson distance and depth (only when asked for).
// float32 and float64 without contraction (-fmad=false), IEEE division and square root.
#include <cuda_runtime.h>

#include "motion_score.cuh"

namespace ofdis {

namespace {

constexpr int kHypThreads = 128;
constexpr int kRefitThreads = 256;
constexpr int kChunk = 32;
constexpr int kJacobiSweeps = 8;

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }
__device__ __forceinline__ double qnan64() { return __longlong_as_double(0x7ff8000000000000ll); }

// The Sampson test in pixels (step 3 of the header), F = g against the pixel correspondence c = (x, y, x', y'); the
// float32 quantities are returned for the per-pixel distance
__device__ __forceinline__ bool sampson_terms(const float* g, float4 c, float t, float& e, float& den) {
  const float a0 = (g[0] * c.x + g[1] * c.y) + g[2], a1 = (g[3] * c.x + g[4] * c.y) + g[5];
  const float a2 = (g[6] * c.x + g[7] * c.y) + g[8];
  const float b0 = (g[0] * c.z + g[3] * c.w) + g[6], b1 = (g[1] * c.z + g[4] * c.w) + g[7];
  e = (c.z * a0 + c.w * a1) + a2;
  den = (a0 * a0 + a1 * a1) + (b0 * b0 + b1 * b1);
  return e * e <= (t * t) * den;
}
struct SampsonTest {
  static __device__ __forceinline__ int inlier(const float* g, float4 c, float t) {
    float e, den;
    return sampson_terms(g, c, t, e, den) ? 1 : 0;
  }
};

// normalized coordinates of a pixel correspondence (float32): ((float)px - cx) / fx, ...
__device__ __forceinline__ void rp_norm(const RelposeGeom& rg, float4 c, float& x, float& y, float& xp, float& yp) {
  x = (c.x - rg.cx) / rg.fx;
  y = (c.y - rg.cy) / rg.fy;
  xp = (c.z - rg.cx) / rg.fx;
  yp = (c.w - rg.cy) / rg.fy;
}

// F = K^-T E K^-1 rounded to float32
__device__ __forceinline__ void rp_fmat(const RelposeGeom& rg, const double* E, float* g) {
  const double ifx = 1.0 / (double)rg.fx, ify = 1.0 / (double)rg.fy;
  const double ux = -((double)rg.cx * ifx), uy = -((double)rg.cy * ify);
  double G[9];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    G[3 * i] = E[3 * i] * ifx;
    G[3 * i + 1] = E[3 * i + 1] * ify;
    G[3 * i + 2] = ((E[3 * i] * ux) + (E[3 * i + 1] * uy)) + E[3 * i + 2];
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    g[j] = (float)(ifx * G[j]);
    g[3 + j] = (float)(ify * G[3 + j]);
    g[6 + j] = (float)(((ux * G[j]) + (uy * G[3 + j])) + G[6 + j]);
  }
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
__device__ __forceinline__ void unit3(double* a) {
  const double L = sqrt(dot3(a, a));
  for (int i = 0; i < 3; ++i) a[i] = a[i] / L;
}

// The null vector of the 8 x 9 system by full pivoting (step 2 of the header); false when a pivot is not > 0 or an
// entry of the unit vector is not finite
__device__ __forceinline__ bool rp_null(double (&A)[8][9], double (&e)[9]) {
  int perm[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) perm[c] = c;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    double best = -1.0;
    int pr = j, pc = j;
#pragma unroll
    for (int i = j; i < 8; ++i)
#pragma unroll
      for (int c = j; c < 9; ++c) {
        const double a = fabs(A[i][c]);
        if (a > best) best = a, pr = i, pc = c;
      }
    if (!(best > 0.0)) return false;
#pragma unroll
    for (int i = j + 1; i < 8; ++i)
      if (i == pr)
#pragma unroll
        for (int c = j; c < 9; ++c) {
          const double t = A[j][c];
          A[j][c] = A[i][c];
          A[i][c] = t;
        }
#pragma unroll
    for (int c = j + 1; c < 9; ++c)
      if (c == pc) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const double t = A[i][j];
          A[i][j] = A[i][c];
          A[i][c] = t;
        }
        const int t = perm[j];
        perm[j] = perm[c];
        perm[c] = t;
      }
#pragma unroll
    for (int i = j + 1; i < 8; ++i) {
      const double f = A[i][j] / A[j][j];
#pragma unroll
      for (int c = j + 1; c < 9; ++c) A[i][c] = A[i][c] - f * A[j][c];
    }
  }
  double y[9];
  y[8] = 1.0;
#pragma unroll
  for (int i = 7; i >= 0; --i) {
    double s = -A[i][8];
#pragma unroll
    for (int c = i + 1; c < 8; ++c) s = s - A[i][c] * y[c];
    y[i] = s / A[i][i];
  }
#pragma unroll
  for (int d = 0; d < 9; ++d) {
    e[d] = 0.0;
#pragma unroll
    for (int c = 0; c < 9; ++c)
      if (perm[c] == d) e[d] = y[c];
  }
  double n2 = 0.0;
#pragma unroll
  for (int d = 0; d < 9; ++d) n2 = n2 + e[d] * e[d];
  const double L = sqrt(n2);
  bool ok = true;
#pragma unroll
  for (int d = 0; d < 9; ++d) {
    e[d] = e[d] / L;
    ok = ok && isfinite(e[d]);
  }
  return ok;
}

// ---- hypotheses ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kHypThreads) relpose_hyp_kernel(RelposeGeom rg, MotionWork ws) {
  const MotionGeom& mg = rg.mg;
  const int h = blockIdx.x * kHypThreads + threadIdx.x, k = blockIdx.y;
  if (h >= mg.nh) return;
  const int m = ws.m[k];
  MotionHyp rec{};
  double e[9];
  bool ok = false;
  if (m >= 8) {
    const float4* corr = ws.corr + (size_t)k * mg.cell_cap;
    double A[8][9];
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      float xf, yf, xpf, ypf;
      rp_norm(rg, corr[motion_draw(mg.seed, h, d, m)], xf, yf, xpf, ypf);
      const double x = xf, y = yf, xp = xpf, yp = ypf;
      A[d][0] = xp * x, A[d][1] = xp * y, A[d][2] = xp;
      A[d][3] = yp * x, A[d][4] = yp * y, A[d][5] = yp;
      A[d][6] = x, A[d][7] = y, A[d][8] = 1.0;
    }
    ok = rp_null(A, e);
  }
  double* hp = ws.hp + ((size_t)k * mg.hyp_cap + h) * 9;
  if (ok) {
#pragma unroll
    for (int i = 0; i < 9; ++i) hp[i] = e[i];
    rp_fmat(rg, e, rec.g);
  }
  rec.ok = ok ? 1 : 0;
  ws.hg[(size_t)k * mg.hyp_cap + h] = rec;
}

// ---- refits ----------------------------------------------------------------------------------------------------------
// The four (R, t) of E (step 4 of the header): row-major R[q] (9) and t[q] (3), q = (R1, u3), (R1, -u3), (R2, u3),
// (R2, -u3)
__device__ void rp_decompose(const double* E, double (&R)[4][9], double (&T)[4][3]) {
  double S[3][3], V[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      S[i][j] = ((E[i] * E[j]) + (E[3 + i] * E[3 + j])) + (E[6 + i] * E[6 + j]);
      V[i][j] = i == j ? 1.0 : 0.0;
    }
#pragma unroll
  for (int sw = 0; sw < kJacobiSweeps; ++sw)
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      const double apq = S[p][q];
      if (apq == 0.0) continue;
      const double th = (S[q][q] - S[p][p]) / (2.0 * apq);
      double t = 1.0 / (fabs(th) + sqrt(th * th + 1.0));
      if (th < 0.0) t = -t;
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      for (int r = 0; r < 3; ++r) {
        const double a = S[r][p], b = S[r][q];
        S[r][p] = c * a - s * b;
        S[r][q] = s * a + c * b;
      }
      for (int r = 0; r < 3; ++r) {
        const double a = S[p][r], b = S[q][r];
        S[p][r] = c * a - s * b;
        S[q][r] = s * a + c * b;
      }
      for (int r = 0; r < 3; ++r) {
        const double a = V[r][p], b = V[r][q];
        V[r][p] = c * a - s * b;
        V[r][q] = s * a + c * b;
      }
    }
  // i1: the largest eigenvalue (first on a tie), i2: the larger of the other two (first on a tie)
  const double d0 = S[0][0], d1 = S[1][1], d2 = S[2][2];
  const int i1 = d1 > d0 ? (d2 > d1 ? 2 : 1) : (d2 > d0 ? 2 : 0);
  const int i2 = i1 == 0 ? (d2 > d1 ? 2 : 1) : i1 == 1 ? (d2 > d0 ? 2 : 0) : (d1 > d0 ? 1 : 0);
  double v1[3], v2[3], v3[3], u1[3], u2[3], u3[3], w[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    v1[i] = i1 == 0 ? V[i][0] : i1 == 1 ? V[i][1] : V[i][2];
    v2[i] = i2 == 0 ? V[i][0] : i2 == 1 ? V[i][1] : V[i][2];
  }
  unit3(v1);
  cross3(v1, v2, v3);
  unit3(v3);
  cross3(v3, v1, v2);
  for (int i = 0; i < 3; ++i) {
    u1[i] = ((E[3 * i] * v1[0]) + (E[3 * i + 1] * v1[1])) + (E[3 * i + 2] * v1[2]);
    w[i] = ((E[3 * i] * v2[0]) + (E[3 * i + 1] * v2[1])) + (E[3 * i + 2] * v2[2]);
  }
  unit3(u1);
  cross3(u1, w, u3);
  unit3(u3);
  cross3(u3, u1, u2);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double r1 = ((u2[i] * v1[j]) - (u1[i] * v2[j])) + (u3[i] * v3[j]);
      const double r2 = ((u1[i] * v2[j]) - (u2[i] * v1[j])) + (u3[i] * v3[j]);
      R[0][3 * i + j] = R[1][3 * i + j] = r1;
      R[2][3 * i + j] = R[3][3 * i + j] = r2;
    }
  for (int i = 0; i < 3; ++i) {
    T[0][i] = T[2][i] = u3[i];
    T[1][i] = T[3][i] = -u3[i];
  }
}

// y = R (x, y, 1)
__device__ __forceinline__ void rp_rot(const double* R, double x, double y, double* o) {
  for (int i = 0; i < 3; ++i) o[i] = ((R[3 * i] * x) + (R[3 * i + 1] * y)) + R[3 * i + 2];
}
// in front of both cameras: lambda0 = -((r1 x y).(r1 x t)) / |r1 x y|^2 > 0 and lambda0 y_2 + t_2 > 0
__device__ __forceinline__ bool rp_front(const double* y, const double* r1, const double* t) {
  double c1[3], c2[3];
  cross3(r1, y, c1);
  cross3(r1, t, c2);
  const double lam = -dot3(c1, c2) / dot3(c1, c1);
  return lam > 0.0 && lam * y[2] + t[2] > 0.0;
}

__global__ void __launch_bounds__(kRefitThreads) relpose_refit_kernel(RelposeGeom rg, MotionWork ws, RelposeOut* outs) {
  const MotionGeom& mg = rg.mg;
  __shared__ double Rs[9], ts[3], Es[9], B[2][3], Rw[9];
  __shared__ double cand_R[4][9], cand_t[4][3];
  __shared__ float gs[9];
  __shared__ int count, stop, refits, votes[4];
  const int k = blockIdx.x;
  const int m = ws.m[k];
  const unsigned long long key = ws.key[k];
  RelposeOut* out = outs + k;
  const int status = m < 8 ? 1 : key == 0ull ? 2 : 0;
  if (status) {
    if (threadIdx.x == 0) {
      for (int i = 0; i < 12; ++i) out->pose[i] = qnan64();
      out->st = ofdis_motion_stats{status, m, -1, 0, 0, 0};
    }
    return;
  }
  const int best = (int)(0xFFFFFFFFu - (unsigned)key);
  const float4* corr = ws.corr + (size_t)k * mg.cell_cap;
  if (threadIdx.x == 0) {
    double E[9], R[4][9], T[4][3];
    const double* hp = ws.hp + ((size_t)k * mg.hyp_cap + best) * 9;
    for (int i = 0; i < 9; ++i) E[i] = hp[i];
    rp_decompose(E, R, T);
    for (int q = 0; q < 4; ++q) {
      for (int i = 0; i < 9; ++i) cand_R[q][i] = R[q][i];
      for (int i = 0; i < 3; ++i) cand_t[q][i] = T[q][i];
      votes[q] = 0;
    }
    for (int i = 0; i < 9; ++i) gs[i] = ws.hg[(size_t)k * mg.hyp_cap + best].g[i];
    refits = 0;
  }
  __syncthreads();
  // the cheirality vote over the inliers of the best hypothesis
  {
    float g[9];
    for (int i = 0; i < 9; ++i) g[i] = gs[i];
    int local[4] = {0, 0, 0, 0};
    for (int i = threadIdx.x; i < m; i += kRefitThreads) {
      const float4 c = corr[i];
      if (!SampsonTest::inlier(g, c, mg.t)) continue;
      float xf, yf, xpf, ypf;
      rp_norm(rg, c, xf, yf, xpf, ypf);
      const double r1[3] = {xpf, ypf, 1.0};
      for (int q = 0; q < 4; ++q) {
        double y[3];
        rp_rot(cand_R[q], xf, yf, y);
        local[q] += rp_front(y, r1, cand_t[q]) ? 1 : 0;
      }
    }
    for (int q = 0; q < 4; ++q) atomicAdd(&votes[q], local[q]);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int qb = 0;
    for (int q = 1; q < 4; ++q)
      if (votes[q] > votes[qb]) qb = q;
    for (int i = 0; i < 9; ++i) Rs[i] = cand_R[qb][i];
    for (int i = 0; i < 3; ++i) ts[i] = cand_t[qb][i];
  }
  double* chunk = ws.chunk + (size_t)k * mg.chunk_cap * RELPOSE_NE;
  const int nc = (m + kChunk - 1) / kChunk;
  int P = 1;
  while (P < nc) P <<= 1;
  const double fx = rg.fx, fy = rg.fy, ifx = 1.0 / fx, ify = 1.0 / fy;
  for (int r = 0;; ++r) {
    if (threadIdx.x == 0) {
      // E = [t]x R, its F, and the tangent basis of t: b1 = unit(t x e_a) with a the first axis of the smallest |t_a|,
      // b2 = t x b1
      const double* t = ts;
      for (int j = 0; j < 3; ++j) {
        Es[j] = (-(t[2] * Rs[3 + j])) + (t[1] * Rs[6 + j]);
        Es[3 + j] = (t[2] * Rs[j]) - (t[0] * Rs[6 + j]);
        Es[6 + j] = (-(t[1] * Rs[j])) + (t[0] * Rs[3 + j]);
      }
      rp_fmat(rg, Es, gs);
      // the twisted pair of R, (2 t t^T - I) R: the other rotation that explains the same E
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
          double v = 0.0;
          for (int k2 = 0; k2 < 3; ++k2) v = v + ((2.0 * (t[i] * t[k2])) - (i == k2 ? 1.0 : 0.0)) * Rs[3 * k2 + j];
          Rw[3 * i + j] = v;
        }
      int a = 0;
      for (int i = 1; i < 3; ++i)
        if (fabs(t[i]) < fabs(t[a])) a = i;
      const double ea[3] = {a == 0 ? 1.0 : 0.0, a == 1 ? 1.0 : 0.0, a == 2 ? 1.0 : 0.0};
      double b1[3], b2[3];
      cross3(t, ea, b1);
      unit3(b1);
      cross3(t, b1, b2);
      for (int i = 0; i < 3; ++i) B[0][i] = b1[i], B[1][i] = b2[i];
      count = 0;
      stop = 0;
    }
    __syncthreads();
    float g[9];
    double R[9], t[3], E[9], b1[3], b2[3];
    for (int i = 0; i < 9; ++i) g[i] = gs[i], R[i] = Rs[i], E[i] = Es[i];
    for (int i = 0; i < 3; ++i) t[i] = ts[i], b1[i] = B[0][i], b2[i] = B[1][i];
    const bool acc = r < mg.refine;
    int local = 0;
    for (int ch = threadIdx.x; ch < nc; ch += kRefitThreads) {
      double s[RELPOSE_NE];
#pragma unroll
      for (int e = 0; e < RELPOSE_NE; ++e) s[e] = 0.0;
      const int end = min(m, (ch + 1) * kChunk);
      for (int i = ch * kChunk; i < end; ++i) {
        const float4 c = corr[i];
        if (!SampsonTest::inlier(g, c, mg.t)) continue;  // adds +0.0: no change
        ++local;
        float xf, yf, xpf, ypf;
        rp_norm(rg, c, xf, yf, xpf, ypf);
        const double x = xf, y = yf, xp = xpf, yp = ypf;
        const double z[3] = {xp, yp, 1.0};
        double Ry[3], a[3], b[3], zt[3], gw[3], yz[3], J[5];
        rp_rot(R, x, y, Ry);
        for (int q = 0; q < 3; ++q) {
          a[q] = ((E[3 * q] * x) + (E[3 * q + 1] * y)) + E[3 * q + 2];
          b[q] = ((E[q] * xp) + (E[3 + q] * yp)) + E[6 + q];
        }
        const double res = ((xp * a[0]) + (yp * a[1])) + a[2];
        const double s0 = a[0] * ifx, s1 = a[1] * ify, s2 = b[0] * ifx, s3 = b[1] * ify;
        const double wt = 1.0 / sqrt(((s0 * s0 + s1 * s1) + s2 * s2) + s3 * s3);
        const double rr = wt * res;
        cross3(z, t, zt);
        cross3(Ry, zt, gw);
        cross3(Ry, z, yz);
        for (int q = 0; q < 3; ++q) J[q] = wt * (2.0 * gw[q]);
        J[3] = wt * dot3(b1, yz);
        J[4] = wt * dot3(b2, yz);
        int e = 0;
#pragma unroll
        for (int p = 0; p < 5; ++p)
#pragma unroll
          for (int q = p; q < 5; ++q) s[e] = s[e] + (J[p] * J[q]), ++e;
#pragma unroll
        for (int p = 0; p < 5; ++p) s[e] = s[e] + -(J[p] * rr), ++e;
        const double dx = fx * (xp - Ry[0] / Ry[2]), dy = fy * (yp - Ry[1] / Ry[2]);
        s[e] = s[e] + sqrt(dx * dx + dy * dy), ++e;
        rp_rot(Rw, x, y, Ry);
        const double wx = fx * (xp - Ry[0] / Ry[2]), wy = fy * (yp - Ry[1] / Ry[2]);
        s[e] = s[e] + sqrt(wx * wx + wy * wy);
      }
#pragma unroll
      for (int e = 0; e < RELPOSE_NE; ++e) chunk[(size_t)ch * RELPOSE_NE + e] = s[e];
    }
    atomicAdd(&count, local);
    __syncthreads();
    refit_tree<RELPOSE_NE>(chunk, nc, P, kRefitThreads);
    if (!acc || count < 8) break;  // uniform: every thread reads the same shared values
    if (threadIdx.x == 0) {
      double A[5][5], bb[5], x[5];
      int e = 0;
      for (int p = 0; p < 5; ++p)
        for (int q = p; q < 5; ++q) A[p][q] = A[q][p] = chunk[e++];
      for (int p = 0; p < 5; ++p) bb[p] = chunk[e++];
      if (motion_solve<5>(A, bb, x)) {
        double C[3][3], Rn[9], tn[3];
        cayley(x, C);
        for (int i = 0; i < 3; ++i)
          for (int j = 0; j < 3; ++j) Rn[3 * i + j] = ((C[i][0] * Rs[j]) + (C[i][1] * Rs[3 + j])) + (C[i][2] * Rs[6 + j]);
        for (int i = 0; i < 3; ++i) tn[i] = (ts[i] + x[3] * B[0][i]) + x[4] * B[1][i];
        unit3(tn);
        for (int i = 0; i < 9; ++i) Rs[i] = Rn[i];
        for (int i = 0; i < 3; ++i) ts[i] = tn[i];
        ++refits;
      } else {
        stop = 1;
      }
    }
    __syncthreads();
    if (stop) break;
  }
  if (threadIdx.x == 0) {
    // the smaller derotated flow of R and its twisted pair: without translation one of them explains the flow alone
    const double pr = chunk[RELPOSE_NE - 2], pw = chunk[RELPOSE_NE - 1];
    const double parallax = (pw < pr ? pw : pr) / (double)count;
    const int st = parallax >= (double)rg.min_parallax ? 0 : 3;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) out->pose[4 * i + j] = st || isnan(Rs[3 * i + j]) ? qnan64() : Rs[3 * i + j];
      out->pose[4 * i + 3] = st || isnan(ts[i]) ? qnan64() : ts[i];
    }
    for (int i = 0; i < 9; ++i) out->g[i] = gs[i];
    out->st = ofdis_motion_stats{st, m, best, (int)(key >> 32), refits, count};
  }
}

// ---- per-pixel outputs -----------------------------------------------------------------------------------------------
template <bool FB>
__global__ void __launch_bounds__(256) relpose_apply_kernel(LevelGeom g, int fa, int fb, RelposeGeom rg,
                                                            const RelposeOut* outs, RelposeOutputs o) {
  const MotionGeom& mg = rg.mg;
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y, k = blockIdx.z;
  const int w = mg.w, h = mg.h;
  if (X >= w || Y >= h) return;
  const size_t px = (size_t)k * w * h + (size_t)Y * w + X;
  const RelposeOut& ro = outs[k];
  float samp = qnan(), depth = qnan();
  unsigned char mask = 2;
  if (ro.st.status == 0) {
    const float* F = g.flow + (size_t)frame_of(g, fa, k) * g.flow_frame_stride;
    float f[2] = {0.f, 0.f};
    upsample_at<2>(g, F, X, Y, mg.crop_x, mg.crop_y, [&f](int ch, float v) { f[ch] = v; });
    const float fX = (float)X, fY = (float)Y, xs = fX + f[0], ys = fY + f[1];
    bool known = fabsf(f[0]) <= 1e9f && fabsf(f[1]) <= 1e9f && in_frame_f(xs, ys, w, h);
    if (FB && known) {
      const float* Bf = g.flow + (size_t)frame_of(g, fb, k) * g.flow_frame_stride;
      consistency_at<2>(g, Bf, f, X, Y, w, h, mg.crop_x, mg.crop_y, mg.alpha, mg.beta,
                        [&known](unsigned char cm, float) { known = cm == 0; });
    }
    if (known) {
      const float4 c = make_float4(fX, fY, xs, ys);
      float e, den;
      mask = sampson_terms(ro.g, c, mg.t, e, den) ? 0 : 1;
      samp = sqrtf((e * e) / den);
      samp = isnan(samp) ? qnan() : samp;
      float R[9], t[3], x, y, xp, yp;
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) R[3 * i + j] = (float)ro.pose[4 * i + j];
        t[i] = (float)ro.pose[4 * i + 3];
      }
      rp_norm(rg, c, x, y, xp, yp);
      float q[3], c1[3], c2[3];
      for (int i = 0; i < 3; ++i) q[i] = (R[3 * i] * x + R[3 * i + 1] * y) + R[3 * i + 2];
      c1[0] = yp * q[2] - q[1], c1[1] = q[0] - xp * q[2], c1[2] = xp * q[1] - yp * q[0];
      c2[0] = yp * t[2] - t[1], c2[1] = t[0] - xp * t[2], c2[2] = xp * t[1] - yp * t[0];
      const float lam = -((c1[0] * c2[0] + c1[1] * c2[1]) + c1[2] * c2[2]) / ((c1[0] * c1[0] + c1[1] * c1[1]) + c1[2] * c1[2]);
      if (lam > 0.f && lam * q[2] + t[2] > 0.f) depth = lam;
    }
  }
  if (o.mask) o.mask[px] = mask;
  if (o.sampson) o.sampson[px] = samp;
  if (o.depth) o.depth[px] = depth;
}

}  // namespace

int launch_relpose(const LevelGeom& g, int fa, int fb, int n, const RelposeGeom& rg, const MotionWork& ws,
                   RelposeOut* out, const RelposeOutputs& o, cudaStream_t st) {
  const MotionGeom& mg = rg.mg;
  if (g.nop != 2 || launch_motion_corr(g, fa, fb, n, mg, ws, st) < 0) return -1;
  relpose_hyp_kernel<<<dim3((mg.nh + kHypThreads - 1) / kHypThreads, n), kHypThreads, 0, st>>>(rg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  if (launch_motion_score<SampsonTest>(mg, ws, n, st) < 0) return -1;
  relpose_refit_kernel<<<n, kRefitThreads, 0, st>>>(rg, ws, out);
  if (cudaGetLastError() != cudaSuccess) return -1;
  if (!o.mask && !o.sampson && !o.depth) return 5;
  const dim3 block(32, 8), grid((mg.w + 31) / 32, (mg.h + 7) / 8, n);
  if (mg.fb_check) relpose_apply_kernel<true><<<grid, block, 0, st>>>(g, fa, fb, rg, out, o);
  else relpose_apply_kernel<false><<<grid, block, 0, st>>>(g, fa, fb, rg, out, o);
  return cudaGetLastError() == cudaSuccess ? 6 : -1;
}

}  // namespace ofdis

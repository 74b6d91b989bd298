// Camera tracking against the TSDF volume (ofdis_fuse_track; the header states the contract, preprocess.fuse_track
// restates it bit for bit).  One kernel per (frame, round), whatever the data:
//   fuse_track_kernel  one warp per chunk of 32 cells: each lane gathers its cell's residual and gradient, the warp's 28
//                      terms per cell go through shared memory and lanes 0..27 sum one term each over the 32 cells in
//                      cell order; the chunk sums go to the workspace.  The last CTA to arrive (an arrival counter,
//                      reset for the next launch) runs the pairwise tree over the chunk sums, the solve, the Cayley
//                      update and the stop and guard rules, and writes the pose the next launch reads.  The sums'
//                      order is fixed by the cells, so the arrival order cannot change a bit.  A launch for a frame
//                      that has stopped returns at once.
// The push of an integrating call is the existing fuse_integrate_kernel with n = 1 (weighted for a weighted call),
// reading its float32 world-to-camera pose from FuseTrack::g.  float32 and float64 without contraction, IEEE division and square root.
#include <cfloat>

#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr int FT_WARPS = 4, FT_THREADS = 32 * FT_WARPS;
constexpr int FT_PAD = 33;  // a term's 32 cells plus one: the column sums read across banks

// step 1 of the header: T(k-1) inv(M_k), or T(k-1) without motions
__device__ __forceinline__ void ft_predict(const FuseTrack& t, int k, double (&M)[12]) {
  const double* P = t.state->prev;
  if (!t.has_motion) {
#pragma unroll
    for (int i = 0; i < 12; ++i) M[i] = P[i];
    return;
  }
  const double* m = t.motion + 12 * k;
  double Ri[3][3], ti[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) Ri[r][c] = m[4 * c + r];
    ti[r] = -(((m[r] * m[3]) + (m[4 + r] * m[7])) + (m[8 + r] * m[11]));
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) M[4 * r + c] = ((P[4 * r] * Ri[0][c]) + (P[4 * r + 1] * Ri[1][c])) + (P[4 * r + 2] * Ri[2][c]);
    M[4 * r + 3] = (((P[4 * r] * ti[0]) + (P[4 * r + 1] * ti[1])) + (P[4 * r + 2] * ti[2])) + P[4 * r + 3];
  }
}

// step 2 at cell c: false when the cell is not valid, else its residual r, gradient G and the world point Pw
__device__ __forceinline__ bool ft_cell(const FuseGeom& g, const FuseVolume& v, const FuseTrack& t, const float* D,
                                        const float* gp, int c, float& res, float (&G)[3], float (&Pw)[3]) {
  const DispCamera& cam = t.cam;
  const int px = min((c % t.ncx) * t.s + t.s / 2, t.w - 1), py = min((c / t.ncx) * t.s + t.s / 2, t.h - 1);
  const float d = __ldg(D + (size_t)py * t.w + px);
  const float sd = d + cam.doffs;
  if (!known_d(d) || !(sd > 0.0f)) return false;
  const float Z = cam.fb / sd;
  if (!(Z <= t.max_depth)) return false;
  const float X = (((float)px - cam.cx) * Z) / cam.fx, Y = (((float)py - cam.cy) * Z) / cam.fy;
  const float o[3] = {g.ox, g.oy, g.oz};
  const int n[3] = {g.nx, g.ny, g.nz};
  int i0[3];
  float fr[3];
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    Pw[e] = ((gp[4 * e] * X + gp[4 * e + 1] * Y) + gp[4 * e + 2] * Z) + gp[4 * e + 3];
    const float q = (Pw[e] - o[e]) / g.voxel;
    const float fl = floorf(q);
    if (!(fl >= 0.0f && fl <= (float)(n[e] - 2))) return false;
    i0[e] = (int)fl;
    fr[e] = q - fl;
  }
  const long long sy = g.nx, sz = (long long)g.nx * g.ny;
  const long long base = ((long long)i0[2] * g.ny + i0[1]) * g.nx + i0[0];
  const long long off[8] = {0, 1, sy, sy + 1, sz, sz + 1, sz + sy, sz + sy + 1};
  float cc[8];
#pragma unroll
  for (int q8 = 0; q8 < 8; ++q8) {
    const float W = __ldg(v.W + base + off[q8]), T = __ldg(v.T + base + off[q8]);
    if (!(W >= t.min_weight && fabsf(T) < 1.0f)) return false;
    cc[q8] = T;
  }
  const float gx = 1.0f - fr[0], gy = 1.0f - fr[1], gz = 1.0f - fr[2];
  const float x00 = cc[0] * gx + cc[1] * fr[0], x10 = cc[2] * gx + cc[3] * fr[0];
  const float x01 = cc[4] * gx + cc[5] * fr[0], x11 = cc[6] * gx + cc[7] * fr[0];
  const float y0 = x00 * gy + x10 * fr[1], y1 = x01 * gy + x11 * fr[1];
  res = y0 * gz + y1 * fr[2];
  G[0] = (((cc[1] - cc[0]) * gy + (cc[3] - cc[2]) * fr[1]) * gz + ((cc[5] - cc[4]) * gy + (cc[7] - cc[6]) * fr[1]) * fr[2]) /
         g.voxel;
  G[1] = ((x10 - x00) * gz + (x11 - x01) * fr[2]) / g.voxel;
  G[2] = (y1 - y0) / g.voxel;
  return true;
}

// steps 3 and 4 after the evaluation of M at round r (the last CTA's thread 0): s the 28 sums, cnt the valid cells
__device__ void ft_finish(const FuseTrack& t, int k, int r, const double (&M)[12], const double* s, int cnt) {
  FuseTrackState* S = t.state;
  if (r == 0) {
    for (int i = 0; i < 12; ++i) S->pred[i] = M[i];
    S->cost0 = s[27];
    S->rounds = 0;
  }
  int status = cnt < t.min_corr && r == 0 ? 1 : 0;
  bool stop = cnt < t.min_corr || r == t.rounds;
  if (!stop) {
    double A[6][6], b[6], x[6];
    int e = 0;
    for (int a = 0; a < 6; ++a)
      for (int bb = a; bb < 6; ++bb) A[a][bb] = A[bb][a] = s[e++];
    for (int a = 0; a < 6; ++a) b[a] = s[e++];
    for (int a = 0; a < 6; ++a) A[a][a] = A[a][a] + t.damping;
    if (!motion_solve<6>(A, b, x)) {
      stop = true;
    } else {
      double mx = 0.0;
      for (int i = 0; i < 6; ++i) mx = fmax(mx, fabs(x[i]));
      if (mx <= t.eps) {
        stop = true;
      } else {
        // the Cayley rotation of ofdis_egomotion_fullres's refits: R <- C R, t <- C t + tau
        const double q = (x[0] * x[0] + x[1] * x[1]) + x[2] * x[2], dg = 1.0 - q, dn = 1.0 + q;
        const double K[3][3] = {{0.0, -x[2], x[1]}, {x[2], 0.0, -x[0]}, {-x[1], x[0], 0.0}};
        double C[3][3];
        for (int i = 0; i < 3; ++i)
          for (int j = 0; j < 3; ++j) C[i][j] = (((i == j ? dg : 0.0) + (2.0 * (x[i] * x[j]))) + (2.0 * K[i][j])) / dn;
        for (int i = 0; i < 3; ++i) {
          for (int j = 0; j < 4; ++j) S->cur[4 * i + j] = ((C[i][0] * M[j]) + (C[i][1] * M[4 + j])) + (C[i][2] * M[8 + j]);
          S->cur[4 * i + 3] = S->cur[4 * i + 3] + x[3 + i];
        }
        S->rounds = r + 1;
      }
    }
  }
  S->done = stop ? 1 : 0;
  if (!stop) return;
  const double* Pp = S->pred;
  if (!status) {
    const double dt[3] = {M[3] - Pp[3], M[7] - Pp[7], M[11] - Pp[11]};
    const double shift = sqrt((dt[0] * dt[0] + dt[1] * dt[1]) + dt[2] * dt[2]);
    double si[3];
    for (int i = 0; i < 3; ++i)
      si[i] = ((M[4 * i] * Pp[4 * i]) + (M[4 * i + 1] * Pp[4 * i + 1])) + (M[4 * i + 2] * Pp[4 * i + 2]);
    const double cosv = (((si[0] + si[1]) + si[2]) - 1.0) / 2.0;
    status = shift <= t.max_shift && cosv >= t.min_cos ? 0 : 2;
  }
  double F[12];
  for (int i = 0; i < 12; ++i) F[i] = status ? Pp[i] : M[i];
  for (int i = 0; i < 12; ++i) {
    t.pose[12 * k + i] = F[i];
    S->prev[i] = F[i];
  }
  t.stats[k] = ofdis_fuse_track_stats{status, cnt, S->rounds, S->cost0, s[27]};
  // ofdis_fuse_push's world-to-camera pose of F, formed in float64 and rounded once
  for (int rr = 0; rr < 3; ++rr) {
    for (int c = 0; c < 3; ++c) t.g[4 * rr + c] = (float)F[4 * c + rr];
    t.g[4 * rr + 3] = (float)(-(((F[rr] * F[3]) + (F[4 + rr] * F[7])) + (F[8 + rr] * F[11])));
  }
}

// WEIGHTED: ofdis_fuse_track_weighted -- a cell is valid only where its weight c = wk[py * w + px] is finite and > 0,
// and its Huber
// weight becomes wt * c.  The false instance is ofdis_fuse_track (wk unused, after the parameters it reads).
template <bool WEIGHTED>
__global__ void __launch_bounds__(FT_THREADS) fuse_track_kernel(FuseGeom g, FuseVolume v, FuseTrack t, int k, int r,
                                                                 const float* wk) {
  __shared__ double terms[FT_WARPS][FTRACK_NE][FT_PAD];
  __shared__ double Ms[12];
  __shared__ float gs[12];
  __shared__ int last;
  FuseTrackState* S = t.state;
  if (r > 0 && S->done) return;  // uniform: written by an earlier launch
  if (threadIdx.x == 0) {
    double M[12];
    if (r == 0) ft_predict(t, k, M);
    else
      for (int i = 0; i < 12; ++i) M[i] = S->cur[i];
    for (int i = 0; i < 12; ++i) Ms[i] = M[i], gs[i] = (float)M[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int chunk = blockIdx.x * FT_WARPS + warp, c = chunk * 32 + lane;
  double (*tw)[FT_PAD] = terms[warp];
  float res = 0.0f, G[3], Pw[3];
  bool valid = c < t.cells && ft_cell(g, v, t, t.disp + (size_t)k * t.disp_stride, gs, c, res, G, Pw);
  float cw = 1.0f;
  if constexpr (WEIGHTED) {
    if (valid) {
      const int px = min((c % t.ncx) * t.s + t.s / 2, t.w - 1), py = min((c / t.ncx) * t.s + t.s / 2, t.h - 1);
      cw = __ldg(wk + (size_t)py * t.w + px);
      valid = cw > 0.0f && cw <= FLT_MAX;
    }
  }
  if (valid) {
    const double a[3] = {(double)G[0], (double)G[1], (double)G[2]};
    const double w0 = 2.0 * (double)Pw[0], w1 = 2.0 * (double)Pw[1], w2 = 2.0 * (double)Pw[2];
    const double J[6] = {(a[1] * -w2) + (a[2] * w1), (a[0] * w2) + (a[2] * -w0), (a[0] * -w1) + (a[1] * w0),
                         a[0], a[1], a[2]};
    const float ar = fabsf(res);
    const float wf = ar <= t.huber ? 1.0f : t.huber / ar;
    const double wt = (double)(WEIGHTED ? wf * cw : wf), rd = (double)res;
    int e = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      const double vi = wt * J[i];
#pragma unroll
      for (int j = i; j < 6; ++j) tw[e++][lane] = vi * J[j];
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) tw[21 + i][lane] = -((wt * J[i]) * rd);
    tw[27][lane] = (wt * rd) * rd;
  } else {
#pragma unroll
    for (int e = 0; e < FTRACK_NE; ++e) tw[e][lane] = 0.0;
  }
  const unsigned nv = __popc(__ballot_sync(0xffffffffu, valid));
  if (lane == 0 && nv) atomicAdd(&S->count, nv);
  __syncwarp();
  if (lane < FTRACK_NE && chunk < t.nchunks) {
    double sum = 0.0;
#pragma unroll 8
    for (int i = 0; i < 32; ++i) sum = sum + tw[lane][i];
    t.chunk[(size_t)chunk * FTRACK_NE + lane] = sum;
  }
  __threadfence();  // the chunk sums and the count reach L2 before this CTA arrives
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&S->arrived, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  // the pairwise tree over the chunk sums, padded with +0.0 to P leaves, in place: v_j += v_(j + stride)
  const int nc = t.nchunks;
  int P = 1;
  while (P < nc) P <<= 1;
  for (int stride = 1; stride < P; stride <<= 1) {
    const int pairs = (nc + 2 * stride - 1) / (2 * stride);
    for (int q = threadIdx.x; q < pairs * FTRACK_NE; q += FT_THREADS) {
      const int j = (q / FTRACK_NE) * 2 * stride, e = q % FTRACK_NE, o = j + stride;
      double* dst = t.chunk + (size_t)j * FTRACK_NE + e;
      *dst = __ldcg(dst) + (o < nc ? __ldcg(t.chunk + (size_t)o * FTRACK_NE + e) : 0.0);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double s[FTRACK_NE], M[12];
    for (int e = 0; e < FTRACK_NE; ++e) s[e] = __ldcg(t.chunk + e);
    for (int i = 0; i < 12; ++i) M[i] = Ms[i];
    const int cnt = (int)atomicExch(&S->count, 0u);
    ft_finish(t, k, r, M, s, cnt);
    S->arrived = 0;
  }
}

}  // namespace

int launch_fuse_track_eval(const FuseGeom& g, const FuseVolume& v, const FuseTrack& t, int k, int r, cudaStream_t st,
                           const float* wk) {
  const int blocks = (t.nchunks + FT_WARPS - 1) / FT_WARPS;
  if (wk) fuse_track_kernel<true><<<blocks, FT_THREADS, 0, st>>>(g, v, t, k, r, wk);
  else fuse_track_kernel<false><<<blocks, FT_THREADS, 0, st>>>(g, v, t, k, r, wk);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ofdis

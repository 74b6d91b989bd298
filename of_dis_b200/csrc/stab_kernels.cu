// Video stabilisation (ofdis_stab_push / ofdis_stab_finish; the header states the contract, preprocess.stabilize
// restates it bit for bit).  Two launches per call, whatever the number of frames it emits:
//   stab_path_kernel  one thread per emitted frame: the float64 path over its window of the model ring, the limit's
//                     bisection with the float32 corner test, a0..a8 and the frame's record;
//   stab_warp_kernel  the hot path: one thread per 4 horizontally adjacent output pixels of a frame, the frame ring
//                     read through L1/L2 by bil_u8, the 4 pixels stored as 32-bit words.
// float64 and float32 without contraction (-fmad=false), IEEE division: the path is computed here rather than on the
// host so that its bits do not depend on the host compiler's contraction.
#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr int kPathThreads = 64;
constexpr int kWarpPx = 4;  // output pixels per thread of stab_warp_kernel

__device__ __forceinline__ void mat_eye(double* A) {
  for (int i = 0; i < 9; ++i) A[i] = (i % 4 == 0) ? 1.0 : 0.0;
}

// C = A * B, (A*B)_ij = (A_i0*B_0j + A_i1*B_1j) + A_i2*B_2j
__device__ __forceinline__ void mat_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = (A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j]) + A[3 * i + 2] * B[6 + j];
}

// norm(A) in place; false where the divisor is zero or not finite or an entry is not finite
__device__ __forceinline__ bool mat_norm(double* A) {
  const double d = A[8];
  if (!(isfinite(d) && d != 0.0)) return false;
  bool ok = true;
  for (int i = 0; i < 9; ++i) {
    A[i] = A[i] / d;
    ok = ok && isfinite(A[i]);
  }
  return ok;
}

// C = inv(A): the adjugate in the header's order, then norm
__device__ __forceinline__ bool mat_inv(const double* a, double* C) {
  C[0] = a[4] * a[8] - a[5] * a[7];
  C[1] = a[2] * a[7] - a[1] * a[8];
  C[2] = a[1] * a[5] - a[2] * a[4];
  C[3] = a[5] * a[6] - a[3] * a[8];
  C[4] = a[0] * a[8] - a[2] * a[6];
  C[5] = a[2] * a[3] - a[0] * a[5];
  C[6] = a[3] * a[7] - a[4] * a[6];
  C[7] = a[1] * a[6] - a[0] * a[7];
  C[8] = a[0] * a[4] - a[1] * a[3];
  return mat_norm(C);
}

// model k as received: divided by its m22, or the identity
__device__ __forceinline__ void stab_model(const StabGeom& sg, const double* ring, long long k, double* M) {
  const double* m = ring + (size_t)(k % sg.mring) * 9;
  const double d = m[8];
  bool ok = isfinite(d) && d != 0.0;
  for (int i = 0; i < 9; ++i) {
    M[i] = m[i] / d;
    ok = ok && isfinite(M[i]);
  }
  if (ok) {
    const double a = M[0] * M[4] - M[1] * M[3];
    ok = isfinite(a) && a != 0.0;
  }
  if (!ok) mat_eye(M);
}

// S of frame t; false where the path is undefined
__device__ bool stab_path(const StabGeom& sg, const double* ring, long long t, double* S) {
  const long long a = t - sg.radius > 0 ? t - sg.radius : 0;
  const long long b = sg.cut && sg.last < t + sg.radius ? sg.last : t + sg.radius;
  double acc[9], P[9], M[9], Q[9];
  const double w0 = sg.wt[0];
  for (int i = 0; i < 9; ++i) acc[i] = (i % 4 == 0) ? w0 : 0.0;
  double wsum = w0;
  mat_eye(P);
  for (int d = 1; d <= (int)(b - t); ++d) {
    stab_model(sg, ring, t + d - 1, M);
    mat_mul(M, P, Q);
    if (!mat_norm(Q)) return false;
    for (int i = 0; i < 9; ++i) {
      P[i] = Q[i];
      acc[i] = acc[i] + sg.wt[d] * P[i];
    }
    wsum = wsum + sg.wt[d];
  }
  mat_eye(P);
  for (int d = 1; d <= (int)(t - a); ++d) {
    stab_model(sg, ring, t - d, M);
    if (!mat_inv(M, Q)) return false;
    mat_mul(Q, P, M);
    if (!mat_norm(M)) return false;
    for (int i = 0; i < 9; ++i) {
      P[i] = M[i];
      acc[i] = acc[i] + sg.wt[d] * P[i];
    }
    wsum = wsum + sg.wt[d];
  }
  bool ok = true;
  for (int i = 0; i < 9; ++i) {
    S[i] = acc[i] / wsum;
    ok = ok && isfinite(S[i]);
  }
  return ok;
}

// S(l) into SL and A(l) rounded to float32 into a; false where A(l) is undefined
__device__ bool stab_warp_map(const StabGeom& sg, const double* S, double l, double* SL, float* a) {
  for (int i = 0; i < 9; ++i) SL[i] = (i % 4 == 0) ? (1.0 - l) + l * S[i] : l * S[i];
  const double s = 1.0 - 2.0 * (double)sg.crop, cx = 0.5 * (double)(sg.w - 1), cy = 0.5 * (double)(sg.h - 1);
  const double Z[9] = {s, 0.0, cx * (1.0 - s), 0.0, s, cy * (1.0 - s), 0.0, 0.0, 1.0};
  double Si[9], A[9];
  if (!mat_inv(SL, Si)) return false;
  mat_mul(Si, Z, A);
  if (!mat_norm(A)) return false;
  for (int i = 0; i < 9; ++i) a[i] = (float)A[i];
  return true;
}

// output pixel (X, Y) -> (xw, yw) and wq of the per-pixel rule; true where the frame is sampled there
__device__ __forceinline__ bool stab_source(const float* a, float X, float Y, int w, int h, float& xw, float& yw) {
  const float mx = (a[0] * X + a[1] * Y) + a[2], my = (a[3] * X + a[4] * Y) + a[5];
  const float wq = (a[6] * X + a[7] * Y) + a[8];
  xw = mx / wq;
  yw = my / wq;
  return wq > 0.f && in_frame_f(xw, yw, w, h);
}

__device__ bool stab_passes(const StabGeom& sg, const double* S, double l, double* SL, float* a) {
  if (!stab_warp_map(sg, S, l, SL, a)) return false;
  const float X1 = (float)(sg.w - 1), Y1 = (float)(sg.h - 1);
  float xw, yw;
  return stab_source(a, 0.f, 0.f, sg.w, sg.h, xw, yw) && stab_source(a, X1, 0.f, sg.w, sg.h, xw, yw) &&
         stab_source(a, 0.f, Y1, sg.w, sg.h, xw, yw) && stab_source(a, X1, Y1, sg.w, sg.h, xw, yw);
}

__global__ void __launch_bounds__(kPathThreads) stab_path_kernel(StabGeom sg, StabWork ws) {
  const int i = blockIdx.x * kPathThreads + threadIdx.x;
  if (i >= sg.count) return;
  const long long t = sg.next + i;
  double S[9], SL[9];
  float a[9];
  double l = 1.0;
  bool ok = stab_path(sg, ws.models, t, S);
  if (ok && !sg.limit) {
    ok = stab_warp_map(sg, S, 1.0, SL, a);
  } else if (ok && !stab_passes(sg, S, 1.0, SL, a)) {
    double lo = 0.0, hi = 1.0;
    for (int k = 0; k < 20; ++k) {
      const double mid = 0.5 * (lo + hi);
      if (stab_passes(sg, S, mid, SL, a)) lo = mid;
      else hi = mid;
    }
    l = lo;
    stab_warp_map(sg, S, l, SL, a);
  }
  if (!ok) {
    mat_eye(S);
    l = 0.0;
    stab_warp_map(sg, S, l, SL, a);
  }
  StabRec& r = ws.rec[i];
  for (int k = 0; k < 9; ++k) r.a[k] = a[k];
  r.info.frame = t;
  r.info.status = ok ? 0 : 1;
  r.info.lambda = l;
  for (int k = 0; k < 9; ++k) r.info.correction[k] = SL[k];
}

template <int NOC>
__global__ void __launch_bounds__(256) stab_warp_kernel(StabGeom sg, StabWork ws, unsigned char* out) {
  const int w = sg.w, h = sg.h, k = blockIdx.z;
  const int X0 = (blockIdx.x * blockDim.x + threadIdx.x) * kWarpPx, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X0 >= w || Y >= h) return;
  float a[9];
  for (int i = 0; i < 9; ++i) a[i] = ws.rec[k].a[i];
  const size_t hwc = (size_t)w * h * NOC;
  const int slot = (sg.slot0 + k) % sg.ring;
  const unsigned char* I = ws.frames + (size_t)slot * hwc;
  unsigned char v[kWarpPx * NOC];
  const float fY = (float)Y;
#pragma unroll
  for (int j = 0; j < kWarpPx; ++j) {
    float xw, yw, s[NOC];
    const bool in = X0 + j < w && stab_source(a, (float)(X0 + j), fY, w, h, xw, yw);
    if (in) bil_u8<NOC>(I, w, h, xw, yw, s);
#pragma unroll
    for (int c = 0; c < NOC; ++c) v[j * NOC + c] = in ? round_u8(s[c]) : (unsigned char)0;
  }
  unsigned char* q = out + (size_t)k * hwc + ((size_t)Y * w + X0) * NOC;
  if (sg.vec) {  // X0 + 4 <= w and q 4-byte aligned
    unsigned int* q4 = reinterpret_cast<unsigned int*>(q);
#pragma unroll
    for (int i = 0; i < NOC; ++i)
      q4[i] = (unsigned int)v[4 * i] | ((unsigned int)v[4 * i + 1] << 8) | ((unsigned int)v[4 * i + 2] << 16) |
              ((unsigned int)v[4 * i + 3] << 24);
  } else {
    for (int j = 0; j < kWarpPx && X0 + j < w; ++j)
#pragma unroll
      for (int c = 0; c < NOC; ++c) q[j * NOC + c] = v[j * NOC + c];
  }
}

}  // namespace

int launch_stab(const StabGeom& sg, const StabWork& ws, unsigned char* out, cudaStream_t st) {
  if ((sg.noc != 1 && sg.noc != 3) || sg.count < 1) return -1;
  stab_path_kernel<<<(sg.count + kPathThreads - 1) / kPathThreads, kPathThreads, 0, st>>>(sg, ws);
  if (cudaGetLastError() != cudaSuccess) return -1;
  const dim3 block(32, 8), grid((sg.w + 32 * kWarpPx - 1) / (32 * kWarpPx), (sg.h + 7) / 8, sg.count);
  if (sg.noc == 3) stab_warp_kernel<3><<<grid, block, 0, st>>>(sg, ws, out);
  else stab_warp_kernel<1><<<grid, block, 0, st>>>(sg, ws, out);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

}  // namespace ofdis

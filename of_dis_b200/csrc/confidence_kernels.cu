// Per-pixel confidence of the last run's flows and disparities (ofdis_confidence_fullres; the header states the
// contract, preprocess.confidence restates it bit for bit).  One launch for all pairs (blockIdx.z is the pair):
//   confidence_kernel  a CTA owns a CF_TX x CF_TY tile of one pair.  It first stages, for every position of the tile
//                      and its r-pixel halo (clamped to the frame), I0's brightness, its two central differences and
//                      the brightness of I1 warped by that position's own flow (NaN where the target leaves the frame)
//                      in shared memory; every window sum of the tile's pixels then reads shared memory only.
// F is read through upsample_at and the forward-backward term through consistency_at; no full-resolution copy of a
// flow is stored.  Float32 without contraction, IEEE division and square root.
#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr int CF_TX = 32, CF_TY = 8, CF_THREADS = CF_TX * CF_TY;
constexpr int CF_SW = CF_TX + 2 * OFDIS_CONF_MAX_RADIUS, CF_SH = CF_TY + 2 * OFDIS_CONF_MAX_RADIUS;

// the brightness of I1 at an in-frame position: bil_u8's rule on the brightness of the four corners
template <int NOC>
__device__ __forceinline__ float gray_bil(const unsigned char* I, int w, int h, float xs, float ys) {
  const int x0 = (int)floorf(xs), y0 = (int)floorf(ys);
  const int x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);
  const float fx = xs - (float)x0, fy = ys - (float)y0, gx = 1.0f - fx, gy = 1.0f - fy;
  const float r0 = gray_at<NOC>(I, w, x0, y0) * gx + gray_at<NOC>(I, w, x1, y0) * fx;
  const float r1 = gray_at<NOC>(I, w, x0, y1) * gx + gray_at<NOC>(I, w, x1, y1) * fx;
  return r0 * gy + r1 * fy;
}

template <int NOP, int NOC>
__global__ void __launch_bounds__(CF_THREADS) confidence_kernel(LevelGeom g, int fa, int fb, ConfArgs a) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  __shared__ float s_g0[CF_SH * CF_SW], s_iw[CF_SH * CF_SW], s_ix[CF_SH * CF_SW], s_iy[CF_SH * CF_SW];
  const int w = a.w, h = a.h, r = a.r, pair = blockIdx.z;
  const int x0 = blockIdx.x * CF_TX - r, y0 = blockIdx.y * CF_TY - r;
  const int sw = CF_TX + 2 * r, sh = CF_TY + 2 * r;
  const unsigned char* I0 = a.i0 + (size_t)pair * a.stride;
  const unsigned char* I1 = a.i1 + (size_t)pair * a.stride;
  const float* F = g.flow + (size_t)frame_of(g, fa, pair) * g.flow_frame_stride;
  const float qnan = __int_as_float(0x7fc00000);
  for (int q = threadIdx.x; q < sw * sh; q += CF_THREADS) {
    const int ly = q / sw, lx = q - ly * sw;
    const int xc = clampi(x0 + lx, w), yc = clampi(y0 + ly, h);
    float f[2] = {0.f, 0.f};
    upsample_at<NOP>(g, F, xc, yc, a.crop_x, a.crop_y, [&f](int c, float v) { f[c] = v; });
    const float xs = (float)xc + f[0], ys = (float)yc + (NOP == 2 ? f[1] : 0.f);
    const int s = ly * CF_SW + lx;
    s_g0[s] = gray_at<NOC>(I0, w, xc, yc);
    s_ix[s] = (gray_at<NOC>(I0, w, min(xc + 1, w - 1), yc) - gray_at<NOC>(I0, w, max(xc - 1, 0), yc)) * 0.5f;
    s_iy[s] = (gray_at<NOC>(I0, w, xc, min(yc + 1, h - 1)) - gray_at<NOC>(I0, w, xc, max(yc - 1, 0))) * 0.5f;
    s_iw[s] = in_frame_f(xs, ys, w, h) ? gray_bil<NOC>(I1, w, h, xs, ys) : qnan;
  }
  __syncthreads();
  const int tx = threadIdx.x % CF_TX, ty = threadIdx.x / CF_TX;
  const int X = blockIdx.x * CF_TX + tx, Y = blockIdx.y * CF_TY + ty;
  if (X >= w || Y >= h) return;
  // pass 1: the in-frame samples, their sums, and the structure tensor over the whole window
  int n = 0;
  float s0 = 0.0f, s1 = 0.0f, ta = 0.0f, tb = 0.0f, td = 0.0f;
  for (int dy = -r; dy <= r; ++dy) {
    const int row = (ty + r + dy) * CF_SW + tx + r;
    for (int dx = -r; dx <= r; ++dx) {
      const float ix = s_ix[row + dx], iy = s_iy[row + dx], b = s_iw[row + dx];
      ta = ta + ix * ix;
      tb = tb + ix * iy;
      td = td + iy * iy;
      if (b == b) {
        ++n;
        s0 = s0 + s_g0[row + dx];
        s1 = s1 + b;
      }
    }
  }
  const float dd = ta - td;
  const float lam = (ta + td) * 0.5f - sqrtf(dd * dd * 0.25f + tb * tb);
  float z = qnan;
  if (n >= a.min_count) {
    // pass 2: centred second moments of the in-frame samples
    const float m0 = s0 / (float)n, m1 = s1 / (float)n;
    float c00 = 0.0f, c11 = 0.0f, c01 = 0.0f;
    for (int dy = -r; dy <= r; ++dy) {
      const int row = (ty + r + dy) * CF_SW + tx + r;
      for (int dx = -r; dx <= r; ++dx) {
        const float b = s_iw[row + dx];
        if (b == b) {
          const float p = s_g0[row + dx] - m0, qv = b - m1;
          c00 = c00 + p * p;
          c11 = c11 + qv * qv;
          c01 = c01 + p * qv;
        }
      }
    }
    const float den = c00 * c11;
    if (den > 0.0f) z = c01 / sqrtf(den);
  }
  float e = qnan, ce = 1.0f;
  if (fb >= 0) {
    const float* B = g.flow + (size_t)frame_of(g, fb, pair) * g.flow_frame_stride;
    float f[2] = {0.f, 0.f};
    upsample_at<NOP>(g, F, X, Y, a.crop_x, a.crop_y, [&f](int c, float v) { f[c] = v; });
    consistency_at<NOP>(g, B, f, X, Y, w, h, a.crop_x, a.crop_y, 0.0f, 0.0f, [&e](unsigned char, float ev) { e = ev; });
    ce = e >= 0.0f ? a.s_fb / (a.s_fb + e) : 0.0f;
  }
  const float cz = z > 0.0f ? z : 0.0f;
  const float cl = lam > 0.0f ? lam / (lam + a.s_tex) : 0.0f;
  const size_t o = ((size_t)pair * h + Y) * w + X;
  if (a.conf) a.conf[o] = (cz * ce) * cl;
  if (a.terms) {
    a.terms[3 * o] = z;
    a.terms[3 * o + 1] = e;
    a.terms[3 * o + 2] = lam;
  }
}

template <int NOP>
int launch_nop(const LevelGeom& g, int fa, int fb, int n, int noc, const ConfArgs& a, cudaStream_t st) {
  const dim3 grid((a.w + CF_TX - 1) / CF_TX, (a.h + CF_TY - 1) / CF_TY, n);
  if (noc == 3) confidence_kernel<NOP, 3><<<grid, CF_THREADS, 0, st>>>(g, fa, fb, a);
  else confidence_kernel<NOP, 1><<<grid, CF_THREADS, 0, st>>>(g, fa, fb, a);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace

int launch_confidence(const LevelGeom& g, int fa, int fb, int n, int noc, const ConfArgs& a, cudaStream_t st) {
  if (noc != 1 && noc != 3) return -1;
  return g.nop == 2 ? launch_nop<2>(g, fa, fb, n, noc, a, st) : launch_nop<1>(g, fa, fb, n, noc, a, st);
}

}  // namespace ofdis

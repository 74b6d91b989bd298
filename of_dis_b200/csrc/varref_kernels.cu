// Variational refinement of the DIS hot path on sm_90a (K5..K12 of SURVEY.md):
// VarRefClass (refine_variational.cpp:25-336) and the FDF1.0.1 routines it calls
// (opticalflow_aux.c:17-548, image.c:376-502, solver.c:77-466).
//
//   varref_setup_kernel  image_warp + copyimage + get_derivatives (5-tap, horizontal replicate / vertical
//                        folded coeffs) through shared-memory stages, and the first inner iteration's records
//   assemble_kernel  compute_smoothness + compute_data[_DE] + sub_laplacian (x2) + the 2x2 block
//                    inversion of sor_coupled's first sweep, fused; smoothness staged through
//                    shared-memory tiles; writes one 32-byte SOR record per pixel (inner iterations 2..n)
//   sor_wave_kernel  all sweeps of the lexicographic SOR as a systolic wavefront, one CTA or one
//                    thread-block cluster per frame (sor_wave_kernel.cuh)
//
// Every expression keeps the reference's operand order; the TU is compiled with
// -fmad=false so nothing is contracted (bit-exactness, DESIGN.md section 4).
#include "ofdis_internal.cuh"

#include <map>
#include <mutex>
#include <type_traits>
#include <utility>

namespace ofdis {

namespace {

#define DATANORM (0.1f * 0.1f)       /* opticalflow_aux.c:10 */
#define EPS_COLOR (0.001f * 0.001f)  /* :11 */
#define EPS_GRAD (0.001f * 0.001f)   /* :12 */
#define EPS_SMOOTH (0.001f * 0.001f) /* :14 */

// convolve_extract_coeffs(even=0) of {0,-8/12,1/12} and {0,-0.5} (image.c:338-342,
// refine_variational.cpp:45-48)
struct Coef5 { float c0, c1, c2, c3, c4; };
__device__ __forceinline__ Coef5 coef5() {
  Coef5 c;
  c.c0 = 1.0f / 12.0f;
  c.c1 = -8.0f / 12.0f;
  c.c2 = -0.0f;
  c.c3 = -(-8.0f / 12.0f);
  c.c4 = -(1.0f / 12.0f);
  return c;
}

// convolve_vert_fast_5 (image.c:401-434): border rows fold the coefficients
__device__ __forceinline__ float conv_v5(const float* q, int pitch, int h, int j, const Coef5& c) {
  if (j == 0) return (c.c0 + c.c1 + c.c2) * q[0] + c.c3 * q[pitch] + c.c4 * q[2 * pitch];
  if (j == 1) return (c.c0 + c.c1) * q[-pitch] + c.c2 * q[0] + c.c3 * q[pitch] + c.c4 * q[2 * pitch];
  if (j == h - 2) return c.c0 * q[-2 * pitch] + c.c1 * q[-pitch] + c.c2 * q[0] + (c.c3 + c.c4) * q[pitch];
  if (j == h - 1) return c.c0 * q[-2 * pitch] + c.c1 * q[-pitch] + (c.c2 + c.c3 + c.c4) * q[0];
  return c.c0 * q[-2 * pitch] + c.c1 * q[-pitch] + c.c2 * q[0] + c.c3 * q[pitch] + c.c4 * q[2 * pitch];
}

// convolve_horiz_fast_5 (image.c:466-502): replicate borders, five products, on a staged row whose first entry is
// column `lo`
__device__ __forceinline__ float conv_h5s(const float* row, int lo, int w, int i, const Coef5& c) {
  return c.c0 * row[clampi(i - 2, w) - lo] + c.c1 * row[clampi(i - 1, w) - lo] + c.c2 * row[i - lo] +
         c.c3 * row[clampi(i + 1, w) - lo] + c.c4 * row[clampi(i + 2, w) - lo];
}

// ---------------------------------------------------------------------------
// One inner fixed-point iteration, everything except the solver:
// compute_smoothness (opticalflow_aux.c:123-165), compute_data / compute_data_DE
// (:309-548), sub_laplacian on b1 (and b2) (:172-199), and for flow the in-place
// 2x2 inversion of sor_coupled's first sweep (solver.c:115-120).
constexpr int TX = 32, TY = 8;

// smoothness weight s = quarter_alpha / sqrt(ux^2+uy^2+vx^2+vy^2+eps) on the tile + 1 halo, from uu, vv staged at
// the clamped positions of the tile + `o` halo (o >= 2)
template <int TH, int SW>
__device__ __forceinline__ void smoothness_tile(const float2 (*s_uv)[SW], float (*s_s)[TX + 2], int o, int x0, int y0,
                                                int w, int h, float quarter_alpha, int tid) {
  const float c0 = -0.5f, c1 = -0.0f, c2 = 0.5f;  // {0,-0.5} -> [-0.5,-0,0.5]
  for (int idx = tid; idx < (TH + 2) * (TX + 2); idx += TX * TY) {
    const int cy = idx / (TX + 2), cx = idx - cy * (TX + 2);
    const int gx = x0 - 1 + cx, gy = y0 - 1 + cy;
    if (gx < 0 || gx >= w || gy < 0 || gy >= h) continue;
    const int sx = cx + o - 1, sy = cy + o - 1;  // position in s_uv
    const float2 l = s_uv[sy][sx - 1], m = s_uv[sy][sx], r = s_uv[sy][sx + 1];
    const float2 t = s_uv[sy - 1][sx], b = s_uv[sy + 1][sx];
    const float ux = c0 * l.x + c1 * m.x + c2 * r.x;
    const float vx = c0 * l.y + c1 * m.y + c2 * r.y;
    float uy, vy;
    if (gy == 0) {  // convolve_vert_fast_3 (image.c:383-398)
      uy = (c0 + c1) * m.x + c2 * b.x;
      vy = (c0 + c1) * m.y + c2 * b.y;
    } else if (gy == h - 1) {
      uy = c0 * t.x + (c1 + c2) * m.x;
      vy = c0 * t.y + (c1 + c2) * m.y;
    } else {
      uy = c0 * t.x + c1 * m.x + c2 * b.x;
      vy = c0 * t.y + c1 * m.y + c2 * b.y;
    }
    s_s[cy][cx] = quarter_alpha / sqrtf(ux * ux + uy * uy + vx * vx + vy * vy + EPS_SMOOTH);
  }
}

// The SOR record of pixel (i, j) from its derivatives D(k, c) (k: Ix Iy Iz Ixx Ixy Iyy Ixz Iyz), (du, dv) = (u, v),
// mask m and the smoothness sums hh = sh(i,j), hl = sh(i-1,j), vv = sv(i,j), vt = sv(i,j-1); fc is the flow w at the
// pixel.  rec points at the pixel's first record field.
template <int C, int NOP, int MODE, class Deriv>
__device__ __forceinline__ void pixel_record(const Deriv& D, float u, float v, float m, float hh, float hl, float vv,
                                             float vt, const float* fc, int i, int j, int w, int h,
                                             const VarRefParams& vp, float* rec) {
  constexpr bool fast = (MODE == 1), lane = (MODE == 2);
  const int fs = fast ? 1 : 4;  // floats between consecutive record fields of a pixel
  const float hdo3 = vp.half_delta_over3, hgo3 = vp.half_gamma_over3;
  float A11 = 0.f, A12 = 0.f, A22 = 0.f, B1 = 0.f, B2 = 0.f;
  if (C == 1) {
    const float ix = D(0, 0), iy = D(1, 0), iz = D(2, 0), ixx = D(3, 0), ixy = D(4, 0), iyy = D(5, 0), ixz = D(6, 0),
                iyz = D(7, 0);
    float t, t2, nn, n2;
    if (hdo3 != 0.0f) {
      t = (NOP == 2) ? iz + ix * u + iy * v : iz + ix * u;
      nn = ix * ix + iy * iy + DATANORM;
      t = m * hdo3 / sqrtf(3 * t * t / nn + EPS_COLOR);
      t /= nn;
      A11 += t * ix * ix;
      B1 -= t * iz * ix;
      if (NOP == 2) {
        A12 += t * ix * iy;
        A22 += t * iy * iy;
        B2 -= t * iz * iy;
      }
    }
    nn = ixx * ixx + ixy * ixy + DATANORM;
    n2 = iyy * iyy + ixy * ixy + DATANORM;
    t = (NOP == 2) ? ixz + ixx * u + ixy * v : ixz + ixx * u;
    t2 = (NOP == 2) ? iyz + ixy * u + iyy * v : iyz + ixy * u;
    t = m * hgo3 / sqrtf(3 * t * t / nn + 3 * t2 * t2 / n2 + EPS_GRAD);
    t2 = t / n2;
    t /= nn;
    A11 += t * ixx * ixx + t2 * ixy * ixy;
    B1 -= t * ixx * ixz + t2 * ixy * iyz;
    if (NOP == 2) {
      A12 += t * ixx * ixy + t2 * ixy * iyy;
      A22 += t2 * iyy * iyy + t * ixy * ixy;
      B2 -= t2 * iyy * iyz + t * ixy * ixz;
    }
    A11 *= 3;
    B1 *= 3;
    if (NOP == 2) {
      A12 *= 3;
      A22 *= 3;
      B2 *= 3;
    }
  } else {
    float tc[3], nc[3], tg[6], ng[6], acc, t;
    if (hdo3 != 0.0f) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float ix = D(0, c), iy = D(1, c), iz = D(2, c);
        tc[c] = (NOP == 2) ? iz + ix * u + iy * v : iz + ix * u;
        nc[c] = ix * ix + iy * iy + DATANORM;
      }
      acc = tc[0] * tc[0] / nc[0] + tc[1] * tc[1] / nc[1] + tc[2] * tc[2] / nc[2] + EPS_COLOR;
      t = m * hdo3 / sqrtf(acc);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float ix = D(0, c), iy = D(1, c), iz = D(2, c);
        const float tt = t / nc[c];
        A11 += tt * ix * ix;
        B1 -= tt * iz * ix;
        if (NOP == 2) {
          A12 += tt * ix * iy;
          A22 += tt * iy * iy;
          B2 -= tt * iz * iy;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float ixx = D(3, c), ixy = D(4, c), iyy = D(5, c), ixz = D(6, c), iyz = D(7, c);
      ng[2 * c] = ixx * ixx + ixy * ixy + DATANORM;
      ng[2 * c + 1] = iyy * iyy + ixy * ixy + DATANORM;
      tg[2 * c] = (NOP == 2) ? ixz + ixx * u + ixy * v : ixz + ixx * u;
      tg[2 * c + 1] = (NOP == 2) ? iyz + ixy * u + iyy * v : iyz + ixy * u;
    }
    acc = tg[0] * tg[0] / ng[0] + tg[1] * tg[1] / ng[1] + tg[2] * tg[2] / ng[2] + tg[3] * tg[3] / ng[3] +
          tg[4] * tg[4] / ng[4] + tg[5] * tg[5] / ng[5] + EPS_GRAD;
    t = m * hgo3 / sqrtf(acc);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float ixx = D(3, c), ixy = D(4, c), iyy = D(5, c), ixz = D(6, c), iyz = D(7, c);
      const float ta = t / ng[2 * c], tb = t / ng[2 * c + 1];
      A11 += ta * ixx * ixx + tb * ixy * ixy;
      B1 -= ta * ixx * ixz + tb * ixy * iyz;
      if (NOP == 2) {
        A12 += ta * ixx * ixy + tb * ixy * iyy;
        A22 += tb * iyy * iyy + ta * ixy * ixy;
        B2 -= tb * iyy * iyz + ta * ixy * ixz;
      }
    }
  }

  // sub_laplacian (opticalflow_aux.c:172-199), per-pixel order -h(i-1) +h(i) -v(j-1) +v(j)
  {
    const float wxc = fc[0];
    if (i > 0) B1 -= hl * (wxc - fc[-NOP]);
    if (i < w - 1) B1 += hh * (fc[NOP] - wxc);
    if (j > 0) B1 -= vt * (wxc - fc[-w * NOP]);
    if (j < h - 1) B1 += vv * (fc[w * NOP] - wxc);
    if (NOP == 2) {
      const float wyc = fc[1];
      if (i > 0) B2 -= hl * (wyc - fc[-NOP + 1]);
      if (i < w - 1) B2 += hh * (fc[NOP + 1] - wyc);
      if (j > 0) B2 -= vt * (wyc - fc[-w * NOP + 1]);
      if (j < h - 1) B2 += vv * (fc[w * NOP + 1] - wyc);
    }
  }

  if (NOP == 2) {
    // solver.c:115-120 (+ twins for first/last line): invert the 2x2 block
    float dps;
    if (j == 0) dps = hl + hh + vv;
    else if (j == h - 1) dps = hl + hh + vt;
    else dps = hl + hh + vt + vv;
    const float iA11 = A22 + dps, iA22 = A11 + dps;
    const float det = iA11 * iA22 - A12 * A12;
    // record fields: a11^-1, a12^-1, a22^-1, b1, b2, sh, sv, sv(row above); two float4 per pixel in the lane and
    // the band layouts, one float per field in the fast mode's natural layout
    if (!fast) {
      float4* const r4 = reinterpret_cast<float4*>(rec);
      r4[0] = make_float4(iA11 / det, A12 / -det, iA22 / det, B1);
      r4[lane ? 32 : 1] = make_float4(B2, hh, vv, vt);
    } else {
    rec[0] = iA11 / det;
    rec[fs] = A12 / -det;
    rec[2 * fs] = iA22 / det;
    rec[3 * fs] = B1;
    rec[4 * fs] = B2;
    rec[5 * fs] = hh;
    rec[6 * fs] = vv;
    rec[7 * fs] = vt;
    }
  } else {
    // sor_coupled_slow_but_readable_DE (solver.c:438-460): A11 = a11 + sum_dpsis (top,left,bottom,right)
    float sum = 0.0f;
    if (j > 0) sum += vt;
    if (i > 0) sum += hl;
    if (j < h - 1) sum += vv;
    if (i < w - 1) sum += hh;
    // stereo record fields: A11 = a11 + sum, b1, sh, sv, sv(row above)
    if (lane) {
      float4* const r4 = reinterpret_cast<float4*>(rec);
      r4[0] = make_float4(A11 + sum, B1, hh, vv);
      r4[32] = make_float4(vt, 0.f, 0.f, 0.f);
    } else {
    rec[0] = A11 + sum;
    rec[fs] = B1;
    rec[2 * fs] = hh;
    rec[3 * fs] = vv;
    rec[4 * fs] = vt;
    }
  }
}

// Records and (du,dv) of pixel (x,y).  Exact mode: the band-skewed lane rows (band_f4): flow records are two float4
// per pixel, stereo records one float4 per field of the block's 4 pixels (band_rec_f); du is chunk nq of the block, dv
// chunk nq+1.  Fast mode (red-black SOR): natural layout, 8 floats per pixel, (du,dv) in the current ping-pong planes.
// Lane mode (sor_lane_kernel): lane-skewed layout, the record is two float4 (lane_rec_f4), (du,dv) one float2.
template <int MODE>
struct RecLayout {
  static constexpr bool fast = (MODE == 1), lane = (MODE == 2);
  float* rec;
  float* dudv;
  int dv_off;  // from du to dv
  __device__ __forceinline__ RecLayout(const VarRefPlanes& pl, int fr) {
    rec = fast ? pl.frec + (size_t)fr * pl.frec_stride : reinterpret_cast<float*>(pl.rec + (size_t)fr * pl.rec_stride);
    dudv = fast ? pl.fdu + (size_t)fr * pl.fdu_stride + (size_t)pl.fcur * 2 * pl.plane : rec;
    dv_off = lane ? 1 : (fast ? (int)pl.plane : 4);
  }
  __device__ __forceinline__ static int rec_idx(const VarRefPlanes& pl, int pitch, int x, int y) {
    return lane ? (int)lane_rec_f4(pl, x, y, 0) * 4 : (fast ? (y * pitch + x) * 8 : (int)band_rec_f(pl, x, y, 0));
  }
  __device__ __forceinline__ static int du_idx(const VarRefPlanes& pl, int pitch, int x, int y) {
    return lane ? (int)lane_dudv_f(pl, x, y) : (fast ? y * pitch + x : (int)band_f4(pl, x >> 2, y, pl.nq) * 4 + (x & 3));
  }
};

// ---------------------------------------------------------------------------
// The set-up of a level and its first inner iteration, per tile of 32 x 8R pixels: image_warp (opticalflow_aux.c:
// 17-60) on the padded interleaved I1 with the first loop of get_derivatives (:80-84), the derivative planes of
// get_derivatives (:86-92) and the mask; with n_inner > 0 also the records of the first inner iteration (du = dv = 0,
// uu = w: refine_variational.cpp:181-190), and (du,dv) reset to zero, which the SOR's first sweep reads.  The warp
// runs over the tile + 4, Ix over the tile + 2, Iy over the tile + 2 rows, in shared memory.  Every stage holds at a
// position outside the level the value of the clamped pixel, which is the replicate border of the horizontal 5-tap
// derivatives; the vertical ones fold their coefficients by global row (conv_v5).  RGB runs the stages once per
// channel on the same buffers and reads the derivative planes it wrote back for the data term.
template <int C, int NOP, int R, int MODE>
__global__ void __launch_bounds__(TX * TY) varref_setup_kernel(LevelGeom g, VarRefPlanes pl, VarRefParams vp, int f0) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  constexpr int TH = TY * R, SW = TX + 8, SH = TH + 8;
  __shared__ float2 s_uv[SH][SW];  // w over the tile + 4
  __shared__ float s_iz[SH][SW];   // I1w - I0 over the tile + 4
  __shared__ union {
    float avg[SH][SW];             // 0.5 * (I1w + I0) over the tile + 4, dead once Ix and Iy exist
    float s[TH + 2][TX + 2];       // then the smoothness weights over the tile + 1
  } s_a;
  __shared__ float s_ix[TH + 4][TX + 4], s_iy[TH + 4][TX];
  const int fr = blockIdx.z, frame = frame_of(g, f0, fr);
  const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TH;
  const int tid = threadIdx.y * TX + threadIdx.x;
  const int w = g.w, h = g.h, pitch = g.pitch;
  const float* const flow = g.flow + (size_t)frame * g.flow_frame_stride;
  const Coef5 c5 = coef5();

  for (int idx = tid; idx < SH * SW; idx += TX * TY) {
    const int cy = idx / SW, cx = idx - cy * SW;
    const float* f = flow + (clampi(y0 - 4 + cy, h) * w + clampi(x0 - 4 + cx, w)) * NOP;
    float2 uv;
    uv.x = f[0];
    uv.y = (NOP == 2) ? f[1] : 0.0f;
    s_uv[cy][cx] = uv;
  }

  const int i = x0 + threadIdx.x;
  const float* const i1 = g.img[3] + (size_t)frame * g.img_fs[3];
  const float* const i0 = g.img[0] + (size_t)frame * g.img_fs[0];
  // the 8 derivatives of pixel (i, j) of channel c: written to their planes and returned in d
  auto derivs = [&](int c, int j, float* d) {
    const int sx = i - x0, sy = j - y0;
    d[0] = s_ix[sy + 2][sx + 2];
    d[1] = s_iy[sy + 2][sx];
    d[2] = s_iz[sy + 4][sx + 4];
    d[3] = conv_h5s(s_ix[sy + 2], x0 - 2, w, i, c5);
    d[4] = conv_v5(&s_ix[sy + 2][sx + 2], TX + 4, h, j, c5);
    d[5] = conv_v5(&s_iy[sy + 2][sx], TX, h, j, c5);
    d[6] = conv_h5s(s_iz[sy + 4], x0 - 4, w, i, c5);
    d[7] = conv_v5(&s_iz[sy + 4][sx + 4], SW, h, j, c5);
    const size_t po = ((size_t)fr * C + c) * pl.plane + j * pitch + i;
#pragma unroll
    for (int k = 0; k < 8; ++k) pl.deriv[k][po] = d[k];
  };
  for (int c = 0; c < C; ++c) {
    __syncthreads();  // w is staged; the previous channel's stages are read
    for (int idx = tid; idx < SH * SW; idx += TX * TY) {
      const int cy = idx / SW, cx = idx - cy * SW;
      const int px = clampi(x0 - 4 + cx, w), py = clampi(y0 - 4 + cy, h);
      const float2 fl = s_uv[cy][cx];
      const float xx = px + fl.x, yy = py + fl.y;
      const int x = (int)floorf(xx), y = (int)floorf(yy);
      const float dx = xx - x, dy = yy - y;
      const int x1 = clampi(x, w), x2 = clampi(x + 1, w), y1 = clampi(y, h), y2 = clampi(y + 1, h);
      const float s11 = i1[((y1 + g.pad) * g.tmp_w + x1 + g.pad) * C + c];
      const float s12 = i1[((y1 + g.pad) * g.tmp_w + x2 + g.pad) * C + c];
      const float s21 = i1[((y2 + g.pad) * g.tmp_w + x1 + g.pad) * C + c];
      const float s22 = i1[((y2 + g.pad) * g.tmp_w + x2 + g.pad) * C + c];
      const float wv = s11 * (1.0f - dx) * (1.0f - dy) + s12 * dx * (1.0f - dy) + s21 * (1.0f - dx) * dy +
                       s22 * dx * dy;
      const float im1 = i0[((py + g.pad) * g.tmp_w + px + g.pad) * C + c];
      s_a.avg[cy][cx] = 0.5f * (wv + im1);
      s_iz[cy][cx] = wv - im1;
    }
    __syncthreads();
    for (int idx = tid; idx < (TH + 4) * (TX + 4); idx += TX * TY) {
      const int cy = idx / (TX + 4), cx = idx - cy * (TX + 4);
      const int px = clampi(x0 - 2 + cx, w), py = clampi(y0 - 2 + cy, h);
      const int sy = py - y0 + 4;
      s_ix[cy][cx] = conv_h5s(s_a.avg[sy], x0 - 4, w, px, c5);
      if (cx >= 2 && cx < TX + 2) s_iy[cy][cx - 2] = conv_v5(&s_a.avg[sy][px - x0 + 4], SW, h, py, c5);
    }
    __syncthreads();
    if (C > 1 && i < w) {
#pragma unroll 1
      for (int rr = 0; rr < R; ++rr) {
        const int j = y0 + threadIdx.y + TY * rr;
        if (j >= h) break;
        float d[8];
        derivs(c, j, d);
      }
    }
  }
  if (vp.n_inner > 0) {
    smoothness_tile<TH, SW>(s_uv, s_a.s, 4, x0, y0, w, h, vp.quarter_alpha, tid);
    __syncthreads();
  }

  if (i >= w) return;
  const RecLayout<MODE> L(pl, fr);
#pragma unroll 1
  for (int rr = 0; rr < R; ++rr) {
  const int ly = threadIdx.y + TY * rr, j = y0 + ly;
  if (j >= h) break;
  const int o = j * pitch + i;
  float d[8];
  if (C == 1) derivs(0, j, d);
  const float2 fl = s_uv[ly + 4][threadIdx.x + 4];
  const float xx = i + fl.x, yy = j + fl.y;
  const float m = (xx >= 0 && xx <= g.w - 1 && yy >= 0 && yy <= g.h - 1) ? 1.0f : 0.0f;
  pl.mask[(size_t)fr * pl.plane + o] = m;
  if (vp.n_inner == 0) continue;

  const int cx = threadIdx.x + 1, cy = ly + 1;
  const float sc = s_a.s[cy][cx];
  const float hh = (i < w - 1) ? sc + s_a.s[cy][cx + 1] : 0.0f;  // sh(i,j)   (opticalflow_aux.c:150-154)
  const float hl = (i > 0) ? s_a.s[cy][cx - 1] + sc : 0.0f;      // sh(i-1,j)
  const float vv = (j < h - 1) ? sc + s_a.s[cy + 1][cx] : 0.0f;  // sv(i,j)   (:159-163)
  const float vt = (j > 0) ? s_a.s[cy - 1][cx] + sc : 0.0f;      // sv(i,j-1)
  // the first inner iteration starts from du = dv = 0 and resets the stored values (refine_variational.cpp:181-182).
  // The last thread of a row also clears the columns >= w of the row's last block, which the exact SOR updates but
  // nobody reads.
  const int bd = L.du_idx(pl, pitch, i, j);
  L.dudv[bd] = 0.0f;
  L.dudv[bd + L.dv_off] = 0.0f;
  if (MODE == 0 && i == w - 1)
    for (int t = (i & 3) + 1; t < 4; ++t) L.dudv[bd + t - (i & 3)] = L.dudv[bd + 4 + t - (i & 3)] = 0.0f;
  // gray: this pixel's derivatives in registers; RGB: the planes this thread wrote
  auto D = [&](int k, int c) { return C == 1 ? d[k] : pl.deriv[k][((size_t)fr * C + c) * pl.plane + o]; };
  pixel_record<C, NOP, MODE>(D, 0.0f, 0.0f, m, hh, hl, vv, vt, flow + (j * w + i) * NOP, i, j, w, h, vp,
                             L.rec + L.rec_idx(pl, pitch, i, j));
  }  // rows of this thread
}

// The later inner iterations (uu = w + du): R rows per thread (tile 32 x 8R): the halo work of the two staging
// phases -- (TH+4)x36 flow values and (TH+2)x34 smoothness weights per 32 x TH pixels -- shrinks from 1.69x / 1.33x
// (R=1) to 1.27x / 1.13x (R=4).  All indices inside a frame are 32-bit.
// MODE: 0 = records for sor_wave_kernel (band_f4 lane rows), 1 = fast mode (natural layout), 2 = sor_lane_kernel
// (lane-skewed layout); a template parameter so that the layout arithmetic of the other modes costs nothing.
template <int C, int NOP, int R, int MODE>
__global__ void __launch_bounds__(TX * TY) assemble_kernel(LevelGeom g, VarRefPlanes pl, VarRefParams vp, int f0) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  constexpr int TH = TY * R;
  __shared__ float2 s_uv[TH + 4][TX + 4];
  __shared__ float s_s[TH + 2][TX + 2];
  const int fr = blockIdx.z, frame = frame_of(g, f0, fr);
  const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TH;
  const int tid = threadIdx.y * TX + threadIdx.x;
  const int w = g.w, h = g.h, pitch = g.pitch;
  const float* const flow = g.flow + (size_t)frame * g.flow_frame_stride;
  const RecLayout<MODE> L(pl, fr);

  // uu = wx + du (vv likewise) (refine_variational.cpp:189-190).  Coordinates are clamped, which also realises the
  // replicate border of the 3-tap horizontal derivative (image.c:448-454).
  for (int idx = tid; idx < (TH + 4) * (TX + 4); idx += TX * TY) {
    const int cy = idx / (TX + 4), cx = idx - cy * (TX + 4);
    const int gx = clampi(x0 - 2 + cx, w), gy = clampi(y0 - 2 + cy, h);
    const float* f = flow + (gy * w + gx) * NOP;
    float2 uv;
    uv.x = f[0];
    uv.y = (NOP == 2) ? f[1] : 0.0f;
    const int b = L.du_idx(pl, pitch, gx, gy);
    const float dx = L.dudv[b];
    if (NOP == 2) {
      uv.x = uv.x + dx;
      uv.y = uv.y + L.dudv[b + L.dv_off];
    } else {  // minps / maxps with zero (refine_variational.cpp:299-314)
      const float t = uv.x + dx;
      uv.x = (camlr_of(g, frame) == 0) ? (t < 0.0f ? t : 0.0f) : (t > 0.0f ? t : 0.0f);
    }
    s_uv[cy][cx] = uv;
  }
  __syncthreads();
  smoothness_tile<TH, TX + 4>(s_uv, s_s, 2, x0, y0, w, h, vp.quarter_alpha, tid);
  __syncthreads();

  const int i = x0 + threadIdx.x;
  if (i >= w) return;
  const float* const maskp = pl.mask + (size_t)fr * pl.plane;

#pragma unroll 1
  for (int rr = 0; rr < R; ++rr) {
  const int ly = threadIdx.y + TY * rr, j = y0 + ly;
  if (j >= h) break;
  const int cx = threadIdx.x + 1, cy = ly + 1;
  const float sc = s_s[cy][cx];
  const float hh = (i < w - 1) ? sc + s_s[cy][cx + 1] : 0.0f;    // sh(i,j)   (opticalflow_aux.c:150-154)
  const float hl = (i > 0) ? s_s[cy][cx - 1] + sc : 0.0f;        // sh(i-1,j)
  const float vv = (j < h - 1) ? sc + s_s[cy + 1][cx] : 0.0f;    // sv(i,j)   (:159-163)
  const float vt = (j > 0) ? s_s[cy - 1][cx] + sc : 0.0f;        // sv(i,j-1)

  const int o = j * pitch + i;
  const int bd = L.du_idx(pl, pitch, i, j);
  const float u = L.dudv[bd], v = (NOP == 2) ? L.dudv[bd + L.dv_off] : 0.0f;
  auto D = [&](int k, int c) { return pl.deriv[k][((size_t)fr * C + c) * pl.plane + o]; };
  pixel_record<C, NOP, MODE>(D, u, v, maskp[o], hh, hl, vv, vt, flow + (j * w + i) * NOP, i, j, w, h, vp,
                             L.rec + L.rec_idx(pl, pitch, i, j));
  }  // rows of this thread
}

// ---------------------------------------------------------------------------
// Shared-memory access helpers of the SOR kernel (explicit 128-bit forms).
__device__ __forceinline__ float4 lds128(unsigned addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
// predicated forms: lanes without a block issue no shared-memory wavefronts.  The result registers of such a
// lane keep whatever they held (no zero-fill: 44 CS2R per super-step); its arithmetic runs on that garbage and
// is never stored, and no branch of the kernel depends on data of a lane without a block.
__device__ __forceinline__ float4 lds128_if(bool p, unsigned addr) {
  float4 v;
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %5, 0;\n\t@q ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];\n\t}"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(addr), "r"((unsigned)p)
               : "memory");
  return v;
}
__device__ __forceinline__ float lds32_if(bool p, unsigned addr) {
  float v;
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q ld.shared.f32 %0, [%1];\n\t}" : "=f"(v) : "r"(addr), "r"((unsigned)p) : "memory");
  return v;
}
__device__ __forceinline__ void sts128_if(bool p, unsigned addr, const float4& v) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %5, 0;\n\t@q st.shared.v4.f32 [%0], {%1,%2,%3,%4};\n\t}" ::"r"(addr), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w), "r"((unsigned)p)
               : "memory");
}
__device__ __forceinline__ void sts128(unsigned addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

#include "sor_wave_kernel.cuh"
#include "sor_lane_kernel.cuh"
#include "sor_redblack_kernel.cuh"

// K12 at the end of the level: flow = w + dw (refine_variational.cpp:210-221; stereo clamp
// :299-314).  Kept out of the SOR kernel: the flow array is row-major per frame, so reading it
// from one-thread-per-row SOR lanes costs 32 cache lines per load instruction.
template <int NOP>
__global__ void __launch_bounds__(256) flow_update_kernel(LevelGeom g, VarRefPlanes pl, int f0) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
  const int fr = blockIdx.z, frame = frame_of(g, f0, fr);
  if (i >= g.w || j >= g.h) return;
  const bool fast = pl.fast != 0, lane = pl.lane != 0;
  const float* dudv = fast ? pl.fdu + (size_t)fr * pl.fdu_stride + (size_t)pl.fcur * 2 * pl.plane
                           : reinterpret_cast<const float*>(pl.rec + (size_t)fr * pl.rec_stride);
  const size_t b = lane ? lane_dudv_f(pl, i, j) : (fast ? (size_t)j * g.pitch + i : band_f4(pl, i >> 2, j, pl.nq) * 4 + (i & 3));
  const size_t dv_off = lane ? 1 : (fast ? pl.plane : 4);
  float* f = g.flow + (size_t)frame * g.flow_frame_stride + ((size_t)j * g.w + i) * NOP;
  if (NOP == 2) {
    const float2 wv = *reinterpret_cast<const float2*>(f);
    *reinterpret_cast<float2*>(f) = make_float2(wv.x + dudv[b], wv.y + dudv[b + dv_off]);
  } else {
    const float t = f[0] + dudv[b];
    f[0] = (camlr_of(g, frame) == 0) ? (t < 0.0f ? t : 0.0f) : (t > 0.0f ? t : 0.0f);
  }
}

}  // namespace

// Opt-in of `smem` bytes of dynamic shared memory for `kern` on the current device (and, with `nonportable`, of
// clusters of more than 8 CTAs).  The attributes belong to the kernel, so the cache is keyed by device and kernel:
// it only ever raises a kernel's setting, whichever of the launches that share the kernel (gray and RGB levels,
// contexts of other patch sizes, sor_max_cluster_size) comes first.  A cache per launcher once let an RGB level that
// needed less shared memory lower the setting behind a gray level's cache, and the gray level's next larger launch
// failed.  Setting the attribute to each launch's own size would fail the same way across contexts: another thread's
// smaller launch can lower it between this thread's set and launch, and a graph captured at the larger size can be
// replayed after it.
cudaError_t smem_optin(const void* kern, size_t smem, bool nonportable) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, std::pair<size_t, bool>> done;  // (device, kernel) -> (smem, nonportable)
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  std::pair<size_t, bool>& d = done[{dev, kern}];
  if (d.first < smem) {
    if ((e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
    d.first = smem;
  }
  if (nonportable && !d.second) {
    if ((e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1)) != cudaSuccess) return e;
    d.second = true;
  }
  return cudaSuccess;
}

// Can a sor_wave_kernel CTA of `hpad` lanes keep K sweeps in flight: K * hpad compute threads + the producer warp
// within the kernel's launch bound, stage ring + board within the shared memory of an SM?
constexpr bool sor_wave_fits(int nop, int hpad, int rt, int K) {
  return K * hpad + 32 <= sor_max_threads(hpad) && sor_smem_bytes(nop, hpad, rt, K, hpad) <= SMEM_OPTIN_MAX;
}
// band of a chain plan: the largest that fits one sweep; the only chain instantiation per (nop, rt)
constexpr int sor_chain_hpad(int nop, int rt) {
  int p = 256;
  while (p > 32 && !sor_wave_fits(nop, p, rt, 1)) p /= 2;
  return p;
}

bool sor_plan(const LevelGeom& L, int K, const SorOptions& o, int frames, const VarRefPlanes& buffers, SorPlan* plan) {
  SorPlan p{};
  VarRefPlanes& pl = p.pl;
  pl = buffers;
  const int nop = L.nop, rt = o.rt, k1 = K < 1 ? 1 : K;
  const int lanes = (L.h + rt - 1) / rt;  // lanes the whole level needs
  int hpad = 0;
  // all K sweeps in flight if some band size allows it, else as many as the band found for one sweep holds
  for (int kk = k1; !hpad; kk = 1) {
    for (int q = 32; q <= 128 && !hpad; q *= 2)
      if (lanes <= q && lanes <= o.single_max && sor_wave_fits(nop, q, rt, kk)) hpad = q;
    for (int q = 32; q <= 256 && !hpad; q *= 2)
      if (lanes > q && (lanes + q - 1) / q <= o.max_cluster && sor_wave_fits(nop, q, rt, kk)) hpad = q;
    if (kk == 1) break;
  }
  pl.chain = !hpad;
  if (pl.chain) hpad = sor_chain_hpad(nop, rt);
  if (!sor_wave_fits(nop, hpad, rt, 1)) return false;
  pl.hpad = hpad;
  pl.rt = rt;
  pl.rtshift = rt == 1 ? 0 : (rt == 2 ? 1 : 2);
  pl.hbshift = (hpad == 32 ? 5 : (hpad == 64 ? 6 : (hpad == 128 ? 7 : 8))) + pl.rtshift;
  pl.nb = (lanes + hpad - 1) / hpad;
  pl.ndiag = (L.w + 3) / 4 + hpad + 2;
  pl.nq = nop == 2 ? 8 : 5;
  pl.lpitch = sor_lane_pitch(nop, rt);
  pl.rec_stride = (size_t)pl.nb * pl.ndiag * pl.hpad * pl.lpitch;
  pl.lane = 0;
  pl.fast = o.fast;
  pl.plane = (size_t)L.pitch * L.h;
  pl.frec_stride = pl.plane * 8;  // fast mode: natural layout at this level's plane size
  pl.fdu_stride = pl.plane * 4;
  p.kind = pl.chain ? SOR_WAVE_CHAIN : (pl.nb > 1 ? SOR_WAVE_CLUSTER : SOR_WAVE_SINGLE);
  p.sweeps = pl.chain ? 1 : k1;  // a chain runs one sweep per launch
  while (p.sweeps > 1 && !sor_wave_fits(nop, hpad, rt, p.sweeps)) --p.sweeps;
  p.ml = sor_stage_lanes(hpad, rt, L.w, L.h, p.kind != SOR_WAVE_SINGLE);
  // sor_lane_kernel, bands of 32 rows.  By default where it beats the block wavefront (tools/lane_ab.py): one or two
  // bands with all sweeps in one launch.  Every further band adds 33 steps of start-up skew, which makes taller
  // levels slower with it.
  const int nb32 = (L.h + 31) / 32, kl32 = sl_sweeps_per_launch(nb32, K);
  if (!o.fast && kl32 >= 1 &&
      (o.lane == 1 || (o.lane == 2 && frames <= SOR_LANE_AUTO_FRAMES && nb32 <= 2 && kl32 >= k1))) {
    p.kind = SOR_LANE;
    pl.lane = 1;
    pl.nb = nb32;
    pl.ndiag = lane_ndiag(L.w);
    pl.rec_stride = lane_frame_f4(L.w, L.h);
    p.sweeps = kl32;
  }
  if (o.fast) {  // sor_redblack_kernel: all K sweeps in one launch
    p.kind = SOR_REDBLACK;
    p.sweeps = k1;
  }
  auto smem = [&](int k) {
    return p.kind == SOR_REDBLACK ? rb_smem_bytes(nop, k)
                                  : (p.kind == SOR_LANE ? sl_smem_bytes(nb32, k) : sor_smem_bytes(nop, hpad, rt, k, p.ml));
  };
  p.smem = smem(p.sweeps);
  p.tail_smem = K % p.sweeps > 0 ? smem(K % p.sweeps) : p.smem;
  p.chain_nb = p.kind == SOR_WAVE_CHAIN ? pl.nb : 0;
  if (p.kind == SOR_REDBLACK && (K < 1 || p.smem > SMEM_OPTIN_MAX)) return false;  // the tile's halo grows with K
  *plan = p;
  return true;
}

// assemble_kernel: as many rows per thread (less halo work) as still leave >= 256 CTAs
int assemble_rows_per_thread(int w, int h, int frames) {
  const long tiles_x = (w + TX - 1) / TX;
  for (int r = 4; r > 1; r >>= 1)
    if (tiles_x * ((h + TY * r - 1) / (TY * r)) * frames >= 256) return r;
  return 1;
}

template <int NOP, int HPAD, int RT, int BM>
static cudaError_t launch_sor_t(const LevelGeom& g, const SorPlan& p, const VarRefParams& vp, int nf, int kk,
                                size_t smem, cudaStream_t st, int* sync, unsigned long long* div_fb) {
  constexpr bool CL = (BM == SOR_CLUSTER);
  auto kern = sor_wave_kernel<NOP, HPAD, RT, BM>;
  const cudaError_t e = smem_optin((const void*)kern, smem, CL);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(nf * (BM != SOR_SINGLE ? p.pl.nb : 1)));
  cfg.blockDim = dim3((unsigned)(kk * HPAD + 32));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (CL) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = (unsigned)p.pl.nb;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (g.pdl) {  // see pdl_wait (ofdis_internal.cuh)
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, g, p.pl, vp, kk, p.ml, sync, div_fb);
}

template <int NOP, int RT>
static cudaError_t launch_sor_rt(const LevelGeom& g, const SorPlan& p, const VarRefParams& vp, int nf, int kk,
                                 size_t smem, cudaStream_t st, int* sync, unsigned long long* div_fb) {
  if (p.kind == SOR_WAVE_CHAIN) {
    constexpr int HC = sor_chain_hpad(NOP, RT);
    if (p.pl.hpad != HC || kk != 1 || !sync) return cudaErrorInvalidValue;
    return launch_sor_t<NOP, HC, RT, SOR_CHAIN>(g, p, vp, nf, kk, smem, st, sync, div_fb);
  }
  const bool cl = p.kind == SOR_WAVE_CLUSTER;
  constexpr int C1 = SOR_CLUSTER, S1 = SOR_SINGLE;
  switch (p.pl.hpad) {
    case 32: return cl ? launch_sor_t<NOP, 32, RT, C1>(g, p, vp, nf, kk, smem, st, sync, div_fb) : launch_sor_t<NOP, 32, RT, S1>(g, p, vp, nf, kk, smem, st, sync, div_fb);
    case 64: return cl ? launch_sor_t<NOP, 64, RT, C1>(g, p, vp, nf, kk, smem, st, sync, div_fb) : launch_sor_t<NOP, 64, RT, S1>(g, p, vp, nf, kk, smem, st, sync, div_fb);
    case 128: return cl ? launch_sor_t<NOP, 128, RT, C1>(g, p, vp, nf, kk, smem, st, sync, div_fb) : launch_sor_t<NOP, 128, RT, S1>(g, p, vp, nf, kk, smem, st, sync, div_fb);
    case 256: return cl ? launch_sor_t<NOP, 256, RT, C1>(g, p, vp, nf, kk, smem, st, sync, div_fb) : launch_sor_t<NOP, 256, RT, S1>(g, p, vp, nf, kk, smem, st, sync, div_fb);
  }
  return cudaErrorInvalidValue;
}

template <int NOP>
static cudaError_t launch_sor(const LevelGeom& g, const SorPlan& p, const VarRefParams& vp, int nf, int kk, size_t smem,
                              cudaStream_t st, int* sync, unsigned long long* div_fb) {
  if (p.pl.rt == 1) return launch_sor_rt<NOP, 1>(g, p, vp, nf, kk, smem, st, sync, div_fb);
  if (p.pl.rt == 2) return launch_sor_rt<NOP, 2>(g, p, vp, nf, kk, smem, st, sync, div_fb);
  if (p.pl.rt == 4) return launch_sor_rt<NOP, 4>(g, p, vp, nf, kk, smem, st, sync, div_fb);
  return cudaErrorInvalidValue;
}

// varref_setup_kernel and assemble_kernel share the grid and the instance rule: (C, NOP, rows per thread, the layout
// of the level's SOR plan)
using TileKernel = void (*)(LevelGeom, VarRefPlanes, VarRefParams, int);
template <int C, int NOP, int MODE>
static TileKernel tile_kernel(bool setup, int rows) {
  if (rows == 4) return setup ? varref_setup_kernel<C, NOP, 4, MODE> : assemble_kernel<C, NOP, 4, MODE>;
  if (rows == 2) return setup ? varref_setup_kernel<C, NOP, 2, MODE> : assemble_kernel<C, NOP, 2, MODE>;
  return setup ? varref_setup_kernel<C, NOP, 1, MODE> : assemble_kernel<C, NOP, 1, MODE>;
}
template <int C, int NOP>
static TileKernel tile_kernel(bool setup, int rows, const VarRefPlanes& pl) {
  if (pl.fast) return tile_kernel<C, NOP, 1>(setup, rows);
  if (pl.lane) return tile_kernel<C, NOP, 2>(setup, rows);
  return tile_kernel<C, NOP, 0>(setup, rows);
}

template <int C, int NOP>
static int launch_varref_t(const LevelGeom& g, const SorPlan& plan, const VarRefParams& vp, int f0, int f1,
                           cudaStream_t st, Profiler* prof, int* chain_sync, unsigned long long* div_fb) {
  VarRefPlanes pl = plan.pl;  // fast mode toggles the (du,dv) ping-pong buffer
  const bool pdl = g.pdl != 0 && prof == nullptr;  // the profiler's events between launches would serialise them anyway
  pl.fcur = 0;
  int launches = 0;
  const int nf = f1 - f0;
  const dim3 block(TX, TY), grid((g.w + TX - 1) / TX, (g.h + TY - 1) / TY, nf);
  const int rows_per_thread = assemble_rows_per_thread(g.w, g.h, nf);
  const dim3 grid_a(grid.x, (g.h + TY * rows_per_thread - 1) / (TY * rows_per_thread), nf);
  {  // derivatives, mask and the first inner iteration's records
    ProfScope scope(prof, KC_VR_SETUP);
    launch_k(pdl, tile_kernel<C, NOP>(true, rows_per_thread, pl), grid_a, block, 0, st, g, pl, vp, f0);
  }
  ++launches;
  // SOR: the launches of the level's plan (sor_plan); the sweeps are sequential, so K sweeps in ceil(K / sweeps)
  // launches give the same result
  const int K = vp.n_solver;
  for (int it = 0; it < vp.n_inner; ++it) {
    if (it > 0) {
      ProfScope scope(prof, KC_VR_ASSEMBLE);
      launch_k(pdl, tile_kernel<C, NOP>(false, rows_per_thread, pl), grid_a, block, 0, st, g, pl, vp, f0);
      ++launches;
    }
    for (int s = 0; s < K; s += plan.sweeps) {
      ProfScope scope(prof, KC_VR_SOR);
      const int kk = (K - s < plan.sweeps) ? K - s : plan.sweeps;
      const size_t smem = kk == plan.sweeps ? plan.smem : plan.tail_smem;
      cudaError_t e;
      if (plan.kind == SOR_REDBLACK) {  // opt-in red-black solver, (du,dv) ping-pong
        const dim3 grid_rb((g.w + RB_TILE - 1) / RB_TILE, (g.h + RB_TILE - 1) / RB_TILE, nf);
        if ((e = smem_optin((const void*)sor_redblack_kernel<NOP>, smem, false)) == cudaSuccess)
          e = launch_k(pdl, sor_redblack_kernel<NOP>, grid_rb, dim3(256), smem, st, g, pl, vp);
      } else if (plan.kind == SOR_LANE) {  // pixel wavefront, warps synchronised through shared-memory flags
        if ((e = smem_optin((const void*)sor_lane_kernel<NOP>, smem, false)) == cudaSuccess)
          e = launch_k(pdl, sor_lane_kernel<NOP>, dim3(nf), dim3(pl.nb * kk * 32), smem, st, g, pl, vp, kk, div_fb);
      } else {
        e = launch_sor<NOP>(g, plan, vp, nf, kk, smem, st, chain_sync, div_fb);
      }
      if (e != cudaSuccess) return -1;
      ++launches;
    }
    pl.fcur ^= pl.fast;
  }
  if (vp.n_inner > 0) {
    ProfScope scope(prof, KC_VR_SETUP);
    launch_k(pdl, flow_update_kernel<NOP>, grid, block, 0, st, g, pl, f0);
    ++launches;
  }
  return cudaGetLastError() == cudaSuccess ? launches : -1;
}

int sor_max_cluster_size() {
  // 16 CTAs is a non-portable cluster size: ask the occupancy calculator whether one such cluster
  // of the largest SOR configuration (256-row bands, one sweep) fits this device
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 8;
  if (cached[dev]) return cached[dev];
  int best = 8;
  auto kern = sor_wave_kernel<2, 128, 1, SOR_CLUSTER>;
  const size_t smem = sor_smem_bytes(2, 128, 1, 3, 128);  // 128-row bands, 3 sweeps in flight: the largest common configuration
  if (smem_optin((const void*)kern, smem, true) == cudaSuccess) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(16);
    cfg.blockDim = dim3(3 * 128 + 32);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 16;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) == cudaSuccess && n >= 1) best = 16;
  }
  cudaGetLastError();  // a refused query must not poison later launches
  cached[dev] = best;
  return best;
}

int launch_varref(const LevelGeom& g, const SorPlan& plan, const VarRefParams& vp, int f0, int f1,
                  cudaStream_t st, Profiler* prof, int* chain_sync, unsigned long long* div_fb) {
  if (g.noc == 1 && g.nop == 2) return launch_varref_t<1, 2>(g, plan, vp, f0, f1, st, prof, chain_sync, div_fb);
  if (g.noc == 3 && g.nop == 2) return launch_varref_t<3, 2>(g, plan, vp, f0, f1, st, prof, chain_sync, div_fb);
  if (g.noc == 1 && g.nop == 1) return launch_varref_t<1, 1>(g, plan, vp, f0, f1, st, prof, chain_sync, div_fb);
  if (g.noc == 3 && g.nop == 1) return launch_varref_t<3, 1>(g, plan, vp, f0, f1, st, prof, chain_sync, div_fb);
  return -1;
}

}  // namespace ofdis

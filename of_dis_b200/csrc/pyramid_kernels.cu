// Image pyramid, gradients and output upsampling on the device -- the callers either side of the
// hot path (SURVEY.md 8f rank 1 and 2): ConstructImgPyramide (run_dense.cpp:130-178), the
// divisibility padding (run_dense.cpp:298-311) and the final resize/crop (run_dense.cpp:407-414).
// Expression order follows of_dis_b200/preprocess.py, which for 8-bit input is bit-identical to
// OpenCV (every intermediate is a dyadic rational that float32 holds exactly).
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

// Level `g.level` of both images of a pair, straight from the 8-bit frames: the 2^l x 2^l box sum
// is exact in int32 and (for l <= 8) in float32, so it equals l successive cv::resize(0.5) steps.
// The divisibility padding (replicate, floor(pad/2) left/top) and the per-level border padding
// (replicate, g.pad) are folded into the index clamps.  One thread per padded destination pixel.
// PYR_PAIRS: s.frames = [pair][2][..], grid.z = 2 x pairs (pair, side).  PYR_SEQ: s.frames = [n + 1][..]
// consecutive frames, grid.z = n + 1; frame t is computed once and stored as I0 of pair t (t < n) and as I1 of
// pair t - 1 (t >= 1).  PYR_BIDIR: as PYR_SEQ, and also as I0 of the backward pair n + t - 1 (t >= 1) and as I1 of
// the backward pair n + t (t < n), pair n + t holding (frame t + 1, frame t).
enum PyrMode { PYR_PAIRS, PYR_SEQ, PYR_BIDIR };

// PYR_BIDIR: the element at offset o of frame t in the pairs that hold it, nullptr where a pair does not exist:
// I0 of pair t, I1 of pair t - 1, I0 of backward pair n + t - 1, I1 of backward pair n + t
__device__ __forceinline__ void bidir_dsts(const LevelGeom& g, int f0, int n, int t, size_t o, float* d[4]) {
  float* i0 = const_cast<float*>(g.img[0]) + o;
  float* i1 = const_cast<float*>(g.img[3]) + o;
  d[0] = t < n ? i0 + (size_t)frame_of(g, f0, t) * g.img_fs[0] : nullptr;
  d[1] = t >= 1 ? i1 + (size_t)frame_of(g, f0, t - 1) * g.img_fs[3] : nullptr;
  d[2] = t >= 1 ? i0 + (size_t)frame_of(g, f0, n + t - 1) * g.img_fs[0] : nullptr;
  d[3] = t < n ? i1 + (size_t)frame_of(g, f0, n + t) * g.img_fs[3] : nullptr;
}

template <int MODE>
__global__ void __launch_bounds__(256) pyr_from_u8_kernel(LevelGeom g, int f0, PyrSourceU8 s, int n) {
  constexpr bool SEQ = MODE != PYR_PAIRS;
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int xp = blockIdx.x * blockDim.x + threadIdx.x, yp = blockIdx.y * blockDim.y + threadIdx.y;
  if (xp >= g.tmp_w || yp >= g.tmp_h) return;
  const int fr = SEQ ? (int)blockIdx.z : (int)(blockIdx.z >> 1), k = blockIdx.z & 1;  // pairs: k 0 = I0, 1 = I1
  const int C = g.noc, sh = g.level, nb = 1 << sh;
  const unsigned char* src = s.frames + (SEQ ? (size_t)fr : (size_t)fr * 2 + k) * s.image_bytes;
  const size_t o = ((size_t)yp * g.tmp_w + xp) * C;
  const int x = clampi(xp - g.pad, g.w), y = clampi(yp - g.pad, g.h);
  const float scale = __int_as_float((127 - 2 * sh) << 23);  // 4^-l
  int sum[3] = {0, 0, 0};
  for (int dy = 0; dy < nb; ++dy) {
    const int Y = clampi((y << sh) + dy - s.pad_top, s.h_org);
    const unsigned char* row = src + (size_t)Y * s.w_org * C;
    for (int dx = 0; dx < nb; ++dx) {
      const int X = clampi((x << sh) + dx - s.pad_left, s.w_org);
      for (int c = 0; c < C; ++c) sum[c] += (int)__ldg(row + X * C + c);
    }
  }
  if constexpr (MODE == PYR_SEQ) {
    float* d0 = fr < n ? const_cast<float*>(g.img[0]) + (size_t)frame_of(g, f0, fr) * g.img_fs[0] + o : nullptr;
    float* d1 = fr >= 1 ? const_cast<float*>(g.img[3]) + (size_t)frame_of(g, f0, fr - 1) * g.img_fs[3] + o : nullptr;
    for (int c = 0; c < C; ++c) {
      const float v = (float)sum[c] * scale;
      if (d0) d0[c] = v;
      if (d1) d1[c] = v;
    }
  } else if constexpr (MODE == PYR_BIDIR) {
    float* d[4];
    bidir_dsts(g, f0, n, fr, o, d);
    for (int c = 0; c < C; ++c) {
      const float v = (float)sum[c] * scale;
      for (int j = 0; j < 4; ++j)
        if (d[j]) d[j][c] = v;
    }
  } else {
    const int arr = k ? 3 : 0;
    float* dst = const_cast<float*>(g.img[arr]) + (size_t)frame_of(g, f0, fr) * g.img_fs[arr] + o;
    for (int c = 0; c < C; ++c) dst[c] = (float)sum[c] * scale;
  }
}

// Border padding of un-padded float images of level g.level ([frame][2][h][w][C], I0 then I1).
__global__ void __launch_bounds__(256) pyr_from_level_kernel(LevelGeom g, int f0, const float* stage) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int xp = blockIdx.x * blockDim.x + threadIdx.x, yp = blockIdx.y * blockDim.y + threadIdx.y;
  if (xp >= g.tmp_w || yp >= g.tmp_h) return;
  const int fr = blockIdx.z >> 1, k = blockIdx.z & 1;
  const int C = g.noc, arr = k ? 3 : 0;
  const float* src = stage + ((size_t)fr * 2 + k) * ((size_t)g.w * g.h * C);
  float* dst = const_cast<float*>(g.img[arr]) + (size_t)frame_of(g, f0, fr) * g.img_fs[arr] + ((size_t)yp * g.tmp_w + xp) * C;
  const int x = clampi(xp - g.pad, g.w), y = clampi(yp - g.pad, g.h);
  for (int c = 0; c < C; ++c) dst[c] = __ldg(src + ((size_t)y * g.w + x) * C + c);
}

// cv::resize(0.5, 0.5, INTER_LINEAR) of an even-sized image == 2x2 box mean (run_dense.cpp:150),
// ((a+b)+(c+d))*0.25 with a,b the even row; reads the interior of the padded level gs, writes
// level gd = gs+1 including its replicate border.  MODE as in pyr_from_u8_kernel: frame t of the n + 1
// consecutive frames reads its finer level from the pair that holds it (I0 of pair t, or I1 of pair n - 1 for
// the last frame) and writes every pair that holds it.
template <int MODE>
__global__ void __launch_bounds__(256) pyr_down_kernel(LevelGeom gs, LevelGeom gd, int f0, int n) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int xp = blockIdx.x * blockDim.x + threadIdx.x, yp = blockIdx.y * blockDim.y + threadIdx.y;
  if (xp >= gd.tmp_w || yp >= gd.tmp_h) return;
  const int C = gd.noc;
  const size_t o = ((size_t)yp * gd.tmp_w + xp) * C;
  const int x = clampi(xp - gd.pad, gd.w), y = clampi(yp - gd.pad, gd.h);
  const size_t so = ((size_t)(2 * y + gs.pad) * gs.tmp_w + (2 * x + gs.pad)) * C;
  if constexpr (MODE == PYR_BIDIR) {
    const int t = blockIdx.z, sa = t < n ? 0 : 3, sf = t < n ? t : t - 1;
    const float* r0 = gs.img[sa] + (size_t)frame_of(gd, f0, sf) * gs.img_fs[sa] + so;
    const float* r1 = r0 + (size_t)gs.tmp_w * C;
    float* d[4];
    bidir_dsts(gd, f0, n, t, o, d);
    for (int c = 0; c < C; ++c) {
      const float v = ((r0[c] + r0[C + c]) + (r1[c] + r1[C + c])) * 0.25f;
      for (int j = 0; j < 4; ++j)
        if (d[j]) d[j][c] = v;
    }
  } else if constexpr (MODE == PYR_SEQ) {
    const int t = blockIdx.z, sa = t < n ? 0 : 3, sf = t < n ? t : t - 1;
    const float* r0 = gs.img[sa] + (size_t)frame_of(gd, f0, sf) * gs.img_fs[sa] + so;
    const float* r1 = r0 + (size_t)gs.tmp_w * C;
    float* d0 = t < n ? const_cast<float*>(gd.img[0]) + (size_t)frame_of(gd, f0, t) * gd.img_fs[0] + o : nullptr;
    float* d1 = t >= 1 ? const_cast<float*>(gd.img[3]) + (size_t)frame_of(gd, f0, t - 1) * gd.img_fs[3] + o : nullptr;
    for (int c = 0; c < C; ++c) {
      const float v = ((r0[c] + r0[C + c]) + (r1[c] + r1[C + c])) * 0.25f;
      if (d0) d0[c] = v;
      if (d1) d1[c] = v;
    }
  } else {
    const int fr = blockIdx.z >> 1, k = blockIdx.z & 1;
    const int arr = k ? 3 : 0;
    const float* r0 = gs.img[arr] + (size_t)frame_of(gd, f0, fr) * gs.img_fs[arr] + so;
    const float* r1 = r0 + (size_t)gs.tmp_w * C;
    float* dst = const_cast<float*>(gd.img[arr]) + (size_t)frame_of(gd, f0, fr) * gd.img_fs[arr] + o;
    for (int c = 0; c < C; ++c) dst[c] = ((r0[c] + r0[C + c]) + (r1[c] + r1[C + c])) * 0.25f;
  }
}

// Gradients of I0 on the device (the first "next" row of SURVEY 8f): cv::Sobel(CV_32F, 3x3,
// scale 1/8, BORDER_DEFAULT = reflect101) on the un-padded level image, zero border of width
// `pad` (run_dense.cpp:156-157,171-172).  Same expression order as of_dis_b200/preprocess.py
// (row difference first, then the [1 2 1]/8 column sum, and vice versa for dy); for images that
// come from 8-bit input every intermediate is exact, so this equals OpenCV bit for bit.
__global__ void __launch_bounds__(256) sobel_kernel(LevelGeom g, int f0) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int xp = blockIdx.x * blockDim.x + threadIdx.x, yp = blockIdx.y * blockDim.y + threadIdx.y;
  const int frame = frame_of(g, f0, blockIdx.z);
  if (xp >= g.tmp_w || yp >= g.tmp_h) return;
  const int C = g.noc, w = g.w, h = g.h, P = g.pad;
  const float* im = g.img[0] + (size_t)frame * g.img_fs[0];
  float* gx = const_cast<float*>(g.img[1]) + (size_t)frame * g.img_fs[1];
  float* gy = const_cast<float*>(g.img[2]) + (size_t)frame * g.img_fs[2];
  const int x = xp - P, y = yp - P;
  const size_t o = ((size_t)yp * g.tmp_w + xp) * C;
  if (x < 0 || y < 0 || x >= w || y >= h) {
    for (int c = 0; c < C; ++c) {
      gx[o + c] = 0.f;
      gy[o + c] = 0.f;
    }
    return;
  }
  auto r101 = [](int v, int n) { return n == 1 ? 0 : (v < 0 ? -v : (v >= n ? 2 * (n - 1) - v : v)); };
  const int xm = r101(x - 1, w) + P, x0 = x + P, xq = r101(x + 1, w) + P;
  const int ym = r101(y - 1, h) + P, y0 = y + P, yq = r101(y + 1, h) + P;
  for (int c = 0; c < C; ++c) {
#define IM(X, Y) im[((size_t)(Y) * g.tmp_w + (X)) * C + c]
    const float t0 = IM(xq, ym) - IM(xm, ym), t1 = IM(xq, y0) - IM(xm, y0), t2 = IM(xq, yq) - IM(xm, yq);
    gx[o + c] = (t0 * 0.125f + t1 * 0.25f) + t2 * 0.125f;
    const float s0 = (IM(xm, ym) * 0.125f + IM(x0, ym) * 0.25f) + IM(xq, ym) * 0.125f;
    const float s2 = (IM(xm, yq) * 0.125f + IM(x0, yq) * 0.25f) + IM(xq, yq) * 0.125f;
    gy[o + c] = s2 - s0;
#undef IM
  }
}

// One thread per full-resolution pixel (upsample_at, ofdis_internal.cuh).
template <int NOP>
__global__ void __launch_bounds__(256) flow_upsample_kernel(LevelGeom g, int f0, float* out, int w_org, int h_org,
                                                            int crop_x, int crop_y) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X >= w_org || Y >= h_org) return;
  const int fr = blockIdx.z;
  const float* fl = g.flow + (size_t)frame_of(g, f0, fr) * g.flow_frame_stride;
  float* o = out + ((size_t)fr * h_org * w_org + (size_t)Y * w_org + X) * NOP;
  upsample_at<NOP>(g, fl, X, Y, crop_x, crop_y, [o](int c, float v) { o[c] = v; });
}

// The full-resolution flow F of flow_upsample_kernel, encoded per pixel (ofdis_get_flow_fullres_encoded; the header
// states the format contract, preprocess.encode_f16 / encode_kitti restate it), float32 without contraction:
//   OFDIS_ENC_F16:   every channel __float2half_rn(F), a NaN of any sign or payload 0x7e00;
//   OFDIS_ENC_KITTI: flow (R, G, B) = (clamp(u * 64 + 32768), clamp(v * 64 + 32768), 1) when neither is NaN, else 0;
//                    stereo d = -F (F where the slot is marked swapped), clamp(d * 256, 1, 65535) when d >= 0, else 0.
// The float32 F itself is never stored.  One thread per full-resolution pixel.
template <int NOP, int ENC>
__global__ void __launch_bounds__(256) flow_encode_kernel(LevelGeom g, int f0, unsigned short* out, int w_org,
                                                          int h_org, int crop_x, int crop_y) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X >= w_org || Y >= h_org) return;
  const int fr = blockIdx.z, frame = frame_of(g, f0, fr);
  const float* fl = g.flow + (size_t)frame * g.flow_frame_stride;
  const size_t o = (size_t)fr * h_org * w_org + (size_t)Y * w_org + X;
  float f[2] = {0.f, 0.f};
  upsample_at<NOP>(g, fl, X, Y, crop_x, crop_y, [&f](int c, float v) { f[c] = v; });
  if constexpr (ENC == OFDIS_ENC_F16) {
    for (int c = 0; c < NOP; ++c)
      out[o * NOP + c] = isnan(f[c]) ? (unsigned short)0x7e00 : __half_as_ushort(__float2half_rn(f[c]));
  } else if constexpr (NOP == 2) {
    const bool valid = !isnan(f[0]) && !isnan(f[1]);
    auto q = [](float x) { return (unsigned short)fminf(fmaxf(x * 64.0f + 32768.0f, 0.0f), 65535.0f); };
    out[o * 3] = valid ? q(f[0]) : (unsigned short)0;
    out[o * 3 + 1] = valid ? q(f[1]) : (unsigned short)0;
    out[o * 3 + 2] = valid ? (unsigned short)1 : (unsigned short)0;
  } else {
    const float d = swapped_of(g, frame) ? f[0] : -f[0];  // KITTI's positive disparity; NaN fails d >= 0, -0 passes
    out[o] = d >= 0.0f ? (unsigned short)fminf(fmaxf(d * 256.0f, 1.0f), 65535.0f) : (unsigned short)0;
  }
}

// Color coding of the full-resolution flow F (ofdis_flow_color_fullres; the header states the contract,
// preprocess.atan2_f32 / flow_to_color / disp_to_color restate it bit for bit).  The tables, built once at compile
// time in float32: Middlebury's color wheel (makecolorwheel, integer division) divided by 255, and the eight-entry
// map of KITTI's stereo devkit (disp_to_color) with its bin weights and cumulative bin edges.
constexpr float PI_F = OFDIS_PI_F;
constexpr int WHEEL = 55;
struct ColorTables {
  float wheel[WHEEL][3];  // W[k][b] / 255.0f
  float disp_map[8][3];   // M[i][0..2]
  float disp_wt[7];       // 1000.0f / M[i][3]
  float disp_cum[8];      // cum[0] = 0, cum[i + 1] = cum[i] + M[i][3] / 1000.0f
  float atan_c[8];        // the polynomial of atan2_f32
};
constexpr ColorTables make_color_tables() {
  ColorTables t{};
  constexpr int seg[6] = {15, 6, 4, 11, 13, 6};  // RY, YG, GC, CB, BM, MR
  int k = 0;
  for (int s = 0; s < 6; ++s)
    for (int i = 0; i < seg[s]; ++i, ++k) {
      const int up = 255 * i / seg[s], down = 255 - 255 * i / seg[s];
      const int w[6][3] = {{255, up, 0}, {down, 255, 0}, {0, 255, up}, {0, down, 255}, {up, 0, 255}, {255, 0, down}};
      for (int b = 0; b < 3; ++b) t.wheel[k][b] = (float)w[s][b] / 255.0f;
    }
  constexpr int M[8][4] = {{0, 0, 0, 114}, {0, 0, 1, 185}, {1, 0, 0, 114}, {1, 0, 1, 174},
                           {0, 1, 0, 114}, {0, 1, 1, 185}, {1, 1, 0, 114}, {1, 1, 1, 0}};
  for (int i = 0; i < 8; ++i)
    for (int c = 0; c < 3; ++c) t.disp_map[i][c] = (float)M[i][c];
  t.disp_cum[0] = 0.0f;
  for (int i = 0; i < 7; ++i) {
    t.disp_wt[i] = 1000.0f / (float)M[i][3];
    t.disp_cum[i + 1] = t.disp_cum[i] + (float)M[i][3] / 1000.0f;
  }
  // atan(t) ~ t * (C0 + s * (C1 + ... + s * C7)), s = t * t, fitted on [0, 1] (|error| < 4e-8 before rounding)
  constexpr float C[8] = {OFDIS_ATAN2_C};
  for (int k = 0; k < 8; ++k) t.atan_c[k] = C[k];
  return t;
}
__constant__ ColorTables kColor = make_color_tables();

// The library's float32 atan2 (ofdis_internal.cuh) on the color tables' coefficients
__device__ __forceinline__ float atan2_f32(float y, float x) { return ofdis::atan2_f32(y, x, kColor.atan_c); }

// What the automatic scale is the maximum of: flow the radius of a known pixel (|u|, |v| <= 1e9, so NaN and the
// infinities are unknown), stereo the valid disparity d (0 <= d <= 1e9; d = -F, +F in a slot marked swapped).  +0
// elsewhere, never -0, so the bit patterns order as the values do.
template <int NOP>
__device__ __forceinline__ float color_magnitude(const LevelGeom& g, int frame, const float f[2]) {
  if constexpr (NOP == 2) {
    const bool known = fabsf(f[0]) <= 1e9f && fabsf(f[1]) <= 1e9f;
    return known ? sqrtf(f[0] * f[0] + f[1] * f[1]) : 0.0f;
  } else {
    const float d = swapped_of(g, frame) ? f[0] : -f[0];
    return d > 0.0f && d <= 1e9f ? d : 0.0f;
  }
}

// The automatic scale's maximum of slot fr: a block max of color_magnitude over the slot's full-resolution pixels,
// then an atomicMax of its bit pattern (non-negative floats order as their patterns) into words[fr], which the
// launcher zeroes first.  One thread per full-resolution pixel, blocks of 32 x 8.
template <int NOP>
__global__ void __launch_bounds__(256) flow_color_scale_kernel(LevelGeom g, int f0, unsigned int* words, int w_org,
                                                               int h_org, int crop_x, int crop_y) {
  __shared__ float warp_max[8];
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  const int fr = blockIdx.z, frame = frame_of(g, f0, fr);
  float m = 0.0f;
  if (X < w_org && Y < h_org) {
    float f[2] = {0.f, 0.f};
    upsample_at<NOP>(g, g.flow + (size_t)frame * g.flow_frame_stride, X, Y, crop_x, crop_y,
                     [&f](int c, float v) { f[c] = v; });
    m = color_magnitude<NOP>(g, frame, f);
  }
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (threadIdx.x == 0) warp_max[threadIdx.y] = m;
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    for (int k = 1; k < 8; ++k) m = fmaxf(m, warp_max[k]);
    if (m > 0.0f) atomicMax(words + fr, __float_as_uint(m));
  }
}

// The color image of slot fr, 3 bytes (R, G, B) per full-resolution pixel, from F (upsample_at) without storing it:
//   flow (Middlebury's computeColor): unknown black; else fx = u / scale, fy = v / scale, rad = |(fx, fy)|,
//     a = atan2_f32(-v, -u) / PI_F of the unscaled flow, fk = (a + 1) / 2 * 54, the wheel entries k0 = (int)fk and
//     (k0 + 1) % 55 mixed by f = fk - k0, whitened towards the centre (rad <= 1) or darkened by 0.75 beyond it;
//   stereo (KITTI's disp_to_color): invalid black; else val = clamp(d / scale, 0, 1) in the first bin i with
//     val < cum[i + 1] (else 6), mixed between map entries i and i + 1.
// scale = max_value when it is > 0, else the slot's maximum (words[fr]): flow 1 where it is 0, stereo at least 1;
// where scale_out is given, pixel (0, 0) writes it to scale_out[fr].  One thread per full-resolution pixel.
template <int NOP>
__global__ void __launch_bounds__(256) flow_color_kernel(LevelGeom g, int f0, const unsigned int* words,
                                                         float max_value, unsigned char* rgb, float* scale_out,
                                                         int w_org, int h_org, int crop_x, int crop_y) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X >= w_org || Y >= h_org) return;
  const int fr = blockIdx.z, frame = frame_of(g, f0, fr);
  float scale = max_value;
  if (!(max_value > 0.0f)) {
    const float m = __uint_as_float(words[fr]);
    scale = NOP == 2 ? (m == 0.0f ? 1.0f : m) : fmaxf(m, 1.0f);
  }
  if (scale_out && X == 0 && Y == 0) scale_out[fr] = scale;
  float f[2] = {0.f, 0.f};
  upsample_at<NOP>(g, g.flow + (size_t)frame * g.flow_frame_stride, X, Y, crop_x, crop_y,
                   [&f](int c, float v) { f[c] = v; });
  unsigned char col[3] = {0, 0, 0};
  if constexpr (NOP == 2) {
    const float u = f[0], v = f[1];
    if (fabsf(u) <= 1e9f && fabsf(v) <= 1e9f) {
      const float fx = u / scale, fy = v / scale, rad = sqrtf(fx * fx + fy * fy);
      const float a = atan2_f32(-v, -u) / PI_F;
      const float fk = (a + 1.0f) / 2.0f * (float)(WHEEL - 1);
      const int k0 = (int)fk, k1 = (k0 + 1) % WHEEL;
      const float fr_k = fk - (float)k0;
      for (int b = 0; b < 3; ++b) {
        float c = (1.0f - fr_k) * kColor.wheel[k0][b] + fr_k * kColor.wheel[k1][b];
        c = rad <= 1.0f ? 1.0f - rad * (1.0f - c) : c * 0.75f;
        col[b] = (unsigned char)(255.0f * c);
      }
    }
  } else {
    const float d = swapped_of(g, frame) ? f[0] : -f[0];
    if (d >= 0.0f && d <= 1e9f) {  // NaN fails, -0 passes
      const float val = fminf(fmaxf(d / scale, 0.0f), 1.0f);
      int i = 6;
#pragma unroll
      for (int k = 6; k >= 0; --k) i = val < kColor.disp_cum[k + 1] ? k : i;  // the first bin that holds val
      const float w = 1.0f - (val - kColor.disp_cum[i]) * kColor.disp_wt[i];
      for (int c = 0; c < 3; ++c)
        col[c] = (unsigned char)fminf(
            fmaxf((w * kColor.disp_map[i][c] + (1.0f - w) * kColor.disp_map[i + 1][c]) * 255.0f, 0.0f), 255.0f);
    }
  }
  unsigned char* o = rgb + ((size_t)fr * h_org * w_org + (size_t)Y * w_org + X) * 3;
  for (int b = 0; b < 3; ++b) o[b] = col[b];
}

// Forward-backward (flow) / left-right (stereo) consistency (Sundaram, Brox, Keutzer, ECCV 2010) of frame fa's
// full-resolution flow F against frame fb's B, both exactly what flow_upsample_kernel writes, evaluated from the
// level flows (upsample_at) where they are needed instead of through a full-resolution copy.  Per pixel, in
// float32 without contraction (preprocess.consistency_check restates it):
//   (xs, ys) = (x, y) + F(x, y); outside [0, w_org-1] x [0, h_org-1] (or NaN): mask 2, err +inf;
//   b = B bilinear at (xs, ys) (corners x0 = floor(xs), x1 = min(x0 + 1, w_org - 1), horizontal pass first);
//   err = |F + b|^2, mask = err <= alpha (|F|^2 + |b|^2) + beta ? 0 : 1.
// One thread per full-resolution pixel; err may be nullptr.
template <int NOP>
__global__ void __launch_bounds__(256) consistency_kernel(LevelGeom g, int fa, int fb, unsigned char* mask, float* err,
                                                          int w_org, int h_org, int crop_x, int crop_y, float alpha,
                                                          float beta) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X >= w_org || Y >= h_org) return;
  const int fr = blockIdx.z;
  const float* F = g.flow + (size_t)frame_of(g, fa, fr) * g.flow_frame_stride;
  const float* B = g.flow + (size_t)frame_of(g, fb, fr) * g.flow_frame_stride;
  const size_t o = (size_t)fr * h_org * w_org + (size_t)Y * w_org + X;
  float f[2] = {0.f, 0.f};
  upsample_at<NOP>(g, F, X, Y, crop_x, crop_y, [&f](int c, float v) { f[c] = v; });
  consistency_at<NOP>(g, B, f, X, Y, w_org, h_org, crop_x, crop_y, alpha, beta, [&](unsigned char m, float e) {
    mask[o] = m;
    if (err) err[o] = e;
  });
}

// Evaluation of frame f0 + fr's full-resolution flow F (upsample_at, as flow_upsample_kernel writes it) against the
// ground truth G of ofdis_flow_error_fullres (header, and preprocess.flow_error), float32 without contraction:
//   known = G not NaN and |G| <= 1e9 per component; e = sqrtf(du*du + dv*dv) (stereo fabsf(F - G)), g = |G| likewise;
//   err = known ? e : qNaN; the pixel counts for class classes[pixel] (0 without classes) if known and < nclasses.
// One CTA of EV_THREADS per (row, pair).  The row goes through shared memory in chunks of EV_CHUNK pixels: every
// thread computes EV_CHUNK / EV_THREADS of them (coalesced), then thread c < nclasses walks the chunk with x ascending
// and adds class c's errors to its float64 row sum -- the fixed order of the contract -- and its counts.
constexpr int EV_THREADS = 256, EV_CHUNK = 1024, EV_MAX_CLASSES = 16;
constexpr unsigned char EV_SKIP = 0xff;  // the pixel counts for no class

template <int NOP>
__global__ void __launch_bounds__(EV_THREADS) flow_error_kernel(LevelGeom g, int f0, const float* gt,
                                                                const unsigned char* classes, int nclasses, float* err,
                                                                ErrRowPartial* part, int w_org, int h_org, int crop_x,
                                                                int crop_y) {
  __shared__ float se[EV_CHUNK];
  __shared__ unsigned char sk[EV_CHUNK], sf[EV_CHUNK];  // class (EV_SKIP: none) and flags (bit k: test k true)
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int Y = blockIdx.x, fr = blockIdx.y, t = threadIdx.x;
  const float* fl = g.flow + (size_t)frame_of(g, f0, fr) * g.flow_frame_stride;
  const size_t row = ((size_t)fr * h_org + Y) * w_org;
  const float unknown_thresh = 1e9f;
  double sum = 0.0;
  unsigned int cnt[5] = {0, 0, 0, 0, 0};
  for (int x0 = 0; x0 < w_org; x0 += EV_CHUNK) {
    const int m = min(EV_CHUNK, w_org - x0);
    for (int i = t; i < m; i += EV_THREADS) {
      const int X = x0 + i;
      const size_t o = row + X;
      float f[2] = {0.f, 0.f};
      upsample_at<NOP>(g, fl, X, Y, crop_x, crop_y, [&f](int c, float v) { f[c] = v; });
      float e, gm;
      bool known;
      if constexpr (NOP == 2) {
        const float Gu = gt[2 * o], Gv = gt[2 * o + 1];  // a caller's device array may be only 4-byte aligned
        known = fabsf(Gu) <= unknown_thresh && fabsf(Gv) <= unknown_thresh;  // NaN fails both
        const float du = f[0] - Gu, dv = f[1] - Gv;
        e = sqrtf(du * du + dv * dv);
        gm = sqrtf(Gu * Gu + Gv * Gv);
      } else {
        const float G = gt[o];
        known = fabsf(G) <= unknown_thresh;
        e = fabsf(f[0] - G);
        gm = fabsf(G);
      }
      if (err) err[o] = known ? e : __int_as_float(0x7fc00000);
      const int k = classes ? classes[o] : 0;
      se[i] = e;
      sk[i] = known && k < nclasses ? (unsigned char)k : EV_SKIP;
      sf[i] = (e > 1.0f ? 1 : 0) | (e > 3.0f ? 2 : 0) | (e > 5.0f ? 4 : 0) | (e > 3.0f && e > 0.05f * gm ? 8 : 0);
    }
    __syncthreads();
    if (t < nclasses) {
      for (int i = 0; i < m; ++i) {
        const bool mine = sk[i] == t;
        const unsigned int fl8 = sf[i];
        sum += mine ? (double)se[i] : 0.0;  // + 0.0 leaves a sum of non-negative terms as it is
        cnt[0] += mine ? 1u : 0u;
        for (int b = 0; b < 4; ++b) cnt[b + 1] += mine ? (fl8 >> b) & 1u : 0u;
      }
    }
    __syncthreads();
  }
  if (t < nclasses) {
    ErrRowPartial& p = part[((size_t)fr * nclasses + t) * h_org + Y];
    p.sum = sum;
    for (int b = 0; b < 5; ++b) p.n[b] = cnt[b];
  }
}

// Sums the row partials of one (pair, class) -- blockIdx.x = pair * nclasses + class -- with y ascending: the threads
// stage EV_THREADS rows at a time in shared memory, thread 0 adds them in order.
__global__ void __launch_bounds__(EV_THREADS) flow_error_reduce_kernel(const ErrRowPartial* part, int h_org,
                                                                       ofdis_error_stats* stats) {
  __shared__ double ss[EV_THREADS];
  __shared__ unsigned int sn[5][EV_THREADS];
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const ErrRowPartial* p = part + (size_t)blockIdx.x * h_org;
  const int t = threadIdx.x;
  double total = 0.0;
  long long cnt[5] = {0, 0, 0, 0, 0};
  for (int y0 = 0; y0 < h_org; y0 += EV_THREADS) {
    const int m = min(EV_THREADS, h_org - y0);
    if (t < m) {
      ss[t] = p[y0 + t].sum;
      for (int b = 0; b < 5; ++b) sn[b][t] = p[y0 + t].n[b];
    }
    __syncthreads();
    if (t == 0) {
      for (int i = 0; i < m; ++i) {
        total += ss[i];
        for (int b = 0; b < 5; ++b) cnt[b] += sn[b][i];
      }
    }
    __syncthreads();
  }
  if (t == 0) {
    ofdis_error_stats& s = stats[blockIdx.x];
    s.n = cnt[0];
    for (int b = 0; b < 3; ++b) s.n_over[b] = cnt[b + 1];
    s.n_outlier = cnt[4];
    s.sum_err = total;
  }
}

// Init flow of the reference's disabled file input (run_dense.cpp:355-378): the full-resolution flow
// [frame][h_org][w_org][NOP], replicate-padded to the context (clamped reads, floor(pad/2) left/top), times
// 2^-(sc_f+1), then cv::resize(INTER_AREA) by the integer factor s = 2^(sc_f+1).  That is OpenCV's area-fast path:
// sum = 0, then for the s x s terms of the block in row-major order, groups of four add as
// sum += ((t0 + t1) + t2) + t3, and the result is sum * (1/s^2); for s = 2 with one channel its SIMD body,
// ((a + b) + (c + d)) * 0.25 (preprocess.initflow_from_fullres).  g: level sc_f, stepped by the context's directions;
// writes level sc_f+1 (g.flow_prev) of the forward grid of every pair, and with usefbcon zeroes the backward grid's,
// which the reference does not initialise (oflow.cpp:217-220).
// TEAM == 1 (s <= 8): one thread per output pixel.  TEAM == 256: one CTA per output pixel; the threads form the
// independent group partials of up to 1024 groups in shared memory, and thread c adds channel c's in order.
template <int NOP, int TEAM>
__global__ void __launch_bounds__(256) initflow_prepare_kernel(LevelGeom g, int f0, const float* src, int w_org,
                                                               int h_org, int pad_left, int pad_top) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int W = g.w >> 1, H = g.h >> 1, sh = g.level + 1, s = 1 << sh;
  const int pix = TEAM == 1 ? (int)(blockIdx.x * blockDim.x + threadIdx.x) : (int)blockIdx.x, fr = blockIdx.y;
  if (pix >= W * H) return;
  const int x0 = (pix % W) * s - pad_left, y0 = (pix / W) * s - pad_top;
  const float* fl = src + (size_t)fr * h_org * w_org * NOP;
  const float sc = __int_as_float((127 - sh) << 23), inv_area = __int_as_float((127 - 2 * sh) << 23);
  auto term = [&](int k, int c) {  // term k (row-major in the block) of channel c, scaled
    const int X = clampi(x0 + (k & (s - 1)), w_org), Y = clampi(y0 + (k >> sh), h_org);
    return __ldg(fl + ((size_t)Y * w_org + X) * NOP + c) * sc;
  };
  auto group = [&](int gi, int c) {
    const int k = 4 * gi;
    return ((term(k, c) + term(k + 1, c)) + term(k + 2, c)) + term(k + 3, c);
  };
  const int ng = (s * s) >> 2;
  float* dst = const_cast<float*>(g.flow_prev) + (size_t)frame_of(g, f0, fr) * g.flow_prev_frame_stride + (size_t)pix * NOP;
  if constexpr (TEAM == 1) {
    for (int c = 0; c < NOP; ++c) {
      float v;
      if (NOP == 1 && s == 2) {
        v = ((term(0, c) + term(1, c)) + (term(2, c) + term(3, c))) * 0.25f;
      } else {
        float sum = 0.f;
        for (int gi = 0; gi < ng; ++gi) sum += group(gi, c);
        v = sum * inv_area;
      }
      dst[c] = v;
      if (g.fstep == 2) dst[g.flow_prev_frame_stride + c] = 0.f;
    }
  } else {
    __shared__ float part[NOP][1024 + 1];  // +1: the channels' rows start in different banks
    float sum = 0.f;                       // thread c < NOP: channel c
    for (int base = 0; base < ng; base += 1024) {
      const int m = min(1024, ng - base);
      for (int i = threadIdx.x; i < m; i += TEAM)
        for (int c = 0; c < NOP; ++c) part[c][i] = group(base + i, c);
      __syncthreads();
      if (threadIdx.x < NOP) {
        const float* p = part[threadIdx.x];
#pragma unroll 8
        for (int i = 0; i < m; ++i) sum += p[i];
      }
      __syncthreads();
    }
    if (threadIdx.x < NOP) {
      dst[threadIdx.x] = sum * inv_area;
      if (g.fstep == 2) dst[g.flow_prev_frame_stride + threadIdx.x] = 0.f;
    }
  }
}

}  // namespace

static dim3 padded_grid(const LevelGeom& g, int nz) { return dim3((g.tmp_w + 31) / 32, (g.tmp_h + 7) / 8, nz); }

int launch_sobel(const LevelGeom& g, int f0, int f1, cudaStream_t st) {
  sobel_kernel<<<padded_grid(g, f1 - f0), dim3(32, 8), 0, st>>>(g, f0);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_pyr_from_u8(const LevelGeom& g, int f0, int f1, const PyrSourceU8& s, cudaStream_t st) {
  pyr_from_u8_kernel<PYR_PAIRS><<<padded_grid(g, 2 * (f1 - f0)), dim3(32, 8), 0, st>>>(g, f0, s, 0);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_pyr_from_u8_seq(const LevelGeom& g, int f0, int n, const PyrSourceU8& s, cudaStream_t st) {
  pyr_from_u8_kernel<PYR_SEQ><<<padded_grid(g, n + 1), dim3(32, 8), 0, st>>>(g, f0, s, n);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_pyr_from_u8_bidir(const LevelGeom& g, int f0, int n, const PyrSourceU8& s, cudaStream_t st) {
  pyr_from_u8_kernel<PYR_BIDIR><<<padded_grid(g, n + 1), dim3(32, 8), 0, st>>>(g, f0, s, n);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_pyr_from_level(const LevelGeom& g, int f0, int f1, const float* stage, cudaStream_t st) {
  pyr_from_level_kernel<<<padded_grid(g, 2 * (f1 - f0)), dim3(32, 8), 0, st>>>(g, f0, stage);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_pyr_down(const LevelGeom& gs, const LevelGeom& gd, int f0, int f1, cudaStream_t st) {
  pyr_down_kernel<PYR_PAIRS><<<padded_grid(gd, 2 * (f1 - f0)), dim3(32, 8), 0, st>>>(gs, gd, f0, 0);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_pyr_down_seq(const LevelGeom& gs, const LevelGeom& gd, int f0, int n, cudaStream_t st) {
  pyr_down_kernel<PYR_SEQ><<<padded_grid(gd, n + 1), dim3(32, 8), 0, st>>>(gs, gd, f0, n);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_pyr_down_bidir(const LevelGeom& gs, const LevelGeom& gd, int f0, int n, cudaStream_t st) {
  pyr_down_kernel<PYR_BIDIR><<<padded_grid(gd, n + 1), dim3(32, 8), 0, st>>>(gs, gd, f0, n);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_flow_upsample(const LevelGeom& g, int f0, int f1, float* out, int w_org, int h_org, int crop_x, int crop_y,
                         cudaStream_t st) {
  const dim3 block(32, 8), grid((w_org + 31) / 32, (h_org + 7) / 8, f1 - f0);
  if (g.nop == 2) flow_upsample_kernel<2><<<grid, block, 0, st>>>(g, f0, out, w_org, h_org, crop_x, crop_y);
  else flow_upsample_kernel<1><<<grid, block, 0, st>>>(g, f0, out, w_org, h_org, crop_x, crop_y);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_flow_encode(const LevelGeom& g, int f0, int n, int enc, unsigned short* out, int w_org, int h_org,
                       int crop_x, int crop_y, cudaStream_t st) {
  const dim3 block(32, 8), grid((w_org + 31) / 32, (h_org + 7) / 8, n);
  if (enc == OFDIS_ENC_F16) {
    if (g.nop == 2)
      flow_encode_kernel<2, OFDIS_ENC_F16><<<grid, block, 0, st>>>(g, f0, out, w_org, h_org, crop_x, crop_y);
    else
      flow_encode_kernel<1, OFDIS_ENC_F16><<<grid, block, 0, st>>>(g, f0, out, w_org, h_org, crop_x, crop_y);
  } else if (enc == OFDIS_ENC_KITTI) {
    if (g.nop == 2)
      flow_encode_kernel<2, OFDIS_ENC_KITTI><<<grid, block, 0, st>>>(g, f0, out, w_org, h_org, crop_x, crop_y);
    else
      flow_encode_kernel<1, OFDIS_ENC_KITTI><<<grid, block, 0, st>>>(g, f0, out, w_org, h_org, crop_x, crop_y);
  } else {
    return -1;
  }
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_flow_color(const LevelGeom& g, int f0, int n, unsigned int* words, float max_value, unsigned char* rgb,
                      float* scale, int w_org, int h_org, int crop_x, int crop_y, cudaStream_t st) {
  const dim3 block(32, 8), grid((w_org + 31) / 32, (h_org + 7) / 8, n);
  const bool automatic = !(max_value > 0.0f);
  if (automatic) {
    if (cudaMemsetAsync(words, 0, sizeof(unsigned int) * n, st) != cudaSuccess) return -1;
    if (g.nop == 2) flow_color_scale_kernel<2><<<grid, block, 0, st>>>(g, f0, words, w_org, h_org, crop_x, crop_y);
    else flow_color_scale_kernel<1><<<grid, block, 0, st>>>(g, f0, words, w_org, h_org, crop_x, crop_y);
    if (cudaGetLastError() != cudaSuccess) return -1;
  }
  if (g.nop == 2)
    flow_color_kernel<2><<<grid, block, 0, st>>>(g, f0, words, max_value, rgb, scale, w_org, h_org, crop_x, crop_y);
  else
    flow_color_kernel<1><<<grid, block, 0, st>>>(g, f0, words, max_value, rgb, scale, w_org, h_org, crop_x, crop_y);
  if (cudaGetLastError() != cudaSuccess) return -1;
  return automatic ? 2 : 1;
}

int launch_consistency(const LevelGeom& g, int fa, int fb, int n, unsigned char* mask, float* err, int w_org,
                       int h_org, int crop_x, int crop_y, float alpha, float beta, cudaStream_t st) {
  const dim3 block(32, 8), grid((w_org + 31) / 32, (h_org + 7) / 8, n);
  if (g.nop == 2)
    consistency_kernel<2><<<grid, block, 0, st>>>(g, fa, fb, mask, err, w_org, h_org, crop_x, crop_y, alpha, beta);
  else
    consistency_kernel<1><<<grid, block, 0, st>>>(g, fa, fb, mask, err, w_org, h_org, crop_x, crop_y, alpha, beta);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_flow_error(const LevelGeom& g, int f0, int n, const float* gt, const unsigned char* classes, int nclasses,
                      float* err, ErrRowPartial* part, ofdis_error_stats* stats, int w_org, int h_org, int crop_x,
                      int crop_y, cudaStream_t st) {
  if (nclasses < 1 || nclasses > EV_MAX_CLASSES) return -1;
  const dim3 grid(h_org, n);
  if (g.nop == 2)
    flow_error_kernel<2><<<grid, EV_THREADS, 0, st>>>(g, f0, gt, classes, nclasses, err, part, w_org, h_org, crop_x, crop_y);
  else
    flow_error_kernel<1><<<grid, EV_THREADS, 0, st>>>(g, f0, gt, classes, nclasses, err, part, w_org, h_org, crop_x, crop_y);
  if (cudaGetLastError() != cudaSuccess) return -1;
  flow_error_reduce_kernel<<<n * nclasses, EV_THREADS, 0, st>>>(part, h_org, stats);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_initflow_prepare(const LevelGeom& g, int f0, int n, const float* flow, int w_org, int h_org, int pad_left,
                            int pad_top, cudaStream_t st) {
  const int npix = (g.w >> 1) * (g.h >> 1);
  if ((2 << g.level) <= 8) {
    const dim3 grid((npix + 255) / 256, n);
    if (g.nop == 2) initflow_prepare_kernel<2, 1><<<grid, 256, 0, st>>>(g, f0, flow, w_org, h_org, pad_left, pad_top);
    else initflow_prepare_kernel<1, 1><<<grid, 256, 0, st>>>(g, f0, flow, w_org, h_org, pad_left, pad_top);
  } else {
    const dim3 grid(npix, n);
    if (g.nop == 2) initflow_prepare_kernel<2, 256><<<grid, 256, 0, st>>>(g, f0, flow, w_org, h_org, pad_left, pad_top);
    else initflow_prepare_kernel<1, 256><<<grid, 256, 0, st>>>(g, f0, flow, w_org, h_org, pad_left, pad_top);
  }
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ofdis

// Trajectory descriptors along the tracker's tracks (ofdis_traj_begin / ofdis_traj_advance; the header states the
// contract, preprocess.traj_descriptors restates it bit for bit): the single-scale pipeline of Wang and Schmid's
// improved dense trajectories (ICCV 2013) -- trajectory shape, HOG, HOF and MBH of the camera-compensated residual flow
// R per segment of L steps.  ofdis_capi.cu interleaves them with the tracker's five kernels; per pair it launches
//   traj_field_kernel  one thread per pixel: R, and the orientation bin and weights of the four vector fields;
//   traj_hist_kernel   one warp per live track (the hot path): the patch's cell histograms, their RootSIFT
//                      normalisation and the temporal cell's sums, the position and displacement of the step;
// then, after the tracker's compaction (whose keep flags and block offsets they reuse, without changing it),
//   traj_flag_kernel   one thread per track slot: the survivor's index in the next list, the tests of a completed
//                      segment, its output offset within the scan block and the counters;
//   traj_scan_kernel   one CTA: the scan blocks' output offsets and the pair's count;
//   traj_move_kernel   one warp per track slot: the emitted record and descriptor, the state's move into the next
//                      list, the seeds' fresh segments.
// Every kernel reads the live counts from the device state, so a call enqueues all its pairs without a host round
// trip.  Float32 without contraction, IEEE division and square root; every sum in the order the header states.
#include <cfloat>

#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

__constant__ float kAtanC[8] = {OFDIS_ATAN2_C};
constexpr float TWO_PI_F = 6.28318530717958647692f;   // 6.2831855f
constexpr float BIN_SCALE = 1.27323954473516268615f;  // 8 / (2 pi): 1.2732395f
constexpr unsigned char NO_BIN = 255;
constexpr int HIST_WARPS = 4;
constexpr int MOVE_WARPS = 4;
constexpr int SCAN_THREADS = 1024;
__constant__ int kBinLo[4] = {0, 8, 17, 25};  // first entry of HOG, HOF, MBHx, MBHy in a cell's 33

// a[c] of a kernel parameter's two-list array without indexing the parameter (which would copy it to the stack)
template <typename T>
__device__ __forceinline__ T* pick(T* const (&a)[2], int c) { return c ? a[1] : a[0]; }

// The orientation bin of a vector (a, b): none where |(a, b)| = sqrtf(a*a + b*b) is not finite; else angle =
// atan2_f32(b, a), + 2 pi below 0, fbin = angle * 8 / (2 pi), bin0 = floor(fbin) (8 wraps to 0), mag1 = (fbin -
// floor(fbin)) * mag, mag0 = mag - mag1.
__device__ __forceinline__ void orient(float a, float b, unsigned char& bin, float& m0, float& m1) {
  const float mag = sqrtf(a * a + b * b);
  bin = NO_BIN;
  m0 = m1 = 0.f;
  if (!(mag <= FLT_MAX)) return;
  float ang = atan2_f32(b, a, kAtanC);
  if (ang < 0.f) ang = ang + TWO_PI_F;
  const float fbin = ang * BIN_SCALE;
  const float fb0 = floorf(fbin);
  const int b0 = (int)fb0;
  m1 = (fbin - fb0) * mag;
  m0 = mag - m1;
  bin = (unsigned char)(b0 >= 8 ? 0 : b0);
}

// R at pixel (X, Y): F (upsample_at) minus the model's flow; known where |u|, |v| <= 1e9, wq > 0 and R is finite
__device__ __forceinline__ bool residual_at(const LevelGeom& g, const float* F, const float* m, int X, int Y,
                                            int crop_x, int crop_y, float& ru, float& rv) {
  float f[2] = {0.f, 0.f};
  upsample_at<2>(g, F, X, Y, crop_x, crop_y, [&f](int c, float v) { f[c] = v; });
  const float fX = (float)X, fY = (float)Y;
  const float mx = (m[0] * fX + m[1] * fY) + m[2], my = (m[3] * fX + m[4] * fY) + m[5];
  const float wq = (m[6] * fX + m[7] * fY) + m[8];
  ru = f[0] - (mx / wq - fX);
  rv = f[1] - (my / wq - fY);
  return fabsf(f[0]) <= 1e9f && fabsf(f[1]) <= 1e9f && wq > 0.f && fabsf(ru) <= FLT_MAX && fabsf(rv) <= FLT_MAX;
}

template <int NOC>
__global__ void __launch_bounds__(256) traj_field_kernel(LevelGeom g, int fa, TrajGeom tg, TrajWork tw,
                                                         const unsigned char* I, const float* mp, int crop_x,
                                                         int crop_y) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  const int w = tg.w, h = tg.h;
  if (X >= w || Y >= h) return;
  float m[9];
  for (int i = 0; i < 9; ++i) m[i] = mp[i];
  const float* F = g.flow + (size_t)fa * g.flow_frame_stride;
  const int xl = max(X - 1, 0), xr = min(X + 1, w - 1), yu = max(Y - 1, 0), yd = min(Y + 1, h - 1);
  uchar4 b;
  float4 a, e;
  const float ix = (gray_at<NOC>(I, w, xr, Y) - gray_at<NOC>(I, w, xl, Y)) * 0.5f;
  const float iy = (gray_at<NOC>(I, w, X, yd) - gray_at<NOC>(I, w, X, yu)) * 0.5f;
  orient(ix, iy, b.x, a.x, a.y);
  float ru, rv;
  const bool known = residual_at(g, F, m, X, Y, crop_x, crop_y, ru, rv);
  const float qnan = __int_as_float(0x7fc00000);
  tw.res[(size_t)Y * w + X] = known ? make_float2(ru, rv) : make_float2(qnan, qnan);
  b.y = NO_BIN;
  a.z = a.w = 0.f;
  if (known) {
    orient(ru, rv, b.y, a.z, a.w);
    if (b.y != NO_BIN && sqrtf(ru * ru + rv * rv) <= tg.min_flow) {
      b.y = 8;  // the zero bin
      a.z = 1.f;
      a.w = 0.f;
    }
  }
  float lu, lv, rru, rrv, uu, uv, du, dv;
  bool kn = residual_at(g, F, m, xl, Y, crop_x, crop_y, lu, lv);
  kn = residual_at(g, F, m, xr, Y, crop_x, crop_y, rru, rrv) && kn;
  kn = residual_at(g, F, m, X, yu, crop_x, crop_y, uu, uv) && kn;
  kn = residual_at(g, F, m, X, yd, crop_x, crop_y, du, dv) && kn;
  b.z = b.w = NO_BIN;
  e = make_float4(0.f, 0.f, 0.f, 0.f);
  if (kn) {
    orient((rru - lu) * 0.5f, (du - uu) * 0.5f, b.z, e.x, e.y);
    orient((rrv - lv) * 0.5f, (dv - uv) * 0.5f, b.w, e.z, e.w);
  }
  const size_t o = (size_t)Y * w + X;
  tw.bins[o] = b;
  tw.mag[2 * o] = a;
  tw.mag[2 * o + 1] = e;
}

// One warp per live track of list[cur]: the step's position and displacement, then per spatial cell the 33 bin sums
// (lane l sums the cell's pixels q = l, l + 32, ... in row-major order into its own shared-memory row; the cell's sum
// is lane 0's + lane 1's + ... + lane 31's, + eps), every descriptor's sum over its entries in layout order, and
// sqrtf(v / sum) into the temporal cell.
__global__ void __launch_bounds__(HIST_WARPS * 32) traj_hist_kernel(TrajGeom tg, TrajWork tw, TrackWork ws, int cur) {
  __shared__ float hs[HIST_WARPS][32 * TRAJ_BINS];
  __shared__ float cv[HIST_WARPS][TRAJ_MAX_NS * TRAJ_MAX_NS * TRAJ_BINS];
  __shared__ float ds[HIST_WARPS][4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * HIST_WARPS + warp;
  if (i >= ws.state->alive) return;
  const ofdis_track_point p = pick(ws.list, cur)[i];
  const int t = pick(tw.meta, cur)[i].x;
  float* S = pick(tw.st, cur) + (size_t)i * tg.ss;
  const int w = tg.w;
  const int xr = (int)floorf(p.x + 0.5f), yr = (int)floorf(p.y + 0.5f);
  if (lane == 0) {
    const float2 d = tw.res[(size_t)yr * w + xr];
    S[2 * t] = p.x;
    S[2 * t + 1] = p.y;
    S[tg.pos + 2 * t] = d.x;
    S[tg.pos + 2 * t + 1] = d.y;
  }
  const int ox = min(max(xr - tg.N / 2, 0), w - tg.N), oy = min(max(yr - tg.N / 2, 0), tg.h - tg.N);
  const int c = tg.c, cc = c * c, ns = tg.ns, nc = ns * ns;
  float* hl = hs[warp] + lane * TRAJ_BINS;
  for (int xc = 0; xc < ns; ++xc)
    for (int yc = 0; yc < ns; ++yc) {
      for (int k = 0; k < TRAJ_BINS; ++k) hl[k] = 0.f;
      const int x0 = ox + xc * c, y0 = oy + yc * c;
      for (int q = lane; q < cc; q += 32) {
        const int py = q / c, px = q - py * c;
        const size_t o = (size_t)(y0 + py) * w + (x0 + px);
        const uchar4 b = tw.bins[o];
        const float4 a = tw.mag[2 * o], e = tw.mag[2 * o + 1];
        if (b.x != NO_BIN) {
          hl[b.x] += a.x;
          hl[(b.x + 1) & 7] += a.y;
        }
        if (b.y != NO_BIN) {
          hl[8 + b.y] += a.z;
          hl[8 + ((b.y + 1) & 7)] += a.w;
        }
        if (b.z != NO_BIN) {
          hl[17 + b.z] += e.x;
          hl[17 + ((b.z + 1) & 7)] += e.y;
        }
        if (b.w != NO_BIN) {
          hl[25 + b.w] += e.z;
          hl[25 + ((b.w + 1) & 7)] += e.w;
        }
      }
      __syncwarp();
      float* v = cv[warp] + (xc * ns + yc) * TRAJ_BINS;
      for (int k = lane; k < TRAJ_BINS; k += 32) {
        float s = hs[warp][k];
        for (int l = 1; l < 32; ++l) s = s + hs[warp][l * TRAJ_BINS + k];
        v[k] = s + tg.eps;
      }
      __syncwarp();
    }
  if (lane < 4) {
    const int lo = kBinLo[lane], nb = lane == 1 ? 9 : 8;
    float s = 0.f;
    for (int cell = 0; cell < nc; ++cell)
      for (int k = 0; k < nb; ++k) s = s + cv[warp][cell * TRAJ_BINS + lo + k];
    ds[warp][lane] = s;
  }
  __syncwarp();
  float* A = S + tg.pos + tg.dis + (t / tg.tl) * nc * TRAJ_BINS;
  const bool first = t % tg.tl == 0;
  for (int e = lane; e < nc * TRAJ_BINS; e += 32) {
    const int k = e % TRAJ_BINS, d = k < 8 ? 0 : k < 17 ? 1 : k < 25 ? 2 : 3;
    const float r = sqrtf(cv[warp][e] / ds[warp][d]);
    A[e] = first ? r : A[e] + r;
  }
}

// The tests of a completed segment whose L + 1 positions and L displacements are in S: 0 emitted, 1 static,
// 2 erratic, 3 jump, 4 camera; the record's statistics and the sum of |d_i| go to sg.
__device__ int segment_test(const TrajGeom& tg, const float* S, TrajSeg& sg) {
  const int L = tg.L;
  const float fn = (float)(L + 1);
  float sx = 0.f, sy = 0.f;
  for (int j = 0; j <= L; ++j) {
    sx = sx + S[2 * j];
    sy = sy + S[2 * j + 1];
  }
  const float mx = sx / fn, my = sy / fn;
  float vx = 0.f, vy = 0.f;
  for (int j = 0; j <= L; ++j) {
    const float dx = S[2 * j] - mx, dy = S[2 * j + 1] - my;
    vx = vx + dx * dx;
    vy = vy + dy * dy;
  }
  const float sdx = sqrtf(vx / fn), sdy = sqrtf(vy / fn);
  float len = 0.f, smax = 0.f;
  for (int j = 0; j < L; ++j) {
    const float dx = S[2 * j + 2] - S[2 * j], dy = S[2 * j + 3] - S[2 * j + 1];
    const float s = sqrtf(dx * dx + dy * dy);
    len = len + s;
    if (s > smax) smax = s;
  }
  float dsum = 0.f, dmax = 0.f;
  bool known = true;
  for (int j = 0; j < L; ++j) {
    const float du = S[tg.pos + 2 * j], dv = S[tg.pos + 2 * j + 1];
    const float a = sqrtf(du * du + dv * dv);
    known = known && a <= FLT_MAX;
    dsum = dsum + a;
    if (a > dmax) dmax = a;
  }
  sg.rec.mean_x = mx;
  sg.rec.mean_y = my;
  sg.rec.sd_x = sdx;
  sg.rec.sd_y = sdy;
  sg.rec.length = len;
  sg.dsum = dsum;
  if (sdx < tg.min_var && sdy < tg.min_var) return 1;
  if (sdx > tg.max_var || sdy > tg.max_var) return 2;
  if (smax > tg.max_dis && smax > 0.7f * len) return 3;
  if (!known || dmax <= tg.min_disp) return 4;
  return 0;
}

// One thread per track slot, one CTA per scan block of the tracker.
__global__ void __launch_bounds__(TRACK_BLOCK) traj_flag_kernel(TrajGeom tg, TrajWork tw, TrackWork ws, int cur) {
  __shared__ unsigned int sw[TRACK_BLOCK / 32];
  const int i = blockIdx.x * TRACK_BLOCK + threadIdx.x;  // the grid is exactly cap_pad threads
  const bool keep = ws.flags[i] != 0;
  unsigned int total;
  const unsigned int loc = block_exclusive_scan<TRACK_BLOCK>(keep ? 1u : 0u, sw, total);
  int why = -1;  // -1 no completed segment, 0 emitted, 1 static, 2 erratic, 3 jump, 4 camera
  if (keep) {
    const int2 mt = pick(tw.meta, cur)[i];
    if (mt.x + 1 == tg.L) {
      float* S = pick(tw.st, cur) + (size_t)i * tg.ss;
      const ofdis_track_point p = pick(ws.list, cur)[i];  // the advanced position
      S[2 * tg.L] = p.x;
      S[2 * tg.L + 1] = p.y;
      TrajSeg sg;
      why = segment_test(tg, S, sg);
      sg.rec.id = p.id;
      sg.rec.start = mt.y;
      if (why == 0) tw.seg[i] = sg;
    }
  }
  tw.dst[i] = keep ? (int)(ws.bsum[blockIdx.x] + loc) : -1;
  const unsigned int eloc = block_exclusive_scan<TRACK_BLOCK>(why == 0 ? 1u : 0u, sw, total);
  tw.eoff[i] = why == 0 ? (int)eloc : -1;
  if (threadIdx.x == 0) tw.ebsum[blockIdx.x] = total;
  const unsigned int lane = threadIdx.x & 31u;
#pragma unroll
  for (int r = 1; r <= 4; ++r) {
    const unsigned int m = __ballot_sync(0xffffffffu, why == r);
    if (m && lane == 0) atomicAdd(&tw.state->reason[r - 1], (unsigned long long)__popc(m));
  }
}

// One CTA: exclusive output offsets of the scan blocks, the pair's count and the call's running total.
__global__ void __launch_bounds__(SCAN_THREADS) traj_scan_kernel(TrajWork tw, int nb, int k) {
  __shared__ unsigned int sw[SCAN_THREADS / 32];
  unsigned int carry = 0;
  for (int base = 0; base < nb; base += SCAN_THREADS) {
    const int i = base + threadIdx.x;
    const unsigned int v = i < nb ? tw.ebsum[i] : 0u;
    unsigned int total;
    const unsigned int ex = block_exclusive_scan<SCAN_THREADS>(v, sw, total);
    if (i < nb) tw.ebsum[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) {
    TrajState* s = tw.state;
    s->base = s->total;
    s->total += (int)carry;
    s->emitted += carry;
    tw.ndesc[k] = (int)carry;
  }
}

// One warp per track slot of list[cur] (and of the next list, for the seeds).
__global__ void __launch_bounds__(MOVE_WARPS * 32) traj_move_kernel(TrajGeom tg, TrajWork tw, TrackWork ws, int cur,
                                                                     int fr, ofdis_traj_record* rec, float* desc) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * MOVE_WARPS + warp;  // the grid is exactly cap_pad warps
  const int d = tw.dst[i];
  const int nc = tg.ns * tg.ns;
  if (d >= 0) {
    const int2 mt = pick(tw.meta, cur)[i];
    const int t1 = mt.x + 1;
    const float* S = pick(tw.st, cur) + (size_t)i * tg.ss;
    if (t1 == tg.L) {
      const int eo = tw.eoff[i];
      if (eo >= 0) {
        const size_t o = (size_t)tw.state->base + tw.ebsum[i / TRACK_BLOCK] + (unsigned int)eo;
        const TrajSeg& sg = tw.seg[i];
        if (lane == 0) rec[o] = sg.rec;
        float* D = desc + o * tg.dim;
        const float dsum = sg.dsum, div = (float)tg.tl;
        for (int j = lane; j < tg.dim; j += 32) {
          float v;
          if (j < tg.dis) {
            v = S[tg.pos + j] / dsum;
          } else {
            // HOG, HOF, MBHx, MBHy, each [nt][ns][ns][bins], from the state's [nt][ns^2][33]
            int r = j - tg.dis, q = 0;
            for (; q < 3; ++q) {
              const int part = tg.nt * nc * (q == 1 ? 9 : 8);
              if (r < part) break;
              r -= part;
            }
            const int nb = q == 1 ? 9 : 8, tc = r / (nc * nb), cell = (r / nb) % nc, b = r % nb;
            v = S[tg.pos + tg.dis + (tc * nc + cell) * TRAJ_BINS + kBinLo[q] + b] / div;
          }
          D[j] = v;
        }
      }
      if (lane == 0) pick(tw.meta, cur ^ 1)[d] = make_int2(0, mt.y + tg.L);
    } else {
      float* T = pick(tw.st, cur ^ 1) + (size_t)d * tg.ss;
      for (int j = lane; j < 2 * t1; j += 32) {
        T[j] = S[j];
        T[tg.pos + j] = S[tg.pos + j];
      }
      const int na = ((t1 - 1) / tg.tl + 1) * nc * TRAJ_BINS;
      for (int j = lane; j < na; j += 32) T[tg.pos + tg.dis + j] = S[tg.pos + tg.dis + j];
      if (lane == 0) pick(tw.meta, cur ^ 1)[d] = make_int2(t1, mt.y);
    }
  }
  if (lane == 0 && i >= ws.state->survivors && i < ws.state->alive) pick(tw.meta, cur ^ 1)[i] = make_int2(0, fr + 1);
}

}  // namespace

int launch_traj_frame(const LevelGeom& g, int fa, const TrajGeom& tg, const TrackGeom& t, const TrajWork& tw,
                      const TrackWork& ws, int noc, const unsigned char* I, const float* m, int cur, int crop_x,
                      int crop_y, cudaStream_t st) {
  if (g.nop != 2 || (noc != 1 && noc != 3)) return -1;
  const dim3 block(32, 8), grid((tg.w + 31) / 32, (tg.h + 7) / 8);
  if (noc == 3) traj_field_kernel<3><<<grid, block, 0, st>>>(g, fa, tg, tw, I, m, crop_x, crop_y);
  else traj_field_kernel<1><<<grid, block, 0, st>>>(g, fa, tg, tw, I, m, crop_x, crop_y);
  traj_hist_kernel<<<t.cap_pad / HIST_WARPS, HIST_WARPS * 32, 0, st>>>(tg, tw, ws, cur);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_traj_step(const TrajGeom& tg, const TrackGeom& t, const TrajWork& tw, const TrackWork& ws, int cur, int fr,
                     int k, ofdis_traj_record* rec, float* desc, cudaStream_t st) {
  const int nb = t.cap_pad / TRACK_BLOCK;
  traj_flag_kernel<<<nb, TRACK_BLOCK, 0, st>>>(tg, tw, ws, cur);
  traj_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(tw, nb, k);
  traj_move_kernel<<<t.cap_pad / MOVE_WARPS, MOVE_WARPS * 32, 0, st>>>(tg, tw, ws, cur, fr, rec, desc);
  return cudaGetLastError() == cudaSuccess ? 3 : -1;
}

}  // namespace ofdis

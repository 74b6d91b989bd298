// Volumetric TSDF fusion (ofdis_fuse_push / ofdis_fuse_extract / ofdis_fuse_render; the header states the contract,
// preprocess.fuse_integrate, fuse_extract and fuse_render restate it bit for bit).  Float32 without contraction.
//   fuse_integrate_kernel  one thread per voxel for the whole call: T, W (and colour) loaded once, the n frames in
//                          order, one store.  The volume's HBM traffic is then 2 x 8 (11) bytes per voxel per call; the
//                          disparity and colour gathers of neighbouring voxels fall on neighbouring pixels and go
//                          through L2.
//   fuse_count_kernel      crossings per scan block of FUSE_BLOCK voxels (4 consecutive voxels per thread);
//   fuse_scan_kernel       one CTA: the blocks' exclusive offsets (64-bit) and the total;
//   fuse_write_kernel      the block's crossings again, scanned within the CTA, written at their global index while it
//                          is below the capacity: the order of the header, whatever the grid.
//   fuse_render_kernel     one thread per (pose, pixel), fixed-step ray march to the first sign change.
#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr int FUSE_THREADS = 256;
constexpr int FUSE_VPT = FUSE_BLOCK / FUSE_THREADS;  // voxels per thread of the count and write kernels
constexpr int FUSE_SCAN_THREADS = 1024;
constexpr int FUSE_RENDER_ROWS = 8;                 // a render CTA is 32 x 8 pixels of one pose

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }

__global__ void __launch_bounds__(FUSE_THREADS) fuse_integrate_kernel(FuseGeom g, FuseVolume v, FusePush p) {
  const long long a = (long long)blockIdx.x * FUSE_THREADS + threadIdx.x;
  if (a >= g.count) return;
  const int i = (int)(a % g.nx);
  const long long r = a / g.nx;
  const int j = (int)(r % g.ny), k = (int)(r / g.ny);
  const float X = g.ox + (float)i * g.voxel, Y = g.oy + (float)j * g.voxel, Z = g.oz + (float)k * g.voxel;
  float T = v.T[a], Wt = v.W[a];
  unsigned char c[3] = {0, 0, 0};
  if (v.C) {
    c[0] = v.C[3 * a];
    c[1] = v.C[3 * a + 1];
    c[2] = v.C[3 * a + 2];
  }
  const DispCamera& cam = p.cam;
  for (int f = 0; f < p.n; ++f) {
    const float* q = p.g + 12 * f;
    const float Zc = ((q[8] * X + q[9] * Y) + q[10] * Z) + q[11];
    if (!(Zc > 0.0f)) continue;
    const float Xc = ((q[0] * X + q[1] * Y) + q[2] * Z) + q[3];
    const float Yc = ((q[4] * X + q[5] * Y) + q[6] * Z) + q[7];
    const float uu = ((cam.fx * Xc) / Zc + cam.cx) + 0.5f, vv = ((cam.fy * Yc) / Zc + cam.cy) + 0.5f;
    if (!(uu >= 0.0f && uu < (float)p.w && vv >= 0.0f && vv < (float)p.h)) continue;
    const int px = (int)floorf(uu), py = (int)floorf(vv);
    const size_t o = (size_t)py * p.w + px;
    const float d = __ldg(p.disp + f * p.disp_stride + o);
    const float s = d + cam.doffs;
    if (!known_d(d) || !(s > 0.0f)) continue;
    const float z = cam.fb / s;
    if (z > p.max_depth) continue;
    const float sdf = z - Zc;
    if (sdf < -g.mu) continue;
    const float fv = fminf(1.0f, sdf / g.mu);
    const float W1 = Wt + 1.0f;
    T = (T * Wt + fv) / W1;
    if (v.C) {
      const unsigned char* I = p.frames + f * p.frame_stride + o * p.noc;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float obs = (float)__ldg(I + (p.noc == 3 ? ch : 0));
        c[ch] = (unsigned char)floorf(((float)c[ch] * Wt + obs) / W1 + 0.5f);
      }
    }
    Wt = fminf(W1, g.max_weight);
  }
  v.T[a] = T;
  v.W[a] = Wt;
  if (v.C) {
    v.C[3 * a] = c[0];
    v.C[3 * a + 1] = c[1];
    v.C[3 * a + 2] = c[2];
  }
}

// bit e (0 x, 1 y, 2 z): voxel a = (i, j, k) and its neighbour along e form a crossing
__device__ __forceinline__ unsigned crossings(const FuseGeom& g, const FuseVolume& v, float minw, long long a) {
  if (a >= g.count) return 0u;
  const float Ta = v.T[a], Wa = v.W[a];
  if (!(Wa >= minw && fabsf(Ta) < 1.0f)) return 0u;
  const int i = (int)(a % g.nx);
  const long long r = a / g.nx;
  const int j = (int)(r % g.ny), k = (int)(r / g.ny);
  const bool in[3] = {i + 1 < g.nx, j + 1 < g.ny, k + 1 < g.nz};
  const long long step[3] = {1, g.nx, (long long)g.nx * g.ny};
  unsigned m = 0;
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    if (!in[e]) continue;
    const float Tb = v.T[a + step[e]], Wb = v.W[a + step[e]];
    if (Wb >= minw && fabsf(Tb) < 1.0f && ((Ta > 0.0f) != (Tb > 0.0f))) m |= 1u << e;
  }
  return m;
}

__global__ void __launch_bounds__(FUSE_THREADS) fuse_count_kernel(FuseGeom g, FuseVolume v, float minw,
                                                                  unsigned long long* bsum) {
  __shared__ unsigned int sw[FUSE_THREADS / 32];
  const long long a0 = (long long)blockIdx.x * FUSE_BLOCK + (long long)threadIdx.x * FUSE_VPT;
  unsigned cnt = 0;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) cnt += __popc(crossings(g, v, minw, a0 + q));
  unsigned int total;
  block_exclusive_scan<FUSE_THREADS>(cnt, sw, total);
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

// exclusive 64-bit scan of the nb block counts in place; the sum to *total
__global__ void __launch_bounds__(FUSE_SCAN_THREADS) fuse_scan_kernel(unsigned long long* bsum, int nb,
                                                                      unsigned long long* total) {
  __shared__ unsigned long long sw[FUSE_SCAN_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long carry = 0;
  for (int base = 0; base < nb; base += FUSE_SCAN_THREADS) {
    const int idx = base + threadIdx.x;
    const unsigned long long val = idx < nb ? bsum[idx] : 0ull;
    unsigned long long x = val;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) sw[warp] = x;
    __syncthreads();
    if (warp == 0) {
      unsigned long long s = sw[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += y;
      }
      sw[lane] = s;
    }
    __syncthreads();
    if (idx < nb) bsum[idx] = carry + x - val + (warp ? sw[warp - 1] : 0ull);
    carry += sw[FUSE_SCAN_THREADS / 32 - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(FUSE_THREADS) fuse_write_kernel(FuseGeom g, FuseVolume v, float minw,
                                                                  const unsigned long long* bsum,
                                                                  ofdis_fuse_point* out, long long cap) {
  __shared__ unsigned int sw[FUSE_THREADS / 32];
  const long long a0 = (long long)blockIdx.x * FUSE_BLOCK + (long long)threadIdx.x * FUSE_VPT;
  unsigned m[FUSE_VPT], cnt = 0;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) {
    m[q] = crossings(g, v, minw, a0 + q);
    cnt += __popc(m[q]);
  }
  unsigned int total;
  const unsigned int ex = block_exclusive_scan<FUSE_THREADS>(cnt, sw, total);
  unsigned long long o = bsum[blockIdx.x] + ex;
  if (!cnt || o >= (unsigned long long)cap) return;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) {
    if (!m[q]) continue;
    const long long a = a0 + q;
    const int i = (int)(a % g.nx);
    const long long r = a / g.nx;
    const int j = (int)(r % g.ny), k = (int)(r / g.ny);
    const long long sy = g.nx, sz = (long long)g.nx * g.ny;
    const float* T = v.T;
    const float Ta = T[a];
    const float gx = T[a - i + min(i + 1, g.nx - 1)] - T[a - i + max(i - 1, 0)];
    const float gy = T[a + (min(j + 1, g.ny - 1) - j) * sy] - T[a + (max(j - 1, 0) - j) * sy];
    const float gz = T[a + (min(k + 1, g.nz - 1) - k) * sz] - T[a + (max(k - 1, 0) - k) * sz];
    const float L = sqrtf((gx * gx + gy * gy) + gz * gz);
    const float nrm[3] = {L > 0.0f ? gx / L : qnan(), L > 0.0f ? gy / L : qnan(), L > 0.0f ? gz / L : qnan()};
    const float P[3] = {g.ox + (float)i * g.voxel, g.oy + (float)j * g.voxel, g.oz + (float)k * g.voxel};
    const long long step[3] = {1, sy, sz};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      if (!((m[q] >> e) & 1u)) continue;
      if (o >= (unsigned long long)cap) return;
      const long long b = a + step[e];
      const float Tb = T[b];
      const float t = Ta / (Ta - Tb);
      const float dt = t * g.voxel;
      ofdis_fuse_point rec;
      rec.x = e == 0 ? P[0] + dt : P[0];
      rec.y = e == 1 ? P[1] + dt : P[1];
      rec.z = e == 2 ? P[2] + dt : P[2];
      rec.nx = nrm[0];
      rec.ny = nrm[1];
      rec.nz = nrm[2];
      const long long src = t < 0.5f ? a : b;
      rec.r = v.C ? v.C[3 * src] : 0;
      rec.g = v.C ? v.C[3 * src + 1] : 0;
      rec.b = v.C ? v.C[3 * src + 2] : 0;
      rec.pad = 0;
      out[o++] = rec;
    }
  }
}

// trilinear T at voxel coordinates q, or false where a corner lies outside or has W < minw
__device__ __forceinline__ bool fuse_sample(const FuseGeom& g, const FuseVolume& v, float minw, const float (&q)[3],
                                            float& out) {
  const int n[3] = {g.nx, g.ny, g.nz};
  int i0[3];
  float fr[3];
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    const float fl = floorf(q[e]);
    if (!(fl >= 0.0f && fl <= (float)(n[e] - 2))) return false;
    i0[e] = (int)fl;
    fr[e] = q[e] - fl;
  }
  const long long sy = g.nx, sz = (long long)g.nx * g.ny;
  const long long base = ((long long)i0[2] * g.ny + i0[1]) * g.nx + i0[0];
  const long long off[8] = {0, 1, sy, sy + 1, sz, sz + 1, sz + sy, sz + sy + 1};
  float c[8];
#pragma unroll
  for (int q8 = 0; q8 < 8; ++q8)
    if (!(__ldg(v.W + base + off[q8]) >= minw)) return false;
#pragma unroll
  for (int q8 = 0; q8 < 8; ++q8) c[q8] = __ldg(v.T + base + off[q8]);
  const float gx = 1.0f - fr[0], gy = 1.0f - fr[1], gz = 1.0f - fr[2];
  const float x00 = c[0] * gx + c[1] * fr[0], x10 = c[2] * gx + c[3] * fr[0];
  const float x01 = c[4] * gx + c[5] * fr[0], x11 = c[6] * gx + c[7] * fr[0];
  const float y0 = x00 * gy + x10 * fr[1], y1 = x01 * gy + x11 * fr[1];
  out = y0 * gz + y1 * fr[2];
  return true;
}

__global__ void __launch_bounds__(32 * FUSE_RENDER_ROWS) fuse_render_kernel(FuseGeom g, FuseVolume v, FuseRender p) {
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * FUSE_RENDER_ROWS + threadIdx.y, k = blockIdx.z;
  if (x >= p.w || y >= p.h) return;
  const float* P = p.pose + 12 * k;
  const DispCamera& cam = p.cam;
  const float r0 = ((float)x - cam.cx) / cam.fx, r1 = ((float)y - cam.cy) / cam.fy;
  float depth = qnan();
  bool prev = false;
  float Tp = 0.0f, Zp = 0.0f;
  for (int s = 0; s <= FUSE_MAX_SAMPLES; ++s) {
    const float Zs = p.z_near + (float)s * p.step;
    if (!(Zs <= p.z_far)) break;
    const float cx = r0 * Zs, cy = r1 * Zs;
    float q[3];
    q[0] = ((((P[0] * cx + P[1] * cy) + P[2] * Zs) + P[3]) - g.ox) / g.voxel;
    q[1] = ((((P[4] * cx + P[5] * cy) + P[6] * Zs) + P[7]) - g.oy) / g.voxel;
    q[2] = ((((P[8] * cx + P[9] * cy) + P[10] * Zs) + P[11]) - g.oz) / g.voxel;
    float T;
    const bool known = fuse_sample(g, v, p.min_weight, q, T);
    if (known && prev && Tp > 0.0f && T <= 0.0f) {
      depth = Zp + p.step * (Tp / (Tp - T));
      break;
    }
    prev = known;
    Tp = T;
    Zp = Zs;
  }
  p.depth[((size_t)k * p.h + y) * p.w + x] = depth;
}

}  // namespace

int launch_fuse_push(const FuseGeom& g, const FuseVolume& v, const FusePush& p, cudaStream_t st) {
  const long long blocks = (g.count + FUSE_THREADS - 1) / FUSE_THREADS;
  fuse_integrate_kernel<<<(unsigned)blocks, FUSE_THREADS, 0, st>>>(g, v, p);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_fuse_count(const FuseGeom& g, const FuseVolume& v, float min_weight, const FuseWork& ws, cudaStream_t st) {
  const int nb = (int)((g.count + FUSE_BLOCK - 1) / FUSE_BLOCK);
  fuse_count_kernel<<<nb, FUSE_THREADS, 0, st>>>(g, v, min_weight, ws.bsum);
  fuse_scan_kernel<<<1, FUSE_SCAN_THREADS, 0, st>>>(ws.bsum, nb, ws.total);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_fuse_write(const FuseGeom& g, const FuseVolume& v, float min_weight, const FuseWork& ws,
                      ofdis_fuse_point* out, long long cap, cudaStream_t st) {
  const int nb = (int)((g.count + FUSE_BLOCK - 1) / FUSE_BLOCK);
  fuse_write_kernel<<<nb, FUSE_THREADS, 0, st>>>(g, v, min_weight, ws.bsum, out, cap);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_fuse_render(const FuseGeom& g, const FuseVolume& v, const FuseRender& p, int n, cudaStream_t st) {
  const dim3 block(32, FUSE_RENDER_ROWS), grid((p.w + 31) / 32, (p.h + FUSE_RENDER_ROWS - 1) / FUSE_RENDER_ROWS, n);
  fuse_render_kernel<<<grid, block, 0, st>>>(g, v, p);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ofdis

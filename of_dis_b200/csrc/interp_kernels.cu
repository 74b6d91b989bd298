// Frame interpolation from bidirectional flows (ofdis_interpolate_fullres; the header states the contract,
// preprocess.interpolate_frames restates it bit for bit).  The algorithm follows the description of the
// interpolation of Baker et al., "A Database and Evaluation Methodology for Optical Flow" (IJCV 2011): forward splat
// of the flow to time t with the lowest match cost winning, outside-in hole filling, and occlusion-aware blending of
// the two frames.  Four kernels per call, between which ofdis_capi.cu launches the consistency masks and runs the
// hole-filling rounds:
//   interp_splat_kernel    one thread per source pixel of I0: match cost, then atomicMin of its 64-bit key into the
//                          (up to four) target pixels around X + t F(X);
//   interp_resolve_kernel  one thread per target: u_t = F of the winning source, or the pixel joins the hole list;
//   interp_fill_kernel     one round of the Jacobi hole filling over the hole list;
//   interp_blend_kernel    one thread per target: the two samples, the occlusion flags, the output bytes.
// F is read through upsample_at; no full-resolution copy of a flow is stored.  Float32 without contraction.
#include <algorithm>
#include <climits>

#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr unsigned long long kNoSource = ~0ull;

__device__ __forceinline__ bool in_frame(float x, float y, int w, int h) {
  return x >= 0.f && x <= (float)(w - 1) && y >= 0.f && y <= (float)(h - 1);
}

// Appends index `o` of every lane with `put` to list[0, *count) with one atomic per warp (order is irrelevant: the
// rounds are Jacobi rounds).  All 32 lanes of the warp take part.
__device__ __forceinline__ void warp_append(bool put, unsigned int o, unsigned int* list, unsigned int* count) {
  const unsigned int lane = threadIdx.x & 31u;
  const unsigned int m = __ballot_sync(0xffffffffu, put);
  if (!m) return;
  const int leader = __ffs(m) - 1;
  unsigned int base = 0;
  if ((int)lane == leader) base = atomicAdd(count, (unsigned int)__popc(m));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (put) list[base + __popc(m & ((1u << lane) - 1u))] = o;
}

// Match cost and forward splat of source pixel (X, Y) of pair blockIdx.z.
template <int NOP, int NOC>
__global__ void __launch_bounds__(256) interp_splat_kernel(LevelGeom g, int fa, InterpSrc s, InterpWork ws) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  const int w = s.w, h = s.h;
  if (X >= w || Y >= h) return;
  const int fr = blockIdx.z;
  const float* F = g.flow + (size_t)frame_of(g, fa, fr) * g.flow_frame_stride;
  float f[2] = {0.f, 0.f};
  upsample_at<NOP>(g, F, X, Y, s.crop_x, s.crop_y, [&f](int c, float v) { f[c] = v; });
  const float u = f[0], v = NOP == 2 ? f[1] : 0.f;
  if (!(fabsf(u) <= 1e9f && fabsf(v) <= 1e9f)) return;  // unknown (NaN fails): splats nowhere
  const size_t pix = (size_t)w * h;
  const float xs = (float)X + u, ys = (float)Y + v;
  float c = __int_as_float(0x7f800000);
  if (in_frame(xs, ys, w, h)) {
    float b[NOC];
    bil_u8<NOC>(s.i1 + fr * s.stride, w, h, xs, ys, b);
    const unsigned char* p = s.i0 + fr * s.stride + ((size_t)Y * w + X) * NOC;
    c = 0.f;
    for (int k = 0; k < NOC; ++k) c += fabsf((float)p[k] - b[k]);
  }
  const unsigned long long key = ((unsigned long long)__float_as_uint(c) << 32) | (unsigned int)(Y * w + X);
  const float px = (float)X + s.t * u, py = (float)Y + s.t * v;
  if (!(px > -1.f && px < (float)w && py > -1.f && py < (float)h)) return;  // no target in the frame
  const float flx = floorf(px), fly = floorf(py);
  const int tx = (int)flx, ty = (int)fly, nx = px > flx ? 2 : 1, ny = py > fly ? 2 : 1;
  unsigned long long* K = ws.keys + fr * pix;
  bool hit = false;
  for (int dy = 0; dy < ny; ++dy) {
    const int yy = ty + dy;
    if (yy < 0 || yy >= h) continue;
    for (int dx = 0; dx < nx; ++dx) {
      const int xx = tx + dx;
      if (xx < 0 || xx >= w) continue;
      atomicMin(K + (size_t)yy * w + xx, key);
      hit = true;
    }
  }
  if (hit) ws.any[fr] = 1;
}

// u_t of every target: F of its winning source (stamp 0); 0 (stamp 0) in a pair no source reached; else a hole
// (stamp INT_MAX) appended to list[0].
template <int NOP>
__global__ void __launch_bounds__(256) interp_resolve_kernel(LevelGeom g, int fa, InterpSrc s, InterpWork ws) {
  pdl_wait();
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  const int w = s.w, h = s.h, fr = blockIdx.z;
  const bool inside = X < w && Y < h;
  const size_t o = (size_t)fr * w * h + (size_t)Y * w + X;
  bool hole = false;
  if (inside) {
    const unsigned long long key = ws.keys[o];
    float* ut = ws.ut + o * NOP;
    if (key != kNoSource) {
      const unsigned int src = (unsigned int)key;
      const float* F = g.flow + (size_t)frame_of(g, fa, fr) * g.flow_frame_stride;
      upsample_at<NOP>(g, F, (int)(src % (unsigned int)w), (int)(src / (unsigned int)w), s.crop_x, s.crop_y,
                       [ut](int c, float v) { ut[c] = v; });
      ws.stamp[o] = 0;
    } else if (!ws.any[fr]) {
      for (int c = 0; c < NOP; ++c) ut[c] = 0.f;
      ws.stamp[o] = 0;
    } else {
      ws.stamp[o] = INT_MAX;
      hole = true;
    }
  }
  warp_append(hole, (unsigned int)o, ws.list[0], ws.count);
}

// Round r of the hole filling: a hole with a neighbour (left, right, up, down) filled before round r (stamp < r)
// takes the mean of those neighbours and stamp r; the others go to the next round's list.  A pixel filled in this
// round has stamp r, so no other hole reads it before round r + 1: the round is a Jacobi round whatever the order.
template <int NOP>
__global__ void __launch_bounds__(256) interp_fill_kernel(InterpWork ws, int w, int h, int r) {
  pdl_wait();
  const unsigned int n_in = ws.count[r - 1];
  const unsigned int* in = ws.list[(r - 1) & 1];
  unsigned int* out = ws.list[r & 1];
  const size_t pix = (size_t)w * h;
  for (unsigned int base = blockIdx.x * blockDim.x; base < n_in; base += gridDim.x * blockDim.x) {
    const unsigned int i = base + threadIdx.x;
    bool keep = false;
    unsigned int o = 0;
    if (i < n_in) {
      o = in[i];
      const unsigned int p = (unsigned int)(o % pix);
      const int x = (int)(p % (unsigned int)w), y = (int)(p / (unsigned int)w);
      const size_t nb[4] = {o - 1, o + 1, o - w, o + w};
      const bool ok[4] = {x > 0, x < w - 1, y > 0, y < h - 1};
      float sum[NOP];
      for (int c = 0; c < NOP; ++c) sum[c] = 0.f;
      int k = 0;
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        if (!ok[d] || ws.stamp[nb[d]] >= r) continue;
        for (int c = 0; c < NOP; ++c) sum[c] += ws.ut[nb[d] * NOP + c];
        ++k;
      }
      if (k) {
        for (int c = 0; c < NOP; ++c) ws.ut[(size_t)o * NOP + c] = sum[c] / (float)k;
        ws.stamp[o] = r;
      } else {
        keep = true;
      }
    }
    warp_append(keep, o, out, ws.count + r);
  }
}

// The output bytes of target (X, Y): samples of I0 at X - t u_t and of I1 at X + (1 - t) u_t, chosen by the frame
// tests and the occlusion flags of the consistency masks.
template <int NOP, int NOC>
__global__ void __launch_bounds__(256) interp_blend_kernel(InterpSrc s, InterpWork ws, unsigned char* out) {
  pdl_wait();
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  const int w = s.w, h = s.h;
  if (X >= w || Y >= h) return;
  const int fr = blockIdx.z;
  const size_t pix = (size_t)w * h, o = (size_t)fr * pix + (size_t)Y * w + X;
  const float u = ws.ut[o * NOP], v = NOP == 2 ? ws.ut[o * NOP + 1] : 0.f;
  const float t = s.t;
  const float x0 = (float)X - t * u, y0 = (float)Y - t * v;
  const float x1 = (float)X + (1.0f - t) * u, y1 = (float)Y + (1.0f - t) * v;
  const bool in0 = in_frame(x0, y0, w, h), in1 = in_frame(x1, y1, w, h);
  const float wm = (float)(w - 1), hm = (float)(h - 1);
  float s0[NOC], s1[NOC];
  bil_u8<NOC>(s.i0 + fr * s.stride, w, h, fminf(fmaxf(x0, 0.f), wm), fminf(fmaxf(y0, 0.f), hm), s0);
  bil_u8<NOC>(s.i1 + fr * s.stride, w, h, fminf(fmaxf(x1, 0.f), wm), fminf(fmaxf(y1, 0.f), hm), s1);
  const bool o0 = in0 && ws.m0[fr * pix + (size_t)(int)floorf(y0 + 0.5f) * w + (int)floorf(x0 + 0.5f)] != 0;
  const bool o1 = in1 && ws.m1[fr * pix + (size_t)(int)floorf(y1 + 0.5f) * w + (int)floorf(x1 + 0.5f)] != 0;
  const bool only0 = (in0 && !in1) || (o0 && !o1), only1 = (in1 && !in0) || (o1 && !o0);
  unsigned char* q = out + o * NOC;
  for (int c = 0; c < NOC; ++c) {
    const float val = only0 ? s0[c] : only1 ? s1[c] : (1.0f - t) * s0[c] + t * s1[c];
    q[c] = round_u8(val);
  }
}

template <int NOP>
int splat_noc(const LevelGeom& g, int fa, int n, const InterpSrc& s, const InterpWork& ws, cudaStream_t st) {
  const dim3 block(32, 8), grid((s.w + 31) / 32, (s.h + 7) / 8, n);
  if (g.noc == 3) interp_splat_kernel<NOP, 3><<<grid, block, 0, st>>>(g, fa, s, ws);
  else interp_splat_kernel<NOP, 1><<<grid, block, 0, st>>>(g, fa, s, ws);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

template <int NOP>
int blend_noc(int noc, int n, const InterpSrc& s, const InterpWork& ws, unsigned char* out, cudaStream_t st) {
  const dim3 block(32, 8), grid((s.w + 31) / 32, (s.h + 7) / 8, n);
  if (noc == 3) interp_blend_kernel<NOP, 3><<<grid, block, 0, st>>>(s, ws, out);
  else interp_blend_kernel<NOP, 1><<<grid, block, 0, st>>>(s, ws, out);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace

int launch_interp_splat(const LevelGeom& g, int fa, int n, const InterpSrc& s, const InterpWork& ws, cudaStream_t st) {
  if (g.noc != 1 && g.noc != 3) return -1;
  return g.nop == 2 ? splat_noc<2>(g, fa, n, s, ws, st) : splat_noc<1>(g, fa, n, s, ws, st);
}

int launch_interp_resolve(const LevelGeom& g, int fa, int n, const InterpSrc& s, const InterpWork& ws,
                          cudaStream_t st) {
  const dim3 block(32, 8), grid((s.w + 31) / 32, (s.h + 7) / 8, n);
  if (g.nop == 2) interp_resolve_kernel<2><<<grid, block, 0, st>>>(g, fa, s, ws);
  else interp_resolve_kernel<1><<<grid, block, 0, st>>>(g, fa, s, ws);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_interp_fill(int nop, const InterpWork& ws, int w, int h, int r0, int rounds, unsigned int bound,
                       cudaStream_t st) {
  const unsigned int blocks = std::min<unsigned int>((bound + 255) / 256, 1024u);
  for (int r = r0; r < r0 + rounds; ++r) {
    if (nop == 2) interp_fill_kernel<2><<<std::max(blocks, 1u), 256, 0, st>>>(ws, w, h, r);
    else interp_fill_kernel<1><<<std::max(blocks, 1u), 256, 0, st>>>(ws, w, h, r);
    if (cudaGetLastError() != cudaSuccess) return -1;
  }
  return rounds;
}

int launch_interp_blend(int nop, int noc, int n, const InterpSrc& s, const InterpWork& ws, unsigned char* out,
                        cudaStream_t st) {
  if (noc != 1 && noc != 3) return -1;
  return nop == 2 ? blend_noc<2>(noc, n, s, ws, out, st) : blend_noc<1>(noc, n, s, ws, out, st);
}

}  // namespace ofdis

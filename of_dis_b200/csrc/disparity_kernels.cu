// Filtered disparities, depth and point clouds from stereo flows (ofdis_disparity_fullres; the header states the
// contract, preprocess.disparity_filter restates it bit for bit).  Every pair of a call is in one grid dimension, so
// a call launches the same kernels whatever its number of pairs:
//   disp_classify_kernel     one thread per pixel: the positive disparity d, the status (range, left-right check) and
//                            the initial union-find parent;
//   disp_ccl_tile_kernel     speckles: union-find of the joined 4-neighbours inside a 32 x 32 tile in shared memory,
//                            the tile roots written as frame pixel indices;
//   disp_ccl_border_kernel   speckles: one thread per pixel pair across a tile border, merged with atomicMin on the
//                            global parents;
//   disp_ccl_count_kernel    speckles: every parent flattened to its root, the component sizes by atomicAdd there;
//   disp_fill_rows_kernel    fill: one warp per row, the nearest value on each side by ballots and shuffles;
//   disp_fill_links_kernel   fill: one warp per pair, the nearest rows with a value above and below every row;
//   disp_output_kernel       one thread per pixel: the column pass, depth and xyz, and the outputs.
// The union-find always hangs the larger root under the smaller one, so a component's root is its smallest pixel
// index whatever order the atomics land in; only membership and sizes leave the stage.  Float32 without contraction.
#include <algorithm>

#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr int CCL_TILE = 32;  // tile edge of disp_ccl_tile_kernel: 32 x 8 threads, four rows each
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }

// d_p and d_q of two status-0 4-neighbours join one component
__device__ __forceinline__ bool joined(float dp, float dq, float diff) { return fabsf(dp - dq) <= diff; }

// Root of x in a parent array whose entries only ever decrease towards a root (L[r] == r), with path halving: every
// visited entry is lowered to its grandparent with atomicMin, which is still an ancestor in the same set, so a
// concurrent merge (which also only lowers entries) never loses a link.  L reads the entries (volatile shared memory,
// or global loads that bypass L1, so that a thread sees the other SMs' atomics), A is the same array for the atomics.
template <typename P>
__device__ __forceinline__ int find_root(P L, int* A, int x) {
  while (true) {
    const int p = L[x];
    if (p == x) return x;
    const int gp = L[p];
    if (gp == p) return p;
    atomicMin(A + x, gp);
    x = gp;
  }
}
struct GlobalParents {
  int* L;
  __device__ __forceinline__ int operator[](int i) const { return __ldcg(L + i); }
};

// Union of the sets of a and b (Playne & Hawick 2018): the larger root goes under the smaller one with atomicMin;
// when another thread moved that root first, retry from what it found
template <typename P>
__device__ __forceinline__ void merge(P L, int* A, int a, int b) {
  bool done;
  do {
    a = find_root(L, A, a);
    b = find_root(L, A, b);
    if (a < b) {
      const int old = atomicMin(A + b, a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const int old = atomicMin(A + a, b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

// The status of a pixel once the speckles are known: 4 for a status-0 pixel of a component of at most S pixels
__device__ __forceinline__ unsigned char speckle_status(unsigned char st, const int* parent, const int* size, size_t o,
                                                        size_t base, int S) {
  return st == 0 && size[base + parent[o]] <= S ? (unsigned char)4 : st;
}

// d = -F (+F in a slot marked swapped); status 3 outside [0, 1e9] (NaN fails, -0 passes), else with lr the mask of
// consistency_at against frame fb's flow; every pixel its own parent and no size yet.
__global__ void __launch_bounds__(256) disp_classify_kernel(LevelGeom g, int fa, int fb, int lr, float alpha,
                                                            float beta, DispWork ws, int w_org, int h_org, int crop_x,
                                                            int crop_y) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X >= w_org || Y >= h_org) return;
  const int fr = blockIdx.z, frame = frame_of(g, fa, fr);
  const float* F = g.flow + (size_t)frame * g.flow_frame_stride;
  float f[2] = {0.f, 0.f};
  upsample_at<1>(g, F, X, Y, crop_x, crop_y, [&f](int c, float v) { f[c] = v; });
  const float d = swapped_of(g, frame) ? f[0] : -f[0];
  unsigned char st = d >= 0.0f && d <= 1e9f ? 0 : 3;
  if (st == 0 && lr) {
    const float* B = g.flow + (size_t)frame_of(g, fb, fr) * g.flow_frame_stride;
    consistency_at<1>(g, B, f, X, Y, w_org, h_org, crop_x, crop_y, alpha, beta, [&st](unsigned char m, float) { st = m; });
  }
  const int p = Y * w_org + X;
  const size_t o = (size_t)fr * h_org * w_org + p;
  ws.val[o] = d;
  ws.status[o] = st;
  ws.parent[o] = p;
  ws.size[o] = 0;
}

// Connected components of the status-0 pixels inside one 32 x 32 tile: union-find on tile indices (row-major, so the
// order of frame indices) in shared memory, flattened; every pixel's parent becomes its tile root as a frame index.
__global__ void __launch_bounds__(256) disp_ccl_tile_kernel(DispWork ws, float diff, int w_org, int h_org) {
  __shared__ int lab[CCL_TILE * CCL_TILE];
  __shared__ float sd[CCL_TILE * CCL_TILE];
  __shared__ unsigned char ok[CCL_TILE * CCL_TILE];
  const int lx = threadIdx.x, x0 = blockIdx.x * CCL_TILE, y0 = blockIdx.y * CCL_TILE, x = x0 + lx;
  const size_t base = (size_t)blockIdx.z * h_org * w_org;
  for (int k = 0; k < CCL_TILE / 8; ++k) {
    const int ly = threadIdx.y + 8 * k, y = y0 + ly, i = ly * CCL_TILE + lx;
    const bool in = x < w_org && y < h_org;
    const size_t o = base + (size_t)y * w_org + x;
    ok[i] = in && ws.status[o] == 0;
    sd[i] = in ? ws.val[o] : 0.f;
    lab[i] = i;
  }
  __syncthreads();
  volatile int* vl = lab;
  for (int k = 0; k < CCL_TILE / 8; ++k) {
    const int ly = threadIdx.y + 8 * k, i = ly * CCL_TILE + lx;
    if (!ok[i]) continue;
    if (lx > 0 && ok[i - 1] && joined(sd[i], sd[i - 1], diff)) merge(vl, lab, i, i - 1);
    if (ly > 0 && ok[i - CCL_TILE] && joined(sd[i], sd[i - CCL_TILE], diff)) merge(vl, lab, i, i - CCL_TILE);
  }
  __syncthreads();
  for (int k = 0; k < CCL_TILE / 8; ++k) {
    const int ly = threadIdx.y + 8 * k, y = y0 + ly, i = ly * CCL_TILE + lx;
    if (x >= w_org || y >= h_org || !ok[i]) continue;
    const int r = find_root(vl, lab, i);
    ws.parent[base + (size_t)y * w_org + x] = (y0 + r / CCL_TILE) * w_org + x0 + r % CCL_TILE;
  }
}

// One thread per pixel pair across a tile border: the vertical borders (x = 32 bx, bx >= 1, against x - 1) first,
// then the horizontal ones (y = 32 by, against y - 1); joined pairs are merged in the pair's global parents.
__global__ void __launch_bounds__(256) disp_ccl_border_kernel(DispWork ws, float diff, int w_org, int h_org,
                                                              long long nv, long long nh) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nv + nh) return;
  int x, y, q;
  if (t < nv) {
    x = (int)(t / h_org + 1) * CCL_TILE;
    y = (int)(t % h_org);
    q = y * w_org + x - 1;
  } else {
    const long long u = t - nv;
    x = (int)(u % w_org);
    y = (int)(u / w_org + 1) * CCL_TILE;
    q = (y - 1) * w_org + x;
  }
  const int p = y * w_org + x;
  const size_t base = (size_t)blockIdx.y * h_org * w_org;
  if (ws.status[base + p] != 0 || ws.status[base + q] != 0 || !joined(ws.val[base + p], ws.val[base + q], diff)) return;
  int* L = ws.parent + base;
  merge(GlobalParents{L}, L, p, q);
}

// Every status-0 pixel's parent flattened to its root, and the root's size counted.  The finds halve the paths with
// atomicMin, not plain stores: a root is the smallest index on every path to it, so an entry that has reached its root
// (a pixel's own final store included) is never raised again by another warp's halving.  Within a warp (32 pixels of a
// row) the pixels that share a tile root walk from it once, and the pixels that share a root add their count with one
// atomicAdd.
__global__ void __launch_bounds__(256) disp_ccl_count_kernel(DispWork ws, int w_org, int h_org) {
  const int lane = threadIdx.x & 31;
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  const size_t base = (size_t)blockIdx.z * h_org * w_org;
  const int p = Y * w_org + X;
  const bool v = X < w_org && Y < h_org && ws.status[base + p] == 0;
  int* L = ws.parent + base;
  const int t = v ? __ldcg(L + p) : -1;
  const unsigned same_t = __match_any_sync(FULL, t);
  int r = 0;
  if (v && lane == __ffs(same_t) - 1) r = find_root(GlobalParents{L}, L, t);
  r = __shfl_sync(FULL, r, __ffs(same_t) - 1);
  if (v && r != t) atomicMin(L + p, r);
  const unsigned same_r = __match_any_sync(FULL, v ? r : -1);
  if (v && lane == __ffs(same_r) - 1) atomicAdd(ws.size + base + r, __popc(same_r));
}

// The row pass, one warp per row: with speckles the status becomes final (4); then left to right the nearest value
// at or left of every pixel (into the parent array, no longer needed), right to left the nearest at or right of it,
// and the row's values into val: d where the status is 0, else the smaller of the two (the left one where they are
// equal), the one that exists, or qNaN.  rowfull: the row has a value.
__global__ void __launch_bounds__(256) disp_fill_rows_kernel(DispWork ws, int speckle, int S, int w_org, int h_org) {
  const int lane = threadIdx.x & 31, y = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (y >= h_org) return;
  const size_t base = (size_t)blockIdx.y * h_org * w_org, row = base + (size_t)y * w_org;
  int* lbuf = ws.parent;
  float carry = qnan();
  bool any = false;
  for (int x0 = 0; x0 < w_org; x0 += 32) {
    const int x = x0 + lane;
    const size_t o = row + x;
    bool valid = false;
    float d = 0.f;
    if (x < w_org) {
      unsigned char st = ws.status[o];
      if (speckle) {
        const unsigned char s2 = speckle_status(st, ws.parent, ws.size, o, base, S);
        if (s2 != st) ws.status[o] = s2;
        st = s2;
      }
      valid = st == 0;
      d = ws.val[o];
    }
    const unsigned m = __ballot_sync(FULL, valid), le = m & (FULL >> (31 - lane));
    const float from = __shfl_sync(FULL, d, le ? 31 - __clz(le) : 0);
    const float last = __shfl_sync(FULL, d, m ? 31 - __clz(m) : 0);
    if (x < w_org) lbuf[o] = __float_as_int(le ? from : carry);
    if (m) carry = last;
    any |= m != 0;
  }
  carry = qnan();
  for (int x0 = (w_org - 1) / 32 * 32; x0 >= 0; x0 -= 32) {
    const int x = x0 + lane;
    const size_t o = row + x;
    const bool valid = x < w_org && ws.status[o] == 0;
    const float d = valid ? ws.val[o] : 0.f;
    const unsigned m = __ballot_sync(FULL, valid), ge = m & (FULL << lane);
    const float from = __shfl_sync(FULL, d, ge ? __ffs(ge) - 1 : 0);
    const float first = __shfl_sync(FULL, d, m ? __ffs(m) - 1 : 0);
    if (x < w_org) {
      const float L = __int_as_float(lbuf[o]), R = ge ? from : carry;
      ws.val[o] = valid ? d : isnan(L) ? R : isnan(R) ? L : std_min(L, R);
    }
    if (m) carry = first;
  }
  if (lane == 0) ws.rowfull[(size_t)blockIdx.y * h_org + y] = any ? 1 : 0;
}

// One warp per pair: for every row the nearest row with a value above (up) and below (down) it, -1 where none
__global__ void __launch_bounds__(32) disp_fill_links_kernel(DispWork ws, int h_org) {
  const int lane = threadIdx.x;
  const size_t rb = (size_t)blockIdx.x * h_org;
  int carry = -1;
  for (int y0 = 0; y0 < h_org; y0 += 32) {
    const int y = y0 + lane;
    const unsigned m = __ballot_sync(FULL, y < h_org && ws.rowfull[rb + y]), lt = m & ((1u << lane) - 1u);
    if (y < h_org) ws.up[rb + y] = lt ? y0 + 31 - __clz(lt) : carry;
    if (m) carry = y0 + 31 - __clz(m);
  }
  carry = -1;
  for (int y0 = (h_org - 1) / 32 * 32; y0 >= 0; y0 -= 32) {
    const int y = y0 + lane;
    const unsigned m = __ballot_sync(FULL, y < h_org && ws.rowfull[rb + y]), gt = m & ~((2u << lane) - 1u);
    if (y < h_org) ws.down[rb + y] = gt ? y0 + __ffs(gt) - 1 : carry;
    if (m) carry = y0 + __ffs(m) - 1;
  }
}

__device__ __forceinline__ float canon(float v) { return isnan(v) ? qnan() : v; }

// The column pass (a row without a value takes the smaller of the nearest rows above and below, the upper one where
// they are equal, or the one that exists), the final status (speckles, when the row pass did not run), depth and xyz.
__global__ void __launch_bounds__(256) disp_output_kernel(DispWork ws, DispOutputs out, int speckle, int S, int fill,
                                                          DispCamera cam, int w_org, int h_org) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X >= w_org || Y >= h_org) return;
  const size_t base = (size_t)blockIdx.z * h_org * w_org, o = base + (size_t)Y * w_org + X;
  unsigned char st = ws.status[o];
  if (speckle && !fill) st = speckle_status(st, ws.parent, ws.size, o, base, S);
  float D;
  if (fill) {
    const size_t r = (size_t)blockIdx.z * h_org + Y;
    if (ws.rowfull[r]) {
      D = ws.val[o];
    } else {
      const int a = ws.up[r], b = ws.down[r];
      const float va = a >= 0 ? ws.val[base + (size_t)a * w_org + X] : qnan();
      const float vb = b >= 0 ? ws.val[base + (size_t)b * w_org + X] : qnan();
      D = a < 0 ? vb : b < 0 ? va : std_min(va, vb);
    }
  } else {
    D = st == 0 ? ws.val[o] : qnan();
  }
  if (out.status) out.status[o] = st;
  if (out.disp) out.disp[o] = D;
  if (out.depth || out.xyz) {
    const float s = D + cam.doffs;
    const float Z = s > 0.0f ? canon(cam.fb / s) : qnan();
    if (out.depth) out.depth[o] = Z;
    if (out.xyz) {
      float* q = out.xyz + o * 3;
      q[0] = canon((((float)X - cam.cx) * Z) / cam.fx);
      q[1] = canon((((float)Y - cam.cy) * Z) / cam.fy);
      q[2] = Z;
    }
  }
}

}  // namespace

int launch_disparity(const LevelGeom& g, int fa, int fb, int n, const DispFilter& f, const DispCamera& cam,
                     const DispWork& ws, const DispOutputs& out, int w_org, int h_org, int crop_x, int crop_y,
                     cudaStream_t st) {
  const dim3 block(32, 8), grid((w_org + 31) / 32, (h_org + 7) / 8, n);
  const bool speckle = f.speckle_size > 0;
  int k = 0;
  disp_classify_kernel<<<grid, block, 0, st>>>(g, fa, fb, f.lr_check, f.alpha, f.beta, ws, w_org, h_org, crop_x, crop_y);
  ++k;
  if (speckle) {
    const int tx = (w_org + CCL_TILE - 1) / CCL_TILE, ty = (h_org + CCL_TILE - 1) / CCL_TILE;
    disp_ccl_tile_kernel<<<dim3(tx, ty, n), block, 0, st>>>(ws, f.speckle_diff, w_org, h_org);
    const long long nv = (long long)(tx - 1) * h_org, nh = (long long)(ty - 1) * w_org;
    const unsigned nbk = (unsigned)std::max((nv + nh + 255) / 256, 1LL);
    disp_ccl_border_kernel<<<dim3(nbk, n), 256, 0, st>>>(ws, f.speckle_diff, w_org, h_org, nv, nh);
    disp_ccl_count_kernel<<<grid, block, 0, st>>>(ws, w_org, h_org);
    k += 3;
  }
  if (f.fill) {
    disp_fill_rows_kernel<<<dim3((h_org + 7) / 8, n), 256, 0, st>>>(ws, speckle, f.speckle_size, w_org, h_org);
    disp_fill_links_kernel<<<n, 32, 0, st>>>(ws, h_org);
    k += 2;
  }
  disp_output_kernel<<<grid, block, 0, st>>>(ws, out, speckle, f.speckle_size, f.fill, cam, w_org, h_org);
  ++k;
  return cudaGetLastError() == cudaSuccess ? k : -1;
}

}  // namespace ofdis

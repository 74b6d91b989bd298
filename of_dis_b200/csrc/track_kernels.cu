// Dense point tracking through a clip's bidirectional flows (ofdis_track_begin / ofdis_track_advance; the header
// states the contract, preprocess.track_points restates it bit for bit).  The tracker of Sundaram, Brox and Keutzer
// (ECCV 2010): a track follows the forward flow with sub-pixel precision, ends where the forward-backward test fails
// or at a motion boundary, and new tracks start in empty, textured cells of a regular grid.  Per pair ofdis_capi.cu
// launches
//   track_advance_kernel  one thread per track slot: the new position, the end reason, the occupied cell;
//   track_seed_kernel     one thread per cell: occupancy, the structure tensor's smaller eigenvalue, the candidate;
//   track_count_kernel    flags per scan block;
//   track_scan_kernel     one CTA: the blocks' offsets, the admitted seeds, the new live count and counters;
//   track_scatter_kernel  survivors in list order, then the admitted seeds in cell order, into the other list and
//                         the frame's output records.
// Grids are sized by the capacity and the cell count; every kernel reads the live count from the device state, so a
// call enqueues all its pairs without a host round trip.  The compaction sums integers, so it is the same whatever
// the order of the atomics.  Float32 without contraction.
#include <climits>

#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr int TRACK_THREADS = 256;  // threads of every kernel but the scan; a scan block is 4 flags per thread
static_assert(TRACK_BLOCK == 4 * TRACK_THREADS, "a scan block is one 32-bit word of flags per thread");

template <int NOP>
__global__ void __launch_bounds__(TRACK_THREADS) track_advance_kernel(LevelGeom g, int fa, int fb, TrackGeom t,
                                                                      TrackWork ws, ofdis_track_point* list,
                                                                      int crop_x, int crop_y) {
  pdl_wait();  // programmatic dependent launch: nothing of the previous kernel is touched before this
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // the grid is exactly cap_pad threads
  const int w = t.w, h = t.h;
  int why = -1;  // -1 no track, 0 survives, 1 leaves, 2 inconsistent, 3 boundary
  if (i < ws.state->alive) {
    ofdis_track_point* p = list + i;
    const float x = p->x, y = p->y;
    const float* F = g.flow + (size_t)fa * g.flow_frame_stride;
    const float* B = g.flow + (size_t)fb * g.flow_frame_stride;
    float f[2] = {0.f, 0.f};
    flow_bilinear_at<NOP>(g, F, x, y, w, h, crop_x, crop_y, f);
    const float u = f[0], v = NOP == 2 ? f[1] : 0.f;
    const float xn = x + u, yn = y + v;
    if (!(xn >= 0.f && xn <= (float)(w - 1) && yn >= 0.f && yn <= (float)(h - 1))) {
      why = 1;
    } else {
      float b[2] = {0.f, 0.f};
      flow_bilinear_at<NOP>(g, B, xn, yn, w, h, crop_x, crop_y, b);
      const float du = u + b[0], dv = NOP == 2 ? v + b[1] : 0.f;
      const float e = du * du + dv * dv;
      const float mag = (u * u + v * v) + (b[0] * b[0] + b[1] * b[1]);
      if (!(e <= t.alpha * mag + t.beta)) {
        why = 2;
      } else {
        // motion boundary: central differences of F at the rounded source pixel, clamped neighbours
        const int xr = (int)floorf(x + 0.5f), yr = (int)floorf(y + 0.5f);
        float l[2], r[2], up[2], dn[2];
        upsample_at<NOP>(g, F, max(xr - 1, 0), yr, crop_x, crop_y, [&l](int c, float val) { l[c] = val; });
        upsample_at<NOP>(g, F, min(xr + 1, w - 1), yr, crop_x, crop_y, [&r](int c, float val) { r[c] = val; });
        upsample_at<NOP>(g, F, xr, max(yr - 1, 0), crop_x, crop_y, [&up](int c, float val) { up[c] = val; });
        upsample_at<NOP>(g, F, xr, min(yr + 1, h - 1), crop_x, crop_y, [&dn](int c, float val) { dn[c] = val; });
        const float ux = (r[0] - l[0]) * 0.5f, uy = (dn[0] - up[0]) * 0.5f;
        float g2 = ux * ux + uy * uy;
        if (NOP == 2) {
          const float vx = (r[1] - l[1]) * 0.5f, vy = (dn[1] - up[1]) * 0.5f;
          g2 = g2 + (vx * vx + vy * vy);
        }
        if (g2 > t.mb_alpha * (u * u + v * v) + t.mb_beta) {
          why = 3;
        } else {
          why = 0;
          p->x = xn;
          p->y = yn;
          ws.occ[((int)yn / t.s) * t.ncx + (int)xn / t.s] = 1;
        }
      }
    }
  }
  ws.flags[i] = why == 0 ? 1 : 0;
  // exact end counts: one 64-bit atomic per warp and reason
  const unsigned int lane = threadIdx.x & 31u;
#pragma unroll
  for (int r = 1; r <= 3; ++r) {
    const unsigned int m = __ballot_sync(0xffffffffu, why == r);
    if (m && lane == 0) atomicAdd(&ws.state->ended[r - 1], (unsigned long long)__popc(m));
  }
}

// candidate flag of cell c: not occupied after the advance, and the smaller eigenvalue of the structure tensor over
// the 5 x 5 window around the seed pixel at least min_eig.  Clears the cell's occupancy for the next pair.
template <int NOC>
__global__ void __launch_bounds__(TRACK_THREADS) track_seed_kernel(TrackGeom t, TrackWork ws, const unsigned char* I) {
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;  // the grid is exactly cells_pad threads
  bool cand = false;
  if (c < t.cells) {
    const bool occupied = ws.occ[c] != 0;
    ws.occ[c] = 0;
    if (!occupied) {
      const int w = t.w, h = t.h;
      const int cx = min((c % t.ncx) * t.s + t.s / 2, w - 1), cy = min((c / t.ncx) * t.s + t.s / 2, h - 1);
      float a = 0.f, b = 0.f, d2 = 0.f;
      for (int dy = -2; dy <= 2; ++dy) {
        const int py = clampi(cy + dy, h);
        for (int dx = -2; dx <= 2; ++dx) {
          const int px = clampi(cx + dx, w);
          const float ix = (gray_at<NOC>(I, w, min(px + 1, w - 1), py) - gray_at<NOC>(I, w, max(px - 1, 0), py)) * 0.5f;
          const float iy = (gray_at<NOC>(I, w, px, min(py + 1, h - 1)) - gray_at<NOC>(I, w, px, max(py - 1, 0))) * 0.5f;
          a += ix * ix;
          b += ix * iy;
          d2 += iy * iy;
        }
      }
      const float d = a - d2;
      const float lam = (a + d2) * 0.5f - sqrtf(d * d * 0.25f + b * b);
      cand = lam >= t.min_eig;
    }
  }
  ws.flags[t.cap_pad + c] = cand ? 1 : 0;
}

// flags of every scan block (each flag is 0 or 1, so a word's popcount is its count)
__global__ void __launch_bounds__(TRACK_THREADS) track_count_kernel(TrackWork ws) {
  pdl_wait();
  __shared__ unsigned int sw[TRACK_THREADS / 32];
  const unsigned int word = reinterpret_cast<const unsigned int*>(ws.flags)[blockIdx.x * TRACK_THREADS + threadIdx.x];
  unsigned int total;
  block_exclusive_scan<TRACK_THREADS>((unsigned int)__popc(word), sw, total);
  if (threadIdx.x == 0) ws.bsum[blockIdx.x] = total;
}

// One CTA: exclusive offsets of the keep blocks [0, nb_keep) and, separately, of the candidate blocks; then the
// admission (up to `capacity` live tracks, ids below INT_MAX) and the state update.
constexpr int TRACK_SCAN_THREADS = 1024;
__global__ void __launch_bounds__(TRACK_SCAN_THREADS) track_scan_kernel(TrackWork ws, int nb_keep, int nb_all,
                                                                         int capacity, int k) {
  pdl_wait();
  __shared__ unsigned int sw[TRACK_SCAN_THREADS / 32];
  unsigned int seg[2];
  for (int part = 0; part < 2; ++part) {
    const int lo = part ? nb_keep : 0, hi = part ? nb_all : nb_keep;
    unsigned int carry = 0;
    for (int base = lo; base < hi; base += TRACK_SCAN_THREADS) {
      const int i = base + threadIdx.x;
      const unsigned int v = i < hi ? ws.bsum[i] : 0u;
      unsigned int total;
      const unsigned int ex = block_exclusive_scan<TRACK_SCAN_THREADS>(v, sw, total);
      if (i < hi) ws.bsum[i] = carry + ex;
      carry += total;
    }
    seg[part] = carry;
  }
  if (threadIdx.x == 0) {
    TrackState* s = ws.state;
    const int S = (int)seg[0], C = (int)seg[1];
    const int adm = min(C, min(capacity - S, INT_MAX - s->next_id));
    s->survivors = S;
    s->admitted = adm;
    s->base_id = s->next_id;
    s->alive = S + adm;
    s->next_id += adm;
    s->seeded += (unsigned long long)adm;
    s->dropped += (unsigned long long)(C - adm);
    ws.counts[k] = S + adm;
  }
}

// Survivors of src in list order, then the admitted candidates in cell order, into dst and out.
__global__ void __launch_bounds__(TRACK_THREADS) track_scatter_kernel(TrackGeom t, TrackWork ws,
                                                                      const ofdis_track_point* src,
                                                                      ofdis_track_point* dst, ofdis_track_point* out) {
  pdl_wait();
  __shared__ unsigned int sw[TRACK_THREADS / 32];
  const int e0 = blockIdx.x * TRACK_BLOCK + threadIdx.x * 4;
  const unsigned int word = reinterpret_cast<const unsigned int*>(ws.flags)[e0 >> 2];
  unsigned int total;
  unsigned int off = ws.bsum[blockIdx.x] + block_exclusive_scan<TRACK_THREADS>((unsigned int)__popc(word), sw, total);
  if (!word) return;
  const TrackState* s = ws.state;
  for (int j = 0; j < 4; ++j) {
    if (!((word >> (8 * j)) & 0xffu)) continue;
    const int e = e0 + j;
    if (e < t.cap_pad) {
      const ofdis_track_point q = src[e];
      dst[off] = q;
      out[off] = q;
    } else if ((int)off < s->admitted) {
      const int c = e - t.cap_pad;
      ofdis_track_point q;
      q.id = s->base_id + (int)off;
      q.x = (float)min((c % t.ncx) * t.s + t.s / 2, t.w - 1);
      q.y = (float)min((c / t.ncx) * t.s + t.s / 2, t.h - 1);
      dst[s->survivors + off] = q;
      out[s->survivors + off] = q;
    }
    ++off;
  }
}

}  // namespace

int launch_track_advance(const LevelGeom& g, int fa, int fb, const TrackGeom& t, const TrackWork& ws, int cur,
                         int crop_x, int crop_y, cudaStream_t st) {
  const int blocks = t.cap_pad / TRACK_THREADS;
  if (g.nop == 2) track_advance_kernel<2><<<blocks, TRACK_THREADS, 0, st>>>(g, fa, fb, t, ws, ws.list[cur], crop_x, crop_y);
  else track_advance_kernel<1><<<blocks, TRACK_THREADS, 0, st>>>(g, fa, fb, t, ws, ws.list[cur], crop_x, crop_y);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_track_seed_compact(const TrackGeom& t, const TrackWork& ws, int noc, const unsigned char* I, int cur,
                              ofdis_track_point* out, int k, cudaStream_t st) {
  if (noc != 1 && noc != 3) return -1;
  const int nb_keep = t.cap_pad / TRACK_BLOCK, nb_all = nb_keep + t.cells_pad / TRACK_BLOCK;
  if (noc == 3) track_seed_kernel<3><<<t.cells_pad / TRACK_THREADS, TRACK_THREADS, 0, st>>>(t, ws, I);
  else track_seed_kernel<1><<<t.cells_pad / TRACK_THREADS, TRACK_THREADS, 0, st>>>(t, ws, I);
  track_count_kernel<<<nb_all, TRACK_THREADS, 0, st>>>(ws);
  track_scan_kernel<<<1, TRACK_SCAN_THREADS, 0, st>>>(ws, nb_keep, nb_all, t.capacity, k);
  track_scatter_kernel<<<nb_all, TRACK_THREADS, 0, st>>>(t, ws, ws.list[cur], ws.list[cur ^ 1], out);
  return cudaGetLastError() == cudaSuccess ? 4 : -1;
}

}  // namespace ofdis

// Fisher vectors of descriptors (ofdis_fisher_push / ofdis_fisher_take; the header states the contract,
// preprocess.FisherStream restates it bit for bit): PCA per block, posteriors of a diagonal GMM and the float64
// statistics of the improved Fisher vector (Perronnin, Sanchez and Mensink, ECCV 2010).  Per chunk of at most
// FISHER_CHUNK descriptors a push launches
//   fisher_project_kernel  a register-tiled SIMT GEMM: 64 descriptors x 64 outputs per CTA, 4 x 4 per thread, mean
//                          subtracted on load, each output summed in increasing i;
//   fisher_post_kernel     32 descriptors x all K Gaussians of one block per CTA: q_k over the d-tiles in order
//                          (mu and 1/sigma staged through shared memory), then the max, exp_f32, the sequential k-sum
//                          and gamma, the skip flags and the block's counts;
//   fisher_stats_kernel    one thread per (block, k, d): its S1 and S2 (and S0 for d = 0) in registers across the
//                          chunk, the descriptors in order, z recomputed with the posterior stage's expression;
// and a take launches fisher_norm_kernel, one CTA per block: the vector, power and L2 normalised in the fixed order.
// Float32 without contraction, IEEE division and square root; the statistics and the normalisation in float64.
#include <cfloat>

#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr int PJ_T = 64, PJ_I = 16;              // projection: tile of descriptors and outputs, i per stage
constexpr int PO_D = 32, PO_K = 64, PO_DT = 32;  // posteriors: descriptors per CTA, Gaussians and dims per tile
constexpr int ST_C = 16;                         // statistics: descriptors per shared-memory stage
constexpr int NORM_T = 256;                      // the take: threads, and the partial sums of the L2 norm

__device__ __forceinline__ const float* cb_mean(const FisherGeom& g, const float* cb, int b) { return cb + g.poff[b]; }
__device__ __forceinline__ const float* cb_proj(const FisherGeom& g, const float* cb, int b) {
  return cb + g.poff[b] + g.din[b];
}
__device__ __forceinline__ const float* cb_mu(const FisherGeom& g, const float* cb, int b) {
  return cb_proj(g, cb, b) + (size_t)g.dim[b] * g.din[b];
}
__device__ __forceinline__ const float* cb_isig(const FisherGeom& g, const float* cb, int b) {
  return cb_mu(g, cb, b) + (size_t)g.K * g.dim[b];
}
__device__ __forceinline__ const float* cb_c(const FisherGeom& g, const float* cb, int b) {
  return cb_isig(g, cb, b) + (size_t)g.K * g.dim[b];
}
__device__ __forceinline__ const float* cb_w(const FisherGeom& g, const float* cb, int b) { return cb_c(g, cb, b) + g.K; }

// y[c][yoff + d] = sum_i proj[d][i] * (x[c][off + i] - mean[i]), from +0.0f in increasing i.  Grid (descriptor
// tiles, output tiles, blocks), 16 x 16 threads; thread (tx, ty) owns rows ty + 16a and outputs tx + 16b.
__global__ void __launch_bounds__(256) fisher_project_kernel(FisherGeom g, const float* __restrict__ cb,
                                                             const float* __restrict__ x, int n, float* __restrict__ y) {
  const int b = blockIdx.z, din = g.din[b], dim = g.dim[b];
  const int r0 = blockIdx.x * PJ_T, d0 = blockIdx.y * PJ_T;
  if (d0 >= dim) return;
  __shared__ float xs[PJ_I][PJ_T];
  __shared__ float ps[PJ_I][PJ_T + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const float* mean = cb_mean(g, cb, b);
  const float* proj = cb_proj(g, cb, b);
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[a][c] = 0.0f;
  for (int i0 = 0; i0 < din; i0 += PJ_I) {
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = threadIdx.x + 256 * e, ii = idx & (PJ_I - 1), rr = idx >> 4, i = i0 + ii;
      const int r = r0 + rr, d = d0 + rr;
      // out-of-range i: both factors 0, so the product adds +0 (the sum never holds -0)
      xs[ii][rr] = (i < din && r < n) ? x[(size_t)r * g.desc_dim + g.off[b] + i] - mean[i] : 0.0f;
      ps[ii][rr] = (i < din && d < dim) ? proj[(size_t)d * din + i] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int ii = 0; ii < PJ_I; ++ii) {
      float xv[4], pv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) xv[a] = xs[ii][ty + 16 * a];
#pragma unroll
      for (int c = 0; c < 4; ++c) pv[c] = ps[ii][tx + 16 * c];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = acc[a][c] + pv[c] * xv[a];
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int r = r0 + ty + 16 * a;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int d = d0 + tx + 16 * c;
      if (r < n && d < dim) y[(size_t)r * g.ydim + g.yoff[b] + d] = acc[a][c];
    }
  }
}

// gamma of descriptors r0 .. r0+31 for block blockIdx.y.  Thread (tk = tid % 64, grp = tid / 64) computes q of
// Gaussian kt + tk for descriptors grp*8 .. grp*8+7; ll goes to shared memory, then warp w finishes descriptors
// 4w .. 4w+3.  Skipped: a y_d, a q_k or the max not finite.
__global__ void __launch_bounds__(256) fisher_post_kernel(FisherGeom g, const float* __restrict__ cb,
                                                          const float* __restrict__ y, int n,
                                                          float* __restrict__ gamma, unsigned char* __restrict__ skip,
                                                          unsigned long long* __restrict__ count) {
  extern __shared__ float ll[];  // [PO_D][K]
  __shared__ float mus[PO_DT][PO_K], iss[PO_DT][PO_K];
  __shared__ __align__(16) float ys[PO_DT][PO_D];
  __shared__ int bad[PO_D];
  __shared__ unsigned int cnt[2];
  const int b = blockIdx.y, K = g.K, dim = g.dim[b], r0 = blockIdx.x * PO_D;
  const int tk = threadIdx.x & (PO_K - 1), grp = threadIdx.x >> 6;
  const float* mu = cb_mu(g, cb, b);
  const float* isig = cb_isig(g, cb, b);
  const float* cc = cb_c(g, cb, b);
  if (threadIdx.x < PO_D) bad[threadIdx.x] = r0 + (int)threadIdx.x < n ? 0 : 1;
  if (threadIdx.x < 2) cnt[threadIdx.x] = 0u;
  for (int kt = 0; kt < K; kt += PO_K) {
    float q[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) q[j] = 0.0f;
    for (int dt = 0; dt < dim; dt += PO_DT) {
      __syncthreads();
      for (int idx = threadIdx.x; idx < PO_DT * PO_K; idx += 256) {
        const int dd = idx / PO_K, kk = idx % PO_K, k = kt + kk, d = dt + dd;
        const bool in = k < K && d < dim;
        mus[dd][kk] = in ? mu[(size_t)k * dim + d] : 0.0f;
        iss[dd][kk] = in ? isig[(size_t)k * dim + d] : 0.0f;
      }
      for (int idx = threadIdx.x; idx < PO_DT * PO_D; idx += 256) {
        const int rr = idx / PO_DT, dd = idx % PO_DT, r = r0 + rr, d = dt + dd;
        float v = 0.0f;
        if (r < n && d < dim) {
          v = y[(size_t)r * g.ydim + g.yoff[b] + d];
          if (!(fabsf(v) <= FLT_MAX)) bad[rr] = 1;
        }
        ys[dd][rr] = v;
      }
      __syncthreads();
      const int nd = min(PO_DT, dim - dt);
      for (int dd = 0; dd < nd; ++dd) {
        const float m = mus[dd][tk], s = iss[dd][tk];
        const float4 ya = *reinterpret_cast<const float4*>(&ys[dd][grp * 8]);
        const float4 yb = *reinterpret_cast<const float4*>(&ys[dd][grp * 8 + 4]);
        const float yv[8] = {ya.x, ya.y, ya.z, ya.w, yb.x, yb.y, yb.z, yb.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float z = (yv[j] - m) * s;
          q[j] = q[j] + z * z;
        }
      }
    }
    const int k = kt + tk;
    if (k < K) {
      const float ck = cc[k];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (!(q[j] <= FLT_MAX)) bad[grp * 8 + j] = 1;
        ll[(grp * 8 + j) * K + k] = ck - 0.5f * q[j];
      }
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = 0; j < 4; ++j) {
    const int rr = warp * 4 + j;
    float* l = ll + rr * K;
    float m = -INFINITY;
    for (int k = lane; k < K; k += 32) m = fmaxf(m, l[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const bool sk = bad[rr] || !(fabsf(m) <= FLT_MAX);
    if (!sk)
      for (int k = lane; k < K; k += 32) l[k] = exp_f32(l[k] - m);
    __syncwarp();
    float s = 0.0f;
    if (lane == 0 && !sk)
      for (int k = 0; k < K; ++k) s = s + l[k];
    s = __shfl_sync(0xffffffffu, s, 0);
    const int r = r0 + rr;
    if (r < n) {
      if (!sk)
        for (int k = lane; k < K; k += 32) gamma[((size_t)r * g.nblocks + b) * K + k] = l[k] / s;
      if (lane == 0) {
        skip[(size_t)r * g.nblocks + b] = sk ? 1 : 0;
        atomicAdd(&cnt[sk ? 1 : 0], 1u);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 && cnt[threadIdx.x])
    atomicAdd(&count[threadIdx.x * FISHER_MAX_BLOCKS + b], (unsigned long long)cnt[threadIdx.x]);
}

// Thread t of block blockIdx.y's K*dim accumulators: k = t / dim, d = t % dim; S0 with d = 0.  The chunk's
// descriptors in order, ST_C at a time through shared memory (gamma of the Gaussians this CTA covers, y of the block).
__global__ void __launch_bounds__(256) fisher_stats_kernel(FisherGeom g, const float* __restrict__ cb,
                                                           const float* __restrict__ y, const float* __restrict__ gamma,
                                                           const unsigned char* __restrict__ skip, int n,
                                                           double* __restrict__ stats) {
  extern __shared__ float sm[];  // gs[ST_C][nk], then ys[ST_C][dim]
  __shared__ unsigned char sk[ST_C];
  const int b = blockIdx.y, K = g.K, dim = g.dim[b], t0 = blockIdx.x * 256;
  if (t0 >= K * dim) return;
  const int t = t0 + threadIdx.x, kmin = t0 / dim, kmax = min(K - 1, (t0 + 255) / dim), nk = kmax - kmin + 1;
  const bool live = t < K * dim;
  const int k = live ? t / dim : kmin, d = live ? t % dim : 0;
  float* gs = sm;
  float* ys = sm + ST_C * nk;
  const float m = cb_mu(g, cb, b)[(size_t)k * dim + d], s = cb_isig(g, cb, b)[(size_t)k * dim + d];
  double* S0 = stats + g.soff[b];
  double* S1 = S0 + K;
  double* S2 = S1 + (size_t)K * dim;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  if (live) {
    s1 = S1[t];
    s2 = S2[t];
    if (d == 0) s0 = S0[k];
  }
  for (int c0 = 0; c0 < n; c0 += ST_C) {
    const int nc = min(ST_C, n - c0);
    __syncthreads();
    for (int idx = threadIdx.x; idx < nc * nk; idx += 256) {
      const int c = idx / nk, kk = idx % nk;
      gs[idx] = gamma[((size_t)(c0 + c) * g.nblocks + b) * K + kmin + kk];
    }
    for (int idx = threadIdx.x; idx < nc * dim; idx += 256) {
      const int c = idx / dim, dd = idx % dim;
      ys[idx] = y[(size_t)(c0 + c) * g.ydim + g.yoff[b] + dd];
    }
    if (threadIdx.x < nc) sk[threadIdx.x] = skip[(size_t)(c0 + threadIdx.x) * g.nblocks + b];
    __syncthreads();
    if (!live) continue;
    for (int c = 0; c < nc; ++c) {
      if (sk[c]) continue;
      const double gd = (double)gs[c * nk + k - kmin];
      const double zd = (double)((ys[c * dim + d] - m) * s);
      s1 = s1 + gd * zd;
      s2 = s2 + gd * (zd * zd);
      if (d == 0) s0 = s0 + gd;
    }
  }
  if (live) {
    S1[t] = s1;
    S2[t] = s2;
    if (d == 0) S0[k] = s0;
  }
}

// f_i of block b's vector (i < 2 K dim) before the L2 normalisation
__device__ __forceinline__ double fisher_entry(const FisherGeom& g, const float* w, const double* S0, int b, int i,
                                               double N) {
  const int K = g.K, dim = g.dim[b], kd = K * dim;
  const bool second = i >= kd;
  const int j = second ? i - kd : i, k = j / dim;
  const double* S1 = S0 + K;
  const double wk = (double)w[k];
  double t;
  if (!second) t = S1[j] / (N * sqrt(wk));
  else t = (S1[kd + j] - S0[k]) / (N * sqrt(2.0 * wk));
  const double r = sqrt(fabs(t));
  return t < 0.0 ? -r : r;
}

__global__ void __launch_bounds__(NORM_T) fisher_norm_kernel(FisherGeom g, const float* __restrict__ cb,
                                                             const double* __restrict__ stats,
                                                             const unsigned long long* __restrict__ count,
                                                             float* __restrict__ fv) {
  __shared__ double part[NORM_T];
  __shared__ double norm;
  const int b = blockIdx.x, len = 2 * g.K * g.dim[b];
  const unsigned long long nb = count[b];
  float* out = fv + g.foff[b];
  if (nb == 0) {
    for (int i = threadIdx.x; i < len; i += NORM_T) out[i] = 0.0f;
    return;
  }
  const double N = (double)nb;
  const float* w = cb_w(g, cb, b);
  const double* S0 = stats + g.soff[b];
  double p = 0.0;
  for (int i = threadIdx.x; i < len; i += NORM_T) {
    const double f = fisher_entry(g, w, S0, b, i, N);
    p = p + f * f;
  }
  part[threadIdx.x] = p;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int j = 0; j < NORM_T; ++j) s = s + part[j];
    norm = sqrt(s);
  }
  __syncthreads();
  const double nm = norm;
  for (int i = threadIdx.x; i < len; i += NORM_T) {
    const double f = fisher_entry(g, w, S0, b, i, N);
    out[i] = (float)(nm > 0.0 ? f / nm : f);
  }
}

}  // namespace

int launch_fisher_chunk(const FisherGeom& g, const FisherWork& w, const float* x, int n, cudaStream_t st) {
  if (n <= 0) return 0;
  int maxdim = 0, mindim = FISHER_MAX_DIM, maxkd = 0;
  for (int b = 0; b < g.nblocks; ++b) {
    maxdim = max(maxdim, g.dim[b]);
    mindim = min(mindim, g.dim[b]);
    maxkd = max(maxkd, g.K * g.dim[b]);
  }
  // the dynamic shared memory of the posteriors (ll) and the statistics (gamma of at most 255 / dim + 2 Gaussians per
  // CTA and y), above the 48 KB default with the static part
  const size_t post_smem = (size_t)PO_D * g.K * sizeof(float);
  const size_t stats_smem = (size_t)ST_C * (min(g.K, 255 / mindim + 2) + maxdim) * sizeof(float);
  if (cudaFuncSetAttribute(fisher_post_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)post_smem) !=
          cudaSuccess ||
      cudaFuncSetAttribute(fisher_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stats_smem) !=
          cudaSuccess)
    return -1;
  fisher_project_kernel<<<dim3((n + PJ_T - 1) / PJ_T, (maxdim + PJ_T - 1) / PJ_T, g.nblocks), 256, 0, st>>>(
      g, w.cb, x, n, w.y);
  fisher_post_kernel<<<dim3((n + PO_D - 1) / PO_D, g.nblocks), 256, post_smem, st>>>(g, w.cb, w.y, n, w.gamma, w.skip,
                                                                                    w.count);
  fisher_stats_kernel<<<dim3((maxkd + 255) / 256, g.nblocks), 256, stats_smem, st>>>(g, w.cb, w.y, w.gamma, w.skip, n,
                                                                                     w.stats);
  return cudaGetLastError() == cudaSuccess ? 3 : -1;
}

int launch_fisher_take(const FisherGeom& g, const FisherWork& w, float* fv, cudaStream_t st) {
  fisher_norm_kernel<<<g.nblocks, NORM_T, 0, st>>>(g, w.cb, w.stats, w.count, fv);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ofdis

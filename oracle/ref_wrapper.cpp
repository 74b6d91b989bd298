// oracle/_ref wrapper -- TEST INFRASTRUCTURE ONLY.
//
// Thin extern "C" entry points around the UNMODIFIED reference classes
// (compiled in place from the reference checkout by oracle/Makefile against
// oracle/eigen_shim).  Used by tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference leg only; the product never links this.
//
//   ofdis_ref_run            -> OFC::OFClass ctor            (oflow.cpp:32-363)
//   ofdis_ref_level_patches  -> PatGridClass one level       (patchgrid.cpp:98-397)
//   ofdis_ref_level_varref   -> VarRefClass one level        (refine_variational.cpp:25-116)
//   ofdis_ref_run_many       -> OFClass ctor over many pairs on a std::thread pool (frame-parallel CPU
//                               baseline without any Python in the timed region)
//   ofdis_ref_run_many_u8    -> the same from 8-bit frames to full-resolution flow: the callers either side
//                               of OFClass (run_dense.cpp:130-178,298-311,407-421) restated without OpenCV
//
// One shared object is built per (SELECTMODE, SELECTCHANNEL) pair because the
// reference selects flow/stereo and gray/RGB at compile time (CMakeLists.txt:25-46).
#include <iostream>
#include <string>
#include <vector>
#include <cmath>
#include <cstring>
#include <algorithm>
#include <sys/time.h>
#include <atomic>
#include <thread>

#include <Eigen/Core>

// test-harness access to per-patch state (p_iter, pweight, flags); the
// reference sources themselves are not touched.
#define private public
#include "patchgrid.h"
#include "refine_variational.h"
#undef private

using namespace OFC;

extern "C" {

struct ofdis_ref_params {
  int sc_f, sc_l, max_iter, min_iter;
  float dp_thresh, dr_thresh, res_thresh;
  int p_samp_s;
  float patove;
  int usefbcon, costfct, noc, patnorm, usetvref;
  float tv_alpha, tv_gamma, tv_delta;
  int tv_innerit, tv_solverit;
  float tv_sor;
  int verbosity;
};

int ofdis_ref_mode(void) { return SELECTMODE; }
int ofdis_ref_channels(void) { return SELECTCHANNEL; }

// Whole coarse-to-fine run == reference "O.Flow Run-Time" region.
void ofdis_ref_run(const float** i0, const float** i0x, const float** i0y,
                   const float** i1, const float** i1x, const float** i1y,
                   int imgpadding, float* outflow, const float* initflow,
                   int width, int height, const ofdis_ref_params* p) {
  OFClass ofc(i0, i0x, i0y, i1, i1x, i1y, imgpadding, outflow, initflow, width, height,
              p->sc_f, p->sc_l, p->max_iter, p->min_iter, p->dp_thresh, p->dr_thresh,
              p->res_thresh, p->p_samp_s, p->patove, p->usefbcon != 0, p->costfct, p->noc,
              p->patnorm, p->usetvref != 0, p->tv_alpha, p->tv_gamma, p->tv_delta,
              p->tv_innerit, p->tv_solverit, p->tv_sor, p->verbosity);
}

// optparam / camparam exactly as OFClass derives them (oflow.cpp:76-108, 138-157).
static void fill_params(optparam& op, camparam& cpl, camparam& cpr, int width_in, int height_in,
                        int sl, int imgpadding_in, const ofdis_ref_params* p) {
#if (SELECTMODE == 1)
  op.nop = 2;
#else
  op.nop = 1;
#endif
  op.p_samp_s = p->p_samp_s;
  op.outlierthresh = (float)op.p_samp_s / 2;
  op.patove = p->patove;
  op.sc_f = p->sc_f;
  op.sc_l = p->sc_l;
  op.max_iter = p->max_iter;
  op.min_iter = p->min_iter;
  op.dp_thresh = p->dp_thresh * p->dp_thresh;
  op.dr_thresh = p->dr_thresh;
  op.res_thresh = p->res_thresh;
  op.steps = std::max(1, (int)floor(op.p_samp_s * (1 - op.patove)));
  op.novals = p->noc * (p->p_samp_s) * (p->p_samp_s);
  op.usefbcon = p->usefbcon != 0;
  op.costfct = p->costfct;
  op.noc = p->noc;
  op.patnorm = p->patnorm;
  op.verbosity = p->verbosity;
  op.noscales = op.sc_f - op.sc_l + 1;
  op.usetvref = p->usetvref != 0;
  op.tv_alpha = p->tv_alpha;
  op.tv_gamma = p->tv_gamma;
  op.tv_delta = p->tv_delta;
  op.tv_innerit = p->tv_innerit;
  op.tv_solverit = p->tv_solverit;
  op.tv_sor = p->tv_sor;
  op.normoutlier_tmpbsq = (v4sf){op.normoutlier * op.normoutlier, op.normoutlier * op.normoutlier,
                                 op.normoutlier * op.normoutlier, op.normoutlier * op.normoutlier};
  op.normoutlier_tmp2bsq = __builtin_ia32_mulps(op.normoutlier_tmpbsq, op.twos);
  op.normoutlier_tmp4bsq = __builtin_ia32_mulps(op.normoutlier_tmpbsq, op.fours);

  float sc_fct = pow(2, -sl);
  cpl.sc_fct = sc_fct;
  cpl.height = height_in * sc_fct;
  cpl.width = width_in * sc_fct;
  cpl.imgpadding = imgpadding_in;
  cpl.tmp_lb = -(float)op.p_samp_s / 2;
  cpl.tmp_ubw = (float)(cpl.width + op.p_samp_s / 2 - 2);
  cpl.tmp_ubh = (float)(cpl.height + op.p_samp_s / 2 - 2);
  cpl.tmp_w = cpl.width + 2 * imgpadding_in;
  cpl.tmp_h = cpl.height + 2 * imgpadding_in;
  cpl.curr_lv = sl;
  cpl.camlr = 0;
  cpr = cpl;
  cpr.camlr = 1;
}

// One pyramid level of the patch stage: InitializeGrid, SetTargetImage,
// [InitializeFromCoarserOF], Optimize, AggregateFlowDense (oflow.cpp:191-267).
// Returns the number of patches; any output pointer may be null.
int ofdis_ref_level_patches(const float* i0, const float* i0x, const float* i0y, const float* i1,
                            const float* i1x, const float* i1y, int width_full, int height_full,
                            int level, int imgpadding, const ofdis_ref_params* p,
                            const float* flow_prev, float* p_out, float* pweight_out,
                            int* conv_out, int* cnt_out, float* dense_out) {
  optparam op;
  camparam cpl, cpr;
  fill_params(op, cpl, cpr, width_full, height_full, level, imgpadding, p);
  PatGridClass grid(&cpl, &cpr, &op);
  grid.InitializeGrid(i0, i0x, i0y);
  grid.SetTargetImage(i1, i1x, i1y);
  if (flow_prev) grid.InitializeFromCoarserOF(flow_prev);
  grid.Optimize();
  const int np = grid.GetNoPatches();
  for (int i = 0; i < np; ++i) {
    const patchstate* pc = grid.pat[i]->pc;
    if (p_out)
      for (int k = 0; k < op.nop; ++k) p_out[i * op.nop + k] = pc->p_iter[k];
    if (pweight_out) std::memcpy(pweight_out + (size_t)i * op.novals, pc->pweight.data(), sizeof(float) * op.novals);
    if (conv_out) conv_out[i] = pc->hasconverged ? 1 : 0;
    if (cnt_out) cnt_out[i] = pc->cnt;
  }
  if (dense_out) grid.AggregateFlowDense(dense_out);
  return np;
}

// One pyramid level of the variational refinement, in place on flow.
void ofdis_ref_level_varref(const float* i0, const float* i0x, const float* i0y, const float* i1,
                            const float* i1x, const float* i1y, int width_full, int height_full,
                            int level, int imgpadding, const ofdis_ref_params* p, float* flow) {
  optparam op;
  camparam cpl, cpr;
  fill_params(op, cpl, cpr, width_full, height_full, level, imgpadding, p);
  VarRefClass varref(i0, i0x, i0y, i1, i1x, i1y, &cpl, &cpr, &op, flow);
}

// Wall-clock helper for the CPU baseline: runs ofdis_ref_run `reps` times and
// returns the per-run times in ms (timer placement == oflow.cpp:113-114,355-360).
void ofdis_ref_time_run(const float** i0, const float** i0x, const float** i0y, const float** i1,
                        const float** i1x, const float** i1y, int imgpadding, float* outflow,
                        int width, int height, const ofdis_ref_params* p, int reps, double* ms_out) {
  for (int r = 0; r < reps; ++r) {
    struct timeval a, b;
    gettimeofday(&a, nullptr);
    ofdis_ref_run(i0, i0x, i0y, i1, i1x, i1y, imgpadding, outflow, nullptr, width, height, p);
    gettimeofday(&b, nullptr);
    ms_out[r] = (b.tv_sec - a.tv_sec) * 1000.0 + (b.tv_usec - a.tv_usec) / 1000.0;
  }
}

// ---------------------------------------------------------------------------------------------
// Frame-parallel drivers for the CPU baseline.  OFClass instances share no mutable state, so the
// only way the (single-threaded) reference uses a many-core host is one pair per thread.

// `npairs` pairs, pair q = pointer tables [6][nlevels] at ptrs[q*6 + {0:i0,1:i0x,2:i0y,3:i1,4:i1x,5:i1y}];
// `nrep` passes over all pairs on `threads` workers; returns wall seconds of the whole job.
double ofdis_ref_run_many(const float*** ptrs, int npairs, int nrep, int threads, int imgpadding, float* outflow,
                          size_t outflow_stride, int width, int height, const ofdis_ref_params* p) {
  std::atomic<long> next(0);
  const long total = (long)npairs * nrep;
  struct timeval a, b;
  gettimeofday(&a, nullptr);
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&]() {
      // OFClass refines its output array in place, so two passes over the same pair (nrep > 1) must not share it:
      // every run writes a per-thread scratch; the result is copied out afterwards (all passes produce the same bits)
      std::vector<float> scratch(outflow_stride);
      for (long i = next.fetch_add(1); i < total; i = next.fetch_add(1)) {
        const int q = (int)(i % npairs);
        const float*** pp = ptrs + (size_t)q * 6;
        ofdis_ref_run(pp[0], pp[1], pp[2], pp[3], pp[4], pp[5], imgpadding, scratch.data(), nullptr, width, height, p);
        if (i < npairs) std::memcpy(outflow + (size_t)q * outflow_stride, scratch.data(), sizeof(float) * outflow_stride);
      }
    });
  for (auto& th : pool) th.join();
  gettimeofday(&b, nullptr);
  return (b.tv_sec - a.tv_sec) + (b.tv_usec - a.tv_usec) * 1e-6;
}

namespace {
// Callers either side of OFClass in run_dense.cpp, restated without OpenCV (the image holds no
// OpenCV SDK).  For 8-bit input these reproduce cv::resize(0.5, INTER_AREA-equivalent 2x2 mean of the
// reference's INTER_LINEAR at exact half size), cv::Sobel(3x3)/8 with BORDER_REFLECT_101, copyMakeBorder
// and the final cv::resize(INTER_LINEAR) exactly (tests/test_preprocess.py pins the same arithmetic
// of of_dis_b200/preprocess.py to cv2).
struct Img {
  int w = 0, h = 0, c = 1;
  std::vector<float> px;
  float& at(int x, int y, int k) { return px[((size_t)y * w + x) * c + k]; }
  float at(int x, int y, int k) const { return px[((size_t)y * w + x) * c + k]; }
};
inline int clampi(int v, int n) { return v < 0 ? 0 : (v > n - 1 ? n - 1 : v); }
inline int refl(int v, int n) {
  if (n == 1) return 0;
  while (v < 0 || v >= n) v = v < 0 ? -v : 2 * (n - 1) - v;
  return v;
}
// all outputs are resized in place: a worker thread reuses its buffers from pair to pair
void border(const Img& s, int pad, bool replicate, Img& d) {  // copyMakeBorder (run_dense.cpp:163-172)
  d.w = s.w + 2 * pad; d.h = s.h + 2 * pad; d.c = s.c;
  d.px.assign((size_t)d.w * d.h * d.c, 0.f);
  const int rowf = s.w * s.c;
  for (int y = 0; y < d.h; ++y) {
    const int sy = y - pad;
    if (!replicate && (sy < 0 || sy >= s.h)) continue;
    const float* src = &s.px[(size_t)clampi(sy, s.h) * rowf];
    float* dst = &d.px[(size_t)y * d.w * d.c];
    std::memcpy(dst + (size_t)pad * s.c, src, sizeof(float) * rowf);
    if (replicate)
      for (int x = 0; x < pad; ++x)
        for (int k = 0; k < s.c; ++k) {
          dst[x * s.c + k] = src[k];
          dst[(size_t)(pad + s.w + x) * s.c + k] = src[(size_t)(s.w - 1) * s.c + k];
        }
  }
}
void half(const Img& s, Img& d) {  // cv::resize(.5,.5) on even sizes (run_dense.cpp:150)
  d.w = s.w / 2; d.h = s.h / 2; d.c = s.c;
  d.px.resize((size_t)d.w * d.h * d.c);
  for (int y = 0; y < d.h; ++y)
    for (int x = 0; x < d.w; ++x)
      for (int k = 0; k < s.c; ++k)
        d.at(x, y, k) = ((s.at(2 * x, 2 * y, k) + s.at(2 * x + 1, 2 * y, k)) + (s.at(2 * x, 2 * y + 1, k) + s.at(2 * x + 1, 2 * y + 1, k))) * 0.25f;
}
void sobel(const Img& s, Img& dx, Img& dy) {  // cv::Sobel 3x3, scale 1/8 (run_dense.cpp:156-157)
  dx.w = dy.w = s.w; dx.h = dy.h = s.h; dx.c = dy.c = s.c;
  dx.px.resize(s.px.size());
  dy.px.resize(s.px.size());
  const int c = s.c;
  for (int y = 0; y < s.h; ++y) {
    const float* rm = &s.px[(size_t)refl(y - 1, s.h) * s.w * c];
    const float* r0 = &s.px[(size_t)y * s.w * c];
    const float* rp = &s.px[(size_t)refl(y + 1, s.h) * s.w * c];
    float* ox = &dx.px[(size_t)y * s.w * c];
    float* oy = &dy.px[(size_t)y * s.w * c];
    for (int x = 0; x < s.w; ++x) {
      const int xm = refl(x - 1, s.w) * c, xp = refl(x + 1, s.w) * c, x0 = x * c;
      for (int k = 0; k < c; ++k) {
        const float t0 = rm[xp + k] - rm[xm + k], t1 = r0[xp + k] - r0[xm + k], t2 = rp[xp + k] - rp[xm + k];
        ox[x0 + k] = (t0 * 0.125f + t1 * 0.25f) + t2 * 0.125f;
        const float s0 = (rm[xm + k] * 0.125f + rm[x0 + k] * 0.25f) + rm[xp + k] * 0.125f;
        const float s2 = (rp[xm + k] * 0.125f + rp[x0 + k] * 0.25f) + rp[xp + k] * 0.125f;
        oy[x0 + k] = s2 - s0;
      }
    }
  }
}
struct Pyr {
  std::vector<Img> raw, rdx, rdy, im, dx, dy;
  std::vector<const float*> pim, pdx, pdy;
  void build(const unsigned char* u8, int w_org, int h_org, int c, int W, int H, int lv_f, int pad) {
    const size_t n = lv_f + 1;
    if (raw.size() != n) {
      raw.resize(n); rdx.resize(n); rdy.resize(n); im.resize(n); dx.resize(n); dy.resize(n);
      pim.resize(n); pdx.resize(n); pdy.resize(n);
    }
    // divisibility padding: replicate, floor(pad/2) left/top (run_dense.cpp:298-311), then float
    Img& base = raw[0];
    base.w = W; base.h = H; base.c = c;
    base.px.resize((size_t)W * H * c);
    const int pl = (W - w_org) / 2, pt = (H - h_org) / 2;
    for (int y = 0; y < H; ++y) {
      const unsigned char* src = u8 + (size_t)clampi(y - pt, h_org) * w_org * c;
      float* dst = &base.px[(size_t)y * W * c];
      for (int x = 0; x < W; ++x) {
        const int sx = clampi(x - pl, w_org) * c;
        for (int k = 0; k < c; ++k) dst[x * c + k] = (float)src[sx + k];
      }
    }
    for (size_t i = 0; i < n; ++i) {
      if (i > 0) half(raw[i - 1], raw[i]);
      sobel(raw[i], rdx[i], rdy[i]);
    }
    for (size_t i = 0; i < n; ++i) {
      border(raw[i], pad, true, im[i]);
      border(rdx[i], pad, false, dx[i]);
      border(rdy[i], pad, false, dy[i]);
      pim[i] = im[i].px.data(); pdx[i] = dx[i].px.data(); pdy[i] = dy[i].px.data();
    }
  }
};
// flow of level sc_l -> x 2^sc_l, cv::resize(INTER_LINEAR) by 2^sc_l, crop (run_dense.cpp:407-414)
void upsample_crop(const float* fl, int w, int h, int nop, int sc, int w_org, int h_org, int W, int H, float* out) {
  const float scale = (float)sc;
  const int cx = (W - w_org) / 2, cy = (H - h_org) / 2;
  std::vector<int> x0(W), x1(W), y0(H), y1(H);
  std::vector<float> fx(W), fy(H);
  auto taps = [&](int ns, int nd, std::vector<int>& a, std::vector<int>& b, std::vector<float>& f) {
    for (int x = 0; x < nd; ++x) {
      const float t = ((float)x + 0.5f) / scale - 0.5f;
      const int i = (int)floorf(t);
      f[x] = i < 0 ? 0.f : t - (float)i;
      a[x] = clampi(i, ns);
      b[x] = clampi(i + 1, ns);
    }
  };
  taps(w, W, x0, x1, fx);
  taps(h, H, y0, y1, fy);
  for (int y = 0; y < h_org; ++y)
    for (int x = 0; x < w_org; ++x) {
      const int X = x + cx, Y = y + cy;
      for (int k = 0; k < nop; ++k) {
        auto S = [&](int xx, int yy) { return fl[((size_t)yy * w + xx) * nop + k] * scale; };
        const float r0 = S(x0[X], y0[Y]) * (1.0f - fx[X]) + S(x1[X], y0[Y]) * fx[X];
        const float r1 = S(x0[X], y1[Y]) * (1.0f - fx[X]) + S(x1[X], y1[Y]) * fx[X];
        out[((size_t)y * w_org + x) * nop + k] = r0 * (1.0f - fy[Y]) + r1 * fy[Y];
      }
    }
}
}  // namespace

// 8-bit frames [pair][2][h_org][w_org][noc] in, full-resolution flow [pair][h_org][w_org][nop] out: what
// one run_OF_INT invocation computes between imread and SaveFlowFile.  Returns wall seconds.
double ofdis_ref_run_many_u8(const unsigned char* frames, int npairs, int nrep, int threads, int w_org, int h_org,
                             float* out, const ofdis_ref_params* p) {
  const int nop = (SELECTMODE == 1) ? 2 : 1, c = p->noc, scf = 1 << p->sc_f;
  const int W = (w_org + scf - 1) / scf * scf, H = (h_org + scf - 1) / scf * scf;
  const size_t img = (size_t)w_org * h_org * c;
  std::atomic<long> next(0);
  const long total = (long)npairs * nrep;
  struct timeval a, b;
  gettimeofday(&a, nullptr);
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&]() {
      Pyr A, B;  // per-thread buffers, reused from pair to pair
      std::vector<float> fl;
      for (long i = next.fetch_add(1); i < total; i = next.fetch_add(1)) {
        const int q = (int)(i % npairs);
        A.build(frames + (size_t)q * 2 * img, w_org, h_org, c, W, H, p->sc_f, p->p_samp_s);
        B.build(frames + (size_t)q * 2 * img + img, w_org, h_org, c, W, H, p->sc_f, p->p_samp_s);
        const int w = W >> p->sc_l, h = H >> p->sc_l;
        fl.resize((size_t)w * h * nop);
        ofdis_ref_run(A.pim.data(), A.pdx.data(), A.pdy.data(), B.pim.data(), B.pdx.data(), B.pdy.data(), p->p_samp_s,
                      fl.data(), nullptr, W, H, p);
        upsample_crop(fl.data(), w, h, nop, 1 << p->sc_l, w_org, h_org, W, H, out + (size_t)q * w_org * h_org * nop);
      }
    });
  for (auto& th : pool) th.join();
  gettimeofday(&b, nullptr);
  return (b.tv_sec - a.tv_sec) + (b.tv_usec - a.tv_usec) * 1e-6;
}

}  // extern "C"

// Host-side C++ classes over the C-ABI; see ofdis_host.h.
#include "ofdis_host.h"

#include <sys/time.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

namespace OFC {

namespace {

void check(int rc, ofdis_ctx* ctx, const char* what) {
  if (rc != OFDIS_OK) {
    std::string msg = std::string(what) + ": status " + std::to_string(rc);
    if (ctx) msg += std::string(" (") + ofdis_last_error(ctx) + ")";
    throw std::runtime_error(msg);
  }
}

ofdis_params to_params(const optparam& op, int sc_f, int sc_l) {
  ofdis_params p;
  std::memset(&p, 0, sizeof(p));
  p.sc_f = sc_f;
  p.sc_l = sc_l;
  p.max_iter = op.max_iter;
  p.min_iter = op.min_iter;
  p.dp_thresh = std::sqrt(op.dp_thresh);  // exact squared value is installed with ofdis_set_dp_thresh_sq
  p.dr_thresh = op.dr_thresh;
  p.res_thresh = op.res_thresh;
  p.p_samp_s = op.p_samp_s;
  p.patove = op.patove;
  p.usefbcon = op.usefbcon ? 1 : 0;
  p.costfct = op.costfct;
  p.noc = op.noc;
  p.patnorm = op.patnorm;
  p.usetvref = 1;
  p.tv_alpha = op.tv_alpha;
  p.tv_gamma = op.tv_gamma;
  p.tv_delta = op.tv_delta;
  p.tv_innerit = op.tv_innerit;
  p.tv_solverit = op.tv_solverit;
  p.tv_sor = op.tv_sor;
  p.verbosity = op.verbosity;
  return p;
}

// one-level context for the per-level classes
ofdis_ctx* level_context(const camparam* cpt, const optparam* op, int device) {
  ofdis_params p = to_params(*op, cpt->curr_lv, cpt->curr_lv);
  p.usefbcon = 0;
  ofdis_ctx* ctx = nullptr;
  check(ofdis_create(&ctx, device, nullptr, &p, op->nop, cpt->width << cpt->curr_lv, cpt->height << cpt->curr_lv,
                     cpt->imgpadding, 1),
        nullptr, "ofdis_create");
  ofdis_set_dp_thresh_sq(ctx, op->dp_thresh);
  ofdis_set_camlr(ctx, cpt->camlr);
  return ctx;
}

double ms_between(const timeval& a, const timeval& b) {
  return (b.tv_sec - a.tv_sec) * 1000.0 + (b.tv_usec - a.tv_usec) / 1000.0;
}

}  // namespace

void FillOptParam(optparam& op, int nop, int sc_f, int sc_l, int max_iter, int min_iter, float dp_thresh,
                  float dr_thresh, float res_thresh, int p_samp_s, float patove, bool usefbcon, int costfct,
                  int noc, int patnorm, bool usetvref, float tv_alpha, float tv_gamma, float tv_delta,
                  int tv_innerit, int tv_solverit, float tv_sor, int verbosity) {
  op.nop = nop;
  op.p_samp_s = p_samp_s;
  op.outlierthresh = (float)op.p_samp_s / 2;
  op.patove = patove;
  op.sc_f = sc_f;
  op.sc_l = sc_l;
  op.max_iter = max_iter;
  op.min_iter = min_iter;
  op.dp_thresh = dp_thresh * dp_thresh;
  op.dr_thresh = dr_thresh;
  op.res_thresh = res_thresh;
  op.steps = std::max(1, (int)floor(op.p_samp_s * (1 - op.patove)));
  op.novals = noc * p_samp_s * p_samp_s;
  op.usefbcon = usefbcon;
  op.costfct = costfct;
  op.noc = noc;
  op.patnorm = patnorm;
  op.verbosity = verbosity;
  op.noscales = op.sc_f - op.sc_l + 1;
  op.usetvref = usetvref;
  op.tv_alpha = tv_alpha;
  op.tv_gamma = tv_gamma;
  op.tv_delta = tv_delta;
  op.tv_innerit = tv_innerit;
  op.tv_solverit = tv_solverit;
  op.tv_sor = tv_sor;
}

void FillCamParam(camparam& cp, const optparam& op, int width_full, int height_full, int level, int imgpadding,
                  int camlr) {
  const float sc_fct = (float)pow(2, -level);
  cp.sc_fct = sc_fct;
  cp.height = (int)(height_full * sc_fct);
  cp.width = (int)(width_full * sc_fct);
  cp.imgpadding = imgpadding;
  cp.tmp_lb = -(float)op.p_samp_s / 2;
  cp.tmp_ubw = (float)(cp.width + op.p_samp_s / 2 - 2);
  cp.tmp_ubh = (float)(cp.height + op.p_samp_s / 2 - 2);
  cp.tmp_w = cp.width + 2 * imgpadding;
  cp.tmp_h = cp.height + 2 * imgpadding;
  cp.curr_lv = level;
  cp.camlr = camlr;
}

// ---------------------------------------------------------------------------
namespace {

// What the level loop starts from and where its result goes: the reference's float pyramids and
// level-sc_l flow (oflow.h:84-111), or -- extension -- 8-bit frames in and full-resolution flow out
// with pyramid, gradients, paddings, upsampling and crop on the device (run_dense.cpp:130-178,
// 298-311,407-414).
struct RunIO {
  const float **im_ao = nullptr, **im_ao_dx = nullptr, **im_ao_dy = nullptr, **im_bo = nullptr, **im_bo_dx = nullptr,
              **im_bo_dy = nullptr;
  const unsigned char* frames = nullptr;  // [2][height_org][width_org][noc]
  int width_org = 0, height_org = 0;
  float* outflow = nullptr;
  const float* initflow = nullptr;           // level sc_f+1 (oflow.h:91)
  const float* initflow_fullres = nullptr;   // [height_org][width_org][nop], with `frames` only
};

void run_ofclass(const RunIO& io, const ofdis_params& p, int nop, int width, int height, int imgpadding, int device) {
  timeval t0, t1;
  const int verbosity = p.verbosity, sc_f = p.sc_f, sc_l = p.sc_l;
  if (verbosity > 0) gettimeofday(&t0, nullptr);
  ofdis_ctx* ctx = nullptr;
  check(ofdis_create(&ctx, device, nullptr, &p, nop, width, height, imgpadding, 1), nullptr, "ofdis_create");
  try {
    if (verbosity > 1) {
      gettimeofday(&t1, nullptr);
      printf("TIME (Grid Memo. Alloc. ) (ms): %3g\n", ms_between(t0, t1));
    }
    if (io.frames)
      check(ofdis_upload_frames_u8(ctx, 0, 1, io.frames, io.width_org, io.height_org, OFDIS_MEM_HOST), ctx,
            "ofdis_upload_frames_u8");
    else
      for (int sl = sc_l; sl <= sc_f; ++sl)
        check(ofdis_upload_level_fb(ctx, 0, sl, io.im_ao[sl], io.im_ao_dx[sl], io.im_ao_dy[sl], io.im_bo[sl],
                                    io.im_bo_dx ? io.im_bo_dx[sl] : nullptr, io.im_bo_dy ? io.im_bo_dy[sl] : nullptr,
                                    OFDIS_MEM_HOST),
              ctx, "ofdis_upload_level_fb");
    if (io.initflow) check(ofdis_set_flow(ctx, 0, sc_f + 1, io.initflow, OFDIS_MEM_HOST), ctx, "ofdis_set_flow");
    if (io.initflow_fullres)
      check(ofdis_set_initflow_fullres(ctx, 0, 1, io.initflow_fullres, io.width_org, io.height_org, OFDIS_MEM_HOST),
            ctx, "ofdis_set_initflow_fullres");
    const bool use_initflow = io.initflow || io.initflow_fullres;
    if (verbosity > 1) {
      // per-level timing like oflow.cpp:303 (stages are timed with a stream sync each)
      for (int sl = sc_f; sl >= sc_l; --sl) {
        timeval a, b, c, d;
        int w, h, nopw, noph, steps;
        ofdis_level_info(ctx, sl, &w, &h, &nopw, &noph, &steps);
        ofdis_sync(ctx);
        gettimeofday(&a, nullptr);
        check(ofdis_patgrid_optimize(ctx, sl, 0, 1, (sl < sc_f) || use_initflow), ctx, "patgrid_optimize");
        ofdis_sync(ctx);
        gettimeofday(&b, nullptr);
        check(ofdis_patgrid_aggregate(ctx, sl, 0, 1), ctx, "patgrid_aggregate");
        ofdis_sync(ctx);
        gettimeofday(&c, nullptr);
        if (p.usetvref) check(ofdis_varref_refine(ctx, sl, 0, 1), ctx, "varref_refine");
        ofdis_sync(ctx);
        gettimeofday(&d, nullptr);
        printf("TIME (Sc: %i, #p:%6i, pconst, pinit, poptim, cflow, tvopt, total): %8.2f %8.2f %8.2f %8.2f %8.2f -> %8.2f ms.\n",
               sl, nopw * noph, 0.0, 0.0, ms_between(a, b), ms_between(b, c), ms_between(c, d), ms_between(a, d));
      }
    } else {
      check(ofdis_run(ctx, 1, use_initflow ? 1 : 0), ctx, "ofdis_run");
    }
    if (io.frames) {
      check(ofdis_get_flow_fullres(ctx, 0, 1, io.outflow, io.width_org, io.height_org, OFDIS_MEM_HOST), ctx,
            "ofdis_get_flow_fullres");
      check(ofdis_sync(ctx), ctx, "ofdis_sync");
    } else {
      check(ofdis_get_flow(ctx, 0, sc_l, io.outflow, OFDIS_MEM_HOST), ctx, "ofdis_get_flow");
    }
  } catch (...) {
    ofdis_destroy(ctx);
    throw;
  }
  ofdis_destroy(ctx);
  if (verbosity > 0) {
    gettimeofday(&t1, nullptr);
    printf("TIME (O.Flow Run-Time   ) (ms): %3g\n", ms_between(t0, t1));
  }
}

ofdis_params make_params(int sc_f, int sc_l, int max_iter, int min_iter, float dp_thresh, float dr_thresh,
                         float res_thresh, int p_samp_s, float patove, bool usefbcon, int costfct, int noc, int patnorm,
                         bool usetvref, float tv_alpha, float tv_gamma, float tv_delta, int tv_innerit, int tv_solverit,
                         float tv_sor, int verbosity) {
  ofdis_params p;
  std::memset(&p, 0, sizeof(p));
  p.sc_f = sc_f;
  p.sc_l = sc_l;
  p.max_iter = max_iter;
  p.min_iter = min_iter;
  p.dp_thresh = dp_thresh;
  p.dr_thresh = dr_thresh;
  p.res_thresh = res_thresh;
  p.p_samp_s = p_samp_s;
  p.patove = patove;
  p.usefbcon = usefbcon ? 1 : 0;
  p.costfct = costfct;
  p.noc = noc;
  p.patnorm = patnorm;
  p.usetvref = usetvref ? 1 : 0;
  p.tv_alpha = tv_alpha;
  p.tv_gamma = tv_gamma;
  p.tv_delta = tv_delta;
  p.tv_innerit = tv_innerit;
  p.tv_solverit = tv_solverit;
  p.tv_sor = tv_sor;
  p.verbosity = verbosity;
  return p;
}

}  // namespace

OFClass::OFClass(const float** im_ao_in, const float** im_ao_dx_in, const float** im_ao_dy_in,
                 const float** im_bo_in, const float** im_bo_dx_in, const float** im_bo_dy_in,
                 const int imgpadding_in, float* outflow, const float* initflow, const int width_in,
                 const int height_in, const int sc_f_in, const int sc_l_in, const int max_iter_in,
                 const int min_iter_in, const float dp_thresh_in, const float dr_thresh_in,
                 const float res_thresh_in, const int padval_in, const float patove_in, const bool usefbcon_in,
                 const int costfct_in, const int noc_in, const int patnorm_in, const bool usetvref_in,
                 const float tv_alpha_in, const float tv_gamma_in, const float tv_delta_in,
                 const int tv_innerit_in, const int tv_solverit_in, const float tv_sor_in,
                 const int verbosity_in, const int nop_in, const int device) {
  RunIO io;
  io.im_ao = im_ao_in;
  io.im_ao_dx = im_ao_dx_in;
  io.im_ao_dy = im_ao_dy_in;
  io.im_bo = im_bo_in;
  io.im_bo_dx = im_bo_dx_in;  // only the forward-backward grid reads them (oflow.cpp:193-197)
  io.im_bo_dy = im_bo_dy_in;
  io.outflow = outflow;
  io.initflow = initflow;
  run_ofclass(io,
              make_params(sc_f_in, sc_l_in, max_iter_in, min_iter_in, dp_thresh_in, dr_thresh_in, res_thresh_in,
                          padval_in, patove_in, usefbcon_in, costfct_in, noc_in, patnorm_in, usetvref_in, tv_alpha_in,
                          tv_gamma_in, tv_delta_in, tv_innerit_in, tv_solverit_in, tv_sor_in, verbosity_in),
              nop_in, width_in, height_in, imgpadding_in, device);
}

OFClass::OFClass(const unsigned char* frame_ao, const unsigned char* frame_bo, const int width_org,
                 const int height_org, float* outflow_fullres, const float* initflow, const int sc_f_in,
                 const int sc_l_in, const int max_iter_in, const int min_iter_in, const float dp_thresh_in,
                 const float dr_thresh_in, const float res_thresh_in, const int padval_in, const float patove_in,
                 const bool usefbcon_in, const int costfct_in, const int noc_in, const int patnorm_in,
                 const bool usetvref_in, const float tv_alpha_in, const float tv_gamma_in, const float tv_delta_in,
                 const int tv_innerit_in, const int tv_solverit_in, const float tv_sor_in, const int verbosity_in,
                 const int nop_in, const int device, const float* initflow_fullres) {
  const size_t n = (size_t)width_org * height_org * noc_in;
  std::vector<unsigned char> frames(2 * n);
  std::memcpy(frames.data(), frame_ao, n);
  std::memcpy(frames.data() + n, frame_bo, n);
  const int scf = 1 << (initflow_fullres ? sc_f_in + 1 : sc_f_in);  // run_dense.cpp:298-311
  RunIO io;
  io.frames = frames.data();
  io.width_org = width_org;
  io.height_org = height_org;
  io.outflow = outflow_fullres;
  io.initflow = initflow;
  io.initflow_fullres = initflow_fullres;
  run_ofclass(io,
              make_params(sc_f_in, sc_l_in, max_iter_in, min_iter_in, dp_thresh_in, dr_thresh_in, res_thresh_in,
                          padval_in, patove_in, usefbcon_in, costfct_in, noc_in, patnorm_in, usetvref_in, tv_alpha_in,
                          tv_gamma_in, tv_delta_in, tv_innerit_in, tv_solverit_in, tv_sor_in, verbosity_in),
              nop_in, (width_org + scf - 1) / scf * scf, (height_org + scf - 1) / scf * scf, padval_in, device);
}

// ---------------------------------------------------------------------------
PatGridClass::PatGridClass(const camparam* cpt_in, const camparam* cpo_in, const optparam* op_in, int device)
    : cpt(cpt_in), op(op_in) {
  (void)cpo_in;
  // patchgrid.cpp:42-48
  steps = op->steps;
  nopw = (int)ceil((float)cpt->width / (float)steps);
  noph = (int)ceil((float)cpt->height / (float)steps);
  offw = (cpt->width - (nopw - 1) * steps) / 2;
  offh = (cpt->height - (noph - 1) * steps) / 2;
  nopatches = nopw * noph;
  device_id = device;
  ctx = level_context(cpt, op, device);
}

PatGridClass::Couple::~Couple() { ofdis_destroy(ctx); }

PatGridClass::~PatGridClass() {
  if (couple) {
    couple->grid[role] = nullptr;
    ctx = nullptr;  // owned by the couple
  }
  ofdis_destroy(ctx);
}

void PatGridClass::SetComplGrid(PatGridClass* cg) {
  if (!cg || cg == this) throw std::runtime_error("PatGridClass::SetComplGrid: need the other grid");
  if (couple) {
    if (couple->grid[role ^ 1] == cg) return;  // second half of oflow.cpp:169-170
    throw std::runtime_error("PatGridClass::SetComplGrid: this grid already has a complementary grid");
  }
  if (cg->couple) throw std::runtime_error("PatGridClass::SetComplGrid: the other grid already has a complementary grid");
  // one engine context with both directions: this grid becomes the forward one
  auto c = std::make_shared<Couple>();
  ofdis_params p = to_params(*op, cpt->curr_lv, cpt->curr_lv);
  p.usefbcon = 1;
  check(ofdis_create(&c->ctx, device_id, nullptr, &p, op->nop, cpt->width << cpt->curr_lv, cpt->height << cpt->curr_lv,
                     cpt->imgpadding, 1),
        nullptr, "ofdis_create (forward-backward couple)");
  ofdis_set_dp_thresh_sq(c->ctx, op->dp_thresh);
  c->grid[0] = this;
  c->grid[1] = cg;
  for (PatGridClass* g : {this, cg}) {
    ofdis_destroy(g->ctx);  // the stand-alone one-direction context
    g->ctx = c->ctx;
    g->couple = c;
    g->fetched = false;
  }
  role = 0;
  cg->role = 1;
}

void PatGridClass::select() const {
  if (couple) check(ofdis_set_direction(ctx, role), ctx, "ofdis_set_direction");
}

void PatGridClass::flush() {
  if (!couple || couple->uploaded) return;
  PatGridClass *f = couple->grid[0], *b = couple->grid[1];
  if (!f || !b || !f->i0 || !b->i0 || !f->tgt || !b->tgt)
    throw std::runtime_error("PatGridClass: both grids of a couple need InitializeGrid and SetTargetImage first");
  // forward: template = its own image, target = the other grid's template (oflow.cpp:191-197)
  check(ofdis_upload_level_fb(ctx, 0, cpt->curr_lv, f->i0, f->i0x, f->i0y, b->i0, b->i0x, b->i0y, OFDIS_MEM_HOST), ctx,
        "ofdis_upload_level_fb");
  couple->uploaded = true;
}

void PatGridClass::InitializeGrid(const float* a, const float* ax, const float* ay) {
  i0 = a;
  i0x = ax;
  i0y = ay;
  from_coarser = false;  // p_init reset (patchgrid.cpp:113)
  fetched = false;
  if (couple) couple->uploaded = false;
}

void PatGridClass::SetTargetImage(const float* b, const float*, const float*) {
  if (!i0) throw std::runtime_error("PatGridClass::SetTargetImage before InitializeGrid");
  tgt = b;
  if (couple) {
    couple->uploaded = false;
  } else {
    check(ofdis_upload_level(ctx, 0, cpt->curr_lv, i0, i0x, i0y, b, OFDIS_MEM_HOST), ctx, "ofdis_upload_level");
  }
  fetched = false;
}

void PatGridClass::InitializeFromCoarserOF(const float* flow_prev) {
  select();
  check(ofdis_set_flow(ctx, 0, cpt->curr_lv + 1, flow_prev, OFDIS_MEM_HOST), ctx, "ofdis_set_flow");
  from_coarser = true;
}

void PatGridClass::Optimize() {
  flush();
  select();
  check(ofdis_patgrid_optimize(ctx, cpt->curr_lv, 0, 1, from_coarser ? 1 : 0), ctx, "ofdis_patgrid_optimize");
  fetched = false;
}

void PatGridClass::AggregateFlowDense(float* flowout) const {
  select();
  check(ofdis_patgrid_aggregate(ctx, cpt->curr_lv, 0, 1), ctx, "ofdis_patgrid_aggregate");
  check(ofdis_get_flow(ctx, 0, cpt->curr_lv, flowout, OFDIS_MEM_HOST), ctx, "ofdis_get_flow");
}

void PatGridClass::fetch() const {
  if (fetched) return;
  p_host.resize((size_t)nopatches * op->nop);
  select();
  check(ofdis_get_patches(ctx, 0, cpt->curr_lv, p_host.data(), nullptr, nullptr, nullptr), ctx, "ofdis_get_patches");
  fetched = true;
}

Vector2f PatGridClass::GetRefPatchPos(int i) const {
  const int x = i / noph, y = i - x * noph;  // patchgrid.cpp:62-69
  return Vector2f{{(float)(x * steps + offw), (float)(y * steps + offh)}};
}

Vector2f PatGridClass::GetQuePatchPos(int i) const {
  fetch();
  Vector2f r = GetRefPatchPos(i);
  r[0] = r[0] + p_host[(size_t)i * op->nop];                      // patch.cpp:217-219
  if (op->nop == 2) r[1] = r[1] + p_host[(size_t)i * op->nop + 1];
  return r;
}

Vector2f PatGridClass::GetQuePatchDis(int i) const { return GetRefPatchPos(i) - GetQuePatchPos(i); }

// ---------------------------------------------------------------------------
VarRefClass::VarRefClass(const float* im_ao_in, const float* im_ao_dx_in, const float* im_ao_dy_in,
                         const float* im_bo_in, const float*, const float*, const camparam* cpt_in,
                         const camparam*, const optparam* op_in, float* flowout, int device) {
  ofdis_ctx* ctx = level_context(cpt_in, op_in, device);
  try {
    check(ofdis_upload_level(ctx, 0, cpt_in->curr_lv, im_ao_in, im_ao_dx_in, im_ao_dy_in, im_bo_in, OFDIS_MEM_HOST),
          ctx, "ofdis_upload_level");
    check(ofdis_set_flow(ctx, 0, cpt_in->curr_lv, flowout, OFDIS_MEM_HOST), ctx, "ofdis_set_flow");
    check(ofdis_varref_refine(ctx, cpt_in->curr_lv, 0, 1), ctx, "ofdis_varref_refine");
    check(ofdis_get_flow(ctx, 0, cpt_in->curr_lv, flowout, OFDIS_MEM_HOST), ctx, "ofdis_get_flow");
  } catch (...) {
    ofdis_destroy(ctx);
    throw;
  }
  ofdis_destroy(ctx);
}

}  // namespace OFC

/* oracle/dis_oracle.c -- CPU restatement of the DIS hot path (TEST INFRASTRUCTURE ONLY).
 *
 * See dis_oracle.h.  Every function cites the reference lines it follows
 * (paths relative to the reference checkout).  All arithmetic is IEEE binary32, one
 * operation per rounding (build with -ffp-contract=off), in the expression
 * order of the reference, because the result must be bitwise equal to the
 * reference build (oracle/_ref) -- SURVEY.md finding 2.
 */
#include "dis_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ */
/* geometry                                                            */
/* ------------------------------------------------------------------ */

/* oflow.cpp:81-92,142-157 and patchgrid.cpp:42-48 */
void dis_make_level(dis_level* L, int width_full, int height_full, int level, int pad,
                    const dis_params* p, int nop, int camlr) {
  float sc_fct = (float)pow(2, -level);
  L->h = (int)(height_full * sc_fct);
  L->w = (int)(width_full * sc_fct);
  L->pad = pad;
  L->tmp_w = L->w + 2 * pad;
  L->noc = p->noc;
  L->nop = nop;
  L->P = p->p_samp_s;
  L->steps = (int)floor(p->p_samp_s * (1 - p->patove));
  if (L->steps < 1) L->steps = 1;
  L->nopw = (int)ceil((float)L->w / (float)L->steps);
  L->noph = (int)ceil((float)L->h / (float)L->steps);
  L->offw = (L->w - (L->nopw - 1) * L->steps) / 2; /* floor of a non-negative int quotient */
  L->offh = (L->h - (L->noph - 1) * L->steps) / 2;
  L->level = level;
  L->camlr = camlr;
  L->lb = -(float)p->p_samp_s / 2;
  L->ubw = (float)(L->w + p->p_samp_s / 2 - 2);
  L->ubh = (float)(L->h + p->p_samp_s / 2 - 2);
  L->outlierthresh = (float)p->p_samp_s / 2;
}

/* ------------------------------------------------------------------ */
/* reductions in the order the reference build uses (Eigen shim)       */
/* ------------------------------------------------------------------ */

/* Sum of f(i), i in [0,n): 8 strided partial sums (two 4-wide accumulators),
 * folded 8->4, optional 4-wide remainder, then (a0+a2)+(a1+a3), scalar tail. */
typedef float (*elem_fn)(const void* ctx, int i);

static float sum_packet_order(int n, elem_fn f, const void* ctx) {
  int n4 = (n / 4) * 4, n8 = (n / 8) * 8, l, idx, i;
  float res;
  if (n4) {
    float a[4], b[4];
    for (l = 0; l < 4; ++l) a[l] = f(ctx, l);
    if (n4 > 4) {
      for (l = 0; l < 4; ++l) b[l] = f(ctx, 4 + l);
      for (idx = 8; idx < n8; idx += 8)
        for (l = 0; l < 4; ++l) {
          a[l] = a[l] + f(ctx, idx + l);
          b[l] = b[l] + f(ctx, idx + 4 + l);
        }
      for (l = 0; l < 4; ++l) a[l] = a[l] + b[l];
      if (n4 > n8)
        for (l = 0; l < 4; ++l) a[l] = a[l] + f(ctx, n8 + l);
    }
    {
      float t0 = a[0] + a[2], t1 = a[1] + a[3];
      res = t0 + t1;
    }
    for (i = n4; i < n; ++i) res = res + f(ctx, i);
  } else {
    res = f(ctx, 0);
    for (i = 1; i < n; ++i) res = res + f(ctx, i);
  }
  return res;
}

typedef struct { const float* a; const float* b; } two_vecs;
static float el_id(const void* c, int i) { return ((const two_vecs*)c)->a[i]; }
static float el_abs(const void* c, int i) { return fabsf(((const two_vecs*)c)->a[i]); }
static float el_mul(const void* c, int i) {
  const two_vecs* t = (const two_vecs*)c;
  return t->a[i] * t->b[i];
}
static float vsum(const float* a, int n) { two_vecs t = {a, 0}; return sum_packet_order(n, el_id, &t); }
static float vabssum(const float* a, int n) { two_vecs t = {a, 0}; return sum_packet_order(n, el_abs, &t); }
static float vdot(const float* a, const float* b, int n) { two_vecs t = {a, b}; return sum_packet_order(n, el_mul, &t); }

float dis_sum_packet_order(const float* v, int n) { return vsum(v, n); }

/* ------------------------------------------------------------------ */
/* patch stage                                                         */
/* ------------------------------------------------------------------ */

/* PatClass::getPatchStaticNNGrad (patch.cpp:287-332): integer-position gather of
 * template and gradients, (y, x, c) order, optional joint mean subtraction. */
static void patch_template(const dis_level* L, int patnorm, const float* i0, const float* i0x,
                           const float* i0y, float cx, float cy, float* T, float* gx, float* gy) {
  int P = L->P, C = L->noc, n = C * P * P, k = 0, x, y, c;
  int px = (int)roundf(cx) + L->pad, py = (int)roundf(cy) + L->pad;
  for (y = -P / 2; y <= P / 2 - 1; ++y)
    for (x = -P / 2; x <= P / 2 - 1; ++x) {
      int idx = ((px + x) + (py + y) * L->tmp_w) * C;
      for (c = 0; c < C; ++c, ++k) {
        T[k] = i0[idx + c];
        gx[k] = i0x[idx + c];
        gy[k] = i0y[idx + c];
      }
    }
  if (patnorm > 0) {
    float m = vsum(T, n) / n;
    for (k = 0; k < n; ++k) T[k] = T[k] - m;
  }
}

/* PatClass::getPatchStaticBil (patch.cpp:335-402): one weight set per patch,
 * taps a=(ceil(x+1e-5), ceil(y+1e-5)), b=a-1px, c=row above, d=c-1px. */
static void patch_bilinear(const dis_level* L, int patnorm, const float* i1, float mx, float my,
                           float* out) {
  int P = L->P, C = L->noc, n = C * P * P, k = 0, x, y, c;
  int pcx = (int)ceilf(mx + .00001f), pcy = (int)ceilf(my + .00001f);
  int pfx = (int)floorf(mx), pfy = (int)floorf(my);
  float rx = mx - (float)pfx, ry = my - (float)pfy;
  float w0 = rx * ry, w1 = (1 - rx) * ry, w2 = rx * (1 - ry), w3 = (1 - rx) * (1 - ry);
  pcx += L->pad;
  pcy += L->pad;
  for (y = -P / 2; y <= P / 2 - 1; ++y)
    for (x = -P / 2; x <= P / 2 - 1; ++x) {
      const float* a = i1 + ((pcx + x) + (pcy + y) * L->tmp_w) * C;
      const float* b = a - C;
      const float* cc = a - L->tmp_w * C;
      const float* d = cc - C;
      for (c = 0; c < C; ++c, ++k) out[k] = w0 * a[c] + w1 * b[c] + w2 * cc[c] + w3 * d[c];
    }
  if (patnorm > 0) {
    float m = vsum(out, n) / n;
    for (k = 0; k < n; ++k) out[k] = out[k] - m;
  }
}

/* PatClass::LossComputeErrorImage (patch.cpp:223-262).  costfct outside {0,1,2}
 * leaves both vectors untouched, as the reference does. */
static void patch_loss(int costfct, int n, float* pdiff, float* pweight, const float* T) {
  int k;
  const float bsq = 5.0f * 5.0f, two_bsq = bsq * 2.0f; /* normoutlier = 5 (oflow.h:63, oflow.cpp:106-107) */
  if (costfct == 0) {
    for (k = 0; k < n; ++k) {
      pdiff[k] = pdiff[k] - T[k];
      pweight[k] = fabsf(pdiff[k]);
    }
  } else if (costfct == 1) {
    for (k = 0; k < n; ++k) {
      float d = pdiff[k] - T[k];
      pdiff[k] = copysignf(sqrtf(fabsf(d)), d);
      pweight[k] = fabsf(pdiff[k]);
    }
  } else if (costfct == 2) {
    for (k = 0; k < n; ++k) {
      float d = pdiff[k] - T[k];
      float h = sqrtf((sqrtf(1.0f + (d * d) / bsq) - 1.0f) * two_bsq);
      /* orps(sign(d), h): h >= 0 (or NaN), so this is copysign */
      pdiff[k] = copysignf(h, d);
      pweight[k] = fabsf(pdiff[k]);
    }
  }
}

typedef struct {
  float H00, H01, H11;     /* Hessian (patch.cpp:71-88) */
  float L00, L10, L11;     /* its (possibly partial) Cholesky factor */
} patch_hess;

/* PatClass::ComputeHessian (patch.cpp:71-88) + Eigen LLT (shim).  *branch (nullable) receives the
 * DIS_HESS_* bits of the data-dependent fallbacks taken; they do not change the arithmetic. */
static void patch_hessian(int nop, int n, const float* gx, const float* gy, patch_hess* h, int* branch) {
  int b = 0;
  if (nop == 2) {
    h->H00 = vdot(gx, gx, n);
    h->H01 = vdot(gx, gy, n);
    h->H11 = vdot(gy, gy, n);
    if (h->H00 * h->H11 - h->H01 * h->H01 == 0) {
      b |= h->H00 == 0 ? DIS_HESS_SINGULAR_ZERO : DIS_HESS_SINGULAR;
      h->H00 = (float)(h->H00 + 1e-10);
      h->H11 = (float)(h->H11 + 1e-10);
    }
    h->L00 = h->H00;
    h->L10 = h->H01;
    h->L11 = h->H11;
    if (h->H00 > 0) {
      float x;
      h->L00 = sqrtf(h->H00);
      h->L10 = h->H01 / h->L00;
      x = h->H11 - h->L10 * h->L10;
      if (x > 0) h->L11 = sqrtf(x);
      else b |= DIS_HESS_NOT_PD;
    }
  } else {
    h->H00 = vdot(gx, gx, n);
    if (h->H00 == 0) {
      b |= DIS_HESS_STEREO_ZERO;
      h->H00 = (float)(h->H00 + 1e-10);
    }
    h->L00 = h->H00 > 0 ? sqrtf(h->H00) : h->H00;
    h->H01 = h->H11 = h->L10 = h->L11 = 0;
  }
  if (branch) *branch = b;
}

/* PatClass::OptimizeIter / OptimizeStart / OptimizeComputeErrImg (patch.cpp:119-212, 264-284) */
static void patch_optimize(const dis_level* L, const dis_params* prm, const float* i1, float refx,
                           float refy, const float* T, const float* gx, const float* gy,
                           const patch_hess* H, const float* p_in, float* p_out, float* pdiff,
                           float* pweight, int* conv_out, int* cnt_out) {
  const int nop = L->nop, n = L->noc * L->P * L->P;
  const float dp_thresh_sq = prm->dp_thresh * prm->dp_thresh; /* oflow.cpp:88 */
  float p[2] = {0, 0}, dp[2] = {0, 0};
  float ptx, pty, stx, sty;
  float dpsq = 1e-10f, dpsq_init = 1e-10f, mares = 1e5f, mares_old = 1e20f;
  int cnt = 0, conv = 0, k;

  for (k = 0; k < nop; ++k) p[k] = p_in[k];
  ptx = refx + p[0];
  pty = (nop == 2) ? refy + p[1] : refy;
  stx = ptx;
  sty = pty;

  if (ptx < L->lb || pty < L->lb || ptx > L->ubw || pty > L->ubh) {
    /* patch.cpp:135-141: converged at once; pdiff=template, pweight never written */
    for (k = 0; k < n; ++k) pdiff[k] = T[k];
    conv = 1;
  } else {
    for (;;) {
      /* OptimizeComputeErrImg (patch.cpp:264-284) */
      patch_bilinear(L, prm->patnorm, i1, ptx, pty, pdiff);
      patch_loss(prm->costfct, n, pdiff, pweight, T);
      dpsq = (nop == 2) ? dp[0] * dp[0] + dp[1] * dp[1] : dp[0] * dp[0];
      if (cnt == 1) dpsq_init = dpsq;
      mares_old = mares;
      mares = vabssum(pweight, n) / n;
      if (!((cnt < prm->max_iter) & (mares > prm->res_thresh) &
            ((cnt < prm->min_iter) | (dpsq / dpsq_init >= dp_thresh_sq)) &
            ((cnt < prm->min_iter) | (mares / mares_old <= prm->dr_thresh))))
        conv = 1;
      if (conv) break;

      /* one Gauss-Newton step (patch.cpp:174-208) */
      cnt++;
      if (nop == 2) {
        float b0 = vdot(gx, pdiff, n), b1 = vdot(gy, pdiff, n);
        float y0 = b0 / H->L00;
        float y1 = (b1 - H->L10 * y0) / H->L11;
        dp[1] = y1 / H->L11;
        dp[0] = (y0 - H->L10 * dp[1]) / H->L00;
        p[0] = p[0] - dp[0];
        p[1] = p[1] - dp[1];
        ptx = refx + p[0];
        pty = refy + p[1];
      } else {
        float b0 = vdot(gx, pdiff, n);
        dp[0] = (b0 / H->L00) / H->L00;
        p[0] = p[0] - dp[0];
        /* std::min / std::max operand order (patch.cpp:188-193) */
        if (L->camlr == 0) p[0] = (0.0f < p[0]) ? 0.0f : p[0];
        else p[0] = (p[0] < 0.0f) ? 0.0f : p[0];
        ptx = refx + p[0];
      }
      {
        float ex = stx - ptx, ey = sty - pty;
        if (sqrtf(ex * ex + ey * ey) > L->outlierthresh || ptx < L->lb || pty < L->lb ||
            ptx > L->ubw || pty > L->ubh) {
          for (k = 0; k < nop; ++k) p[k] = p_in[k];
          ptx = refx + p[0];
          if (nop == 2) pty = refy + p[1];
          conv = 1; /* the error image is still recomputed once (patch.cpp:210) */
        }
      }
      if (conv) {
        patch_bilinear(L, prm->patnorm, i1, ptx, pty, pdiff);
        patch_loss(prm->costfct, n, pdiff, pweight, T);
        break;
      }
    }
  }
  for (k = 0; k < nop; ++k) p_out[k] = p[k];
  *conv_out = conv;
  *cnt_out = cnt;
}

int dis_patches_level(const dis_level* L, const dis_params* prm, const float* i0, const float* i0x,
                      const float* i0y, const float* i1, const float* flow_prev, float* p_out,
                      float* pweight_out, int* conv_out, int* cnt_out) {
  const int n = L->noc * L->P * L->P, np = L->nopw * L->noph;
  float* buf = (float*)calloc((size_t)5 * n, sizeof(float));
  float *T = buf, *gx = buf + n, *gy = buf + 2 * n, *pdiff = buf + 3 * n, *pw = buf + 4 * n;
  int px, py;
  for (px = 0; px < L->nopw; ++px)
    for (py = 0; py < L->noph; ++py) {
      const int ip = px * L->noph + py; /* patchgrid.cpp:62-69 */
      const float refx = (float)(px * L->steps + L->offw), refy = (float)(py * L->steps + L->offh);
      float pin[2] = {0, 0}, pout[2];
      patch_hess H;
      int conv, cnt;
      if (flow_prev) { /* InitializeFromCoarserOF, patchgrid.cpp:195-211 */
        int x = (int)floorf(refx / 2), y = (int)floorf(refy / 2);
        int i = y * (L->w / 2) + x;
        if (L->nop == 2) {
          pin[0] = flow_prev[2 * i] * 2;
          pin[1] = flow_prev[2 * i + 1] * 2;
        } else
          pin[0] = flow_prev[i] * 2;
      }
      patch_template(L, prm->patnorm, i0, i0x, i0y, refx, refy, T, gx, gy);
      patch_hessian(L->nop, n, gx, gy, &H, NULL);
      memset(pw, 0, sizeof(float) * n); /* fresh PatClass per level: zeroed storage (shim) */
      patch_optimize(L, prm, i1, refx, refy, T, gx, gy, &H, pin, pout, pdiff, pw, &conv, &cnt);
      if (p_out) memcpy(p_out + (size_t)ip * L->nop, pout, sizeof(float) * L->nop);
      if (pweight_out) memcpy(pweight_out + (size_t)ip * n, pw, sizeof(float) * n);
      if (conv_out) conv_out[ip] = conv;
      if (cnt_out) cnt_out[ip] = cnt;
    }
  free(buf);
  return np;
}

int dis_patches_level_branches(const dis_level* L, const dis_params* prm, const float* i0, const float* i0x,
                               const float* i0y, int* branch_out) {
  const int n = L->noc * L->P * L->P, np = L->nopw * L->noph;
  float* buf = (float*)calloc((size_t)3 * n, sizeof(float));
  int px, py;
  for (px = 0; px < L->nopw; ++px)
    for (py = 0; py < L->noph; ++py) {
      const int ip = px * L->noph + py;
      patch_hess H;
      patch_template(L, prm->patnorm, i0, i0x, i0y, (float)(px * L->steps + L->offw),
                     (float)(py * L->steps + L->offh), buf, buf + n, buf + 2 * n);
      patch_hessian(L->nop, n, buf + n, buf + 2 * n, &H, branch_out + ip);
    }
  free(buf);
  return np;
}

/* PatGridClass::AggregateFlowDense without the fwd/bwd merge (patchgrid.cpp:213-275,377-394).
 * Written as the per-pixel gather the GPU uses: covering patches visited in
 * ascending ip = px*noph+py, which is the order the reference's scatter adds them. */
#define STD_MAX(a, b) (((a) < (b)) ? (b) : (a)) /* std::max operand order */
void dis_densify(const dis_level* L, const dis_params* prm, const float* p, const float* pweight,
                 float* flow_out) {
  const int P = L->P, C = L->noc, n = C * P * P, nop = L->nop;
  const float minerrval = 2.0f; /* oflow.h:62 */
  int xi, yi, px, py, c, k;
  (void)prm;
  for (yi = 0; yi < L->h; ++yi)
    for (xi = 0; xi < L->w; ++xi) {
      float we = 0, acc[2] = {0, 0};
      for (px = 0; px < L->nopw; ++px) {
        int dx = xi - (px * L->steps + L->offw);
        if (dx < -P / 2 || dx > P / 2 - 1) continue;
        for (py = 0; py < L->noph; ++py) {
          int dy = yi - (py * L->steps + L->offh), ip = px * L->noph + py;
          const float* pw;
          float absw;
          if (dy < -P / 2 || dy > P / 2 - 1) continue;
          {
            /* patchgrid.cpp:243-259: the weight cursor advances by 1 for a patch
             * pixel outside the image and by C for one inside, so for C==3 the
             * index of pixel k is k + 2*(in-image pixels before k). */
            int rx = dx + P / 2, ry = dy + P / 2, cx = px * L->steps + L->offw, cy = py * L->steps + L->offh;
            int x0 = cx - P / 2 < 0 ? P / 2 - cx : 0, y0 = cy - P / 2 < 0 ? P / 2 - cy : 0;
            int x1 = cx + P / 2 - 1 > L->w - 1 ? L->w - 1 - cx + P / 2 : P - 1;
            int inb = (ry - y0) * (x1 - x0 + 1) + (rx - x0);
            pw = pweight + (size_t)ip * n + (ry * P + rx) + (C - 1) * inb;
          }
          if (C == 1)
            absw = 1.0f / STD_MAX(minerrval, pw[0]);
          else {
            absw = STD_MAX(minerrval, pw[0]);
            for (c = 1; c < C; ++c) absw += STD_MAX(minerrval, pw[c]);
            absw = 1.0f / absw;
          }
          we += absw;
          for (k = 0; k < nop; ++k) acc[k] += p[ip * nop + k] * absw;
        }
      }
      for (k = 0; k < nop; ++k) flow_out[(yi * L->w + xi) * nop + k] = we > 0 ? acc[k] / we : acc[k];
    }
}

/* ------------------------------------------------------------------ */
/* variational refinement                                              */
/* ------------------------------------------------------------------ */

#define DATANORM (0.1f * 0.1f)      /* opticalflow_aux.c:10 */
#define EPS_COLOR (0.001f * 0.001f) /* :11 */
#define EPS_GRAD (0.001f * 0.001f)  /* :12 */
#define EPS_SMOOTH (0.001f * 0.001f) /* :14 */

static int clampi(int v, int n) { return v < 0 ? 0 : (v > n - 1 ? n - 1 : v); }

/* image_warp (opticalflow_aux.c:17-60) fused with VarRefClass::copyimage
 * (refine_variational.cpp:119-149): reads the padded interleaved image directly. */
void dis_warp(const dis_level* L, const float* i1p, const float* wx, const float* wy, float* warped,
              float* mask) {
  const int w = L->w, h = L->h, C = L->noc;
  int i, j, c;
  for (j = 0; j < h; ++j)
    for (i = 0; i < w; ++i) {
      const int o = j * w + i;
      float xx = i + wx[o], yy = j + wy[o];
      int x = (int)floor(xx), y = (int)floor(yy);
      float dx = xx - x, dy = yy - y;
      int x1 = clampi(x, w), x2 = clampi(x + 1, w), y1 = clampi(y, h), y2 = clampi(y + 1, h);
      mask[o] = (xx >= 0 && xx <= w - 1 && yy >= 0 && yy <= h - 1);
      for (c = 0; c < C; ++c) {
#define PIX(X, Y) i1p[(((Y) + L->pad) * L->tmp_w + (X) + L->pad) * C + c]
        warped[c * w * h + o] = PIX(x1, y1) * (1.0f - dx) * (1.0f - dy) + PIX(x2, y1) * dx * (1.0f - dy) +
                                PIX(x1, y2) * (1.0f - dx) * dy + PIX(x2, y2) * dx * dy;
#undef PIX
      }
    }
}

/* convolve_horiz_fast_5 (image.c:466-502): replicate borders, all five products */
static float conv_h5(const float* s, int w, int i, const float* c) {
  return c[0] * s[clampi(i - 2, w)] + c[1] * s[clampi(i - 1, w)] + c[2] * s[i] + c[3] * s[clampi(i + 1, w)] +
         c[4] * s[clampi(i + 2, w)];
}
/* convolve_vert_fast_5 (image.c:401-434): border rows fold the COEFFICIENTS */
static float conv_v5(const float* s, int w, int h, int i, int j, const float* c) {
  const float* q = s + j * w + i;
  if (j == 0) return (c[0] + c[1] + c[2]) * q[0] + c[3] * q[w] + c[4] * q[2 * w];
  if (j == 1) return (c[0] + c[1]) * q[-w] + c[2] * q[0] + c[3] * q[w] + c[4] * q[2 * w];
  if (j == h - 2) return c[0] * q[-2 * w] + c[1] * q[-w] + c[2] * q[0] + (c[3] + c[4]) * q[w];
  if (j == h - 1) return c[0] * q[-2 * w] + c[1] * q[-w] + (c[2] + c[3] + c[4]) * q[0];
  return c[0] * q[-2 * w] + c[1] * q[-w] + c[2] * q[0] + c[3] * q[w] + c[4] * q[2 * w];
}
/* convolve_horiz_fast_3 (image.c:436-464) / convolve_vert_fast_3 (image.c:376-399) */
static float conv_h3(const float* s, int w, int i, const float* c) {
  return c[0] * s[clampi(i - 1, w)] + c[1] * s[i] + c[2] * s[clampi(i + 1, w)];
}
static float conv_v3(const float* s, int w, int h, int i, int j, const float* c) {
  const float* q = s + j * w + i;
  if (j == 0) return (c[0] + c[1]) * q[0] + c[2] * q[w];
  if (j == h - 1) return c[0] * q[-w] + (c[1] + c[2]) * q[0];
  return c[0] * q[-w] + c[1] * q[0] + c[2] * q[w];
}

/* convolve_extract_coeffs, even=0 (image.c:338-342) with the filters of
 * refine_variational.cpp:45-48 */
static void deriv5_coeffs(float* c) {
  const float half[3] = {0.0f, -8.0f / 12.0f, 1.0f / 12.0f};
  int i;
  for (i = 0; i <= 2; ++i) {
    c[2 - i] = +half[i];
    c[2 + i] = -half[i];
  }
}
static void deriv3_coeffs(float* c) {
  const float half[2] = {0.0f, -0.5f};
  int i;
  for (i = 0; i <= 1; ++i) {
    c[1 - i] = +half[i];
    c[1 + i] = -half[i];
  }
}

/* get_derivatives (opticalflow_aux.c:64-116); planar per channel */
void dis_derivatives(const dis_level* L, const float* i0p, const float* warped, float* Ix, float* Iy,
                     float* Iz, float* Ixx, float* Ixy, float* Iyy, float* Ixz, float* Iyz) {
  const int w = L->w, h = L->h, C = L->noc, n = w * h;
  float c5[5];
  float* avg = (float*)malloc(sizeof(float) * n);
  int i, j, c;
  deriv5_coeffs(c5);
  for (c = 0; c < C; ++c) {
    const int b = c * n;
    for (j = 0; j < h; ++j)
      for (i = 0; i < w; ++i) {
        float im1 = i0p[((j + L->pad) * L->tmp_w + i + L->pad) * C + c], im2 = warped[b + j * w + i];
        avg[j * w + i] = 0.5f * (im2 + im1);
        Iz[b + j * w + i] = im2 - im1;
      }
    for (j = 0; j < h; ++j)
      for (i = 0; i < w; ++i) {
        Ix[b + j * w + i] = conv_h5(avg + j * w, w, i, c5);
        Iy[b + j * w + i] = conv_v5(avg, w, h, i, j, c5);
        Ixz[b + j * w + i] = conv_h5(Iz + b + j * w, w, i, c5);
        Iyz[b + j * w + i] = conv_v5(Iz + b, w, h, i, j, c5);
      }
    for (j = 0; j < h; ++j)
      for (i = 0; i < w; ++i) {
        Ixx[b + j * w + i] = conv_h5(Ix + b + j * w, w, i, c5);
        Ixy[b + j * w + i] = conv_v5(Ix + b, w, h, i, j, c5);
        Iyy[b + j * w + i] = conv_v5(Iy + b, w, h, i, j, c5);
      }
  }
  free(avg);
}

/* compute_smoothness (opticalflow_aux.c:123-165) */
void dis_smoothness(int w, int h, const float* uu, const float* vv, float qa, float* sh, float* sv) {
  float c3[3];
  float* s = (float*)malloc(sizeof(float) * w * h);
  int i, j;
  deriv3_coeffs(c3);
  for (j = 0; j < h; ++j)
    for (i = 0; i < w; ++i) {
      float ux = conv_h3(uu + j * w, w, i, c3), vx = conv_h3(vv + j * w, w, i, c3);
      float uy = conv_v3(uu, w, h, i, j, c3), vy = conv_v3(vv, w, h, i, j, c3);
      s[j * w + i] = qa / sqrtf(ux * ux + uy * uy + vx * vx + vy * vy + EPS_SMOOTH);
    }
  for (j = 0; j < h; ++j)
    for (i = 0; i < w; ++i) {
      sh[j * w + i] = (i < w - 1) ? s[j * w + i] + s[j * w + i + 1] : 0.0f;
      sv[j * w + i] = (j < h - 1) ? s[j * w + i] + s[(j + 1) * w + i] : 0.0f;
    }
  free(s);
}

/* compute_data / compute_data_DE (opticalflow_aux.c:309-438, 445-548).
 * nop==1 drops every dv/a12/a22/b2 term exactly as compute_data_DE does. */
void dis_data_term(const dis_level* L, const float* mask, const float* du, const float* dv,
                   const float* Ix, const float* Iy, const float* Iz, const float* Ixx,
                   const float* Ixy, const float* Iyy, const float* Ixz, const float* Iyz, float hdo3,
                   float hgo3, float* a11, float* a12, float* a22, float* b1, float* b2) {
  const int n = L->w * L->h, C = L->noc, flow = (L->nop == 2);
  int o, c;
  for (o = 0; o < n; ++o) {
    float A11 = 0, A12 = 0, A22 = 0, B1 = 0, B2 = 0, t, t2 = 0, nn, n2;
    const float u = du[o], v = flow ? dv[o] : 0.0f, m = mask[o];
    if (C == 1) {
      const float ix = Ix[o], iy = Iy[o], iz = Iz[o], ixx = Ixx[o], ixy = Ixy[o], iyy = Iyy[o],
                  ixz = Ixz[o], iyz = Iyz[o];
      if (hdo3) {
        t = flow ? iz + ix * u + iy * v : iz + ix * u;
        nn = ix * ix + iy * iy + DATANORM;
        t = m * hdo3 / sqrtf(3 * t * t / nn + EPS_COLOR);
        t /= nn;
        A11 += t * ix * ix;
        B1 -= t * iz * ix;
        if (flow) {
          A12 += t * ix * iy;
          A22 += t * iy * iy;
          B2 -= t * iz * iy;
        }
      }
      nn = ixx * ixx + ixy * ixy + DATANORM;
      n2 = iyy * iyy + ixy * ixy + DATANORM;
      t = flow ? ixz + ixx * u + ixy * v : ixz + ixx * u;
      t2 = flow ? iyz + ixy * u + iyy * v : iyz + ixy * u;
      t = m * hgo3 / sqrtf(3 * t * t / nn + 3 * t2 * t2 / n2 + EPS_GRAD);
      t2 = t / n2;
      t /= nn;
      A11 += t * ixx * ixx + t2 * ixy * ixy;
      B1 -= t * ixx * ixz + t2 * ixy * iyz;
      if (flow) {
        A12 += t * ixx * ixy + t2 * ixy * iyy;
        A22 += t2 * iyy * iyy + t * ixy * ixy;
        B2 -= t2 * iyy * iyz + t * ixy * ixz;
      }
      A11 *= 3;
      B1 *= 3;
      if (flow) {
        A12 *= 3;
        A22 *= 3;
        B2 *= 3;
      }
    } else {
      float tc[3], nc[3], tg[6], ng[6], acc;
      if (hdo3) {
        for (c = 0; c < 3; ++c) {
          const float ix = Ix[c * n + o], iy = Iy[c * n + o], iz = Iz[c * n + o];
          tc[c] = flow ? iz + ix * u + iy * v : iz + ix * u;
          nc[c] = ix * ix + iy * iy + DATANORM;
        }
        acc = tc[0] * tc[0] / nc[0] + tc[1] * tc[1] / nc[1] + tc[2] * tc[2] / nc[2] + EPS_COLOR;
        t = m * hdo3 / sqrtf(acc);
        for (c = 0; c < 3; ++c) {
          const float ix = Ix[c * n + o], iy = Iy[c * n + o], iz = Iz[c * n + o];
          const float tt = t / nc[c];
          A11 += tt * ix * ix;
          B1 -= tt * iz * ix;
          if (flow) {
            A12 += tt * ix * iy;
            A22 += tt * iy * iy;
            B2 -= tt * iz * iy;
          }
        }
      }
      for (c = 0; c < 3; ++c) {
        const float ixx = Ixx[c * n + o], ixy = Ixy[c * n + o], iyy = Iyy[c * n + o],
                    ixz = Ixz[c * n + o], iyz = Iyz[c * n + o];
        ng[2 * c] = ixx * ixx + ixy * ixy + DATANORM;
        ng[2 * c + 1] = iyy * iyy + ixy * ixy + DATANORM;
        tg[2 * c] = flow ? ixz + ixx * u + ixy * v : ixz + ixx * u;
        tg[2 * c + 1] = flow ? iyz + ixy * u + iyy * v : iyz + ixy * u;
      }
      acc = tg[0] * tg[0] / ng[0] + tg[1] * tg[1] / ng[1] + tg[2] * tg[2] / ng[2] + tg[3] * tg[3] / ng[3] +
            tg[4] * tg[4] / ng[4] + tg[5] * tg[5] / ng[5] + EPS_GRAD;
      t = m * hgo3 / sqrtf(acc);
      for (c = 0; c < 3; ++c) {
        const float ixx = Ixx[c * n + o], ixy = Ixy[c * n + o], iyy = Iyy[c * n + o],
                    ixz = Ixz[c * n + o], iyz = Iyz[c * n + o];
        const float ta = t / ng[2 * c], tb = t / ng[2 * c + 1];
        A11 += ta * ixx * ixx + tb * ixy * ixy;
        B1 -= ta * ixx * ixz + tb * ixy * iyz;
        if (flow) {
          A12 += ta * ixx * ixy + tb * ixy * iyy;
          A22 += tb * iyy * iyy + ta * ixy * ixy;
          B2 -= tb * iyy * iyz + ta * ixy * ixz;
        }
      }
    }
    a11[o] = A11;
    b1[o] = B1;
    if (flow) {
      a12[o] = A12;
      a22[o] = A22;
      b2[o] = B2;
    }
  }
}

/* sub_laplacian (opticalflow_aux.c:172-199): per pixel, in the order the two
 * reference passes touch it: -t_h(i-1), +t_h(i), -t_v(j-1), +t_v(j). */
void dis_sub_laplacian(int w, int h, float* b, const float* src, const float* sh, const float* sv) {
  int i, j;
  for (j = 0; j < h; ++j)
    for (i = 0; i < w; ++i) {
      const int o = j * w + i;
      float v = b[o];
      if (i > 0) v -= sh[o - 1] * (src[o] - src[o - 1]);
      if (i < w - 1) v += sh[o] * (src[o + 1] - src[o]);
      if (j > 0) v -= sv[o - w] * (src[o] - src[o - w]);
      if (j < h - 1) v += sv[o] * (src[o + w] - src[o]);
      b[o] = v;
    }
}

/* sor_coupled (solver.c:77-421), per pixel in raster order.  Right/bottom
 * neighbours are still the previous sweep's values when pixel o is visited,
 * left/top are already this sweep's; the reference's row copies (solver.c:
 * 108-110) give the same thing. */
void dis_sor_coupled(int w, int h, float* du, float* dv, float* a11, float* a12, float* a22,
                     const float* b1, const float* b2, const float* sh, const float* sv, int iterations,
                     float omega) {
  int it, i, j;
  if (w < 2 || h < 2 || iterations < 1) return; /* reference falls back to another solver; not on this path */
  for (it = 0; it < iterations; ++it)
    for (j = 0; j < h; ++j)
      for (i = 0; i < w; ++i) {
        const int o = j * w + i;
        const float hl = i > 0 ? sh[o - 1] : 0.0f, hh = sh[o];
        const float dur = i < w - 1 ? du[o + 1] : 0.0f, dvr = i < w - 1 ? dv[o + 1] : 0.0f;
        float s1, s2, B1, B2;
        if (it == 0) { /* solver.c:115-120 and twins */
          float dps, A11, A22, det;
          if (j == 0) dps = hl + hh + sv[o];
          else if (j == h - 1) dps = hl + hh + sv[o - w];
          else dps = hl + hh + sv[o - w] + sv[o];
          A11 = a22[o] + dps;
          A22 = a11[o] + dps;
          det = A11 * A22 - a12[o] * a12[o];
          a11[o] = A11 / det;
          a22[o] = A22 / det;
          a12[o] = a12[o] / -det;
        }
        if (j == 0) {
          s1 = hh * dur + sv[o] * du[o + w] + b1[o];
          s2 = hh * dvr + sv[o] * dv[o + w] + b2[o];
        } else if (j == h - 1) {
          s1 = hh * dur + sv[o - w] * du[o - w] + b1[o];
          s2 = hh * dvr + sv[o - w] * dv[o - w] + b2[o];
        } else {
          s1 = hh * dur + sv[o - w] * du[o - w] + sv[o] * du[o + w] + b1[o];
          s2 = hh * dvr + sv[o - w] * dv[o - w] + sv[o] * dv[o + w] + b2[o];
        }
        if (i == 0) {
          B1 = s1;
          B2 = s2;
        } else {
          B1 = hl * du[o - 1] + s1;
          B2 = hl * dv[o - 1] + s2;
        }
        du[o] += omega * (a11[o] * B1 + a12[o] * B2 - du[o]);
        dv[o] += omega * (a12[o] * B1 + a22[o] * B2 - dv[o]);
      }
}

/* sor_coupled_slow_but_readable_DE (solver.c:428-466) */
void dis_sor_de(int w, int h, float* du, const float* a11, const float* b1, const float* sh,
                const float* sv, int iterations, float omega) {
  int it, i, j;
  for (it = 0; it < iterations; ++it)
    for (j = 0; j < h; ++j)
      for (i = 0; i < w; ++i) {
        const int o = j * w + i;
        float sigma = 0.0f, sum = 0.0f, A11, B1;
        if (j > 0) { sigma -= sv[o - w] * du[o - w]; sum += sv[o - w]; }
        if (i > 0) { sigma -= sh[o - 1] * du[o - 1]; sum += sh[o - 1]; }
        if (j < h - 1) { sigma -= sv[o] * du[o + w]; sum += sv[o]; }
        if (i < w - 1) { sigma -= sh[o] * du[o + 1]; sum += sh[o]; }
        A11 = a11[o] + sum;
        B1 = b1[o] - sigma;
        du[o] = (1.0f - omega) * du[o] + omega * (B1 / A11);
      }
}

/* VarRefClass ctor + RefLevelOF / RefLevelDE (refine_variational.cpp:25-116,152-241,244-336) */
void dis_varref_level(const dis_level* L, const dis_params* prm, const float* i0, const float* i1,
                      float* flow) {
  const int w = L->w, h = L->h, n = w * h, C = L->noc, nop = L->nop;
  const int n_inner = prm->tv_innerit * (L->level + 1);
  const float qa = 0.25f * prm->tv_alpha;
  const float hgo3 = prm->tv_gamma * 0.5f / 3.0f;
  const float hdo3 = prm->tv_delta * 0.5f / 3.0f;
  const int nplanes = 14 + 9 * C;
  float* buf = (float*)calloc((size_t)nplanes * n, sizeof(float));
  float *wx = buf, *wy = wx + n, *du = wy + n, *dv = du + n, *uu = dv + n, *vv = uu + n, *mask = vv + n,
        *sh = mask + n, *sv = sh + n, *a11 = sv + n, *a12 = a11 + n, *a22 = a12 + n, *b1 = a22 + n,
        *b2 = b1 + n;
  float *warped = b2 + n, *Ix = warped + C * n, *Iy = Ix + C * n, *Iz = Iy + C * n, *Ixx = Iz + C * n,
        *Ixy = Ixx + C * n, *Iyy = Ixy + C * n, *Ixz = Iyy + C * n, *Iyz = Ixz + C * n;
  int o, it;
  for (o = 0; o < n; ++o) {
    wx[o] = flow[o * nop];
    wy[o] = nop == 2 ? flow[o * nop + 1] : 0.0f;
  }
  dis_warp(L, i1, wx, wy, warped, mask);
  dis_derivatives(L, i0, warped, Ix, Iy, Iz, Ixx, Ixy, Iyy, Ixz, Iyz);
  memcpy(uu, wx, sizeof(float) * n);
  memcpy(vv, wy, sizeof(float) * n);
  for (it = 0; it < n_inner; ++it) {
    dis_smoothness(w, h, uu, vv, qa, sh, sv);
    dis_data_term(L, mask, du, dv, Ix, Iy, Iz, Ixx, Ixy, Iyy, Ixz, Iyz, hdo3, hgo3, a11, a12, a22, b1, b2);
    dis_sub_laplacian(w, h, b1, wx, sh, sv);
    if (nop == 2) {
      dis_sub_laplacian(w, h, b2, wy, sh, sv);
      dis_sor_coupled(w, h, du, dv, a11, a12, a22, b1, b2, sh, sv, prm->tv_solverit, prm->tv_sor);
      for (o = 0; o < n; ++o) {
        uu[o] = wx[o] + du[o];
        vv[o] = wy[o] + dv[o];
      }
    } else {
      dis_sor_de(w, h, du, a11, b1, sh, sv, prm->tv_solverit, prm->tv_sor);
      for (o = 0; o < n; ++o) { /* minps / maxps with zero (refine_variational.cpp:299-314) */
        float t = wx[o] + du[o];
        uu[o] = L->camlr == 0 ? (t < 0.0f ? t : 0.0f) : (t > 0.0f ? t : 0.0f);
      }
    }
  }
  for (o = 0; o < n; ++o) {
    flow[o * nop] = uu[o];
    if (nop == 2) flow[o * nop + 1] = vv[o];
  }
  free(buf);
}

/* The second loop of PatGridClass::AggregateFlowDense (patchgrid.cpp:278-375): the complementary
 * grid's patches, at their displaced positions, splat their NEGATED flow bilinearly.  Gather form:
 * for one cell the reference's scatter visits the patches in ascending ip and, inside a patch, the
 * pixels in raster order, so a cell receives at most four terms per patch -- from the patch pixels
 * at (cx,cy) [weight wbil0], (cx+1,cy) [wbil1], (cx,cy+1) [wbil2], (cx+1,cy+1) [wbil3], in that order. */
static void densify_cg_cell(const dis_level* L, const float* cg_p, const float* cg_pweight, int xi, int yi,
                            float* we, float* acc) {
  const int P = L->P, C = L->noc, n = C * P * P, nop = L->nop, lb = -P / 2, ub = P / 2 - 1;
  const float minerrval = 2.0f;
  int px, py, t, c, k;
  for (px = 0; px < L->nopw; ++px)
    for (py = 0; py < L->noph; ++py) {
      const int ip = px * L->noph + py;
      const float refx = (float)(px * L->steps + L->offw), refy = (float)(py * L->steps + L->offh);
      /* GetPointPos() == pt_iter == pt_ref + p_iter (patch.cpp:214-221; stereo keeps the row) */
      const float rpx = refx + cg_p[ip * nop], rpy = (nop == 2) ? refy + cg_p[ip * nop + 1] : refy;
      const int pos0 = (int)ceil(rpx + .00001), pos1 = (int)ceil(rpy + .00001); /* double literal: patchgrid.cpp:308-309 */
      const int pos2 = (int)floorf(rpx), pos3 = (int)floorf(rpy);
      float wbil[4], r0, r1;
      int x0, x1, y0;
      if (xi < pos0 + lb - 1 || xi > pos0 + ub || yi < pos1 + lb - 1 || yi > pos1 + ub) continue;
      r0 = rpx - pos2;
      r1 = rpy - pos3;
      wbil[0] = r0 * r1;
      wbil[1] = (1 - r0) * r1;
      wbil[2] = r0 * (1 - r1);
      wbil[3] = (1 - r0) * (1 - r1);
      /* in-image rectangle of this patch (the reference's test xt>=1, yt>=1, xt<w-1, yt<h-1), patch coordinates */
      x0 = 1 - pos0 - lb; if (x0 < 0) x0 = 0;
      x1 = L->w - 2 - pos0 - lb; if (x1 > P - 1) x1 = P - 1;
      y0 = 1 - pos1 - lb; if (y0 < 0) y0 = 0;
      for (t = 0; t < 4; ++t) {
        const int xt = xi + (t & 1), yt = yi + (t >> 1);
        const int rx = xt - pos0 - lb, ry = yt - pos1 - lb; /* pixel inside the patch, 0..P-1 */
        const float* pw;
        float absw;
        if (rx < 0 || rx > P - 1 || ry < 0 || ry > P - 1) continue;
        if (!(xt >= 1 && yt >= 1 && xt < L->w - 1 && yt < L->h - 1)) continue;
        /* weight cursor: +1 per pixel, +(C-1) more per in-image pixel before this one (patchgrid.cpp:331-339) */
        pw = cg_pweight + (size_t)ip * n + (ry * P + rx) + (C - 1) * ((ry - y0) * (x1 - x0 + 1) + (rx - x0));
        if (C == 1)
          absw = 1.0f / STD_MAX(minerrval, pw[0]);
        else {
          absw = STD_MAX(minerrval, pw[0]);
          for (c = 1; c < C; ++c) absw += STD_MAX(minerrval, pw[c]);
          absw = 1.0f / absw;
        }
        *we += wbil[t] * absw;
        for (k = 0; k < nop; ++k) acc[k] -= wbil[t] * (cg_p[ip * nop + k] * absw);
      }
    }
}

/* AggregateFlowDense with the forward-backward merge (usefbcon): own patches, then the
 * complementary grid's, then the normalisation (patchgrid.cpp:213-394). */
void dis_densify_fb(const dis_level* L, const dis_params* prm, const float* p, const float* pweight,
                    const float* cg_p, const float* cg_pweight, float* flow_out) {
  const int P = L->P, C = L->noc, n = C * P * P, nop = L->nop;
  const float minerrval = 2.0f;
  int xi, yi, px, py, c, k;
  (void)prm;
  for (yi = 0; yi < L->h; ++yi)
    for (xi = 0; xi < L->w; ++xi) {
      float we = 0, acc[2] = {0, 0};
      for (px = 0; px < L->nopw; ++px) {
        int dx = xi - (px * L->steps + L->offw);
        if (dx < -P / 2 || dx > P / 2 - 1) continue;
        for (py = 0; py < L->noph; ++py) {
          int dy = yi - (py * L->steps + L->offh), ip = px * L->noph + py;
          const float* pw;
          float absw;
          if (dy < -P / 2 || dy > P / 2 - 1) continue;
          {
            int rx = dx + P / 2, ry = dy + P / 2, cx = px * L->steps + L->offw, cy = py * L->steps + L->offh;
            int x0 = cx - P / 2 < 0 ? P / 2 - cx : 0, y0 = cy - P / 2 < 0 ? P / 2 - cy : 0;
            int x1 = cx + P / 2 - 1 > L->w - 1 ? L->w - 1 - cx + P / 2 : P - 1;
            int inb = (ry - y0) * (x1 - x0 + 1) + (rx - x0);
            pw = pweight + (size_t)ip * n + (ry * P + rx) + (C - 1) * inb;
          }
          if (C == 1)
            absw = 1.0f / STD_MAX(minerrval, pw[0]);
          else {
            absw = STD_MAX(minerrval, pw[0]);
            for (c = 1; c < C; ++c) absw += STD_MAX(minerrval, pw[c]);
            absw = 1.0f / absw;
          }
          we += absw;
          for (k = 0; k < nop; ++k) acc[k] += p[ip * nop + k] * absw;
        }
      }
      if (cg_p) densify_cg_cell(L, cg_p, cg_pweight, xi, yi, &we, acc);
      for (k = 0; k < nop; ++k) flow_out[(yi * L->w + xi) * nop + k] = we > 0 ? acc[k] / we : acc[k];
    }
}

/* OFClass::OFClass level loop (oflow.cpp:184-295) including the forward-backward variant:
 * a second grid on the swapped images (camlr = 1), merged at every densification; the backward
 * flow is densified and refined on all but the last level. */
int dis_run_fb(const float** i0, const float** i0x, const float** i0y, const float** i1, const float** i1x,
               const float** i1y, int pad, float* outflow, const float* initflow, int width, int height,
               const dis_params* prm, int nop) {
  float *prev = NULL, *prev_bw = NULL;
  const int fb = prm->usefbcon != 0;
  int sl;
  if (fb && (!i1x || !i1y)) return -1;
  for (sl = prm->sc_f; sl >= prm->sc_l; --sl) {
    dis_level L, Lb;
    int np, n;
    float *p, *pw, *cur, *pb = NULL, *pwb = NULL, *cur_bw = NULL;
    dis_make_level(&L, width, height, sl, pad, prm, nop, 0);
    dis_make_level(&Lb, width, height, sl, pad, prm, nop, 1);
    np = L.nopw * L.noph;
    n = L.noc * L.P * L.P;
    p = (float*)malloc(sizeof(float) * np * nop);
    pw = (float*)malloc(sizeof(float) * (size_t)np * n);
    cur = (sl == prm->sc_l) ? outflow : (float*)malloc(sizeof(float) * L.w * L.h * nop);
    dis_patches_level(&L, prm, i0[sl], i0x[sl], i0y[sl], i1[sl], sl < prm->sc_f ? prev : initflow, p, pw, NULL, NULL);
    if (fb) {
      pb = (float*)malloc(sizeof(float) * np * nop);
      pwb = (float*)malloc(sizeof(float) * (size_t)np * n);
      dis_patches_level(&Lb, prm, i1[sl], i1x[sl], i1y[sl], i0[sl], sl < prm->sc_f ? prev_bw : NULL, pb, pwb, NULL,
                        NULL);
    }
    dis_densify_fb(&L, prm, p, pw, pb, pwb, cur);
    if (fb && sl > prm->sc_l) {
      cur_bw = (float*)malloc(sizeof(float) * L.w * L.h * nop);
      dis_densify_fb(&Lb, prm, pb, pwb, p, pw, cur_bw);
    }
    if (prm->usetvref) {
      dis_varref_level(&L, prm, i0[sl], i1[sl], cur);
      if (cur_bw) dis_varref_level(&Lb, prm, i1[sl], i0[sl], cur_bw);
    }
    free(p);
    free(pw);
    free(pb);
    free(pwb);
    free(prev);
    free(prev_bw);
    prev = (sl == prm->sc_l) ? NULL : cur;
    prev_bw = cur_bw;
  }
  free(prev_bw);
  return 0;
}

int dis_run(const float** i0, const float** i0x, const float** i0y, const float** i1, int pad,
            float* outflow, const float* initflow, int width, int height, const dis_params* prm,
            int nop) {
  if (prm->usefbcon) return -1; /* needs the gradients of the second image: dis_run_fb */
  return dis_run_fb(i0, i0x, i0y, i1, NULL, NULL, pad, outflow, initflow, width, height, prm, nop);
}

/* oracle/dis_oracle.h -- CPU restatement of the DIS hot path (TEST INFRASTRUCTURE ONLY).
 *
 * Plain scalar C, one pixel / one patch at a time, written in the per-element
 * form the CUDA kernels use.  It is the checker for tests/, smoke() and the
 * "port" CPU baseline of bench.py; the product never links or imports it.
 *
 * Pinned: tests/test_oracle.py requires BITWISE equality with
 * oracle/_ref (the reference's own sources compiled in place) on every stage
 * and on whole runs; small golden fixtures of those runs live in tests/golden/.
 * Unpinned boundary: Eigen's reduction order (see oracle/eigen_shim/Eigen/Core).
 */
#ifndef DIS_ORACLE_H
#define DIS_ORACLE_H

#ifdef __cplusplus
extern "C" {
#endif

/* same binary layout as ofdis_params (include/ofdis_b200.h) */
typedef struct dis_params {
  int sc_f, sc_l, max_iter, min_iter;
  float dp_thresh, dr_thresh, res_thresh;
  int p_samp_s;
  float patove;
  int usefbcon, costfct, noc, patnorm, usetvref;
  float tv_alpha, tv_gamma, tv_delta;
  int tv_innerit, tv_solverit;
  float tv_sor;
  int verbosity;
} dis_params;

/* level geometry (oflow.cpp:91,142-151; patchgrid.cpp:42-48) */
typedef struct dis_level {
  int w, h, pad, tmp_w, noc, nop, P, steps, nopw, noph, offw, offh, level, camlr;
  float lb, ubw, ubh, outlierthresh;
} dis_level;

void dis_make_level(dis_level* L, int width_full, int height_full, int level, int pad,
                    const dis_params* p, int nop, int camlr);

/* Eigen-3.3/SSE packet-order sum of n floats (see eigen_shim/Eigen/Core). */
float dis_sum_packet_order(const float* v, int n);

/* K1+K2+K3: template/Hessian, init from coarser flow (nullable), GN iterations.
 * Outputs (any may be NULL): p_out[np*nop], pweight_out[np*novals], conv_out[np], cnt_out[np]. */
int dis_patches_level(const dis_level* L, const dis_params* prm, const float* i0, const float* i0x,
                      const float* i0y, const float* i1, const float* flow_prev, float* p_out,
                      float* pweight_out, int* conv_out, int* cnt_out);

/* Data-dependent fallbacks of PatClass::ComputeHessian + Eigen LLT (patch.cpp:71-88), as bits:
 * flow, det H == 0 with H00 == 0 / with H00 > 0 (both diagonals get +1e-10); flow, the Cholesky pivot
 * H11 - L10^2 <= 0 (L11 keeps H11); stereo, H00 == 0. */
#define DIS_HESS_SINGULAR_ZERO 1
#define DIS_HESS_SINGULAR 2
#define DIS_HESS_NOT_PD 4
#define DIS_HESS_STEREO_ZERO 8

/* Test query, no result of the run depends on it: for every patch of the level (ip order) the
 * DIS_HESS_* bits its Hessian took into branch_out[np].  Returns np. */
int dis_patches_level_branches(const dis_level* L, const dis_params* prm, const float* i0, const float* i0x,
                               const float* i0y, int* branch_out);

/* K4: densification (patchgrid.cpp:213-275,377-394). flow_out[h*w*nop] interleaved. */
void dis_densify(const dis_level* L, const dis_params* prm, const float* p, const float* pweight,
                 float* flow_out);

/* K5-K12 pieces on planar w*h arrays (pitch == w). */
void dis_warp(const dis_level* L, const float* i1_padded, const float* wx, const float* wy,
              float* warped /*noc planes*/, float* mask);
void dis_derivatives(const dis_level* L, const float* i0_padded, const float* warped, float* Ix,
                     float* Iy, float* Iz, float* Ixx, float* Ixy, float* Iyy, float* Ixz, float* Iyz);
void dis_smoothness(int w, int h, const float* uu, const float* vv, float quarter_alpha, float* sh,
                    float* sv);
void dis_data_term(const dis_level* L, const float* mask, const float* du, const float* dv,
                   const float* Ix, const float* Iy, const float* Iz, const float* Ixx,
                   const float* Ixy, const float* Iyy, const float* Ixz, const float* Iyz,
                   float half_delta_over3, float half_gamma_over3, float* a11, float* a12, float* a22,
                   float* b1, float* b2);
void dis_sub_laplacian(int w, int h, float* b, const float* src, const float* sh, const float* sv);
/* sor_coupled (solver.c:77-421): inverts the 2x2 blocks in place on sweep 1 */
void dis_sor_coupled(int w, int h, float* du, float* dv, float* a11, float* a12, float* a22,
                     const float* b1, const float* b2, const float* sh, const float* sv, int iterations,
                     float omega);
/* sor_coupled_slow_but_readable_DE (solver.c:428-466) */
void dis_sor_de(int w, int h, float* du, const float* a11, const float* b1, const float* sh,
                const float* sv, int iterations, float omega);

/* One level of variational refinement in place on flow[h*w*nop] (refine_variational.cpp:25-116). */
void dis_varref_level(const dis_level* L, const dis_params* prm, const float* i0, const float* i1,
                      float* flow);

/* K4 with the forward-backward merge (patchgrid.cpp:213-394): cg_p / cg_pweight are the complementary
 * grid's results (NULL: no merge, == dis_densify). */
void dis_densify_fb(const dis_level* L, const dis_params* prm, const float* p, const float* pweight,
                    const float* cg_p, const float* cg_pweight, float* flow_out);

/* Whole run including usefbcon (second grid on the swapped images; needs i1x, i1y). */
int dis_run_fb(const float** i0, const float** i0x, const float** i0y, const float** i1, const float** i1x,
               const float** i1y, int pad, float* outflow, const float* initflow, int width, int height,
               const dis_params* prm, int nop);

/* Whole coarse-to-fine run == OFClass ctor (oflow.cpp:32-363), usefbcon must be 0. */
int dis_run(const float** i0, const float** i0x, const float** i0y, const float** i1, int pad,
            float* outflow, const float* initflow, int width, int height, const dis_params* prm,
            int nop);

#ifdef __cplusplus
}
#endif
#endif

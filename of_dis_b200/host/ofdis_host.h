// Host-side C++ mirror of the reference's three classes, implemented on the
// C-ABI of libofdis_b200 (include/ofdis_b200.h).  Same namespace, names,
// argument order and argument meaning as
//   OFC::OFClass       oflow.h:84-111
//   OFC::PatGridClass  patchgrid.h:19-44
//   OFC::VarRefClass   refine_variational.h:37-39
// so a caller written against the reference (run_dense.cpp:391-400) compiles
// unchanged.  Differences by design: SELECTMODE / SELECTCHANNEL are run-time
// (optparam::nop / optparam::noc), Eigen::Vector2f is replaced by a 2-float POD,
// and failures throw std::runtime_error instead of exit(1) (image.c:17-28).
#ifndef OFDIS_HOST_H
#define OFDIS_HOST_H

#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ofdis_b200.h"

namespace OFC {

struct Vector2f {
  float v[2];
  float& operator[](int i) { return v[i]; }
  const float& operator[](int i) const { return v[i]; }
  Vector2f operator-(const Vector2f& o) const { return Vector2f{{v[0] - o.v[0], v[1] - o.v[1]}}; }
  Vector2f operator+(const Vector2f& o) const { return Vector2f{{v[0] + o.v[0], v[1] + o.v[1]}}; }
};

// oflow.h:16-29
typedef struct {
  int width, height, imgpadding;
  float tmp_lb, tmp_ubw, tmp_ubh;
  int tmp_w, tmp_h;
  float sc_fct;
  int curr_lv;
  int camlr;
} camparam;

// oflow.h:31-76 (without the SSE helper vectors)
typedef struct {
  int sc_f, sc_l, p_samp_s, max_iter, min_iter;
  float dp_thresh;  // squared, as OFClass stores it (oflow.cpp:88)
  float dr_thresh, res_thresh;
  int patnorm, verbosity;
  bool usefbcon;
  int costfct;
  bool usetvref;
  float tv_alpha, tv_gamma, tv_delta;
  int tv_innerit, tv_solverit;
  float tv_sor;
  int nop;
  float patove, outlierthresh;
  int steps, novals, noc, noscales;
  float minerrval = 2.0f;
  float normoutlier = 5.0f;
} optparam;

// Fills optparam / per-level camparam exactly as OFClass does (oflow.cpp:76-108,138-157).
void FillOptParam(optparam& op, int nop, int sc_f, int sc_l, int max_iter, int min_iter, float dp_thresh,
                  float dr_thresh, float res_thresh, int p_samp_s, float patove, bool usefbcon, int costfct,
                  int noc, int patnorm, bool usetvref, float tv_alpha, float tv_gamma, float tv_delta,
                  int tv_innerit, int tv_solverit, float tv_sor, int verbosity);
void FillCamParam(camparam& cp, const optparam& op, int width_full, int height_full, int level, int imgpadding,
                  int camlr);

class OFClass {
 public:
  // oflow.h:84-111; `nop_in` (2 flow / 1 stereo) replaces the compile-time SELECTMODE.
  OFClass(const float** im_ao_in, const float** im_ao_dx_in, const float** im_ao_dy_in,
          const float** im_bo_in, const float** im_bo_dx_in, const float** im_bo_dy_in, const int imgpadding_in,
          float* outflow, const float* initflow, const int width_in, const int height_in, const int sc_f_in,
          const int sc_l_in, const int max_iter_in, const int min_iter_in, const float dp_thresh_in,
          const float dr_thresh_in, const float res_thresh_in, const int padval_in, const float patove_in,
          const bool usefbcon_in, const int costfct_in, const int noc_in, const int patnorm_in,
          const bool usetvref_in, const float tv_alpha_in, const float tv_gamma_in, const float tv_delta_in,
          const int tv_innerit_in, const int tv_solverit_in, const float tv_sor_in, const int verbosity_in,
          const int nop_in = 2, const int device = 0);
  // Extension (SURVEY 8f rank 1-2): 8-bit frames ([height_org][width_org][noc]) in, flow of the
  // original frame size out; divisibility padding, pyramid, gradients, border padding, x2^sc_l
  // upsampling and crop (run_dense.cpp:130-178,298-311,407-414) run on the device.  `initflow` keeps the
  // reference's meaning (level sc_f+1); `initflow_fullres` ([height_org][width_org][nop]) is instead a flow of the
  // original frame size, prepared on the device like run_dense.cpp:355-378 (ofdis_set_initflow_fullres) -- the
  // frames are then padded to multiples of 2^(sc_f+1).
  OFClass(const unsigned char* frame_ao, const unsigned char* frame_bo, const int width_org, const int height_org,
          float* outflow_fullres, const float* initflow, const int sc_f_in, const int sc_l_in, const int max_iter_in,
          const int min_iter_in, const float dp_thresh_in, const float dr_thresh_in, const float res_thresh_in,
          const int padval_in, const float patove_in, const bool usefbcon_in, const int costfct_in, const int noc_in,
          const int patnorm_in, const bool usetvref_in, const float tv_alpha_in, const float tv_gamma_in,
          const float tv_delta_in, const int tv_innerit_in, const int tv_solverit_in, const float tv_sor_in,
          const int verbosity_in, const int nop_in = 2, const int device = 0, const float* initflow_fullres = nullptr);
};

class PatGridClass {
 public:
  PatGridClass(const camparam* cpt_in, const camparam* cpo_in, const optparam* op_in, int device = 0);
  ~PatGridClass();
  void InitializeGrid(const float* im_ao_in, const float* im_ao_dx_in, const float* im_ao_dy_in);
  void SetTargetImage(const float* im_bo_in, const float* im_bo_dx_in, const float* im_bo_dy_in);
  void InitializeFromCoarserOF(const float* flow_prev);
  void AggregateFlowDense(float* flowout) const;
  void Optimize();
  // patchgrid.h:36: joins this grid and `cg_in` (the grid on the swapped images) so that
  // AggregateFlowDense merges the complementary grid's flow (patchgrid.cpp:278-375).  Both grids
  // then live in one two-direction engine context; call it on both objects like oflow.cpp:166-170.
  void SetComplGrid(PatGridClass* cg_in);
  inline int GetNoPatches() const { return nopatches; }
  inline int GetNoph() const { return noph; }
  inline int GetNopw() const { return nopw; }
  Vector2f GetRefPatchPos(int i) const;
  Vector2f GetQuePatchPos(int i) const;
  Vector2f GetQuePatchDis(int i) const;

 private:
  void fetch() const;
  void select() const;   // couple: address this grid's direction in the shared context
  void flush();          // couple: upload both grids' images once both are bound
  struct Couple {         // two grids joined by SetComplGrid share one usefbcon context
    ofdis_ctx* ctx = nullptr;
    PatGridClass* grid[2] = {nullptr, nullptr};
    bool uploaded = false;
    ~Couple();
  };
  std::shared_ptr<Couple> couple;
  int role = 0;          // 0 = forward grid of the couple, 1 = backward
  const float *tgt = nullptr;
  int device_id = 0;
  const camparam* cpt;
  const optparam* op;
  ofdis_ctx* ctx = nullptr;
  const float *i0 = nullptr, *i0x = nullptr, *i0y = nullptr;
  bool from_coarser = false;
  int steps, nopw, noph, nopatches, offw, offh;
  mutable std::vector<float> p_host;
  mutable bool fetched = false;
};

class VarRefClass {
 public:
  // refine_variational.h:37-39: refines `flowout` in place.
  VarRefClass(const float* im_ao_in, const float* im_ao_dx_in, const float* im_ao_dy_in, const float* im_bo_in,
              const float* im_bo_dx_in, const float* im_bo_dy_in, const camparam* cpt_in, const camparam* cpo_in,
              const optparam* op_in, float* flowout, int device = 0);
};

}  // namespace OFC

#endif

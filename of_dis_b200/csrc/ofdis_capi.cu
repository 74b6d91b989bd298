// C-ABI of libofdis_b200 (include/ofdis_b200.h): context, device workspaces,
// level loop (OFClass::OFClass, oflow.cpp:76-108,138-157,184-295) and transfers.
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <climits>
#include <cstdint>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "../../include/ofdis_b200.h"
#include "ofdis_internal.cuh"

using namespace ofdis;

// A lazily allocated device buffer that only grows (the workspaces of the stages outside ofdis_run)
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  // at least n bytes: nothing when the buffer holds them, else the stream synchronised, the old buffer freed and a new
  // one allocated; on failure p is null, bytes 0, and the error OFDIS_ERR_NOMEM with `what`
  int reserve(ofdis_ctx* ctx, size_t n, const char* what);
};

// Hands out consecutive typed arrays of a workspace, each on a 16-byte boundary.  Without a base it only counts, so
// one layout function both sizes a workspace (size()) and places its arrays; offsets stay integers until placed.
struct Carve {
  char* base = nullptr;
  size_t off = 0;
  template <class T>
  T* take(size_t count) {
    const size_t at = (off + 15) & ~(size_t)15;
    off = at + sizeof(T) * count;
    return base ? reinterpret_cast<T*>(base + at) : nullptr;
  }
  // the same room, but null unless `want`: an output a call does not ask for keeps its place in the layout
  template <class T>
  T* take(size_t count, bool want) {
    T* p = take<T>(count);
    return want ? p : nullptr;
  }
  size_t size() const { return (off + 15) & ~(size_t)15; }
};

struct ofdis_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  ofdis_params prm{};
  int nop = 2, width = 0, height = 0, pad = 0, max_frames = 0;
  // usefbcon: every pair occupies two internal frames (2*f forward, 2*f+1 the grid on the swapped
  // images); dirs = 2, cap = max_frames * dirs internal frames are allocated
  int dirs = 1, cap = 0;
  int last_vr_fstep = 1;
  int sel_dir = -1;                // ofdis_set_direction: -1 = both directions / the forward grid
  // SOR options (sor_plan).  max_cluster: 8 = portable limit, 16 where the device grants it (sor_dev_cluster); rt:
  // set in ofdis_create.  lane: pixel wavefront (sor_lane_kernel) instead of the block wavefront on levels of few
  // 32-row bands, 0 never, 1 always, 2 (default) for launches of up to SOR_LANE_AUTO_FRAMES frames on levels of one
  // or two bands: there it is faster per launch (H100, 700 W, one stream, operating point 2: 1 pair 0.344 vs 0.456 ms
  // per step, 8 pairs 0.365 vs 0.470 ms), but it needs 200 KB of shared memory per CTA at 56-row levels (one CTA per
  // SM), which costs 10-13 % of throughput when ten streams of 32 or 64 frames overlap (bench.py `value`)
  SorOptions sor{/*lane*/ 2, /*fast*/ 0, /*rt*/ 1, /*single_max*/ 128, /*max_cluster*/ 8};
  int sor_dev_cluster = 8;
  SorPlan last_sor{};  // plan of the last refinement (ofdis_debug_get decodes its planes)
  // programmatic dependent launch of the level loop's kernels (pdl_wait, ofdis_internal.cuh): 0 never, 1 always,
  // 2 (default) for launches of up to SOR_LANE_AUTO_FRAMES frames: H100, one stream, graph replay: 1 pair
  // 0.374 -> 0.344 ms, 8 pairs 0.390 -> 0.363 ms; 64 pairs 0.659 -> 0.690 ms, and 5-14 % less throughput when ten
  // streams of 32 or 64 frames overlap (waiting CTAs of the next kernel take SM slots from the tail of the current one)
  int pdl = 2;
  // lanes per patch of the P = 8 gray patch kernel (patch_p8c1_kernel): 8 or 4, 0 (default) = 4 for launches of more
  // than SOR_LANE_AUTO_FRAMES frames, 8 below (DESIGN.md section 5.9)
  int patch_lanes = 0;
  int nlev = 0;                   // sc_f - sc_l + 1
  std::vector<LevelGeom> lev;      // index: level - sc_l
  std::vector<size_t> img_off;     // [lev][4] offsets (floats) inside one packed frame
  size_t frame_floats = 0;
  size_t images_floats = 0;        // leading part of a packed frame that holds I0,I1 of all levels
  float* d_img = nullptr;          // [max_frames][frame_floats]
  // swapped marks (ofdis_set_swapped_slots), one byte per internal frame, in the same allocation right in front of
  // d_img (LevelGeom::swap_off); this is the pointer the allocation is freed by
  unsigned char* d_swapped = nullptr;
  // The workspaces below (DevBuf) are lazily allocated and never touched by ofdis_run.
  // staging of host inputs (ofdis_upload_frames_u8, ofdis_upload_finest_level, ...) and the scratch of host outputs
  // (ofdis_get_flow_fullres, ...)
  DevBuf d_stage, d_full;
  // ofdis_flow_error_fullres: the row partials [max_frames][16][height], then the device stats [max_frames][16]
  DevBuf d_eval;
  // ofdis_flow_color_fullres: the automatic scales' maxima [max_frames] as float bit patterns
  DevBuf d_color;
  // ofdis_interpolate_fullres (InterpWork for max_frames pairs of width x height pixels)
  DevBuf d_interp;
  InterpWork interp{};
  // the tracker of ofdis_track_begin / ofdis_track_advance: its workspace (TrackWork, then the host-output records of
  // max_frames pairs), the geometry of the last begin and the list that holds the live tracks
  DevBuf d_track;
  TrackWork track{};
  ofdis_track_point* track_out = nullptr;
  TrackGeom tgeom{};
  int track_cur = 0;
  bool track_on = false;
  // the descriptor stage of ofdis_traj_begin / ofdis_traj_advance on top of the tracker: its workspace (TrajWork, then
  // the host-output records and descriptors of max_frames pairs), the geometry of the last begin and the frames seen
  // since it; ended by ofdis_track_begin and ofdis_track_advance
  DevBuf d_traj;
  TrajWork traj{};
  TrajGeom trgeom{};
  ofdis_traj_record* traj_rec = nullptr;
  float* traj_desc = nullptr;
  int traj_frame = 0;
  bool traj_on = false;
  // ofdis_disparity_fullres (DispWork for max_frames pairs of width x height pixels)
  DevBuf d_disp;
  // ofdis_scene_flow_fullres's counters ([max_frames][16] ofdis_sf_stats)
  DevBuf d_sf;
  // ofdis_global_motion_fullres (MotionWork for max_frames pairs of motion_cells cells and motion_hyps hypotheses)
  DevBuf d_motion;
  size_t motion_cells = 0, motion_hyps = 0;
  MotionWork motion{};
  // ofdis_egomotion_fullres (EgoWork for max_frames pairs of ego_cells cells and ego_hyps hypotheses)
  DevBuf d_ego;
  size_t ego_cells = 0, ego_hyps = 0;
  EgoWork ego{};
  // ofdis_relpose_fullres (global motion's MotionWork layout with float64 E per hypothesis and RELPOSE_NE chunk sums,
  // then the RelposeOut records, for max_frames pairs of relpose_cells cells and relpose_hyps hypotheses)
  DevBuf d_relpose;
  size_t relpose_cells = 0, relpose_hyps = 0;
  MotionWork relpose{};
  RelposeOut* relpose_out = nullptr;
  // the stabiliser of ofdis_stab_begin / ofdis_stab_push / ofdis_stab_finish: its workspace (StabWork: the frame ring,
  // the model ring, the per-frame records), the geometry and weights of the last begin, L and the next frame to emit
  DevBuf d_stab;
  StabWork stab{};
  StabGeom sgeom{};
  long long stab_last = 0, stab_next = 0;
  bool stab_on = false;
  // the Fisher encoder of ofdis_fisher_begin / ofdis_fisher_push / ofdis_fisher_take: its workspace (FisherWork), the
  // geometry of the last begin and the descriptors pushed since it or the last take
  DevBuf d_fisher;
  FisherWork fisher{};
  FisherGeom fgeom{};
  long long fisher_pushed = 0;
  bool fisher_on = false;
  // the volume of ofdis_fuse_begin / ofdis_fuse_push / ofdis_fuse_extract / ofdis_fuse_render: T, W, the colour bytes,
  // then FuseWork's poses and scan blocks; the geometry of the last begin
  DevBuf d_fuse;
  FuseGeom fuse_geom{};
  FuseVolume fuse_vol{};
  FuseWork fuse_ws{};
  bool fuse_on = false;
  // ofdis_fuse_mesh (FuseMeshWork: the per-voxel first vertex indices, the second scan blocks and their total)
  DevBuf d_mesh;
  // ofdis_fuse_track (the pose chain's state, motions, poses and stats, the push pose, then the chunk sums)
  DevBuf d_ftrack;
  std::vector<float*> d_flow;   // index level - sc_l, plus one extra entry for level sc_f+1 (initflow)
  std::vector<size_t> flow_floats;
  VarRefPlanes planes{};
  float* d_planes = nullptr;
  float* d_fast = nullptr;          // fast-mode records and (du,dv) ping-pong planes (ofdis_set_option "sor_fast")
  int* d_chain = nullptr;           // SOR chain: ticket counter + progress words [frame][band], zero between launches
  size_t rec_f4 = 0;                // float4 per frame of the SOR's lane rows in d_planes
  int chain_nb = 0;                 // bands per frame d_chain holds
  unsigned long long* d_div_fb = nullptr;  // stereo SOR work redone with the plain division (ofdis_debug_sor_div_fallbacks)
  int last_vr_fcur = 0;
  PatchParams pp{};
  long launches = 0;
  int last_vr_level = -1, last_vr_f0 = 0;
  bool graph_mode = false;
  Profiler* prof = nullptr;         // non-null only inside ofdis_profile_run
  std::map<long, cudaGraphExec_t> graphs;
  std::map<long, long> graph_launches;
  std::string err;
};

namespace {

// NVTX range per stage and level ("patch L3", "densify L3", "varref L3", "pyramid", "upsample"): free
// when no profiler is attached, names the stages in Nsight Systems / ncu --nvtx timelines.
struct NvtxRange {
  NvtxRange(const char* stage, int level) {
    char name[48];
    if (level >= 0) snprintf(name, sizeof(name), "ofdis %s L%d", stage, level);
    else snprintf(name, sizeof(name), "ofdis %s", stage);
    nvtxRangePushA(name);
  }
  ~NvtxRange() { nvtxRangePop(); }
};

int fail(ofdis_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess) {
  if (c) {
    c->err = what;
    if (e != cudaSuccess) {
      c->err += ": ";
      c->err += cudaGetErrorString(e);
    }
  }
  return code;
}

#define CK(call)                                                        \
  do {                                                                  \
    cudaError_t e__ = (call);                                           \
    if (e__ != cudaSuccess) return fail(ctx, OFDIS_ERR_CUDA, #call, e__); \
  } while (0)

// ofdis_debug_div: the stereo SOR's division helpers (ofdis_internal.cuh), exactly as the SOR kernels call them
__global__ void debug_div_kernel(const float* a, const float* b, long n, float* q_fast, float* q_plain,
                                 unsigned char* unsafe) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float A = a[i], B = b[i];
  q_fast[i] = fdiv_quot(A, B, fdiv_rcp(A));
  q_plain[i] = B / A;
  unsafe[i] = fdiv_unsafe(A, B) ? 1 : 0;
}

// camparam / optparam derivation (oflow.cpp:81-92,142-157; patchgrid.cpp:42-48)
void make_level(LevelGeom& L, const ofdis_ctx* c, int sl) {
  const ofdis_params& p = c->prm;
  const float sc_fct = (float)pow(2, -sl);
  L.h = (int)(c->height * sc_fct);
  L.w = (int)(c->width * sc_fct);
  L.pad = c->pad;
  L.tmp_w = L.w + 2 * c->pad;
  L.tmp_h = L.h + 2 * c->pad;
  L.noc = p.noc;
  L.nop = c->nop;
  L.P = p.p_samp_s;
  L.novals = p.noc * p.p_samp_s * p.p_samp_s;
  L.steps = (int)floor(p.p_samp_s * (1 - p.patove));
  if (L.steps < 1) L.steps = 1;
  L.nopw = (int)ceil((float)L.w / (float)L.steps);
  L.noph = (int)ceil((float)L.h / (float)L.steps);
  L.np = L.nopw * L.noph;
  L.offw = (L.w - (L.nopw - 1) * L.steps) / 2;
  L.offh = (L.h - (L.noph - 1) * L.steps) / 2;
  L.level = sl;
  L.camlr = 0;
  L.swap_off = 0;
  L.pitch = ((L.w + 3) / 4) * 4;
  L.lb = -(float)p.p_samp_s / 2;
  L.ubw = (float)(L.w + p.p_samp_s / 2 - 2);
  L.ubh = (float)(L.h + p.p_samp_s / 2 - 2);
  L.outlierthresh = (float)p.p_samp_s / 2;
  L.pat_p = L.pat_w = nullptr;
  L.pat_conv = L.pat_cnt = nullptr;
  L.fb = 0;
  L.fstep = 1;
  L.fb_pos = nullptr;
  L.fb_wbil = nullptr;
  L.fb_reach = nullptr;
}

// programmatic dependent launch for a launch of `frames` internal frames (ofdis_set_option "pdl")
int pdl_for(const ofdis_ctx* c, int frames) { return c->pdl == 1 || (c->pdl == 2 && frames <= SOR_LANE_AUTO_FRAMES) ? 1 : 0; }

// lanes per patch of patch_p8c1_kernel for a launch of `frames` internal frames (ofdis_set_option "patch_lanes")
int patch_lanes_for(const ofdis_ctx* c, int frames) {
  if (c->patch_lanes) return c->patch_lanes;
  return frames > SOR_LANE_AUTO_FRAMES ? 4 : 8;
}

LevelGeom* level_of(ofdis_ctx* c, int level) {
  if (level < c->prm.sc_l || level > c->prm.sc_f) return nullptr;
  return &c->lev[level - c->prm.sc_l];
}

// copy of a level's geometry whose launches address every `fstep`-th internal frame
LevelGeom stepped(const LevelGeom& L, int fstep) {
  LevelGeom g = L;
  g.fstep = fstep;
  return g;
}

cudaMemcpyKind kind_in(int memkind) { return memkind == OFDIS_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice; }
cudaMemcpyKind kind_out(int memkind) { return memkind == OFDIS_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost; }

int run_levels(ofdis_ctx* ctx, int nframes, int use_initflow) {
  for (int sl = ctx->prm.sc_f; sl >= ctx->prm.sc_l; --sl) {
    const bool from_coarser = (sl < ctx->prm.sc_f) || use_initflow;
    if (ctx->prof) ctx->prof->level = sl;
    int rc = ofdis_patgrid_optimize(ctx, sl, 0, nframes, from_coarser ? 1 : 0);
    if (rc) return rc;
    rc = ofdis_patgrid_aggregate(ctx, sl, 0, nframes);
    if (rc) return rc;
    if (ctx->prm.usetvref) {
      rc = ofdis_varref_refine(ctx, sl, 0, nframes);
      if (rc) return rc;
    }
  }
  return OFDIS_OK;
}

// Float4 per frame of the SOR's lane rows and most bands of a chain that the plans (sor_plan) of every level need,
// over sor_single_max, sor_rows_per_thread and sor_lane with sor_max_cluster in mc_lo .. mc_hi (powers of two).
void sor_workspace_need(const ofdis_ctx* c, int mc_lo, int mc_hi, size_t* recf4, int* chain_nb) {
  *recf4 = 0;
  *chain_nb = 0;
  for (const LevelGeom& L : c->lev)
    for (int mc = mc_lo; mc <= mc_hi; mc *= 2)
      for (int sm = 32; sm <= 128; sm *= 2)
        for (int rt = 1; rt <= 4; rt *= 2)
          for (int lane = 0; lane <= 1; ++lane) {
            SorPlan p;
            if (sor_plan(L, c->prm.tv_solverit, SorOptions{lane, 0, rt, sm, mc}, 1, VarRefPlanes{}, &p)) {
              *recf4 = std::max(*recf4, p.pl.rec_stride);
              *chain_nb = std::max(*chain_nb, p.chain_nb);
            }
          }
}

// (Re)allocates the refinement planes of the finest level (mask, 8 x deriv[C]) behind `recf4` float4 of SOR
// lane rows per frame, and the chain's scratch for `chain_nb` bands per frame; all of it zeroed.  On failure the
// previous buffers stay in place.
bool alloc_refinement(ofdis_ctx* ctx, size_t recf4, int chain_nb) {
  const LevelGeom& Lf = ctx->lev[0];
  const size_t plane = (size_t)Lf.pitch * Lf.h, cap = (size_t)ctx->cap;
  const int C = ctx->prm.noc;
  const size_t per_frame = plane * (1 + 8 * C) + recf4 * 4, chain_ints = 1 + (size_t)chain_nb * cap;
  float* planes = nullptr;
  int* chain = nullptr;
  if (cudaMalloc((void**)&planes, sizeof(float) * per_frame * cap) != cudaSuccess) return false;
  if (cudaMalloc((void**)&chain, sizeof(int) * chain_ints) != cudaSuccess) {
    cudaFree(planes);
    return false;
  }
  if (ctx->d_planes || ctx->d_chain) cudaStreamSynchronize(ctx->stream);  // nothing in flight uses the old buffers
  cudaFree(ctx->d_planes);
  cudaFree(ctx->d_chain);
  ctx->d_planes = planes;
  ctx->d_chain = chain;
  // never-written lane rows (wavefront ramps, padded lanes) are read by idle SOR lanes: keep them finite
  cudaMemsetAsync(planes, 0, sizeof(float) * per_frame * cap, ctx->stream);
  cudaMemsetAsync(chain, 0, sizeof(int) * chain_ints, ctx->stream);
  float* q = planes;
  VarRefPlanes& P = ctx->planes;
  P.rec = reinterpret_cast<float4*>(q); q += recf4 * 4 * cap;   // first (alignment)
  P.mask = q; q += plane * cap;
  for (int k = 0; k < 8; ++k) { P.deriv[k] = q; q += plane * C * cap; }
  P.plane = plane;
  ctx->rec_f4 = recf4;
  ctx->chain_nb = chain_nb;
  return true;
}

}  // namespace

int DevBuf::reserve(ofdis_ctx* ctx, size_t n, const char* what) {
  if (bytes >= n) return OFDIS_OK;
  CK(cudaStreamSynchronize(ctx->stream));
  cudaFree(p);
  p = nullptr;
  bytes = 0;
  if (cudaMalloc(&p, n) != cudaSuccess) {
    p = nullptr;
    return fail(ctx, OFDIS_ERR_NOMEM, what);
  }
  bytes = n;
  return OFDIS_OK;
}

// The bytes of the workspace `layout` lays out
template <class F>
static size_t measure(F&& layout) {
  Carve c;
  layout(c);
  return c.size();
}

// Reserves buf for `layout` and at least `floor` bytes, then has `layout` place its arrays in it
template <class F>
static int carve(ofdis_ctx* ctx, DevBuf& buf, const char* what, F&& layout, size_t floor = 0) {
  const int rc = buf.reserve(ctx, std::max(measure(layout), floor), what);
  if (rc) return rc;
  Carve c{static_cast<char*>(buf.p)};
  layout(c);
  return OFDIS_OK;
}

// The scratch of host outputs for frames of pix pixels: at least the pix * nop * max_frames floats
// ofdis_get_flow_fullres asks for, so that host-memory calls that alternate with it never reallocate
template <class F>
static int carve_full(ofdis_ctx* ctx, size_t pix, F&& layout) {
  return carve(ctx, ctx->d_full, "full-resolution flow buffer", layout,
               sizeof(float) * pix * ctx->nop * (size_t)ctx->max_frames);
}

// The staging of host inputs
template <class F>
static int carve_stage(ofdis_ctx* ctx, F&& layout) {
  return carve(ctx, ctx->d_stage, "staging buffer", layout);
}

// The staging of host 8-bit frames of hwc bytes: at least two frames per pair of max_frames, as the pair upload
// needs, so that the uploads, the tracker, confidence and interpolation never reallocate when they alternate
template <class F>
static int carve_stage_u8(ofdis_ctx* ctx, size_t hwc, F&& layout) {
  return carve(ctx, ctx->d_stage, "staging buffer", layout, hwc * 2 * (size_t)ctx->max_frames);
}

extern "C" {

const char* ofdis_version(void) { return "ofdis_b200 0.1 (sm_90a)"; }

const char* ofdis_last_error(const ofdis_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int ofdis_create(ofdis_ctx** out, int device, void* stream, const ofdis_params* prm, int nop, int width,
                 int height, int imgpadding, int max_frames) {
  if (!out || !prm) return OFDIS_ERR_ARG;
  *out = nullptr;
  if (nop != 1 && nop != 2) return OFDIS_ERR_ARG;
  if (prm->noc != 1 && prm->noc != 3) return OFDIS_ERR_ARG;
  if (prm->sc_l < 0 || prm->sc_f < prm->sc_l || prm->sc_f > 16) return OFDIS_ERR_ARG;
  if (prm->p_samp_s < 2 || (prm->p_samp_s & 1) || (prm->noc * prm->p_samp_s * prm->p_samp_s) % 4) return OFDIS_ERR_ARG;
  if (imgpadding < prm->p_samp_s) return OFDIS_ERR_ARG;  // window of a patch at the bounds must stay inside the padding
  if (width <= 0 || height <= 0 || (width % (1 << prm->sc_f)) || (height % (1 << prm->sc_f))) return OFDIS_ERR_ARG;
  if (max_frames < 1 || prm->max_iter < 0) return OFDIS_ERR_ARG;
  if (prm->usetvref && ((height >> prm->sc_f) < 4 || (width >> prm->sc_f) < 2)) return OFDIS_ERR_ARG;  // image.c:401-434 needs >= 4 rows
  // tallest refinement level: SOR_MAX_ROWS (levels beyond the largest cluster run as a chain of bands)
  if (prm->usetvref && (height >> prm->sc_l) > SOR_MAX_ROWS) return OFDIS_ERR_UNSUPPORTED;
  // launches that put the frames in gridDim.y / .z (at most 65535): the derivative kernels max_frames x dirs x noc,
  // the pyramid kernels 2 x max_frames (both images of a pair), every other one max_frames x dirs or fewer
  if ((long)max_frames * std::max(2, (prm->usefbcon ? 2 : 1) * prm->noc) > OFDIS_MAX_GRID_FRAMES) return OFDIS_ERR_UNSUPPORTED;
  // patches too large for the generic patch kernel's smallest CTA: the library builds for sm_90a only, so its
  // opt-in ceiling is a constant and the refusal needs no device (RGB P >= 32, gray P >= 54)
  size_t patch_smem;
  patch_generic_threads(prm->noc * prm->p_samp_s * prm->p_samp_s, &patch_smem);
  if (patch_smem > SMEM_OPTIN_MAX) return OFDIS_ERR_UNSUPPORTED;

  ofdis_ctx* ctx = new (std::nothrow) ofdis_ctx();
  if (!ctx) return OFDIS_ERR_NOMEM;
  ctx->device = device;
  ctx->prm = *prm;
  ctx->nop = nop;
  ctx->width = width;
  ctx->height = height;
  ctx->pad = imgpadding;
  ctx->max_frames = max_frames;
  ctx->dirs = prm->usefbcon ? 2 : 1;
  ctx->cap = max_frames * ctx->dirs;
  const int cap = ctx->cap;
  ctx->nlev = prm->sc_f - prm->sc_l + 1;
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    delete ctx;
    return OFDIS_ERR_CUDA;
  }
  if (stream) ctx->stream = (cudaStream_t)stream;
  else {
    e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
      delete ctx;
      return OFDIS_ERR_CUDA;
    }
    ctx->own_stream = true;
  }
  if (prm->usetvref) {
    // Defaults (compare with tools/big_configs.py, bench.py --opt): the largest cluster the device grants (an H100
    // grants 16 CTAs), two rows per SOR thread for stereo, one for flow.
    ctx->sor_dev_cluster = sor_max_cluster_size();
    ctx->sor.max_cluster = ctx->sor_dev_cluster;
    ctx->sor.rt = (nop == 1) ? 2 : 1;
  }
  ctx->pp.max_iter = prm->max_iter;
  ctx->pp.min_iter = prm->min_iter;
  ctx->pp.costfct = prm->costfct;
  ctx->pp.patnorm = prm->patnorm;
  ctx->pp.dp_thresh_sq = prm->dp_thresh * prm->dp_thresh;  // oflow.cpp:88
  ctx->pp.dr_thresh = prm->dr_thresh;
  ctx->pp.res_thresh = prm->res_thresh;

  // geometry + packed image layout: per frame, level sc_f down to sc_l, I0 I0x I0y I1
  ctx->lev.resize(ctx->nlev);
  ctx->img_off.resize((size_t)ctx->nlev * 4);
  // packed frame: [for level sc_f..sc_l: I0, I1] then [for level sc_f..sc_l: I0x, I0y].  The image
  // block is contiguous so that ofdis_upload_packed_images can move it with one 2-D copy and derive
  // the gradients on the device.
  size_t off = 0;
  for (int pass = 0; pass < 2; ++pass)
    for (int sl = prm->sc_f; sl >= prm->sc_l; --sl) {
      LevelGeom& L = ctx->lev[sl - prm->sc_l];
      if (pass == 0) make_level(L, ctx, sl);
      const size_t n = (size_t)L.tmp_w * L.tmp_h * L.noc;
      const int which[2][2] = {{0, 3}, {1, 2}};  // pass 0: I0, I1; pass 1: I0x, I0y
      for (int k = 0; k < 2; ++k) {
        ctx->img_off[(size_t)(sl - prm->sc_l) * 4 + which[pass][k]] = off;
        off += (n + 3) / 4 * 4;  // keep every array 16-byte aligned
      }
    }
  ctx->frame_floats = off;
  ctx->images_floats = ctx->img_off[(size_t)(prm->sc_f - prm->sc_l) * 4 + 1];  // first gradient array starts where the images end

  auto dalloc = [&](void** p, size_t bytes) -> bool {
    return cudaMalloc(p, bytes ? bytes : 16) == cudaSuccess;
  };
  // the swapped marks take the first 256 bytes per 256 internal frames of the image allocation (alignment kept)
  const size_t marks = ((size_t)cap + 255) / 256 * 256;
  // LevelGeom::swap_off counts 16-byte units back from a level's I0 (inside the image block): an int reaches 32 GB
  if ((marks + sizeof(float) * ctx->images_floats) / 16 > (size_t)INT_MAX) {
    ofdis_destroy(ctx);
    return OFDIS_ERR_UNSUPPORTED;
  }
  bool ok = dalloc((void**)&ctx->d_swapped, marks + sizeof(float) * ctx->frame_floats * cap);
  if (ok) {
    ctx->d_img = reinterpret_cast<float*>(ctx->d_swapped + marks);
    cudaMemsetAsync(ctx->d_swapped, 0, marks, ctx->stream);
  }
  ctx->d_flow.assign(ctx->nlev + 1, nullptr);
  ctx->flow_floats.assign(ctx->nlev + 1, 0);
  for (int li = 0; li <= ctx->nlev && ok; ++li) {
    const int sl = prm->sc_l + li;
    const size_t n = (size_t)(width >> sl) * (height >> sl) * nop;
    ctx->flow_floats[li] = n;
    ok = dalloc((void**)&ctx->d_flow[li], sizeof(float) * n * cap);
    if (ok) cudaMemsetAsync(ctx->d_flow[li], 0, sizeof(float) * n * cap, ctx->stream);
  }
  for (int li = 0; li < ctx->nlev && ok; ++li) {
    LevelGeom& L = ctx->lev[li];
    // device layout == the packed host frame: [frame][I0,I1 of all levels | I0x,I0y of all levels], so that
    // ofdis_upload_packed is ONE contiguous copy (two 64-row 2-D copies reached 44 of the link's 54 GB/s)
    for (int k = 0; k < 4; ++k) {
      L.img[k] = ctx->d_img + ctx->img_off[(size_t)li * 4 + k];
      L.img_fs[k] = ctx->frame_floats;
    }
    // marks (a multiple of 256 bytes) and every array offset (a multiple of 4 floats) are 16-byte multiples
    L.swap_off = ok ? -(int)((marks + sizeof(float) * ctx->img_off[(size_t)li * 4]) / 16) : 0;
    L.flow = ctx->d_flow[li];
    L.flow_frame_stride = ctx->flow_floats[li];
    L.flow_prev = ctx->d_flow[li + 1];
    L.flow_prev_frame_stride = ctx->flow_floats[li + 1];
    ok = ok && dalloc((void**)&L.pat_p, sizeof(float) * L.np * nop * cap);
    ok = ok && dalloc((void**)&L.pat_w, sizeof(float) * (size_t)L.np * L.novals * cap);
    ok = ok && dalloc((void**)&L.pat_conv, sizeof(int) * L.np * cap);
    ok = ok && dalloc((void**)&L.pat_cnt, sizeof(int) * L.np * cap);
    L.fb = ctx->dirs == 2 ? 1 : 0;
    L.fstep = 1;
    L.fb_pos = nullptr;
    L.fb_wbil = nullptr;
    L.fb_reach = nullptr;
    if (L.fb) {
      ok = ok && dalloc((void**)&L.fb_pos, sizeof(int) * 2 * L.np * cap);
      ok = ok && dalloc((void**)&L.fb_wbil, sizeof(float) * 4 * L.np * cap);
      ok = ok && dalloc((void**)&L.fb_reach, sizeof(int) * cap);
    }
  }
  if (ok && prm->usetvref) {
    // sized for the plans of the clusters the device grants (8 and 16 CTAs); a smaller sor_max_cluster, which only
    // trades clusters for chains, grows the workspace in ofdis_set_option when its plans need more
    size_t recf4 = 0;
    int chain_nb = 0;
    sor_workspace_need(ctx, 8, ctx->sor_dev_cluster, &recf4, &chain_nb);
    ok = alloc_refinement(ctx, recf4, chain_nb) && dalloc((void**)&ctx->d_div_fb, sizeof(unsigned long long));
    if (ok) cudaMemsetAsync(ctx->d_div_fb, 0, sizeof(unsigned long long), ctx->stream);
  }
  if (!ok) {
    ofdis_destroy(ctx);
    return OFDIS_ERR_NOMEM;
  }
  *out = ctx;
  return OFDIS_OK;
}

int ofdis_destroy(ofdis_ctx* ctx) {
  if (!ctx) return OFDIS_OK;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  for (auto& kv : ctx->graphs) cudaGraphExecDestroy(kv.second);
  cudaFree(ctx->d_swapped);  // d_img lies in the same allocation
  for (DevBuf* b : {&ctx->d_stage, &ctx->d_full, &ctx->d_eval, &ctx->d_color, &ctx->d_interp, &ctx->d_track,
                    &ctx->d_disp, &ctx->d_sf, &ctx->d_motion, &ctx->d_ego, &ctx->d_relpose, &ctx->d_traj, &ctx->d_stab, &ctx->d_fisher,
                    &ctx->d_fuse, &ctx->d_mesh, &ctx->d_ftrack})
    cudaFree(b->p);
  for (float* p : ctx->d_flow) cudaFree(p);
  for (LevelGeom& L : ctx->lev) {
    cudaFree(L.pat_p);
    cudaFree(L.pat_w);
    cudaFree(L.pat_conv);
    cudaFree(L.pat_cnt);
    cudaFree(L.fb_pos);
    cudaFree(L.fb_wbil);
    cudaFree(L.fb_reach);
  }
  cudaFree(ctx->d_planes);
  cudaFree(ctx->d_fast);
  cudaFree(ctx->d_chain);
  cudaFree(ctx->d_div_fb);
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return OFDIS_OK;
}

int ofdis_set_camlr(ofdis_ctx* ctx, int camlr) {
  if (!ctx || (camlr != 0 && camlr != 1)) return OFDIS_ERR_ARG;
  for (LevelGeom& L : ctx->lev) L.camlr = camlr;
  for (auto& kv : ctx->graphs) cudaGraphExecDestroy(kv.second);  // kernel arguments changed
  ctx->graphs.clear();
  return OFDIS_OK;
}

int ofdis_set_dp_thresh_sq(ofdis_ctx* ctx, float dp_thresh_sq) {
  if (!ctx) return OFDIS_ERR_ARG;
  ctx->pp.dp_thresh_sq = dp_thresh_sq;
  for (auto& kv : ctx->graphs) cudaGraphExecDestroy(kv.second);
  ctx->graphs.clear();
  return OFDIS_OK;
}

int ofdis_level_info(const ofdis_ctx* ctx, int level, int* w, int* h, int* nopw, int* noph, int* steps) {
  if (!ctx) return OFDIS_ERR_ARG;
  const LevelGeom* L = level_of(const_cast<ofdis_ctx*>(ctx), level);
  if (!L) return OFDIS_ERR_ARG;
  if (w) *w = L->w;
  if (h) *h = L->h;
  if (nopw) *nopw = L->nopw;
  if (noph) *noph = L->noph;
  if (steps) *steps = L->steps;
  return OFDIS_OK;
}

int ofdis_upload_level(ofdis_ctx* ctx, int frame, int level, const float* i0, const float* i0x,
                       const float* i0y, const float* i1, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  LevelGeom* L = level_of(ctx, level);
  if (!L || frame < 0 || frame >= ctx->max_frames || !i0 || !i0x || !i0y || !i1) return fail(ctx, OFDIS_ERR_ARG, "upload_level: bad argument");
  CK(cudaSetDevice(ctx->device));
  if (ctx->dirs == 2) return fail(ctx, OFDIS_ERR_ARG, "upload_level: usefbcon needs the gradients of the second image, use ofdis_upload_level_fb");
  const size_t n = (size_t)L->tmp_w * L->tmp_h * L->noc;
  const float* src[4] = {i0, i0x, i0y, i1};
  for (int k = 0; k < 4; ++k)
    CK(cudaMemcpyAsync(const_cast<float*>(L->img[k]) + (size_t)frame * L->img_fs[k], src[k], sizeof(float) * n,
                       kind_in(memkind), ctx->stream));
  return OFDIS_OK;
}

int ofdis_upload_level_fb(ofdis_ctx* ctx, int frame, int level, const float* i0, const float* i0x, const float* i0y,
                          const float* i1, const float* i1x, const float* i1y, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  LevelGeom* L = level_of(ctx, level);
  if (!L || frame < 0 || frame >= ctx->max_frames || !i0 || !i0x || !i0y || !i1) return fail(ctx, OFDIS_ERR_ARG, "upload_level_fb: bad argument");
  if (ctx->dirs == 2 && (!i1x || !i1y)) return fail(ctx, OFDIS_ERR_ARG, "upload_level_fb: usefbcon needs i1x, i1y");
  CK(cudaSetDevice(ctx->device));
  const size_t n = (size_t)L->tmp_w * L->tmp_h * L->noc;
  // forward frame: template I0 (+ gradients), target I1; backward frame: the swapped pair (oflow.cpp:191-197)
  const float* src[2][4] = {{i0, i0x, i0y, i1}, {i1, i1x, i1y, i0}};
  for (int d = 0; d < ctx->dirs; ++d)
    for (int k = 0; k < 4; ++k)
      CK(cudaMemcpyAsync(const_cast<float*>(L->img[k]) + (size_t)(frame * ctx->dirs + d) * L->img_fs[k], src[d][k],
                         sizeof(float) * n, kind_in(memkind), ctx->stream));
  return OFDIS_OK;
}

int ofdis_get_level(ofdis_ctx* ctx, int frame, int level, int which, float* dst, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  LevelGeom* L = level_of(ctx, level);
  if (!L || frame < 0 || frame >= ctx->max_frames || which < 0 || which > 3 || !dst) return fail(ctx, OFDIS_ERR_ARG, "get_level: bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t n = (size_t)L->tmp_w * L->tmp_h * L->noc;
  // the forward frame unless a direction is selected (usefbcon: the backward frame holds the swapped pair)
  const size_t q = (size_t)frame * ctx->dirs + std::max(ctx->sel_dir, 0);
  CK(cudaMemcpyAsync(dst, L->img[which] + q * L->img_fs[which], sizeof(float) * n, kind_out(memkind), ctx->stream));
  if (memkind != OFDIS_MEM_DEVICE) CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

size_t ofdis_packed_frame_floats(const ofdis_ctx* ctx) { return ctx ? ctx->frame_floats : 0; }

size_t ofdis_packed_offset(const ofdis_ctx* ctx, int level, int which) {
  if (!ctx || level < ctx->prm.sc_l || level > ctx->prm.sc_f || which < 0 || which > 3) return (size_t)-1;
  return ctx->img_off[(size_t)(level - ctx->prm.sc_l) * 4 + which];
}

int ofdis_upload_packed(ofdis_ctx* ctx, int f0, int f1, const float* packed, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !packed) return fail(ctx, OFDIS_ERR_ARG, "upload_packed: bad argument");
  if (ctx->dirs == 2) return fail(ctx, OFDIS_ERR_UNSUPPORTED, "upload_packed: a packed frame has no gradients of the second image; with usefbcon use ofdis_upload_level_fb or one of the image-only uploads");
  CK(cudaSetDevice(ctx->device));
  // host and device share the frame layout: one contiguous copy
  CK(cudaMemcpyAsync(ctx->d_img + (size_t)f0 * ctx->frame_floats, packed, sizeof(float) * ctx->frame_floats * (f1 - f0),
                     kind_in(memkind), ctx->stream));
  return OFDIS_OK;
}

// Images of the forward frames are in place: fill the backward frames with the swapped pair
// (usefbcon) and derive the template gradients of every internal frame on every level.
static int finish_gradients(ofdis_ctx* ctx, int f0, int f1) {
  const int D = ctx->dirs, q0 = f0 * D, q1 = f1 * D;
  for (int sl = ctx->prm.sc_f; sl >= ctx->prm.sc_l; --sl) {
    const LevelGeom& L = ctx->lev[sl - ctx->prm.sc_l];
    if (D == 2) {
      if (launch_swap_images(L, q0, q1, ctx->stream) < 0) return fail(ctx, OFDIS_ERR_CUDA, "swap_images_kernel launch", cudaGetLastError());
      ctx->launches += 1;
    }
    if (launch_sobel(L, q0, q1, ctx->stream) < 0) return fail(ctx, OFDIS_ERR_CUDA, "sobel_kernel launch", cudaGetLastError());
    ctx->launches += 1;
  }
  return OFDIS_OK;
}

size_t ofdis_packed_images_frame_floats(const ofdis_ctx* ctx) { return ctx ? ctx->images_floats : 0; }

int ofdis_upload_packed_images(ofdis_ctx* ctx, int f0, int f1, const float* packed, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !packed) return fail(ctx, OFDIS_ERR_ARG, "upload_packed_images: bad argument");
  CK(cudaSetDevice(ctx->device));
  // the image part of every (forward) frame: one 2-D copy, a row per frame
  const int D = ctx->dirs;
  const size_t nif = ctx->images_floats;
  CK(cudaMemcpy2DAsync(ctx->d_img + (size_t)f0 * D * ctx->frame_floats, sizeof(float) * ctx->frame_floats * D, packed,
                       sizeof(float) * nif, sizeof(float) * nif, (size_t)(f1 - f0), kind_in(memkind), ctx->stream));
  return finish_gradients(ctx, f0, f1);
}

// Coarser levels by 2x2 box means (forward frames), then finish_gradients.  SEQ: the pairs hold consecutive
// frames (ofdis_upload_sequence_u8), BIDIR: the forward and the backward pairs of consecutive frames in two halves
// (ofdis_upload_sequence_bidir_u8); each frame's levels are built once.
enum PyramidSource { PAIRS, SEQ, BIDIR };
static int finish_pyramid(ofdis_ctx* ctx, int f0, int f1, PyramidSource src = PAIRS) {
  NvtxRange nvtx("pyramid", -1);
  const int D = ctx->dirs, q0 = f0 * D, nq = f1 - f0;
  for (int sl = ctx->prm.sc_l + 1; sl <= ctx->prm.sc_f; ++sl) {
    const LevelGeom gs = stepped(ctx->lev[sl - 1 - ctx->prm.sc_l], D), gd = stepped(ctx->lev[sl - ctx->prm.sc_l], D);
    const int rc = src == SEQ     ? launch_pyr_down_seq(gs, gd, q0, nq, ctx->stream)
                   : src == BIDIR ? launch_pyr_down_bidir(gs, gd, q0, nq / 2, ctx->stream)
                                  : launch_pyr_down(gs, gd, q0, q0 + nq, ctx->stream);
    if (rc < 0) return fail(ctx, OFDIS_ERR_CUDA, "pyr_down_kernel launch", cudaGetLastError());
    ctx->launches += 1;
  }
  return finish_gradients(ctx, f0, f1);
}

static int org_padding(ofdis_ctx* ctx, int width_org, int height_org, int* padl, int* padt) {
  // run_dense.cpp:299-311: pad up to the next multiple of 2^lv_f -- or of 2^(lv_f+1), as for a run with an init flow
  // (run_dense.cpp:301) -- floor(pad/2) on the left/top
  auto pads_to = [&](int m) {
    return (width_org + m - 1) / m * m == ctx->width && (height_org + m - 1) / m * m == ctx->height;
  };
  const int scf = 1 << ctx->prm.sc_f;
  if (width_org <= 0 || height_org <= 0 || !(pads_to(scf) || pads_to(2 * scf)))
    return fail(ctx, OFDIS_ERR_ARG, "frame size does not pad to the context's width/height");
  *padl = (ctx->width - width_org) / 2;
  *padt = (ctx->height - height_org) / 2;
  return OFDIS_OK;
}

int ofdis_upload_frames_u8(ofdis_ctx* ctx, int f0, int f1, const unsigned char* frames, int width_org, int height_org,
                           int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !frames) return fail(ctx, OFDIS_ERR_ARG, "upload_frames_u8: bad argument");
  if (ctx->prm.sc_l > 8) return fail(ctx, OFDIS_ERR_UNSUPPORTED, "upload_frames_u8: box sums are exact in float32 up to level 8");
  PyrSourceU8 src;
  int rc = org_padding(ctx, width_org, height_org, &src.pad_left, &src.pad_top);
  if (rc) return rc;
  CK(cudaSetDevice(ctx->device));
  src.w_org = width_org;
  src.h_org = height_org;
  src.image_bytes = (size_t)width_org * height_org * ctx->prm.noc;
  src.frames = frames;
  if (memkind != OFDIS_MEM_DEVICE) {
    unsigned char* st = nullptr;
    rc = carve_stage_u8(ctx, src.image_bytes,
                        [&](Carve& c) { st = c.take<unsigned char>(src.image_bytes * 2 * (size_t)ctx->max_frames); });
    if (rc) return rc;
    CK(cudaMemcpyAsync(st, frames, src.image_bytes * 2 * (size_t)(f1 - f0), cudaMemcpyHostToDevice, ctx->stream));
    src.frames = st;
  }
  if (launch_pyr_from_u8(stepped(ctx->lev[0], ctx->dirs), f0 * ctx->dirs, f0 * ctx->dirs + (f1 - f0), src, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "pyr_from_u8_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  return finish_pyramid(ctx, f0, f1);
}

int ofdis_upload_sequence_u8(ofdis_ctx* ctx, int f0, int f1, const unsigned char* frames, int width_org, int height_org,
                             int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !frames) return fail(ctx, OFDIS_ERR_ARG, "upload_sequence_u8: bad argument");
  if (ctx->prm.sc_l > 8) return fail(ctx, OFDIS_ERR_UNSUPPORTED, "upload_sequence_u8: box sums are exact in float32 up to level 8");
  PyrSourceU8 src;
  int rc = org_padding(ctx, width_org, height_org, &src.pad_left, &src.pad_top);
  if (rc) return rc;
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0;
  src.w_org = width_org;
  src.h_org = height_org;
  src.image_bytes = (size_t)width_org * height_org * ctx->prm.noc;
  src.frames = frames;
  if (memkind != OFDIS_MEM_DEVICE) {
    unsigned char* st = nullptr;
    rc = carve_stage_u8(ctx, src.image_bytes,
                        [&](Carve& c) { st = c.take<unsigned char>(src.image_bytes * (size_t)(ctx->max_frames + 1)); });
    if (rc) return rc;
    CK(cudaMemcpyAsync(st, frames, src.image_bytes * (size_t)(n + 1), cudaMemcpyHostToDevice, ctx->stream));
    src.frames = st;
  }
  if (launch_pyr_from_u8_seq(stepped(ctx->lev[0], ctx->dirs), f0 * ctx->dirs, n, src, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "pyr_from_u8_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  return finish_pyramid(ctx, f0, f1, SEQ);
}

int ofdis_upload_sequence_bidir_u8(ofdis_ctx* ctx, int f0, int n, const unsigned char* frames, int width_org,
                                   int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || n < 1 || n > ctx->max_frames || f0 > ctx->max_frames - 2 * n || !frames)
    return fail(ctx, OFDIS_ERR_ARG, "upload_sequence_bidir_u8: bad argument");
  if (ctx->prm.sc_l > 8) return fail(ctx, OFDIS_ERR_UNSUPPORTED, "upload_sequence_bidir_u8: box sums are exact in float32 up to level 8");
  PyrSourceU8 src;
  int rc = org_padding(ctx, width_org, height_org, &src.pad_left, &src.pad_top);
  if (rc) return rc;
  CK(cudaSetDevice(ctx->device));
  NvtxRange nvtx("upload", -1);
  src.w_org = width_org;
  src.h_org = height_org;
  src.image_bytes = (size_t)width_org * height_org * ctx->prm.noc;
  src.frames = frames;
  if (memkind != OFDIS_MEM_DEVICE) {
    unsigned char* st = nullptr;
    const size_t cap = src.image_bytes * (size_t)(ctx->max_frames / 2 + 1);
    rc = carve_stage_u8(ctx, src.image_bytes, [&](Carve& c) { st = c.take<unsigned char>(cap); });
    if (rc) return rc;
    CK(cudaMemcpyAsync(st, frames, src.image_bytes * (size_t)(n + 1), cudaMemcpyHostToDevice, ctx->stream));
    src.frames = st;
  }
  const int D = ctx->dirs;
  if (launch_pyr_from_u8_bidir(stepped(ctx->lev[0], D), f0 * D, n, src, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "pyr_from_u8_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  rc = finish_pyramid(ctx, f0, f0 + 2 * n, BIDIR);
  if (rc) return rc;
  // only once the pyramids are enqueued: the backward half runs as the right camera (stereo)
  CK(cudaMemsetAsync(ctx->d_swapped + (size_t)f0 * D, 0, (size_t)n * D, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_swapped + (size_t)(f0 + n) * D, 1, (size_t)n * D, ctx->stream));
  return OFDIS_OK;
}

int ofdis_set_swapped_slots(ofdis_ctx* ctx, int f0, int f1, int swapped) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || (swapped != 0 && swapped != 1))
    return fail(ctx, OFDIS_ERR_ARG, "set_swapped_slots: bad argument");
  CK(cudaSetDevice(ctx->device));
  // stream-ordered: runs enqueued before keep the marks they were enqueued with; graphs read the marks at replay
  CK(cudaMemsetAsync(ctx->d_swapped + (size_t)f0 * ctx->dirs, swapped, (size_t)(f1 - f0) * ctx->dirs, ctx->stream));
  return OFDIS_OK;
}

size_t ofdis_finest_level_frame_floats(const ofdis_ctx* ctx) {
  return ctx ? (size_t)2 * ctx->lev[0].w * ctx->lev[0].h * ctx->lev[0].noc : 0;
}

int ofdis_upload_finest_level(ofdis_ctx* ctx, int f0, int f1, const float* packed, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !packed) return fail(ctx, OFDIS_ERR_ARG, "upload_finest_level: bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t per = ofdis_finest_level_frame_floats(ctx);
  const float* src = packed;
  if (memkind != OFDIS_MEM_DEVICE) {
    float* st = nullptr;
    int rc = carve_stage(ctx, [&](Carve& c) { st = c.take<float>(per * (size_t)ctx->max_frames); });
    if (rc) return rc;
    CK(cudaMemcpyAsync(st, packed, sizeof(float) * per * (size_t)(f1 - f0), cudaMemcpyHostToDevice, ctx->stream));
    src = st;
  }
  if (launch_pyr_from_level(stepped(ctx->lev[0], ctx->dirs), f0 * ctx->dirs, f0 * ctx->dirs + (f1 - f0), src, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "pyr_from_level_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  return finish_pyramid(ctx, f0, f1);
}

// Level sc_f+1 of pairs [f0, f0 + n) from full-resolution device flows (run_dense.cpp:355-378).  The context must
// be padded to multiples of 2^(sc_f+1): a patch at x of level sc_f reads the init flow at x/2 with row stride w/2
// (patchgrid.cpp:195-211).
static int prepare_initflow(ofdis_ctx* ctx, int f0, int n, const float* flow, int width_org, int height_org) {
  NvtxRange nvtx("initflow", -1);
  int padl, padt;
  const int rc = org_padding(ctx, width_org, height_org, &padl, &padt);
  if (rc) return rc;
  if (launch_initflow_prepare(stepped(ctx->lev[ctx->nlev - 1], ctx->dirs), f0 * ctx->dirs, n, flow, width_org,
                              height_org, padl, padt, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "initflow_prepare_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  return OFDIS_OK;
}

static int check_initflow_ctx(ofdis_ctx* ctx, const char* what) {
  const int s = 2 << ctx->prm.sc_f;
  if (ctx->width % s || ctx->height % s) return fail(ctx, OFDIS_ERR_ARG, what);
  return OFDIS_OK;
}

int ofdis_set_initflow_fullres(ofdis_ctx* ctx, int f0, int f1, const float* flow, int width_org, int height_org,
                               int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !flow) return fail(ctx, OFDIS_ERR_ARG, "set_initflow_fullres: bad argument");
  int rc = check_initflow_ctx(ctx, "set_initflow_fullres: the context's width/height are not multiples of 2^(sc_f+1)");
  if (rc) return rc;
  int padl, padt;
  rc = org_padding(ctx, width_org, height_org, &padl, &padt);
  if (rc) return rc;
  CK(cudaSetDevice(ctx->device));
  const size_t per = (size_t)width_org * height_org * ctx->nop;
  const float* src = flow;
  if (memkind != OFDIS_MEM_DEVICE) {
    float* st = nullptr;
    rc = carve_stage(ctx, [&](Carve& c) { st = c.take<float>(per * (size_t)ctx->max_frames); });
    if (rc) return rc;
    CK(cudaMemcpyAsync(st, flow, sizeof(float) * per * (size_t)(f1 - f0), cudaMemcpyHostToDevice, ctx->stream));
    src = st;
  }
  return prepare_initflow(ctx, f0, f1 - f0, src, width_org, height_org);
}

int ofdis_set_initflow_from_result(ofdis_ctx* ctx, int f0, int f1, int src_f0, int width_org, int height_org) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || src_f0 < 0 || src_f0 + (f1 - f0) > ctx->max_frames)
    return fail(ctx, OFDIS_ERR_ARG, "set_initflow_from_result: bad argument");
  int rc = check_initflow_ctx(ctx, "set_initflow_from_result: the context's width/height are not multiples of 2^(sc_f+1)");
  if (rc) return rc;
  int cx, cy;
  rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  CK(cudaSetDevice(ctx->device));
  // exactly ofdis_get_flow_fullres(DEVICE) into the full-resolution scratch, then ofdis_set_initflow_fullres(DEVICE);
  // the source (level sc_l) and the destination (level sc_f+1) are different buffers, so the slots may overlap
  const size_t pix = (size_t)width_org * height_org;
  float* flow = nullptr;
  rc = carve_full(ctx, pix, [&](Carve& c) { flow = c.take<float>(pix * ctx->nop * (size_t)ctx->max_frames); });
  if (rc) return rc;
  {
    NvtxRange nvtx("upsample", -1);
    if (launch_flow_upsample(stepped(ctx->lev[0], ctx->dirs), src_f0 * ctx->dirs, src_f0 * ctx->dirs + (f1 - f0),
                             flow, width_org, height_org, cx, cy, ctx->stream) < 0)
      return fail(ctx, OFDIS_ERR_CUDA, "flow_upsample_kernel launch", cudaGetLastError());
    ctx->launches += 1;
  }
  return prepare_initflow(ctx, f0, f1 - f0, flow, width_org, height_org);
}

int ofdis_get_flow_fullres(ofdis_ctx* ctx, int f0, int f1, float* out, int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !out) return fail(ctx, OFDIS_ERR_ARG, "get_flow_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("upsample", -1);
  CK(cudaSetDevice(ctx->device));
  const size_t pix = (size_t)width_org * height_org, per = pix * ctx->nop;
  float* dst = out;
  if (memkind != OFDIS_MEM_DEVICE) {
    rc = carve_full(ctx, pix, [&](Carve& c) { dst = c.take<float>(per * (size_t)ctx->max_frames); });
    if (rc) return rc;
  }
  if (launch_flow_upsample(stepped(ctx->lev[0], ctx->dirs), f0 * ctx->dirs, f0 * ctx->dirs + (f1 - f0), dst, width_org, height_org,
                           cx, cy, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "flow_upsample_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  if (memkind != OFDIS_MEM_DEVICE)
    CK(cudaMemcpyAsync(out, dst, sizeof(float) * per * (size_t)(f1 - f0), cudaMemcpyDeviceToHost, ctx->stream));
  return OFDIS_OK;
}

int ofdis_get_flow_fullres_encoded(ofdis_ctx* ctx, int f0, int f1, int encoding, void* out, int width_org,
                                   int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !out ||
      (encoding != OFDIS_ENC_F16 && encoding != OFDIS_ENC_KITTI) ||
      (memkind == OFDIS_MEM_DEVICE && reinterpret_cast<uintptr_t>(out) % 2))
    return fail(ctx, OFDIS_ERR_ARG, "get_flow_fullres_encoded: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("encode", -1);
  CK(cudaSetDevice(ctx->device));
  const size_t pix = (size_t)width_org * height_org;
  // uint16 values per slot: nop binary16, or KITTI's 3 (flow) / 1 (stereo)
  const size_t per = encoding == OFDIS_ENC_F16 ? pix * ctx->nop : pix * (ctx->nop == 2 ? 3 : 1);
  unsigned short* dst = static_cast<unsigned short*>(out);
  if (memkind != OFDIS_MEM_DEVICE) {
    rc = carve_full(ctx, pix, [&](Carve& c) { dst = c.take<unsigned short>(per * (size_t)ctx->max_frames); });
    if (rc) return rc;
  }
  if (launch_flow_encode(stepped(ctx->lev[0], ctx->dirs), f0 * ctx->dirs, f1 - f0, encoding, dst, width_org, height_org,
                         cx, cy, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "flow_encode_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  if (memkind != OFDIS_MEM_DEVICE)
    CK(cudaMemcpyAsync(out, dst, sizeof(unsigned short) * per * (size_t)(f1 - f0), cudaMemcpyDeviceToHost, ctx->stream));
  return OFDIS_OK;
}

int ofdis_flow_color_fullres(ofdis_ctx* ctx, int f0, int f1, unsigned char* rgb, float* scale, float max_value,
                             int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !rgb || !(max_value >= 0.f && max_value <= FLT_MAX) ||
      (memkind == OFDIS_MEM_DEVICE && reinterpret_cast<uintptr_t>(scale) % sizeof(float)))
    return fail(ctx, OFDIS_ERR_ARG, "flow_color_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("color", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0;
  const size_t pix = (size_t)width_org * height_org;
  unsigned int* dmax = nullptr;
  rc = carve(ctx, ctx->d_color, "flow_color_fullres workspace",
             [&](Carve& c) { dmax = c.take<unsigned int>(ctx->max_frames); });
  if (rc) return rc;
  unsigned char* drgb = rgb;
  float* dscale = scale;
  if (memkind != OFDIS_MEM_DEVICE) {
    rc = carve_full(ctx, pix, [&](Carve& c) {
      drgb = c.take<unsigned char>(3 * pix * ctx->max_frames);
      dscale = c.take<float>(ctx->max_frames, scale);
    });
    if (rc) return rc;
  }
  const int k = launch_flow_color(stepped(ctx->lev[0], ctx->dirs), f0 * ctx->dirs, n, dmax, max_value, drgb,
                                  dscale, width_org, height_org, cx, cy, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "flow_color_kernel launch", cudaGetLastError());
  ctx->launches += k;
  if (memkind != OFDIS_MEM_DEVICE) {
    CK(cudaMemcpyAsync(rgb, drgb, 3 * pix * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (scale) CK(cudaMemcpyAsync(scale, dscale, sizeof(float) * n, cudaMemcpyDeviceToHost, ctx->stream));
  }
  return OFDIS_OK;
}

int ofdis_consistency_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, unsigned char* mask, float* err, float alpha,
                              float beta, int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || b0 < 0 || b0 > ctx->max_frames - (f1 - f0) || !mask ||
      !(alpha >= 0.f && alpha <= FLT_MAX) || !(beta >= 0.f && beta <= FLT_MAX))
    return fail(ctx, OFDIS_ERR_ARG, "consistency_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("consistency", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0;
  const size_t pix = (size_t)width_org * height_org;
  unsigned char* dmask = mask;
  float* derr = err;
  if (memkind != OFDIS_MEM_DEVICE) {
    rc = carve_full(ctx, pix, [&](Carve& c) {
      derr = c.take<float>(pix * ctx->max_frames, err);
      dmask = c.take<unsigned char>(pix * ctx->max_frames);
    });
    if (rc) return rc;
  }
  const int D = ctx->dirs;
  if (launch_consistency(stepped(ctx->lev[0], D), f0 * D, b0 * D, n, dmask, derr, width_org, height_org, cx, cy, alpha,
                         beta, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "consistency_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  if (memkind != OFDIS_MEM_DEVICE) {
    CK(cudaMemcpyAsync(mask, dmask, pix * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (err) CK(cudaMemcpyAsync(err, derr, sizeof(float) * pix * n, cudaMemcpyDeviceToHost, ctx->stream));
  }
  return OFDIS_OK;
}

int ofdis_confidence_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_conf_params* p,
                             const unsigned char* frames0, const unsigned char* frames1, size_t frame_stride,
                             float* conf, float* terms, int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  const int side = p ? 2 * p->radius + 1 : 0;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || (b0 >= 0 && b0 > ctx->max_frames - (f1 - f0)) || !p ||
      p->radius < 1 || p->radius > OFDIS_CONF_MAX_RADIUS || !(p->s_fb > 0.f && p->s_fb <= FLT_MAX) ||
      !(p->s_tex > 0.f && p->s_tex <= FLT_MAX) || p->min_count < 1 || p->min_count > side * side || !frames0 ||
      !frames1 || (!conf && !terms) ||
      (dev && (reinterpret_cast<uintptr_t>(conf) % sizeof(float) || reinterpret_cast<uintptr_t>(terms) % sizeof(float))))
    return fail(ctx, OFDIS_ERR_ARG, "confidence_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  const size_t pix = (size_t)width_org * height_org, hwc = pix * ctx->prm.noc;
  if (frame_stride < hwc) return fail(ctx, OFDIS_ERR_ARG, "confidence_fullres: frame_stride below one frame");
  NvtxRange nvtx("confidence", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0, D = ctx->dirs;
  ConfArgs a{frames0, frames1, frame_stride, conf, terms, width_org, height_org, cx, cy, p->radius, p->min_count,
             p->s_fb, p->s_tex};
  if (!dev) {
    unsigned char *i0 = nullptr, *i1 = nullptr;
    rc = carve_stage_u8(ctx, hwc, [&](Carve& c) {
      i0 = c.take<unsigned char>(hwc * ctx->max_frames);
      i1 = c.take<unsigned char>(hwc * ctx->max_frames);
    });
    if (rc) return rc;
    rc = carve_full(ctx, pix, [&](Carve& c) {
      a.conf = c.take<float>(pix * ctx->max_frames, conf);
      a.terms = c.take<float>(3 * pix * ctx->max_frames, terms);
    });
    if (rc) return rc;
    CK(cudaMemcpy2DAsync(i0, hwc, frames0, frame_stride, hwc, n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpy2DAsync(i1, hwc, frames1, frame_stride, hwc, n, cudaMemcpyHostToDevice, ctx->stream));
    a.i0 = i0, a.i1 = i1, a.stride = hwc;
  }
  if (launch_confidence(stepped(ctx->lev[0], D), f0 * D, b0 >= 0 ? b0 * D : -1, n, ctx->prm.noc, a, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "confidence_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  if (!dev) {
    if (conf) CK(cudaMemcpyAsync(conf, a.conf, sizeof(float) * pix * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (terms) CK(cudaMemcpyAsync(terms, a.terms, sizeof(float) * 3 * pix * n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return OFDIS_OK;
}

// The workspace of ofdis_interpolate_fullres for max_frames pairs of the context's size (InterpWork), allocated on
// the first call: per pixel and pair the keys (8 bytes), u_t (4 nop), the fill stamps (4), two hole lists (4 + 4) and
// the two consistency masks (1 + 1); then one word per pair and width + height round counts.
static int ensure_interp(ofdis_ctx* ctx) {
  const size_t P = (size_t)ctx->max_frames * ctx->width * ctx->height;
  if (P > UINT_MAX) return fail(ctx, OFDIS_ERR_UNSUPPORTED, "interpolate_fullres: more than 2^32 pixels per call");
  InterpWork& ws = ctx->interp;
  return carve(ctx, ctx->d_interp, "interpolate_fullres workspace", [&](Carve& c) {
    ws.keys = c.take<unsigned long long>(P);
    ws.ut = c.take<float>(ctx->nop * P);
    ws.stamp = c.take<int>(P);
    ws.list[0] = c.take<unsigned int>(P);
    ws.list[1] = c.take<unsigned int>(P);
    ws.any = c.take<int>(ctx->max_frames);
    ws.count = c.take<unsigned int>(ctx->width + ctx->height);
    ws.m0 = c.take<unsigned char>(P);
    ws.m1 = c.take<unsigned char>(P);
  });
}

int ofdis_interpolate_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* i0, const unsigned char* i1,
                              size_t frame_stride, float t, float alpha, float beta, unsigned char* out, float* flow_t,
                              int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || b0 < 0 || b0 > ctx->max_frames - (f1 - f0) || !i0 || !i1 ||
      !out || !(t > 0.f && t < 1.f) || !(alpha >= 0.f && alpha <= FLT_MAX) || !(beta >= 0.f && beta <= FLT_MAX) ||
      (memkind == OFDIS_MEM_DEVICE && reinterpret_cast<uintptr_t>(flow_t) % sizeof(float)))
    return fail(ctx, OFDIS_ERR_ARG, "interpolate_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  const size_t pix = (size_t)width_org * height_org, hwc = pix * ctx->prm.noc;
  if (frame_stride < hwc) return fail(ctx, OFDIS_ERR_ARG, "interpolate_fullres: frame_stride below one frame");
  NvtxRange nvtx("interpolate", -1);
  CK(cudaSetDevice(ctx->device));
  rc = ensure_interp(ctx);
  if (rc) return rc;
  const int n = f1 - f0, D = ctx->dirs, nop = ctx->nop;
  const InterpWork& ws = ctx->interp;
  InterpSrc s{i0, i1, frame_stride, width_org, height_org, cx, cy, t};
  unsigned char* dout = out;
  if (memkind != OFDIS_MEM_DEVICE) {
    unsigned char *s0 = nullptr, *s1 = nullptr;
    rc = carve_stage_u8(ctx, hwc, [&](Carve& c) {
      s0 = c.take<unsigned char>(hwc * ctx->max_frames);
      s1 = c.take<unsigned char>(hwc * ctx->max_frames);
    });
    if (rc) return rc;
    rc = carve_full(ctx, pix, [&](Carve& c) { dout = c.take<unsigned char>(hwc * ctx->max_frames); });
    if (rc) return rc;
    CK(cudaMemcpy2DAsync(s0, hwc, i0, frame_stride, hwc, n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpy2DAsync(s1, hwc, i1, frame_stride, hwc, n, cudaMemcpyHostToDevice, ctx->stream));
    s = InterpSrc{s0, s1, hwc, width_org, height_org, cx, cy, t};
  }
  const LevelGeom g = stepped(ctx->lev[0], D);
  CK(cudaMemsetAsync(ws.keys, 0xff, sizeof(unsigned long long) * pix * n, ctx->stream));
  CK(cudaMemsetAsync(ws.any, 0, sizeof(int) * n, ctx->stream));
  CK(cudaMemsetAsync(ws.count, 0, sizeof(unsigned int) * (ctx->width + ctx->height), ctx->stream));
  if (launch_consistency(g, f0 * D, b0 * D, n, ws.m0, nullptr, width_org, height_org, cx, cy, alpha, beta,
                         ctx->stream) < 0 ||
      launch_consistency(g, b0 * D, f0 * D, n, ws.m1, nullptr, width_org, height_org, cx, cy, alpha, beta,
                         ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "consistency_kernel launch", cudaGetLastError());
  if (launch_interp_splat(g, f0 * D, n, s, ws, ctx->stream) < 0 || launch_interp_resolve(g, f0 * D, n, s, ws, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "interp_splat_kernel launch", cudaGetLastError());
  ctx->launches += 4;
  // Hole filling: round r fills the holes 4-neighbour distance r from the nearest splatted pixel, so every hole is
  // filled after width + height - 2 rounds.  The rounds go out in batches of 8, 16, ... 256 launches; the count of
  // holes left is read after each batch, so that holes a few pixels wide cost one read, and a frame filled from one
  // pixel one read per 256 rounds once the batches have grown.  Rounds after the last hole do nothing.
  const int max_rounds = width_org + height_org - 2;
  unsigned int bound = (unsigned int)(pix * n), left = 0;
  for (int r = 0, batch = 8; r < max_rounds; batch = std::min(2 * batch, 256)) {
    const int rounds = std::min(batch, max_rounds - r);
    if (launch_interp_fill(nop, ws, width_org, height_org, r + 1, rounds, bound, ctx->stream) < 0)
      return fail(ctx, OFDIS_ERR_CUDA, "interp_fill_kernel launch", cudaGetLastError());
    ctx->launches += rounds;
    r += rounds;
    CK(cudaMemcpyAsync(&left, ws.count + r, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (!left) break;
    bound = left;
  }
  if (left) return fail(ctx, OFDIS_ERR_CUDA, "interpolate_fullres: holes left after the last fill round");
  if (launch_interp_blend(nop, ctx->prm.noc, n, s, ws, dout, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "interp_blend_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  if (memkind != OFDIS_MEM_DEVICE) CK(cudaMemcpyAsync(out, dout, hwc * n, cudaMemcpyDeviceToHost, ctx->stream));
  if (flow_t)
    CK(cudaMemcpyAsync(flow_t, ws.ut, sizeof(float) * pix * nop * n, kind_out(memkind), ctx->stream));
  return OFDIS_OK;
}

// The workspace of ofdis_disparity_fullres for max_frames pairs of the context's size, allocated on the first call:
// per pixel and pair d, the parent and the component size (4 bytes each) and the status (1); per row and pair the
// row pass's flag and the nearest full rows above and below (4 bytes each).  A call of a smaller frame size packs its
// pairs densely at the front of each array.
static int ensure_disp(ofdis_ctx* ctx, DispWork* ws) {
  const size_t P = (size_t)ctx->max_frames * ctx->width * ctx->height, R = (size_t)ctx->max_frames * ctx->height;
  return carve(ctx, ctx->d_disp, "disparity_fullres workspace", [&](Carve& c) {
    ws->val = c.take<float>(P);
    ws->parent = c.take<int>(P);
    ws->size = c.take<int>(P);
    ws->rowfull = c.take<int>(R);
    ws->up = c.take<int>(R);
    ws->down = c.take<int>(R);
    ws->status = c.take<unsigned char>(P);
  });
}

static bool finite_ge0(float v) { return v >= 0.f && v <= FLT_MAX; }
static bool finite_gt0(float v) { return v > 0.f && v <= FLT_MAX; }
static bool finite_f32(float v) { return v >= -FLT_MAX && v <= FLT_MAX; }

int ofdis_disparity_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_disp_filter* filt,
                            const ofdis_stereo_camera* cam, float* disp, unsigned char* status, float* depth,
                            float* xyz, int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  auto misaligned = [dev](const float* p) { return dev && reinterpret_cast<uintptr_t>(p) % sizeof(float); };
  const bool need_cam = depth || xyz;
  if (ctx->nop != 1 || f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !filt ||
      (filt->lr_check && (b0 < 0 || b0 > ctx->max_frames - (f1 - f0))) ||
      (filt->lr_check != 0 && filt->lr_check != 1) || (filt->fill != 0 && filt->fill != 1) ||
      !finite_ge0(filt->alpha) || !finite_ge0(filt->beta) || filt->speckle_size < 0 ||
      !finite_ge0(filt->speckle_diff) || (!disp && !status && !depth && !xyz) ||
      (need_cam && (!cam || !finite_gt0(cam->fx) || !finite_gt0(cam->fy) || !finite_gt0(cam->baseline) ||
                    !finite_f32(cam->cx) || !finite_f32(cam->cy) || !finite_f32(cam->doffs))) ||
      misaligned(disp) || misaligned(depth) || misaligned(xyz))
    return fail(ctx, OFDIS_ERR_ARG, "disparity_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  const size_t pix = (size_t)width_org * height_org;
  if (pix > (size_t)INT_MAX) return fail(ctx, OFDIS_ERR_UNSUPPORTED, "disparity_fullres: 2^31 pixels or more per frame");
  NvtxRange nvtx("disparity", -1);
  CK(cudaSetDevice(ctx->device));
  DispWork ws;
  rc = ensure_disp(ctx, &ws);
  if (rc) return rc;
  const int n = f1 - f0, D = ctx->dirs;
  const size_t np = pix * n;
  DispOutputs out{disp, status, depth, xyz};
  if (!dev) {
    const size_t cap = pix * ctx->max_frames;
    rc = carve_full(ctx, pix, [&](Carve& c) {
      out.disp = c.take<float>(cap, disp);
      out.depth = c.take<float>(cap, depth);
      out.xyz = c.take<float>(3 * cap, xyz);
      out.status = c.take<unsigned char>(cap, status);
    });
    if (rc) return rc;
  }
  const DispFilter f{filt->lr_check, filt->alpha, filt->beta, filt->speckle_size, filt->speckle_diff, filt->fill};
  DispCamera c{};
  if (need_cam) c = DispCamera{cam->fx * cam->baseline, cam->fx, cam->fy, cam->cx, cam->cy, cam->doffs};
  const int k = launch_disparity(stepped(ctx->lev[0], D), f0 * D, (filt->lr_check ? b0 : f0) * D, n, f, c, ws, out,
                                 width_org, height_org, cx, cy, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "disp_classify_kernel launch", cudaGetLastError());
  ctx->launches += k;
  if (!dev) {
    if (disp) CK(cudaMemcpyAsync(disp, out.disp, sizeof(float) * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (depth) CK(cudaMemcpyAsync(depth, out.depth, sizeof(float) * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (xyz) CK(cudaMemcpyAsync(xyz, out.xyz, sizeof(float) * 3 * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (status) CK(cudaMemcpyAsync(status, out.status, np, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return OFDIS_OK;
}

// The workspace of ofdis_global_motion_fullres for max_frames pairs of at least `cells` cells and `hyps` hypotheses:
// per cell the correspondence (16 bytes), its flag (1) and the refit's chunk sums (44 doubles per 32 cells, 11); per
// hypothesis its float64 parameters (64) and MotionHyp (48); per pair MotionOut, the key and the count.  The cell and
// hypothesis capacities grow independently, never shrink.
static int ensure_motion(ofdis_ctx* ctx, size_t cells, size_t hyps) {
  cells = std::max((cells + 31) / 32 * 32, ctx->motion_cells);
  hyps = std::max(hyps, ctx->motion_hyps);
  const size_t n = (size_t)ctx->max_frames;
  MotionWork& ws = ctx->motion;
  const int rc = carve(ctx, ctx->d_motion, "global_motion_fullres workspace", [&](Carve& c) {
    ws.corr = c.take<float4>(n * cells);
    ws.chunk = c.take<double>(n * (cells / 32) * MOTION_NE);
    ws.hp = c.take<double>(n * hyps * 8);
    ws.hg = c.take<MotionHyp>(n * hyps);
    ws.out = c.take<MotionOut>(n);
    ws.key = c.take<unsigned long long>(n);
    ws.m = c.take<int>(n);
    ws.flag = c.take<unsigned char>(n * cells);
  });
  ctx->motion_cells = rc ? 0 : cells;
  ctx->motion_hyps = rc ? 0 : hyps;
  return rc;
}

int ofdis_global_motion_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_motion_params* p,
                                const unsigned char* i1, size_t frame_stride, double* model,
                                ofdis_motion_stats* stats, unsigned char* mask, float* residual,
                                unsigned char* registered, int width_org, int height_org, int memkind) {
  static_assert(sizeof(ofdis_motion_stats) == 24, "ofdis_motion_stats: 24 bytes, as api.MotionStats");
  if (!ctx) return OFDIS_ERR_ARG;
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  if (ctx->nop != 2 || f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !p ||
      (p->fb_check && (b0 < 0 || b0 > ctx->max_frames - (f1 - f0))) ||
      p->model < OFDIS_MOTION_SIMILARITY || p->model > OFDIS_MOTION_HOMOGRAPHY || p->step < 1 ||
      (p->fb_check != 0 && p->fb_check != 1) || !finite_ge0(p->alpha) || !finite_ge0(p->beta) ||
      p->hypotheses < 1 || p->hypotheses > 65536 || !finite_gt0(p->threshold) || p->refine < 0 || p->refine > 16 ||
      !model || !stats || (registered && !i1) || (dev && reinterpret_cast<uintptr_t>(residual) % sizeof(float)))
    return fail(ctx, OFDIS_ERR_ARG, "global_motion_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  const size_t pix = (size_t)width_org * height_org, noc = (size_t)ctx->prm.noc, hwc = pix * noc;
  if (registered && frame_stride < hwc) return fail(ctx, OFDIS_ERR_ARG, "global_motion_fullres: frame_stride below one frame");
  const int s = p->step, ncx = (width_org - 1) / s + 1, ncy = (height_org - 1) / s + 1;
  if ((long long)ncx * ncy > (1ll << 24)) return fail(ctx, OFDIS_ERR_ARG, "global_motion_fullres: more than 2^24 cells");
  NvtxRange nvtx("global_motion", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0, D = ctx->dirs;
  rc = ensure_motion(ctx, (size_t)ncx * ncy, (size_t)p->hypotheses);
  if (rc) return rc;
  MotionGeom mg{};
  mg.w = width_org, mg.h = height_org, mg.s = s, mg.ncx = ncx, mg.cells = ncx * ncy, mg.model = p->model;
  mg.n_min = p->model + 1, mg.nh = p->hypotheses, mg.fb_check = p->fb_check, mg.refine = p->refine;
  mg.crop_x = cx, mg.crop_y = cy, mg.noc = ctx->prm.noc, mg.alpha = p->alpha, mg.beta = p->beta;
  mg.cx = 0.5f * (float)(width_org - 1);
  mg.cy = 0.5f * (float)(height_org - 1);
  mg.sigma = 2.0f / (float)std::max(width_org, height_org);
  mg.t = p->threshold * mg.sigma;
  mg.thr = p->threshold;
  mg.seed = p->seed;
  mg.cell_cap = ctx->motion_cells, mg.chunk_cap = ctx->motion_cells / 32, mg.hyp_cap = ctx->motion_hyps;
  MotionOutputs o{mask, residual, registered, i1, frame_stride};
  if (!dev && (mask || residual || registered)) {
    const size_t cap = pix * ctx->max_frames;
    rc = carve_full(ctx, pix, [&](Carve& c) {
      o.residual = c.take<float>(2 * cap, residual);
      o.mask = c.take<unsigned char>(cap, mask);
      o.registered = c.take<unsigned char>(noc * cap, registered);
    });
    if (rc) return rc;
    if (registered) {
      unsigned char* st = nullptr;
      rc = carve_stage(ctx, [&](Carve& c) { st = c.take<unsigned char>(hwc * ctx->max_frames); });
      if (rc) return rc;
      CK(cudaMemcpy2DAsync(st, hwc, i1, frame_stride, hwc, n, cudaMemcpyHostToDevice, ctx->stream));
      o.i1 = st;
      o.stride = hwc;
    }
  }
  const int k = launch_global_motion(stepped(ctx->lev[0], D), f0 * D, (p->fb_check ? b0 : f0) * D, n, mg, ctx->motion,
                                     o, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "motion kernel launch", cudaGetLastError());
  ctx->launches += k;
  if (!dev) {
    if (residual) CK(cudaMemcpyAsync(residual, o.residual, sizeof(float) * 2 * pix * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (mask) CK(cudaMemcpyAsync(mask, o.mask, pix * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (registered) CK(cudaMemcpyAsync(registered, o.registered, hwc * n, cudaMemcpyDeviceToHost, ctx->stream));
  }
  std::vector<MotionOut> res(n);
  CK(cudaMemcpyAsync(res.data(), ctx->motion.out, sizeof(MotionOut) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int q = 0; q < n; ++q) {
    std::memcpy(model + 9 * (size_t)q, res[q].M, sizeof(res[q].M));
    stats[q] = res[q].st;
  }
  return OFDIS_OK;
}

// The workspace of ofdis_egomotion_fullres for max_frames pairs of at least `cells` cells and `hyps` hypotheses: per
// cell the correspondence (32 bytes), its flag (1) and the refit's chunk sums (27 doubles per 32 cells); per hypothesis
// its float64 [R | t] (96) and EgoHyp (64); per pair EgoOut, the key and the count.  The cell and hypothesis
// capacities grow independently, never shrink.
static int ensure_ego(ofdis_ctx* ctx, size_t cells, size_t hyps) {
  cells = std::max((cells + 31) / 32 * 32, ctx->ego_cells);
  hyps = std::max(hyps, ctx->ego_hyps);
  const size_t n = (size_t)ctx->max_frames;
  EgoWork& ws = ctx->ego;
  const int rc = carve(ctx, ctx->d_ego, "egomotion_fullres workspace", [&](Carve& c) {
    ws.corr = c.take<EgoCorr>(n * cells);
    ws.chunk = c.take<double>(n * (cells / 32) * EGO_NE);
    ws.hp = c.take<double>(n * hyps * 12);
    ws.hg = c.take<EgoHyp>(n * hyps);
    ws.out = c.take<EgoOut>(n);
    ws.key = c.take<unsigned long long>(n);
    ws.m = c.take<int>(n);
    ws.flag = c.take<unsigned char>(n * cells);
  });
  ctx->ego_cells = rc ? 0 : cells;
  ctx->ego_hyps = rc ? 0 : hyps;
  return rc;
}

int ofdis_egomotion_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_egomotion_params* p,
                            const float* disp0, const float* disp1, size_t disp_stride,
                            const ofdis_stereo_camera* cam, double* pose, ofdis_motion_stats* stats,
                            unsigned char* mask, float* residual, float* object_motion,
                            int width_org, int height_org, int memkind) {
  static_assert(sizeof(EgoCorr) == 32 && sizeof(EgoHyp) == 64 && sizeof(EgoOut) == 128, "egomotion records");
  if (!ctx) return OFDIS_ERR_ARG;
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  auto misaligned = [dev](const float* q) { return dev && reinterpret_cast<uintptr_t>(q) % sizeof(float); };
  const size_t pix = (size_t)std::max(width_org, 0) * std::max(height_org, 0);
  if (ctx->nop != 2 || f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !p ||
      (p->fb_check && (b0 < 0 || b0 > ctx->max_frames - (f1 - f0))) || p->step < 1 ||
      (p->fb_check != 0 && p->fb_check != 1) || !finite_ge0(p->alpha) || !finite_ge0(p->beta) ||
      !(p->edge_diff >= 0.f) || p->hypotheses < 1 || p->hypotheses > 65536 || !finite_gt0(p->threshold) ||
      p->refine < 0 || p->refine > 16 || !cam || !finite_gt0(cam->fx) || !finite_gt0(cam->fy) ||
      !finite_gt0(cam->baseline) || !finite_f32(cam->cx) || !finite_f32(cam->cy) || !finite_f32(cam->doffs) ||
      !disp0 || !disp1 || !pose || !stats || disp_stride < pix || misaligned(disp0) || misaligned(disp1) ||
      misaligned(residual) || misaligned(object_motion))
    return fail(ctx, OFDIS_ERR_ARG, "egomotion_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  const int s = p->step, ncx = (width_org - 1) / s + 1, ncy = (height_org - 1) / s + 1;
  if ((long long)ncx * ncy > (1ll << 24)) return fail(ctx, OFDIS_ERR_ARG, "egomotion_fullres: more than 2^24 cells");
  NvtxRange nvtx("egomotion", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0, D = ctx->dirs;
  const size_t np = pix * n;
  rc = ensure_ego(ctx, (size_t)ncx * ncy, (size_t)p->hypotheses);
  if (rc) return rc;
  EgoGeom eg{};
  eg.w = width_org, eg.h = height_org, eg.s = s, eg.ncx = ncx, eg.cells = ncx * ncy, eg.nh = p->hypotheses;
  eg.fb_check = p->fb_check, eg.refine = p->refine, eg.crop_x = cx, eg.crop_y = cy;
  eg.alpha = p->alpha, eg.beta = p->beta, eg.edge_diff = p->edge_diff, eg.thr = p->threshold;
  eg.cam = DispCamera{cam->fx * cam->baseline, cam->fx, cam->fy, cam->cx, cam->cy, cam->doffs};
  eg.seed = p->seed;
  eg.cell_cap = ctx->ego_cells, eg.chunk_cap = ctx->ego_cells / 32, eg.hyp_cap = ctx->ego_hyps;
  eg.disp0 = disp0, eg.disp1 = disp1, eg.stride = disp_stride;
  EgoOutputs o{mask, residual, object_motion};
  if (!dev) {
    // disp0 and disp1 packed to one map per pair
    const size_t cap = pix * ctx->max_frames;
    float *d0 = nullptr, *d1 = nullptr;
    rc = carve_stage(ctx, [&](Carve& c) {
      d0 = c.take<float>(cap);
      d1 = c.take<float>(cap);
    });
    if (rc) return rc;
    const size_t row = sizeof(float) * pix, pitch = sizeof(float) * disp_stride;
    CK(cudaMemcpy2DAsync(d0, row, disp0, pitch, row, n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpy2DAsync(d1, row, disp1, pitch, row, n, cudaMemcpyHostToDevice, ctx->stream));
    eg.disp0 = d0, eg.disp1 = d1, eg.stride = pix;
    if (mask || residual || object_motion) {
      rc = carve_full(ctx, pix, [&](Carve& c) {
        o.residual = c.take<float>(2 * cap, residual);
        o.object_motion = c.take<float>(3 * cap, object_motion);
        o.mask = c.take<unsigned char>(cap, mask);
      });
      if (rc) return rc;
    }
  }
  const int k = launch_egomotion(stepped(ctx->lev[0], D), f0 * D, (p->fb_check ? b0 : f0) * D, n, eg, ctx->ego, o,
                                 ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "egomotion kernel launch", cudaGetLastError());
  ctx->launches += k;
  if (!dev) {
    if (residual) CK(cudaMemcpyAsync(residual, o.residual, sizeof(float) * 2 * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (object_motion)
      CK(cudaMemcpyAsync(object_motion, o.object_motion, sizeof(float) * 3 * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (mask) CK(cudaMemcpyAsync(mask, o.mask, np, cudaMemcpyDeviceToHost, ctx->stream));
  }
  std::vector<EgoOut> res(n);
  CK(cudaMemcpyAsync(res.data(), ctx->ego.out, sizeof(EgoOut) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int q = 0; q < n; ++q) {
    std::memcpy(pose + 12 * (size_t)q, res[q].pose, sizeof(res[q].pose));
    stats[q] = res[q].st;
  }
  return OFDIS_OK;
}

// The workspace of ofdis_relpose_fullres for max_frames pairs of at least `cells` cells and `hyps` hypotheses: per cell
// the correspondence (16 bytes), its flag (1) and the refit's chunk sums (21 doubles per 32 cells); per hypothesis its
// float64 E (72) and MotionHyp (48); per pair RelposeOut, the key and the count.  The cell and hypothesis capacities
// grow independently, never shrink.
static int ensure_relpose(ofdis_ctx* ctx, size_t cells, size_t hyps) {
  cells = std::max((cells + 31) / 32 * 32, ctx->relpose_cells);
  hyps = std::max(hyps, ctx->relpose_hyps);
  const size_t n = (size_t)ctx->max_frames;
  MotionWork& ws = ctx->relpose;
  const int rc = carve(ctx, ctx->d_relpose, "relpose_fullres workspace", [&](Carve& c) {
    ws.corr = c.take<float4>(n * cells);
    ws.chunk = c.take<double>(n * (cells / 32) * RELPOSE_NE);
    ws.hp = c.take<double>(n * hyps * 9);
    ws.hg = c.take<MotionHyp>(n * hyps);
    ctx->relpose_out = c.take<RelposeOut>(n);
    ws.key = c.take<unsigned long long>(n);
    ws.m = c.take<int>(n);
    ws.flag = c.take<unsigned char>(n * cells);
  });
  ctx->relpose_cells = rc ? 0 : cells;
  ctx->relpose_hyps = rc ? 0 : hyps;
  return rc;
}

int ofdis_relpose_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_relpose_params* p, double* pose,
                          ofdis_motion_stats* stats, unsigned char* mask, float* sampson, float* depth, int width_org,
                          int height_org, int memkind) {
  static_assert(sizeof(RelposeOut) == 160, "relpose record");
  if (!ctx) return OFDIS_ERR_ARG;
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  auto misaligned = [dev](const float* q) { return dev && reinterpret_cast<uintptr_t>(q) % sizeof(float); };
  if (ctx->nop != 2 || f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !p ||
      (p->fb_check && (b0 < 0 || b0 > ctx->max_frames - (f1 - f0))) || p->step < 1 ||
      (p->fb_check != 0 && p->fb_check != 1) || !finite_ge0(p->alpha) || !finite_ge0(p->beta) ||
      !finite_gt0(p->fx) || !finite_gt0(p->fy) || !finite_f32(p->cx) || !finite_f32(p->cy) ||
      p->hypotheses < 1 || p->hypotheses > 65536 || !finite_gt0(p->threshold) || p->refine < 0 || p->refine > 16 ||
      !finite_ge0(p->min_parallax) || !pose || !stats || misaligned(sampson) || misaligned(depth))
    return fail(ctx, OFDIS_ERR_ARG, "relpose_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  const size_t pix = (size_t)width_org * height_org;
  const int s = p->step, ncx = (width_org - 1) / s + 1, ncy = (height_org - 1) / s + 1;
  if ((long long)ncx * ncy > (1ll << 24)) return fail(ctx, OFDIS_ERR_ARG, "relpose_fullres: more than 2^24 cells");
  NvtxRange nvtx("relpose", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0, D = ctx->dirs;
  const size_t np = pix * n;
  rc = ensure_relpose(ctx, (size_t)ncx * ncy, (size_t)p->hypotheses);
  if (rc) return rc;
  RelposeGeom rg{};
  MotionGeom& mg = rg.mg;
  mg.w = width_org, mg.h = height_org, mg.s = s, mg.ncx = ncx, mg.cells = ncx * ncy, mg.model = 0;
  mg.n_min = 8, mg.nh = p->hypotheses, mg.fb_check = p->fb_check, mg.refine = p->refine;
  mg.crop_x = cx, mg.crop_y = cy, mg.noc = ctx->prm.noc, mg.alpha = p->alpha, mg.beta = p->beta;
  mg.cx = 0.f, mg.cy = 0.f, mg.sigma = 1.f;  // global motion's correspondences in pixel coordinates
  mg.t = p->threshold, mg.thr = p->threshold;
  mg.seed = p->seed;
  mg.cell_cap = ctx->relpose_cells, mg.chunk_cap = ctx->relpose_cells / 32, mg.hyp_cap = ctx->relpose_hyps;
  rg.fx = p->fx, rg.fy = p->fy, rg.cx = p->cx, rg.cy = p->cy, rg.min_parallax = p->min_parallax;
  RelposeOutputs o{mask, sampson, depth};
  if (!dev && (mask || sampson || depth)) {
    const size_t cap = pix * ctx->max_frames;
    rc = carve_full(ctx, pix, [&](Carve& c) {
      o.sampson = c.take<float>(cap, sampson);
      o.depth = c.take<float>(cap, depth);
      o.mask = c.take<unsigned char>(cap, mask);
    });
    if (rc) return rc;
  }
  const int k = launch_relpose(stepped(ctx->lev[0], D), f0 * D, (p->fb_check ? b0 : f0) * D, n, rg, ctx->relpose,
                               ctx->relpose_out, o, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "relpose kernel launch", cudaGetLastError());
  ctx->launches += k;
  if (!dev) {
    if (sampson) CK(cudaMemcpyAsync(sampson, o.sampson, sizeof(float) * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (depth) CK(cudaMemcpyAsync(depth, o.depth, sizeof(float) * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (mask) CK(cudaMemcpyAsync(mask, o.mask, np, cudaMemcpyDeviceToHost, ctx->stream));
  }
  std::vector<RelposeOut> res(n);
  CK(cudaMemcpyAsync(res.data(), ctx->relpose_out, sizeof(RelposeOut) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int q = 0; q < n; ++q) {
    std::memcpy(pose + 12 * (size_t)q, res[q].pose, sizeof(res[q].pose));
    stats[q] = res[q].st;
  }
  return OFDIS_OK;
}

static bool fuse_cam_ok(const ofdis_stereo_camera* cam) {
  return cam && finite_gt0(cam->fx) && finite_gt0(cam->fy) && finite_gt0(cam->baseline) && finite_f32(cam->cx) &&
         finite_f32(cam->cy) && finite_f32(cam->doffs);
}

// n poses [n][12] float64 (camera-to-world) into ctx->fuse_ws.g as float32: world-to-camera (invert) or as given
static int fuse_poses(ofdis_ctx* ctx, int n, const double* P, bool invert) {
  std::vector<float> g((size_t)12 * n);
  for (int k = 0; k < n; ++k) {
    const double* p = P + (size_t)12 * k;
    float* q = g.data() + (size_t)12 * k;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 4; ++c) {
        if (!(std::fabs(p[4 * r + c]) <= DBL_MAX)) return fail(ctx, OFDIS_ERR_ARG, "fuse: a pose entry is not finite");
        if (!invert) q[4 * r + c] = (float)p[4 * r + c];
      }
      if (invert) {
        for (int c = 0; c < 3; ++c) q[4 * r + c] = (float)p[4 * c + r];
        q[4 * r + 3] = (float)(-(((p[r] * p[3]) + (p[4 + r] * p[7])) + (p[8 + r] * p[11])));
      }
    }
  }
  CK(cudaMemcpyAsync(ctx->fuse_ws.g, g.data(), sizeof(float) * g.size(), cudaMemcpyHostToDevice, ctx->stream));
  // g is pageable host memory: the copy has left it when cudaMemcpyAsync returns
  return OFDIS_OK;
}

int ofdis_fuse_begin(ofdis_ctx* ctx, const ofdis_fuse_params* p) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (!p || p->nx < 1 || p->ny < 1 || p->nz < 1 || (long long)p->nx * p->ny * p->nz > (1ll << 30) ||
      !finite_f32(p->origin[0]) || !finite_f32(p->origin[1]) || !finite_f32(p->origin[2]) || !finite_gt0(p->voxel) ||
      !finite_gt0(p->trunc) || !(p->max_weight >= 1.0f && p->max_weight <= FLT_MAX) || (p->color != 0 && p->color != 1))
    return fail(ctx, OFDIS_ERR_ARG, "fuse_begin: bad argument");
  NvtxRange nvtx("fuse", -1);
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)p->nx * p->ny * p->nz, nb = (N + FUSE_BLOCK - 1) / FUSE_BLOCK;
  FuseVolume& v = ctx->fuse_vol;
  auto layout = [&](Carve& c) {
    v.T = c.take<float>(N);
    v.W = c.take<float>(N);
    v.C = p->color ? c.take<unsigned char>(3 * N) : nullptr;
    ctx->fuse_ws.g = c.take<float>(12 * (size_t)(ctx->max_frames + 1));
    ctx->fuse_ws.bsum = c.take<unsigned long long>(nb);
    ctx->fuse_ws.total = c.take<unsigned long long>(1);
  };
  if (measure(layout) > ctx->d_fuse.bytes) ctx->fuse_on = false;  // the live volume goes with the old buffer
  const int rc = carve(ctx, ctx->d_fuse, "fuse volume", layout);
  if (rc) return rc;
  FuseGeom& g = ctx->fuse_geom;
  g.count = (long long)N;
  g.nx = p->nx, g.ny = p->ny, g.nz = p->nz;
  g.ox = p->origin[0], g.oy = p->origin[1], g.oz = p->origin[2];
  g.voxel = p->voxel, g.mu = p->trunc, g.max_weight = p->max_weight;
  CK(cudaMemsetAsync(v.T, 0, 4 * N, ctx->stream));
  CK(cudaMemsetAsync(v.W, 0, 4 * N, ctx->stream));
  if (v.C) CK(cudaMemsetAsync(v.C, 0, 3 * N, ctx->stream));
  ctx->fuse_on = true;
  return OFDIS_OK;
}

// Host inputs of n frames of the fusion calls through the staging buffer: the disparity maps, the frames and the
// weights (those not null) are copied there and replaced by their copies.  The layout holds max_frames + 1 of each,
// with the frames' room whenever the volume has colour and the weights' whenever the call is weighted.
static int fuse_stage(ofdis_ctx* ctx, int n, size_t pix, size_t hwc, bool color, const float** disp,
                      size_t* disp_stride, const unsigned char** frames, size_t* frame_stride, const float** weight,
                      size_t* weight_stride) {
  const size_t F = (size_t)ctx->max_frames + 1;
  float *d = nullptr, *w = nullptr;
  unsigned char* f = nullptr;
  const int rc = carve_stage(ctx, [&](Carve& c) {
    d = c.take<float>(pix * F);
    if (color) f = c.take<unsigned char>(hwc * F);
    if (*weight) w = c.take<float>(pix * F);
  });
  if (rc) return rc;
  CK(cudaMemcpy2DAsync(d, sizeof(float) * pix, *disp, sizeof(float) * *disp_stride, sizeof(float) * pix, n,
                       cudaMemcpyHostToDevice, ctx->stream));
  *disp = d, *disp_stride = pix;
  if (*frames) {
    CK(cudaMemcpy2DAsync(f, hwc, *frames, *frame_stride, hwc, n, cudaMemcpyHostToDevice, ctx->stream));
    *frames = f, *frame_stride = hwc;
  }
  if (*weight) {
    CK(cudaMemcpy2DAsync(w, sizeof(float) * pix, *weight, sizeof(float) * *weight_stride, sizeof(float) * pix, n,
                         cudaMemcpyHostToDevice, ctx->stream));
    *weight = w, *weight_stride = pix;
  }
  return OFDIS_OK;
}

// ofdis_fuse_push (weighted false) and ofdis_fuse_push_weighted
static int fuse_push_impl(ofdis_ctx* ctx, bool weighted, int n, const float* disp, size_t disp_stride,
                          const double* poses, const ofdis_stereo_camera* cam, float max_depth,
                          const unsigned char* frames, size_t frame_stride, const float* weight, size_t weight_stride,
                          int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  const char* name = weighted ? "fuse_push_weighted" : "fuse_push";
  if (!ctx->fuse_on) return fail(ctx, OFDIS_ERR_ARG, (std::string(name) + ": no live volume (ofdis_fuse_begin)").c_str());
  const bool dev = memkind == OFDIS_MEM_DEVICE, color = ctx->fuse_vol.C != nullptr;
  const size_t pix = (size_t)std::max(width_org, 0) * std::max(height_org, 0), hwc = pix * ctx->prm.noc;
  if (n < 1 || n > ctx->max_frames + 1 || !disp || !poses || (color && !frames) || !fuse_cam_ok(cam) ||
      !(max_depth > 0.0f) || disp_stride < pix || (color && frame_stride < hwc) ||
      (dev && reinterpret_cast<uintptr_t>(disp) % sizeof(float)) ||
      (weighted && (!weight || weight_stride < pix || (dev && reinterpret_cast<uintptr_t>(weight) % sizeof(float)))))
    return fail(ctx, OFDIS_ERR_ARG, (std::string(name) + ": bad argument").c_str());
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("fuse", -1);
  CK(cudaSetDevice(ctx->device));
  FusePush fp{};
  fp.disp = disp, fp.disp_stride = disp_stride;
  fp.frames = color ? frames : nullptr, fp.frame_stride = frame_stride;
  fp.n = n, fp.w = width_org, fp.h = height_org, fp.noc = ctx->prm.noc, fp.max_depth = max_depth;
  fp.cam = DispCamera{cam->fx * cam->baseline, cam->fx, cam->fy, cam->cx, cam->cy, cam->doffs};
  fp.g = ctx->fuse_ws.g;
  fp.weight = weighted ? weight : nullptr, fp.weight_stride = weight_stride;
  rc = fuse_poses(ctx, n, poses, true);
  if (rc) return rc;
  if (!dev) {
    rc = fuse_stage(ctx, n, pix, hwc, color, &fp.disp, &fp.disp_stride, &fp.frames, &fp.frame_stride, &fp.weight,
                    &fp.weight_stride);
    if (rc) return rc;
  }
  const int k = launch_fuse_push(ctx->fuse_geom, ctx->fuse_vol, fp, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_integrate_kernel launch", cudaGetLastError());
  ctx->launches += k;
  return OFDIS_OK;
}

int ofdis_fuse_push(ofdis_ctx* ctx, int n, const float* disp, size_t disp_stride, const double* poses,
                    const ofdis_stereo_camera* cam, float max_depth, const unsigned char* frames, size_t frame_stride,
                    int width_org, int height_org, int memkind) {
  return fuse_push_impl(ctx, false, n, disp, disp_stride, poses, cam, max_depth, frames, frame_stride, nullptr, 0,
                        width_org, height_org, memkind);
}

int ofdis_fuse_push_weighted(ofdis_ctx* ctx, int n, const float* disp, size_t disp_stride, const double* poses,
                             const ofdis_stereo_camera* cam, float max_depth, const unsigned char* frames,
                             size_t frame_stride, const float* weight, size_t weight_stride, int width_org,
                             int height_org, int memkind) {
  return fuse_push_impl(ctx, true, n, disp, disp_stride, poses, cam, max_depth, frames, frame_stride, weight,
                        weight_stride, width_org, height_org, memkind);
}

int ofdis_fuse_extract(ofdis_ctx* ctx, float min_weight, ofdis_fuse_point* pts, long capacity, long* count,
                       int memkind) {
  static_assert(sizeof(ofdis_fuse_point) == 28, "ofdis_fuse_point: 28 bytes, as preprocess.FUSE_POINT_DTYPE");
  if (!ctx) return OFDIS_ERR_ARG;
  if (!ctx->fuse_on) return fail(ctx, OFDIS_ERR_ARG, "fuse_extract: no live volume (ofdis_fuse_begin)");
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  if (!count || capacity < 0 || (capacity > 0 && !pts) || std::isnan(min_weight) ||
      (dev && reinterpret_cast<uintptr_t>(pts) % sizeof(float)))
    return fail(ctx, OFDIS_ERR_ARG, "fuse_extract: bad argument");
  NvtxRange nvtx("fuse", -1);
  CK(cudaSetDevice(ctx->device));
  int k = launch_fuse_count(ctx->fuse_geom, ctx->fuse_vol, min_weight, ctx->fuse_ws, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_count_kernel launch", cudaGetLastError());
  ctx->launches += k;
  unsigned long long total = 0;
  ofdis_fuse_point* out = pts;
  long long cap = capacity;
  if (!dev) {
    // the total decides how much of the full-resolution scratch the host output needs
    CK(cudaMemcpyAsync(&total, ctx->fuse_ws.total, sizeof(total), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    cap = (long long)std::min<unsigned long long>(total, (unsigned long long)capacity);
    const int rc = carve(ctx, ctx->d_full, "full-resolution flow buffer",
                         [&](Carve& c) { out = c.take<ofdis_fuse_point>((size_t)cap); });
    if (rc) return rc;
  }
  k = launch_fuse_write(ctx->fuse_geom, ctx->fuse_vol, min_weight, ctx->fuse_ws, out, cap, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_write_kernel launch", cudaGetLastError());
  ctx->launches += k;
  if (!dev && cap > 0)
    CK(cudaMemcpyAsync(pts, out, sizeof(ofdis_fuse_point) * (size_t)cap, cudaMemcpyDeviceToHost, ctx->stream));
  if (dev) CK(cudaMemcpyAsync(&total, ctx->fuse_ws.total, sizeof(total), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  *count = (long)total;
  return OFDIS_OK;
}

int ofdis_fuse_render(ofdis_ctx* ctx, int n, const double* poses, const ofdis_stereo_camera* cam, float z_near,
                      float z_far, float step, float min_weight, float* depth, int width_org, int height_org,
                      int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (!ctx->fuse_on) return fail(ctx, OFDIS_ERR_ARG, "fuse_render: no live volume (ofdis_fuse_begin)");
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  if (n < 1 || n > ctx->max_frames + 1 || !poses || !depth || !fuse_cam_ok(cam) || !finite_gt0(z_near) ||
      !finite_gt0(step) || !(z_far >= z_near && z_far <= FLT_MAX) || !((z_far - z_near) / step <= 65536.0f) ||
      std::isnan(min_weight) || (dev && reinterpret_cast<uintptr_t>(depth) % sizeof(float)))
    return fail(ctx, OFDIS_ERR_ARG, "fuse_render: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("fuse", -1);
  CK(cudaSetDevice(ctx->device));
  const size_t np = (size_t)width_org * height_org * n;
  FuseRender fr{};
  fr.depth = depth;
  if (!dev) {
    const size_t pix = (size_t)width_org * height_org;
    rc = carve_full(ctx, pix, [&](Carve& c) { fr.depth = c.take<float>(pix * (ctx->max_frames + 1)); });
    if (rc) return rc;
  }
  rc = fuse_poses(ctx, n, poses, false);
  if (rc) return rc;
  fr.pose = ctx->fuse_ws.g;
  fr.w = width_org, fr.h = height_org;
  fr.z_near = z_near, fr.z_far = z_far, fr.step = step, fr.min_weight = min_weight;
  fr.cam = DispCamera{cam->fx * cam->baseline, cam->fx, cam->fy, cam->cx, cam->cy, cam->doffs};
  const int k = launch_fuse_render(ctx->fuse_geom, ctx->fuse_vol, fr, n, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_render_kernel launch", cudaGetLastError());
  ctx->launches += k;
  if (!dev) {
    CK(cudaMemcpyAsync(depth, fr.depth, sizeof(float) * np, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return OFDIS_OK;
}

int ofdis_fuse_get_volume(ofdis_ctx* ctx, float* T, float* W, unsigned char* color, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (!ctx->fuse_on) return fail(ctx, OFDIS_ERR_ARG, "fuse_get_volume: no live volume (ofdis_fuse_begin)");
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  const FuseVolume& v = ctx->fuse_vol;
  if ((color && !v.C) || (dev && (reinterpret_cast<uintptr_t>(T) % 4 || reinterpret_cast<uintptr_t>(W) % 4)))
    return fail(ctx, OFDIS_ERR_ARG, "fuse_get_volume: bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)ctx->fuse_geom.count;
  const cudaMemcpyKind kind = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  if (T) CK(cudaMemcpyAsync(T, v.T, 4 * N, kind, ctx->stream));
  if (W) CK(cudaMemcpyAsync(W, v.W, 4 * N, kind, ctx->stream));
  if (color) CK(cudaMemcpyAsync(color, v.C, 3 * N, kind, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

int ofdis_fuse_mesh(ofdis_ctx* ctx, float min_weight, ofdis_fuse_point* pts, long pt_capacity, long* pt_count,
                    unsigned int* faces, long face_capacity, long* face_count, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (!ctx->fuse_on) return fail(ctx, OFDIS_ERR_ARG, "fuse_mesh: no live volume (ofdis_fuse_begin)");
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  if (!pt_count || !face_count || pt_capacity < 0 || face_capacity < 0 || (pt_capacity > 0 && !pts) ||
      (face_capacity > 0 && !faces) || std::isnan(min_weight) ||
      (dev && (reinterpret_cast<uintptr_t>(pts) % sizeof(float) || reinterpret_cast<uintptr_t>(faces) % 4)))
    return fail(ctx, OFDIS_ERR_ARG, "fuse_mesh: bad argument");
  NvtxRange nvtx("fuse", -1);
  CK(cudaSetDevice(ctx->device));
  const FuseGeom& g = ctx->fuse_geom;
  const size_t N = (size_t)g.count, nb = (N + FUSE_BLOCK - 1) / FUSE_BLOCK;
  FuseMeshWork mw;
  const int rc = carve(ctx, ctx->d_mesh, "fuse_mesh workspace", [&](Carve& c) {
    mw.vbase = c.take<unsigned int>(N);
    mw.bsum = c.take<unsigned long long>(nb);
    mw.total = c.take<unsigned long long>(1);
  });
  if (rc) return rc;
  int k = launch_fuse_count(g, ctx->fuse_vol, min_weight, ctx->fuse_ws, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_count_kernel launch", cudaGetLastError());
  ctx->launches += k;
  k = launch_fuse_cube_count(g, ctx->fuse_vol, min_weight, mw, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_cube_count_kernel launch", cudaGetLastError());
  ctx->launches += k;
  unsigned long long total[2] = {0, 0};  // vertices, triangles
  ofdis_fuse_point* out = pts;
  unsigned int* fout = faces;
  long long pcap = pt_capacity, fcap = face_capacity;
  if (!dev) {
    // the totals decide how much of the full-resolution scratch the host outputs need: the points, then the faces
    CK(cudaMemcpyAsync(&total[0], ctx->fuse_ws.total, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(&total[1], mw.total, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    pcap = (long long)std::min<unsigned long long>(total[0], (unsigned long long)pt_capacity);
    fcap = (long long)std::min<unsigned long long>(total[1], (unsigned long long)face_capacity);
    const int rc = carve(ctx, ctx->d_full, "full-resolution flow buffer", [&](Carve& c) {
      out = c.take<ofdis_fuse_point>((size_t)pcap);
      fout = c.take<unsigned int>(3 * (size_t)fcap);
    });
    if (rc) return rc;
  }
  k = launch_fuse_write(g, ctx->fuse_vol, min_weight, ctx->fuse_ws, out, pcap, ctx->stream, mw.vbase);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_write_kernel launch", cudaGetLastError());
  ctx->launches += k;
  k = launch_fuse_faces(g, ctx->fuse_vol, min_weight, mw, fout, fcap, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_face_kernel launch", cudaGetLastError());
  ctx->launches += k;
  if (!dev && pcap > 0)
    CK(cudaMemcpyAsync(pts, out, sizeof(ofdis_fuse_point) * (size_t)pcap, cudaMemcpyDeviceToHost, ctx->stream));
  if (!dev && fcap > 0)
    CK(cudaMemcpyAsync(faces, fout, 12 * (size_t)fcap, cudaMemcpyDeviceToHost, ctx->stream));
  if (dev) {
    CK(cudaMemcpyAsync(&total[0], ctx->fuse_ws.total, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(&total[1], mw.total, 8, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  *pt_count = (long)total[0];
  *face_count = (long)total[1];
  return OFDIS_OK;
}

int ofdis_fuse_set_volume(ofdis_ctx* ctx, const float* T, const float* W, const unsigned char* color, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (!ctx->fuse_on) return fail(ctx, OFDIS_ERR_ARG, "fuse_set_volume: no live volume (ofdis_fuse_begin)");
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  const FuseVolume& v = ctx->fuse_vol;
  if ((color && !v.C) || (dev && (reinterpret_cast<uintptr_t>(T) % 4 || reinterpret_cast<uintptr_t>(W) % 4)))
    return fail(ctx, OFDIS_ERR_ARG, "fuse_set_volume: bad argument");
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)ctx->fuse_geom.count;
  const cudaMemcpyKind kind = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  if (T) CK(cudaMemcpyAsync(v.T, T, 4 * N, kind, ctx->stream));
  if (W) CK(cudaMemcpyAsync(v.W, W, 4 * N, kind, ctx->stream));
  if (color) CK(cudaMemcpyAsync(v.C, color, 3 * N, kind, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

static bool finite_f64(double v) { return std::fabs(v) <= DBL_MAX; }

// ofdis_fuse_track (weighted false) and ofdis_fuse_track_weighted
static int fuse_track_impl(ofdis_ctx* ctx, bool weighted, int n, const float* disp, size_t disp_stride,
                           const double* motions, const double* prev, const ofdis_stereo_camera* cam,
                           const ofdis_fuse_track_params* p, const unsigned char* frames, size_t frame_stride,
                           const float* weight, size_t weight_stride, double* poses, ofdis_fuse_track_stats* stats,
                           int width_org, int height_org, int memkind) {
  static_assert(sizeof(ofdis_fuse_track_stats) == 32, "ofdis_fuse_track_stats: 32 bytes, as FUSE_TRACK_STATS_DTYPE");
  if (!ctx) return OFDIS_ERR_ARG;
  const char* name = weighted ? "fuse_track_weighted" : "fuse_track";
  if (!ctx->fuse_on) return fail(ctx, OFDIS_ERR_ARG, (std::string(name) + ": no live volume (ofdis_fuse_begin)").c_str());
  const bool dev = memkind == OFDIS_MEM_DEVICE, color = ctx->fuse_vol.C != nullptr;
  const size_t pix = (size_t)std::max(width_org, 0) * std::max(height_org, 0), hwc = pix * ctx->prm.noc;
  bool ok = n >= 1 && n <= ctx->max_frames + 1 && disp && prev && poses && stats && fuse_cam_ok(cam) && p &&
            disp_stride >= pix && !(dev && reinterpret_cast<uintptr_t>(disp) % sizeof(float));
  ok = ok && (!weighted || (weight && weight_stride >= pix &&
                            !(dev && reinterpret_cast<uintptr_t>(weight) % sizeof(float))));
  ok = ok && p->step >= 1 && p->rounds >= 0 && p->rounds <= 32 && !std::isnan(p->min_weight) &&
       p->max_depth > 0.0f && finite_gt0(p->huber) && finite_f64(p->damping) && p->damping >= 0.0 &&
       p->min_corr >= 6 && finite_f64(p->max_shift) && p->max_shift > 0.0 && p->min_cos >= -1.0 && p->min_cos <= 1.0 &&
       finite_f64(p->eps) && p->eps >= 0.0 && (p->integrate == 0 || p->integrate == 1);
  const bool use_frames = ok && p->integrate && color;
  ok = ok && (!use_frames || (frames && frame_stride >= hwc));
  for (int i = 0; ok && i < 12; ++i) ok = finite_f64(prev[i]);
  for (size_t i = 0; ok && motions && i < (size_t)12 * n; ++i) ok = finite_f64(motions[i]);
  if (!ok) return fail(ctx, OFDIS_ERR_ARG, (std::string(name) + ": bad argument").c_str());
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("fuse", -1);
  CK(cudaSetDevice(ctx->device));
  FuseTrack t{};
  t.w = width_org, t.h = height_org, t.s = p->step;
  t.ncx = (width_org - 1) / p->step + 1;
  t.cells = t.ncx * ((height_org - 1) / p->step + 1);
  t.nchunks = (t.cells + 31) / 32;
  t.rounds = p->rounds, t.min_corr = p->min_corr, t.has_motion = motions != nullptr;
  t.min_weight = p->min_weight, t.max_depth = p->max_depth, t.huber = p->huber;
  t.damping = p->damping, t.max_shift = p->max_shift, t.min_cos = p->min_cos, t.eps = p->eps;
  t.cam = DispCamera{cam->fx * cam->baseline, cam->fx, cam->fy, cam->cx, cam->cy, cam->doffs};
  // the workspace: the state, the motions, poses and stats of max_frames + 1 frames, the push pose, the chunk sums;
  // host inputs through the staging buffer as the push's
  const size_t F = (size_t)ctx->max_frames + 1;
  rc = carve(ctx, ctx->d_ftrack, "fuse_track workspace", [&](Carve& c) {
    t.state = c.take<FuseTrackState>(1);
    t.motion = c.take<double>(12 * F);
    t.pose = c.take<double>(12 * F);
    t.stats = c.take<ofdis_fuse_track_stats>(F);
    t.g = c.take<float>(12);
    t.chunk = c.take<double>(FTRACK_NE * (size_t)t.nchunks);
  });
  if (rc) return rc;
  t.disp = disp, t.disp_stride = disp_stride;
  const unsigned char* fr = use_frames ? frames : nullptr;
  size_t fstride = frame_stride;
  const float* wt = weighted ? weight : nullptr;
  size_t wstride = weight_stride;
  if (!dev) {
    rc = fuse_stage(ctx, n, pix, hwc, color, &t.disp, &t.disp_stride, &fr, &fstride, &wt, &wstride);
    if (rc) return rc;
  }
  FuseTrackState init{};
  std::memcpy(init.prev, prev, sizeof(init.prev));
  CK(cudaMemcpyAsync(t.state, &init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
  if (motions)
    CK(cudaMemcpyAsync(const_cast<double*>(t.motion), motions, sizeof(double) * 12 * n, cudaMemcpyHostToDevice,
                       ctx->stream));
  // init and motions are pageable host memory: the copies have left them when cudaMemcpyAsync returns
  FusePush fp{};
  fp.g = t.g;
  fp.n = 1, fp.w = width_org, fp.h = height_org, fp.noc = ctx->prm.noc, fp.max_depth = p->max_depth;
  fp.cam = t.cam;
  for (int k = 0; k < n; ++k) {
    for (int r = 0; r <= p->rounds; ++r) {
      const int kk = launch_fuse_track_eval(ctx->fuse_geom, ctx->fuse_vol, t, k, r, ctx->stream,
                                            wt ? wt + (size_t)k * wstride : nullptr);
      if (kk < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_track_kernel launch", cudaGetLastError());
      ctx->launches += kk;
    }
    if (!p->integrate) continue;
    fp.disp = t.disp + (size_t)k * t.disp_stride, fp.disp_stride = t.disp_stride;
    fp.frames = fr ? fr + (size_t)k * fstride : nullptr, fp.frame_stride = fstride;
    fp.weight = wt ? wt + (size_t)k * wstride : nullptr, fp.weight_stride = wstride;
    const int kk = launch_fuse_push(ctx->fuse_geom, ctx->fuse_vol, fp, ctx->stream);
    if (kk < 0) return fail(ctx, OFDIS_ERR_CUDA, "fuse_integrate_kernel launch", cudaGetLastError());
    ctx->launches += kk;
  }
  std::vector<double> P((size_t)12 * n);
  std::vector<ofdis_fuse_track_stats> S(n);
  CK(cudaMemcpyAsync(P.data(), t.pose, sizeof(double) * P.size(), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(S.data(), t.stats, sizeof(ofdis_fuse_track_stats) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  std::memcpy(poses, P.data(), sizeof(double) * P.size());
  std::memcpy(stats, S.data(), sizeof(ofdis_fuse_track_stats) * n);
  return OFDIS_OK;
}

int ofdis_fuse_track(ofdis_ctx* ctx, int n, const float* disp, size_t disp_stride, const double* motions,
                     const double* prev, const ofdis_stereo_camera* cam, const ofdis_fuse_track_params* p,
                     const unsigned char* frames, size_t frame_stride, double* poses, ofdis_fuse_track_stats* stats,
                     int width_org, int height_org, int memkind) {
  return fuse_track_impl(ctx, false, n, disp, disp_stride, motions, prev, cam, p, frames, frame_stride, nullptr, 0,
                         poses, stats, width_org, height_org, memkind);
}

int ofdis_fuse_track_weighted(ofdis_ctx* ctx, int n, const float* disp, size_t disp_stride, const double* motions,
                              const double* prev, const ofdis_stereo_camera* cam, const ofdis_fuse_track_params* p,
                              const unsigned char* frames, size_t frame_stride, const float* weight,
                              size_t weight_stride, double* poses, ofdis_fuse_track_stats* stats, int width_org,
                              int height_org, int memkind) {
  return fuse_track_impl(ctx, true, n, disp, disp_stride, motions, prev, cam, p, frames, frame_stride, weight,
                         weight_stride, poses, stats, width_org, height_org, memkind);
}

// The tracker's workspace for geometry t: the state, two track lists, the flags, the occupancy, the scan blocks'
// sums, the counts of max_frames pairs, then the host-output records of max_frames pairs.  Grows, never shrinks.
static int ensure_track(ofdis_ctx* ctx, const TrackGeom& t) {
  const size_t nflags = (size_t)t.cap_pad + t.cells_pad;
  TrackWork& ws = ctx->track;
  return carve(ctx, ctx->d_track, "track workspace", [&](Carve& c) {
    ws.state = c.take<TrackState>(1);
    ws.list[0] = c.take<ofdis_track_point>(t.capacity);
    ws.list[1] = c.take<ofdis_track_point>(t.capacity);
    ws.flags = c.take<unsigned char>(nflags);
    ws.occ = c.take<unsigned char>(t.cells);
    ws.bsum = c.take<unsigned int>(nflags / TRACK_BLOCK);
    ws.counts = c.take<int>(ctx->max_frames);
    ctx->track_out = c.take<ofdis_track_point>((size_t)t.capacity * ctx->max_frames);
  });
}

// n host frames of hwc bytes, *stride apart, packed into the staging buffer; *frames and *stride then name the copy
static int stage_frames_u8(ofdis_ctx* ctx, int n, size_t hwc, const unsigned char** frames, size_t* stride) {
  unsigned char* st = nullptr;
  const int rc = carve_stage_u8(ctx, hwc, [&](Carve& c) { st = c.take<unsigned char>(hwc * ctx->max_frames); });
  if (rc) return rc;
  CK(cudaMemcpy2DAsync(st, hwc, *frames, *stride, hwc, n, cudaMemcpyHostToDevice, ctx->stream));
  *frames = st, *stride = hwc;
  return OFDIS_OK;
}

int ofdis_track_begin(ofdis_ctx* ctx, const ofdis_track_params* params, const unsigned char* frame,
                      ofdis_track_point* points, int* count, int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  auto finite_nonneg = [](float v) { return v >= 0.f && v <= FLT_MAX; };
  if (!params || params->capacity < 1 || params->capacity > (1 << 24) || params->spacing < 1 ||
      !finite_nonneg(params->alpha) || !finite_nonneg(params->beta) || !finite_nonneg(params->mb_alpha) ||
      !finite_nonneg(params->mb_beta) || std::isnan(params->min_eig) || !frame || !points || !count ||
      (memkind == OFDIS_MEM_DEVICE && reinterpret_cast<uintptr_t>(points) % 4))
    return fail(ctx, OFDIS_ERR_ARG, "track_begin: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("track", -1);
  CK(cudaSetDevice(ctx->device));
  ctx->track_on = false;
  ctx->traj_on = false;
  TrackGeom t{};
  t.w = width_org;
  t.h = height_org;
  t.s = params->spacing;
  t.ncx = (width_org - 1) / t.s + 1;
  const long long cells = (long long)t.ncx * ((height_org - 1) / t.s + 1);
  if (cells > INT_MAX - TRACK_BLOCK) return fail(ctx, OFDIS_ERR_UNSUPPORTED, "track_begin: too many cells");
  t.cells = (int)cells;
  t.cells_pad = (t.cells + TRACK_BLOCK - 1) / TRACK_BLOCK * TRACK_BLOCK;
  t.capacity = params->capacity;
  t.cap_pad = (t.capacity + TRACK_BLOCK - 1) / TRACK_BLOCK * TRACK_BLOCK;
  t.alpha = params->alpha;
  t.beta = params->beta;
  t.mb_alpha = params->mb_alpha;
  t.mb_beta = params->mb_beta;
  t.min_eig = params->min_eig;
  rc = ensure_track(ctx, t);
  if (rc) return rc;
  ctx->tgeom = t;
  const TrackWork& ws = ctx->track;
  const size_t hwc = (size_t)width_org * height_org * ctx->prm.noc;
  const unsigned char* I = frame;
  if (memkind != OFDIS_MEM_DEVICE) {
    unsigned char* st = nullptr;
    rc = carve_stage_u8(ctx, hwc, [&](Carve& c) { st = c.take<unsigned char>(hwc); });
    if (rc) return rc;
    CK(cudaMemcpyAsync(st, frame, hwc, cudaMemcpyHostToDevice, ctx->stream));
    I = st;
  }
  // no track yet: every keep flag and every cell's occupancy is 0
  CK(cudaMemsetAsync(ws.state, 0, sizeof(TrackState), ctx->stream));
  CK(cudaMemsetAsync(ws.flags, 0, t.cap_pad, ctx->stream));
  CK(cudaMemsetAsync(ws.occ, 0, t.cells, ctx->stream));
  ofdis_track_point* out = memkind == OFDIS_MEM_DEVICE ? points : ctx->track_out;
  const int k = launch_track_seed_compact(t, ws, ctx->prm.noc, I, 0, out, 0, ctx->stream);
  if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "track_seed_kernel launch", cudaGetLastError());
  ctx->launches += k;
  ctx->track_cur = 1;
  CK(cudaMemcpyAsync(count, ws.counts, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (memkind != OFDIS_MEM_DEVICE && *count > 0) {
    CK(cudaMemcpyAsync(points, out, sizeof(ofdis_track_point) * *count, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  ctx->track_on = true;
  return OFDIS_OK;
}

int ofdis_track_advance(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* frames, size_t frame_stride,
                        ofdis_track_point* points, int* counts, int width_org, int height_org, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || b0 < 0 || b0 > ctx->max_frames - (f1 - f0) || !frames ||
      !points || !counts || (memkind == OFDIS_MEM_DEVICE && reinterpret_cast<uintptr_t>(points) % 4))
    return fail(ctx, OFDIS_ERR_ARG, "track_advance: bad argument");
  if (!ctx->track_on) return fail(ctx, OFDIS_ERR_ARG, "track_advance: no ofdis_track_begin");
  ctx->traj_on = false;
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  const TrackGeom& t = ctx->tgeom;
  if (width_org != t.w || height_org != t.h)
    return fail(ctx, OFDIS_ERR_ARG, "track_advance: frame size differs from ofdis_track_begin's");
  const size_t hwc = (size_t)width_org * height_org * ctx->prm.noc;
  if (frame_stride < hwc) return fail(ctx, OFDIS_ERR_ARG, "track_advance: frame_stride below one frame");
  NvtxRange nvtx("track", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0, D = ctx->dirs;
  const TrackWork& ws = ctx->track;
  const unsigned char* src = frames;
  size_t stride = frame_stride;
  if (memkind != OFDIS_MEM_DEVICE) {
    rc = stage_frames_u8(ctx, n, hwc, &src, &stride);
    if (rc) return rc;
  }
  ofdis_track_point* out = memkind == OFDIS_MEM_DEVICE ? points : ctx->track_out;
  const LevelGeom g = stepped(ctx->lev[0], D);
  // a call that fails on the way leaves the tracker to a new ofdis_track_begin
  ctx->track_on = false;
  int cur = ctx->track_cur;
  for (int k = 0; k < n; ++k) {
    if (launch_track_advance(g, (f0 + k) * D, (b0 + k) * D, t, ws, cur, cx, cy, ctx->stream) < 0)
      return fail(ctx, OFDIS_ERR_CUDA, "track_advance_kernel launch", cudaGetLastError());
    const int l = launch_track_seed_compact(t, ws, ctx->prm.noc, src + k * stride, cur, out + (size_t)k * t.capacity,
                                            k, ctx->stream);
    if (l < 0) return fail(ctx, OFDIS_ERR_CUDA, "track_seed_kernel launch", cudaGetLastError());
    ctx->launches += 1 + l;
    cur ^= 1;
  }
  ctx->track_cur = cur;
  CK(cudaMemcpyAsync(counts, ws.counts, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (memkind != OFDIS_MEM_DEVICE) {
    for (int k = 0; k < n; ++k)
      if (counts[k] > 0)
        CK(cudaMemcpyAsync(points + (size_t)k * t.capacity, out + (size_t)k * t.capacity,
                           sizeof(ofdis_track_point) * counts[k], cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  ctx->track_on = true;
  return OFDIS_OK;
}

int ofdis_track_stats_get(const ofdis_ctx* ctx, ofdis_track_stats* out) {
  if (!ctx || !out || !ctx->track_on) return OFDIS_ERR_ARG;
  TrackState s;
  if (cudaSetDevice(ctx->device) != cudaSuccess ||
      cudaMemcpyAsync(&s, ctx->track.state, sizeof(s), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return OFDIS_ERR_CUDA;
  out->seeded = (long long)s.seeded;
  out->ended_leaves = (long long)s.ended[0];
  out->ended_inconsistent = (long long)s.ended[1];
  out->ended_boundary = (long long)s.ended[2];
  out->dropped = (long long)s.dropped;
  out->alive = s.alive;
  out->next_id = s.next_id;
  return OFDIS_OK;
}

// A received model through the stabiliser's validity rule (stab_kernels.cu): divided by its m22 into q, which stays
// as it is (the identity) when m22 is not finite and non-zero, an entry is not finite or m00*m11 - m01*m10 is not
// finite and non-zero
static void stab_valid_model(const double* m, double* q) {
  const double d = m[8];
  double M[9];
  bool ok = std::isfinite(d) && d != 0.0;
  for (int i = 0; i < 9; ++i) {
    M[i] = m[i] / d;
    ok = ok && std::isfinite(M[i]);
  }
  if (ok) {
    const double a = M[0] * M[4] - M[1] * M[3];
    ok = std::isfinite(a) && a != 0.0;
  }
  if (ok) std::memcpy(q, M, sizeof(M));
}

// The bound of the segments a call of n pairs emits (ofdis_traj_advance's header)
static size_t traj_bound(const TrajGeom& tg, int capacity, int n) {
  return (size_t)capacity * (size_t)((n + tg.L - 1 + tg.L - 1) / tg.L);
}

// The descriptor stage's workspace for tracker geometry t and descriptor geometry tg: the state, two state lists and
// their metadata, the per-slot scan arrays, the per-pixel fields, the models of max_frames pairs, the kept frame,
// then the host-output records and descriptors of max_frames pairs.  Grows, never shrinks.
static int ensure_traj(ofdis_ctx* ctx, const TrackGeom& t, const TrajGeom& tg) {
  const size_t cp = (size_t)t.cap_pad, px = (size_t)tg.w * tg.h;
  const size_t bound = traj_bound(tg, t.capacity, ctx->max_frames);
  TrajWork& tw = ctx->traj;
  return carve(ctx, ctx->d_traj, "traj workspace", [&](Carve& c) {
    tw.state = c.take<TrajState>(1);
    tw.st[0] = c.take<float>(tg.ss * cp);
    tw.st[1] = c.take<float>(tg.ss * cp);
    tw.meta[0] = c.take<int2>(cp);
    tw.meta[1] = c.take<int2>(cp);
    tw.bins = c.take<uchar4>(px);
    tw.mag = c.take<float4>(2 * px);
    tw.res = c.take<float2>(px);
    tw.models = c.take<float>(9 * ctx->max_frames);
    tw.dst = c.take<int>(cp);
    tw.eoff = c.take<int>(cp);
    tw.seg = c.take<TrajSeg>(cp);
    tw.ebsum = c.take<unsigned int>(cp / TRACK_BLOCK);
    tw.ndesc = c.take<int>(ctx->max_frames);
    tw.frame = c.take<unsigned char>(px * ctx->prm.noc);
    ctx->traj_rec = c.take<ofdis_traj_record>(bound);
    ctx->traj_desc = c.take<float>(tg.dim * bound);
  });
}

int ofdis_traj_begin(ofdis_ctx* ctx, const ofdis_track_params* params, const ofdis_traj_params* traj,
                     const unsigned char* frame, ofdis_track_point* points, int* count, int width_org, int height_org,
                     int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  auto finite = [](float v) { return std::isfinite(v); };
  if (ctx->nop != 2 || !traj || traj->L < 1 || traj->L > 64 || traj->nt < 1 || traj->L % traj->nt ||
      traj->ns < 1 || traj->ns > TRAJ_MAX_NS || traj->N < 1 || traj->N % traj->ns ||
      traj->N > std::min(width_org, height_org) || !finite(traj->min_flow) || !finite(traj->eps) ||
      !(traj->eps > 0.f) || !finite(traj->min_disp) || !(traj->min_disp >= 0.f) || !finite(traj->min_var) ||
      !finite(traj->max_var) || !finite(traj->max_dis))
    return fail(ctx, OFDIS_ERR_ARG, "traj_begin: bad argument");
  int rc = ofdis_track_begin(ctx, params, frame, points, count, width_org, height_org, memkind);
  if (rc) return rc;
  NvtxRange nvtx("traj", -1);
  TrajGeom tg{};
  tg.w = width_org;
  tg.h = height_org;
  tg.L = traj->L;
  tg.nt = traj->nt;
  tg.N = traj->N;
  tg.ns = traj->ns;
  tg.c = traj->N / traj->ns;
  tg.tl = traj->L / traj->nt;
  tg.pos = 2 * (tg.L + 1);
  tg.dis = 2 * tg.L;
  tg.nacc = tg.nt * tg.ns * tg.ns * TRAJ_BINS;
  tg.ss = (tg.pos + tg.dis + tg.nacc + 3) / 4 * 4;
  tg.dim = tg.dis + tg.nacc;
  tg.min_flow = traj->min_flow;
  tg.eps = traj->eps;
  tg.min_disp = traj->min_disp;
  tg.min_var = traj->min_var;
  tg.max_var = traj->max_var;
  tg.max_dis = traj->max_dis;
  const TrackGeom& t = ctx->tgeom;
  rc = ensure_traj(ctx, t, tg);
  if (rc) return rc;
  ctx->trgeom = tg;
  const TrajWork& tw = ctx->traj;
  const size_t hwc = (size_t)width_org * height_org * ctx->prm.noc;
  // frame 0's tracks start their first segment at frame 0; track_begin staged a host frame in d_stage
  CK(cudaMemsetAsync(tw.state, 0, sizeof(TrajState), ctx->stream));
  CK(cudaMemsetAsync(tw.meta[ctx->track_cur], 0, sizeof(int2) * t.cap_pad, ctx->stream));
  CK(cudaMemcpyAsync(tw.frame, memkind == OFDIS_MEM_DEVICE ? frame : static_cast<const unsigned char*>(ctx->d_stage.p),
                     hwc, cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->traj_frame = 0;
  ctx->traj_on = true;
  return OFDIS_OK;
}

static int fisher_push_chunks(ofdis_ctx* ctx, const float* desc, long n, bool host);

// ofdis_traj_advance, and with to_fisher (records and desc unused) ofdis_traj_advance_fisher: the emitted segments'
// descriptors stay in the stage's device output and go into the live encoder
static int traj_advance_impl(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* frames, size_t frame_stride,
                             const double* models, ofdis_track_point* points, int* counts, ofdis_traj_record* records,
                             float* desc, int* n_desc, int width_org, int height_org, int memkind, bool to_fisher) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (ctx->nop != 2 || f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || b0 < 0 || b0 > ctx->max_frames - (f1 - f0) ||
      !frames || !points || !counts || (!to_fisher && (!records || !desc)) || !n_desc ||
      (memkind == OFDIS_MEM_DEVICE && (reinterpret_cast<uintptr_t>(points) % 4 ||
                                       reinterpret_cast<uintptr_t>(records) % 4 ||
                                       reinterpret_cast<uintptr_t>(desc) % 4)))
    return fail(ctx, OFDIS_ERR_ARG, "traj_advance: bad argument");
  if (!ctx->traj_on || !ctx->track_on) return fail(ctx, OFDIS_ERR_ARG, "traj_advance: no ofdis_traj_begin");
  if (to_fisher && (!ctx->fisher_on || ctx->fgeom.desc_dim != ctx->trgeom.dim))
    return fail(ctx, OFDIS_ERR_ARG, "traj_advance_fisher: no live encoder of the descriptors' size");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  const TrackGeom& t = ctx->tgeom;
  const TrajGeom& tg = ctx->trgeom;
  if (width_org != t.w || height_org != t.h)
    return fail(ctx, OFDIS_ERR_ARG, "traj_advance: frame size differs from ofdis_traj_begin's");
  const size_t hwc = (size_t)width_org * height_org * ctx->prm.noc;
  if (frame_stride < hwc) return fail(ctx, OFDIS_ERR_ARG, "traj_advance: frame_stride below one frame");
  NvtxRange nvtx("traj", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0, D = ctx->dirs;
  // the models through the stabiliser's validity rule, rounded to float32 (models == NULL: the identity)
  std::vector<float> m32(9 * (size_t)n);
  for (int k = 0; k < n; ++k) {
    double q[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (models) stab_valid_model(models + 9 * (size_t)k, q);
    for (int i = 0; i < 9; ++i) m32[9 * (size_t)k + i] = (float)q[i];
  }
  const TrackWork& ws = ctx->track;
  const TrajWork& tw = ctx->traj;
  const unsigned char* src = frames;
  size_t stride = frame_stride;
  if (memkind != OFDIS_MEM_DEVICE) {
    rc = stage_frames_u8(ctx, n, hwc, &src, &stride);
    if (rc) return rc;
  }
  ofdis_track_point* out = memkind == OFDIS_MEM_DEVICE ? points : ctx->track_out;
  ofdis_traj_record* rout = memkind == OFDIS_MEM_DEVICE && !to_fisher ? records : ctx->traj_rec;
  float* dout = memkind == OFDIS_MEM_DEVICE && !to_fisher ? desc : ctx->traj_desc;
  const LevelGeom g = stepped(ctx->lev[0], D);
  // a call that fails on the way leaves the tracker and the descriptor stage to a new ofdis_traj_begin
  ctx->track_on = false;
  ctx->traj_on = false;
  CK(cudaMemcpyAsync(tw.models, m32.data(), sizeof(float) * m32.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(&tw.state->total, 0, sizeof(int), ctx->stream));
  int cur = ctx->track_cur;
  for (int k = 0; k < n; ++k) {
    const unsigned char* I = k == 0 ? tw.frame : src + (k - 1) * stride;
    const int l0 = launch_traj_frame(g, (f0 + k) * D, tg, t, tw, ws, ctx->prm.noc, I, tw.models + 9 * k, cur, cx, cy,
                                     ctx->stream);
    if (l0 < 0) return fail(ctx, OFDIS_ERR_CUDA, "traj_field_kernel launch", cudaGetLastError());
    if (launch_track_advance(g, (f0 + k) * D, (b0 + k) * D, t, ws, cur, cx, cy, ctx->stream) < 0)
      return fail(ctx, OFDIS_ERR_CUDA, "track_advance_kernel launch", cudaGetLastError());
    const int l = launch_track_seed_compact(t, ws, ctx->prm.noc, src + k * stride, cur, out + (size_t)k * t.capacity,
                                            k, ctx->stream);
    if (l < 0) return fail(ctx, OFDIS_ERR_CUDA, "track_seed_kernel launch", cudaGetLastError());
    const int l1 = launch_traj_step(tg, t, tw, ws, cur, ctx->traj_frame + k, k, rout, dout, ctx->stream);
    if (l1 < 0) return fail(ctx, OFDIS_ERR_CUDA, "traj_flag_kernel launch", cudaGetLastError());
    ctx->launches += l0 + 1 + l + l1;
    cur ^= 1;
  }
  ctx->track_cur = cur;
  CK(cudaMemcpyAsync(tw.frame, src + (n - 1) * stride, hwc, cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaMemcpyAsync(counts, ws.counts, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(n_desc, tw.ndesc, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (memkind != OFDIS_MEM_DEVICE) {
    for (int k = 0; k < n; ++k)
      if (counts[k] > 0)
        CK(cudaMemcpyAsync(points + (size_t)k * t.capacity, out + (size_t)k * t.capacity,
                           sizeof(ofdis_track_point) * counts[k], cudaMemcpyDeviceToHost, ctx->stream));
    size_t total = 0;
    for (int k = 0; k < n; ++k) total += (size_t)n_desc[k];
    if (total && !to_fisher) {
      CK(cudaMemcpyAsync(records, rout, sizeof(ofdis_traj_record) * total, cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaMemcpyAsync(desc, dout, sizeof(float) * tg.dim * total, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream));
  }
  if (to_fisher) {
    long total = 0;
    for (int k = 0; k < n; ++k) total += n_desc[k];
    rc = fisher_push_chunks(ctx, dout, total, false);
    if (rc) return rc;
  }
  ctx->traj_frame += n;
  ctx->track_on = true;
  ctx->traj_on = true;
  return OFDIS_OK;
}

int ofdis_traj_advance(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* frames, size_t frame_stride,
                       const double* models, ofdis_track_point* points, int* counts, ofdis_traj_record* records,
                       float* desc, int* n_desc, int width_org, int height_org, int memkind) {
  return traj_advance_impl(ctx, f0, f1, b0, frames, frame_stride, models, points, counts, records, desc, n_desc,
                           width_org, height_org, memkind, false);
}

int ofdis_traj_advance_fisher(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* frames,
                              size_t frame_stride, const double* models, ofdis_track_point* points, int* counts,
                              int* n_desc, int width_org, int height_org, int memkind) {
  return traj_advance_impl(ctx, f0, f1, b0, frames, frame_stride, models, points, counts, nullptr, nullptr, n_desc,
                           width_org, height_org, memkind, true);
}

int ofdis_traj_stats_get(const ofdis_ctx* ctx, ofdis_traj_stats* out) {
  if (!ctx || !out || !ctx->traj_on) return OFDIS_ERR_ARG;
  TrajState s;
  if (cudaSetDevice(ctx->device) != cudaSuccess ||
      cudaMemcpyAsync(&s, ctx->traj.state, sizeof(s), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return OFDIS_ERR_CUDA;
  out->emitted = (long long)s.emitted;
  out->rejected_static = (long long)s.reason[0];
  out->rejected_erratic = (long long)s.reason[1];
  out->rejected_jump = (long long)s.reason[2];
  out->rejected_camera = (long long)s.reason[3];
  return OFDIS_OK;
}

// The stabiliser's workspace for frames of hwc bytes at radius r: the frame ring (r + max_frames frames), the model
// ring (2r + max_frames models) and max(r, max_frames) records.  Grows, never shrinks.
static int ensure_stab(ofdis_ctx* ctx, size_t hwc, int r) {
  const int ring = r + ctx->max_frames, mring = 2 * r + ctx->max_frames, nrec = std::max(r, ctx->max_frames);
  const int rc = carve(ctx, ctx->d_stab, "stab workspace", [&](Carve& c) {
    ctx->stab.frames = c.take<unsigned char>(hwc * ring);
    ctx->stab.models = c.take<double>(9 * (size_t)mring);
    ctx->stab.rec = c.take<StabRec>(nrec);
  });
  if (rc) return rc;
  ctx->sgeom.ring = ring;
  ctx->sgeom.mring = mring;
  return OFDIS_OK;
}

int ofdis_stab_begin(ofdis_ctx* ctx, const ofdis_stab_params* p, const double* weights, const unsigned char* frame0,
                     int width_org, int height_org, int memkind) {
  static_assert(sizeof(ofdis_stab_frame) == 96, "ofdis_stab_frame: 96 bytes, as preprocess.STAB_FRAME_DTYPE");
  if (!ctx) return OFDIS_ERR_ARG;
  bool ok = p && p->radius >= 1 && p->radius <= STAB_MAX_RADIUS && p->crop >= 0.f && p->crop < 0.5f &&
            (p->limit == 0 || p->limit == 1) && weights && frame0 && weights[0] > 0.0;
  for (int d = 0; ok && d <= p->radius; ++d) ok = weights[d] >= 0.0 && weights[d] <= DBL_MAX;
  if (!ok) return fail(ctx, OFDIS_ERR_ARG, "stab_begin: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("stab", -1);
  CK(cudaSetDevice(ctx->device));
  ctx->stab_on = false;
  const size_t hwc = (size_t)width_org * height_org * ctx->prm.noc;
  rc = ensure_stab(ctx, hwc, p->radius);
  if (rc) return rc;
  StabGeom& sg = ctx->sgeom;
  sg.w = width_org;
  sg.h = height_org;
  sg.noc = ctx->prm.noc;
  sg.radius = p->radius;
  sg.limit = p->limit;
  sg.crop = p->crop;
  for (int d = 0; d <= STAB_MAX_RADIUS; ++d) sg.wt[d] = d <= p->radius ? weights[d] : 0.0;
  CK(cudaMemcpyAsync(ctx->stab.frames, frame0, hwc,
                     memkind == OFDIS_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->stab_last = ctx->stab_next = 0;
  ctx->stab_on = true;
  return OFDIS_OK;
}

// Emits frames stab_next .. stab_next + count - 1 (windows cut at L with cut) to out and info, then synchronises.
static int stab_emit(ofdis_ctx* ctx, int count, int cut, unsigned char* out, ofdis_stab_frame* info, int memkind) {
  StabGeom sg = ctx->sgeom;
  sg.count = count;
  sg.cut = cut;
  sg.next = ctx->stab_next;
  sg.last = ctx->stab_last;
  sg.slot0 = (int)(ctx->stab_next % sg.ring);
  const size_t pix = (size_t)sg.w * sg.h, hwc = pix * sg.noc;
  std::vector<StabRec> rec(count);
  if (count > 0) {
    unsigned char* dout = out;
    if (memkind != OFDIS_MEM_DEVICE) {
      // at the scratch's start, which sg.vec finds aligned
      const size_t frames = (size_t)std::max(sg.radius, ctx->max_frames);
      const int rc = carve_full(ctx, pix, [&](Carve& c) { dout = c.take<unsigned char>(hwc * frames); });
      if (rc) return rc;
    }
    sg.vec = sg.w % 4 == 0 && reinterpret_cast<uintptr_t>(dout) % 4 == 0;
    const int k = launch_stab(sg, ctx->stab, dout, ctx->stream);
    if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "stab kernel launch", cudaGetLastError());
    ctx->launches += k;
    if (memkind != OFDIS_MEM_DEVICE) CK(cudaMemcpyAsync(out, dout, hwc * count, cudaMemcpyDeviceToHost, ctx->stream));
    if (info) CK(cudaMemcpyAsync(rec.data(), ctx->stab.rec, sizeof(StabRec) * count, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < count && info; ++i) info[i] = rec[i].info;
  return OFDIS_OK;
}

int ofdis_stab_push(ofdis_ctx* ctx, int n, const double* models, const unsigned char* frames, size_t frame_stride,
                    unsigned char* out, ofdis_stab_frame* info, int* n_out, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (n < 1 || n > ctx->max_frames || !models || !frames || !out || !n_out)
    return fail(ctx, OFDIS_ERR_ARG, "stab_push: bad argument");
  if (!ctx->stab_on) return fail(ctx, OFDIS_ERR_ARG, "stab_push: no live stabiliser (ofdis_stab_begin)");
  const StabGeom& sg = ctx->sgeom;
  const size_t hwc = (size_t)sg.w * sg.h * sg.noc;
  if (frame_stride < hwc) return fail(ctx, OFDIS_ERR_ARG, "stab_push: frame_stride below one frame");
  NvtxRange nvtx("stab", -1);
  CK(cudaSetDevice(ctx->device));
  *n_out = 0;
  // a call that fails on the way leaves the stabiliser to a new ofdis_stab_begin
  ctx->stab_on = false;
  const long long L = ctx->stab_last;
  const cudaMemcpyKind kin = memkind == OFDIS_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  // frames L+1 .. L+n and models L .. L+n-1 into their rings, in at most two runs each across the wrap
  for (int k = 0, run; k < n; k += run) {
    const int slot = (int)((L + 1 + k) % sg.ring);
    run = std::min(n - k, sg.ring - slot);
    CK(cudaMemcpy2DAsync(ctx->stab.frames + (size_t)slot * hwc, hwc, frames + (size_t)k * frame_stride, frame_stride,
                         hwc, run, kin, ctx->stream));
  }
  for (int k = 0, run; k < n; k += run) {
    const int slot = (int)((L + k) % sg.mring);
    run = std::min(n - k, sg.mring - slot);
    CK(cudaMemcpyAsync(ctx->stab.models + (size_t)slot * 9, models + (size_t)k * 9, sizeof(double) * 9 * run,
                       cudaMemcpyHostToDevice, ctx->stream));
  }
  ctx->stab_last = L + n;
  const long long last_emitted = ctx->stab_last - sg.radius;
  const int count = last_emitted >= ctx->stab_next ? (int)(last_emitted - ctx->stab_next + 1) : 0;
  const int rc = stab_emit(ctx, count, 0, out, info, memkind);
  if (rc) return rc;
  ctx->stab_next += count;
  *n_out = count;
  ctx->stab_on = true;
  return OFDIS_OK;
}

int ofdis_stab_finish(ofdis_ctx* ctx, unsigned char* out, ofdis_stab_frame* info, int* n_out, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (!out || !n_out) return fail(ctx, OFDIS_ERR_ARG, "stab_finish: bad argument");
  if (!ctx->stab_on) return fail(ctx, OFDIS_ERR_ARG, "stab_finish: no live stabiliser (ofdis_stab_begin)");
  NvtxRange nvtx("stab", -1);
  CK(cudaSetDevice(ctx->device));
  *n_out = 0;
  ctx->stab_on = false;
  const int count = (int)(ctx->stab_last - ctx->stab_next + 1);
  const int rc = stab_emit(ctx, count, 1, out, info, memkind);
  if (rc) return rc;
  ctx->stab_next += count;
  *n_out = count;
  return OFDIS_OK;
}

// The encoder's workspace for geometry g: the codebook (body floats), the statistics, the counts, per chunk the
// staging, y, the posteriors and the skip flags, then the host-output vector.  Grows, never shrinks.
static int ensure_fisher(ofdis_ctx* ctx, const FisherGeom& g, size_t body, size_t nstats) {
  const size_t C = FISHER_CHUNK;
  FisherWork& w = ctx->fisher;
  return carve(ctx, ctx->d_fisher, "fisher workspace", [&](Carve& c) {
    w.cb = c.take<float>(body);
    w.stats = c.take<double>(nstats);
    w.count = c.take<unsigned long long>(2 * FISHER_MAX_BLOCKS);
    w.x = c.take<float>(C * g.desc_dim);
    w.y = c.take<float>(C * g.ydim);
    w.gamma = c.take<float>(C * g.nblocks * g.K);
    w.skip = c.take<unsigned char>(C * g.nblocks);
    w.fv = c.take<float>(2 * (size_t)g.K * g.ydim);
  });
}

static size_t fisher_nstats(const FisherGeom& g) {
  size_t n = 0;
  for (int b = 0; b < g.nblocks; ++b) n += (size_t)g.K * (1 + 2 * g.dim[b]);
  return n;
}

// zero statistics and counts for a new clip (enqueued)
static int fisher_reset(ofdis_ctx* ctx) {
  CK(cudaMemsetAsync(ctx->fisher.stats, 0, sizeof(double) * fisher_nstats(ctx->fgeom), ctx->stream));
  CK(cudaMemsetAsync(ctx->fisher.count, 0, sizeof(unsigned long long) * 2 * FISHER_MAX_BLOCKS, ctx->stream));
  ctx->fisher_pushed = 0;
  return OFDIS_OK;
}

int ofdis_fisher_begin(ofdis_ctx* ctx, const ofdis_fisher_codebook* cb) {
  static_assert(sizeof(ofdis_fisher_stats) == 136, "ofdis_fisher_stats: 136 bytes, as preprocess.FISHER_STATS_DTYPE");
  static_assert(OFDIS_FISHER_MAX_BLOCKS == FISHER_MAX_BLOCKS, "one block limit");
  if (!ctx) return OFDIS_ERR_ARG;
  bool ok = cb && cb->params && cb->K >= 1 && cb->K <= FISHER_MAX_K && cb->nblocks >= 1 &&
            cb->nblocks <= FISHER_MAX_BLOCKS && cb->desc_dim >= 1;
  FisherGeom g{};
  size_t body = 0, fv = 0, nst = 0;
  for (int b = 0; ok && b < cb->nblocks; ++b) {
    const ofdis_fisher_block& bl = cb->blocks[b];
    ok = bl.dim >= 1 && bl.dim <= bl.dim_in && bl.dim_in <= FISHER_MAX_DIM && bl.offset >= 0 &&
         (long long)bl.offset + bl.dim_in <= cb->desc_dim;
    if (!ok) break;
    const size_t K = cb->K, D = bl.dim_in, P = bl.dim;
    g.off[b] = bl.offset;
    g.din[b] = bl.dim_in;
    g.dim[b] = bl.dim;
    g.yoff[b] = g.ydim;
    g.ydim += bl.dim;
    g.poff[b] = (long long)body;
    g.foff[b] = (long long)fv;
    g.soff[b] = (long long)nst;
    // mean, proj and mu finite; isig finite and > 0; c finite; w finite and > 0
    const float* a = cb->params + body;
    for (size_t i = 0; ok && i < D + P * D + K * P; ++i) ok = finite_f32(a[i]);
    a += D + P * D + K * P;
    for (size_t i = 0; ok && i < K * P; ++i) ok = finite_gt0(a[i]);
    a += K * P;
    for (size_t i = 0; ok && i < K; ++i) ok = finite_f32(a[i]);
    a += K;
    for (size_t i = 0; ok && i < K; ++i) ok = finite_gt0(a[i]);
    body += D + P * D + 2 * K * P + 2 * K;
    fv += 2 * K * P;
    nst += K * (1 + 2 * P);
  }
  if (!ok) return fail(ctx, OFDIS_ERR_ARG, "fisher_begin: bad codebook");
  g.K = cb->K;
  g.nblocks = cb->nblocks;
  g.desc_dim = cb->desc_dim;
  NvtxRange nvtx("fisher", -1);
  CK(cudaSetDevice(ctx->device));
  ctx->fisher_on = false;
  int rc = ensure_fisher(ctx, g, body, nst);
  if (rc) return rc;
  ctx->fgeom = g;
  CK(cudaMemcpyAsync(ctx->fisher.cb, cb->params, sizeof(float) * body, cudaMemcpyHostToDevice, ctx->stream));
  rc = fisher_reset(ctx);
  if (rc) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->fisher_on = true;
  return OFDIS_OK;
}

// n descriptors into the live encoder, in chunks (host input through the staging buffer), one synchronise at the end
static int fisher_push_chunks(ofdis_ctx* ctx, const float* desc, long n, bool host) {
  // a call that fails on the way leaves the encoder to a new ofdis_fisher_begin
  ctx->fisher_on = false;
  const FisherGeom& g = ctx->fgeom;
  for (long c0 = 0; c0 < n; c0 += FISHER_CHUNK) {
    const int m = (int)std::min<long>(FISHER_CHUNK, n - c0);
    const float* x = desc + (size_t)c0 * g.desc_dim;
    if (host) {
      CK(cudaMemcpyAsync(ctx->fisher.x, x, sizeof(float) * (size_t)m * g.desc_dim, cudaMemcpyHostToDevice,
                         ctx->stream));
      x = ctx->fisher.x;
    }
    const int k = launch_fisher_chunk(g, ctx->fisher, x, m, ctx->stream);
    if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fisher kernel launch", cudaGetLastError());
    ctx->launches += k;
  }
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->fisher_pushed += n;
  ctx->fisher_on = true;
  return OFDIS_OK;
}

int ofdis_fisher_push(ofdis_ctx* ctx, const float* desc, long n, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (n < 0 || (!desc && n > 0) || (memkind == OFDIS_MEM_DEVICE && reinterpret_cast<uintptr_t>(desc) % 4 != 0))
    return fail(ctx, OFDIS_ERR_ARG, "fisher_push: bad argument");
  if (!ctx->fisher_on) return fail(ctx, OFDIS_ERR_ARG, "fisher_push: no live encoder (ofdis_fisher_begin)");
  if (n == 0) return OFDIS_OK;
  NvtxRange nvtx("fisher", -1);
  CK(cudaSetDevice(ctx->device));
  return fisher_push_chunks(ctx, desc, n, memkind != OFDIS_MEM_DEVICE);
}

int ofdis_fisher_take(ofdis_ctx* ctx, float* fv, double* stats, ofdis_fisher_stats* out, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  if (dev && (reinterpret_cast<uintptr_t>(fv) % 4 != 0 || reinterpret_cast<uintptr_t>(stats) % 8 != 0))
    return fail(ctx, OFDIS_ERR_ARG, "fisher_take: bad argument");
  if (!ctx->fisher_on) return fail(ctx, OFDIS_ERR_ARG, "fisher_take: no live encoder (ofdis_fisher_begin)");
  NvtxRange nvtx("fisher", -1);
  CK(cudaSetDevice(ctx->device));
  ctx->fisher_on = false;
  const FisherGeom& g = ctx->fgeom;
  const cudaMemcpyKind kout = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  if (fv) {
    float* dfv = dev ? fv : ctx->fisher.fv;
    const int k = launch_fisher_take(g, ctx->fisher, dfv, ctx->stream);
    if (k < 0) return fail(ctx, OFDIS_ERR_CUDA, "fisher kernel launch", cudaGetLastError());
    ctx->launches += k;
    if (!dev) CK(cudaMemcpyAsync(fv, dfv, sizeof(float) * 2 * g.K * g.ydim, kout, ctx->stream));
  }
  if (stats) CK(cudaMemcpyAsync(stats, ctx->fisher.stats, sizeof(double) * fisher_nstats(g), kout, ctx->stream));
  unsigned long long cnt[2 * FISHER_MAX_BLOCKS];
  CK(cudaMemcpyAsync(cnt, ctx->fisher.count, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
  const long long pushed = ctx->fisher_pushed;
  const int rc = fisher_reset(ctx);
  if (rc) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  if (out) {
    std::memset(out, 0, sizeof(*out));
    out->pushed = pushed;
    for (int b = 0; b < g.nblocks; ++b) {
      out->n[b] = (long long)cnt[b];
      out->skipped[b] = (long long)cnt[FISHER_MAX_BLOCKS + b];
    }
  }
  ctx->fisher_on = true;
  return OFDIS_OK;
}

static constexpr int kEvalMaxClasses = 16;

int ofdis_flow_error_fullres(ofdis_ctx* ctx, int f0, int f1, const float* gt, const unsigned char* classes,
                             int nclasses, ofdis_error_stats* stats, float* err, int width_org, int height_org,
                             int memkind) {
  static_assert(sizeof(ofdis_error_stats) == 48, "ofdis_error_stats: 48 bytes, as api.ERROR_STATS_DTYPE");
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !gt || !stats || nclasses < 1 || nclasses > kEvalMaxClasses ||
      (!classes && nclasses > 1))
    return fail(ctx, OFDIS_ERR_ARG, "flow_error_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("evaluate", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0;
  const size_t pix = (size_t)width_org * height_org, nop = (size_t)ctx->nop;
  ErrRowPartial* part = nullptr;
  ofdis_error_stats* dstats = nullptr;
  rc = carve(ctx, ctx->d_eval, "flow_error_fullres workspace", [&](Carve& c) {
    part = c.take<ErrRowPartial>((size_t)ctx->max_frames * kEvalMaxClasses * ctx->height);
    dstats = c.take<ofdis_error_stats>((size_t)ctx->max_frames * kEvalMaxClasses);
  });
  if (rc) return rc;
  const float* dgt = gt;
  const unsigned char* dcls = classes;
  float* derr = err;
  if (memkind != OFDIS_MEM_DEVICE) {
    // gt and the classes go in, err comes out through the same scratch
    const size_t cap = pix * ctx->max_frames;
    float* sgt = nullptr;
    unsigned char* scls = nullptr;
    rc = carve_full(ctx, pix, [&](Carve& c) {
      sgt = c.take<float>(nop * cap);
      derr = c.take<float>(cap, err);
      scls = c.take<unsigned char>(cap);
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(sgt, gt, sizeof(float) * pix * nop * n, cudaMemcpyHostToDevice, ctx->stream));
    dgt = sgt;
    if (classes) {
      CK(cudaMemcpyAsync(scls, classes, pix * n, cudaMemcpyHostToDevice, ctx->stream));
      dcls = scls;
    }
  }
  const int D = ctx->dirs;
  if (launch_flow_error(stepped(ctx->lev[0], D), f0 * D, n, dgt, dcls, nclasses, derr, part, dstats, width_org,
                        height_org, cx, cy, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "flow_error_kernel launch", cudaGetLastError());
  ctx->launches += 2;
  if (memkind != OFDIS_MEM_DEVICE && err)
    CK(cudaMemcpyAsync(err, derr, sizeof(float) * pix * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(stats, dstats, sizeof(ofdis_error_stats) * n * nclasses, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

int ofdis_scene_flow_fullres(ofdis_ctx* ctx, int f0, int f1, const float* disp0, const float* disp1,
                             size_t disp_stride, float edge_diff, const ofdis_stereo_camera* cam,
                             float* disp1_warped, unsigned char* status, float* motion,
                             const ofdis_sf_gt* gt, const unsigned char* classes, int nclasses,
                             ofdis_sf_stats* stats, int width_org, int height_org, int memkind) {
  static_assert(sizeof(ofdis_sf_stats) == 64, "ofdis_sf_stats: 64 bytes, as api.SF_STATS_DTYPE");
  if (!ctx) return OFDIS_ERR_ARG;
  const bool dev = memkind == OFDIS_MEM_DEVICE;
  auto misaligned = [dev](const float* p) { return dev && reinterpret_cast<uintptr_t>(p) % sizeof(float); };
  const size_t pix = (size_t)std::max(width_org, 0) * std::max(height_org, 0);
  if (ctx->nop != 2 || f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !disp0 || !disp1 || disp_stride < pix ||
      !(edge_diff >= 0.f) || (!disp1_warped && !status && !motion && !stats) || (!gt != !stats) ||
      (gt && (!gt->disp0 || !gt->disp1 || !gt->flow)) || nclasses < 1 || nclasses > kEvalMaxClasses ||
      (!classes && nclasses > 1) ||
      (motion && (!cam || !finite_gt0(cam->fx) || !finite_gt0(cam->fy) || !finite_gt0(cam->baseline) ||
                  !finite_f32(cam->cx) || !finite_f32(cam->cy) || !finite_f32(cam->doffs))) ||
      misaligned(disp0) || misaligned(disp1) || misaligned(disp1_warped) || misaligned(motion) ||
      (gt && (misaligned(gt->disp0) || misaligned(gt->disp1) || misaligned(gt->flow))))
    return fail(ctx, OFDIS_ERR_ARG, "scene_flow_fullres: bad argument");
  int cx, cy;
  int rc = org_padding(ctx, width_org, height_org, &cx, &cy);
  if (rc) return rc;
  NvtxRange nvtx("sceneflow", -1);
  CK(cudaSetDevice(ctx->device));
  const int n = f1 - f0, D = ctx->dirs;
  const size_t np = pix * n;
  ofdis_sf_stats* dstats = nullptr;
  if (stats) {
    rc = carve(ctx, ctx->d_sf, "scene_flow_fullres counters",
               [&](Carve& c) { dstats = c.take<ofdis_sf_stats>((size_t)ctx->max_frames * kEvalMaxClasses); });
    if (rc) return rc;
  }
  SfArgs a{};
  a.disp0 = disp0;
  a.disp1 = disp1;
  a.stride = disp_stride;
  a.edge_diff = edge_diff;
  if (motion) a.cam = DispCamera{cam->fx * cam->baseline, cam->fx, cam->fy, cam->cx, cam->cy, cam->doffs};
  a.disp1w = disp1_warped;
  a.status = status;
  a.motion = motion;
  if (gt) {
    a.gt_d0 = gt->disp0;
    a.gt_d1 = gt->disp1;
    a.gt_flow = gt->flow;
    a.classes = classes;
    a.stats = dstats;
  }
  a.nclasses = nclasses;
  if (!dev) {
    // disp0 and disp1 packed to one map per pair, then gt's disp0, disp1 and flow and the classes (those given)
    const size_t cap = pix * ctx->max_frames;
    float *d0 = nullptr, *d1 = nullptr, *g0 = nullptr, *g1 = nullptr, *gf = nullptr;
    unsigned char* cls = nullptr;
    rc = carve_stage(ctx, [&](Carve& c) {
      d0 = c.take<float>(cap);
      d1 = c.take<float>(cap);
      g0 = c.take<float>(cap);
      g1 = c.take<float>(cap);
      gf = c.take<float>(2 * cap);
      cls = c.take<unsigned char>(cap);
    });
    if (rc) return rc;
    const size_t row = sizeof(float) * pix, pitch = sizeof(float) * disp_stride;
    CK(cudaMemcpy2DAsync(d0, row, disp0, pitch, row, n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpy2DAsync(d1, row, disp1, pitch, row, n, cudaMemcpyHostToDevice, ctx->stream));
    a.disp0 = d0;
    a.disp1 = d1;
    a.stride = pix;
    if (gt) {
      CK(cudaMemcpyAsync(g0, gt->disp0, sizeof(float) * np, cudaMemcpyHostToDevice, ctx->stream));
      CK(cudaMemcpyAsync(g1, gt->disp1, sizeof(float) * np, cudaMemcpyHostToDevice, ctx->stream));
      CK(cudaMemcpyAsync(gf, gt->flow, sizeof(float) * 2 * np, cudaMemcpyHostToDevice, ctx->stream));
      a.gt_d0 = g0;
      a.gt_d1 = g1;
      a.gt_flow = gf;
      if (classes) {
        CK(cudaMemcpyAsync(cls, classes, np, cudaMemcpyHostToDevice, ctx->stream));
        a.classes = cls;
      }
    }
    rc = carve_full(ctx, pix, [&](Carve& c) {
      a.disp1w = c.take<float>(cap, disp1_warped);
      a.motion = c.take<float>(3 * cap, motion);
      a.status = c.take<unsigned char>(cap, status);
    });
    if (rc) return rc;
  }
  if (stats) CK(cudaMemsetAsync(dstats, 0, sizeof(ofdis_sf_stats) * n * nclasses, ctx->stream));
  if (launch_scene_flow(stepped(ctx->lev[0], D), f0 * D, n, a, width_org, height_org, cx, cy, ctx->stream) < 0)
    return fail(ctx, OFDIS_ERR_CUDA, "sceneflow_kernel launch", cudaGetLastError());
  ctx->launches += 1;
  if (!dev) {
    if (disp1_warped) CK(cudaMemcpyAsync(disp1_warped, a.disp1w, sizeof(float) * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (motion) CK(cudaMemcpyAsync(motion, a.motion, sizeof(float) * 3 * np, cudaMemcpyDeviceToHost, ctx->stream));
    if (status) CK(cudaMemcpyAsync(status, a.status, np, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (stats)
    CK(cudaMemcpyAsync(stats, dstats, sizeof(ofdis_sf_stats) * n * nclasses, cudaMemcpyDeviceToHost, ctx->stream));
  if (!dev || stats) CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

int ofdis_patgrid_optimize(ofdis_ctx* ctx, int level, int f0, int f1, int init_from_coarser) {
  if (!ctx) return OFDIS_ERR_ARG;
  LevelGeom* L = level_of(ctx, level);
  if (!L || f0 < 0 || f1 > ctx->max_frames || f0 >= f1) return fail(ctx, OFDIS_ERR_ARG, "patgrid_optimize: bad argument");
  CK(cudaSetDevice(ctx->device));
  if (ctx->sel_dir >= 0 && f1 != f0 + 1) return fail(ctx, OFDIS_ERR_ARG, "patgrid_optimize: one frame at a time while a direction is selected");
  NvtxRange nvtx("patch", level);
  const int q0 = ctx->sel_dir >= 0 ? f0 * ctx->dirs + ctx->sel_dir : f0 * ctx->dirs;
  const int q1 = ctx->sel_dir >= 0 ? q0 + 1 : f1 * ctx->dirs;
  L->pdl = pdl_for(ctx, q1 - q0);
  cudaError_t optin = cudaSuccess;
  const int n = launch_patch_optimize(*L, ctx->pp, q0, q1, init_from_coarser != 0, patch_lanes_for(ctx, q1 - q0),
                                      ctx->stream, ctx->prof, &optin);
  if (optin != cudaSuccess) return fail(ctx, OFDIS_ERR_CUDA, "patch kernel launch: shared-memory opt-in (smem_optin)", optin);
  if (n < 0) return fail(ctx, OFDIS_ERR_CUDA, "patch_optimize_kernel launch", cudaGetLastError());
  ctx->launches += n;
  return OFDIS_OK;
}

int ofdis_patgrid_aggregate(ofdis_ctx* ctx, int level, int f0, int f1) {
  if (!ctx) return OFDIS_ERR_ARG;
  LevelGeom* L = level_of(ctx, level);
  if (!L || f0 < 0 || f1 > ctx->max_frames || f0 >= f1) return fail(ctx, OFDIS_ERR_ARG, "patgrid_aggregate: bad argument");
  CK(cudaSetDevice(ctx->device));
  NvtxRange nvtx("densify", level);
  L->pdl = pdl_for(ctx, (f1 - f0) * ctx->dirs);
  int n;
  if (ctx->dirs == 2) {
    // both grids' patch positions first; the backward flow is not densified on the last level (oflow.cpp:269-270)
    if (launch_fb_prepare(*L, f0 * 2, f1 * 2, ctx->stream) < 0) return fail(ctx, OFDIS_ERR_CUDA, "fb_prepare_kernel launch", cudaGetLastError());
    ctx->launches += 1;
    if (ctx->sel_dir >= 0)  // one grid of the couple (PatGridClass::AggregateFlowDense of either stand-alone grid)
      n = launch_densify(stepped(*L, 2), f0 * 2 + ctx->sel_dir, f0 * 2 + ctx->sel_dir + (f1 - f0), ctx->stream, ctx->prof);
    else
      n = (level == ctx->prm.sc_l) ? launch_densify(stepped(*L, 2), f0 * 2, f0 * 2 + (f1 - f0), ctx->stream, ctx->prof)
                                   : launch_densify(*L, f0 * 2, f1 * 2, ctx->stream, ctx->prof);
  } else {
    n = launch_densify(*L, f0, f1, ctx->stream, ctx->prof);
  }
  if (n < 0) return fail(ctx, OFDIS_ERR_CUDA, "densify_kernel launch", cudaGetLastError());
  ctx->launches += n;
  return OFDIS_OK;
}

static int varref_impl(ofdis_ctx* ctx, int level, int f0, int f1, int n_inner_override) {
  if (!ctx) return OFDIS_ERR_ARG;
  LevelGeom* L = level_of(ctx, level);
  if (!L || f0 < 0 || f1 > ctx->max_frames || f0 >= f1) return fail(ctx, OFDIS_ERR_ARG, "varref_refine: bad argument");
  if (!ctx->d_planes) return fail(ctx, OFDIS_ERR_ARG, "varref_refine: context created with usetvref=0");
  CK(cudaSetDevice(ctx->device));
  NvtxRange nvtx("varref", level);
  VarRefParams vp;
  // refine_variational.cpp:36-43
  vp.n_inner = n_inner_override >= 0 ? n_inner_override : ctx->prm.tv_innerit * (level + 1);
  vp.n_solver = ctx->prm.tv_solverit;
  vp.omega = ctx->prm.tv_sor;
  vp.quarter_alpha = 0.25f * ctx->prm.tv_alpha;
  vp.half_gamma_over3 = ctx->prm.tv_gamma * 0.5f / 3.0f;
  vp.half_delta_over3 = ctx->prm.tv_delta * 0.5f / 3.0f;
  const int nlaunch = (f1 - f0) * ctx->dirs;  // frames per launch
  SorPlan plan;
  if (!sor_plan(*L, ctx->prm.tv_solverit, ctx->sor, nlaunch, ctx->planes, &plan))
    return fail(ctx, OFDIS_ERR_UNSUPPORTED, "varref_refine: no SOR band fits one CTA");
  if (plan.pl.rec_stride > ctx->rec_f4 || plan.chain_nb > ctx->chain_nb)
    return fail(ctx, OFDIS_ERR_UNSUPPORTED, "varref_refine: the SOR plan exceeds the refinement workspace");
  L->pdl = pdl_for(ctx, nlaunch);
  // usefbcon: both directions are refined except on the last level (oflow.cpp:285-294)
  const int D = ctx->dirs;
  const bool fwd_only = (D == 2 && level == ctx->prm.sc_l);
  const int n = fwd_only ? launch_varref(stepped(*L, 2), plan, vp, f0 * 2, f0 * 2 + (f1 - f0), ctx->stream, ctx->prof, ctx->d_chain, ctx->d_div_fb)
                         : launch_varref(*L, plan, vp, f0 * D, f1 * D, ctx->stream, ctx->prof, ctx->d_chain, ctx->d_div_fb);
  if (n < 0) return fail(ctx, OFDIS_ERR_CUDA, "varref kernels launch", cudaGetLastError());
  ctx->launches += n;
  ctx->last_vr_level = level;
  ctx->last_sor = plan;
  ctx->last_vr_fcur = vp.n_inner & 1;
  ctx->last_vr_f0 = f0;
  ctx->last_vr_fstep = fwd_only ? 1 : D;  // workspace slots per user frame
  return OFDIS_OK;
}

int ofdis_varref_refine(ofdis_ctx* ctx, int level, int f0, int f1) { return varref_impl(ctx, level, f0, f1, -1); }

int ofdis_debug_varref_iters(ofdis_ctx* ctx, int level, int f0, int f1, int n_inner) {
  return varref_impl(ctx, level, f0, f1, n_inner);
}

int ofdis_set_direction(ofdis_ctx* ctx, int dir) {
  if (!ctx || dir < -1 || dir > 1 || (dir >= 0 && ctx->dirs != 2)) return OFDIS_ERR_ARG;
  ctx->sel_dir = dir;
  return OFDIS_OK;
}

int ofdis_set_option(ofdis_ctx* ctx, const char* name, int value) {
  if (!ctx || !name) return OFDIS_ERR_ARG;
  if (!strcmp(name, "sor_single_max")) {
    if (value != 32 && value != 64 && value != 128) return fail(ctx, OFDIS_ERR_ARG, "sor_single_max: 32, 64 or 128");
    ctx->sor.single_max = value;
  } else if (!strcmp(name, "sor_max_cluster")) {  // at most this many bands per cluster; levels with more are chained
    if (value != 1 && value != 2 && value != 4 && value != 8 && value != 16) return fail(ctx, OFDIS_ERR_ARG, "sor_max_cluster: 1, 2, 4, 8 or 16");
    if (value > ctx->sor_dev_cluster) return fail(ctx, OFDIS_ERR_UNSUPPORTED, "sor_max_cluster: the device does not grant clusters of 16 CTAs");
    if (ctx->d_planes) {  // the plans of a smaller cluster may need a larger workspace (chains of larger bands)
      size_t recf4 = 0;
      int chain_nb = 0;
      sor_workspace_need(ctx, value, value, &recf4, &chain_nb);
      if (recf4 > ctx->rec_f4 || chain_nb > ctx->chain_nb) {
        CK(cudaSetDevice(ctx->device));
        if (!alloc_refinement(ctx, std::max(recf4, ctx->rec_f4), std::max(chain_nb, ctx->chain_nb)))
          return fail(ctx, OFDIS_ERR_NOMEM, "sor_max_cluster: refinement workspace");
      }
    }
    ctx->sor.max_cluster = value;
  } else if (!strcmp(name, "sor_lane")) {
    if (value < 0 || value > 2) return fail(ctx, OFDIS_ERR_ARG, "sor_lane: 0, 1 or 2");
    ctx->sor.lane = value;
  } else if (!strcmp(name, "pdl")) {
    if (value < 0 || value > 2) return fail(ctx, OFDIS_ERR_ARG, "pdl: 0, 1 or 2");
    ctx->pdl = value;
  } else if (!strcmp(name, "patch_lanes")) {
    if (value != 0 && value != 4 && value != 8) return fail(ctx, OFDIS_ERR_ARG, "patch_lanes: 0, 4 or 8");
    ctx->patch_lanes = value;
  } else if (!strcmp(name, "sor_fast")) {
    if (value != 0 && value != 1) return fail(ctx, OFDIS_ERR_ARG, "sor_fast: 0 or 1");
    if (!ctx->d_planes) return fail(ctx, OFDIS_ERR_ARG, "sor_fast: context created with usetvref=0");
    SorOptions o = ctx->sor;
    o.fast = 1;
    SorPlan p;
    if (value && !sor_plan(ctx->lev[0], ctx->prm.tv_solverit, o, 1, ctx->planes, &p))
      return fail(ctx, OFDIS_ERR_UNSUPPORTED, "sor_fast: too many sweeps for the tile's halo");
    if (value && !ctx->d_fast) {  // records 8 floats per pixel + 2 x 2 planes of (du,dv), finest level x frames
      const size_t plane = ctx->planes.plane;
      CK(cudaSetDevice(ctx->device));
      if (cudaMalloc((void**)&ctx->d_fast, sizeof(float) * plane * 12 * ctx->cap) != cudaSuccess)
        return fail(ctx, OFDIS_ERR_NOMEM, "sor_fast workspace");
      cudaMemsetAsync(ctx->d_fast, 0, sizeof(float) * plane * 12 * ctx->cap, ctx->stream);
      ctx->planes.frec = ctx->d_fast;
      ctx->planes.fdu = ctx->d_fast + plane * 8 * ctx->cap;
    }
    ctx->sor.fast = value;
  } else if (!strcmp(name, "sor_rows_per_thread")) {
    if (value != 1 && value != 2 && value != 4) return fail(ctx, OFDIS_ERR_ARG, "sor_rows_per_thread: 1, 2 or 4");
    ctx->sor.rt = value;
  } else {
    return fail(ctx, OFDIS_ERR_ARG, "set_option: unknown option");
  }
  for (auto& kv : ctx->graphs) cudaGraphExecDestroy(kv.second);  // launch geometry changed
  ctx->graphs.clear();
  return OFDIS_OK;
}

int ofdis_set_graph_mode(ofdis_ctx* ctx, int enabled) {
  if (!ctx) return OFDIS_ERR_ARG;
  ctx->graph_mode = enabled != 0;
  return OFDIS_OK;
}

int ofdis_run(ofdis_ctx* ctx, int nframes, int use_initflow) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (nframes < 1 || nframes > ctx->max_frames) return fail(ctx, OFDIS_ERR_ARG, "run: bad frame count");
  CK(cudaSetDevice(ctx->device));
  NvtxRange nvtx(ctx->graph_mode ? "run (graph)" : "run", -1);
  if (!ctx->graph_mode) return run_levels(ctx, nframes, use_initflow);
  const long key = (long)nframes * 2 + (use_initflow ? 1 : 0);
  auto it = ctx->graphs.find(key);
  if (it == ctx->graphs.end()) {
    const long before = ctx->launches;
    cudaGraph_t graph = nullptr;
    CK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    const int rc = run_levels(ctx, nframes, use_initflow);
    cudaError_t e = cudaStreamEndCapture(ctx->stream, &graph);
    if (rc || e != cudaSuccess) {
      if (graph) cudaGraphDestroy(graph);
      return rc ? rc : fail(ctx, OFDIS_ERR_CUDA, "cudaStreamEndCapture", e);
    }
    cudaGraphExec_t exec = nullptr;
    e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) return fail(ctx, OFDIS_ERR_CUDA, "cudaGraphInstantiate", e);
    ctx->graph_launches[key] = ctx->launches - before;
    ctx->launches = before;  // capture does not execute
    it = ctx->graphs.emplace(key, exec).first;
  }
  CK(cudaGraphLaunch(it->second, ctx->stream));
  ctx->launches += ctx->graph_launches[key];
  return OFDIS_OK;
}

int ofdis_sync(ofdis_ctx* ctx) {
  if (!ctx) return OFDIS_ERR_ARG;
  CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

static int flow_index(const ofdis_ctx* ctx, int level) {
  if (level < ctx->prm.sc_l || level > ctx->prm.sc_f + 1) return -1;
  return level - ctx->prm.sc_l;
}

int ofdis_get_flow(ofdis_ctx* ctx, int frame, int level, float* dst, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  const int li = flow_index(ctx, level);
  if (li < 0 || frame < 0 || frame >= ctx->max_frames || !dst) return fail(ctx, OFDIS_ERR_ARG, "get_flow: bad argument");
  CK(cudaMemcpyAsync(dst, ctx->d_flow[li] + (size_t)(frame * ctx->dirs + std::max(ctx->sel_dir, 0)) * ctx->flow_floats[li],
                     sizeof(float) * ctx->flow_floats[li], kind_out(memkind), ctx->stream));
  if (memkind == OFDIS_MEM_HOST) CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

int ofdis_set_flow(ofdis_ctx* ctx, int frame, int level, const float* src, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  const int li = flow_index(ctx, level);
  if (li < 0 || frame < 0 || frame >= ctx->max_frames || !src) return fail(ctx, OFDIS_ERR_ARG, "set_flow: bad argument");
  CK(cudaMemcpyAsync(ctx->d_flow[li] + (size_t)(frame * ctx->dirs + std::max(ctx->sel_dir, 0)) * ctx->flow_floats[li], src,
                     sizeof(float) * ctx->flow_floats[li], kind_in(memkind), ctx->stream));
  return OFDIS_OK;
}

int ofdis_get_flow_batch(ofdis_ctx* ctx, int f0, int f1, float* dst, int memkind) {
  if (!ctx) return OFDIS_ERR_ARG;
  if (f0 < 0 || f1 > ctx->max_frames || f0 >= f1 || !dst) return fail(ctx, OFDIS_ERR_ARG, "get_flow_batch: bad argument");
  const size_t nfl = ctx->flow_floats[0];
  if (ctx->dirs == 1)
    CK(cudaMemcpyAsync(dst, ctx->d_flow[0] + (size_t)f0 * nfl, sizeof(float) * nfl * (f1 - f0), kind_out(memkind), ctx->stream));
  else  // forward frames only
    CK(cudaMemcpy2DAsync(dst, sizeof(float) * nfl, ctx->d_flow[0] + (size_t)f0 * 2 * nfl, sizeof(float) * nfl * 2,
                         sizeof(float) * nfl, (size_t)(f1 - f0), kind_out(memkind), ctx->stream));
  return OFDIS_OK;
}

int ofdis_get_patches(ofdis_ctx* ctx, int frame, int level, float* p, float* pweight, int* conv, int* cnt) {
  if (!ctx) return OFDIS_ERR_ARG;
  LevelGeom* L = level_of(ctx, level);
  if (!L || frame < 0 || frame >= ctx->max_frames) return fail(ctx, OFDIS_ERR_ARG, "get_patches: bad argument");
  const size_t np = L->np;
  frame = frame * ctx->dirs + std::max(ctx->sel_dir, 0);  // the forward grid unless a direction is selected
  if (p) CK(cudaMemcpyAsync(p, L->pat_p + frame * np * L->nop, sizeof(float) * np * L->nop, cudaMemcpyDeviceToHost, ctx->stream));
  if (pweight) CK(cudaMemcpyAsync(pweight, L->pat_w + frame * np * L->novals, sizeof(float) * np * L->novals, cudaMemcpyDeviceToHost, ctx->stream));
  if (conv) CK(cudaMemcpyAsync(conv, L->pat_conv + frame * np, sizeof(int) * np, cudaMemcpyDeviceToHost, ctx->stream));
  if (cnt) CK(cudaMemcpyAsync(cnt, L->pat_cnt + frame * np, sizeof(int) * np, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

long ofdis_debug_get(ofdis_ctx* ctx, const char* name, int frame, float* dst, size_t max_floats) {
  if (!ctx || !name || !dst || ctx->last_vr_level < 0) return OFDIS_ERR_ARG;
  LevelGeom* L = level_of(ctx, ctx->last_vr_level);
  const int fr = (frame - ctx->last_vr_f0) * ctx->last_vr_fstep;
  if (!L || fr < 0) return OFDIS_ERR_ARG;
  const size_t plane = (size_t)L->pitch * L->h;
  const int C = L->noc;
  static const char* dn[8] = {"Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz"};
  const float* src = nullptr;
  size_t n = 0;
  for (int k = 0; k < 8; ++k)
    if (!strcmp(name, dn[k])) {
      src = ctx->planes.deriv[k] + (size_t)fr * C * plane;
      n = plane * C;
    }
  if (!strcmp(name, "mask")) { src = ctx->planes.mask + (size_t)fr * plane; n = plane; }
  if (!strcmp(name, "dudv") || !strcmp(name, "rec")) {
    // stored in the layout of the last refinement's plan (see VarRefPlanes); returned in natural (h, pitch,
    // per-pixel) order
    const bool is_rec = name[0] == 'r';
    const VarRefPlanes& sp = ctx->last_sor.pl;  // its layout; the buffers are the context's current ones
    const int per = is_rec ? sp.nq : 2;  // floats per pixel
    if (plane * per > max_floats) return OFDIS_ERR_ARG;
    if (sp.fast) {  // natural layout: records 8 floats per pixel, (du,dv) two planes of the current buffer
      std::vector<float> raw(is_rec ? plane * 8 : plane * 2);
      const float* src_f = is_rec ? ctx->planes.frec + (size_t)fr * sp.frec_stride
                                  : ctx->planes.fdu + (size_t)fr * sp.fdu_stride + (size_t)ctx->last_vr_fcur * 2 * plane;
      if (cudaMemcpyAsync(raw.data(), src_f, sizeof(float) * raw.size(), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return OFDIS_ERR_CUDA;
      if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return OFDIS_ERR_CUDA;
      for (size_t o = 0; o < plane; ++o)
        for (int e = 0; e < per; ++e) dst[o * per + e] = is_rec ? raw[o * 8 + e] : raw[(size_t)e * plane + o];
      return (long)(plane * per);
    }
    std::vector<float> raw(sp.rec_stride * 4);
    if (cudaMemcpyAsync(raw.data(), ctx->planes.rec + (size_t)fr * sp.rec_stride, sizeof(float) * raw.size(), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return OFDIS_ERR_CUDA;
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return OFDIS_ERR_CUDA;
    for (int j = 0; j < L->h; ++j)
      for (int i = 0; i < L->w; ++i)
        for (int e = 0; e < per; ++e) {
          // lane layout: a record is two float4 (lane_rec_f4), (du,dv) consecutive floats (lane_dudv_f); band lane
          // rows: records as band_rec_f places them, (du,dv) are chunks nq, nq+1
          const size_t k = sp.lane ? (is_rec ? lane_rec_f4(sp, i, j, e >> 2) * 4 + (e & 3) : lane_dudv_f(sp, i, j) + e)
                                   : (is_rec ? band_rec_f(sp, i, j, e) : band_f4(sp, i >> 2, j, sp.nq + e) * 4 + (i & 3));
          dst[((size_t)j * L->pitch + i) * per + e] = raw[k];
        }
    return (long)(plane * per);
  }
  if (!src || n > max_floats) return OFDIS_ERR_ARG;
  if (cudaMemcpyAsync(dst, src, sizeof(float) * n, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return OFDIS_ERR_CUDA;
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return OFDIS_ERR_CUDA;
  return (long)n;
}

int ofdis_debug_div(ofdis_ctx* ctx, const float* a, const float* b, long n, float* q_fast, float* q_plain,
                    unsigned char* unsafe) {
  if (!ctx || n < 0 || (n && (!a || !b || !q_fast || !q_plain || !unsafe))) return OFDIS_ERR_ARG;
  if (!n) return OFDIS_OK;
  CK(cudaSetDevice(ctx->device));
  float* d = nullptr;  // a, b, q_fast, q_plain, then the flags
  CK(cudaMalloc((void**)&d, (size_t)n * (4 * sizeof(float) + 1)));
  cudaError_t e = cudaMemcpyAsync(d, a, sizeof(float) * n, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + n, b, sizeof(float) * n, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) {
    debug_div_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d, d + n, n, d + 2 * n, d + 3 * n,
                                                                           reinterpret_cast<unsigned char*>(d + 4 * n));
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(q_fast, d + 2 * n, sizeof(float) * n, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(q_plain, d + 3 * n, sizeof(float) * n, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(unsafe, d + 4 * n, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  cudaFree(d);
  if (e != cudaSuccess) return fail(ctx, OFDIS_ERR_CUDA, "debug_div", e);
  return OFDIS_OK;
}

int ofdis_debug_sor_div_fallbacks(ofdis_ctx* ctx, unsigned long long* count, int reset) {
  if (!ctx || !count) return OFDIS_ERR_ARG;
  if (!ctx->d_div_fb) return fail(ctx, OFDIS_ERR_ARG, "debug_sor_div_fallbacks: context created with usetvref=0");
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemcpyAsync(count, ctx->d_div_fb, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  if (reset) CK(cudaMemsetAsync(ctx->d_div_fb, 0, sizeof(unsigned long long), ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return OFDIS_OK;
}

int ofdis_debug_sor_plan(int w, int h, int nop, int noc, int solverit, int frames, int lane, int fast, int rt,
                         int single_max, int max_cluster, int* out) {
  if (w < 2 || h < 4 || h > SOR_MAX_ROWS || (nop != 1 && nop != 2) || (noc != 1 && noc != 3) || solverit < 1 ||
      frames < 1 || lane < 0 || lane > 2 || (fast != 0 && fast != 1) || (rt != 1 && rt != 2 && rt != 4) ||
      (single_max != 32 && single_max != 64 && single_max != 128) ||
      (max_cluster != 1 && max_cluster != 2 && max_cluster != 4 && max_cluster != 8 && max_cluster != 16) || !out)
    return OFDIS_ERR_ARG;
  LevelGeom L{};
  L.w = w;
  L.h = h;
  L.nop = nop;
  L.noc = noc;
  L.pitch = ((w + 3) / 4) * 4;
  SorPlan p;
  if (!sor_plan(L, solverit, SorOptions{lane, fast, rt, single_max, max_cluster}, frames, VarRefPlanes{}, &p))
    return OFDIS_ERR_UNSUPPORTED;
  out[0] = p.kind;
  out[1] = p.pl.hpad;
  out[2] = p.pl.rt;
  out[3] = p.ml;
  out[4] = p.pl.nb;
  out[5] = p.sweeps;
  out[6] = solverit % p.sweeps;
  out[7] = assemble_rows_per_thread(w, h, frames);
  out[8] = p.kind == SOR_REDBLACK ? 1 : (p.kind == SOR_LANE ? 2 : 0);  // launch_varref_t's MODE
  return OFDIS_OK;
}

long ofdis_launch_count(const ofdis_ctx* ctx) { return ctx ? ctx->launches : 0; }

int ofdis_profile_run(ofdis_ctx* ctx, int nframes, int steps, double* ms_by_class, long* launches_by_class) {
  return ofdis_profile_levels(ctx, nframes, steps, ms_by_class, launches_by_class, nullptr);
}

int ofdis_profile_levels(ofdis_ctx* ctx, int nframes, int steps, double* ms_by_class, long* launches_by_class,
                         double* ms_by_level_class) {
  if (!ctx || steps < 1 || !ms_by_class || !launches_by_class) return OFDIS_ERR_ARG;
  if (nframes < 1 || nframes > ctx->max_frames) return fail(ctx, OFDIS_ERR_ARG, "profile_run: bad frame count");
  CK(cudaSetDevice(ctx->device));
  Profiler prof;
  prof.st = ctx->stream;
  ctx->prof = &prof;
  int rc = OFDIS_OK;
  for (int s = 0; s < steps && rc == OFDIS_OK; ++s) rc = run_levels(ctx, nframes, 0);
  ctx->prof = nullptr;
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  for (int k = 0; k < KC_COUNT; ++k) {
    ms_by_class[k] = 0.0;
    launches_by_class[k] = 0;
  }
  if (ms_by_level_class)
    for (int k = 0; k < ctx->nlev * KC_COUNT; ++k) ms_by_level_class[k] = 0.0;
  for (auto& r : prof.recs) {
    float ms = 0.f;
    if (e == cudaSuccess && cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
      ms_by_class[r.cls] += ms;
      launches_by_class[r.cls] += 1;
      if (ms_by_level_class && r.level >= ctx->prm.sc_l && r.level <= ctx->prm.sc_f)
        ms_by_level_class[(r.level - ctx->prm.sc_l) * KC_COUNT + r.cls] += ms;
    }
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  if (rc) return rc;
  if (e != cudaSuccess) return fail(ctx, OFDIS_ERR_CUDA, "profile_run sync", e);
  return OFDIS_OK;
}

}  // extern "C"

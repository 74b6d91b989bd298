/* ofdis_b200.h -- C-ABI of the CUDA (sm_90a, H100) DIS optical-flow hot path.
 *
 * This is the drop-in boundary (DESIGN.md section 1): plain C, plain pointers
 * and sizes, no C++/torch types.  Everything the reference's three classes do
 * on the hot path is reachable from here:
 *
 *   reference interface (file:line)                       -> entry point
 *   ------------------------------------------------------------------------
 *   OFC::OFClass::OFClass            oflow.h:84-111,        ofdis_create + ofdis_upload_* +
 *                                    oflow.cpp:32-363        ofdis_run + ofdis_get_flow
 *   PatGridClass::InitializeGrid /   patchgrid.h:25-26,     ofdis_upload_level (binds I0,dI0,I1 of a level)
 *     SetTargetImage                 patchgrid.cpp:98-132
 *   PatGridClass::InitializeFromCoarserOF  patchgrid.cpp:195-211   ofdis_set_flow(level+1) / implicit in ofdis_run
 *   PatGridClass::Optimize           patchgrid.cpp:134-141  ofdis_patgrid_optimize
 *     (PatClass::InitializePatch, OptimizeIter  patch.cpp:57-88,119-212 -- fused into the same kernel)
 *   PatGridClass::AggregateFlowDense patchgrid.cpp:213-397  ofdis_patgrid_aggregate
 *   PatGridClass::SetComplGrid       patchgrid.h:36 + oflow.cpp:162-170   ofdis_params.usefbcon = 1 (both grids of a pair
 *                                                            live in the context; ofdis_upload_level_fb,
 *                                                            ofdis_set_direction)
 *   PatGridClass::GetQuePatchDis &c  patchgrid.h:42-44      ofdis_get_patches
 *   VarRefClass::VarRefClass         refine_variational.h:37-39,    ofdis_varref_refine
 *                                    refine_variational.cpp:25-116
 *     (image_warp, get_derivatives, compute_smoothness, compute_data[_DE],
 *      sub_laplacian, sor_coupled / sor_coupled_slow_but_readable_DE;
 *      FDF1.0.1/opticalflow_aux.c:17-548, solver.c:77-466 -- device kernels)
 *
 * Unlike the reference (no status, exit(1) on OOM, image.c:17-28) every call
 * returns an int status and never exits.  A context is bound to one CUDA
 * device and one stream; all work is asynchronous on that stream unless the
 * call copies to pageable host memory.  `frames` is the batch dimension that
 * sits BELOW the reference API: one context processes frame pairs
 * [0, max_frames) per launch.
 *
 * Threads and shared devices: one context is used by one host thread at a
 * time (calls on the same context must not overlap; which thread makes them
 * may change).  Different contexts may share a device and a stream, and
 * each gives the same bits as it would alone.  Contexts on different streams
 * may be used from different threads at once, in graph mode or not.  A
 * context in graph mode captures its stream while ofdis_run records a graph
 * (the first run of a frame count after ofdis_set_graph_mode(1) or after a
 * call that discards its graphs, such as ofdis_set_option): whatever else is
 * enqueued on that stream meanwhile, from any thread, is recorded into the
 * graph or breaks the capture, and a synchronisation of the stream breaks
 * it.  So contexts that share a stream, and the caller's own work on it,
 * are used from one thread at a time once one of them is in graph mode.  A
 * context on a caller's stream only enqueues its own work there, in call
 * order, and leaves the stream's other work alone; ofdis_destroy waits for
 * that stream.  Process-wide state is guarded inside the library (DESIGN.md
 * section 5.13).
 *
 * Arithmetic contract: IEEE binary32, no FMA contraction, expression order of
 * the reference, so results are bitwise equal to the reference CPU build on
 * the same inputs (tests/test_gpu_parity.py).
 */
#ifndef OFDIS_B200_H
#define OFDIS_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ofdis_ctx ofdis_ctx;

/* The 21 run-time scalars of OFClass's constructor (oflow.h:93-111), CLI
 * semantics of run_dense.cpp:225-294.  dp_thresh is the un-squared CLI value. */
typedef struct ofdis_params {
  int sc_f, sc_l;          /* first (coarsest) / last (finest) pyramid level */
  int max_iter, min_iter;  /* Gauss-Newton iterations per patch */
  float dp_thresh, dr_thresh, res_thresh;
  int p_samp_s;            /* patch edge length P (even, P*P*noc % 4 == 0) */
  float patove;            /* patch overlap in [0,1) */
  int usefbcon;            /* forward-backward merge (oflow.cpp:162-170, patchgrid.cpp:278-375): doubles the patch work */
  int costfct;             /* 0 L2, 1 L1, 2 pseudo-Huber */
  int noc;                 /* image channels: 1 or 3 */
  int patnorm;             /* mean-normalise patches */
  int usetvref;            /* run the variational refinement */
  float tv_alpha, tv_gamma, tv_delta;
  int tv_innerit, tv_solverit;
  float tv_sor;
  int verbosity;
} ofdis_params;

enum {
  OFDIS_OK = 0,
  OFDIS_ERR_ARG = -1,         /* bad argument / unsupported geometry */
  OFDIS_ERR_CUDA = -2,        /* a CUDA call failed; see ofdis_last_error */
  OFDIS_ERR_UNSUPPORTED = -3, /* valid in the reference but not built here (a finest refinement level of more than 16384 rows, more frames than OFDIS_MAX_GRID_FRAMES allows, or a patch too large for the generic patch kernel's shared memory -- RGB p_samp_s >= 32, gray p_samp_s >= 54; the largest accepted are RGB 30 and gray 52 -- refused by ofdis_create before it touches a device; ofdis_upload_packed with usefbcon).  The reference has none of these limits. */
  OFDIS_ERR_NOMEM = -4
};
/* Kernels put the frames of a launch in a grid dimension of at most 65535 blocks: ofdis_create refuses
 * max_frames * max(2, dirs * noc) > OFDIS_MAX_GRID_FRAMES (dirs = 2 with usefbcon, else 1) with
 * OFDIS_ERR_UNSUPPORTED.  The largest contexts are 32767 frames (gray, or usefbcon gray), 21845 (RGB) and
 * 10922 (usefbcon RGB). */
enum { OFDIS_MAX_GRID_FRAMES = 65535 };
enum { OFDIS_MEM_HOST = 0, OFDIS_MEM_DEVICE = 1 };

/* nop: 2 = optical flow (run_OF_*), 1 = stereo disparity (run_DE_*).
 * width/height: level-0 size, divisible by 2^sc_f (oflow.h:87).  imgpadding:
 * border of every level image, at least p_samp_s (OFDIS_ERR_ARG otherwise; run_dense.cpp:343 passes the
 * patch size).  A wider border gives the same flow: no read reaches beyond p_samp_s of the image.
 * stream: a cudaStream_t to enqueue on, or NULL for a private stream. */
int ofdis_create(ofdis_ctx** out, int device, void* stream, const ofdis_params* prm, int nop,
                 int width, int height, int imgpadding, int max_frames);
int ofdis_destroy(ofdis_ctx* ctx);
const char* ofdis_last_error(const ofdis_ctx* ctx);
const char* ofdis_version(void);

/* camparam::camlr (oflow.h:28; 0 = left/forward grid clamps disparity <= 0, 1 = right/backward
 * clamps >= 0, patch.cpp:188-193, refine_variational.cpp:299-314).  Default 0, as OFClass's
 * forward grid uses.  Only meaningful for nop == 1; with usefbcon the forward grid is 0 and the
 * backward grid 1 whatever is set here. */
int ofdis_set_camlr(ofdis_ctx* ctx, int camlr);
/* optparam::dp_thresh is stored SQUARED by OFClass (oflow.cpp:88); callers that already hold
 * the squared value (PatGridClass built from an optparam) set it here bit-exactly. */
int ofdis_set_dp_thresh_sq(ofdis_ctx* ctx, float dp_thresh_sq);

/* level geometry (oflow.cpp:142-151, patchgrid.cpp:42-48) */
int ofdis_level_info(const ofdis_ctx* ctx, int level, int* w, int* h, int* nopw, int* noph, int* steps);

/* Images of one level of one frame pair: padded, row-major, channel-interleaved
 * float32, (h+2*pad) x (w+2*pad) x noc, exactly what OFClass receives
 * (oflow.h:84-86).  The gradients of I1 are only read by the forward-backward grid
 * (oflow.cpp:193-197); without usefbcon they are not needed (ofdis_upload_level_fb otherwise). */
int ofdis_upload_level(ofdis_ctx* ctx, int frame, int level, const float* i0, const float* i0x,
                       const float* i0y, const float* i1, int memkind);

/* Like ofdis_upload_level plus the gradients of the second image (im_bo_dx, im_bo_dy of oflow.h:84-86),
 * which the forward-backward grid needs as its template gradients (oflow.cpp:193-197).  Required when the
 * context was created with usefbcon = 1; i1x, i1y may be NULL otherwise. */
int ofdis_upload_level_fb(ofdis_ctx* ctx, int frame, int level, const float* i0, const float* i0x,
                          const float* i0y, const float* i1, const float* i1x, const float* i1y, int memkind);

/* Packed transfer: all levels sc_f..sc_l of frames [f0,f1) in the context's own
 * layout (per frame: I0,I1 of levels sc_f..sc_l, then I0x,I0y of the same levels; use
 * ofdis_packed_offset), one copy.  Not available with usefbcon (a packed frame has no gradients of
 * the second image: OFDIS_ERR_UNSUPPORTED); the image-only transfers below are. */
size_t ofdis_packed_frame_floats(const ofdis_ctx* ctx);
size_t ofdis_packed_offset(const ofdis_ctx* ctx, int level, int which /*0 I0,1 I0x,2 I0y,3 I1*/);
int ofdis_upload_packed(ofdis_ctx* ctx, int f0, int f1, const float* packed, int memkind);

/* Images-only transfer (extension, SURVEY 8f rank 1): the leading ofdis_packed_images_frame_floats()
 * floats of a packed frame are I0,I1 of all levels (offsets as ofdis_packed_offset reports them);
 * `packed` holds only those, frame after frame.  One 2-D copy, then the gradients of I0 are derived
 * on the device (Sobel 3x3 / 8, reflect101, zero border: run_dense.cpp:156-157,171-172). */
size_t ofdis_packed_images_frame_floats(const ofdis_ctx* ctx);
int ofdis_upload_packed_images(ofdis_ctx* ctx, int f0, int f1, const float* packed, int memkind);

/* Read-back of one padded array of the device pyramid (which: 0 I0, 1 I0x, 2 I0y, 3 I1); the
 * inverse of ofdis_upload_level, used to check the device-built pyramids.  With usefbcon, after
 * ofdis_set_direction(ctx, 1), the arrays of the pair's backward frame: I1, its gradients, I0. */
int ofdis_get_level(ofdis_ctx* ctx, int frame, int level, int which, float* dst, int memkind);

/* Pyramid on the device (extension, SURVEY 8f rank 1 == ConstructImgPyramide, run_dense.cpp:130-178
 * plus the divisibility padding of run_dense.cpp:298-311).
 * ofdis_upload_frames_u8: `frames` = [frame][2][height_org][width_org][noc] 8-bit pixels (I0 then I1
 *   of each pair); width_org/height_org must pad up to the context's width/height.  Builds levels
 *   sc_l..sc_f of I0, I1 (box means), I0x, I0y (Sobel/8) and both paddings on the device.
 * ofdis_upload_finest_level: `packed` = [frame][2][h][w][noc] float images of level sc_l WITHOUT
 *   the border padding (h = height >> sc_l, ...; ofdis_finest_level_frame_floats() per frame);
 *   coarser levels, gradients and paddings are derived on the device.  Smallest transfer that still
 *   defines the run's input exactly. */
int ofdis_upload_frames_u8(ofdis_ctx* ctx, int f0, int f1, const unsigned char* frames, int width_org, int height_org,
                           int memkind);
/* Consecutive frames (extension): `frames` = [f1-f0+1][height_org][width_org][noc] 8-bit frames; pair slot
 * f0+i gets (frames[i], frames[i+1]).  Same preprocessing as ofdis_upload_frames_u8 (divisibility padding,
 * box-mean levels, Sobel/8, border paddings; usefbcon's swapped frames), each frame uploaded and each of its
 * levels built once.  The following ofdis_run is bitwise what ofdis_upload_frames_u8 of the pairs gives.
 * Same arguments and status codes as ofdis_upload_frames_u8; slots outside [f0, f1) are not touched.  The
 * context keeps no frame between calls: to stream a clip in chunks, pass each chunk's last frame again as the
 * next chunk's first. */
int ofdis_upload_sequence_u8(ofdis_ctx* ctx, int f0, int f1, const unsigned char* frames, int width_org,
                             int height_org, int memkind);
/* Two-way sequence (extension): `frames` = [n+1][height_org][width_org][noc] 8-bit frames.  Slot f0+t gets
 * (frames[t], frames[t+1]), slot f0+n+t gets (frames[t+1], frames[t]); f0 + 2n <= max_frames.  Arguments, padding
 * rules, staging and status codes as ofdis_upload_sequence_u8 (n < 1: OFDIS_ERR_ARG); each frame is uploaded and each
 * of its levels built once.  Every slot's pyramid is bitwise what ofdis_upload_frames_u8 of the forward and the
 * swapped pairs gives.  Marks slots [f0, f0+n) not swapped and [f0+n, f0+2n) swapped (see ofdis_set_swapped_slots);
 * other uploads leave the marks alone. */
int ofdis_upload_sequence_bidir_u8(ofdis_ctx* ctx, int f0, int n, const unsigned char* frames, int width_org,
                                   int height_org, int memkind);
/* Stereo (nop == 1): slots [f0, f1) hold swapped pairs (right image first) and run as the right camera -- every grid
 * of such a slot has its camlr inverted (with usefbcon its forward grid clamps disparities to >= 0, its backward grid
 * to <= 0).  Flow ignores the mark.  Default 0 for every slot; swapped is 0 or 1.  The marks are read when a run
 * executes, so a captured graph follows later changes.  Enqueued on the context's stream. */
int ofdis_set_swapped_slots(ofdis_ctx* ctx, int f0, int f1, int swapped);
/* Forward-backward (flow) / left-right (stereo) consistency of the last run's slots [f0, f1) against partner slots
 * [b0, b0 + f1 - f0), at the original frame size: mask = [f1-f0][height_org][width_org] bytes (0 consistent,
 * 1 inconsistent, 2 leaves the frame), err = the same shape in float32 (may be NULL).  F is slot a's full-resolution
 * flow and B its partner's, both exactly what ofdis_get_flow_fullres returns; per pixel, in float32 without
 * contraction: (xs, ys) = (x, y) + F(x, y); outside [0, width_org-1] x [0, height_org-1] (or NaN): mask 2,
 * err +inf; else b = B sampled bilinearly at (xs, ys) (corners floor and floor + 1 clamped to the frame, horizontal
 * pass first), err = |F + b|^2 and mask = (err <= alpha (|F|^2 + |b|^2) + beta) ? 0 : 1.  Usual choices: flow
 * alpha 0.01, beta 0.5 (Sundaram et al., ECCV 2010); stereo alpha 0, beta 1 (|d_L + d_R(x + d_L)| <= 1 px).
 * alpha, beta finite and >= 0, a non-NULL mask and slots inside the context, else OFDIS_ERR_ARG; frame sizes as
 * ofdis_get_flow_fullres checks them.  Computed from the level flows without a full-resolution copy of either;
 * host output goes through the context's full-resolution scratch.  The flows are not changed. */
int ofdis_consistency_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, unsigned char* mask, float* err, float alpha,
                              float beta, int width_org, int height_org, int memkind);
/* Per-pixel confidence of the last run's slots [f0, f1) (extension): a number in [0, 1] per pixel that ranks how far
 * the flow or disparity there can be trusted, from three terms (the measures surveyed by Hu and Mordohai, PAMI 2012).
 * Flow (nop 2) and stereo (nop 1, v = 0) contexts.  For pair k, F is slot a = f0+k's full-resolution flow, exactly
 * what ofdis_get_flow_fullres returns (computed from the level flows, without a full-resolution copy).  I0 and I1 are
 * frames0 + k*frame_stride and frames1 + k*frame_stride, [H][W][noc] bytes in the context's channel count
 * (frame_stride >= H*W*noc; a clip passes frames1 = frames0 + frame_stride, as ofdis_interpolate_fullres).
 * W = width_org, H = height_org.  Everything is float32 with +, -, *, IEEE / and sqrtf only, without contraction; every
 * sum starts from +0.0f and runs dy = -r .. r outer, dx = -r .. r inner.
 *   Brightness g(I, x, y): the byte, or ((float)b0 + (float)b1 + (float)b2) / 3.0f in memory order (the tracker's).
 *   Window: r = p->radius; window pixel (dx, dy) of (X, Y) is q = (clamp(X + dx), clamp(Y + dy)), clamped to the frame
 *     as the tracker's seeding clamps (border pixels repeat).
 *   Warp: for a window pixel q with flow F(q) = (u, v): (xs, ys) = ((float)qx + u, (float)qy + v); when 0 <= xs <= W-1
 *     and 0 <= ys <= H-1 (NaN fails), Iw(q) = the bilinear rule of ofdis_consistency_fullres on the brightness of I1's
 *     four corners (x0 = floor(xs), x1 = min(x0 + 1, W - 1), fx = xs - x0, the same in y; r0 = g00*(1-fx) + g10*fx,
 *     r1 = g01*(1-fx) + g11*fx, Iw = r0*(1-fy) + r1*fy); else q is not a sample.
 *   z (photometric): over the samples of the window, n their count (int), s0 += g(I0, q), s1 += Iw(q); with
 *     n >= min_count, m0 = s0 / (float)n, m1 = s1 / (float)n, then over the samples again c00 += (g0 - m0)*(g0 - m0),
 *     c11 += (Iw - m1)*(Iw - m1), c01 += (g0 - m0)*(Iw - m1); den = c00 * c11; z = c01 / sqrtf(den) when den > 0.
 *     Otherwise (n < min_count, or zero variance) z = qNaN.
 *   e (forward-backward / left-right): with b0 >= 0, err of ofdis_consistency_fullres of slot a against slot b0+k at
 *     (X, Y), bit for bit (+inf where the target leaves the frame, a NaN of any payload where the partner's flow there is
 *     NaN); with b0 < 0, e = qNaN and it is not used.
 *   lambda (texture): over every window pixel, ix = (g(I0, min(qx+1, W-1), qy) - g(I0, max(qx-1, 0), qy)) * 0.5f,
 *     iy likewise in y, a += ix*ix, b += ix*iy, c += iy*iy; d = a - c; lambda = (a + c)*0.5f - sqrtf(d*d*0.25f + b*b):
 *     the smaller eigenvalue of the structure tensor, at r = 2 the tracker's seeding value bit for bit.
 *   conf = (cz * ce) * cl with cz = z > 0 ? z : 0 (NaN gives 0; rounding may leave z a few ulp above 1),
 *     ce = e >= 0 ? s_fb / (s_fb + e) : 0 (so +inf gives 0 and NaN gives 0), and ce = 1 with b0 < 0,
 *     cl = lambda > 0 ? lambda / (lambda + s_tex) : 0.
 * conf = [f1-f0][H][W] float32, terms = [f1-f0][H][W][3] float32 (z, e, lambda); either may be NULL, not both.
 * frames, conf and terms are in memkind: host frames go through the context's staging buffer (two 2-D copies), host
 * outputs through its full-resolution scratch, and the call then synchronises the stream once.  One kernel for all
 * pairs.  OFDIS_ERR_ARG, with the outputs untouched: slots outside the context, b0 >= 0 with [b0, b0 + f1 - f0)
 * outside it, a NULL p, radius outside 1 .. 7, s_fb or s_tex not finite and > 0, min_count outside 1 .. (2r+1)^2,
 * NULL frames0 or frames1, frame_stride below one frame, both outputs NULL, a device output not 4-byte aligned; frame
 * sizes as ofdis_get_flow_fullres checks them.  Not part of ofdis_run's graph; the flows are not changed. */
typedef struct ofdis_conf_params {
  int radius;           /* window (2r+1)^2, r in 1 .. 7 */
  float s_fb;           /* > 0, finite: scale of the forward-backward term (px^2) */
  float s_tex;          /* > 0, finite: scale of the texture term */
  int min_count;        /* 1 .. (2r+1)^2: in-frame warped samples a window needs */
} ofdis_conf_params;
int ofdis_confidence_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_conf_params* p,
                             const unsigned char* frames0, const unsigned char* frames1, size_t frame_stride,
                             float* conf, float* terms, int width_org, int height_org, int memkind);
/* Error statistics of one (pair, class) of ofdis_flow_error_fullres (48 bytes). */
typedef struct ofdis_error_stats {
  long long n;          /* pixels counted */
  long long n_over[3];  /* e > 1, e > 3, e > 5 */
  long long n_outlier;  /* e > 3.0f && e > 0.05f * g   (KITTI Fl / D1, evaluated in float32 as written) */
  double sum_err;       /* sum of e, in the fixed order below */
} ofdis_error_stats;
/* Evaluation against ground truth (extension) of the last run's slots [f0, f1) at the original frame size.  F is slot
 * a's full-resolution flow, exactly what ofdis_get_flow_fullres returns (computed from the level flows, without a
 * full-resolution copy); gt = G, [f1-f0][height_org][width_org][nop] float32 in this library's convention (stereo: the
 * disparity sign ofdis_get_flow_fullres returns).  In float32 without contraction:
 *   known ground truth: flow G_u, G_v not NaN and |G_u|, |G_v| <= 1e9 (Middlebury's UNKNOWN_FLOW_THRESH, so infinities
 *     are unknown); stereo G not NaN and |G| <= 1e9;
 *   flow: du = F_u - G_u, dv = F_v - G_v, e = sqrtf(du*du + dv*dv), g = sqrtf(G_u*G_u + G_v*G_v);
 *   stereo: e = fabsf(F - G), g = fabsf(G);
 *   err (optional, the same shape without nop): e where the ground truth is known, else the quiet NaN 0x7fc00000;
 *   a pixel counts for (pair, class c) when its ground truth is known and c = classes[pixel] < nclasses (classes:
 *     [f1-f0][height_org][width_org] bytes; NULL means class 0), so a byte of nclasses or more (e.g. 255) is ignored.
 * stats = [f1-f0][nclasses], always host memory.  Counts are exact.  sum_err is summed in this fixed order: per row y a
 * float64 sum starts at +0.0 and adds (double)e of the row's counted pixels of the class with x ascending; a float64
 * total starts at +0.0 and adds the row sums with y ascending.  NaN flows are not special-cased: a NaN e counts, makes
 * sum_err NaN and fails every > test.  gt, classes and err are in memkind (host ones go through the context's
 * full-resolution scratch); classes and err may be NULL.  Slots inside the context, non-NULL gt and stats,
 * 1 <= nclasses <= 16, classes non-NULL when nclasses > 1, else OFDIS_ERR_ARG; frame sizes as ofdis_get_flow_fullres
 * checks them.  The flows are not changed.  Synchronises the context's stream before it returns. */
int ofdis_flow_error_fullres(ofdis_ctx* ctx, int f0, int f1, const float* gt, const unsigned char* classes,
                             int nclasses, ofdis_error_stats* stats, float* err, int width_org, int height_org,
                             int memkind);
size_t ofdis_finest_level_frame_floats(const ofdis_ctx* ctx);
int ofdis_upload_finest_level(ofdis_ctx* ctx, int f0, int f1, const float* packed, int memkind);

/* Output stage on the device (extension, SURVEY 8f rank 2 == run_dense.cpp:407-414): flow of level
 * sc_l times 2^sc_l, bilinear upsampling by 2^sc_l (half-pixel centres, edge clamped), crop of the
 * divisibility padding.  `out` = [f1-f0][height_org][width_org][nop] floats.  Here and in the 8-bit uploads,
 * width_org/height_org pad up to the context's size by multiples of 2^sc_f, or of 2^(sc_f+1) as a run with an init
 * flow pads (run_dense.cpp:301); the crop is floor(pad/2) on the left/top either way. */
int ofdis_get_flow_fullres(ofdis_ctx* ctx, int f0, int f1, float* out, int width_org, int height_org, int memkind);
/* Encoded full-resolution flow (extension): F is each slot's full-resolution flow, exactly what
 * ofdis_get_flow_fullres returns, computed from the level-sc_l flows without a full-resolution float copy, and written
 * in a compact encoding.  Everything is float32, evaluated without contraction; the uint16 values are in host byte
 * order (a PNG writer stores them big-endian).
 *   OFDIS_ENC_F16: out = [f1-f0][height_org][width_org][nop] uint16 holding IEEE binary16.  Each channel is rounded
 *     to nearest even (__float2half_rn), so magnitudes of 65520 and more become +-inf.  Every NaN, whatever its sign
 *     or payload, becomes 0x7e00 (numpy's astype(float16) of the quiet NaN 0x7fc00000).
 *   OFDIS_ENC_KITTI, flow: out = [f1-f0][height_org][width_org][3] uint16, channels R, G, B of KITTI's 16-bit flow
 *     PNG.  Valid when u and v are not NaN: R = (uint16)fminf(fmaxf(u * 64.0f + 32768.0f, 0.0f), 65535.0f), G the
 *     same of v, B = 1.  Invalid: 0, 0, 0.
 *   OFDIS_ENC_KITTI, stereo: out = [f1-f0][height_org][width_org] uint16, KITTI's 16-bit disparity PNG.  d is the
 *     positive disparity: -F for an ordinary slot (the sign SavePFMFile writes), +F for a slot marked swapped
 *     (ofdis_set_swapped_slots, ofdis_upload_sequence_bidir_u8), which holds the right view.  Valid when d >= 0 (NaN
 *     fails, -0 passes): (uint16)fminf(fmaxf(d * 256.0f, 1.0f), 65535.0f); invalid: 0.  Disparities of 256 px and
 *     more are clamped to 65535 here; KITTI's format itself does not say what happens to them.
 * Arguments, slot and frame-size checks and status codes are those of ofdis_get_flow_fullres; an unknown encoding, a
 * NULL out or a device out that is not 2-byte aligned is OFDIS_ERR_ARG.  Host output goes through the context's
 * full-resolution scratch, sized as ofdis_get_flow_fullres sizes it (no encoding is larger than the float flow), so
 * alternating the two calls never reallocates.  Enqueued on the context's stream; not part of ofdis_run's graph.
 * The flows are not changed. */
enum { OFDIS_ENC_F16 = 1, OFDIS_ENC_KITTI = 2 };
int ofdis_get_flow_fullres_encoded(ofdis_ctx* ctx, int f0, int f1, int encoding, void* out, int width_org,
                                   int height_org, int memkind);
/* Color-coded full-resolution flow (extension): F is each slot's full-resolution flow, exactly what
 * ofdis_get_flow_fullres returns, computed from the level-sc_l flows without a full-resolution float copy.
 * rgb = [f1-f0][height_org][width_org][3] bytes, R, G, B; scale = NULL or [f1-f0] floats, the scale each slot was
 * colored with.  Everything is float32 without contraction, with IEEE division and square root; PI_F = (float)M_PI;
 * bytes are (uint8) of a float in [0, 256), by truncation.  preprocess.flow_to_color / disp_to_color restate it.
 *   Flow (nop 2), Middlebury's MotionToColor / computeColor (Baker et al. 2011):
 *     known pixel: u, v not NaN and |u|, |v| <= 1e9 (the rule of ofdis_flow_error_fullres, so +-inf is unknown);
 *     scale: max_value if it is > 0, else m, the maximum of sqrtf(u*u + v*v) over the slot's known pixels starting
 *       from 0, or 1 when m == 0 (an all-zero or all-unknown slot);
 *     unknown pixel: (0, 0, 0);
 *     known pixel: fx = u / scale, fy = v / scale, rad = sqrtf(fx*fx + fy*fy); a = atan2_f32(-v, -u) / PI_F of the
 *       unscaled flow (fx, fy may overflow for a tiny max_value); fk = (a + 1) / 2 * 54, k0 = (int)fk,
 *       k1 = (k0 + 1) % 55, f = fk - k0; per channel b
 *       col = (1.0f - f) * (W[k0][b] / 255.0f) + f * (W[k1][b] / 255.0f),
 *       col = rad <= 1 ? 1 - rad * (1 - col) : col * 0.75f, byte (uint8)(255.0f * col).  Zero flow is white.
 *     W: 55 integer entries of Middlebury's makecolorwheel, integer division, segments RY 15 (255, 255*i/15, 0),
 *       YG 6 (255 - 255*i/6, 255, 0), GC 4 (0, 255, 255*i/4), CB 11 (0, 255 - 255*i/11, 255),
 *       BM 13 (255*i/13, 0, 255), MR 6 (255, 0, 255 - 255*i/6).
 *     atan2_f32(y, x): the library's own float32 atan2, so the contract does not depend on a libm:
 *       ax = |x|, ay = |y|, mx = max(ax, ay), mn = min(ax, ay), t = mx > 0 ? mn / mx : 0, s = t * t,
 *       q = C7, then q = q * s + Ck for k = 6 .. 0, p = t * q with C0..C7 = 0.99999934f, -0.3332986f, 0.19946565f,
 *       -0.13908629f, 0.09642195f, -0.055912293f, 0.021862935f, -0.0040545613f;
 *       p = ay > ax ? PI_F * 0.5f - p : p; p = signbit(x) ? PI_F - p : p; result signbit(y) ? -p : p.
 *       Within 1e-6 of float64 atan2, in [-PI_F, PI_F] for finite input; signed zeros and axes as C's atan2.
 *   Stereo (nop 1), the color map of KITTI's stereo devkit (disp_to_color):
 *     d = -F for an ordinary slot, +F for a slot marked swapped (as OFDIS_ENC_KITTI); valid when 0 <= d <= 1e9 (NaN
 *       fails, -0 passes); scale: max_value if it is > 0, else fmaxf(m, 1), m the maximum valid d, starting from 0;
 *     invalid pixel: (0, 0, 0);
 *     M = {{0,0,0,114},{0,0,1,185},{1,0,0,114},{1,0,1,174},{0,1,0,114},{0,1,1,185},{1,1,0,114},{1,1,1,0}};
 *       wt[i] = 1000.0f / M[i][3]; cum[0] = 0, cum[i+1] = cum[i] + M[i][3] / 1000.0f for i = 0..6 in order;
 *     valid pixel: val = fminf(fmaxf(d / scale, 0), 1); i = the first of 0..6 with val < cum[i+1], else 6 (cum[7] is
 *       1.0f, so val = 1 takes the last bin); w = 1 - (val - cum[i]) * wt[i]; channel c
 *       (uint8)fminf(fmaxf((w * M[i][c] + (1 - w) * M[i+1][c]) * 255.0f, 0), 255).  In float32, w at val = 1 is
 *       3.6e-7 rather than 0, so d >= scale gives (255, 255, 254).
 *     These formulas follow the devkit's description; they have not been compared with the devkit's own output.
 * rgb NULL, max_value NaN, negative or infinite, slots outside the context, or a device scale that is not 4-byte
 * aligned is OFDIS_ERR_ARG; frame-size checks and status codes are those of ofdis_get_flow_fullres.  rgb and scale are
 * in memkind; host output goes through the context's full-resolution scratch at the size ofdis_get_flow_fullres asks
 * for, so alternating the two calls never reallocates.  The automatic scale launches two kernels (a per-slot
 * maximum into a workspace allocated on the first call, then the colors), a fixed scale one.  Enqueued on the context's
 * stream; not part of ofdis_run's graph.  The flows are not changed. */
int ofdis_flow_color_fullres(ofdis_ctx* ctx, int f0, int f1, unsigned char* rgb, float* scale, float max_value,
                             int width_org, int height_org, int memkind);
/* Frame interpolation from bidirectional flows (extension): the frame at time t between I0 and I1 of every pair
 * k < f1-f0.  Slot a = f0+k holds the forward flow F (I0 -> I1) of the last run and slot b0+k its backward partner B
 * (I1 -> I0): the layout of ofdis_upload_sequence_bidir_u8 (b0 = n), or of pairs followed by their swapped copies.
 * F and B are exactly what ofdis_get_flow_fullres returns, computed from the level flows without a full-resolution
 * copy; stereo (nop 1) uses F as a horizontal flow with v = 0, which gives the view at fraction t between the two
 * cameras (swapped marks need no special case).  i0, i1: the 8-bit frames [height_org][width_org][noc] in the
 * context's channel count, frame k at i0 + k*frame_stride and i1 + k*frame_stride, frame_stride >= height_org *
 * width_org * noc (a clip: i1 = i0 + hwc, stride hwc; the pairs of ofdis_upload_frames_u8: stride 2hwc).
 * out = [f1-f0][height_org][width_org][noc] bytes; flow_t = NULL or [f1-f0][height_org][width_org][nop] float32, the
 * filled flow u_t at time t.  The algorithm follows the description of the interpolation in Baker et al.'s
 * evaluation (IJCV 2011); it has not been compared with their implementation.  Everything is float32 without
 * contraction, with IEEE division; preprocess.interpolate_frames restates it.  W = width_org, H = height_org;
 * bil(I, xs, ys) is the bilinear rule of ofdis_consistency_fullres on the (float) byte values: x0 = floor(xs),
 * x1 = min(x0 + 1, W - 1), fx = xs - x0 (the same in y), per channel r0 = I(x0,y0)*(1-fx) + I(x1,y0)*fx,
 * r1 = I(x0,y1)*(1-fx) + I(x1,y1)*fx, bil = r0*(1-fy) + r1*fy.  "In the frame" is 0 <= x <= W-1 and 0 <= y <= H-1.
 * Per pair:
 *   1. m0 = the mask ofdis_consistency_fullres(alpha, beta) gives F against B (every pixel of I0), m1 the mask of B
 *      against F (every pixel of I1), bitwise; a pixel whose mask is not 0 (1, or 2: it leaves the frame) is
 *      occluded in the other frame.
 *   2. Cost of source pixel (X, Y) of I0: xs = X + u, ys = Y + v with (u, v) = F(X, Y); c = +inf when (xs, ys) is
 *      not in the frame (or NaN), else c = 0, then c += fabsf(I0(X,Y)[ch] - bil(I1, xs, ys)[ch]) in channel order.
 *   3. Forward splat: a source with |u| <= 1e9 and |v| <= 1e9 (NaN fails) has the target p = (X + t*u, Y + t*v) and
 *      reaches every pixel of the frame with a non-zero bilinear weight at p: x = floor(px), and floor(px) + 1 when
 *      px > floor(px), the same in y.  Every target keeps the source with the smallest 64-bit key
 *      (bits(c) << 32) | (Y*W + X): the lowest cost, on a tie the lowest source index.  u_t = F of that source.
 *   4. Hole filling: pixels no source reached are holes.  In rounds r = 1, 2, ...: a hole with at least one neighbour
 *      (left, right, up, down) filled before round r takes, per component, s = 0, s += each such neighbour's u_t in
 *      that order, u_t = s / k with k their count; rounds repeat until no hole is left.  A pair that no source
 *      reached has u_t = 0 everywhere.
 *   5. Color: x0 = X - t*u_t, x1 = X + (1.0f - t)*u_t (the same in y); in0, in1 = (x0, y0), (x1, y1) in the frame;
 *      s0 = bil(I0, clamp(x0, y0)), s1 = bil(I1, clamp(x1, y1)) with the coordinates clamped to the frame;
 *      o0 = in0 && m0(rnd(x0), rnd(y0)) != 0, o1 = in1 && m1(rnd(x1), rnd(y1)) != 0, rnd(x) = (int)floorf(x + 0.5f);
 *      value s0 when (in0 && !in1) || (o0 && !o1), s1 when (in1 && !in0) || (o1 && !o0), else
 *      (1.0f - t)*s0 + t*s1; each byte (unsigned char)(fminf(fmaxf(value, 0), 255) + 0.5f).
 * Slots outside the context, NULL i0, i1 or out, t not in (0, 1) (or NaN), frame_stride below one frame, alpha or
 * beta not finite and >= 0, or a device flow_t that is not 4-byte aligned is OFDIS_ERR_ARG; frame-size checks and
 * status codes are those of ofdis_get_flow_fullres.  i0, i1, out and flow_t are in memkind: host frames go through
 * the context's staging buffer (two 2-D copies), host output through its full-resolution scratch at the size
 * ofdis_get_flow_fullres asks for.  The workspace -- per pixel and pair 30 bytes for flow, 26 for stereo (the 64-bit
 * keys, u_t, fill stamps, two hole lists, two masks), for max_frames pairs of the context's size -- is allocated on
 * the first call and freed by ofdis_destroy; a context of more than 2^32 such pixels is OFDIS_ERR_UNSUPPORTED.  Not
 * part of ofdis_run's graph; the flows are not changed.  The hole filling reads a count of the holes left on the host
 * after rounds 8, 24, 56, ... (batches double up to 256 rounds), so the call synchronises the context's stream, once
 * when the holes are at most 8 pixels from a splatted one. */
int ofdis_interpolate_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* i0, const unsigned char* i1,
                              size_t frame_stride, float t, float alpha, float beta, unsigned char* out, float* flow_t,
                              int width_org, int height_org, int memkind);

/* Filtered disparity, depth and point cloud from stereo flows (extension, stereo contexts only).  Everything is
 * float32 without contraction, with IEEE division; preprocess.disparity_filter restates it.  W = width_org,
 * H = height_org, qNaN = the quiet NaN 0x7fc00000; "the smaller of a and b" is (b < a) ? b : a, so of two equal values
 * (+0 and -0 among them) the first one is taken.  For every pair k < f1-f0, in this order:
 *   1. Disparity.  F is slot a = f0+k's full-resolution flow, exactly what ofdis_get_flow_fullres returns (computed from
 *      the level flows without a full-resolution copy); d = -F for an ordinary slot, +F for a slot marked swapped (the
 *      rule of OFDIS_ENC_KITTI and of the stereo color map).
 *   2. Status.  3 when d is not in [0, 1e9] (NaN fails, -0 passes); else, with lr_check, the mask of
 *      ofdis_consistency_fullres(alpha, beta) of slot a against slot b0+k, bitwise (1 inconsistent, 2 leaves the
 *      frame); else 0, valid.
 *   3. Speckles (speckle_size > 0).  Two 4-neighbours of status 0 are joined when fabsf(d_p - d_q) <= speckle_diff
 *      (diagonal neighbours are not); every pixel of a connected component of at most speckle_size pixels gets status 4.
 *   4. Fill (fill = 1).  At first only the pixels of status 0 have a value, d.  Row pass: each maximal run [x1, x2] of
 *      pixels without a value with x1 > 0 and x2 < W-1 takes the smaller of the values at x1-1 and x2+1; pixels left of
 *      the row's first value take that value, pixels right of its last value that one.  Then the same rule along the
 *      columns over what the row pass left.  After the row pass a row is either full or empty, so the column pass
 *      fills the empty rows: bridging empty rows between two full ones is this library's choice (KITTI's devkit is
 *      described as extrapolating up and down only).  A frame without a status-0 pixel stays empty.  These rules
 *      follow the description of the devkit's interpolateBackground; they have not been compared with its output.
 *   5. Outputs, each [n][H][W] in memkind and each may be NULL, but not all four:
 *      disp: d where the status is 0, the filled value where one exists, else qNaN;
 *      status: bytes 0..4; filling does not change it, so status != 0 with a finite disp marks a filled pixel;
 *      depth: with D = disp, Z = (fx * baseline) / (D + doffs) where D + doffs > 0 (NaN fails), else qNaN; the product
 *        fx * baseline is rounded once;
 *      xyz: [n][H][W][3], (((float)x - cx) * Z) / fx, (((float)y - cy) * Z) / fy, Z.
 *      Every NaN written to depth or xyz is qNaN.
 * cam is required for depth and xyz, one camera per call (the right view's depth takes the right camera, e.g.
 * Middlebury's cam1, in a call of its own): fx, fy, baseline finite and > 0, cx, cy, doffs finite.  filt: lr_check and
 * fill 0 or 1, alpha, beta and speckle_diff finite and >= 0, speckle_size >= 0.  b0 is read only with lr_check.
 * OFDIS_ERR_ARG: a flow context (nop 2), slots outside the context, a NULL or bad filt, a missing or bad cam when depth
 * or xyz is asked for, all four outputs NULL, or a device output that is not aligned to its element; frame sizes as
 * ofdis_get_flow_fullres checks them; W * H >= 2^31 is OFDIS_ERR_UNSUPPORTED (the labels are int32 per frame).
 * The workspace -- per pixel and pair 13 bytes (d, the parent, the component size, the status) and per row and pair
 * 12 (the row pass's flag and the nearest full rows), for max_frames pairs of the context's size -- is allocated on
 * the first call, never shrinks, and is freed by ofdis_destroy.  Host outputs go through the context's
 * full-resolution scratch, grown to max_frames x 21 bytes per pixel of the call's size (disp, depth and xyz floats, then
 * the status bytes) and at least what ofdis_get_flow_fullres asks for.  Enqueued on the context's stream with a fixed
 * number of kernels per call whatever the number of pairs (2, + 3 with speckles, + 2 with fill); host outputs
 * synchronise it.  Not part of ofdis_run's graph; the flows are not changed. */
typedef struct ofdis_disp_filter {
  int lr_check;        /* 0 | 1: test slot f0+k against partner slot b0+k */
  float alpha, beta;   /* the rule of ofdis_consistency_fullres (usual: 0, 1) */
  int speckle_size;    /* 0: off; else components of at most this many pixels are removed */
  float speckle_diff;  /* 4-neighbours join a component when |d_p - d_q| <= speckle_diff */
  int fill;            /* 0 | 1: background fill */
} ofdis_disp_filter;
typedef struct ofdis_stereo_camera { float fx, fy, cx, cy, baseline, doffs; } ofdis_stereo_camera;
int ofdis_disparity_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_disp_filter* filt,
                            const ofdis_stereo_camera* cam, float* disp, unsigned char* status, float* depth,
                            float* xyz, int width_org, int height_org, int memkind);

/* Scene flow from a flow and two disparity maps (extension, flow contexts only): the second disparity warped to the
 * first frame, the 3-D motion of every pixel and KITTI 2015's D1, D2, Fl and SF outlier counts.  Everything is
 * float32 without contraction, with IEEE division; preprocess.scene_flow restates it bit for bit.  W = width_org,
 * H = height_org, qNaN = the quiet NaN 0x7fc00000, known(d) = 0 <= d <= 1e9 (NaN fails, -0 passes).  For every pair
 * k < f1-f0 and pixel (x, y):
 *   F = (u, v): slot f0+k's full-resolution flow, exactly what ofdis_get_flow_fullres returns (computed from the level
 *     flows without a full-resolution copy).  d0 = D0(x, y) with D0 = disp0 + k*disp_stride, D1 = disp1 + k*disp_stride,
 *     both [H][W] positive disparities with NaN for unknown (the disp output of ofdis_disparity_fullres, or a decoded
 *     KITTI PNG); disp_stride >= W*H floats, so a clip of n+1 maps passes disp1 = disp0 + W*H.
 *   1. Target.  (xs, ys) = ((float)x + u, (float)y + v); it fails outside [0, W-1] x [0, H-1] (or NaN).
 *   2. d1, the second disparity at the target.  x0 = floor(xs), x1 = min(x0 + 1, W-1), fx = xs - x0 (the same in y).
 *      When the four corners are known and max - min of them <= edge_diff: the bilinear value of
 *      ofdis_consistency_fullres, r0 = D1(x0,y0)*(1-fx) + D1(x1,y0)*fx, r1 = D1(x0,y1)*(1-fx) + D1(x1,y1)*fx,
 *      d1 = r0*(1-fy) + r1*fy.  Otherwise the nearest corner, D1(fx >= 0.5f ? x1 : x0, fy >= 0.5f ? y1 : y0), so that a
 *      depth edge gives one of its sides rather than a "flying" disparity between them.  edge_diff = +inf always blends.
 *   3. status (bytes): bit 0 d0 is not known, bit 1 the target fails, bit 2 d1 is not known (only when bit 1 is clear).
 *   4. disp1_warped = d1 where bits 1 and 2 are clear, else qNaN: KITTI's D2 (disp_occ_1) in frame-t coordinates.
 *   5. motion = [n][H][W][3], needs cam: fb = fx * baseline rounded once; where status = 0, s0 = d0 + doffs > 0 and
 *      s1 = d1 + doffs > 0: Z0 = fb / s0, X0 = (((float)x - cx) * Z0) / fx, Y0 = (((float)y - cy) * Z0) / fy (the xyz of
 *      ofdis_disparity_fullres bit for bit), Z1 = fb / s1, X1 = ((xs - cx) * Z1) / fx, Y1 = ((ys - cy) * Z1) / fy, and
 *      motion = (X1 - X0, Y1 - Y0, Z1 - Z0); elsewhere (qNaN, qNaN, qNaN).  Every NaN written is qNaN.
 *   6. Evaluation (gt and stats).  Ground truth is known as above for gt.disp0 and gt.disp1, and as in
 *      ofdis_flow_error_fullres (|G_u|, |G_v| <= 1e9) for gt.flow.  D1 compares d0 with gt.disp0, D2 disp1_warped with
 *      gt.disp1: e = fabsf(est - G), g = fabsf(G).  Fl compares F with gt.flow: e = sqrtf(du*du + dv*dv) with
 *      (du, dv) = F - G, g = sqrtf(G_u*G_u + G_v*G_v).  An unknown estimate (a disparity that is not known, a flow with
 *      |u| or |v| not <= 1e9) has e = +inf.  A component is an outlier when e > 3.0f && e > 0.05f * g (the KITTI
 *      expression of ofdis_flow_error_fullres), so an unknown estimate is always one.  KITTI's devkit instead fills
 *      unknown estimates from the background before it compares; pass filled disparities (ofdis_disparity_fullres with
 *      fill) for its behaviour.  Each component counts where its ground truth is known; a pixel counts for SF where
 *      all three are known, and is an SF outlier where any of its three components is an outlier.  A pixel counts for
 *      (pair k, class c) with c = classes[k][y][x] < nclasses (classes NULL: class 0), as ofdis_flow_error_fullres.
 * stats = [f1-f0][nclasses] exact counts, always host memory.  disp0, disp1, gt's three arrays ([n][H][W], [n][H][W]
 * and [n][H][W][2], this library's flow convention), classes ([n][H][W] bytes) and the outputs disp1_warped
 * ([n][H][W]), status and motion are in memkind; each output may be NULL, but not all three when stats is NULL.  Host
 * inputs go through the context's staging buffer, host outputs through its full-resolution scratch.  Device
 * disparities may come from another context on the same device (a stereo context's ofdis_disparity_fullres); the
 * caller orders that work before this call, by sharing the stream or with an event.  OFDIS_ERR_ARG: a stereo context,
 * slots outside the context, NULL disp0 or disp1, disp_stride < W*H, edge_diff NaN or negative, all outputs and stats
 * NULL, gt and stats not given together (or a NULL array in gt), nclasses not in 1..16, classes NULL when nclasses > 1,
 * motion without cam, a cam whose fx, fy, baseline are not finite and > 0 or whose cx, cy, doffs are not finite, or a
 * device pointer that is not aligned to its element; frame sizes as ofdis_get_flow_fullres checks them.  The counters,
 * 64 bytes per (pair, class) for max_frames x 16, are allocated on the first call and freed by ofdis_destroy.
 * Enqueued on the context's stream as one kernel, plus one memset of the counters with stats, whatever the number of
 * pairs; host outputs or stats synchronise the stream.  Not part of ofdis_run's graph; the flows are not changed. */
typedef struct ofdis_sf_gt {            /* all three [n][H][W](...) in memkind */
  const float* disp0;                   /* positive disparity at t, NaN = unknown */
  const float* disp1;                   /* positive disparity at t+1 of the point seen at (x, y) in frame t (KITTI disp_occ_1) */
  const float* flow;                    /* [n][H][W][2], this library's convention */
} ofdis_sf_gt;
typedef struct ofdis_sf_stats {         /* per (pair, class), 64 bytes, exact counts */
  long long n_d1, n_d2, n_fl, n_sf;     /* pixels counted */
  long long out_d1, out_d2, out_fl, out_sf;
} ofdis_sf_stats;
int ofdis_scene_flow_fullres(ofdis_ctx* ctx, int f0, int f1, const float* disp0, const float* disp1,
                             size_t disp_stride, float edge_diff, const ofdis_stereo_camera* cam,
                             float* disp1_warped, unsigned char* status, float* motion,
                             const ofdis_sf_gt* gt, const unsigned char* classes, int nclasses,
                             ofdis_sf_stats* stats, int width_org, int height_org, int memkind);

/* Global camera motion from dense flows (extension, flow contexts only): a RANSAC fit of one similarity, affine map
 * or homography per pair, its least-squares refits on the inliers, and from the model per pixel the residual flow, a
 * moving-pixel mask and I1 registered onto I0.  preprocess.global_motion restates it bit for bit.  float32 where
 * marked, float64 in the solver, everything without contraction and with IEEE division.  W = width_org,
 * H = height_org, s = step, qNaN = the quiet NaN 0x7fc00000.  For every pair k < f1-f0, slot a = f0+k:
 *   1. Correspondences.  The cells (i, j) are ceil(W/s) x ceil(H/s) in row-major order (j outer), cell (i, j) has the
 *      pixel cx = min(i*s + s/2, W-1), cy = min(j*s + s/2, H-1) (the seed grid of ofdis_track_begin).  F = (u, v) is
 *      slot a's full-resolution flow at (cx, cy), exactly what ofdis_get_flow_fullres returns.  A cell is valid when
 *      |u| <= 1e9 and |v| <= 1e9 (NaN fails), (xs, ys) = ((float)cx + u, (float)cy + v) lies in [0, W-1] x [0, H-1],
 *      and, with fb_check, the mask of ofdis_consistency_fullres(alpha, beta) of slot a against slot b0+k is 0 there.
 *      The valid cells, in cell order, are the m correspondences (x, y, p, q) in float32 normalized coordinates:
 *      c_x = 0.5f * (float)(W-1), c_y = 0.5f * (float)(H-1), sigma = 2.0f / (float)max(W, H), x = ((float)cx - c_x)
 *      * sigma, y = ((float)cy - c_y) * sigma, p = (xs - c_x) * sigma, q = (ys - c_y) * sigma.  m < n_min: status 1.
 *   2. Hypotheses h = 0 .. hypotheses-1.  Draw d < n_min takes z = mix(seed + (uint64)(8h + d + 1) * G) with
 *      G = 0x9E3779B97F4A7C15 and SplitMix64's finalizer mix(z): z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9,
 *      z = (z ^ (z >> 27)) * 0x94D049BB133111EB, z ^ (z >> 31) (all mod 2^64; this is the (8h+d+1)-th output of the
 *      SplitMix64 generator seeded with `seed`), and the correspondence index (uint32)(((z >> 32) * m) >> 32).  The
 *      draws depend on h, d, m and seed only, so a pair's whole result depends only on its own flows and the params.
 *      The draws give 2 n_min rows, point by point, row x then row y, of (double) of the float32 values:
 *        similarity (k = 4):  [x, -y, 1, 0 | p], [y, x, 0, 1 | q];           H^ = [a, -b, tx; b, a, ty; 0, 0, 1]
 *        affine     (k = 6):  [x, y, 1, 0, 0, 0 | p], [0, 0, 0, x, y, 1 | q]; H^ = [h0, h1, h2; h3, h4, h5; 0, 0, 1]
 *        homography (k = 8):  [x, y, 1, 0, 0, 0, -(x*p), -(y*p) | p], [0, 0, 0, x, y, 1, -(x*q), -(y*q) | q];
 *                             H^ = [h0, h1, h2; h3, h4, h5; h6, h7, 1]
 *      solved by THE elimination of this call: for column j: the pivot row is the first i >= j of the largest
 *      |a_ij|; a pivot that is not > 0 in magnitude fails; swap rows; for each i > j: f = a_ij / a_jj, a_ic = a_ic - f
 *      * a_jc for c > j, b_i = b_i - f * b_j.  Back substitution for i = k-1 .. 0: x_i = b_i, x_i = x_i - a_ic * x_c for
 *      c = i+1 .. k-1, x_i = x_i / a_ii.  A failed pivot or a non-finite x_i makes the hypothesis unsolvable (a repeated
 *      index gives a zero pivot).
 *   3. Scoring.  g0..g8 = H^ rounded to float32, t = threshold * sigma (float32).  Correspondence (x, y, p, q) is an
 *      inlier iff W' > 0 and ex*ex + ey*ey <= (t*W')*(t*W') with X' = (g0*x + g1*y) + g2, Y' = (g3*x + g4*y) + g5,
 *      W' = (g6*x + g7*y) + g8, ex = X' - p*W', ey = Y' - q*W' (reprojection error <= t, without a division).  The best
 *      solvable hypothesis has the most inliers, the lowest h on a tie (the largest (count << 32) | (0xFFFFFFFF - h)).
 *      No solvable hypothesis: status 2.
 *   4. Refits, rounds 1 .. refine: the inliers of the current model (the test above); fewer than n_min: stop.  Normal
 *      equations from each inlier's two rows r1 | b1, r2 | b2: N_ij = (r1_i*r1_j) + (r2_i*r2_j) for i <= j, the
 *      right-hand side (r1_i*b1) + (r2_i*b2), other correspondences +0.0.  Each sum runs over chunks of 32 consecutive
 *      correspondences, each chunk from +0.0 in order, then a pairwise tree over the chunk sums padded with +0.0 to a
 *      power of two (level by level, v_i = v_2i + v_2i+1).  N is mirrored and solved by the elimination; a failure
 *      stops and keeps the model, else the solution replaces it.
 *   5. model (row-major 3 x 3, float64) = T^-1 H^ T in pixel coordinates, mapping an I0 pixel to its I1 position:
 *      with h = H^, S = (double)sigma, Cx = (double)c_x, Cy = (double)c_y, per row r: A_r0 = h_r0*S, A_r1 = h_r1*S,
 *      A_r2 = h_r2 - (A_r0*Cx + A_r1*Cy); M_0c = A_0c/S + Cx*A_2c, M_1c = A_1c/S + Cy*A_2c, M_2c = A_2c; a homography
 *      is then divided entry by entry by the M_22 of before.  Every NaN of the model is the float64 qNaN
 *      0x7ff8000000000000; status != 0: nine of them.
 *   6. Per pixel (X, Y) of the frame, m0..m8 = model rounded to float32: mx = (m0*X + m1*Y) + m2, my = (m3*X + m4*Y)
 *      + m5, w = (m6*X + m7*Y) + m8, the model flow (mx/w - X, my/w - Y).  residual = F - the model flow, per
 *      component, every NaN written as qNaN.  mask: 2 where F is unknown, (X + u, Y + v) leaves the frame or, with
 *      fb_check, the consistency mask is not 0; else 0 where rx*rx + ry*ry <= threshold*threshold (float32), else 1 (moves independently).
 *      registered: with w > 0 and (mx/w, my/w) in the frame, I1 there by the bilinear byte rule and rounding of
 *      ofdis_interpolate_fullres, else 0.  A pair of status != 0 writes residual qNaN, mask 2 and registered 0.
 * stats per pair: status, n_corr = m, best_hypothesis (-1 unless status 0), ransac_inliers (its count), refits (the
 * refits that replaced the model), n_inliers (the final model's count).  model = [n][9] doubles and stats = [n] are
 * host memory.  mask [n][H][W] bytes, residual [n][H][W][2] float32 and registered [n][H][W][noc] bytes are optional
 * (NULL skips them) and in memkind; registered needs i1: the 8-bit frame I1 of pair k at i1 + k*frame_stride, the
 * convention of ofdis_interpolate_fullres (host frames go through the staging buffer, host outputs through the
 * full-resolution scratch).  OFDIS_ERR_ARG: a stereo context, slots outside the context (b0 only with fb_check), a NULL
 * p or one out of range (model 1..3, step >= 1, fb_check 0|1, alpha and beta finite and >= 0, hypotheses 1..65536,
 * threshold finite and > 0, refine 0..16), a NULL model or stats, registered without i1, frame_stride below one frame,
 * a device residual not 4-byte aligned, or more than 2^24 cells per pair; frame sizes as ofdis_get_flow_fullres checks
 * them.  The workspace -- per cell and pair 28 bytes (the correspondence, its flag, the refit's chunk sums), per
 * hypothesis and pair 112 (its float64 parameters and float32 H^) and 128 per pair -- is allocated on the first call,
 * grows, never shrinks and is freed by ofdis_destroy.  Enqueued on the context's stream as 5 kernels, plus one when a
 * per-pixel output is asked for, whatever the number of pairs; the call synchronises the stream once, at the end, for
 * model and stats.  Not part of ofdis_run's graph; the flows are not changed. */
enum { OFDIS_MOTION_SIMILARITY = 1, OFDIS_MOTION_AFFINE = 2, OFDIS_MOTION_HOMOGRAPHY = 3 };
typedef struct ofdis_motion_params {
  int model;                 /* OFDIS_MOTION_*: n_min = 2, 3, 4 points, k = 4, 6, 8 unknowns */
  int step;                  /* correspondence grid step s >= 1 */
  int fb_check;              /* 0 | 1: only correspondences whose consistency mask against slot b0+k is 0 */
  float alpha, beta;         /* the rule of ofdis_consistency_fullres; finite, >= 0 */
  int hypotheses;            /* 1 .. 65536 */
  float threshold;           /* inlier reprojection error in pixels; finite, > 0 */
  int refine;                /* 0 .. 16 least-squares refits on the inliers */
  unsigned long long seed;
} ofdis_motion_params;
typedef struct ofdis_motion_stats {
  int status;                /* 0 fitted, 1 fewer than n_min correspondences, 2 no solvable hypothesis */
  int n_corr, best_hypothesis, ransac_inliers, refits, n_inliers;
} ofdis_motion_stats;
int ofdis_global_motion_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_motion_params* p,
                                const unsigned char* i1, size_t frame_stride, double* model,
                                ofdis_motion_stats* stats, unsigned char* mask, float* residual,
                                unsigned char* registered, int width_org, int height_org, int memkind);

/* Stereo ego-motion from flows and disparities (extension, flow contexts only): a RANSAC fit of one rigid transform
 * [R | t] per pair from the camera at t to the camera at t+1, its Gauss-Newton refits on the inliers, and from the pose
 * per pixel an independent-motion mask, the residual flow and the object motion.  preprocess.egomotion restates it
 * bit for bit.  float32 where marked, float64 in the solver, everything without contraction and with IEEE division
 * and square root; no transcendental function.  W = width_org, H = height_org, s = step, qNaN = the quiet NaN
 * 0x7fc00000, known(d) = 0 <= d <= 1e9, fb = fx * baseline rounded once to float32.  For every pair k < f1-f0, slot
 * a = f0+k, D0 = disp0 + k*disp_stride, D1 = disp1 + k*disp_stride ([H][W] positive disparities, NaN unknown, as
 * ofdis_scene_flow_fullres takes them):
 *   1. Correspondences.  The cells of ofdis_global_motion_fullres at step s, cell (i, j) read at its pixel (px, py).
 *      F = (u, v) is slot a's flow there (ofdis_get_flow_fullres's value), (xs, ys) = ((float)px + u, (float)py + v),
 *      d0 = D0(px, py), d1 = D1 gathered at (xs, ys) by step 2 of ofdis_scene_flow_fullres with edge_diff (when the
 *      target lies in [0, W-1] x [0, H-1]), s0 = d0 + doffs, s1 = d1 + doffs.  A cell is valid when d0 is known,
 *      s0 > 0, the target lies in the frame, d1 is known, s1 > 0 and, with fb_check, the mask of
 *      ofdis_consistency_fullres(alpha, beta) of slot a against slot b0+k is 0 there.  It gives P = (X, Y, Z), the
 *      xyz of scene flow's step 5 (Z = fb / s0, X = (((float)px - cx) * Z) / fx, Y = (((float)py - cy) * Z) / fy) and
 *      the observation (xs, ys, d1).  The valid cells in cell order are the m correspondences; m < 3: status 1.
 *   2. Hypotheses h = 0 .. hypotheses-1.  Draws d = 0, 1, 2 by ofdis_global_motion_fullres's SplitMix64 rule give
 *      correspondences a, b, c.  Q, the t+1 point of an observation, is scene flow's Z1 = fb / s1,
 *      X1 = ((xs - cx) * Z1) / fx, Y1 = ((ys - cy) * Z1) / fy (float32).  In float64 of the float32 values, the triad
 *      of three points A, B, C: u = B - A, L = sqrt((u0*u0 + u1*u1) + u2*u2), e1 = u / L (per component),
 *      n' = e1 x (C - A) with x the cross product (a1*b2 - a2*b1, a2*b0 - a0*b2, a0*b1 - a1*b0),
 *      Ln = sqrt(n'.n') as L, n = n' / Ln, e2 = n x e1.  The triads (e1, e2, n) of P and (f1, f2, q) of Q give
 *      R_ij = ((f1_i*e1_j) + (f2_i*e2_j)) + (q_i*n_j) and t_i = cQ_i - (((R_i0*cP_0) + (R_i1*cP_1)) + (R_i2*cP_2)),
 *      with the centroids c_i = ((a_i + b_i) + c_i) / 3.0.  A length that is not > 0 or a non-finite entry of R or t
 *      makes the hypothesis unsolvable (repeated or collinear draws).
 *   3. Scoring.  g = [R | t] rounded to float32 (row-major, 12), P' = (X', Y', Z') with X' = ((g0*X + g1*Y) + g2*Z)
 *      + g3 (rows 4..7, 8..11 the same).  A correspondence is an inlier iff Z' > 0 and (ex*ex + ey*ey) + ed*ed <=
 *      tz*tz with ex = (fx*X' + cx*Z') - xs*Z', ey = (fy*Y' + cy*Z') - ys*Z', ed = fb - s1*Z', tz = threshold*Z'
 *      (float32): the left-image and disparity reprojection error <= threshold, without a division.  The best
 *      solvable hypothesis has the most inliers, the lowest h on a tie (the largest (count << 32) | (0xFFFFFFFF - h)).
 *      No solvable hypothesis: status 2.
 *   4. Refits, rounds 1 .. refine: the inliers of the current model by the test above; fewer than 3: stop.  For each
 *      inlier, in float64 with P' = R P + t (P'_i = (((R_i0*X) + (R_i1*Y)) + (R_i2*Z)) + t_i), iz = 1.0 / Z',
 *      u = X' * iz, v = Y' * iz, three residuals and their gradients a = d(residual)/dP':
 *        x: r = ((fx*u) + cx) - xs,        a = (fx*iz, 0, -((fx*iz)*u))
 *        y: r = ((fy*v) + cy) - ys,        a = (0, fy*iz, -((fy*iz)*v))
 *        d: r = ((fb*iz) - doffs) - d1,    a = (0, 0, -((fb*iz)*iz))
 *      and the Jacobian row of (omega, tau) with w = 2 P' per component: ((a1*-w2) + (a2*w1), (a0*w2) + (a2*-w0),
 *      (a0*-w1) + (a1*w0), a0, a1, a2).  N_ij = ((Jx_i*Jx_j) + (Jy_i*Jy_j)) + (Jd_i*Jd_j) for i <= j and
 *      b_i = -(((Jx_i*rx) + (Jy_i*ry)) + (Jd_i*rd)), summed as ofdis_global_motion_fullres's refits sum (chunks of 32
 *      from +0.0, then the pairwise tree), mirrored and solved by its elimination.  A failure stops and keeps the
 *      model; else with (omega, tau) = x, q = (w0*w0 + w1*w1) + w2*w2 (w = omega), the Cayley rotation
 *      C_ij = (((i == j ? 1.0 - q : 0.0) + (2.0*(w_i*w_j))) + (2.0*K_ij)) / (1.0 + q) with K = [omega]x =
 *      [0, -w2, w1; w2, 0, -w0; -w1, w0, 0], then [R | t]_ij = ((C_i0*M_0j) + (C_i1*M_1j)) + (C_i2*M_2j) of the old
 *      [R | t] = M for j = 0..3, and t_i = t_i + tau_i.
 *   5. pose = [n][12] float64 row-major [R | t]: camera-t coordinates to camera-t+1 coordinates.  Status != 0: twelve
 *      float64 qNaN 0x7ff8000000000000.
 *   6. Per pixel (X, Y), with g = the pose rounded to float32 and step 1's values at the pixel: mask 2 where the pixel
 *      is not valid by step 1 or Z' <= 0 (or NaN), 0 where it passes step 3's test, else 1 (moves independently).
 *      residual = (u - (((fx*X')/Z' + cx) - (float)X), v - (((fy*Y')/Z' + cy) - (float)Y)) where d0 is known and
 *      s0 > 0, else qNaN: F minus the flow the pose induces.  object_motion = (X1 - X', Y1 - Y', Z1 - Z') with Q as in
 *      step 2, where mask != 2, else qNaN: the pixel's 3-D motion relative to the static scene.  Every NaN written is
 *      qNaN; a pair of status != 0 writes mask 2 and qNaN.
 * stats per pair: the ofdis_motion_stats of ofdis_global_motion_fullres (status, n_corr = m, best_hypothesis,
 * ransac_inliers, refits that replaced the model, n_inliers of the final model).  pose and stats are host memory;
 * mask [n][H][W] bytes, residual [n][H][W][2] and object_motion [n][H][W][3] float32 are optional (NULL skips them)
 * and in memkind, as disp0 and disp1 are.  Host inputs go through the context's staging buffer, host outputs through
 * its full-resolution scratch.  Device disparities may come from another context on the same device; the caller
 * orders that work before this call.  OFDIS_ERR_ARG: a stereo context, slots outside the context (b0 only with
 * fb_check), a NULL p or one out of range (step >= 1, fb_check 0|1, alpha and beta finite and >= 0, edge_diff >= 0
 * (+inf allowed), hypotheses 1..65536, threshold finite and > 0, refine 0..16), a NULL or bad cam (as
 * ofdis_scene_flow_fullres checks it), NULL disp0, disp1, pose or stats, disp_stride < W*H, a device pointer that is
 * not aligned to its element, or more than 2^24 cells per pair; frame sizes as ofdis_get_flow_fullres checks them.
 * The workspace -- per cell and pair 39.75 bytes (the 32-byte correspondence, its flag, the refit's 27 chunk sums per
 * 32 cells), per hypothesis and pair 160 (its float64 [R | t] and the float32 record) and 140 per pair -- is allocated
 * on the first call, grows, never shrinks and is freed by ofdis_destroy.  Enqueued on the context's stream as 5
 * kernels, plus one when a per-pixel output is asked for, whatever the number of pairs; the call synchronises the
 * stream once, at the end, for pose and stats.  Not part of ofdis_run's graph; the flows are not changed. */
typedef struct ofdis_egomotion_params {
  int step;                  /* correspondence grid step s >= 1 (the seed grid of ofdis_track_begin) */
  int fb_check;              /* 0 | 1: only correspondences whose consistency mask against slot b0+k is 0 */
  float alpha, beta;         /* the rule of ofdis_consistency_fullres; finite, >= 0 */
  float edge_diff;           /* the d1 gather of ofdis_scene_flow_fullres; >= 0, +inf allowed */
  int hypotheses;            /* 1 .. 65536 */
  float threshold;           /* inlier stereo reprojection error in pixels; finite, > 0 */
  int refine;                /* 0 .. 16 Gauss-Newton rounds on the inliers */
  unsigned long long seed;
} ofdis_egomotion_params;
int ofdis_egomotion_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_egomotion_params* p,
                            const float* disp0, const float* disp1, size_t disp_stride,
                            const ofdis_stereo_camera* cam, double* pose, ofdis_motion_stats* stats,
                            unsigned char* mask, float* residual, float* object_motion,
                            int width_org, int height_org, int memkind);

/* Monocular relative pose from dense flows (extension, flow contexts only): a RANSAC eight-point fit of one essential
 * matrix per pair with one calibrated camera, its decomposition, Gauss-Newton refits of the 5-DoF motion on the
 * epipolar inliers, a parallax guard, and per pixel an epipolar mask, the Sampson distance and the depth up to scale.
 * preprocess.relpose restates it bit for bit.  float32 where marked, float64 in the solver, everything without
 * contraction and with IEEE division and square root; no transcendental function.  W = width_org, H = height_org,
 * s = step, qNaN = the quiet NaN 0x7fc00000, K = [fx, 0, cx; 0, fy, cy; 0, 0, 1].  For every pair k < f1-f0, slot
 * a = f0+k:
 *   1. Correspondences.  The cells, their order and validity rule of ofdis_global_motion_fullres (fb_check included);
 *      the m valid cells give pixel correspondences c = (px, py, xs, ys) float32 and normalized ones x = ((float)px -
 *      cx) / fx, y = ((float)py - cy) / fy, x' = (xs - cx) / fx, y' = (ys - cy) / fy (float32).  m < 8: status 1.
 *   2. Hypotheses h = 0 .. hypotheses-1.  Draws d = 0..7 by ofdis_global_motion_fullres's SplitMix64 rule give the
 *      rows [x'x, x'y, x', y'x, y'y, y', x, y, 1] (float64 products of the float32 values) of an 8 x 9 system A e = 0.
 *      Its null vector by full pivoting: for j = 0..7 the pivot is the first entry, rows i >= j outer and columns
 *      c >= j inner, of the largest |a_ic| (NaN is never largest); a pivot that is not > 0 fails; rows j and i are
 *      swapped (columns >= j), then columns j and c in every row together with the column permutation; for each
 *      i > j: f = a_ij / a_jj, a_ic = a_ic - f * a_jc for c > j.  Then y_8 = 1 and for i = 7..0: y_i = -a_i8,
 *      y_i = y_i - a_ic * y_c for c = i+1..7, y_i = y_i / a_ii; e is y un-permuted, divided entry by entry by
 *      L = sqrt(((e0*e0 + e1*e1) + ...) + e8*e8) summed in order from +0.0.  A failed pivot or a non-finite entry of
 *      e makes the hypothesis unsolvable (repeated or degenerate draws).  E = e row-major.
 *   3. Scoring.  F = K^-T E K^-1 in float64 with ifx = 1.0/fx, ify = 1.0/fy, ux = -(cx*ifx), uy = -(cy*ify):
 *      G_i0 = E_i0*ifx, G_i1 = E_i1*ify, G_i2 = ((E_i0*ux) + (E_i1*uy)) + E_i2; F_0j = ifx*G_0j, F_1j = ify*G_1j,
 *      F_2j = ((ux*G_0j) + (uy*G_1j)) + G_2j, rounded to float32 g.  With a = g (px, py, 1) (a_r = (g_r0*px + g_r1*py)
 *      + g_r2), b0 = (g0*xs + g3*ys) + g6, b1 = (g1*xs + g4*ys) + g7, e = (xs*a0 + ys*a1) + a2 and den = (a0*a0 +
 *      a1*a1) + (b0*b0 + b1*b1), a correspondence is an inlier iff e*e <= (threshold*threshold) * den (float32): the
 *      Sampson distance in pixels <= threshold, without a division.  The raw E is scored.  The best solvable
 *      hypothesis has the most inliers, the lowest h on a tie.  No solvable hypothesis: status 2.
 *   4. Refits.  The best E: S = E^T E (S_ij = ((E_0i*E_0j) + (E_1i*E_1j)) + (E_2i*E_2j)), V = I, then 8 sweeps of
 *      the pairs (0,1), (0,2), (1,2) of the cyclic Jacobi method: where S_pq != 0, th = (S_qq - S_pp) / (2.0*S_pq),
 *      t = 1.0 / (|th| + sqrt(th*th + 1.0)) negated when th < 0, c = 1.0 / sqrt(t*t + 1.0), s = t*c; the columns p, q
 *      of S, then its rows p, q, then the columns p, q of V become (c*a - s*b, s*a + c*b) of the old (a, b).  v1, v2
 *      are the columns of V of the largest diagonal entry of S and the larger of the other two (first on ties);
 *      unit(a) = a / sqrt((a0*a0 + a1*a1) + a2*a2), x the cross product (a1*b2 - a2*b1, a2*b0 - a0*b2, a0*b1 - a1*b0):
 *      v1 = unit(v1), v3 = unit(v1 x v2), v2 = v3 x v1, u1 = unit(E v1), u3 = unit(u1 x E v2), u2 = u3 x u1 (E v with
 *      rows ((E_i0*v0) + (E_i1*v1)) + (E_i2*v2)).  R1_ij = ((u2_i*v1_j) - (u1_i*v2_j)) + (u3_i*v3_j), R2_ij =
 *      ((u1_i*v2_j) - (u2_i*v1_j)) + (u3_i*v3_j); the candidates q = 0..3 are (R1, u3), (R1, -u3), (R2, u3),
 *      (R2, -u3).  Over the inliers of the best hypothesis (step 3), with r0 = (x, y, 1), r1 = (x', y', 1) in float64
 *      and Y = R r0 (Y_i = ((R_i0*x) + (R_i1*y)) + R_i2), c1 = r1 x Y, c2 = r1 x t, lambda = -(c1.c2) / (c1.c1)
 *      (a.b = (a0*b0 + a1*b1) + a2*b2): the candidate with the most inliers of lambda > 0 and lambda*Y_2 + t_2 > 0
 *      (in front of both cameras), the lowest q on a tie, is the model.  Then rounds r = 0, 1, ...: E = [t]x R
 *      (E_0j = (-(t2*R_1j)) + (t1*R_2j), E_1j = (t2*R_0j) - (t0*R_2j), E_2j = (-(t1*R_0j)) + (t0*R_1j)), g its F as in
 *      step 3, the tangent basis b1 = unit(t x e_a) with e_a the unit axis of the first smallest |t_a|, b2 = t x b1.
 *      The inliers of g (step 3's test), each with Y = R r0, a = E r0 and b = E^T r1 (rows as above, b_j = ((E_0j*x')
 *      + (E_1j*y')) + E_2j), the residual res = ((x'*a0) + (y'*a1)) + a2, the Sampson weight w = 1.0 / sqrt(((s0*s0 +
 *      s1*s1) + s2*s2) + s3*s3) with s = (a0*ifx, a1*ify, b0*ifx, b1*ify), rr = w*res and the Jacobian row of
 *      (omega, delta) J = (w*(2.0*g_0), w*(2.0*g_1), w*(2.0*g_2), w*(b1.n), w*(b2.n)) with g = Y x (r1 x t), n = Y x r1,
 *      give N_pq = J_p*J_q (p <= q), the right side -(J_p*rr), the derotated flow length sqrt(dx*dx + dy*dy),
 *      dx = fx*(x' - Y_0/Y_2), dy = fy*(y' - Y_1/Y_2), and the same length with Y = Rw r0 of the twisted pair
 *      Rw_ij = sum over k = 0..2 from +0.0 of ((2.0*(t_i*t_k)) - (i == k ? 1.0 : 0.0)) * R_kj (the rotation by 180
 *      degrees about t composed with R, which explains the same E), summed as ofdis_global_motion_fullres's refits sum (chunks of
 *      32 from +0.0, then the pairwise tree).  When r = refine or fewer than 8 inliers: stop.  Else N is mirrored
 *      and solved by ofdis_global_motion_fullres's elimination; a failure stops and keeps the model; else R <- C R
 *      with ofdis_egomotion_fullres's Cayley rotation C of omega (R_ij = ((C_i0*R_0j) + (C_i1*R_1j)) + (C_i2*R_2j)),
 *      t_i <- (t_i + delta_0*b1_i) + delta_1*b2_i, t <- unit(t), next round.
 *   5. Parallax guard.  With Lr and Lw the last round's two length sums, parallax = (Lw < Lr ? Lw : Lr) /
 *      (double)its inlier count: the mean derotated flow in pixels under R or its twisted pair, whichever is
 *      smaller.  Without translation E is degenerate and the cheirality vote may pick the twisted candidate; one of
 *      the two rotations then explains the flow alone.  Unless parallax >= min_parallax (a NaN fails): status 3, the
 *      translation is unobservable (identical frames, or a pure rotation of a static scene; an object that moves on
 *      its own among the inliers adds its own parallax to the mean).
 *   6. pose = [n][12] float64 row-major [R | t], |t| = 1, camera-t coordinates to camera-t+1 coordinates (the
 *      convention of ofdis_egomotion_fullres).  Status != 0: twelve float64 qNaN 0x7ff8000000000000.
 *   7. Per pixel (X, Y), F = (u, v) and validity by step 1's rule at the pixel, c = ((float)X, (float)Y, X + u, Y + v):
 *      mask 2 where the pixel is not valid or the status is not 0, else 0 where step 3's test passes with the final
 *      model's g, else 1 (moves on its own, or a bad flow).  sampson = sqrtf((e*e) / den) of that test where mask
 *      != 2, else qNaN.  depth: with the pose rounded to float32 (R, t), x, y, x', y' of step 1 and float32 Y = R r0
 *      (Y_i = (R_i0*x + R_i1*y) + R_i2), c1 = (y'*Y2 - Y1, Y0 - x'*Y2, x'*Y1 - y'*Y0), c2 = (y'*t2 - t1,
 *      t0 - x'*t2, x'*t1 - y'*t0), lambda = -((c1_0*c2_0 + c1_1*c2_1) + c1_2*c2_2) / ((c1_0*c1_0 + c1_1*c1_1) +
 *      c1_2*c1_2): lambda where mask != 2, lambda > 0 and lambda*Y2 + t2 > 0, else qNaN -- the depth at t in units of
 *      |t|.  Every NaN written is qNaN.
 * stats per pair: status (0 fitted, 1 fewer than 8 correspondences, 2 no solvable hypothesis, 3 too little parallax),
 * n_corr = m, best_hypothesis (-1 for status 1 and 2), ransac_inliers (its count), refits (rounds that replaced the
 * model), n_inliers (the final model's count).  pose and stats are host memory; mask [n][H][W] bytes, sampson and depth
 * [n][H][W] float32 are optional (NULL skips them) and in memkind; host outputs go through the full-resolution scratch.
 * OFDIS_ERR_ARG: a stereo context, slots outside the context (b0 only with fb_check), a NULL p or one out of range
 * (fx, fy finite and > 0, cx, cy finite, step >= 1, fb_check 0|1, alpha and beta finite and >= 0, hypotheses
 * 1..65536, threshold finite and > 0, refine 0..16, min_parallax finite and >= 0), NULL pose or stats, a device
 * sampson or depth not 4-byte aligned, or more than 2^24 cells per pair; frame sizes as ofdis_get_flow_fullres checks
 * them.  The workspace -- per cell and pair 22.5 bytes (the correspondence, its flag, the refit's 22 chunk sums per
 * 32 cells), per hypothesis and pair 120 (its float64 E and the float32 F record) and 176 per pair -- is allocated on
 * the first call, grows, never shrinks and is freed by ofdis_destroy.  Enqueued on the context's stream as 5 kernels,
 * plus one when a per-pixel output is asked for, whatever the number of pairs; the call synchronises the stream once,
 * at the end, for pose and stats.  Not part of ofdis_run's graph; the flows are not changed. */
typedef struct ofdis_relpose_params {
  float fx, fy, cx, cy;      /* pinhole intrinsics of both frames; finite, fx, fy > 0 */
  int step;                  /* correspondence grid step s >= 1, as ofdis_global_motion_fullres */
  int fb_check;              /* 0 | 1: only correspondences whose consistency mask against slot b0+k is 0 */
  float alpha, beta;         /* the rule of ofdis_consistency_fullres; finite, >= 0 */
  int hypotheses;            /* 1 .. 65536 */
  float threshold;           /* inlier Sampson distance in pixels; finite, > 0 */
  int refine;                /* 0 .. 16 Gauss-Newton rounds on the inliers */
  float min_parallax;        /* pixels, finite, >= 0: below it status 3 */
  unsigned long long seed;
} ofdis_relpose_params;
int ofdis_relpose_fullres(ofdis_ctx* ctx, int f0, int f1, int b0, const ofdis_relpose_params* p, double* pose,
                          ofdis_motion_stats* stats, unsigned char* mask, float* sampson, float* depth,
                          int width_org, int height_org, int memkind);

/* Volumetric fusion (extension): a truncated signed distance function (TSDF; Curless and Levoy, SIGGRAPH 1996;
 * KinectFusion, Newcombe et al., ISMAR 2011) integrated from a clip's disparity maps and camera poses, its zero
 * crossings as surface points and its depth rendered by ray casting.  The context owns one volume: T, W and, with
 * colour, three bytes per voxel.  It persists across calls and across ofdis_run and the other extensions;
 * ofdis_fuse_begin resets it and ofdis_destroy frees it.  It reads no flow: any context (flow or stereo) may own one.
 * Float32 without contraction, with IEEE division and square root; the pose algebra on the host in float64;
 * preprocess.fuse_integrate, fuse_extract and fuse_render restate it bit for bit.  qNaN = 0x7fc00000, known(d) =
 * 0 <= d <= 1e9 (NaN fails, -0 passes), fb = fx * baseline rounded once, mu = trunc.
 *   Volume.  Voxel (i, j, k), linear index (k*ny + j)*nx + i, sits at X = ox + (float)i * voxel, Y = oy + (float)j *
 *   voxel, Z = oz + (float)k * voxel in the world: frame 0's camera, x right, y down, z forward.  Initially T = +0,
 *   W = 0 and colour (0, 0, 0).
 *   Push.  Frame k's pose P ([3][4] float64 row-major [R | t], camera-to-world, the convention of
 *   preprocess.chain_poses and KITTI) gives the world-to-camera g ([3][4] float32): g_r0..g_r2 = R_0r, R_1r, R_2r and
 *   g_r3 = -(((R_0r*t_0) + (R_1r*t_1)) + (R_2r*t_2)) in float64, each rounded to float32.  Per voxel, for k = 0 .. n-1
 *   in order: Xc = ((g00*X + g01*Y) + g02*Z) + g03 (Yc with row 1, Zc with row 2); skip unless Zc > 0.
 *   u = (fx*Xc)/Zc + cx, v = (fy*Yc)/Zc + cy; skip unless u + 0.5f and v + 0.5f lie in [0, W) and [0, H) (NaN fails);
 *   px = (int)floorf(u + 0.5f), py likewise.  d = D_k(px, py); skip unless known(d) and s = d + doffs > 0.  z = fb / s;
 *   skip when z > max_depth.  sdf = z - Zc; skip when sdf < -mu.  f = fminf(1.0f, sdf / mu); W' = W + 1.0f;
 *   T = (T*W + f) / W'; with colour, per channel c = (unsigned char)floorf(((float)c*W + (float)obs) / W' + 0.5f)
 *   with the W before the update and obs frame k's byte at (px, py) (gray replicated); then W = fminf(W', max_weight).
 *   A push of n frames gives exactly the volume of n pushes of one frame each.
 *   Extract.  For voxel a and axis e (x, y, z), in ascending voxel index and then axis order, with b = a + e inside
 *   the volume: a crossing when W_a >= min_weight, W_b >= min_weight, fabsf(T_a) < 1, fabsf(T_b) < 1 and
 *   (T_a > 0) != (T_b > 0).  Its point is a's (X, Y, Z) with the e component plus t * voxel, t = T_a / (T_a - T_b);
 *   its normal the gradient G = (T(i+1, j, k) - T(i-1, j, k), T(i, j+1, k) - T(i, j-1, k), T(i, j, k+1) - T(i, j, k-1))
 *   at a with indices clamped to the volume, divided per component by L = sqrtf((Gx*Gx + Gy*Gy) + Gz*Gz) when L > 0,
 *   else (qNaN, qNaN, qNaN); its colour a's when t < 0.5f, else b's ((0, 0, 0) without colour); pad 0.
 *   Render.  For pose k (rounded to float32 row-major, p) and pixel (x, y): the ray r = (((float)x - cx)/fx,
 *   ((float)y - cy)/fy, 1); samples s = 0 .. 65536 with Z_s = z_near + (float)s*step while Z_s <= z_far; the sample's
 *   world point Pw_r = ((p_r0*(r0*Z_s) + p_r1*(r1*Z_s)) + p_r2*Z_s) + p_r3 and voxel coordinates q = (Pw - origin) /
 *   voxel per component.  fl = floorf(q) must satisfy 0 <= fl <= (float)(n - 2) on each axis (n = nx, ny, nz), i0 =
 *   (int)fl, fr = q - fl; the sample is known when all 8 corners have W >= min_weight, and its T is trilinear, x first,
 *   then y, then z, each step a*(1.0f - fr) + b*fr.  At the first s with samples s and s+1 both known and T_s > 0 >=
 *   T_s+1: depth = Z_s + step * (T_s / (T_s - T_s+1)); none: qNaN.  The step is fixed: no adaptive skipping. */
typedef struct ofdis_fuse_params {
  int nx, ny, nz;       /* each >= 1, nx * ny * nz <= 2^30 */
  float origin[3];      /* world position of voxel (0, 0, 0), metres; finite */
  float voxel;          /* voxel size, metres; finite, > 0 */
  float trunc;          /* truncation distance mu, metres; finite, > 0 */
  float max_weight;     /* finite, >= 1 */
  int color;            /* 0 | 1: keep three colour bytes per voxel */
} ofdis_fuse_params;
typedef struct ofdis_fuse_point {
  float x, y, z;        /* the zero crossing, world metres */
  float nx, ny, nz;     /* unit normal (towards T > 0, free space), qNaN where the gradient is 0 */
  unsigned char r, g, b, pad;
} ofdis_fuse_point;     /* 28 bytes */
/* Resets the volume: every voxel to T = +0, W = 0, colour 0.  The volume -- 8 bytes per voxel, 11 with colour -- is
 * allocated here, grows, never shrinks and is freed by ofdis_destroy.  A NULL or out-of-range p is OFDIS_ERR_ARG and
 * leaves a live volume as it was.  One memset per array, no kernel. */
int ofdis_fuse_begin(ofdis_ctx* ctx, const ofdis_fuse_params* p);
/* Integrates frames k = 0 .. n-1 in order: disp + k*disp_stride ([H][W] positive disparities, NaN unknown, the maps of
 * ofdis_scene_flow_fullres), poses [n][12] float64 on the host, and with colour frames + k*frame_stride ([H][W][noc]
 * bytes, noc the context's channels; NULL without colour).  W = width_org, H = height_org; max_depth > 0 (+inf
 * allowed).  disp and frames in memkind: host inputs go through the context's staging buffer.  One kernel plus the copy
 * of the n float32 world-to-camera poses, whatever n.  OFDIS_ERR_ARG, with the volume unchanged: no live volume, NULL
 * disp or poses, a NULL frames with colour, a NULL or bad cam (as ofdis_scene_flow_fullres checks it), max_depth NaN or
 * not > 0, disp_stride < W*H, frame_stride below one frame (with colour), n outside 1 .. max_frames + 1, a non-finite
 * pose entry, or a device disp that is not 4-byte aligned; frame sizes as ofdis_get_flow_fullres checks them. */
int ofdis_fuse_push(ofdis_ctx* ctx, int n, const float* disp, size_t disp_stride, const double* poses,
                    const ofdis_stereo_camera* cam, float max_depth, const unsigned char* frames, size_t frame_stride,
                    int width_org, int height_org, int memkind);
/* Confidence-weighted integration: ofdis_fuse_push with weight + k*weight_stride ([H][W] float32 in memkind, for
 * example ofdis_confidence_fullres's conf) for frame k.  An observation at pixel (px, py) with c = weight there is
 * skipped unless 0 < c <= FLT_MAX (NaN, +-0, negative values and +-inf skip); otherwise, in float32, W' = W + c, T = (T*W + f*c) / W',
 * each colour byte floor(((float)col*W + (float)obs*c) / W' + 0.5f) and W = fminf(W', max_weight).  With c = 1.0f
 * everywhere this is ofdis_fuse_push bit for bit (f*1 = f).  W is then a sum of confidences, and min_weight in
 * ofdis_fuse_extract, ofdis_fuse_render, ofdis_fuse_mesh and ofdis_fuse_track compares against that sum.  Host weights go
 * through the staging buffer after the maps and frames.  One kernel, as the push; OFDIS_ERR_ARG as the push, and for a
 * NULL weight, weight_stride < W*H or a device weight that is not 4-byte aligned. */
int ofdis_fuse_push_weighted(ofdis_ctx* ctx, int n, const float* disp, size_t disp_stride, const double* poses,
                             const ofdis_stereo_camera* cam, float max_depth, const unsigned char* frames,
                             size_t frame_stride, const float* weight, size_t weight_stride, int width_org,
                             int height_org, int memkind);
/* The volume's zero crossings in order: *count (host) gets the total, pts ([capacity] in memkind) the first
 * min(capacity, total); capacity 0 counts only (pts may then be NULL).  Three kernels (count, scan, write), then one
 * synchronise.  Host output goes through the context's full-resolution scratch.  OFDIS_ERR_ARG: no live volume, NULL
 * count, capacity < 0, NULL pts with capacity > 0, min_weight NaN, or a device pts that is not 4-byte aligned. */
int ofdis_fuse_extract(ofdis_ctx* ctx, float min_weight, ofdis_fuse_point* pts, long capacity, long* count,
                       int memkind);
/* Ray-cast depth [n][H][W] float32 (memkind) for n poses ([n][12] float64 camera-to-world, host).  One kernel;
 * host output goes through the full-resolution scratch and synchronises the stream.  OFDIS_ERR_ARG: no live volume,
 * NULL poses or depth, a NULL or bad cam, z_near or step not finite and > 0, z_far not finite or below z_near,
 * (z_far - z_near) / step > 65536 (float32), min_weight NaN, n outside 1 .. max_frames + 1, a non-finite pose entry, or
 * a device depth that is not 4-byte aligned; frame sizes as ofdis_get_flow_fullres checks them. */
int ofdis_fuse_render(ofdis_ctx* ctx, int n, const double* poses, const ofdis_stereo_camera* cam, float z_near,
                      float z_far, float step, float min_weight, float* depth, int width_org, int height_org,
                      int memkind);
/* Copies the volume out in memkind: T and W [nz][ny][nx] float32 and color [nz][ny][nx][3] bytes, each may be NULL
 * (color must be NULL for a volume without colour).  Synchronises the stream.  OFDIS_ERR_ARG: no live volume, a
 * colour output without colour, or a device T or W that is not 4-byte aligned. */
int ofdis_fuse_get_volume(ofdis_ctx* ctx, float* T, float* W, unsigned char* color, int memkind);
/* The inverse of ofdis_fuse_get_volume: T, W and color (as it lays them out, in memkind) into the volume; a NULL
 * array leaves that array as it was.  Any float bits are accepted: the comparisons of the contract then apply as
 * written (NaN fails every test).  One copy per array, no kernel; synchronises the stream.  OFDIS_ERR_ARG, with the
 * volume unchanged: no live volume, a colour input for a volume without colour, or a device T or W that is not 4-byte
 * aligned. */
int ofdis_fuse_set_volume(ofdis_ctx* ctx, const float* T, const float* W, const unsigned char* color, int memkind);
/* Marching cubes (extension): the volume's surface as a closed, oriented triangle mesh over the crossings of
 * ofdis_fuse_extract.  preprocess.fuse_mesh restates it bit for bit and preprocess.fuse_mc_table generates its table.
 *   Vertices.  Exactly ofdis_fuse_extract(min_weight)'s points, in its order and bit for bit: the crossing of voxel a
 *   along axis e has vertex index = its position in that list (uint32: a volume has at most 3 * 2^30 crossings).
 *   Cubes.  Cube (i, j, k) exists for i < nx-1, j < ny-1, k < nz-1.  Its corner q = 0 .. 7 is voxel (i + (q&1),
 *   j + ((q>>1)&1), k + (q>>2)).  A cube is meshed when all 8 corners satisfy W >= min_weight && fabsf(T) < 1, the
 *   extraction's per-voxel test; its case is the sum over q of (T_q > 0) << q (-0 and NaN count as solid, but NaN
 *   fails the test).  Every sign-changing edge of a meshed cube therefore joins two voxels that pass the test: it is
 *   an extraction crossing, and every face index refers to an existing vertex.  Edge n = 4*e + r (e the axis) runs
 *   from corner q -- r with a 0 bit inserted at bit e -- to q | (1 << e): edges 0..3 join corners 0-1, 2-3, 4-5, 6-7,
 *   edges 4..7 join 0-2, 1-3, 4-6, 5-7, edges 8..11 join 0-4, 1-5, 2-6, 3-7.  Its vertex is the crossing of corner q's
 *   voxel along e.
 *   Table (preprocess.fuse_mc_table; 820 triangles over the 256 cases, at most 5 per case), from three rules:
 *     face rule: on each cube face the crossing edges are joined by segments; on an ambiguous face (diagonal corners
 *     of equal sign) the segments cut off the two T > 0 corners, so that the solid side stays connected across the
 *     face.  The rule depends only on the face's four signs, so two cubes sharing a face make the same segments and
 *     the mesh has no cracks (the classic 15-case table does not have this property);
 *     loops: the segments link into closed loops (every crossing edge lies on exactly two faces, so the loops are
 *     unique), oriented so that each triangle's normal (p1 - p0) x (p2 - p0) points towards T > 0 -- free space, the
 *     direction of the extraction's normals.  A cube's loops go in the order of their lowest edge numbers, and each
 *     loop v_0 .. v_L-1 starts at its lowest edge;
 *     triangulation: each loop takes the first triangulation, in this enumeration, in which no diagonal joins two
 *     edges on the same cube face.  The triangulations of v_lo .. v_hi: for the apex k = lo+1 .. hi-1 in ascending
 *     order, the triangle (v_lo, v_k, v_hi), then each triangulation of v_lo .. v_k and, within it, of v_k .. v_hi;
 *     that is also the order of the triangles.
 *   Faces.  Meshed cubes in ascending voxel index of corner 0, each cube's triangles in table order, as [3] uint32
 *   vertex indices.
 * *pt_count and *face_count (host) get the totals; pts ([pt_capacity] records) and faces ([face_capacity][3]) in
 * memkind the first min(capacity, total) entries; capacity 0 counts only (the array may then be NULL).  Faces keep
 * their global indices when pt_capacity is below the vertex total.  Six kernels whatever the volume (the extraction's
 * count and scan, a cube count and the same scan, the extraction's write with each crossing voxel's first vertex
 * index, a face write), one synchronise, and with host output one readback of the two totals before the writes; host
 * output goes through the full-resolution scratch.  The workspace (4 bytes per voxel plus 8 per scan block of 1024
 * voxels, and 8 for the total) is allocated at the first call, grows, never shrinks and is freed by ofdis_destroy;
 * OFDIS_ERR_NOMEM when that fails, with the volume intact.  OFDIS_ERR_ARG, with the volume and the outputs untouched:
 * no live volume, NULL pt_count or face_count, a capacity < 0, a NULL array with capacity > 0, min_weight NaN, or a
 * device pts or faces that is not 4-byte aligned. */
int ofdis_fuse_mesh(ofdis_ctx* ctx, float min_weight, ofdis_fuse_point* pts, long pt_capacity, long* pt_count,
                    unsigned int* faces, long face_capacity, long* face_count, int memkind);
/* Camera tracking against the volume (extension): each frame aligned to the TSDF before it is pushed, the SDF
 * formulation of Bylow et al. (RSS 2013): the frame's points, moved into the volume by the camera-to-world pose, should
 * land on T = 0.  preprocess.fuse_track restates it bit for bit.  float32 where marked, float64 in the sums and the
 * pose algebra, everything without contraction and with IEEE division and square root; the terms of the fusion header
 * above (known(d), fb, the volume's layout).  W = width_org, H = height_org.  For k = 0 .. n-1:
 *   1. Prediction (float64).  T(-1) = prev ([12], camera-to-world); P = T(k-1) and M = motions[k] (camera k-1 to
 *      camera k, as ofdis_egomotion_fullres returns it): inv(M) = [Ri | ti] with Ri_rc = M_cr and ti_r =
 *      -(((M_0r*M_03) + (M_1r*M_13)) + (M_2r*M_23)), and T_pred_rc = ((P_r0*Ri_0c) + (P_r1*Ri_1c)) + (P_r2*Ri_2c) for
 *      c < 3, T_pred_r3 = (((P_r0*ti_0) + (P_r1*ti_1)) + (P_r2*ti_2)) + P_r3.  motions NULL: T_pred = T(k-1) as it is.
 *      This can differ in the last bits from preprocess.chain_poses, which inverts with np.linalg.inv.  T(k-1) is frame
 *      k-1's final pose from step 4, so the chain runs through the tracked poses.
 *   2. Evaluation of a pose M (float64 [12]) of frame k: g = M rounded to float32.  The cells of
 *      ofdis_global_motion_fullres at step s, in cell order, cell (i, j) at its pixel (px, py): d = D_k(px, py),
 *      sd = d + doffs, Z = fb / sd, X = (((float)px - cx) * Z) / fx, Y = (((float)py - cy) * Z) / fy (ofdis_scene_flow's
 *      xyz), Pw_r = ((g_r0*X + g_r1*Y) + g_r2*Z) + g_r3 (the push's order), q_e = (Pw_e - origin_e) / voxel (the
 *      render's).  The cell is valid when known(d), sd > 0, Z <= max_depth, fl = floorf(q) satisfies 0 <= fl <= (float)
 *      (n - 2) on each axis (NaN fails), and all 8 corners of the cube at i0 = (int)fl have W >= min_weight and
 *      fabsf(T) < 1.  With fr = q - fl, gx = 1.0f - fr_0 (gy, gz likewise) and the corners c0..c7 in the render's
 *      order: x00 = c0*gx + c1*fr_0, x10 = c2*gx + c3*fr_0, x01 = c4*gx + c5*fr_0, x11 = c6*gx + c7*fr_0,
 *      y0 = x00*gy + x10*fr_1, y1 = x01*gy + x11*fr_1, the residual r = y0*gz + y1*fr_2 (the render's T); the gradient
 *      G_0 = (((c1 - c0)*gy + (c3 - c2)*fr_1)*gz + ((c5 - c4)*gy + (c7 - c6)*fr_1)*fr_2) / voxel,
 *      G_1 = ((x10 - x00)*gz + (x11 - x01)*fr_2) / voxel, G_2 = (y1 - y0) / voxel (float32, the exact partial
 *      derivatives of the trilinear T in metres).  Huber weight wt = 1.0f when fabsf(r) <= huber, else
 *      huber / fabsf(r).  In float64 of those values, a = G and w = 2 Pw per component: the Jacobian row of the left
 *      update J = ((a1*-w2) + (a2*w1), (a0*w2) + (a2*-w0), (a0*-w1) + (a1*w0), a0, a1, a2) (ofdis_egomotion_fullres's
 *      row), v = wt * J per component, N_ij = v_i * J_j for i <= j (21, row-major), b_i = -(v_i * r) (6) and
 *      e = (wt * r) * r (1).  These 28 sums and the count of valid cells run over the cells as the refits of
 *      ofdis_global_motion_fullres sum: chunks of 32 consecutive cells from +0.0 in cell order (an invalid cell or one
 *      past the last adds nothing), then the pairwise tree over the chunk sums padded with +0.0 to a power of two.
 *   3. Rounds r = 0, 1, ...: M = T_pred at r = 0.  Evaluate M (step 2): n_corr = the count, cost = e, and at r = 0
 *      cost0 = e.  Stop when n_corr < min_corr (status 1 when r = 0), when r = rounds, or when N with damping added to
 *      each diagonal entry (N_ii + damping) fails the elimination of ofdis_global_motion_fullres.  Otherwise x = its
 *      solution (omega, tau); stop when max_i fabs(x_i) <= eps (the update is not applied), else M = the Cayley update
 *      of ofdis_egomotion_fullres's step 4 applied to M (R <- C R, t <- C t + tau), rounds = r + 1, next r.  So a frame
 *      takes at most rounds + 1 evaluations and the stats describe the last evaluated pose.
 *   4. Guard.  Unless status 1, with M_f the last evaluated pose and M_p = T_pred: dt = t_f - t_p, the shift
 *      sqrt((dt0*dt0 + dt1*dt1) + dt2*dt2) <= max_shift and, with s_i = ((Rf_i0*Rp_i0) + (Rf_i1*Rp_i1)) +
 *      (Rf_i2*Rp_i2), (((s0 + s1) + s2) - 1.0) / 2.0 >= min_cos (the cosine of the rotation between them): status 0
 *      and T(k) = M_f; else status 2 (NaN fails).  Status 1 or 2: T(k) = T_pred.  poses[k] = T(k).
 *   5. Integration (integrate 1): frame k is pushed at T(k) before frame k+1 is predicted, by exactly ofdis_fuse_push's
 *      rule (its world-to-camera g formed in float64 and rounded once, max_depth, colour from frames + k*frame_stride
 *      when the volume keeps it).  So one call of n frames equals n calls of one frame with prev = the last pose
 *      returned, and equals, frame by frame, a call with integrate 0 followed by ofdis_fuse_push at the returned pose.
 * disp + k*disp_stride ([H][W], the maps of ofdis_fuse_push) and frames are in memkind; host inputs go through the
 * staging buffer.  prev ([12]), motions ([n][12] or NULL), poses ([n][12] float64) and stats ([n]) are host memory.
 * OFDIS_ERR_ARG, with the volume and the outputs untouched: no live volume, n outside 1 .. max_frames + 1, NULL disp,
 * prev, p, poses or stats, a NULL or bad cam (as ofdis_fuse_push checks it), p out of range (see the fields), a NULL
 * frames when integrating into a volume with colour, a non-finite entry of prev or motions, disp_stride < W*H,
 * frame_stride below one frame (when frames are read), or a device disp or frames that is not aligned to its element;
 * frame sizes as ofdis_get_flow_fullres checks them.  The workspace -- 28 doubles of chunk sums per 32 cells, the pose
 * chain (the motions, poses and stats of max_frames + 1 frames and the current frame's poses) and one arrival
 * counter -- is allocated at the first call, grows, never shrinks and is freed by ofdis_destroy; OFDIS_ERR_NOMEM when
 * that fails, with the volume intact.  Enqueued on the context's stream as rounds + 1 evaluation kernels per frame
 * (a frame that stops early makes its later ones return at once) plus, with integrate, one integration kernel per
 * frame: n * (rounds + 1 + integrate) kernels whatever the data.  The call synchronises the stream once, at the end. */
typedef struct ofdis_fuse_track_params {
  int step;             /* >= 1: the correspondence cells of ofdis_global_motion_fullres at this step */
  int rounds;           /* 0 .. 32 Gauss-Newton rounds per frame */
  float min_weight;     /* every one of the 8 corners needs W >= min_weight; not NaN */
  float max_depth;      /* > 0, +inf allowed: used by the alignment and, when integrating, by the push */
  float huber;          /* finite, > 0: Huber threshold on the residual r (units of T) */
  double damping;       /* finite, >= 0: added to the normal matrix's diagonal */
  int min_corr;         /* >= 6 */
  double max_shift;     /* finite, > 0, metres: the guard on translation */
  double min_cos;       /* [-1, 1]: the guard on rotation, (trace(R_f R_p^T) - 1) / 2 >= min_cos */
  double eps;           /* finite, >= 0: an update with max_i |x_i| <= eps ends the frame's rounds */
  int integrate;        /* 0 | 1: push each frame at its final pose before aligning the next */
} ofdis_fuse_track_params;
typedef struct ofdis_fuse_track_stats {
  int status;           /* 0 aligned; 1 fewer than min_corr at the prediction; 2 rejected by the guard */
  int n_corr;           /* valid cells at the last evaluated pose */
  int rounds;           /* updates applied */
  double cost0, cost;   /* sum of wt*r*r at the prediction and at the last evaluated pose */
} ofdis_fuse_track_stats;  /* 32 bytes */
int ofdis_fuse_track(ofdis_ctx* ctx, int n, const float* disp, size_t disp_stride, const double* motions,
                     const double* prev, const ofdis_stereo_camera* cam, const ofdis_fuse_track_params* p,
                     const unsigned char* frames, size_t frame_stride, double* poses, ofdis_fuse_track_stats* stats,
                     int width_org, int height_org, int memkind);
/* Confidence-weighted tracking: ofdis_fuse_track with weight + k*weight_stride ([H][W] float32 in memkind) for frame
 * k.  A cell at pixel (px, py) is valid only when, in addition, 0 < c <= FLT_MAX for c = weight there (NaN and +-inf
 * fail); its weight in N,
 * b and the cost becomes (double)(wt * c), the float32 product of the Huber weight and c.  With integrate, the push is
 * ofdis_fuse_push_weighted's.  With c = 1.0f everywhere this is ofdis_fuse_track bit for bit: poses, stats and volume.
 * Host weights go through the staging buffer after the maps and frames.  The same launches as ofdis_fuse_track;
 * OFDIS_ERR_ARG as ofdis_fuse_track, and for a NULL weight, weight_stride < W*H or a device weight that is not 4-byte
 * aligned. */
int ofdis_fuse_track_weighted(ofdis_ctx* ctx, int n, const float* disp, size_t disp_stride, const double* motions,
                              const double* prev, const ofdis_stereo_camera* cam, const ofdis_fuse_track_params* p,
                              const unsigned char* frames, size_t frame_stride, const float* weight,
                              size_t weight_stride, double* poses, ofdis_fuse_track_stats* stats, int width_org,
                              int height_org, int memkind);

/* Dense point trajectories (extension): the tracker of Sundaram, Brox and Keutzer ("Dense point trajectories by
 * GPU-accelerated large displacement optical flow", ECCV 2010) through consecutive pairs of bidirectional flows.
 * The context owns one tracker: the list of live tracks (sorted by id), the next id and the counters.  It persists
 * across calls and across ofdis_run; ofdis_track_begin resets it and ofdis_destroy frees it.  Everything is float32
 * without contraction, with IEEE division and square root; preprocess.track_points restates it.  W = width_org,
 * H = height_org, s = spacing.
 *   Seeding a frame (ofdis_track_begin: its frame; ofdis_track_advance: every target frame).  The cells (i, j) are
 *   ceil(W/s) x ceil(H/s), in row-major order (j outer); cell (i, j) has the seed pixel cx = min(i*s + s/2, W-1),
 *   cy = min(j*s + s/2, H-1).  A cell is occupied when a live track has ((int)x / s, (int)y / s) == (i, j) after the
 *   frame's advance.  Brightness g: the byte for gray, ((float)c0 + (float)c1 + (float)c2) / 3.0f for 3 channels in
 *   memory order.  Ix = (g(min(x+1, W-1), y) - g(max(x-1, 0), y)) * 0.5f, Iy the same in y.  Over the 5 x 5 window
 *   around the seed pixel (coordinates clamped to the frame; dy outer, dx inner, both ascending; sums from +0.0f):
 *   a = sum Ix*Ix, b = sum Ix*Iy, c = sum Iy*Iy; d = a - c, lambda = (a + c)*0.5f - sqrtf(d*d*0.25f + b*b).  An
 *   unoccupied cell with lambda >= min_eig is a candidate.  Candidates take the ids next_id, next_id + 1, ... in cell
 *   order and are appended after the surviving tracks at (cx, cy), as long as there are fewer than `capacity` live
 *   tracks and next_id stays at most 2^31-1 (ids below 2^31-1); the lowest cells are kept, the others are counted in
 *   `dropped`.
 *   Advancing a track at (x, y) through pair k.  F is slot f0+k's full-resolution flow and B slot b0+k's, both
 *   exactly what ofdis_get_flow_fullres returns, computed from the level flows without a full-resolution copy;
 *   stereo (nop 1) uses v = 0.  bil(F, x, y) is the bilinear rule of ofdis_consistency_fullres (corners floor and
 *   floor + 1 clamped to the frame, horizontal pass first).
 *     (u, v) = bil(F, x, y); (x', y') = (x + u, y + v); outside [0, W-1] x [0, H-1] (or NaN): ends as *leaves*.
 *     b = bil(B, x', y'); err = du*du + dv*dv with (du, dv) = (u + b0, v + b1); mag = (u*u + v*v) + (b0*b0 + b1*b1)
 *     (stereo dv = b1 = 0); ends as *inconsistent* unless err <= alpha*mag + beta.
 *     (xr, yr) = ((int)floorf(x + 0.5f), (int)floorf(y + 0.5f)); ux = (F(min(xr+1, W-1), yr) - F(max(xr-1, 0), yr))
 *     * 0.5f and uy = (F(xr, min(yr+1, H-1)) - F(xr, max(yr-1, 0))) * 0.5f of the u component, vx, vy the same of v;
 *     g2 = (ux*ux + uy*uy) + (vx*vx + vy*vy) (stereo ux*ux + uy*uy); ends as *boundary* if
 *     g2 > mb_alpha*(u*u + v*v) + mb_beta.
 *     Otherwise the track moves to (x', y') and keeps its id; survivors keep their order.
 *   Sundaram et al. use alpha 0.01, beta 0.5 (as ofdis_consistency_fullres) and mb_alpha 0.01, mb_beta 0.002. */
typedef struct ofdis_track_params {
  int capacity;             /* live tracks the tracker holds, 1 .. 1<<24 */
  int spacing;              /* seed grid step s in pixels, >= 1 */
  float alpha, beta;        /* forward-backward test, as ofdis_consistency_fullres; finite and >= 0 */
  float mb_alpha, mb_beta;  /* motion-boundary test; finite and >= 0 */
  float min_eig;            /* seed where the structure tensor's smaller eigenvalue >= min_eig; not NaN */
} ofdis_track_params;
typedef struct ofdis_track_point { int id; float x, y; } ofdis_track_point;  /* 12 bytes */
typedef struct ofdis_track_stats {
  long long seeded, ended_leaves, ended_inconsistent, ended_boundary, dropped;  /* since ofdis_track_begin */
  int alive, next_id;
} ofdis_track_stats;
/* Resets the tracker and seeds `frame` ([height_org][width_org][noc] bytes in memkind); its list goes to points
 * ([capacity] records in memkind) and its length to *count (host).  Allocates the workspace -- the state, two track
 * lists and the output records of max_frames pairs (12 bytes per track), the cell flags -- which grows with capacity
 * and the cell count, never shrinks, and is freed by ofdis_destroy.  A NULL params, frame, points or count, a
 * parameter out of range, or a device `points` that is not 4-byte aligned is OFDIS_ERR_ARG; frame sizes are checked
 * as in ofdis_get_flow_fullres. */
int ofdis_track_begin(ofdis_ctx* ctx, const ofdis_track_params* params, const unsigned char* frame,
                      ofdis_track_point* points, int* count, int width_org, int height_org, int memkind);
/* Pairs k = 0 .. f1-f0-1 in order: advance every live track through slot f0+k (F) and slot b0+k (B) of the last run
 * (the layout of ofdis_upload_sequence_bidir_u8 with b0 = f0 + n, or pairs followed by their swapped copies), then
 * seed target frame k at frames + k*frame_stride (a clip: frames + hwc with stride hwc; the pairs of
 * ofdis_upload_frames_u8: image2 at stride 2hwc).  The list after pair k goes to points + k*capacity and its length
 * to counts[k] (host).  frames and points are in memkind; host frames go through the staging buffer, host records
 * through the workspace.  The pairs are enqueued without a host round trip; the call synchronises the context's
 * stream once, at the end, for the counts.  Slots outside the context, NULL frames, points or counts, frame_stride
 * below one frame, a device `points` that is not 4-byte aligned, or a call before ofdis_track_begin or with another
 * frame size than its is OFDIS_ERR_ARG.  Not part of ofdis_run's graph; the flows are not changed. */
int ofdis_track_advance(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* frames, size_t frame_stride,
                        ofdis_track_point* points, int* counts, int width_org, int height_org, int memkind);
/* The tracker's counters since ofdis_track_begin (synchronises the context's stream); OFDIS_ERR_ARG before the
 * first ofdis_track_begin or with a NULL out. */
int ofdis_track_stats_get(const ofdis_ctx* ctx, ofdis_track_stats* out);

/* Trajectory descriptors (extension): the single-scale pipeline of Wang and Schmid's improved dense trajectories
 * ("Action recognition with improved trajectories", ICCV 2013) on the tracker above.  The tracks are the tracker's,
 * bit for bit (the raw flow F moves them); the descriptors describe the camera-compensated residual flow R.  The
 * context owns one descriptor stage on top of its tracker; ofdis_traj_begin starts both, ofdis_track_begin and
 * ofdis_track_advance end it.  Float32 without contraction, IEEE division and square root, every sum from +0.0f in
 * the order given; preprocess.traj_descriptors restates it bit for bit.  W = width_org, H = height_org.
 *   Segments.  A track seeded at frame b (counted from ofdis_traj_begin's frame, 0) emits one descriptor per complete
 *   segment [b + (j-1)L, b + jL], j = 1, 2, ...: L + 1 positions p_0..p_L, L steps, and the frame histograms of its L
 *   source frames.  The next segment starts at the last point of the previous one; a track that ends partway through
 *   a segment discards it.
 *   Residual flow of pair k.  models[k] (9 float64, ofdis_global_motion_fullres's model) goes through the
 *   stabiliser's validity rule (divided by m22, or the identity; ofdis_stab_push), then each entry is rounded to
 *   float32: m0..m8; models == NULL is the identity (R = F).  F = slot f0+k's full-resolution flow (exactly what
 *   ofdis_get_flow_fullres returns).  At pixel (X, Y): mx = (m0*X + m1*Y) + m2, my = (m3*X + m4*Y) + m5,
 *   wq = (m6*X + m7*Y) + m8, R = (u - (mx/wq - X), v - (my/wq - Y)).  R is unknown where |u| > 1e9, |v| > 1e9 or
 *   either is NaN (F unknown), where wq is not > 0, or where a component of R is not finite.
 *   Vector fields of source frame k (pair k's I0: ofdis_traj_begin's frame, then the previous pair's target frame).
 *   Central differences are clamped: dx(f)(X, Y) = (f(min(X+1, W-1), Y) - f(max(X-1, 0), Y)) * 0.5f, dy the same in y.
 *     HOG:  (dx(g), dy(g)) of the tracker's brightness g.
 *     HOF:  R; unknown where R is.
 *     MBHx: (dx(R_u), dy(R_u)); MBHy: (dx(R_v), dy(R_v)); unknown where R is unknown at one of the four neighbours.
 *   Orientation bins of a vector (a, b).  mag = sqrtf(a*a + b*b); an unknown vector or a non-finite mag gives no
 *   bin.  angle = atan2_f32(b, a) (the color wheel's polynomial, preprocess.atan2_f32); angle < 0: angle + 6.2831855f;
 *   fbin = angle * 1.2732395f (8 / 2pi); bin0 = floorf(fbin), 8 wraps to 0; bin1 = (bin0 + 1) % 8;
 *   mag1 = (fbin - floorf(fbin)) * mag, mag0 = mag - mag1.  HOF with mag <= min_flow: weight 1 into its zero bin 8
 *   instead (HOF has 9 bins, the others 8).
 *   Frame histogram of a track at its position (x, y) before pair k's advance.  (xr, yr) = ((int)floorf(x + 0.5f),
 *   (int)floorf(y + 0.5f)); the N x N patch at ox = min(max(xr - N/2, 0), W - N), oy the same with H; ns x ns cells of
 *   c = N/ns pixels.  In cell (cx, cy) a bin's sum runs over the cell's pixels q = py*c + px (row-major): q mod 32 = l
 *   gives lane l, which sums its pixels in increasing q (mag0 into bin0, mag1 into bin1, for HOG, HOF, MBHx, MBHy);
 *   the cell's sum is lane 0's + lane 1's + ... + lane 31's, and v = sum + eps.  Each descriptor's entries, in the
 *   order (cx, cy, bin), sum to s = v_0 + v_1 + ...; each becomes sqrtf(v / s) (RootSIFT).
 *   Temporal cells: step i of the segment (0 .. L-1) adds its frame histograms to cell i / (L/nt), in step order;
 *   the descriptor holds that sum / (float)(L/nt).
 *   Tests of a completed segment, in order, each counted in its counter: with n = (float)(L+1), mean_x = (x_0 + ...
 *   + x_L) / n, sd_x = sqrtf(((x_0 - mean_x)^2 + ... ) / n), the same in y; *static* if sd_x < min_var and sd_y <
 *   min_var; *erratic* if sd_x > max_var or sd_y > max_var; with steps s_i = |p_{i+1} - p_i|, length = s_0 + ... +
 *   s_{L-1} and smax their largest, *jump* if smax > max_dis and smax > 0.7f*length; with d_i = R at (xr, yr) of p_i
 *   (the step's source pixel), *camera* if any d_i is unknown or not finite in magnitude |d_i| = sqrtf(du*du + dv*dv),
 *   or max |d_i| <= min_disp (the track moves with the camera).  Otherwise the segment is emitted.
 *   Descriptor (dim = 2L + ns*ns*nt*33 floats; 426 with the defaults): the shape d_i / (|d_0| + ... + |d_{L-1}|) as
 *   (du_0, dv_0, du_1, ...), then HOG [nt][ns][ns][8], HOF [nt][ns][ns][9], MBHx and MBHy [nt][ns][ns][8], the
 *   temporal cell outermost, then the x cell, the y cell and the bin.
 *   Order and bound.  Segments are emitted pair by pair, within a pair in list order (id order).  Each takes L (track,
 *   pair) incidences: at most n*capacity fall in a call of n pairs and at most (L-1)*capacity come from before it, so a
 *   call emits at most capacity * ceil((n + L - 1) / L) segments (the caller's output size).
 *   Wang and Schmid use L 15, nt 3, N 32, ns 2, min_flow 0.4, eps 0.05, min_disp 1 (their camera test in pixels at
 *   full resolution), min_var sqrt(3), max_var 50 and max_dis 20. */
typedef struct ofdis_traj_params {
  int L;             /* steps per segment, 1 .. 64, a multiple of nt */
  int nt;            /* temporal cells, >= 1 */
  int N;             /* patch side, a multiple of ns, at most min(W, H) */
  int ns;            /* spatial cells per side, 1 .. 4 */
  float min_flow;    /* HOF's zero-bin magnitude; finite */
  float eps;         /* added to every bin sum; finite and > 0 */
  float min_disp;    /* the camera test; finite and >= 0 */
  float min_var, max_var, max_dis;  /* the static, erratic and jump tests; finite */
} ofdis_traj_params;
typedef struct ofdis_traj_record {
  int id;            /* the track's id */
  int start;         /* the segment's first frame, counted from ofdis_traj_begin's frame */
  float mean_x, mean_y, sd_x, sd_y, length;
} ofdis_traj_record;  /* 28 bytes */
typedef struct ofdis_traj_stats {
  long long emitted, rejected_static, rejected_erratic, rejected_jump, rejected_camera;  /* since ofdis_traj_begin */
} ofdis_traj_stats;
/* ofdis_track_begin (same arguments, outputs and errors) followed by a reset of the descriptor stage, which keeps a
 * device copy of `frame`: pair 0's source frame.  Flow contexts only.  Allocates the descriptor workspace -- per track
 * slot and list (two lists): (2(L+1) + 2L + nt*ns*ns*33 floats rounded up to 16 bytes) + 8 bytes of state, per slot
 * 40 bytes of scan state, per pixel 44 bytes of fields, one frame, and the records and descriptors of max_frames pairs
 * for host outputs (capacity * ceil((max_frames + L - 1) / L) * (28 + 4*dim) bytes) -- which grows, never shrinks and
 * is freed by ofdis_destroy.  The batch command's tracker settings (1024 x 436 gray, capacity 4 x 7040 cells, 64
 * frames) with the defaults: about 420 MB, of which 106 MB the per-track state, 20 MB the fields and 293 MB the host
 * outputs.  A NULL or out-of-range traj, or a stereo context, is OFDIS_ERR_ARG. */
int ofdis_traj_begin(ofdis_ctx* ctx, const ofdis_track_params* params, const ofdis_traj_params* traj,
                     const unsigned char* frame, ofdis_track_point* points, int* count, int width_org, int height_org,
                     int memkind);
/* ofdis_track_advance (same frames, slots, outputs and errors) with the descriptors of every pair: the source frame of
 * pair 0 is the kept frame, of pair k >= 1 frames + (k-1)*frame_stride; the last target frame is kept for the next
 * call.  models: [f1-f0][9] float64 in host memory, or NULL.  The emitted segments' records go to records and their
 * descriptors to desc ([bound][dim] floats), bound = capacity * ceil((f1-f0 + L - 1) / L), both in memkind; pair k's
 * count goes to n_desc[k] (host).  Per pair 5 launches beyond the tracker's 5; no host round trip between pairs; one
 * synchronise at the end (host outputs: a second one after their copies).  A call before ofdis_traj_begin or after an
 * ofdis_track_begin or ofdis_track_advance, NULL records, desc or n_desc, or device outputs not 4-byte aligned is
 * OFDIS_ERR_ARG.  A call that fails on the way leaves the stage to a new ofdis_traj_begin. */
int ofdis_traj_advance(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* frames, size_t frame_stride,
                       const double* models, ofdis_track_point* points, int* counts, ofdis_traj_record* records,
                       float* desc, int* n_desc, int width_org, int height_org, int memkind);
/* The descriptor stage's counters since ofdis_traj_begin (synchronises the context's stream); OFDIS_ERR_ARG without a
 * live stage or with a NULL out. */
int ofdis_traj_stats_get(const ofdis_ctx* ctx, ofdis_traj_stats* out);

/* Fisher vectors of descriptors (extension): one fixed-length vector per clip from its descriptors, the encoding of
 * Wang and Schmid's improved dense trajectories -- PCA per descriptor block, a diagonal GMM per block and the improved
 * Fisher vector (Perronnin, Sanchez and Mensink, ECCV 2010).  The context owns one encoder: the device codebook, the
 * float64 statistics of the clip being encoded and its counters.  It persists across calls and across ofdis_run and the
 * other extensions; ofdis_fisher_begin resets it and ofdis_destroy frees it.  It reads no flow: any context may use
 * it.  Float32 without contraction, IEEE division and square root; the statistics and the normalisation float64;
 * preprocess.FisherStream restates it bit for bit.  Per descriptor x and block b (offset o, dim_in D, dim P):
 *   Projection.  y_d = sum_i proj[d][i] * (x[o+i] - mean[i]), from +0.0f in increasing i.
 *   Log-likelihood.  z_kd = (y_d - mu[k][d]) * isig[k][d]; q_k = sum_d z_kd * z_kd from +0.0f in increasing d;
 *   ll_k = c_k - 0.5f * q_k.
 *   Posteriors.  m = max_k ll_k; e_k = exp_f32(ll_k - m); s = sum_k e_k from +0.0f in increasing k; g_k = e_k / s.
 *   exp_f32 (preprocess.exp_f32): n = rintf(x * 1.44269504f), r = (x - n * 0.693145751953125f) - n * 1.42860677e-06f,
 *   p = 1/k! for k = 7 .. 0 in Horner form (p = p * r + c_k, c_7 .. c_3 = 0.000198412701f, 0.00138888892f,
 *   0.00833333377f, 0.0416666679f, 0.166666672f, then 0.5f, 1, 1), times 2^n built in the exponent field; +0 for x
 *   < -87 (e^x below FLT_MIN), exactly 1 at 0; within 2 ulp of float64 exp on [-87, 0].
 *   Skipped.  The block of x is skipped when some y_d, some q_k or m is not finite (a non-finite z makes q_k infinite;
 *   skipping it keeps 0 * inf out of the sums).  It is counted in the block's `skipped` and adds nothing.
 *   Statistics, float64, per block and Gaussian, plain sequential sums over the clip's descriptors in push order (so
 *   they do not depend on how the clip is cut into pushes): S0_k += (double)g_k; S1_kd += (double)g_k * (double)z_kd;
 *   S2_kd += (double)g_k * ((double)z_kd * (double)z_kd).  N_b counts the descriptors block b did not skip.
 *   Vector, per block, float64: u_kd = S1_kd / (N_b * sqrt(w_k)), v_kd = (S2_kd - S0_k) / (N_b * sqrt(2 * w_k)),
 *   laid out [u (K x P), v (K x P)]; each entry t becomes t < 0 ? -sqrt(|t|) : sqrt(|t|); then the sum of squares,
 *   256 partial sums over the indices = j (mod 256) in increasing index, then the partials in increasing j; each
 *   entry is divided by its square root when that is > 0 and rounded to float32.  N_b = 0 gives a block of zeros.
 *   The clip's vector is the blocks in order, 2K * sum P floats (109,056 with IDT's blocks, P = D / 2, at K = 256).
 *   Departures from VLFeat's vl_fisher: every posterior counts (VLFeat drops those below 1e-6), and the sums are
 *   float64 and sequential.
 * IDT's blocks follow from ofdis_traj_params, as preprocess.fisher_blocks gives them: shape 2L, HOG nt*ns*ns*8, HOF nt*ns*ns*9, MBHx and
 * MBHy nt*ns*ns*8 each -- 30/96/108/96/96 of the 426 floats with the defaults. */
#define OFDIS_FISHER_MAX_BLOCKS 8
typedef struct ofdis_fisher_block { int offset, dim_in, dim; } ofdis_fisher_block;
typedef struct ofdis_fisher_codebook {
  int K;             /* Gaussians per block, 1 .. 256 */
  int desc_dim;      /* floats per descriptor, >= 1 */
  int nblocks;       /* 1 .. OFDIS_FISHER_MAX_BLOCKS */
  ofdis_fisher_block blocks[OFDIS_FISHER_MAX_BLOCKS];  /* 1 <= dim <= dim_in <= 512, offset >= 0, offset + dim_in
                                                         <= desc_dim */
  /* host float32, per block in order: mean[dim_in], proj[dim][dim_in], mu[K][dim], isig[K][dim] (1/sigma, finite,
   * > 0), c[K] (log w_k - sum_d log sigma_kd, finite), w[K] (finite, > 0) -- the body of the codebook file
   * (preprocess.write_fisher_codebook: "OFDISFV1", int32 K, nblocks, desc_dim, offset/dim_in/dim per block, body) */
  const float* params;
} ofdis_fisher_codebook;
typedef struct ofdis_fisher_stats {
  long long pushed;                            /* descriptors pushed since the last begin or take */
  long long n[OFDIS_FISHER_MAX_BLOCKS];        /* N_b */
  long long skipped[OFDIS_FISHER_MAX_BLOCKS];  /* the skipped, per block */
} ofdis_fisher_stats;  /* 136 bytes */
/* Validates the codebook on the host (every range above, every array finite, isig and w > 0, else OFDIS_ERR_ARG,
 * which leaves a live encoder as it was), uploads it and resets the statistics.  Allocates the workspace -- the codebook, 8 * K * sum(1 + 2P) bytes of
 * statistics, and per chunk of 4096 descriptors the host-input staging (4 * desc_dim bytes each), y (4 * sum P),
 * the posteriors (4 * K * nblocks) and the skip flags (nblocks), plus the host-output vector: about 30 MB with IDT's
 * blocks at K = 256 -- which grows, never shrinks and is freed by ofdis_destroy. */
int ofdis_fisher_begin(ofdis_ctx* ctx, const ofdis_fisher_codebook* cb);
/* Adds n descriptors desc ([n][desc_dim] float32 in memkind) to the clip, in order; host input goes through the
 * staging in chunks of 4096.  3 launches per chunk of 4096 descriptors, no host round trip inside the call, one
 * synchronise at the end; n = 0 does nothing.  n < 0, a NULL desc with n > 0, a device desc that is not 4-byte aligned,
 * or no live encoder is OFDIS_ERR_ARG.  A call that fails on the way leaves the encoder to a new ofdis_fisher_begin. */
int ofdis_fisher_push(ofdis_ctx* ctx, const float* desc, long n, int memkind);
/* Ends the clip: its vector to fv (2K * sum P floats, may be NULL), the raw statistics [nblocks]{S0[K], S1[K][P],
 * S2[K][P]} float64 to stats (may be NULL; what an EM step needs), both in memkind (device: fv 4-byte, stats 8-byte
 * aligned, else OFDIS_ERR_ARG), and the counters to *out (host, may be NULL).  Then resets the statistics and
 * counters for the next clip; the codebook stays.  One launch when fv is given, none without; one synchronise at the end.  No live encoder is
 * OFDIS_ERR_ARG; a call that fails on the way leaves the encoder to a new ofdis_fisher_begin. */
int ofdis_fisher_take(ofdis_ctx* ctx, float* fv, double* stats, ofdis_fisher_stats* out, int memkind);
/* ofdis_traj_advance (same frames, slots, points, counts, n_desc and errors) whose emitted segments go, in the order
 * of ofdis_traj_advance's output, straight into the live encoder as an ofdis_fisher_push would take them: the
 * descriptors stay in the descriptor stage's device output and never cross to the host.  Adds 3 launches per chunk of
 * 4096 segments and one synchronise to ofdis_traj_advance's.  No live encoder, or one whose desc_dim is not the
 * descriptors' dim, is OFDIS_ERR_ARG; a call that fails on the way leaves both stages to a new begin. */
int ofdis_traj_advance_fisher(ofdis_ctx* ctx, int f0, int f1, int b0, const unsigned char* frames,
                              size_t frame_stride, const double* models, ofdis_track_point* points, int* counts,
                              int* n_desc, int width_org, int height_org, int memkind);

/* Video stabilisation (extension): a Gaussian-smoothed camera path streamed through a clip, from the per-pair models
 * of ofdis_global_motion_fullres, and every frame warped onto it on the device (the motion filter of Matsushita et al.,
 * "Full-frame video stabilization", CVPR 2005, and of OpenCV's videostab).  The context owns one stabiliser: the
 * params and weights, the index L of the last frame received, the index of the next frame to emit, the models still
 * needed and the frames not emitted yet.  It persists across calls and across ofdis_run and the other extensions;
 * ofdis_stab_begin resets it and ofdis_destroy frees it.  float64 in the path, float32 in the per-pixel warp,
 * everything without contraction and with IEEE division; preprocess.stabilize restates it bit for bit, and its output
 * does not depend on how the clip is cut into calls.  W = width_org, H = height_org, r = radius, I = the identity.
 *   Models as received.  Model k (M_k) maps a pixel of frame k to its position in frame k+1.  Its entries are divided
 *   by its m22; it is replaced by I when m22 is not finite and non-zero, an entry of the divided model is not finite,
 *   or its adjugate's (2,2) entry a = m00*m11 - m01*m10 is not finite and non-zero (I means "camera still"; the nine
 *   NaNs of a status != 0 pair are such a model).
 *   Matrices (3 x 3, row-major, float64).  (A*B)_ij = (A_i0*B_0j + A_i1*B_1j) + A_i2*B_2j.  norm(A): every entry
 *   divided by A_22.  inv(A) = norm(C) of the adjugate C: C00 = a11*a22 - a12*a21, C01 = a02*a21 - a01*a22,
 *   C02 = a01*a12 - a02*a11, C10 = a12*a20 - a10*a22, C11 = a00*a22 - a02*a20, C12 = a02*a10 - a00*a12,
 *   C20 = a10*a21 - a11*a20, C21 = a01*a20 - a00*a21, C22 = a00*a11 - a01*a10 (exact on affine maps, whose products
 *   keep the row (0, 0, 1)).  A norm or inv whose divisor is zero or not finite, or that yields a non-finite entry,
 *   makes the frame's path undefined.
 *   Path of frame t over the window [a, b], a = max(0, t-r); b = t+r in ofdis_stab_push, min(L, t+r) in
 *   ofdis_stab_finish.  P = I, acc = w0*I (w0 on the diagonal, +0.0 elsewhere), wsum = w0.  Forward, d = 1 .. b-t:
 *   P = norm(M_{t+d-1} * P), acc_ij = acc_ij + w_d*P_ij, wsum = wsum + w_d.  Backward from P = I, d = 1 .. t-a:
 *   P = norm(inv(M_{t-d}) * P), the same sums.  S = acc / wsum entry by entry (S_22 is exactly 1: acc_22 and wsum are
 *   summed in the same order); a non-finite entry of S makes the path undefined.  S maps a pixel of frame t to the
 *   weighted mean of its positions in the window's frames: the smoothed camera.
 *   Crop and limit.  s = 1 - 2*(double)crop, c = (0.5*(W-1), 0.5*(H-1)), Z = [s, 0, c_x*(1-s); 0, s, c_y*(1-s);
 *   0, 0, 1] (an output pixel -> its position in the uncropped stabilised frame).  S(l): off-diagonal entries l*S_ij,
 *   diagonal entries (1-l) + l*S_ii.  A(l) = norm(inv(S(l)) * Z), a0..a8 = A(l) rounded to float32.  l passes when
 *   A(l) is defined and each corner (0,0), (W-1,0), (0,H-1), (W-1,H-1) passes the per-pixel test below (wq > 0 and
 *   (mx/wq, my/wq) in [0, W-1] x [0, H-1]).  limit 0: l = 1; limit 1: l = 1 if it passes, else 20 rounds of bisection
 *   from lo = 0, hi = 1 with mid = 0.5*(lo + hi) (mid passes: lo = mid, else hi = mid), l = lo (S(0) = I: no correction).
 *   An undefined path, or limit 0 with A(1) undefined, gives S = I, l = 0 and status 1.
 *   Per pixel (X, Y) of output frame t, in float32: mx = (a0*X + a1*Y) + a2, my = (a3*X + a4*Y) + a5,
 *   wq = (a6*X + a7*Y) + a8; with wq > 0 and (mx/wq, my/wq) in the frame, frame t there by the bilinear byte rule and
 *   rounding of the registered frames of ofdis_global_motion_fullres, else 0. */
typedef struct ofdis_stab_params {
  int radius;   /* r, 1 .. 64: frames on each side of the smoothing window */
  float crop;   /* 0 <= crop < 0.5: the fraction cut from each side, the rest scaled back to the frame */
  int limit;    /* 0 | 1: shrink each correction so that the cropped frame's corners stay inside the source frame */
} ofdis_stab_params;
typedef struct ofdis_stab_frame {
  long long frame;        /* index in the clip, from 0 */
  int status;             /* 0, or 1: the window's path is undefined and the correction is the identity */
  double lambda;          /* l: the share of the correction the limit keeps, 1 without it */
  double correction[9];   /* S(l), row-major: frame pixel -> stabilised position, before the crop */
} ofdis_stab_frame;       /* 96 bytes */
/* Resets the stabiliser: params, weights (host, r+1 finite entries >= 0 with weights[0] > 0; w_d weighs the frames d
 * away, so the caller picks the kernel -- preprocess.gaussian_weights and the batch command make a Gaussian) and frame 0
 * ([H][W][noc] bytes in memkind).  Allocates the workspace -- a device ring of r + max_frames frames (W*H*noc bytes
 * each: 79 x 6.2 MB, about 491 MB, for 1920 x 1080 RGB at r = 15 and 64 frames), a ring of 2r + max_frames models
 * (72 bytes each) and max(r, max_frames) per-frame records (a0..a8 and the ofdis_stab_frame) -- which grows, never
 * shrinks and is freed by ofdis_destroy.  A NULL or out-of-range p, bad weights or a NULL frame is OFDIS_ERR_ARG;
 * frame sizes are checked as in ofdis_get_flow_fullres.  The stabiliser reads no flow: any context may use it. */
int ofdis_stab_begin(ofdis_ctx* ctx, const ofdis_stab_params* p, const double* weights, const unsigned char* frame0,
                     int width_org, int height_org, int memkind);
/* Appends frames L+1 .. L+n: frame k at frames + k*frame_stride (a clip: frames + hwc with stride hwc; the pairs of
 * ofdis_upload_frames_u8: image2 at stride 2hwc), in memkind, and models = [n][9] float64 in host memory, model k
 * mapping frame L+k to frame L+k+1 -- exactly what ofdis_global_motion_fullres returns.  Then emits, in order, every
 * frame t <= L' - r not emitted yet (L' = L+n): at most n frames, exactly n once the clip is longer than r.  Their bytes
 * go to out ([n][H][W][noc] in memkind), their records to info ([n], host, may be NULL) and their count to *n_out.
 * n < 1 or n > max_frames, a NULL models, frames, out or n_out, frame_stride below one frame, or no live stabiliser is
 * OFDIS_ERR_ARG. */
int ofdis_stab_push(ofdis_ctx* ctx, int n, const double* models, const unsigned char* frames, size_t frame_stride,
                    unsigned char* out, ofdis_stab_frame* info, int* n_out, int memkind);
/* Emits the remaining min(r, L+1) frames, each with its window cut at L (out holds r frames), and ends the stabiliser:
 * a push or finish before the next ofdis_stab_begin is OFDIS_ERR_ARG, as are a NULL out or n_out.
 * Host frames are copied straight into the ring, host output goes through the full-resolution scratch.  A push or
 * finish enqueues its copies and, when it emits a frame, 2 kernels, whatever n; it synchronises the context's stream
 * once, at the end.  Not part of ofdis_run's graph; the flows are not changed.  A call that fails on the way leaves
 * the stabiliser to a new ofdis_stab_begin. */
int ofdis_stab_finish(ofdis_ctx* ctx, unsigned char* out, ofdis_stab_frame* info, int* n_out, int memkind);

/* Init flow from a flow of the original frame size (extension; the reference's disabled file input,
 * run_dense.cpp:292-301,355-378).  `flow` = [f1-f0][height_org][width_org][nop] floats.  Prepares the initflow of
 * pairs [f0, f1) that the following ofdis_run(ctx, n, use_initflow = 1) reads: replicate padding to the context,
 * x 2^-(sc_f+1), cv::resize(INTER_AREA) by 2^(sc_f+1) in OpenCV's summation order (DESIGN.md section 1), written to
 * level sc_f+1 of the forward grid; with usefbcon the backward grid's level sc_f+1 is zeroed (the reference
 * initialises only the forward grid, oflow.cpp:217-220).  The context's width and height must be multiples of
 * 2^(sc_f+1) -- the padding of run_dense.cpp:301 -- else OFDIS_ERR_ARG; width_org/height_org must pad up to them.
 * Host input goes through the context's staging buffer.  Slots outside [f0, f1) are not touched.  Otherwise the
 * same arguments and status codes as ofdis_upload_frames_u8. */
int ofdis_set_initflow_fullres(ofdis_ctx* ctx, int f0, int f1, const float* flow, int width_org, int height_org,
                               int memkind);
/* Warm start (extension): the init flow of pairs [f0, f1) from the last run's flow of pairs
 * [src_f0, src_f0 + f1 - f0) -- bitwise ofdis_get_flow_fullres(DEVICE) of those pairs followed by
 * ofdis_set_initflow_fullres(DEVICE), through the context's full-resolution scratch.  Source and destination slots
 * may overlap (they are different buffers).  Same status codes as ofdis_set_initflow_fullres. */
int ofdis_set_initflow_from_result(ofdis_ctx* ctx, int f0, int f1, int src_f0, int width_org, int height_org);

/* Stage operators on frames [f0,f1) of one level. */
int ofdis_patgrid_optimize(ofdis_ctx* ctx, int level, int f0, int f1, int init_from_coarser);
int ofdis_patgrid_aggregate(ofdis_ctx* ctx, int level, int f0, int f1);
int ofdis_varref_refine(ofdis_ctx* ctx, int level, int f0, int f1);

/* Whole coarse-to-fine run on frames [0,nframes): == OFClass ctor per frame.
 * use_initflow != 0 takes the flow stored at level sc_f+1 (ofdis_set_flow,
 * ofdis_set_initflow_fullres, ofdis_set_initflow_from_result) as the reference's
 * `initflow` argument. */
int ofdis_run(ofdis_ctx* ctx, int nframes, int use_initflow);
int ofdis_sync(ofdis_ctx* ctx);

/* Dense flow of a level, (h x w x nop) interleaved float32.  Levels sc_l..sc_f+1
 * are addressable (sc_f+1 only as initflow). */
int ofdis_get_flow(ofdis_ctx* ctx, int frame, int level, float* dst, int memkind);
int ofdis_set_flow(ofdis_ctx* ctx, int frame, int level, const float* src, int memkind);
/* Final flow (level sc_l) of frames [f0,f1), contiguous, one copy. */
int ofdis_get_flow_batch(ofdis_ctx* ctx, int f0, int f1, float* dst, int memkind);

/* Per-patch results of the last ofdis_patgrid_optimize on `level` (any pointer may be
 * NULL): p[np*nop] displacement, pweight[np*novals] abs. residual, conv[np], cnt[np]. */
int ofdis_get_patches(ofdis_ctx* ctx, int frame, int level, float* p, float* pweight, int* conv,
                      int* cnt);

/* Test hook: raw internal planes of the last ofdis_varref_refine / debug run.
 * name in {"Ix","Iy","Iz","Ixx","Ixy","Iyy","Ixz","Iyz","mask","rec","dudv"};
 * returns the number of floats written (or a negative status). */
long ofdis_debug_get(ofdis_ctx* ctx, const char* name, int frame, float* dst, size_t max_floats);
/* Test hook: run only the first n_inner inner iterations of the refinement. */
int ofdis_debug_varref_iters(ofdis_ctx* ctx, int level, int f0, int f1, int n_inner);
/* Test hook: the stereo SOR's division b[i] / a[i] on the context's device and stream, for n host values.
 * q_fast: the exact SOR kernels' written-out IEEE division; q_plain: the compiler's `/`; unsafe[i] = 1 where the
 * kernels' exponent test sends the pair to the plain division (a or, if b != +-0, b outside 2^-60 <= |x| < 2^61).
 * Where unsafe[i] == 0, q_fast[i] is the correctly rounded quotient. */
int ofdis_debug_div(ofdis_ctx* ctx, const float* a, const float* b, long n, float* q_fast, float* q_plain,
                    unsigned char* unsafe);
/* Test hook: how often the stereo SOR took the plain division since create or the last reset -- tiles of
 * sor_wave_kernel and pixel updates of a warp of sor_lane_kernel (0 on ordinary inputs: their operands stay in range).
 * Synchronises the context's stream; reset != 0 zeroes the count after reading it. */
int ofdis_debug_sor_div_fallbacks(ofdis_ctx* ctx, unsigned long long* count, int reset);
/* Test hook, no context and no CUDA call: the launch plan ofdis_varref_refine takes for a w x h level of a nop / noc
 * context with tv_solverit = solverit, `frames` internal frames per launch (pairs, x 2 with usefbcon) and the SOR
 * options "sor_lane", "sor_fast", "sor_rows_per_thread", "sor_single_max", "sor_max_cluster" (ofdis_set_option).
 * out[9]: kind (0 sor_wave_kernel one CTA per frame, 1 a cluster of bands, 2 a chain of bands, 3 sor_lane_kernel,
 * 4 sor_redblack_kernel), lanes per band (sor_wave_kernel), rows per lane, lane-row slots of a stage, bands, sweeps
 * per launch, sweeps of the shorter last launch (0: none), rows per thread of assemble_kernel, assemble_kernel's
 * record layout (0 band lanes, 1 natural, 2 sor_lane_kernel's).  OFDIS_ERR_UNSUPPORTED where no plan exists. */
int ofdis_debug_sor_plan(int w, int h, int nop, int noc, int solverit, int frames, int lane, int fast, int rt,
                         int single_max, int max_cluster, int* out);

/* Number of kernels this library has launched on the context since creation. */
long ofdis_launch_count(const ofdis_ctx* ctx);
/* Eager ofdis_run x steps with a CUDA-event pair around every launch group; sums per class
 * {0 patch, 1 densify, 2 refinement setup (warp+derivatives), 3 assemble, 4 SOR} into
 * ms_by_class[5] / launches_by_class[5] (launch groups, one per stage call). */
int ofdis_profile_run(ofdis_ctx* ctx, int nframes, int steps, double* ms_by_class, long* launches_by_class);
/* The same, additionally split by pyramid level: ms_by_level_class[(level - sc_l) * 5 + class] (may be NULL). */
int ofdis_profile_levels(ofdis_ctx* ctx, int nframes, int steps, double* ms_by_class, long* launches_by_class,
                         double* ms_by_level_class);
/* usefbcon contexts only: address ONE grid of every pair (0 = forward, 1 = the grid on the swapped images)
 * in the following ofdis_patgrid_optimize / ofdis_patgrid_aggregate (one frame per call) / ofdis_set_flow /
 * ofdis_get_flow / ofdis_get_patches / ofdis_get_level calls; -1 (default) restores "both grids; flows and patches of the
 * forward one".  This is what two stand-alone PatGridClass objects joined by SetComplGrid
 * (patchgrid.h:36, oflow.cpp:162-170) are built on. */
int ofdis_set_direction(ofdis_ctx* ctx, int dir);
/* Options.  "sor_fast" 0 (default) | 1 switches the refinement's solver from the reference's lexicographic SOR to a
 *   red-black SOR (same system, omega and sweep count; SURVEY 8f rank 4): NOT bit-identical to the reference --
 *   the flow differs by a few hundredths of a pixel (bench.py reports the delta) -- and never covered by the parity
 *   claim.  All other options are launch geometry (tuning / test hook), results are bit-identical under every setting:
 *   "sor_lane"        2 (default) | 1 | 0: refinement levels of few 32-row bands (bands x sweeps <= 12 warps within the
 *                     shared memory of an SM; more sweeps than fit run in several launches) run the SOR as a wavefront of
 *                     two-pixel blocks whose warps synchronise through shared-memory flags instead of a CTA barrier
 *                     (sor_lane_kernel.cuh): 1 always, 0 never (the block wavefront of sor_wave_kernel everywhere),
 *                     2 for launches of up to 16 frames on levels of up to 64 rows -- there it is 10-20 % faster per
 *                     launch; it holds one CTA per SM at 56-row levels, which costs throughput when several streams of
 *                     large batches overlap, and every further band of rows adds start-up skew
 *   "pdl"             2 (default) | 1 | 0: programmatic dependent launch of the level loop's kernels (every kernel starts
 *                     with griddepcontrol.wait, so the next kernel's launch overlaps the tail of the current one):
 *                     1 always, 0 never, 2 for launches of up to 16 frames (2-5 % of the step there; larger batches lose)
 *   "patch_lanes"     0 (default) | 8 | 4: lanes per patch of the P = 8 gray patch kernel (other patch sizes and RGB
 *                     ignore it): 8 = one template column per lane, 4 patches per warp; 4 = two adjacent columns per
 *                     lane, 8 patches per warp, so the per-patch work its lanes repeat (bilinear weights, reductions,
 *                     Cholesky solve, stop tests) is paid once per 8 patches; 0 = 4 for launches of more than 16
 *                     frames, 8 for smaller ones
 *   "sor_rows_per_thread" 1 (default for flow) | 2 (default for stereo) | 4: rows of the 4-column tile one SOR thread updates per super-step
 *                     (a level needs W/4 + h/rows super-steps; sor_wave_kernel.cuh)
 *   "sor_single_max"  32 | 64 | 128 (default): refinement levels of up to this many SOR lanes (= rows / rows per
 *                     thread) run their SOR in one CTA, taller ones in a thread-block cluster of row bands
 *   "sor_max_cluster" 1 | 2 | 4 | 8 (portable) | 16 (default where the device grants it): at most this many SOR bands
 *                     per thread-block cluster; levels with more bands run as a chain of bands, one sweep per launch.
 *                     The workspace is sized at create for 8 and 16; 1, 2 or 4 reallocate it here when their chains need more */
int ofdis_set_option(ofdis_ctx* ctx, const char* name, int value);
/* CUDA-graph replay of ofdis_run (captured on first use per nframes). */
int ofdis_set_graph_mode(ofdis_ctx* ctx, int enabled);

#ifdef __cplusplus
}
#endif
#endif

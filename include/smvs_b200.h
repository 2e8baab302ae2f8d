/*
 * smvs_b200.h -- C ABI of libsmvs_b200.so: the SMVS per-view depth-refinement
 * hot path (Gauss-Newton construct -> block-Jacobi PCG -> node update /
 * active set, lighting fit, SGM cost volume + 8-path aggregation) as
 * hand-written sm_90a CUDA kernels.
 *
 * The reference (flanggut/smvs) has no FFI layer; the seams this ABI replaces
 * are C++ member calls inside DepthOptimizer and SGMStereo. Each entry point
 * names the reference code it stands in for (paths relative to the reference
 * root). INTEGRATION.md shows the patched bodies of those reference functions.
 *
 * Conventions
 *  - every call returns 0 on success, a negative smvsb_status on error; the
 *    message is available from smvsb_last_error(). No C++ exception crosses.
 *  - the caller owns every host buffer; the library copies in / out. Host
 *    buffers may be pageable or pinned.
 *  - a smvsb_ctx owns its device memory and one CUDA stream on the device it
 *    was created for. Contexts are independent: one per host thread / per
 *    reference view, as the reference runs one DepthOptimizer per pool thread
 *    (app/smvsrecon.cc:658-733). No global mutable state.
 *  - images are interleaved row-major exactly like mve::Image<T>:
 *    data[(y * w + x) * channels + c].
 *  - there is NO CPU fallback: without a CUDA device every call fails with
 *    SMVSB_ERR_CUDA.
 */
#ifndef SMVS_B200_H
#define SMVS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct smvsb_ctx smvsb_ctx;

/* Views (contexts) one smvsb_newton_loop_batch call can advance together. */
#define SMVSB_MAX_BATCH 8

typedef enum smvsb_status
{
    SMVSB_OK = 0,
    SMVSB_ERR_INVALID = -1,   /* bad argument / call order (std::invalid_argument in the reference) */
    SMVSB_ERR_CUDA = -2,      /* CUDA runtime error or no device */
    SMVSB_ERR_ALLOC = -3,     /* device allocation failed */
    SMVSB_ERR_STATE = -4      /* required state (views / surface / system) not set */
} smvsb_status;

/* ConjugateGradient::ReturnInfo, lib/conjugate_gradient.h:22-27 */
typedef enum smvsb_cg_info
{
    SMVSB_CG_CONVERGENCE = 0,
    SMVSB_CG_MAX_ITERATIONS = 1,
    SMVSB_CG_INVALID_INPUT = 2
} smvsb_cg_info;

/* Result of one fused inner Newton loop (smvsb_newton_loop). */
typedef struct smvsb_newton_stats
{
    int32_t newton_steps;        /* lib/depth_optimizer.cc:214,228 */
    int32_t cg_iterations;       /* sum of Status::num_iterations, :257 */
    int32_t nan_break;           /* 1 if the loop left through :267 */
    int32_t reserved;
    uint64_t n_active;           /* active nodes after the last step, :300-303 */
    double pixel_iterations;     /* sum over steps of samples of processed patches */
    double ms_construct;         /* device time, CUDA events */
    double ms_solve;
    double ms_update;
    double ms_total;             /* first launch to last result, incl. the
                                    per-step host read-back of the scalars */
    double cg_block_iterations;  /* sum over solves of (4x4 blocks of the
                                    system, i.e. both nodes active) x iterations */
    double cg_row_iterations;    /* sum over solves of active nodes x iterations */
} smvsb_newton_stats;

/* ---- lifetime ------------------------------------------------------- */

/* Number of CUDA devices this process can use (0 without a GPU or driver);
 * hosts spread their pool threads over them: thread k -> device k mod count,
 * the reference's one-view-per-thread model of app/smvsrecon.cc:658-733. */
int smvsb_device_count (void);
/* Dense fp64 FMA throughput of the device in TFLOP/s, measured on the spot
 * (8 independent DFMA chains per thread, CUDA events, best of 5): the roof the
 * Gauss-Newton construct kernel is reported against. */
int smvsb_measure_fp64_peak (int device, double* tflops_out);
int smvsb_create (int device, smvsb_ctx** out);
void smvsb_destroy (smvsb_ctx* ctx);
/* Message of the last failed call on ctx (or, with ctx == NULL, of the last
 * failed smvsb_create / context-free call on this thread). Never NULL. */
const char* smvsb_last_error (const smvsb_ctx* ctx);
/* Library identification ("smvs_b200 <version> sm_90a"). */
const char* smvsb_version (void);
/* Number of kernel launches issued on this context since creation. */
uint64_t smvsb_launch_count (const smvsb_ctx* ctx);
/* Kernel launches issued by this library in this process (all contexts and
 * smvsb_sgm calls); lets a host prove that the GPU path did the work. */
uint64_t smvsb_global_launch_count (void);
/* The same per device: shows which GPUs a multi-threaded host really used. */
uint64_t smvsb_device_launch_count (int device);

/* ---- inputs --------------------------------------------------------- */

/*
 * Per-scale image data, once per StereoView::set_scale
 * (lib/stereo_view.cc:24-46; consumed at lib/gauss_newton_step.cc:168-198,
 * 435-440).
 *   main_grad          w*h*2   StereoView::get_image_gradients() of the main view
 *   main_shading       w*h     get_shading_image()      or NULL (no -S)
 *   main_shading_grad  w*h*2   get_shading_gradients()  or NULL
 *   flen_px            StereoView::get_flen()          (lib/stereo_view.h:132-139)
 *   inv_flen           StereoView::get_inverse_flen()  (lib/stereo_view.h:141-148)
 *   sub_grad[k]        sub_w[k]*sub_h[k]*2  gradients of neighbour k
 *   sub_hess[k]        sub_w[k]*sub_h[k]*3  Hessian (xx, xy, yy) of neighbour k
 *   Mi                 n_sub*9 row-major, ti n_sub*3: DepthOptimizer::Mi/ti
 *                      (lib/depth_optimizer.cc:679-699)
 */
int smvsb_set_views (smvsb_ctx* ctx, int w, int h, double flen_px,
    double inv_flen, const float* main_grad, const float* main_shading,
    const float* main_shading_grad, int n_sub, const int* sub_w,
    const int* sub_h, const float* const* sub_grad,
    const float* const* sub_hess, const double* Mi, const double* ti);

/*
 * Same as smvsb_set_views, but from the views' BYTE images: StereoView::
 * set_scale (Gaussian blur with sigma = 0.12 * 2^scale + 0.2, then gradient
 * and Hessian; lib/stereo_view.cc:24-46, 97-188) and, with with_shading != 0,
 * StereoView::initialize_linear without gamma (:64-84) run on the device.
 * Images are single-channel (luminance) uint8, w*h each. Bit-identical to the
 * reference's CPU result, 20x less host-to-device traffic.
 */
int smvsb_set_views_u8 (smvsb_ctx* ctx, int scale, int w, int h,
    double flen_px, double inv_flen, const uint8_t* main_img,
    int with_shading, int n_sub, const int* sub_w, const int* sub_h,
    const uint8_t* const* sub_img, const double* Mi, const double* ti);

/* Parity-test access to the device-side images: view 0 = main (grad w*h*2,
 * hess ignored), view k >= 1 = neighbour k-1 (grad, hess w*h*3). */
int smvsb_debug_get_view (smvsb_ctx* ctx, int view, float* grad, float* hess);

/*
 * The Surface and the per-patch visibility lists (DepthOptimizer::subsurfaces).
 *   scale, npx, npy, start_x, start_y   grid of lib/surface.cc:28-37: patch
 *       (idx, idy) has id idy*npx+idx, covers pixels start + id*2^scale;
 *       scale 0..8 (patch size 1..256), larger is SMVSB_ERR_INVALID;
 *       node (idx, idy) has id idy*(npx+1)+idx (lib/surface.h:199-203)
 *   nodes        (npx+1)*(npy+1)*4   f, dx, dy, dxy per node (lib/bicubic_patch.h:29-36)
 *   node_valid   (npx+1)*(npy+1)     0 where Surface::nodes[i] == nullptr
 *   patch_valid  npx*npy             0 where Surface::patches[i] == nullptr
 *   vis_off      npx*npy+1, vis_ids  CSR of subsurfaces[patch] (neighbour ids,
 *                                    in the reference's order); both NULL =
 *                                    nothing visible yet (see smvsb_visibility)
 */
int smvsb_set_surface (smvsb_ctx* ctx, int scale, int npx, int npy,
    int start_x, int start_y, const double* nodes, const uint8_t* node_valid,
    const uint8_t* patch_valid, const uint32_t* vis_off,
    const uint8_t* vis_ids);

/* Replace node values only (same grid / validity / visibility). */
int smvsb_set_nodes (smvsb_ctx* ctx, const double* nodes);

/* ---- the Gauss-Newton step ----------------------------------------- */

/*
 * GaussNewtonStep::construct (lib/gauss_newton_step.cc:33-143): gradient,
 * block-sparse Hessian and inverted block-diagonal preconditioner for the
 * current surface; they stay on the device.
 *   active_nodes  (npx+1)*(npy+1) bytes, or NULL = every valid node active
 *                 (lib/depth_optimizer.cc:204-212)
 *   light16       GlobalLighting parameters or NULL (lighting == nullptr)
 */
int smvsb_gn_construct (smvsb_ctx* ctx, const uint8_t* active_nodes,
    const double* light16, double regularization,
    double light_surf_regularization);

/*
 * ConjugateGradient::solve(H, -g, &x, &P) (lib/conjugate_gradient.h:72-202)
 * on the system of the last smvsb_gn_construct. err_tol < 0 selects the
 * caller's rule of lib/depth_optimizer.cc:247 (0.01 * ||g||). x stays on the
 * device (smvsb_get_delta reads it).
 */
int smvsb_cg_solve (smvsb_ctx* ctx, int max_iter, double err_tol,
    double q_tol, int* iters, int* info);

/* delta = CG solution, (npx+1)*(npy+1)*4 doubles. */
int smvsb_get_delta (smvsb_ctx* ctx, double* delta);
/* Overwrite the CG solution (parity tests of the update step). */
int smvsb_set_delta (smvsb_ctx* ctx, const double* delta);

/*
 * lib/depth_optimizer.cc:271-303: reprojections of every pixel of every
 * processed patch before/after Surface::update_nodes(delta)
 * (lib/surface.cc:957-981), then the new active set (or, with full_opt, only
 * the mean shift, :275-289). The active set used is the one given to the last
 * smvsb_gn_construct; the new one replaces it on the device and is copied to
 * active_out (may be NULL).
 */
int smvsb_update_nodes (smvsb_ctx* ctx, double reproj_thresh, int full_opt,
    uint8_t* active_out, uint64_t* n_active, double* mean_shift);

/*
 * The whole inner loop of DepthOptimizer::run_newton_iterations
 * (lib/depth_optimizer.cc:204-304): all valid nodes active, then
 * construct -> CG (max 200 iterations, tolerance 0.01 * ||g||) -> NaN check
 * -> update -> active set, while active > initial/20 and steps < max_steps.
 */
int smvsb_newton_loop (smvsb_ctx* ctx, const double* light16,
    double regularization, double light_surf_regularization, int max_steps,
    int full_opt, smvsb_newton_stats* stats);

/*
 * The inner Newton loops of `n` views (contexts of the SAME device, each with
 * its own views and surface set) advanced in lock-step: per step the systems
 * of all views that are still iterating are constructed, solved by ONE
 * persistent PCG launch (every view with its own dot products and stopping
 * decisions) and updated. A view leaves the batch when its own loop ends
 * (lib/depth_optimizer.cc:219,267,284). The reference runs one view per pool
 * thread (app/smvsrecon.cc:658-733); this is the same work for the views a
 * GPU holds, with the per-iteration synchronisation cost of the PCG shared.
 * Results per view are bitwise those of smvsb_newton_loop on that view.
 *   light16   n pointers (each 16 doubles or NULL), or NULL for no lighting
 *   stats     n entries; the ms_* fields hold the batch's device times
 * n <= SMVSB_MAX_BATCH. All work runs on the stream of ctxs[0].
 */
int smvsb_newton_loop_batch (smvsb_ctx* const* ctxs, int n,
    const double* const* light16, double regularization,
    double light_surf_regularization, int max_steps, int full_opt,
    smvsb_newton_stats* stats);

/*
 * StereoView::set_scale (lib/stereo_view.cc:24-46, 97-188) for ONE view whose
 * float image (w*h, single channel, what byte_to_float_image made) is on the
 * host: Gaussian blur with sigma = 0.12 * 2^scale + 0.2, then the 3x3
 * quadratic-fit gradient (w*h*2) and Hessian (w*h*3), bit-identical to the
 * reference; results go back to the host arrays a StereoView holds
 * (scaleimage, image_grad, image_hessian; any may be NULL). Needs no views or
 * surface in the context.
 */
int smvsb_view_set_scale (smvsb_ctx* ctx, int w, int h, const float* image,
    int scale, float* scaleimage, float* grad, float* hess);

/*
 * The same for an image of `channels` = 1 or 3 interleaved channels
 * (StereoView::image of a colour view): mve::image::blur_gaussian blurs
 * channel by channel, initialize_image_gradients (lib/stereo_view.cc:48-62)
 * desaturates the blurred image (luminance, 0.21 / 0.72 / 0.07) before the
 * stencil. scaleimage receives the blurred image with all its channels
 * (w*h*channels); grad and hess as above.
 */
int smvsb_view_set_scale_c (smvsb_ctx* ctx, int w, int h, int channels,
    const float* image, int scale, float* scaleimage, float* grad,
    float* hess);

/*
 * DepthOptimizer::depthmap_bilateral_filter (lib/depth_optimizer.cc:957-1004):
 * joint bilateral filter of a depth map (dm_w*dm_h, 0 = no depth) guided by
 * the w*h*channels float image; spatial Gaussian `sigma` over a
 * (2*kernel_size+1)^2 window, range Gaussian 0.1 per channel; out: w*h.
 * Bit-identical to the reference (fp32, same accumulation order, expf as
 * glibc computes it). kernel_size <= 8, channels <= 4.
 */
int smvsb_bilateral_filter (smvsb_ctx* ctx, int w, int h, int channels,
    const float* guide, int dm_w, int dm_h, const float* depth, float sigma,
    int kernel_size, float* out);
/* Host twin of the device expf used above (tests compare it with libm). */
float smvsb_debug_expf (float x);

/* ---- visibility and boundary cutting (the callers' side of the loop) ---- */

/*
 * DepthOptimizer::create_subview_surfaces (lib/depth_optimizer.cc:433-604) in
 * the use_sgm mode, on the surface set by smvsb_set_surface (whose visibility
 * lists may be NULL): z-buffer of every neighbour from the surface's depth map
 * and `sgm_depth` (w*h floats, 0 = no depth), then per (patch, neighbour) the
 * 3 % border test, the 0.95 depth test and the warp-anisotropy test (> 8).
 * Patches no neighbour sees are deleted, nodes without a patch removed, the
 * context's visibility lists replaced.
 * sgm_depth == NULL is the use_sgm = false mode: only the surface's own depth
 * map fills the z-buffers, and a neighbour that passes the three tests must
 * also pass the NCC occlusion filter DepthOptimizer::ncc_for_patch (:795-912)
 * on the colour images set by smvsb_set_color_images -- including the
 * reference's carry-over of the patch's two-pixel rim into the NEXT
 * neighbour's border and depth tests (:508, :514, :551, :579).
 */
int smvsb_visibility (smvsb_ctx* ctx, const float* sgm_depth,
    uint64_t* removed_patches);

/*
 * The colour images ncc_for_patch compares: StereoView::get_image() of the
 * main view (w*h*3 floats, interleaved) and of every neighbour (sub_w*sub_h*3
 * each) at the current scale, sizes as given to smvsb_set_views. Needed only
 * for smvsb_visibility(ctx, NULL, ..); a new smvsb_set_views invalidates them.
 */
int smvsb_set_color_images (smvsb_ctx* ctx, const float* main_rgb, int n_sub,
    const float* const* sub_rgb);

/*
 * One DepthOptimizer::cut_boundaries() (lib/depth_optimizer.cc:360-431):
 * patches across a depth discontinuity, then rim patches with mse_for_patch
 * (:747-793) > 0.05, are deleted; nodes without a patch removed. inv_calib9 =
 * the main camera's fill_inverse_calibration(w, h) (row-major 3x3 floats).
 * Callers repeat while *deleted > 10, like the reference (:192-195).
 */
int smvsb_cut_boundaries (smvsb_ctx* ctx, const float* inv_calib9,
    int* deleted);

/*
 * The context's node / patch validity and visibility lists (what the two
 * calls above and smvsb_set_surface left). Any pointer may be NULL; vis_ids
 * needs room for vis_capacity entries (n_patches * n_sub always suffices).
 */
int smvsb_get_surface_state (smvsb_ctx* ctx, uint8_t* node_valid,
    uint8_t* patch_valid, uint32_t* vis_off, uint8_t* vis_ids,
    uint64_t vis_capacity);

/* ---- surface topology between the Newton loops ------------------------ */

/*
 * Surface::create(bundle, view, scale, init_depth) (lib/surface.cc:19-53 with
 * initialize_node_from_depth :665-760, fill_holes :628-649,
 * remove_nodes_without_patch :762-867): the context's surface becomes the
 * surface of `scale` initialised from init_depth (w*h floats, 0 = no depth).
 * scale 0..8, larger is SMVSB_ERR_INVALID.
 */
int smvsb_surface_create (smvsb_ctx* ctx, int scale, const float* init_depth);
/* Surface::subdivide_patches (lib/surface.cc:983-1107): the surface moves to
 * scale - 1; visibility lists are cleared (the caller runs smvsb_visibility). */
int smvsb_surface_subdivide (smvsb_ctx* ctx);
/* Surface::fill_patches_from_depth (lib/surface.cc:141-153). init_depth NULL:
 * the depth given to smvsb_surface_create (what the reference's Surface
 * keeps); otherwise it replaces it. */
int smvsb_surface_fill_from_depth (smvsb_ctx* ctx, const float* init_depth);
/* Surface::remove_isolated_patches (lib/surface.cc:887-927), with the
 * reference's sequential semantics. */
int smvsb_surface_remove_isolated (smvsb_ctx* ctx);
/* scale, npx, npy, start_x, start_y, patchsize of the context's surface */
/* Surface::expand (lib/surface.cc:482-628): two rounds of extrapolated rim
 * nodes, fill_holes, remove_nodes_without_patch; *filled_out = its return
 * value (patches created). The no-SGM mode's growth step
 * (lib/depth_optimizer.cc:330-337). */
int smvsb_surface_expand (smvsb_ctx* ctx, int* filled_out);
int smvsb_surface_info (smvsb_ctx* ctx, int* info6);

/* DepthOptimizer::Options as far as optimize() in the use_sgm mode reads them
 * (lib/depth_optimizer.h:27-44). */
typedef struct smvsb_optimize_options
{
    double regularization;
    double light_surf_regularization;
    int32_t num_iterations;      /* app/smvsrecon.cc:713: 5 */
    int32_t min_scale;
    int32_t use_shading;
    int32_t full_optimization;
    int32_t no_sgm;              /* 1: Options::use_sgm = false (--no-sgm) */
    int32_t reserved;            /* 0 */
} smvsb_optimize_options;

typedef struct smvsb_optimize_stats
{
    int32_t scales;              /* scales optimised (ladder length) */
    int32_t final_scale;
    int32_t newton_loops;        /* inner Newton loops run */
    int32_t newton_steps;
    int32_t cg_iterations;
    int32_t reserved;
    uint64_t patches;            /* valid patches of the final surface */
    double pixel_iterations;
    double ms_newton;            /* device time of the Newton loops */
} smvsb_optimize_stats;

/*
 * DepthOptimizer::optimize() (lib/depth_optimizer.cc:54-162) in the use_sgm
 * mode, with run_newton_iterations (:164-358), for one reference view whose
 * images are single-channel: bilateral filter of the SGM depth, initial
 * surface, then per scale set_scale of all views, visibility, boundary
 * cutting, Newton loops, isolated-patch removal and the patch-count
 * convergence test, subdivision and hole filling between scales, lighting fit
 * below scale 4 with use_shading. The view stays on the device from the byte
 * images to the depth and normal maps; nothing but scalars comes back in
 * between. The ladder starts at max(ceil(log2(w*h / 1.7e6) / 2) + 4, 4)
 * (:38-39), one scale coarser with no_sgm (:50); a start above scale 8
 * (above 435 MP, 108.8 MP with no_sgm) is SMVSB_ERR_INVALID.
 *   inv_calib9    main camera's fill_inverse_calibration(w, h)
 *   shading, shading_grad   StereoView::get_shading_image / _gradients
 *                 (w*h, w*h*2) or NULL without use_shading
 *   sgm_depth     StereoView::get_sgm_depth(), sgm_w * sgm_h
 *   depth_out     w*h (Surface::get_depth_map), normals_out w*h*3
 *                 (Surface::get_normal_map(inverse flen)); either may be NULL
 *   light16_out   the last fitted lighting (zeros if none), may be NULL
 */
int smvsb_optimize (smvsb_ctx* ctx, int w, int h, double flen_px,
    double inv_flen, const float* inv_calib9, const uint8_t* main_img,
    int n_sub, const int* sub_w, const int* sub_h,
    const uint8_t* const* sub_img, const double* Mi, const double* ti,
    const float* shading, const float* shading_grad, int sgm_w, int sgm_h,
    const float* sgm_depth, const smvsb_optimize_options* opts,
    float* depth_out, float* normals_out, double* light16_out,
    smvsb_optimize_stats* stats);

/*
 * The same for colour views: the images are what StereoView::get_image()
 * holds of a three-channel view (interleaved float RGB in [0, 1], w*h*3 and
 * sub_w*sub_h*3). set_scale blurs the three channels and desaturates
 * (smvsb_view_set_scale_c), the bilateral filter of the SGM depth is guided
 * by the colour image (lib/depth_optimizer.cc:42, 957-1004); everything else
 * is smvsb_optimize.
 * With opts->no_sgm the call is optimize() in the use_sgm = false mode:
 * sgm_depth (then w * h) is the sparse initial depth Surface::create makes of
 * the bundle's features (lib/surface.cc:43-46, 91-128; 0 = no feature), taken
 * without the bilateral filter; the ladder starts one scale coarser (:51);
 * visibility runs the NCC occlusion filter on the colour images (:433-604 with
 * :795-912), and every outer iteration expands the surface by a ring of
 * patches before the next visibility / cutting round (:331-339).
 */
int smvsb_optimize_rgb_f32 (smvsb_ctx* ctx, int w, int h, double flen_px,
    double inv_flen, const float* inv_calib9, const float* main_rgb,
    int n_sub, const int* sub_w, const int* sub_h,
    const float* const* sub_rgb, const double* Mi, const double* ti,
    const float* shading, const float* shading_grad, int sgm_w, int sgm_h,
    const float* sgm_depth, const smvsb_optimize_options* opts,
    float* depth_out, float* normals_out, double* light16_out,
    smvsb_optimize_stats* stats);

/* ---- outputs -------------------------------------------------------- */

int smvsb_get_nodes (smvsb_ctx* ctx, double* nodes_out);
/* Surface::get_depth_map (lib/surface.cc:155-168): w*h floats, 0 outside. */
int smvsb_get_depth (smvsb_ctx* ctx, float* depth_wh);
/* Surface::get_normal_map(inv_flen) (lib/surface.cc:170-183): w*h*3. */
int smvsb_get_normals (smvsb_ctx* ctx, float* normals_wh3);

/*
 * Parity-test access to the linear system in the reference's layout
 * (lib/block_sparse_matrix.h:95-97): blocks sorted by block column then block
 * row, each 4x4 row-major, inner = 4 * block row, outer = num_nodes+1 prefix.
 * Pass NULL for anything not wanted; *nnzb_h / *nnzb_p receive block counts
 * (call once with NULL arrays to size the buffers).
 */
int smvsb_debug_get_system (smvsb_ctx* ctx, double* g, double* Hvals,
    uint64_t* Houter, uint64_t* Hinner, uint64_t* nnzb_h, double* Pvals,
    uint64_t* Pouter, uint64_t* Pinner, uint64_t* nnzb_p);
/* y = H x with the device SpMV kernel (parity of lib/block_sparse_matrix.h:276-298). */
int smvsb_debug_spmv (smvsb_ctx* ctx, const double* x, double* y);

/*
 * LightOptimizer::fit_lighting_to_image (lib/light_optimizer.cc:22-55) on the
 * current surface and the main view's shading image: 16 SH coefficients.
 * nccl_comm: NULL for the reference's per-view behaviour; otherwise an
 * ncclComm_t -- the 16x16+16 normal equations are summed over the
 * communicator before the pseudo inverse (opt-in global lighting, changes
 * results w.r.t. the reference; see DESIGN.md).
 */
int smvsb_fit_lighting (smvsb_ctx* ctx, double* params16_out,
    void* nccl_comm);

/* ---- SGM ------------------------------------------------------------ */

/*
 * SGMStereo::run_sgm (lib/sgm_stereo.cc:98-124) = create_cost_volume
 * (:192-244) + aggregate_sgm_costs (:429-667, SSE branch: constant P2) +
 * depth_from_sgm_volume (:274-306), for one main / neighbour luminance pair
 * that is already at SGM working resolution.
 *   M, t       fp32 reprojection main -> neighbour at these sizes
 *              (mve::CameraInfo::fill_reprojection, lib/sgm_stereo.cc:158-160)
 *   depth_out  w*h floats
 *   cost_out / sgm_out  optional w*h*num_steps uint16 dumps (NULL to skip)
 *   ms_out     optional double[3]: device ms of cost volume, aggregation, WTA
 * num_steps must be a multiple of 32 and <= 256. Runs within the default
 * device budget (smvsb_sgm_ex with opts = NULL).
 */
int smvsb_sgm (int device, int w, int h, const uint8_t* main_lum,
    int nw, int nh, const uint8_t* neigh_lum, const float* M, const float* t,
    float min_depth, float max_depth, int num_steps, uint16_t penalty1,
    uint16_t penalty2, float* depth_out, uint16_t* cost_out,
    uint16_t* sgm_out, double* ms_out);

/*
 * SGMStereo::reconstruct (lib/sgm_stereo.cc:45-96) for one main / neighbour
 * luminance pair at SGM working resolution: run_sgm main -> neighbour and
 * neighbour -> main (both on the device, volumes never leave it), then the
 * consistency check of :64-91 -- a main depth survives if its reprojection
 * lands inside the neighbour's 3 % border on a pixel with depth and the two
 * depths agree within 20 % -- and, if merge_with != NULL, the merge of
 * app/smvsrecon.cc:362-377 with an earlier result for the same main view
 * (mean where both have depth). One depth image leaves the GPU.
 *   M_mn, t_mn   fp32 reprojection main -> neighbour (fill_reprojection at the
 *                working sizes; also used by the consistency check, :66-69)
 *   M_nm, t_nm   the same, neighbour -> main
 *   depth_range_main / _neigh   {min, max} depth of the two runs (:50-61)
 *   merge_with   w*h floats or NULL
 *   ms_out       optional double[2]: device ms of the two run_sgm
 * Runs within the default device budget (smvsb_sgm_reconstruct_ex with
 * opts = NULL).
 */
int smvsb_sgm_reconstruct (int device, int w, int h, const uint8_t* main_lum,
    int nw, int nh, const uint8_t* neigh_lum, const float* M_mn,
    const float* t_mn, const float* M_nm, const float* t_nm,
    const float* depth_range_main, const float* depth_range_neigh,
    int num_steps, uint16_t penalty1, uint16_t penalty2,
    const float* merge_with, float* depth_out, double* ms_out);

/* Device memory of smvsb_sgm_ex and smvsb_sgm_reconstruct_ex. */
typedef struct smvsb_sgm_options
{
    uint64_t device_bytes;       /* the device's SGM workspace holds at most
                                    this much; 0 = the smaller of a quarter of
                                    the card and its free memory (counting
                                    what the workspace holds) less a margin
                                    (1/32 of the card, >= 256 MiB) */
    uint64_t reserved[3];        /* 0 */
} smvsb_sgm_options;

typedef struct smvsb_sgm_stats
{
    int32_t banded;              /* 1: a run took the banded path */
    int32_t bands;               /* bands per run (the larger of a
                                    reconstruct's two); 1 on the volume path */
    uint64_t peak_device_bytes;  /* the workspace's largest size in the call */
    uint64_t host_bytes;         /* partial sums staged in pinned host memory */
    double ms_device;            /* CUDA events over the run_sgm calls */
} smvsb_sgm_stats;

/*
 * smvsb_sgm and smvsb_sgm_reconstruct within a device-memory budget (the
 * per-device workspace holds at most opts->device_bytes after the call).
 * Each run_sgm keeps its whole cost and aggregation volumes on the device
 * (about 10 bytes per voxel) when they fit the budget. Otherwise it runs in
 * bands of image rows: cost per band (census halo recomputed), a top-to-bottom
 * sweep of the downward and horizontal paths that keeps a uint16 partial sum
 * per voxel (on the device, or in pinned host memory when the budget cannot
 * hold it next to a useful band), and a bottom-to-top sweep of the upward
 * paths that adds it and takes the winner. The depth is bit-identical
 * whatever the path and budget. cost_out / sgm_out always take the volume
 * path, whatever the budget. On the banded path the stages interleave:
 * ms_out[0] of smvsb_sgm_ex is the whole run and ms_out[1..2] are 0.
 *   opts    NULL = defaults
 *   stats   may be NULL
 * SMVSB_ERR_INVALID: a device_bytes budget too small for one band of 16 rows
 * and the carried state (the message names the minimum); SMVSB_ERR_ALLOC:
 * the default budget is that small, or the device has not that much memory.
 */
int smvsb_sgm_ex (int device, int w, int h, const uint8_t* main_lum,
    int nw, int nh, const uint8_t* neigh_lum, const float* M, const float* t,
    float min_depth, float max_depth, int num_steps, uint16_t penalty1,
    uint16_t penalty2, float* depth_out, uint16_t* cost_out,
    uint16_t* sgm_out, double* ms_out, const smvsb_sgm_options* opts,
    smvsb_sgm_stats* stats);

int smvsb_sgm_reconstruct_ex (int device, int w, int h,
    const uint8_t* main_lum, int nw, int nh, const uint8_t* neigh_lum,
    const float* M_mn, const float* t_mn, const float* M_nm,
    const float* t_nm, const float* depth_range_main,
    const float* depth_range_neigh, int num_steps, uint16_t penalty1,
    uint16_t penalty2, const float* merge_with, float* depth_out,
    double* ms_out, const smvsb_sgm_options* opts, smvsb_sgm_stats* stats);

/* ---- after the per-view optimisation ------------------------------------ */

/*
 * MeshGenerator::cut_depth_maps (lib/mesh_generator.cc:25-158): the
 * cross-view consistency cut of all depth maps of a scene, on one device:
 * smvsb_cut_depth_maps_multi with the device list { device } and the
 * default budget.
 *   depth[i]      w[i]*h[i], MVE convention (distance along the viewing ray),
 *                 what View::get_float_image(dm_name) holds (:190)
 *   normals[i]    w[i]*h[i]*3, world space (after :192-203)
 *   invproj9      per view: CameraInfo::fill_inverse_calibration(w, h) (:38-40)
 *   cam_to_world16   per view: CameraInfo::fill_cam_to_world (:55)
 *   KR9, t3       per view: MeshGenerator::ViewProjection (:302-312)
 *   depth_out[i]  the cut maps (same convention as depth[i])
 * The matrices are computed by the host with the reference's own camera code;
 * the device only consumes them.
 */
int smvsb_cut_depth_maps (int device, int n_views, const int* w, const int* h,
    const float* const* depth, const float* const* normals,
    const float* invproj9, const float* cam_to_world16, const float* KR9,
    const float* t3, float* const* depth_out);

/* Devices and memory of smvsb_cut_depth_maps_multi. */
typedef struct smvsb_cut_options
{
    const int* devices;          /* one worker per entry; an id may repeat */
    int32_t n_devices;
    int32_t reserved0;           /* 0 */
    uint64_t device_bytes;       /* per device, split among its workers;
                                    0 = free memory at call time less a
                                    margin (1/32 of the card, >= 256 MiB) */
    uint64_t reserved[2];        /* 0 */
} smvsb_cut_options;

typedef struct smvsb_cut_stats
{
    uint64_t reference_pairs;    /* sum of valid pixels x (n_views - 1): the
                                    (pixel, view) pairs of the reference's loop */
    uint64_t evaluated_pairs;    /* pairs left after culling */
    uint64_t bytes_uploaded;     /* host -> device */
    int32_t target_groups;       /* over all workers */
    int32_t source_chunks;
    double ms_device;            /* longest worker, CUDA events */
} smvsb_cut_stats;

/*
 * MeshGenerator::cut_depth_maps (lib/mesh_generator.cc:25-158) for scenes
 * larger than one device, on every device of a list. The maps stay in the
 * caller's host buffers (as the reference keeps them in host RAM). Each
 * worker holds a group of target views (as many as its budget holds) and
 * streams the source views the group needs through pinned staging buffers
 * in ascending j, chunk by chunk; 16x16 tiles of target pixels skip the
 * source views their world-space box cannot project into (behind the camera
 * or outside the image, with fp32 rounding accounted for). Target views come
 * from a shared counter. The cut maps are those of the reference whatever
 * the device list, budget, grouping or chunking.
 *   opts          devices, per-device cap (see smvsb_cut_options)
 *   stats         may be NULL
 * Everything else as smvsb_cut_depth_maps. SMVSB_ERR_INVALID: empty device
 * list, device id out of range, or a device_bytes cap that cannot hold the
 * largest target view next to one source view; SMVSB_ERR_ALLOC: the device
 * has not that much free memory.
 */
int smvsb_cut_depth_maps_multi (const smvsb_cut_options* opts, int n_views,
    const int* w, const int* h, const float* const* depth,
    const float* const* normals, const float* invproj9,
    const float* cam_to_world16, const float* KR9, const float* t3,
    float* const* depth_out, smvsb_cut_stats* stats);

#ifdef __cplusplus
}
#endif

#endif /* SMVS_B200_H */

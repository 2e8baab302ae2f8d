/*
 * common.cuh -- context, device buffers and small helpers shared by the
 * smvs_b200 kernels. sm_90a (H100) only; there is no host fallback anywhere.
 */
#ifndef SMVSB_COMMON_CUH
#define SMVSB_COMMON_CUH

#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/smvs_b200.h"

#define SMVSB_MAX_SUBS 32          /* neighbours per reference view */
#define SMVSB_MAX_SCALE 8          /* coarsest surface scale (patch size 256) */
#define SMVSB_NB_STRIDE 8          /* floats per packed neighbour texel */
#define SMVSB_NUM_EVENTS 6

/* Throws smvsb::Error (caught at the ABI boundary). */
#define CUDA_CHECK(call)                                                     \
    do {                                                                     \
        cudaError_t e__ = (call);                                            \
        if (e__ != cudaSuccess)                                              \
            throw smvsb::Error(SMVSB_ERR_CUDA, std::string(#call) + ": "     \
                + cudaGetErrorString(e__));                                  \
    } while (0)

namespace smvsb {

struct Error
{
    int code;
    std::string msg;
    Error (int c, std::string const& m) : code(c), msg(m) {}
};

/* Owning device buffer; grows, and shrinks only by release(). */
template <typename T>
struct DevBuf
{
    T* p = nullptr;
    size_t cap = 0;      /* elements */

    DevBuf (void) = default;
    DevBuf (DevBuf const&) = delete;
    DevBuf& operator= (DevBuf const&) = delete;
    ~DevBuf (void) { if (p) cudaFree(p); }

    void reserve (size_t n)
    {
        if (n <= cap)
            return;
        if (p) { cudaFree(p); p = nullptr; cap = 0; }
        cudaError_t e = cudaMalloc(&p, n * sizeof(T));
        if (e != cudaSuccess)
        {
            p = nullptr;
            throw Error(SMVSB_ERR_ALLOC, std::string("cudaMalloc of ")
                + std::to_string(n * sizeof(T)) + " bytes: "
                + cudaGetErrorString(e));
        }
        cap = n;
    }

    void release (void)
    {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }

    size_t bytes (void) const { return cap * sizeof(T); }
};

/* One neighbour view on the device: packed texels
 * (gx, gy, hxx, hxy, hyy, 0, 0, 0) -- one 32-byte sector per texel. */
struct SubViewDev
{
    int w = 0, h = 0;
    DevBuf<float> texels;
};

/* Arguments shared by the Gauss-Newton kernels (passed by value). */
struct SurfaceDev
{
    int scale, ps, sampling, npos;      /* npos = ps / sampling */
    int npx, npy, start_x, start_y;
    int n_nodes, n_patches;
    int w, h;                           /* main view size */
    double flen, inv_flen;
    int n_sub;
    double const* nodes;                /* n_nodes * 4 */
    uint8_t const* node_valid;
    uint8_t const* patch_valid;
    uint32_t const* vis_off;
    uint8_t const* vis_ids;
    uint8_t const* active;              /* current active set */
    float const* main_grad;             /* w*h*2 */
    float const* main_shading;          /* w*h or null */
    float const* main_shading_grad;     /* w*h*2 or null */
    float const* const* sub_texels;     /* device array of n_sub pointers */
    int const* sub_dims;                /* device array: w0,h0,w1,h1,... */
    double const* Mt;                   /* device: n_sub * 12 (M 9, t 3) */
    double const* basis_s;              /* sampled positions: 3 * npos * 4 */
    double const* basis_f;              /* all pixel positions: 3 * ps * 4 */
};

/* Page-locked landing places of a context's asynchronous read-backs: each is
 * copied on the context's stream and read after that stream synchronised. */
struct PinnedResults
{
    double cg[3];                       /* cg_result: iterations, info, x0 NaN */
    unsigned long long cg_counts[2];    /* blocks, rows of the solved system */
    double update[3];                   /* upd_result: shift sum, shift count,
                                           active nodes */
    unsigned long long processed;       /* patches count_processed counted */
    unsigned long long vis_flags;       /* smvsb_set_surface's list check */
};

} /* namespace smvsb */

struct smvsb_ctx
{
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[SMVSB_NUM_EVENTS] = {};
    /* smvsb_set_views_u8: the upload of image k + 1 (copy stream) runs under
     * set_scale of image k (two staging buffers) */
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copied[2] = {}, ev_consumed[2] = {};
    std::string last_error;
    uint64_t launches = 0;
    int num_sms = 0;

    /* views */
    bool have_views = false;
    int w = 0, h = 0, n_sub = 0;
    double flen = 0, inv_flen = 0;
    smvsb::DevBuf<float> main_grad, main_shading, main_shading_grad;
    bool have_shading = false;
    smvsb::SubViewDev subs[SMVSB_MAX_SUBS];
    smvsb::DevBuf<float const*> sub_ptrs;
    smvsb::DevBuf<int> sub_dims;
    smvsb::DevBuf<double> Mt;
    smvsb::DevBuf<uint8_t> stage_u8;       /* upload staging (reused) */
    smvsb::DevBuf<uint8_t> stage_u8b;
    smvsb::DevBuf<float> stage_a, stage_b;
    smvsb::DevBuf<float> view_in, view_texels, view_out;   /* smvsb_view_set_scale */

    /* surface */
    bool have_surface = false;
    int scale = 0, ps = 0, sampling = 0, npos = 0;
    int npx = 0, npy = 0, start_x = 0, start_y = 0;
    int n_nodes = 0, n_patches = 0;
    smvsb::DevBuf<double> nodes;
    smvsb::DevBuf<uint8_t> node_valid, patch_valid, vis_ids;
    smvsb::DevBuf<uint32_t> vis_off;
    smvsb::DevBuf<uint8_t> active, active_new;
    smvsb::DevBuf<double> basis_s, basis_f;
    std::vector<uint8_t> h_node_valid, h_patch_valid;

    /* resident pipeline (smvsb_optimize, topology.cu) */
    smvsb::DevBuf<float> init_depth;        /* Surface::depth */
    smvsb::DevBuf<double> nodes_tmp;
    smvsb::DevBuf<uint8_t> node_valid_tmp;
    smvsb::DevBuf<uint8_t> u8_main;
    smvsb::DevBuf<uint8_t> u8_subs[SMVSB_MAX_SUBS];
    smvsb::DevBuf<float> guide;             /* byte_to_float(main image) */

    /* linear system */
    bool have_system = false;
    smvsb::DevBuf<double> patch_H;      /* n_patches * 256 */
    smvsb::DevBuf<double> patch_g;      /* n_patches * 16 */
    smvsb::DevBuf<uint8_t> patch_proc;  /* n_patches */
    smvsb::DevBuf<double> H;            /* n_nodes * 9 * 16 */
    smvsb::DevBuf<double> P;            /* n_nodes * 16 */
    smvsb::DevBuf<double> g;            /* n_nodes * 4 */
    smvsb::DevBuf<double> light;        /* 16 */

    /* CG */
    smvsb::DevBuf<double> x, r, d, d2, z, Ad;
    size_t x_count = 0;                 /* entries of x that belong to the
                                           current surface (0 = none) */
    smvsb::DevBuf<double> cg_partials;
    smvsb::DevBuf<uint16_t> cg_rowmask; /* existing blocks per stencil row */
    smvsb::DevBuf<uint32_t> cg_row_list, cg_block_rows;
    smvsb::DevBuf<unsigned long long> cg_counts;
    uint64_t cg_blocks = 0, cg_rows = 0;    /* of the last solve's system */
    smvsb::PinnedResults* pinned = nullptr;
    smvsb::DevBuf<unsigned int> cg_sync;
    smvsb::DevBuf<double> cg_result;    /* iters, info, ... */

    /* update */
    smvsb::DevBuf<double> patch_shift;  /* n_patches * 2: sum, count */
    smvsb::DevBuf<double> upd_partials, upd_result;
    smvsb::DevBuf<unsigned long long> counters;

    /* visibility / cutting */
    smvsb::DevBuf<unsigned int> zbuf, vis_mask;
    smvsb::DevBuf<unsigned long long> zoff;
    smvsb::DevBuf<float> sgm_depth;
    /* use_sgm = false: colour images of the current scale, rim lists */
    bool have_color = false;
    smvsb::DevBuf<float> color_main;
    smvsb::DevBuf<float> color_subs[SMVSB_MAX_SUBS];
    smvsb::DevBuf<float const*> color_ptrs;
    smvsb::DevBuf<short4> rim_lists;
    int rim_ps = 0;
    int rim_off[9] = {};
    smvsb::DevBuf<uint32_t> vis_counts;

    /* lighting */
    smvsb::DevBuf<double> light_partials;

    /* render */
    smvsb::DevBuf<float> image_out;
};

namespace smvsb {

/* process-wide launch counters (smvsb_global_launch_count,
 * smvsb_device_launch_count) */
#define SMVSB_MAX_DEVICES 64
extern std::atomic<uint64_t> g_launches;
extern std::atomic<uint64_t> g_device_launches[SMVSB_MAX_DEVICES];

inline void
count_device_launches (int device, int n)
{
    g_launches += n;
    if (device >= 0 && device < SMVSB_MAX_DEVICES)
        g_device_launches[device] += n;
}

inline void
count_launches (smvsb_ctx* c, int n)
{
    c->launches += n;
    count_device_launches(c->device, n);
}

/* Throws unless `device` names a CUDA device of this process. */
inline void
check_device (int device)
{
    int count = 0;
    cudaError_t const e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
    {
        cudaGetLastError();
        throw Error(SMVSB_ERR_CUDA, std::string("no CUDA device "
            "(smvs_b200 has no CPU fallback)") + (e != cudaSuccess
            ? std::string(": ") + cudaGetErrorString(e) : std::string()));
    }
    if (device < 0 || device >= count)
        throw Error(SMVSB_ERR_INVALID, "device index out of range");
}

/* Free memory of the current device less a margin left to the runtime and
 * the process's other work (1/32 of the card, at least 256 MiB): the start of
 * the default budget of the calls that size their work to the device.
 * total_out (may be NULL): the card's memory. */
inline size_t
usable_device_bytes (size_t* total_out = nullptr)
{
    size_t free_b = 0, total_b = 0;
    CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    if (total_out != nullptr)
        *total_out = total_b;
    size_t const margin = (total_b / 32 > (size_t(256) << 20))
        ? total_b / 32 : (size_t(256) << 20);
    return free_b > margin ? free_b - margin : 0;
}

inline SurfaceDev
surface_args (smvsb_ctx* c)
{
    SurfaceDev s;
    s.scale = c->scale; s.ps = c->ps; s.sampling = c->sampling;
    s.npos = c->npos;
    s.npx = c->npx; s.npy = c->npy;
    s.start_x = c->start_x; s.start_y = c->start_y;
    s.n_nodes = c->n_nodes; s.n_patches = c->n_patches;
    s.w = c->w; s.h = c->h; s.flen = c->flen; s.inv_flen = c->inv_flen;
    s.n_sub = c->n_sub;
    s.nodes = c->nodes.p; s.node_valid = c->node_valid.p;
    s.patch_valid = c->patch_valid.p;
    s.vis_off = c->vis_off.p; s.vis_ids = c->vis_ids.p;
    s.active = c->active.p;
    s.main_grad = c->main_grad.p;
    s.main_shading = c->have_shading ? c->main_shading.p : nullptr;
    s.main_shading_grad = c->have_shading ? c->main_shading_grad.p : nullptr;
    s.sub_texels = c->sub_ptrs.p; s.sub_dims = c->sub_dims.p;
    s.Mt = c->Mt.p;
    s.basis_s = c->basis_s.p; s.basis_f = c->basis_f.p;
    return s;
}

/* A view's image on the device as StereoView::set_scale takes it: w*h bytes,
 * w*h floats, or w*h*3 interleaved floats of a colour view. */
struct DevImage
{
    enum Kind { U8, F32, RGB_F32 } kind;
    void const* p;
    int w, h;
};

/* kernels / launchers implemented in the .cu files */
void reserve_set_scale_scratch (smvsb_ctx* c, DevImage::Kind kind,
    size_t pixels);
/* StereoView::set_scale of one image: blur, then the gradient (mode 0,
 * float2 per pixel) or the packed neighbour texels (mode 1) into out. The
 * blurred image (the colour image for RGB_F32) goes to blur_out unless it is
 * null. */
void device_set_scale (smvsb_ctx* c, DevImage const& img, int scale, int mode,
    float* out, float* blur_out);
void device_shading_inputs (smvsb_ctx* c, uint8_t const* img_dev, int w, int h,
    float* shading_dev, float* shading_grad_dev);
void device_bilateral_filter (smvsb_ctx* c, float const* ci_dev, int w, int h,
    int channels, float const* dm_dev, int dm_w, int dm_h, float sigma,
    int kernel_size, float* out_dev);
float host_expf_like_glibc (float x);
void device_byte_to_float (smvsb_ctx* c, uint8_t const* img_dev, size_t n,
    float* out_dev);
void device_unpack_texels (smvsb_ctx* c, float const* texels, int n,
    float* grad, float* hess);
void fill_basis_table (std::vector<double>& tab, int ps, int step);
double measure_fp64_peak (int device);
void launch_pack_subview (smvsb_ctx* c, float const* grad, float const* hess,
    float* texels, int w, int h);
void launch_construct (smvsb_ctx* c, bool use_light, double reg,
    double light_reg);
void launch_spmv (smvsb_ctx* c, double const* x, double* y);
void run_cg (smvsb_ctx* c, int max_iter, double err_tol, double q_tol,
    int* iters, int* info, bool* x0_nan);
void cg_enqueue (smvsb_ctx* const* cs, int n, int max_iter, double err_tol,
    double q_tol);
void cg_collect (smvsb_ctx* c, int* iters, int* info, bool* x0_nan);
void launch_update (smvsb_ctx* c, double thresh, bool full_opt,
    uint64_t* n_active, double* mean_shift);
void update_enqueue (smvsb_ctx* c, double thresh, bool full_opt);
void update_collect (smvsb_ctx* c, uint64_t* n_active, double* mean_shift);
void count_processed_enqueue (smvsb_ctx* c);
unsigned long long count_processed_collect (smvsb_ctx* c);
void launch_render_depth (smvsb_ctx* c, float* out_dev);
void launch_render_normals (smvsb_ctx* c, float* out_dev);
void run_fit_lighting (smvsb_ctx* c, double* A_b_host /*272*/);
void launch_count_processed (smvsb_ctx* c, unsigned long long* n_proc_host);
uint64_t run_visibility (smvsb_ctx* c, float const* sgm_depth_host);
uint64_t run_visibility_device (smvsb_ctx* c, bool use_sgm = true);   /* c->sgm_depth already set */
uint64_t run_visibility_ncc (smvsb_ctx* c);      /* use_sgm = false, colour images set */
void launch_remove_nodes (smvsb_ctx* c);
/* off[i] = counts[0] + ... + counts[i - 1] for i = 0 .. n (off[n]: the
 * total); one block of 1024 threads */
void launch_exclusive_scan (smvsb_ctx* c, uint32_t const* counts,
    uint32_t* off, int n);
void topo_fill_from_depth (smvsb_ctx* c);
void topo_set_init_depth (smvsb_ctx* c, float const* src_dev);
void topo_subdivide (smvsb_ctx* c, int* new_npx, int* new_npy, int* new_sx,
    int* new_sy);
void topo_subdivide_finish (smvsb_ctx* c);
void topo_remove_isolated (smvsb_ctx* c);
uint64_t topo_expand (smvsb_ctx* c);
uint64_t topo_count_patches (smvsb_ctx* c);
uint64_t run_cut_boundaries (smvsb_ctx* c, float const* inv_calib9);
void sgm_run (int device, int w, int h, uint8_t const* main_lum, int nw, int nh,
    uint8_t const* neigh_lum, float const* M, float const* t,
    float min_depth, float max_depth, int num_steps, uint16_t penalty1,
    uint16_t penalty2, float* depth_out, uint16_t* cost_out,
    uint16_t* sgm_out, double* ms_out, smvsb_sgm_options const* opts,
    smvsb_sgm_stats* stats);
void sgm_reconstruct (int device, int w, int h, uint8_t const* main_lum,
    int nw, int nh, uint8_t const* neigh_lum, float const* M_mn,
    float const* t_mn, float const* M_nm, float const* t_nm,
    float const* depth_range_main, float const* depth_range_neigh,
    int num_steps, uint16_t penalty1, uint16_t penalty2,
    float const* merge_with, float* depth_out, double* ms_out,
    smvsb_sgm_options const* opts, smvsb_sgm_stats* stats);
void cut_depth_maps_multi (smvsb_cut_options const* opts, int n_views,
    int const* w, int const* h, float const* const* depth,
    float const* const* normals, float const* invproj9,
    float const* cam_to_world16, float const* KR9, float const* t3,
    float* const* depth_out, smvsb_cut_stats* stats);

} /* namespace smvsb */

#endif

/*
 * api.cu -- the C ABI of include/smvs_b200.h over the kernels.
 * Host code here is plumbing: argument checks, uploads, launch order of the
 * Newton loop (lib/depth_optimizer.cc:204-304). No numeric step of the hot
 * path runs on the host; the one exception is the 16x16 pseudo inverse that
 * closes the lighting fit (lib/light_optimizer.cc:50-52), a 16x16 SVD.
 */
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <dlfcn.h>

#include "common.cuh"

namespace smvsb {
std::atomic<uint64_t> g_launches(0);
std::atomic<uint64_t> g_device_launches[SMVSB_MAX_DEVICES];
}

namespace {

thread_local std::string g_last_error = "";

/* A call that fails may have asynchronous copies from the caller's buffers
 * queued: they are finished before the error is returned. */
void
quiesce (smvsb_ctx* ctx)
{
    if (ctx == nullptr)
        return;
    if (ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
}

template <typename F>
int
guarded (smvsb_ctx* ctx, F&& fn)
{
    try
    {
        if (ctx != nullptr)
        {
            cudaError_t e = cudaSetDevice(ctx->device);
            if (e != cudaSuccess)
                throw smvsb::Error(SMVSB_ERR_CUDA,
                    std::string("cudaSetDevice: ") + cudaGetErrorString(e));
        }
        fn();
        return SMVSB_OK;
    }
    catch (smvsb::Error const& e)
    {
        quiesce(ctx);
        if (ctx) ctx->last_error = e.msg; else g_last_error = e.msg;
        return e.code;
    }
    catch (std::exception const& e)
    {
        quiesce(ctx);
        if (ctx) ctx->last_error = e.what(); else g_last_error = e.what();
        return SMVSB_ERR_INVALID;
    }
}

void
require (bool cond, int code, char const* msg)
{
    if (!cond)
        throw smvsb::Error(code, msg);
}

/* smvsb_set_surface: the visibility lists as the kernels will read them --
 * bit 0: offsets not monotone (or beyond the id array), 1: a list longer than
 * the number of neighbours, 2: an id out of range, 3: a neighbour twice. */
__global__ void __launch_bounds__(256)
vis_validate_kernel (int n_patches, int n_sub, uint32_t total,
    uint32_t const* __restrict__ vis_off, uint8_t const* __restrict__ vis_ids,
    unsigned long long* __restrict__ flags)
{
    int const p = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned int bad = 0;
    if (p < n_patches)
    {
        uint32_t const b = vis_off[p], e = vis_off[p + 1];
        if (b > e || e > total)
            bad |= 1u;
        else if (e - b > static_cast<uint32_t>(n_sub))
            bad |= 2u;
        else
        {
            uint32_t seen = 0;
            for (uint32_t i = b; i < e; ++i)
            {
                uint32_t const id = vis_ids[i];
                if (id >= static_cast<uint32_t>(n_sub))
                    bad |= 4u;
                uint32_t const bit = 1u << (id & 31u);
                if (seen & bit)
                    bad |= 8u;
                seen |= bit;
            }
        }
    }
    bad = __reduce_or_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && bad != 0)
        atomicOr(flags, static_cast<unsigned long long>(bad));
}

template <typename T>
void
upload (smvsb_ctx* c, smvsb::DevBuf<T>& buf, T const* host, size_t n)
{
    buf.reserve(std::max<size_t>(n, 1));
    if (n > 0)
        CUDA_CHECK(cudaMemcpyAsync(buf.p, host, n * sizeof(T),
            cudaMemcpyHostToDevice, c->stream));
}

template <typename T>
void
download (smvsb_ctx* c, T* host, T const* dev, size_t n)
{
    CUDA_CHECK(cudaMemcpyAsync(host, dev, n * sizeof(T),
        cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
}

int
sampling_for_scale (int scale)
{
    /* lib/gauss_newton_step.cc:157-161 */
    int sampling = 4;
    if (scale < 5) sampling = 2;
    if (scale < 3) sampling = 1;
    return sampling;
}

/* One-sided Jacobi SVD based pseudo inverse of a symmetric 16x16 matrix,
 * singular values within 1e-12 of zero dropped
 * (math::matrix_pseudo_inverse as called at lib/light_optimizer.cc:51). */
void
pseudo_inverse_16 (double const* A, double* Ainv)
{
    int const N = 16;
    double U[256], V[256];
    std::copy(A, A + 256, U);
    std::fill(V, V + 256, 0.0);
    for (int i = 0; i < N; ++i) V[i * N + i] = 1.0;
    for (int sweep = 0; sweep < 60; ++sweep)
    {
        double off = 0.0;
        for (int p = 0; p < N - 1; ++p)
            for (int q = p + 1; q < N; ++q)
            {
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < N; ++i)
                {
                    alpha += U[i * N + p] * U[i * N + p];
                    beta += U[i * N + q] * U[i * N + q];
                    gamma += U[i * N + p] * U[i * N + q];
                }
                double const lim = std::sqrt(alpha * beta);
                if (gamma == 0.0 || std::abs(gamma) <= 1e-16 * lim)
                    continue;
                off = std::max(off, std::abs(gamma) / (lim > 0 ? lim : 1.0));
                double const zeta = (beta - alpha) / (2.0 * gamma);
                double const t = (zeta >= 0 ? 1.0 : -1.0)
                    / (std::abs(zeta) + std::sqrt(1.0 + zeta * zeta));
                double const cs = 1.0 / std::sqrt(1.0 + t * t);
                double const sn = cs * t;
                for (int i = 0; i < N; ++i)
                {
                    double const up = U[i * N + p], uq = U[i * N + q];
                    U[i * N + p] = cs * up - sn * uq;
                    U[i * N + q] = sn * up + cs * uq;
                    double const vp = V[i * N + p], vq = V[i * N + q];
                    V[i * N + p] = cs * vp - sn * vq;
                    V[i * N + q] = sn * vp + cs * vq;
                }
            }
        if (off < 1e-15)
            break;
    }
    double sinv[16];
    for (int j = 0; j < N; ++j)
    {
        double n = 0.0;
        for (int i = 0; i < N; ++i) n += U[i * N + j] * U[i * N + j];
        n = std::sqrt(n);
        for (int i = 0; i < N; ++i)
            U[i * N + j] = (n > 0.0 ? U[i * N + j] / n : 0.0);
        sinv[j] = (n >= -1e-12 && n <= 1e-12) ? 0.0 : 1.0 / n;
    }
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < N; ++j)
        {
            double s = 0.0;
            for (int k = 0; k < N; ++k)
                s += V[i * N + k] * sinv[k] * U[j * N + k];
            Ainv[i * N + j] = s;
        }
}

/* The lighting parameters from the normal equations Ab = A (16x16) | b (16):
 * pinv(A) b (lib/light_optimizer.cc:50-52). */
void
lighting_from_normal_equations (double const* Ab, double* out16)
{
    double Ainv[256];
    pseudo_inverse_16(Ab, Ainv);
    for (int i = 0; i < 16; ++i)
    {
        double s = 0.0;
        for (int j = 0; j < 16; ++j)
            s += Ainv[i * 16 + j] * Ab[256 + j];
        out16[i] = s;
    }
}

/* New views for the context: the stored grid and visibility ids were checked
 * against the old image size and neighbour count. The colour images
 * (smvsb_set_color_images) stay while the geometry of the views does: the
 * reference's get_image() does not change with the scale. */
void
forget_stale_views (smvsb_ctx* c, int w, int h, int n_sub, int const* sub_w,
    int const* sub_h)
{
    if (c->w != w || c->h != h || c->n_sub != n_sub)
    {
        c->have_surface = false;
        c->have_color = false;
    }
    for (int k = 0; c->have_color && k < n_sub; ++k)
        if (c->subs[k].w != sub_w[k] || c->subs[k].h != sub_h[k])
            c->have_color = false;
}

/* The neighbour tables from arguments the caller checked: each neighbour's
 * size and texel buffer (reserved; the caller fills it), and the device
 * arrays of texel pointers, sizes and M | t that the kernels read. */
void
set_neighbour_tables (smvsb_ctx* c, int n_sub, int const* sub_w,
    int const* sub_h, double const* Mi, double const* ti)
{
    c->n_sub = n_sub;
    std::vector<float const*> ptrs(std::max(n_sub, 1), nullptr);
    std::vector<int> dims(std::max(2 * n_sub, 2), 0);
    std::vector<double> mt(std::max(12 * n_sub, 12), 0.0);
    for (int k = 0; k < n_sub; ++k)
    {
        smvsb::SubViewDev& sv = c->subs[k];
        sv.w = sub_w[k]; sv.h = sub_h[k];
        sv.texels.reserve(static_cast<size_t>(sv.w) * sv.h * SMVSB_NB_STRIDE);
        ptrs[k] = sv.texels.p;
        dims[2 * k] = sv.w; dims[2 * k + 1] = sv.h;
        std::copy(Mi + 9 * k, Mi + 9 * k + 9, mt.begin() + 12 * k);
        std::copy(ti + 3 * k, ti + 3 * k + 3, mt.begin() + 12 * k + 9);
    }
    upload(c, c->sub_ptrs, ptrs.data(), ptrs.size());
    upload(c, c->sub_dims, dims.data(), dims.size());
    upload(c, c->Mt, mt.data(), mt.size());
}

/* The three-channel images of the main view and of each neighbour, at the
 * sizes the context holds, and the device array of the neighbours' image
 * pointers that the NCC filter reads. */
void
upload_color_images (smvsb_ctx* c, float const* main_rgb,
    float const* const* sub_rgb)
{
    upload(c, c->color_main, main_rgb, static_cast<size_t>(c->w) * c->h * 3);
    std::vector<float const*> ptrs(c->n_sub);
    for (int k = 0; k < c->n_sub; ++k)
    {
        upload(c, c->color_subs[k], sub_rgb[k],
            static_cast<size_t>(c->subs[k].w) * c->subs[k].h * 3);
        ptrs[k] = c->color_subs[k].p;
    }
    upload(c, c->color_ptrs, ptrs.data(), ptrs.size());
}

void
ensure_system_buffers (smvsb_ctx* c)
{
    size_t const np = c->n_patches, nn = c->n_nodes;
    c->patch_H.reserve(np * 256);
    c->patch_g.reserve(np * 16);
    c->patch_proc.reserve(np);
    c->H.reserve(nn * 144);
    c->P.reserve(nn * 16);
    c->g.reserve(nn * 4);
    c->x.reserve(nn * 4);
    c->light.reserve(16);
}

void
set_active (smvsb_ctx* c, uint8_t const* active_nodes)
{
    if (active_nodes != nullptr)
        upload(c, c->active, active_nodes, c->n_nodes);
    else
    {
        /* every valid node active, lib/depth_optimizer.cc:204-212 */
        c->active.reserve(c->n_nodes);
        CUDA_CHECK(cudaMemcpyAsync(c->active.p, c->node_valid.p, c->n_nodes,
            cudaMemcpyDeviceToDevice, c->stream));
    }
}

void
construct (smvsb_ctx* c, double const* light16, double reg, double light_reg)
{
    require(c->have_views && c->have_surface, SMVSB_ERR_STATE,
        "smvsb_set_views and smvsb_set_surface must precede construct");
    if (light16 != nullptr)
    {
        require(c->have_shading, SMVSB_ERR_STATE,
            "lighting given but the main view has no shading image");
        upload(c, c->light, light16, 16);
    }
    ensure_system_buffers(c);
    smvsb::launch_construct(c, light16 != nullptr, reg, light_reg);
    c->have_system = true;
}

/* Surfaces exist at scales 0..SMVSB_MAX_SCALE (patch sizes 1..256). */
void
require_surface_scale (int scale)
{
    require(scale >= 0 && scale <= SMVSB_MAX_SCALE, SMVSB_ERR_INVALID,
        "surface scale out of range (0..8)");
}

/* Grid geometry of a Surface at `scale` (lib/surface.cc:28-37) and the tables
 * that depend on it. */
void
configure_grid (smvsb_ctx* c, int scale, int npx, int npy, int start_x,
    int start_y)
{
    require_surface_scale(scale);
    require(npx > 0 && npy > 0, SMVSB_ERR_INVALID, "empty patch grid");
    int const ps = 1 << scale;
    int const sampling = sampling_for_scale(scale);
    require(ps % sampling == 0, SMVSB_ERR_INVALID,
        "patch size below sampling");
    int const npos = ps / sampling;
    require(npos == 1 || npos == 2 || npos == 4 || npos == 8
        || npos == 16 || npos == 32 || npos == 64, SMVSB_ERR_INVALID,
        "unsupported samples per patch");
    require(start_x >= 0 && start_y >= 0
        && start_x + npx * ps <= c->w && start_y + npy * ps <= c->h,
        SMVSB_ERR_INVALID, "patch grid exceeds the main image");
    c->scale = scale; c->ps = ps; c->sampling = sampling; c->npos = npos;
    c->npx = npx; c->npy = npy; c->start_x = start_x; c->start_y = start_y;
    c->n_patches = npx * npy;
    c->n_nodes = (npx + 1) * (npy + 1);
    std::vector<double> tab;
    smvsb::fill_basis_table(tab, ps, sampling);
    upload(c, c->basis_s, tab.data(), tab.size());
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    smvsb::fill_basis_table(tab, ps, 1);
    upload(c, c->basis_f, tab.data(), tab.size());
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
}

/* Host mirrors of the validity flags after the device changed them. */
void
refresh_validity (smvsb_ctx* c)
{
    c->h_node_valid.resize(c->n_nodes);
    c->h_patch_valid.resize(c->n_patches);
    download(c, c->h_node_valid.data(), c->node_valid.p, c->n_nodes);
    download(c, c->h_patch_valid.data(), c->patch_valid.p, c->n_patches);
    set_active(c, nullptr);
    c->have_system = false;
}

/* Empty visibility lists (nothing visible yet). */
void
clear_visibility (smvsb_ctx* c)
{
    c->vis_off.reserve(static_cast<size_t>(c->n_patches) + 1);
    c->vis_ids.reserve(1);
    CUDA_CHECK(cudaMemsetAsync(c->vis_off.p, 0,
        (static_cast<size_t>(c->n_patches) + 1) * sizeof(uint32_t),
        c->stream));
}

/* Surface::Surface(bundle, view, scale, init_depth) (lib/surface.cc:19-53)
 * from an init depth that is already on the device. */
void
surface_create_device (smvsb_ctx* c, int scale, float const* init_dev)
{
    require_surface_scale(scale);
    int const ps = 1 << scale;
    int const npx = (c->w - 2) / ps - 1, npy = (c->h - 2) / ps - 1;
    require(npx > 0 && npy > 0, SMVSB_ERR_INVALID,
        "image too small for a surface at this scale");
    int const sx = (c->w - npx * ps) / 2, sy = (c->h - npy * ps) / 2;
    configure_grid(c, scale, npx, npy, sx, sy);
    size_t const nn = c->n_nodes, np = c->n_patches;
    c->nodes.reserve(nn * 4);
    c->node_valid.reserve(nn);
    c->patch_valid.reserve(np);
    CUDA_CHECK(cudaMemsetAsync(c->nodes.p, 0, nn * 4 * sizeof(double),
        c->stream));
    CUDA_CHECK(cudaMemsetAsync(c->node_valid.p, 0, nn, c->stream));
    CUDA_CHECK(cudaMemsetAsync(c->patch_valid.p, 0, np, c->stream));
    clear_visibility(c);
    smvsb::topo_set_init_depth(c, init_dev);
    smvsb::topo_fill_from_depth(c);
    c->have_surface = true;
    c->x_count = 0;
    refresh_validity(c);
}

void
surface_subdivide_device (smvsb_ctx* c)
{
    require(c->scale >= 1, SMVSB_ERR_INVALID, "cannot subdivide scale 0");
    int npx, npy, sx, sy;
    smvsb::topo_subdivide(c, &npx, &npy, &sx, &sy);
    configure_grid(c, c->scale - 1, npx, npy, sx, sy);
    smvsb::topo_subdivide_finish(c);
    clear_visibility(c);
    c->x_count = 0;
    refresh_validity(c);
}

/* StereoView::set_scale of all views from the images kept on the device
 * (smvsb_optimize): single-channel byte images, or three-channel float
 * images (StereoView::get_image() of a colour view) in the colour buffers. */
void
views_from_resident (smvsb_ctx* c, int scale, bool colour)
{
    smvsb::DevImage::Kind const kind = colour ? smvsb::DevImage::RGB_F32
        : smvsb::DevImage::U8;
    size_t max_pix = static_cast<size_t>(c->w) * c->h;
    for (int k = 0; k < c->n_sub; ++k)
        max_pix = std::max(max_pix, static_cast<size_t>(c->subs[k].w)
            * c->subs[k].h);
    smvsb::reserve_set_scale_scratch(c, kind, max_pix);
    c->main_grad.reserve(static_cast<size_t>(c->w) * c->h * 2);
    smvsb::device_set_scale(c, { kind, colour
        ? static_cast<void const*>(c->color_main.p) : c->u8_main.p, c->w,
        c->h }, scale, 0, c->main_grad.p, nullptr);
    for (int k = 0; k < c->n_sub; ++k)
    {
        smvsb::SubViewDev& sv = c->subs[k];
        sv.texels.reserve(static_cast<size_t>(sv.w) * sv.h * SMVSB_NB_STRIDE);
        smvsb::device_set_scale(c, { kind, colour
            ? static_cast<void const*>(c->color_subs[k].p) : c->u8_subs[k].p,
            sv.w, sv.h }, scale, 1, sv.texels.p, nullptr);
    }
    c->have_system = false;
}

} /* namespace */

extern "C" {

const char*
smvsb_version (void)
{
    return "smvs_b200 0.1.0 sm_90a";
}

const char*
smvsb_last_error (const smvsb_ctx* ctx)
{
    return ctx ? ctx->last_error.c_str() : g_last_error.c_str();
}

uint64_t
smvsb_launch_count (const smvsb_ctx* ctx)
{
    return ctx ? ctx->launches : 0;
}

uint64_t
smvsb_global_launch_count (void)
{
    return smvsb::g_launches.load();
}

uint64_t
smvsb_device_launch_count (int device)
{
    if (device < 0 || device >= SMVSB_MAX_DEVICES)
        return 0;
    return smvsb::g_device_launches[device].load();
}

int
smvsb_device_count (void)
{
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess)
        return 0;
    return count;
}

int
smvsb_measure_fp64_peak (int device, double* tflops_out)
{
    return guarded(nullptr, [&]() {
        require(tflops_out != nullptr, SMVSB_ERR_INVALID, "NULL output");
        smvsb::check_device(device);
        *tflops_out = smvsb::measure_fp64_peak(device);
    });
}

int
smvsb_create (int device, smvsb_ctx** out)
{
    return guarded(nullptr, [&]() {
        require(out != nullptr, SMVSB_ERR_INVALID, "out must not be NULL");
        *out = nullptr;
        smvsb::check_device(device);
        CUDA_CHECK(cudaSetDevice(device));
        smvsb_ctx* c = new smvsb_ctx();
        c->device = device;
        try
        {
            CUDA_CHECK(cudaStreamCreateWithFlags(&c->stream,
                cudaStreamNonBlocking));
            for (int i = 0; i < SMVSB_NUM_EVENTS; ++i)
                CUDA_CHECK(cudaEventCreate(&c->ev[i]));
            CUDA_CHECK(cudaStreamCreateWithFlags(&c->copy_stream,
                cudaStreamNonBlocking));
            for (int i = 0; i < 2; ++i)
            {
                CUDA_CHECK(cudaEventCreateWithFlags(&c->ev_copied[i],
                    cudaEventDisableTiming));
                CUDA_CHECK(cudaEventCreateWithFlags(&c->ev_consumed[i],
                    cudaEventDisableTiming));
            }
            CUDA_CHECK(cudaDeviceGetAttribute(&c->num_sms,
                cudaDevAttrMultiProcessorCount, device));
            CUDA_CHECK(cudaMallocHost(&c->pinned, sizeof(*c->pinned)));
        }
        catch (...)
        {
            if (c->pinned) cudaFreeHost(c->pinned);
            for (int i = 0; i < 2; ++i)
            {
                if (c->ev_copied[i]) cudaEventDestroy(c->ev_copied[i]);
                if (c->ev_consumed[i]) cudaEventDestroy(c->ev_consumed[i]);
            }
            for (int i = 0; i < SMVSB_NUM_EVENTS; ++i)
                if (c->ev[i]) cudaEventDestroy(c->ev[i]);
            if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
            if (c->stream) cudaStreamDestroy(c->stream);
            delete c;
            throw;
        }
        *out = c;
    });
}

void
smvsb_destroy (smvsb_ctx* ctx)
{
    if (ctx == nullptr)
        return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (int i = 0; i < SMVSB_NUM_EVENTS; ++i)
        if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
    if (ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream);
    for (int i = 0; i < 2; ++i)
    {
        if (ctx->ev_copied[i]) cudaEventDestroy(ctx->ev_copied[i]);
        if (ctx->ev_consumed[i]) cudaEventDestroy(ctx->ev_consumed[i]);
    }
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    delete ctx;
}

int
smvsb_set_views (smvsb_ctx* ctx, int w, int h, double flen_px,
    double inv_flen, const float* main_grad, const float* main_shading,
    const float* main_shading_grad, int n_sub, const int* sub_w,
    const int* sub_h, const float* const* sub_grad,
    const float* const* sub_hess, const double* Mi, const double* ti)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(w > 0 && h > 0 && main_grad != nullptr, SMVSB_ERR_INVALID,
            "main view missing");
        require(n_sub >= 0 && n_sub <= SMVSB_MAX_SUBS, SMVSB_ERR_INVALID,
            "n_sub out of range (max 32)");
        require((main_shading == nullptr) == (main_shading_grad == nullptr),
            SMVSB_ERR_INVALID, "shading image and gradient go together");
        require(n_sub == 0 || (sub_w && sub_h && sub_grad && sub_hess && Mi
            && ti), SMVSB_ERR_INVALID, "neighbour arrays missing");
        for (int k = 0; k < n_sub; ++k)
            require(sub_w[k] > 0 && sub_h[k] > 0 && sub_grad[k]
                && sub_hess[k], SMVSB_ERR_INVALID, "neighbour image missing");
        smvsb_ctx* c = ctx;
        forget_stale_views(c, w, h, n_sub, sub_w, sub_h);
        c->w = w; c->h = h; c->flen = flen_px; c->inv_flen = inv_flen;
        size_t const npix = static_cast<size_t>(w) * h;
        upload(c, c->main_grad, main_grad, npix * 2);
        c->have_shading = (main_shading != nullptr);
        if (c->have_shading)
        {
            upload(c, c->main_shading, main_shading, npix);
            upload(c, c->main_shading_grad, main_shading_grad, npix * 2);
        }
        set_neighbour_tables(c, n_sub, sub_w, sub_h, Mi, ti);
        smvsb::DevBuf<float>& stage_g = c->stage_a;
        smvsb::DevBuf<float>& stage_h = c->stage_b;
        for (int k = 0; k < n_sub; ++k)
        {
            smvsb::SubViewDev& sv = c->subs[k];
            size_t const n = static_cast<size_t>(sv.w) * sv.h;
            upload(c, stage_g, sub_grad[k], n * 2);
            upload(c, stage_h, sub_hess[k], n * 3);
            smvsb::launch_pack_subview(c, stage_g.p, stage_h.p, sv.texels.p,
                sv.w, sv.h);
        }
        CUDA_CHECK(cudaStreamSynchronize(c->stream));   /* staging buffers */
        c->have_views = true;
        c->have_system = false;
    });
}

int
smvsb_set_views_u8 (smvsb_ctx* ctx, int scale, int w, int h, double flen_px,
    double inv_flen, const uint8_t* main_img, int with_shading, int n_sub,
    const int* sub_w, const int* sub_h, const uint8_t* const* sub_img,
    const double* Mi, const double* ti)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(w > 2 && h > 2 && main_img != nullptr, SMVSB_ERR_INVALID,
            "main view missing");
        require(scale >= 0 && scale <= 8, SMVSB_ERR_INVALID,
            "scale out of range");
        require(n_sub >= 0 && n_sub <= SMVSB_MAX_SUBS, SMVSB_ERR_INVALID,
            "n_sub out of range (max 32)");
        require(n_sub == 0 || (sub_w && sub_h && sub_img && Mi && ti),
            SMVSB_ERR_INVALID, "neighbour arrays missing");
        size_t max_pix = static_cast<size_t>(w) * h;
        for (int k = 0; k < n_sub; ++k)
        {
            require(sub_w[k] > 2 && sub_h[k] > 2 && sub_img[k],
                SMVSB_ERR_INVALID, "neighbour image missing");
            max_pix = std::max(max_pix, static_cast<size_t>(sub_w[k])
                * sub_h[k]);
        }
        smvsb_ctx* c = ctx;
        forget_stale_views(c, w, h, n_sub, sub_w, sub_h);
        c->w = w; c->h = h; c->flen = flen_px; c->inv_flen = inv_flen;
        set_neighbour_tables(c, n_sub, sub_w, sub_h, Mi, ti);
        c->stage_u8.reserve(max_pix);
        c->stage_u8b.reserve(max_pix);
        smvsb::reserve_set_scale_scratch(c, smvsb::DevImage::U8, max_pix);
        size_t const npix = static_cast<size_t>(w) * h;
        c->main_grad.reserve(npix * 2);
        /* Image k travels on the copy stream into staging buffer k mod 2
         * while set_scale of image k - 1 runs on the context's stream; from
         * page-locked host memory the copies are asynchronous, so the PCIe
         * transfers and the kernels overlap (from pageable memory the same
         * calls simply serialise). Whatever the context's stream still has
         * queued may read the staging buffers: the first copies wait for it. */
        uint8_t* const stage[2] = { c->stage_u8.p, c->stage_u8b.p };
        CUDA_CHECK(cudaEventRecord(c->ev_consumed[0], c->stream));
        CUDA_CHECK(cudaEventRecord(c->ev_consumed[1], c->stream));
        auto stage_image = [&](int k, uint8_t const* img, size_t n) {
            int const slot = k & 1;
            CUDA_CHECK(cudaStreamWaitEvent(c->copy_stream,
                c->ev_consumed[slot], 0));
            CUDA_CHECK(cudaMemcpyAsync(stage[slot], img, n,
                cudaMemcpyHostToDevice, c->copy_stream));
            CUDA_CHECK(cudaEventRecord(c->ev_copied[slot], c->copy_stream));
        };
        auto acquire = [&](int k) -> uint8_t const* {
            CUDA_CHECK(cudaStreamWaitEvent(c->stream, c->ev_copied[k & 1], 0));
            return stage[k & 1];
        };
        auto release = [&](int k) {
            CUDA_CHECK(cudaEventRecord(c->ev_consumed[k & 1], c->stream));
        };
        stage_image(0, main_img, npix);
        if (n_sub > 0)
            stage_image(1, sub_img[0], static_cast<size_t>(sub_w[0]) * sub_h[0]);
        {
            uint8_t const* src = acquire(0);
            smvsb::device_set_scale(c, { smvsb::DevImage::U8, src, w, h },
                scale, 0, c->main_grad.p, nullptr);
            c->have_shading = (with_shading != 0);
            if (c->have_shading)
            {
                c->main_shading.reserve(npix);
                c->main_shading_grad.reserve(npix * 2);
                smvsb::device_shading_inputs(c, src, w, h,
                    c->main_shading.p, c->main_shading_grad.p);
            }
            release(0);
        }
        for (int k = 0; k < n_sub; ++k)
        {
            smvsb::SubViewDev& sv = c->subs[k];
            if (k + 1 < n_sub)
                stage_image(k + 2, sub_img[k + 1],
                    static_cast<size_t>(sub_w[k + 1]) * sub_h[k + 1]);
            uint8_t const* src = acquire(k + 1);
            smvsb::device_set_scale(c, { smvsb::DevImage::U8, src, sv.w,
                sv.h }, scale, 1, sv.texels.p, nullptr);
            release(k + 1);
        }
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
        c->have_views = true;
        c->have_system = false;
    });
}

int
smvsb_debug_get_view (smvsb_ctx* ctx, int view, float* grad, float* hess)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(c->have_views && grad != nullptr, SMVSB_ERR_STATE,
            "views not set");
        require(view >= 0 && view <= c->n_sub, SMVSB_ERR_INVALID,
            "view index out of range");
        if (view == 0)
        {
            download(c, grad, c->main_grad.p,
                static_cast<size_t>(c->w) * c->h * 2);
            return;
        }
        require(hess != nullptr, SMVSB_ERR_INVALID, "hess missing");
        smvsb::SubViewDev& sv = c->subs[view - 1];
        size_t const n = static_cast<size_t>(sv.w) * sv.h;
        smvsb::DevBuf<float> g, hs;
        g.reserve(n * 2); hs.reserve(n * 3);
        smvsb::device_unpack_texels(c, sv.texels.p, static_cast<int>(n), g.p,
            hs.p);
        download(c, grad, g.p, n * 2);
        download(c, hess, hs.p, n * 3);
    });
}

int
smvsb_view_set_scale_c (smvsb_ctx* ctx, int w, int h, int channels,
    const float* image, int scale, float* scaleimage, float* grad,
    float* hess)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(w >= 3 && h >= 3 && image != nullptr, SMVSB_ERR_INVALID,
            "image missing or smaller than 3x3");
        require(channels == 1 || channels == 3, SMVSB_ERR_INVALID,
            "1 or 3 channels");
        require(scale >= 0 && scale <= 8, SMVSB_ERR_INVALID,
            "scale out of range");
        size_t const n = static_cast<size_t>(w) * h;
        size_t const nc = n * channels;
        c->view_in.reserve(nc);
        c->view_texels.reserve(n * SMVSB_NB_STRIDE);
        c->view_out.reserve(n * 5);
        CUDA_CHECK(cudaMemcpyAsync(c->view_in.p, image, nc * sizeof(float),
            cudaMemcpyHostToDevice, c->stream));
        /* the blurred image passes through view_out before the gradient and
         * Hessian are unpacked into it */
        smvsb::device_set_scale(c, { channels == 1 ? smvsb::DevImage::F32
            : smvsb::DevImage::RGB_F32, c->view_in.p, w, h }, scale, 1,
            c->view_texels.p, (scaleimage != nullptr) ? c->view_out.p
            : nullptr);
        if (scaleimage != nullptr)
            CUDA_CHECK(cudaMemcpyAsync(scaleimage, c->view_out.p,
                nc * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        if (grad != nullptr || hess != nullptr)
        {
            smvsb::device_unpack_texels(c, c->view_texels.p,
                static_cast<int>(n), c->view_out.p, c->view_out.p + 2 * n);
            if (grad != nullptr)
                CUDA_CHECK(cudaMemcpyAsync(grad, c->view_out.p,
                    2 * n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
            if (hess != nullptr)
                CUDA_CHECK(cudaMemcpyAsync(hess, c->view_out.p + 2 * n,
                    3 * n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        }
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}

int
smvsb_view_set_scale (smvsb_ctx* ctx, int w, int h, const float* image,
    int scale, float* scaleimage, float* grad, float* hess)
{
    return smvsb_view_set_scale_c(ctx, w, h, 1, image, scale, scaleimage,
        grad, hess);
}

int
smvsb_bilateral_filter (smvsb_ctx* ctx, int w, int h, int channels,
    const float* guide, int dm_w, int dm_h, const float* depth, float sigma,
    int kernel_size, float* out)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(w > 0 && h > 0 && dm_w > 0 && dm_h > 0 && guide && depth
            && out, SMVSB_ERR_INVALID, "bilateral filter: image missing");
        size_t const n = static_cast<size_t>(w) * h;
        size_t const nd = static_cast<size_t>(dm_w) * dm_h;
        c->view_texels.reserve(n * channels);
        c->view_in.reserve(nd);
        c->view_out.reserve(n);
        CUDA_CHECK(cudaMemcpyAsync(c->view_texels.p, guide,
            n * channels * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaMemcpyAsync(c->view_in.p, depth, nd * sizeof(float),
            cudaMemcpyHostToDevice, c->stream));
        smvsb::device_bilateral_filter(c, c->view_texels.p, w, h, channels,
            c->view_in.p, dm_w, dm_h, sigma, kernel_size, c->view_out.p);
        download(c, out, c->view_out.p, n);
    });
}

float
smvsb_debug_expf (float x)
{
    return smvsb::host_expf_like_glibc(x);
}

int
smvsb_set_surface (smvsb_ctx* ctx, int scale, int npx, int npy, int start_x,
    int start_y, const double* nodes, const uint8_t* node_valid,
    const uint8_t* patch_valid, const uint32_t* vis_off,
    const uint8_t* vis_ids)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_views, SMVSB_ERR_STATE,
            "smvsb_set_views must precede smvsb_set_surface");
        require_surface_scale(scale);
        require(npx > 0 && npy > 0, SMVSB_ERR_INVALID, "empty patch grid");
        require(nodes && node_valid && patch_valid, SMVSB_ERR_INVALID,
            "surface arrays missing");
        require((vis_off == nullptr) == (vis_ids == nullptr),
            SMVSB_ERR_INVALID, "vis_off and vis_ids go together");
        smvsb_ctx* c = ctx;
        /* a call that fails leaves the context without a surface */
        c->have_surface = false;
        configure_grid(c, scale, npx, npy, start_x, start_y);
        /* the node and validity arrays travel while the host checks the
         * lists (asynchronous from page-locked buffers) */
        upload(c, c->nodes, nodes, static_cast<size_t>(c->n_nodes) * 4);
        upload(c, c->node_valid, node_valid, c->n_nodes);
        upload(c, c->patch_valid, patch_valid, c->n_patches);
        /* no lists: nothing visible yet (smvsb_visibility fills them) */
        std::vector<uint32_t> no_off;
        uint8_t const no_id = 0;
        if (vis_off == nullptr)
        {
            no_off.assign(static_cast<size_t>(c->n_patches) + 1, 0);
            vis_off = no_off.data();
            vis_ids = &no_id;
        }
        /* the kernels fill a fixed array of SMVSB_MAX_SUBS rows per patch
         * from these lists: offsets must start at 0 and be monotone, a list
         * holds each neighbour at most once. The lists are checked where
         * they land (one thread per patch; 0.5 ms on a host core at 2 MP). */
        require(vis_off[0] == 0, SMVSB_ERR_INVALID, "vis_off[0] must be 0");
        {
            /* the offsets on the host (they bound what is read of vis_ids) */
            uint32_t const n_sub = static_cast<uint32_t>(c->n_sub);
            unsigned int bad_order = 0, bad_len = 0;
            for (int p = 0; p < c->n_patches; ++p)
            {
                bad_order |= vis_off[p] > vis_off[p + 1];
                bad_len |= (vis_off[p + 1] - vis_off[p]) > n_sub;
            }
            require(!bad_order, SMVSB_ERR_INVALID, "vis_off must be monotone");
            require(!bad_len, SMVSB_ERR_INVALID,
                "visibility list longer than the number of neighbours");
        }
        size_t const total_vis = vis_off[c->n_patches];
        upload(c, c->vis_off, vis_off, static_cast<size_t>(c->n_patches) + 1);
        upload(c, c->vis_ids, vis_ids, std::max<size_t>(total_vis, 1));
        c->counters.reserve(8);
        CUDA_CHECK(cudaMemsetAsync(c->counters.p, 0, sizeof(unsigned long long),
            c->stream));
        vis_validate_kernel<<<(c->n_patches + 255) / 256, 256, 0, c->stream>>>(
            c->n_patches, c->n_sub, static_cast<uint32_t>(total_vis),
            c->vis_off.p, c->vis_ids.p, c->counters.p);
        smvsb::count_launches(c, 1);
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(&c->pinned->vis_flags, c->counters.p,
            sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
        c->h_node_valid.assign(node_valid, node_valid + c->n_nodes);
        c->h_patch_valid.assign(patch_valid, patch_valid + c->n_patches);
        set_active(c, nullptr);
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
        unsigned long long const bad = c->pinned->vis_flags;
        require(!(bad & 1u), SMVSB_ERR_INVALID, "vis_off must be monotone");
        require(!(bad & 2u), SMVSB_ERR_INVALID,
            "visibility list longer than the number of neighbours");
        require(!(bad & 4u), SMVSB_ERR_INVALID, "visibility id out of range");
        require(!(bad & 8u), SMVSB_ERR_INVALID,
            "duplicate neighbour in a visibility list");
        c->have_surface = true;
        c->have_system = false;
        c->x_count = 0;
    });
}

int
smvsb_set_nodes (smvsb_ctx* ctx, const double* nodes)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface, SMVSB_ERR_STATE, "no surface set");
        require(nodes != nullptr, SMVSB_ERR_INVALID, "nodes missing");
        upload(ctx, ctx->nodes, nodes, static_cast<size_t>(ctx->n_nodes) * 4);
        CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        ctx->have_system = false;
    });
}

int
smvsb_gn_construct (smvsb_ctx* ctx, const uint8_t* active_nodes,
    const double* light16, double regularization,
    double light_surf_regularization)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_views && ctx->have_surface, SMVSB_ERR_STATE,
            "views / surface not set");
        set_active(ctx, active_nodes);
        construct(ctx, light16, regularization, light_surf_regularization);
        CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    });
}

int
smvsb_cg_solve (smvsb_ctx* ctx, int max_iter, double err_tol, double q_tol,
    int* iters, int* info)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_system, SMVSB_ERR_STATE,
            "smvsb_gn_construct must precede smvsb_cg_solve");
        smvsb::run_cg(ctx, max_iter, err_tol, q_tol, iters, info, nullptr);
        ctx->x_count = static_cast<size_t>(ctx->n_nodes) * 4;
    });
}

int
smvsb_get_delta (smvsb_ctx* ctx, double* delta)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_system && delta, SMVSB_ERR_STATE, "no solution");
        download(ctx, delta, ctx->x.p, static_cast<size_t>(ctx->n_nodes) * 4);
    });
}

int
smvsb_set_delta (smvsb_ctx* ctx, const double* delta)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface && delta, SMVSB_ERR_STATE, "no surface");
        upload(ctx, ctx->x, delta, static_cast<size_t>(ctx->n_nodes) * 4);
        CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        ctx->x_count = static_cast<size_t>(ctx->n_nodes) * 4;
    });
}

int
smvsb_update_nodes (smvsb_ctx* ctx, double reproj_thresh, int full_opt,
    uint8_t* active_out, uint64_t* n_active, double* mean_shift)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface && ctx->x.p != nullptr
            && ctx->x_count == static_cast<size_t>(ctx->n_nodes) * 4,
            SMVSB_ERR_STATE, "no delta for this surface (solve or "
            "smvsb_set_delta after the last smvsb_set_surface)");
        smvsb::launch_update(ctx, reproj_thresh, full_opt != 0, n_active,
            mean_shift);
        if (active_out)
            download(ctx, active_out, ctx->active.p, ctx->n_nodes);
        ctx->have_system = false;
    });
}

/*
 * The inner loop of DepthOptimizer::run_newton_iterations
 * (lib/depth_optimizer.cc:204-304) for n views in lock-step; n = 1 is
 * smvsb_newton_loop. All launches go to the lead context's stream.
 */
static void
newton_loop_batch (smvsb_ctx* const* cs, int n, double const* const* light16,
    double regularization, double light_surf_regularization, int max_steps,
    int full_opt, smvsb_newton_stats* stats)
{
    smvsb_ctx* lead = cs[0];
    /* every context of the batch works on the lead's stream for the duration
     * of the call (its own stream is idle: all entry points synchronise) */
    struct StreamSwap
    {
        smvsb_ctx* const* cs; int n; cudaStream_t saved[SMVSB_MAX_BATCH];
        StreamSwap (smvsb_ctx* const* c, int k) : cs(c), n(k)
        {
            for (int i = 0; i < n; ++i)
            {
                saved[i] = cs[i]->stream;
                cs[i]->stream = cs[0]->stream;
            }
        }
        ~StreamSwap (void)
        {
            for (int i = n - 1; i >= 0; --i)
                cs[i]->stream = saved[i];
        }
    } swap(cs, n);

    smvsb_newton_stats st[SMVSB_MAX_BATCH];
    uint64_t num_initial[SMVSB_MAX_BATCH], num_active[SMVSB_MAX_BATCH];
    bool running[SMVSB_MAX_BATCH];
    for (int k = 0; k < n; ++k)
    {
        smvsb_ctx* c = cs[k];
        std::memset(&st[k], 0, sizeof(st[k]));
        /* lib/depth_optimizer.cc:203-213 */
        set_active(c, nullptr);
        num_initial[k] = 0;
        for (uint8_t v : c->h_node_valid) num_initial[k] += (v != 0);
        num_active[k] = num_initial[k];
        running[k] = true;
    }

    float ms = 0.f;
    double ms_construct = 0, ms_solve = 0, ms_update = 0;
    cudaEvent_t const ev_begin = lead->ev[4], ev_end = lead->ev[5];
    CUDA_CHECK(cudaEventRecord(ev_begin, lead->stream));
    for (;;)
    {
        /* lib/depth_optimizer.cc:219: the views whose loop goes on */
        smvsb_ctx* act[SMVSB_MAX_BATCH];
        int idx[SMVSB_MAX_BATCH];
        int m = 0;
        for (int k = 0; k < n; ++k)
        {
            running[k] = running[k] && st[k].newton_steps < max_steps
                && num_active[k] > num_initial[k] / 20;
            if (running[k])
            {
                act[m] = cs[k];
                idx[m] = k;
                m += 1;
            }
        }
        if (m == 0)
            break;

        CUDA_CHECK(cudaEventRecord(lead->ev[0], lead->stream));
        for (int j = 0; j < m; ++j)
        {
            st[idx[j]].newton_steps += 1;
            smvsb::count_processed_enqueue(act[j]);
            construct(act[j], light16 ? light16[idx[j]] : nullptr,
                regularization, light_surf_regularization);
        }
        CUDA_CHECK(cudaEventRecord(lead->ev[1], lead->stream));
        smvsb::cg_enqueue(act, m, 200, -1.0, 1e-3);
        CUDA_CHECK(cudaEventRecord(lead->ev[2], lead->stream));
        CUDA_CHECK(cudaStreamSynchronize(lead->stream));

        int n_update = 0;
        for (int j = 0; j < m; ++j)
        {
            smvsb_ctx* c = act[j];
            smvsb_newton_stats& s = st[idx[j]];
            double const samples = double(c->npos) * c->npos;
            s.pixel_iterations += samples
                * double(smvsb::count_processed_collect(c));
            int iters = 0, info = 0;
            bool x0_nan = false;
            smvsb::cg_collect(c, &iters, &info, &x0_nan);
            c->x_count = static_cast<size_t>(c->n_nodes) * 4;
            s.cg_iterations += iters;
            s.cg_block_iterations += double(c->cg_blocks) * iters;
            s.cg_row_iterations += double(c->cg_rows) * iters;
            if (x0_nan)     /* lib/depth_optimizer.cc:267 */
            {
                s.nan_break = 1;
                running[idx[j]] = false;
                continue;
            }
            smvsb::update_enqueue(c, 0.15, full_opt != 0);
            n_update += 1;
        }
        CUDA_CHECK(cudaEventRecord(lead->ev[3], lead->stream));
        CUDA_CHECK(cudaEventSynchronize(lead->ev[3]));
        CUDA_CHECK(cudaEventElapsedTime(&ms, lead->ev[0], lead->ev[1]));
        ms_construct += ms;
        CUDA_CHECK(cudaEventElapsedTime(&ms, lead->ev[1], lead->ev[2]));
        ms_solve += ms;
        CUDA_CHECK(cudaEventElapsedTime(&ms, lead->ev[2], lead->ev[3]));
        ms_update += ms;
        for (int j = 0; j < m; ++j)
        {
            int const k = idx[j];
            if (!running[k])
                continue;
            double mean_shift = 0.0;
            smvsb::update_collect(act[j], &num_active[k], &mean_shift);
            /* lib/depth_optimizer.cc:275-289 */
            if (full_opt && mean_shift < 0.01)
                running[k] = false;
        }
    }
    CUDA_CHECK(cudaEventRecord(ev_end, lead->stream));
    CUDA_CHECK(cudaEventSynchronize(ev_end));
    CUDA_CHECK(cudaEventElapsedTime(&ms, ev_begin, ev_end));
    for (int k = 0; k < n; ++k)
    {
        st[k].ms_construct = ms_construct;
        st[k].ms_solve = ms_solve;
        st[k].ms_update = ms_update;
        st[k].ms_total = ms;
        st[k].n_active = num_active[k];
        cs[k]->have_system = false;
        if (stats) stats[k] = st[k];
    }
}

int
smvsb_newton_loop (smvsb_ctx* ctx, const double* light16,
    double regularization, double light_surf_regularization, int max_steps,
    int full_opt, smvsb_newton_stats* stats)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_views && ctx->have_surface, SMVSB_ERR_STATE,
            "views / surface not set");
        smvsb_ctx* cs[1] = { ctx };
        double const* lights[1] = { light16 };
        newton_loop_batch(cs, 1, lights, regularization,
            light_surf_regularization, max_steps, full_opt, stats);
    });
}

int
smvsb_newton_loop_batch (smvsb_ctx* const* ctxs, int n,
    const double* const* light16, double regularization,
    double light_surf_regularization, int max_steps, int full_opt,
    smvsb_newton_stats* stats)
{
    if (ctxs == nullptr || n < 1 || ctxs[0] == nullptr)
        return SMVSB_ERR_INVALID;
    return guarded(ctxs[0], [&]() {
        require(n <= SMVSB_MAX_BATCH, SMVSB_ERR_INVALID,
            "batch larger than SMVSB_MAX_BATCH");
        for (int k = 0; k < n; ++k)
        {
            require(ctxs[k] != nullptr, SMVSB_ERR_INVALID, "NULL context");
            require(ctxs[k]->device == ctxs[0]->device, SMVSB_ERR_INVALID,
                "the contexts of a batch must live on one device");
            for (int j = 0; j < k; ++j)
                require(ctxs[j] != ctxs[k], SMVSB_ERR_INVALID,
                    "a context appears twice in the batch");
            require(ctxs[k]->have_views && ctxs[k]->have_surface,
                SMVSB_ERR_STATE, "views / surface not set");
            if (light16 != nullptr && light16[k] != nullptr)
                require(ctxs[k]->have_shading, SMVSB_ERR_STATE,
                    "lighting given but the main view has no shading image");
            /* pending work of the context's own stream */
            CUDA_CHECK(cudaStreamSynchronize(ctxs[k]->stream));
        }
        newton_loop_batch(ctxs, n, light16, regularization,
            light_surf_regularization, max_steps, full_opt, stats);
    });
}


/* ---- surface topology on the device (topology.cu) ------------------- */

int
smvsb_surface_create (smvsb_ctx* ctx, int scale, const float* init_depth)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(c->have_views, SMVSB_ERR_STATE,
            "smvsb_set_views must precede smvsb_surface_create");
        require(init_depth != nullptr, SMVSB_ERR_INVALID,
            "init depth missing (the bundle-based initialisation of "
            "lib/surface.cc:54-139 is host code)");
        size_t const npix = static_cast<size_t>(c->w) * c->h;
        c->image_out.reserve(npix * 3);
        CUDA_CHECK(cudaMemcpyAsync(c->image_out.p, init_depth,
            npix * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        surface_create_device(c, scale, c->image_out.p);
    });
}

int
smvsb_surface_subdivide (smvsb_ctx* ctx)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface, SMVSB_ERR_STATE, "no surface set");
        surface_subdivide_device(ctx);
    });
}

int
smvsb_surface_fill_from_depth (smvsb_ctx* ctx, const float* init_depth)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(c->have_surface, SMVSB_ERR_STATE, "no surface set");
        size_t const npix = static_cast<size_t>(c->w) * c->h;
        if (init_depth != nullptr)
        {
            c->image_out.reserve(npix * 3);
            CUDA_CHECK(cudaMemcpyAsync(c->image_out.p, init_depth,
                npix * sizeof(float), cudaMemcpyHostToDevice, c->stream));
            smvsb::topo_set_init_depth(c, c->image_out.p);
        }
        require(c->init_depth.p != nullptr && c->init_depth.cap >= npix,
            SMVSB_ERR_STATE, "no init depth on the device");
        smvsb::topo_fill_from_depth(c);
        refresh_validity(c);
    });
}

int
smvsb_surface_remove_isolated (smvsb_ctx* ctx)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface, SMVSB_ERR_STATE, "no surface set");
        smvsb::topo_remove_isolated(ctx);
        refresh_validity(ctx);
    });
}

int
smvsb_surface_expand (smvsb_ctx* ctx, int* filled_out)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface, SMVSB_ERR_STATE, "no surface set");
        uint64_t const filled = smvsb::topo_expand(ctx);
        if (filled_out)
            *filled_out = static_cast<int>(filled);
        refresh_validity(ctx);
    });
}

int
smvsb_surface_info (smvsb_ctx* ctx, int* info6)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface && info6, SMVSB_ERR_STATE, "no surface set");
        info6[0] = ctx->scale; info6[1] = ctx->npx; info6[2] = ctx->npy;
        info6[3] = ctx->start_x; info6[4] = ctx->start_y; info6[5] = ctx->ps;
    });
}

/*
 * DepthOptimizer::optimize() (lib/depth_optimizer.cc:54-162) with
 * run_newton_iterations (:164-358) for the use_sgm mode, the whole view
 * resident on the device from the SGM initialisation to the depth and normal
 * maps.
 */
/* The body of smvsb_optimize / smvsb_optimize_f32. colour: the images are
 * three-channel float images (StereoView::get_image() of a colour view),
 * otherwise single-channel bytes. */
static int
optimize_resident (smvsb_ctx* ctx, int w, int h, double flen_px,
    double inv_flen, const float* inv_calib9, bool colour,
    const void* main_img, int n_sub, const int* sub_w, const int* sub_h,
    const void* const* sub_img, const double* Mi, const double* ti,
    const float* shading, const float* shading_grad, int sgm_w, int sgm_h,
    const float* sgm_depth, const smvsb_optimize_options* opts,
    float* depth_out, float* normals_out, double* light16_out,
    smvsb_optimize_stats* stats_out)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(w > 2 && h > 2 && main_img && inv_calib9 && opts
            && sgm_depth && sgm_w > 0 && sgm_h > 0, SMVSB_ERR_INVALID,
            "smvsb_optimize: main view, options or SGM depth missing");
        require(n_sub >= 1 && n_sub <= SMVSB_MAX_SUBS && sub_w && sub_h
            && sub_img && Mi && ti, SMVSB_ERR_INVALID,
            "smvsb_optimize: neighbour arrays missing");
        require((shading == nullptr) == (shading_grad == nullptr),
            SMVSB_ERR_INVALID, "shading image and gradient go together");
        require(!opts->use_shading || shading != nullptr, SMVSB_ERR_INVALID,
            "use_shading needs the shading image");
        require(opts->num_iterations >= 1 && opts->min_scale >= 0,
            SMVSB_ERR_INVALID, "bad iteration count / min_scale");
        for (int k = 0; k < n_sub; ++k)
            require(sub_w[k] > 2 && sub_h[k] > 2 && sub_img[k],
                SMVSB_ERR_INVALID, "neighbour image missing");
        smvsb_optimize_stats st;
        std::memset(&st, 0, sizeof(st));

        /* ---- inputs: once per view ------------------------------------ */
        c->w = w; c->h = h; c->flen = flen_px; c->inv_flen = inv_flen;
        /* the surface and the colour images are made anew, whatever the
         * geometry of the views */
        c->have_surface = false;
        c->have_color = false;
        set_neighbour_tables(c, n_sub, sub_w, sub_h, Mi, ti);
        size_t const npix = static_cast<size_t>(w) * h;
        if (colour)
        {
            upload_color_images(c, static_cast<float const*>(main_img),
                reinterpret_cast<float const* const*>(sub_img));
            c->have_color = true;
        }
        else
        {
            upload(c, c->u8_main, static_cast<uint8_t const*>(main_img), npix);
            for (int k = 0; k < n_sub; ++k)
                upload(c, c->u8_subs[k],
                    static_cast<uint8_t const*>(sub_img[k]),
                    static_cast<size_t>(sub_w[k]) * sub_h[k]);
        }
        c->have_shading = (shading != nullptr);
        if (c->have_shading)
        {
            upload(c, c->main_shading, shading, npix);
            upload(c, c->main_shading_grad, shading_grad, npix * 2);
        }
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
        c->have_views = true;

        /* ---- create_initial_surface, :35-52 --------------------------- */
        bool const no_sgm = (opts->no_sgm != 0);
        require(!no_sgm || colour, SMVSB_ERR_INVALID,
            "no_sgm needs three-channel views (the NCC filter, "
            "lib/depth_optimizer.cc:795-912, reads channels 0..2)");
        require(!no_sgm || (sgm_w == w && sgm_h == h), SMVSB_ERR_INVALID,
            "no_sgm: the initial depth must have the size of the main view");
        int const init_scale = static_cast<int>(std::max(std::ceil(std::log2(
            w * h / 1.7e6) / 2) + 4, 4.0)) + (no_sgm ? 1 : 0);   /* :37-38, :51 */
        require(init_scale <= SMVSB_MAX_SCALE, SMVSB_ERR_INVALID,
            "image too large: initial scale above 8");
        if (no_sgm)
        {
            /* the sparse depth of the bundle's features (lib/surface.cc:91-128)
             * as the host projected it */
            c->sgm_depth.reserve(npix);
            CUDA_CHECK(cudaMemcpyAsync(c->sgm_depth.p, sgm_depth,
                npix * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        }
        else
        {
            /* depthmap_bilateral_filter(sgm depth, main image), :42 */
            size_t const nd = static_cast<size_t>(sgm_w) * sgm_h;
            float const* guide = c->color_main.p;
            if (!colour)
            {
                c->guide.reserve(npix);
                smvsb::device_byte_to_float(c, c->u8_main.p, npix, c->guide.p);
                guide = c->guide.p;
            }
            c->view_in.reserve(nd);
            CUDA_CHECK(cudaMemcpyAsync(c->view_in.p, sgm_depth,
                nd * sizeof(float), cudaMemcpyHostToDevice, c->stream));
            c->sgm_depth.reserve(npix);
            smvsb::device_bilateral_filter(c, guide, w, h, colour ? 3 : 1,
                c->view_in.p, sgm_w, sgm_h, 5.0f, 5, c->sgm_depth.p);
        }
        surface_create_device(c, init_scale, c->sgm_depth.p);
        views_from_resident(c, c->scale, colour);

        bool have_light = false;
        double light[16];
        /* cut_boundaries until it deletes at most 10 patches */
        auto cut_until_settled = [&]()
        {
            for (uint64_t del = ~0ull; del > 10;)
            {
                del = smvsb::run_cut_boundaries(c, inv_calib9);
                refresh_validity(c);
            }
        };
        auto run_newton_iterations = [&]()
        {
            bool finished = false;
            for (int iter = 0; iter < opts->num_iterations; ++iter)
            {
                uint64_t const num_valid = smvsb::topo_count_patches(c);
                if (iter == 0)
                {
                    /* :189-195 */
                    if (no_sgm)
                        smvsb::run_visibility_ncc(c);
                    else
                        smvsb::run_visibility_device(c);
                    refresh_validity(c);
                    cut_until_settled();
                }
                smvsb_newton_stats ns;
                smvsb_ctx* cs[1] = { c };
                double const* lights[1] = { have_light ? light : nullptr };
                newton_loop_batch(cs, 1, lights, opts->regularization,
                    opts->light_surf_regularization, 200,
                    opts->full_optimization, &ns);
                st.newton_loops += 1;
                st.newton_steps += ns.newton_steps;
                st.cg_iterations += ns.cg_iterations;
                st.pixel_iterations += ns.pixel_iterations;
                st.ms_newton += ns.ms_total;
                if (finished)
                    break;
                /* :322-356 */
                cut_until_settled();
                if (no_sgm)
                {
                    /* :331-339: grow the surface by a ring of patches, see
                     * which neighbours see them, cut again */
                    smvsb::topo_expand(c);
                    refresh_validity(c);
                    smvsb::run_visibility_ncc(c);
                    refresh_validity(c);
                    cut_until_settled();
                }
                smvsb::topo_remove_isolated(c);
                refresh_validity(c);
                uint64_t const num_new = smvsb::topo_count_patches(c);
                double const change = 1.0 - static_cast<double>(
                    std::min(num_new, num_valid)) / static_cast<double>(
                    std::max(num_new, num_valid));
                if (iter > 0 && (num_new <= num_valid
                    || change < 0.05 * c->scale))
                    finished = true;
            }
        };

        run_newton_iterations();
        st.scales = 1;
        while (c->scale > opts->min_scale && c->scale > 0)
        {
            surface_subdivide_device(c);                     /* :90 */
            views_from_resident(c, c->scale, colour);             /* :91-95 */
            smvsb::topo_fill_from_depth(c);                  /* :99 */
            refresh_validity(c);
            if (opts->use_shading && c->scale < 4)           /* :102-109 */
            {
                double Ab[272];
                smvsb::run_fit_lighting(c, Ab);
                lighting_from_normal_equations(Ab, light);
                have_light = true;
            }
            run_newton_iterations();
            st.scales += 1;
        }

        /* ---- outputs, :158-161 ---------------------------------------- */
        c->image_out.reserve(npix * 3);
        if (depth_out != nullptr)
        {
            smvsb::launch_render_depth(c, c->image_out.p);
            download(c, depth_out, c->image_out.p, npix);
        }
        if (normals_out != nullptr)
        {
            smvsb::launch_render_normals(c, c->image_out.p);
            download(c, normals_out, c->image_out.p, npix * 3);
        }
        if (light16_out != nullptr)
            for (int i = 0; i < 16; ++i)
                light16_out[i] = have_light ? light[i] : 0.0;
        st.final_scale = c->scale;
        st.patches = smvsb::topo_count_patches(c);
        if (stats_out) *stats_out = st;
    });
}

int
smvsb_optimize (smvsb_ctx* ctx, int w, int h, double flen_px, double inv_flen,
    const float* inv_calib9, const uint8_t* main_img, int n_sub,
    const int* sub_w, const int* sub_h, const uint8_t* const* sub_img,
    const double* Mi, const double* ti, const float* shading,
    const float* shading_grad, int sgm_w, int sgm_h, const float* sgm_depth,
    const smvsb_optimize_options* opts, float* depth_out, float* normals_out,
    double* light16_out, smvsb_optimize_stats* stats_out)
{
    return optimize_resident(ctx, w, h, flen_px, inv_flen, inv_calib9, false,
        main_img, n_sub, sub_w, sub_h,
        reinterpret_cast<const void* const*>(sub_img), Mi, ti, shading,
        shading_grad, sgm_w, sgm_h, sgm_depth, opts, depth_out, normals_out,
        light16_out, stats_out);
}

int
smvsb_optimize_rgb_f32 (smvsb_ctx* ctx, int w, int h, double flen_px,
    double inv_flen, const float* inv_calib9, const float* main_rgb,
    int n_sub, const int* sub_w, const int* sub_h,
    const float* const* sub_rgb, const double* Mi, const double* ti,
    const float* shading, const float* shading_grad, int sgm_w, int sgm_h,
    const float* sgm_depth, const smvsb_optimize_options* opts,
    float* depth_out, float* normals_out, double* light16_out,
    smvsb_optimize_stats* stats_out)
{
    return optimize_resident(ctx, w, h, flen_px, inv_flen, inv_calib9, true,
        main_rgb, n_sub, sub_w, sub_h,
        reinterpret_cast<const void* const*>(sub_rgb), Mi, ti, shading,
        shading_grad, sgm_w, sgm_h, sgm_depth, opts, depth_out, normals_out,
        light16_out, stats_out);
}

int
smvsb_get_nodes (smvsb_ctx* ctx, double* nodes_out)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface && nodes_out, SMVSB_ERR_STATE,
            "no surface set");
        download(ctx, nodes_out, ctx->nodes.p,
            static_cast<size_t>(ctx->n_nodes) * 4);
    });
}

int
smvsb_visibility (smvsb_ctx* ctx, const float* sgm_depth,
    uint64_t* removed_patches)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_views && ctx->have_surface, SMVSB_ERR_STATE,
            "views / surface not set");
        require(ctx->n_sub <= 32, SMVSB_ERR_INVALID,
            "more than 32 neighbours");
        require(sgm_depth != nullptr || ctx->have_color, SMVSB_ERR_STATE,
            "sgm_depth is NULL (use_sgm = false) but no colour images are "
            "set: call smvsb_set_color_images first");
        uint64_t const removed = (sgm_depth != nullptr)
            ? smvsb::run_visibility(ctx, sgm_depth)
            : smvsb::run_visibility_ncc(ctx);
        refresh_validity(ctx);
        if (removed_patches) *removed_patches = removed;
    });
}

int
smvsb_set_color_images (smvsb_ctx* ctx, const float* main_rgb, int n_sub,
    const float* const* sub_rgb)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_views, SMVSB_ERR_STATE, "views not set");
        require(main_rgb != nullptr && sub_rgb != nullptr
            && n_sub == ctx->n_sub, SMVSB_ERR_INVALID,
            "colour images: one per view of the context");
        for (int k = 0; k < n_sub; ++k)
            require(sub_rgb[k] != nullptr, SMVSB_ERR_INVALID,
                "colour image missing");
        upload_color_images(ctx, main_rgb, sub_rgb);
        CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        ctx->have_color = true;
    });
}

int
smvsb_cut_boundaries (smvsb_ctx* ctx, const float* inv_calib9, int* deleted)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_views && ctx->have_surface, SMVSB_ERR_STATE,
            "views / surface not set");
        require(inv_calib9 != nullptr, SMVSB_ERR_INVALID,
            "inverse calibration missing");
        uint64_t const n = smvsb::run_cut_boundaries(ctx, inv_calib9);
        refresh_validity(ctx);
        if (deleted) *deleted = static_cast<int>(n);
    });
}

int
smvsb_get_surface_state (smvsb_ctx* ctx, uint8_t* node_valid,
    uint8_t* patch_valid, uint32_t* vis_off, uint8_t* vis_ids,
    uint64_t vis_capacity)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(c->have_surface, SMVSB_ERR_STATE, "no surface set");
        if (node_valid)
            download(c, node_valid, c->node_valid.p, c->n_nodes);
        if (patch_valid)
            download(c, patch_valid, c->patch_valid.p, c->n_patches);
        std::vector<uint32_t> off(static_cast<size_t>(c->n_patches) + 1);
        download(c, off.data(), c->vis_off.p, off.size());
        if (vis_off)
            std::copy(off.begin(), off.end(), vis_off);
        if (vis_ids)
        {
            require(off.back() <= vis_capacity, SMVSB_ERR_INVALID,
                "vis_ids capacity too small");
            if (off.back() > 0)
                download(c, vis_ids, c->vis_ids.p, off.back());
        }
    });
}

int
smvsb_get_depth (smvsb_ctx* ctx, float* depth_wh)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface && depth_wh, SMVSB_ERR_STATE,
            "no surface set");
        size_t const n = static_cast<size_t>(ctx->w) * ctx->h;
        ctx->image_out.reserve(n * 3);
        smvsb::launch_render_depth(ctx, ctx->image_out.p);
        download(ctx, depth_wh, ctx->image_out.p, n);
    });
}

int
smvsb_get_normals (smvsb_ctx* ctx, float* normals_wh3)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_surface && normals_wh3, SMVSB_ERR_STATE,
            "no surface set");
        size_t const n = static_cast<size_t>(ctx->w) * ctx->h * 3;
        ctx->image_out.reserve(n);
        smvsb::launch_render_normals(ctx, ctx->image_out.p);
        download(ctx, normals_wh3, ctx->image_out.p, n);
    });
}

int
smvsb_debug_get_system (smvsb_ctx* ctx, double* g, double* Hvals,
    uint64_t* Houter, uint64_t* Hinner, uint64_t* nnzb_h, double* Pvals,
    uint64_t* Pouter, uint64_t* Pinner, uint64_t* nnzb_p)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(c->have_system, SMVSB_ERR_STATE, "no system constructed");
        int const nn = c->n_nodes, ns = c->npx + 1;
        std::vector<uint8_t> active(nn), proc(c->n_patches);
        download(c, active.data(), c->active.p, nn);
        download(c, proc.data(), c->patch_proc.p, c->n_patches);
        if (g)
            download(c, g, c->g.p, static_cast<size_t>(nn) * 4);
        std::vector<double> H, P;
        if (Hvals)
        {
            H.resize(static_cast<size_t>(nn) * 144);
            download(c, H.data(), c->H.p, H.size());
        }
        if (Pvals)
        {
            P.resize(static_cast<size_t>(nn) * 16);
            download(c, P.data(), c->P.p, P.size());
        }
        /* A block (row i, col j) exists in the reference iff some processed
         * patch holds both nodes and both are active
         * (lib/gauss_newton_step.cc:99-121). Walk columns, then rows. */
        uint64_t nh = 0, np = 0;
        for (int j = 0; j < nn; ++j)
        {
            if (Houter) Houter[j] = nh;
            if (Pouter) Pouter[j] = np;
            int const jx = j % ns, jy = j / ns;
            if (!c->h_node_valid[j] || !active[j])
                continue;
            for (int dy = -1; dy <= 1; ++dy)
                for (int dx = -1; dx <= 1; ++dx)
                {
                    int const ix = jx + dx, iy = jy + dy;
                    if (ix < 0 || ix > c->npx || iy < 0 || iy > c->npy)
                        continue;
                    int const i = iy * ns + ix;
                    if (!c->h_node_valid[i] || !active[i])
                        continue;
                    bool shared = false;
                    for (int pb = 0; pb < 2 && !shared; ++pb)
                        for (int pa = 0; pa < 2 && !shared; ++pa)
                        {
                            int const px = jx - 1 + pa, py = jy - 1 + pb;
                            if (px < 0 || px >= c->npx || py < 0
                                || py >= c->npy)
                                continue;
                            if (!proc[py * c->npx + px])
                                continue;
                            if (ix >= px && ix <= px + 1 && iy >= py
                                && iy <= py + 1)
                                shared = true;
                        }
                    if (!shared)
                        continue;
                    /* block (row i, col j) is stencil slot of row i towards
                     * j: offset (jx-ix, jy-iy) = (-dx, -dy) */
                    if (Hvals)
                    {
                        int const k = (-dy + 1) * 3 + (-dx + 1);
                        std::copy(H.begin() + (static_cast<size_t>(i) * 9 + k)
                            * 16, H.begin() + (static_cast<size_t>(i) * 9 + k)
                            * 16 + 16, Hvals + nh * 16);
                    }
                    if (Hinner) Hinner[nh] = static_cast<uint64_t>(i) * 4;
                    nh += 1;
                    if (i == j)
                    {
                        if (Pvals)
                            std::copy(P.begin() + static_cast<size_t>(i) * 16,
                                P.begin() + static_cast<size_t>(i) * 16 + 16,
                                Pvals + np * 16);
                        if (Pinner) Pinner[np] = static_cast<uint64_t>(i) * 4;
                        np += 1;
                    }
                }
        }
        if (Houter) Houter[nn] = nh;
        if (Pouter) Pouter[nn] = np;
        if (nnzb_h) *nnzb_h = nh;
        if (nnzb_p) *nnzb_p = np;
    });
}

int
smvsb_debug_spmv (smvsb_ctx* ctx, const double* x, double* y)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        require(ctx->have_system && x && y, SMVSB_ERR_STATE, "no system");
        size_t const n = static_cast<size_t>(ctx->n_nodes) * 4;
        ctx->r.reserve(n); ctx->Ad.reserve(n);
        upload(ctx, ctx->r, x, n);
        smvsb::launch_spmv(ctx, ctx->r.p, ctx->Ad.p);
        download(ctx, y, ctx->Ad.p, n);
    });
}

int
smvsb_fit_lighting (smvsb_ctx* ctx, double* params16_out, void* nccl_comm)
{
    if (ctx == nullptr) return SMVSB_ERR_INVALID;
    return guarded(ctx, [&]() {
        smvsb_ctx* c = ctx;
        require(c->have_surface && c->have_shading && params16_out,
            SMVSB_ERR_STATE, "surface and shading image required");
        double Ab[272];
        smvsb::run_fit_lighting(c, Ab);
        if (nccl_comm != nullptr)
        {
            /* Opt-in global lighting: sum the normal equations over the
             * communicator. ncclAllReduce is taken from the NCCL already
             * loaded in this process (the one that made the communicator). */
            typedef int (*allreduce_fn)(const void*, void*, size_t, int, int,
                void*, cudaStream_t);
            allreduce_fn fn = reinterpret_cast<allreduce_fn>(
                dlsym(RTLD_DEFAULT, "ncclAllReduce"));
            require(fn != nullptr, SMVSB_ERR_STATE,
                "ncclAllReduce not found in this process");
            c->light_partials.reserve(272);
            upload(c, c->light_partials, Ab, 272);
            int const ncclDouble = 8, ncclSum = 0;
            int const rc = fn(c->light_partials.p, c->light_partials.p, 272,
                ncclDouble, ncclSum, nccl_comm, c->stream);
            require(rc == 0, SMVSB_ERR_CUDA, "ncclAllReduce failed");
            download(c, Ab, c->light_partials.p, 272);
        }
        lighting_from_normal_equations(Ab, params16_out);
    });
}

int
smvsb_sgm (int device, int w, int h, const uint8_t* main_lum, int nw, int nh,
    const uint8_t* neigh_lum, const float* M, const float* t,
    float min_depth, float max_depth, int num_steps, uint16_t penalty1,
    uint16_t penalty2, float* depth_out, uint16_t* cost_out,
    uint16_t* sgm_out, double* ms_out)
{
    return smvsb_sgm_ex(device, w, h, main_lum, nw, nh, neigh_lum, M, t,
        min_depth, max_depth, num_steps, penalty1, penalty2, depth_out,
        cost_out, sgm_out, ms_out, nullptr, nullptr);
}

int
smvsb_sgm_ex (int device, int w, int h, const uint8_t* main_lum, int nw,
    int nh, const uint8_t* neigh_lum, const float* M, const float* t,
    float min_depth, float max_depth, int num_steps, uint16_t penalty1,
    uint16_t penalty2, float* depth_out, uint16_t* cost_out,
    uint16_t* sgm_out, double* ms_out, const smvsb_sgm_options* opts,
    smvsb_sgm_stats* stats)
{
    return guarded(nullptr, [&]() {
        smvsb::sgm_run(device, w, h, main_lum, nw, nh, neigh_lum, M, t,
            min_depth, max_depth, num_steps, penalty1, penalty2, depth_out,
            cost_out, sgm_out, ms_out, opts, stats);
    });
}

int
smvsb_sgm_reconstruct (int device, int w, int h, const uint8_t* main_lum,
    int nw, int nh, const uint8_t* neigh_lum, const float* M_mn,
    const float* t_mn, const float* M_nm, const float* t_nm,
    const float* depth_range_main, const float* depth_range_neigh,
    int num_steps, uint16_t penalty1, uint16_t penalty2,
    const float* merge_with, float* depth_out, double* ms_out)
{
    return smvsb_sgm_reconstruct_ex(device, w, h, main_lum, nw, nh,
        neigh_lum, M_mn, t_mn, M_nm, t_nm, depth_range_main,
        depth_range_neigh, num_steps, penalty1, penalty2, merge_with,
        depth_out, ms_out, nullptr, nullptr);
}

int
smvsb_sgm_reconstruct_ex (int device, int w, int h, const uint8_t* main_lum,
    int nw, int nh, const uint8_t* neigh_lum, const float* M_mn,
    const float* t_mn, const float* M_nm, const float* t_nm,
    const float* depth_range_main, const float* depth_range_neigh,
    int num_steps, uint16_t penalty1, uint16_t penalty2,
    const float* merge_with, float* depth_out, double* ms_out,
    const smvsb_sgm_options* opts, smvsb_sgm_stats* stats)
{
    return guarded(nullptr, [&]() {
        smvsb::sgm_reconstruct(device, w, h, main_lum, nw, nh, neigh_lum,
            M_mn, t_mn, M_nm, t_nm, depth_range_main, depth_range_neigh,
            num_steps, penalty1, penalty2, merge_with, depth_out, ms_out,
            opts, stats);
    });
}

int
smvsb_cut_depth_maps (int device, int n_views, const int* w, const int* h,
    const float* const* depth, const float* const* normals,
    const float* invproj9, const float* cam_to_world16, const float* KR9,
    const float* t3, float* const* depth_out)
{
    smvsb_cut_options opts = {};
    opts.devices = &device;
    opts.n_devices = 1;
    return smvsb_cut_depth_maps_multi(&opts, n_views, w, h, depth, normals,
        invproj9, cam_to_world16, KR9, t3, depth_out, nullptr);
}

int
smvsb_cut_depth_maps_multi (const smvsb_cut_options* opts, int n_views,
    const int* w, const int* h, const float* const* depth,
    const float* const* normals, const float* invproj9,
    const float* cam_to_world16, const float* KR9, const float* t3,
    float* const* depth_out, smvsb_cut_stats* stats)
{
    return guarded(nullptr, [&]() {
        smvsb::cut_depth_maps_multi(opts, n_views, w, h, depth, normals,
            invproj9, cam_to_world16, KR9, t3, depth_out, stats);
    });
}

} /* extern "C" */

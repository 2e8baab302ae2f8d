/*
 * update.cu -- node update + active-set test, depth / normal map rendering,
 * and the lighting normal equations.
 *
 *   K4  reproj_kernel    DepthOptimizer::fill_node_reprojections before and
 *                        after Surface::update_nodes, and the > 0.15 px test
 *                        (lib/depth_optimizer.cc:271-303, 647-677). The
 *                        reference materialises two vectors of
 *                        4 * pixels * neighbours entries; here each patch is
 *                        one block-wide OR / sum.
 *       apply_delta_kernel   Surface::update_nodes (lib/surface.cc:957-981)
 *   render_depth_kernel / render_normals_kernel
 *                        Surface::get_depth_map / get_normal_map
 *                        (lib/surface.cc:155-183, lib/surface_patch.cc:15-55)
 *   K5  light_partials_kernel  LightOptimizer::fit_lighting_to_image sums
 *                        (lib/light_optimizer.cc:22-55)
 */
#include "gn_math.cuh"
#include "patch_eval.cuh"

namespace smvsb {

namespace {

constexpr int UPD_THREADS = 64;

/* depth of the patch at pixel (i, j) of the patch: sum theta * X0 * Y0 */
__device__ __forceinline__ double
eval_depth (double const* theta, double const* X0, double const* Y0)
{
    double w = 0.0;
#pragma unroll
    for (int col = 0; col < 16; ++col)
    {
        int const bx = ((col >> 2) & 1) + 2 * (col & 1);
        int const by = ((col >> 3) & 1) + 2 * ((col >> 1) & 1);
        w += theta[col] * X0[bx] * Y0[by];
    }
    return w;
}

/*
 * G = threads per patch (a power of two <= UPD_THREADS, = min(ps^2, 64));
 * a block holds UPD_THREADS / G patches, so at scale 2 (16 pixels per patch)
 * four patches share a block instead of leaving 48 of 64 threads idle.
 * PS_MAX = the largest patch size the cached basis_f row holds (64 up to
 * scale 6, 256 at scales 7 and 8).
 */
template <int G, int PS_MAX = 64>
__global__ void __launch_bounds__(UPD_THREADS)
reproj_kernel (SurfaceDev const sf, double const* __restrict__ delta,
    double thresh, uint8_t* __restrict__ active_new,
    double* __restrict__ patch_shift)
{
    constexpr int PPB = UPD_THREADS / G;
    __shared__ double s_theta[PPB][16], s_dtheta[PPB][16];
    __shared__ double s_b0[PS_MAX * 4];
    __shared__ double s_sum[UPD_THREADS / 32];
    __shared__ int s_flag[UPD_THREADS / 32];

    int const tid = threadIdx.x;
    int const pl = tid / G, lt = tid % G;
    int const patch = blockIdx.x * PPB + pl;
    int idx = 0, idy = 0, n0 = 0;
    bool proc = false;
    if (patch < sf.n_patches)
    {
        idx = patch % sf.npx; idy = patch / sf.npx;
        n0 = idy * (sf.npx + 1) + idx;
        proc = sf.patch_valid[patch] != 0;
        if (proc)
            proc = (sf.active[n0] | sf.active[n0 + 1]
                | sf.active[n0 + sf.npx + 1] | sf.active[n0 + sf.npx + 2]) != 0;
    }
    for (int i = tid; i < sf.ps * 4; i += UPD_THREADS)
        s_b0[i] = sf.basis_f[i];
    for (int c = lt; c < 16 && proc; c += G)
    {
        int const node = (idy + ((c >> 3) & 1)) * (sf.npx + 1)
            + idx + ((c >> 2) & 1);
        s_theta[pl][c] = sf.nodes[node * 4 + (c & 3)];
        s_dtheta[pl][c] = delta[node * 4 + (c & 3)];
    }
    __syncthreads();

    double sum = 0.0;
    int flag = 0;
    int const npix = sf.ps * sf.ps;
    int n = 0;
    if (proc)
    {
        uint32_t const v0 = sf.vis_off[patch];
        n = static_cast<int>(sf.vis_off[patch + 1] - v0);
        for (int p = lt; p < npix; p += G)
        {
            int const i = p % sf.ps, j = p / sf.ps;
            double const w1 = eval_depth(s_theta[pl], s_b0 + i * 4,
                s_b0 + j * 4);
            double const w2 = w1 + eval_depth(s_dtheta[pl], s_b0 + i * 4,
                s_b0 + j * 4);
            /* no +0.5 here: lib/depth_optimizer.cc:669-670 */
            double const u = sf.start_x + idx * sf.ps + i;
            double const v = sf.start_y + idy * sf.ps + j;
            for (int k = 0; k < n; ++k)
            {
                double const* Mt = sf.Mt + sf.vis_ids[v0 + k] * 12;
                double const pp = Mt[0] * u + Mt[1] * v + Mt[2];
                double const qq = Mt[3] * u + Mt[4] * v + Mt[5];
                double const rr = Mt[6] * u + Mt[7] * v + Mt[8];
                double const d1 = w1 * rr + Mt[11], d2 = w2 * rr + Mt[11];
                double const ex = (w1 * pp + Mt[9]) / d1
                    - (w2 * pp + Mt[9]) / d2;
                double const ey = (w1 * qq + Mt[10]) / d1
                    - (w2 * qq + Mt[10]) / d2;
                double const diff = sqrt(ex * ex + ey * ey);
                sum += diff;
                flag |= (diff > thresh);
            }
        }
    }
    /* reduce over the G threads of the patch (fixed order) */
    constexpr int W = (G < 32) ? G : 32;
    for (int off = W / 2; off > 0; off >>= 1)
    {
        sum += __shfl_down_sync(0xffffffffu, sum, off, W);
        flag |= __shfl_down_sync(0xffffffffu, flag, off, W);
    }
    if (G > 32)
    {
        if ((tid & 31) == 0)
        {
            s_sum[tid >> 5] = sum;
            s_flag[tid >> 5] = flag;
        }
        __syncthreads();
        if (tid == 0)
        {
            sum = 0.0; flag = 0;
            for (int i = 0; i < UPD_THREADS / 32; ++i)
            {
                sum += s_sum[i];
                flag |= s_flag[i];
            }
        }
    }
    if (lt == 0 && patch < sf.n_patches)
    {
        patch_shift[2 * patch] = proc ? sum : 0.0;
        patch_shift[2 * patch + 1] = proc ? double(npix) * n : 0.0;
        if (proc && flag)
        {
            /* every entry of the patch carries all four node ids,
             * lib/depth_optimizer.cc:674-675 */
            active_new[n0] = 1;
            active_new[n0 + 1] = 1;
            active_new[n0 + sf.npx + 1] = 1;
            active_new[n0 + sf.npx + 2] = 1;
        }
    }
}

__global__ void
apply_delta_kernel (int n_nodes, uint8_t const* __restrict__ node_valid,
    double const* __restrict__ delta, double* __restrict__ nodes)
{
    int const i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes * 4)
        return;
    if (node_valid[i >> 2])
        nodes[i] += delta[i];
}

/* Stage 1: each block sums a fixed slice of patch_shift and of the active
 * flags; stage 2 (one block) sums the per-block results in block order. Fixed
 * grid -> deterministic. */
constexpr int RED_BLOCKS = 128;

__global__ void __launch_bounds__(256)
update_reduce_kernel (int n_patches, double const* __restrict__ patch_shift,
    int n_nodes, uint8_t const* __restrict__ active,
    double* __restrict__ partial /* [RED_BLOCKS][3] */)
{
    __shared__ double s_a[256], s_b[256], s_c[256];
    int const tid = threadIdx.x;
    int const gid = blockIdx.x * 256 + tid, gstride = gridDim.x * 256;
    double a = 0.0, b = 0.0, c = 0.0;
    for (int i = gid; i < n_patches; i += gstride)
    {
        a += patch_shift[2 * i];
        b += patch_shift[2 * i + 1];
    }
    for (int i = gid; i < n_nodes; i += gstride)
        c += (active[i] == 1) ? 1.0 : 0.0;
    s_a[tid] = a; s_b[tid] = b; s_c[tid] = c;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1)
    {
        if (tid < off)
        {
            s_a[tid] += s_a[tid + off];
            s_b[tid] += s_b[tid + off];
            s_c[tid] += s_c[tid + off];
        }
        __syncthreads();
    }
    if (tid == 0)
    {
        partial[3 * blockIdx.x + 0] = s_a[0];
        partial[3 * blockIdx.x + 1] = s_b[0];
        partial[3 * blockIdx.x + 2] = s_c[0];
    }
}

__global__ void
update_reduce_final_kernel (int nblocks, double const* __restrict__ partial,
    double* __restrict__ out /* [0] sum, [1] count, [2] n_active */)
{
    if (threadIdx.x < 3)
    {
        double v = 0.0;
        for (int b = 0; b < nblocks; ++b)
            v += partial[3 * b + threadIdx.x];
        out[threadIdx.x] = v;
    }
}

__global__ void
count_processed_kernel (SurfaceDev const sf, unsigned long long* out)
{
    int const patch = blockIdx.x * blockDim.x + threadIdx.x;
    int proc = 0;
    if (patch < sf.n_patches && sf.patch_valid[patch])
    {
        int const idx = patch % sf.npx, idy = patch / sf.npx;
        int const n0 = idy * (sf.npx + 1) + idx;
        proc = (sf.active[n0] | sf.active[n0 + 1]
            | sf.active[n0 + sf.npx + 1] | sf.active[n0 + sf.npx + 2]) != 0;
    }
    unsigned const m = __ballot_sync(0xffffffffu, proc);
    if ((threadIdx.x & 31) == 0 && m)
        atomicAdd(out, (unsigned long long)__popc(m));
}

/* one thread per pixel of the patch grid area */
__global__ void
render_kernel (SurfaceDev const sf, float* __restrict__ out, int normals)
{
    int const gx = blockIdx.x * blockDim.x + threadIdx.x;
    int const gy = blockIdx.y * blockDim.y + threadIdx.y;
    if (gx >= sf.npx * sf.ps || gy >= sf.npy * sf.ps)
        return;
    int const idx = gx / sf.ps, idy = gy / sf.ps;
    int const patch = idy * sf.npx + idx;
    if (!sf.patch_valid[patch])
        return;
    int const i = gx % sf.ps, j = gy % sf.ps;
    /* BicubicPatch::evaluate_f / _dx / _dy on the polynomial coefficients,
     * bitwise the reference's values (patch_eval.cuh): the depth map feeds
     * the visibility z-buffer, where decisions hang on the last bit */
    double theta[16], cf[16];
    load_patch_theta(sf.nodes, sf.npx, idx, idy, theta);
    patch_coefficients(theta, cf);
    PatchSample const smp = normals ? patch_sample<true>(cf, i, j, sf.ps)
        : patch_sample<false>(cf, i, j, sf.ps);
    double const w = smp.w, wx = smp.wx, wy = smp.wy;
    int const px = sf.start_x + gx, py = sf.start_y + gy;
    size_t const pix = static_cast<size_t>(py) * sf.w + px;
    if (!normals)
    {
        out[pix] = static_cast<float>(w);
        return;
    }
    double const x = px + 0.5 - static_cast<double>(sf.w) / 2.0;
    double const y = py + 0.5 - static_cast<double>(sf.h) / 2.0;
    double nrm[3];
    /* get_normal_map takes a FLOAT inv_flen (lib/surface.cc:170-171): the
     * caller's value is narrowed before it reaches fill_normal */
    fill_normal(x, y, static_cast<double>(static_cast<float>(sf.inv_flen)),
        w, wx, wy, nrm);
    out[pix * 3 + 0] = static_cast<float>(nrm[0]);
    out[pix * 3 + 1] = static_cast<float>(nrm[1]);
    out[pix * 3 + 2] = static_cast<float>(nrm[2]);
}

constexpr int LIGHT_THREADS = 256;
constexpr int LIGHT_VALUES = 136 + 16;     /* upper triangle of A, b */

/* Per block partial sums of sh sh^T (upper triangle) and sh * I over the
 * pixels that pass the tests of lib/light_optimizer.cc:36-38; normals are
 * rounded through fp32 like the reference's normal map. */
__global__ void __launch_bounds__(LIGHT_THREADS)
light_partials_kernel (int npix, float const* __restrict__ normals,
    float const* __restrict__ image, double* __restrict__ partials)
{
    __shared__ double s_red[LIGHT_THREADS / 32][LIGHT_VALUES];
    double acc[LIGHT_VALUES];
#pragma unroll
    for (int i = 0; i < LIGHT_VALUES; ++i) acc[i] = 0.0;

    for (int p = blockIdx.x * LIGHT_THREADS + threadIdx.x; p < npix;
        p += gridDim.x * LIGHT_THREADS)
    {
        double nrm[3] = { normals[3 * p], normals[3 * p + 1],
            normals[3 * p + 2] };
        float const iv = image[p];
        double const len = sqrt(nrm[0] * nrm[0] + nrm[1] * nrm[1]
            + nrm[2] * nrm[2]);
        if (fabs(len - 1.0) > 1e-6 || iv < 0.05f)
            continue;
        double sh[16];
        sh_evaluate_4_band(nrm, sh);
        int o = 0;
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int j = i; j < 16; ++j)
                acc[o++] += sh[i] * sh[j];
#pragma unroll
        for (int i = 0; i < 16; ++i)
            acc[136 + i] += sh[i] * static_cast<double>(iv);
    }
    int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < LIGHT_VALUES; ++i)
    {
        double v = acc[i];
        for (int off = 16; off > 0; off >>= 1)
            v += __shfl_down_sync(0xffffffffu, v, off);
        if (lane == 0)
            s_red[warp][i] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < LIGHT_VALUES; i += LIGHT_THREADS)
    {
        double v = 0.0;
        for (int wi = 0; wi < LIGHT_THREADS / 32; ++wi)
            v += s_red[wi][i];
        partials[static_cast<size_t>(blockIdx.x) * LIGHT_VALUES + i] = v;
    }
}

} /* namespace */

void
update_enqueue (smvsb_ctx* c, double thresh, bool full_opt)
{
    SurfaceDev const sf = surface_args(c);
    c->patch_shift.reserve(static_cast<size_t>(c->n_patches) * 2);
    c->active_new.reserve(c->n_nodes);
    c->upd_result.reserve(4);
    CUDA_CHECK(cudaMemsetAsync(c->active_new.p, 0, c->n_nodes, c->stream));
    int const npix_patch = c->ps * c->ps;
    auto grid_for = [&](int g) { int const ppb = UPD_THREADS / g;
        return (c->n_patches + ppb - 1) / ppb; };
    if (c->ps > 64)
        reproj_kernel<64, 256><<<grid_for(64), UPD_THREADS, 0, c->stream>>>(
            sf, c->x.p, thresh, c->active_new.p, c->patch_shift.p);
    else if (npix_patch >= 64)
        reproj_kernel<64><<<grid_for(64), UPD_THREADS, 0, c->stream>>>(sf,
            c->x.p, thresh, c->active_new.p, c->patch_shift.p);
    else if (npix_patch == 16)
        reproj_kernel<16><<<grid_for(16), UPD_THREADS, 0, c->stream>>>(sf,
            c->x.p, thresh, c->active_new.p, c->patch_shift.p);
    else if (npix_patch == 4)
        reproj_kernel<4><<<grid_for(4), UPD_THREADS, 0, c->stream>>>(sf,
            c->x.p, thresh, c->active_new.p, c->patch_shift.p);
    else
        reproj_kernel<1><<<grid_for(1), UPD_THREADS, 0, c->stream>>>(sf,
            c->x.p, thresh, c->active_new.p, c->patch_shift.p);
    CUDA_CHECK(cudaGetLastError());
    int const n4 = c->n_nodes * 4;
    apply_delta_kernel<<<(n4 + 255) / 256, 256, 0, c->stream>>>(c->n_nodes,
        c->node_valid.p, c->x.p, c->nodes.p);
    CUDA_CHECK(cudaGetLastError());
    if (!full_opt)
    {
        /* the new set replaces the old one, lib/depth_optimizer.cc:291-298 */
        CUDA_CHECK(cudaMemcpyAsync(c->active.p, c->active_new.p, c->n_nodes,
            cudaMemcpyDeviceToDevice, c->stream));
    }
    c->upd_partials.reserve(3 * RED_BLOCKS);
    update_reduce_kernel<<<RED_BLOCKS, 256, 0, c->stream>>>(c->n_patches,
        c->patch_shift.p, c->n_nodes, c->active.p, c->upd_partials.p);
    CUDA_CHECK(cudaGetLastError());
    update_reduce_final_kernel<<<1, 32, 0, c->stream>>>(RED_BLOCKS,
        c->upd_partials.p, c->upd_result.p);
    CUDA_CHECK(cudaGetLastError());
    smvsb::count_launches(c, 4);
    CUDA_CHECK(cudaMemcpyAsync(c->pinned->update, c->upd_result.p,
        3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
}

/* after the stream has been synchronised */
void
update_collect (smvsb_ctx* c, uint64_t* n_active, double* mean_shift)
{
    double const* res = c->pinned->update;
    if (n_active) *n_active = static_cast<uint64_t>(res[2]);
    if (mean_shift) *mean_shift = res[0] / res[1];
}

void
launch_update (smvsb_ctx* c, double thresh, bool full_opt,
    uint64_t* n_active, double* mean_shift)
{
    update_enqueue(c, thresh, full_opt);
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    update_collect(c, n_active, mean_shift);
}

void
count_processed_enqueue (smvsb_ctx* c)
{
    SurfaceDev const sf = surface_args(c);
    c->counters.reserve(4);
    CUDA_CHECK(cudaMemsetAsync(c->counters.p, 0, sizeof(unsigned long long),
        c->stream));
    count_processed_kernel<<<(c->n_patches + 255) / 256, 256, 0,
        c->stream>>>(sf, c->counters.p);
    smvsb::count_launches(c, 1);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(&c->pinned->processed, c->counters.p,
        sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
}

unsigned long long
count_processed_collect (smvsb_ctx* c)
{
    return c->pinned->processed;
}

void
launch_count_processed (smvsb_ctx* c, unsigned long long* n_proc_host)
{
    count_processed_enqueue(c);
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    *n_proc_host = count_processed_collect(c);
}

static void
launch_render (smvsb_ctx* c, float* out_dev, int normals)
{
    SurfaceDev const sf = surface_args(c);
    size_t const bytes = static_cast<size_t>(c->w) * c->h
        * (normals ? 3 : 1) * sizeof(float);
    CUDA_CHECK(cudaMemsetAsync(out_dev, 0, bytes, c->stream));
    dim3 const block(32, 8);
    dim3 const grid((c->npx * c->ps + 31) / 32, (c->npy * c->ps + 7) / 8);
    if (grid.x > 0 && grid.y > 0)
        render_kernel<<<grid, block, 0, c->stream>>>(sf, out_dev, normals);
    smvsb::count_launches(c, 1);
    CUDA_CHECK(cudaGetLastError());
}

void
launch_render_depth (smvsb_ctx* c, float* out_dev)
{
    launch_render(c, out_dev, 0);
}

void
launch_render_normals (smvsb_ctx* c, float* out_dev)
{
    launch_render(c, out_dev, 1);
}

/* A_b_host: 16x16 row-major A followed by b (272 doubles), summed over the
 * per-block partials in block order on the host (152 x <= 592 adds). */
void
run_fit_lighting (smvsb_ctx* c, double* A_b_host)
{
    int const npix = c->w * c->h;
    c->image_out.reserve(static_cast<size_t>(npix) * 3);
    launch_render_normals(c, c->image_out.p);
    int const grid = std::max(1, std::min(c->num_sms * 4,
        (npix + LIGHT_THREADS - 1) / LIGHT_THREADS));
    c->light_partials.reserve(static_cast<size_t>(grid) * LIGHT_VALUES);
    light_partials_kernel<<<grid, LIGHT_THREADS, 0, c->stream>>>(npix,
        c->image_out.p, c->main_shading.p, c->light_partials.p);
    smvsb::count_launches(c, 1);
    CUDA_CHECK(cudaGetLastError());
    std::vector<double> part(static_cast<size_t>(grid) * LIGHT_VALUES);
    CUDA_CHECK(cudaMemcpyAsync(part.data(), c->light_partials.p,
        part.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    double tri[LIGHT_VALUES];
    for (int i = 0; i < LIGHT_VALUES; ++i)
    {
        double v = 0.0;
        for (int b = 0; b < grid; ++b)
            v += part[static_cast<size_t>(b) * LIGHT_VALUES + i];
        tri[i] = v;
    }
    int o = 0;
    for (int i = 0; i < 16; ++i)
        for (int j = i; j < 16; ++j)
        {
            A_b_host[i * 16 + j] = tri[o];
            A_b_host[j * 16 + i] = tri[o];
            o += 1;
        }
    for (int i = 0; i < 16; ++i)
        A_b_host[256 + i] = tri[136 + i];
}

} /* namespace smvsb */

/*
 * visibility.cu -- which neighbours see which patch, and where the surface is
 * cut: DepthOptimizer::create_subview_surfaces (lib/depth_optimizer.cc:433-604,
 * both modes; use_sgm = false adds ncc_for_patch :795-912 on the colour
 * images) and DepthOptimizer::cut_boundaries (:360-431) with
 * mse_for_patch (:747-793), Surface::remove_nodes_without_patch
 * (lib/surface.cc:762-867), on the surface resident in the context.
 *
 * All of it is yes/no decisions on fp64 values, so every value a decision
 * looks at is computed bitwise like the CPU (patch_eval.cuh); the reference's
 * order-dependent pieces are order-free here by construction:
 *   - the per-neighbour depth cache (a z-buffer of fp32 minima filled by a
 *     sequential "if (d < cache) cache = d") becomes an atomicMin on an
 *     order-preserving integer image of fp32(d): rounding is monotone, so the
 *     result is the same minimum whatever the order;
 *   - "all pixels of the patch pass" / "largest Jacobian anisotropy" are
 *     and / max reductions;
 *   - mse_for_patch is a sequential sum per patch: one thread per patch adds
 *     in the reference's order (pixels outer, neighbours inner).
 */
#include "patch_eval.cuh"

namespace smvsb {

namespace {

constexpr float ZBUF_FAR = 10000.0f;        /* lib/depth_optimizer.cc:449 */

/* order-preserving fp32 -> u32 (and back) */
__host__ __device__ __forceinline__ unsigned int
float_key (float f)
{
#ifdef __CUDA_ARCH__
    unsigned int const b = __float_as_uint(f);
#else
    unsigned int b;
    memcpy(&b, &f, 4);
#endif
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float
key_float (unsigned int k)
{
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct VisArgs
{
    SurfaceDev s;
    unsigned int* zbuf;             /* all neighbours' caches, concatenated */
    unsigned long long const* zoff; /* n_sub + 1 offsets into zbuf */
    float const* surf_depth;        /* w*h, Surface::get_depth_map */
    float const* sgm_depth;         /* w*h */
    unsigned int* vis_mask;         /* n_patches */
    unsigned long long* counters;   /* [0] removed / deleted patches */
    /* use_sgm = false only */
    float const* color_main;        /* w*h*3 */
    float const* const* color_subs; /* n_sub pointers, sub_w*sub_h*3 each */
    short4 const* rim;              /* the eight rim lists, concatenated */
    int rim_off[9];
};

__global__ void
zbuf_fill_kernel (unsigned int* z, unsigned long long n, unsigned int key)
{
    unsigned long long i = blockIdx.x * static_cast<unsigned long long>(
        blockDim.x) + threadIdx.x;
    unsigned long long const stride = static_cast<unsigned long long>(
        gridDim.x) * blockDim.x;
    for (; i < n; i += stride)
        z[i] = key;
}

/* first pass, :470-500: every surface pixel and every SGM pixel lowers the
 * 3x3 neighbourhood of its projection in every neighbour's cache */
__global__ void __launch_bounds__(256)
zbuf_scatter_kernel (VisArgs const a)
{
    SurfaceDev const& sf = a.s;
    int const pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= sf.w * sf.h)
        return;
    int const x = pix % sf.w, y = pix / sf.w;
    for (int src = 0; src < 2; ++src)
    {
        if (src == 1 && a.sgm_depth == nullptr)
            break;                  /* use_sgm = false: surface pixels only */
        float const dep = (src == 0) ? a.surf_depth[pix] : a.sgm_depth[pix];
        if (dep == 0.0f)
            continue;
        for (int sub = 0; sub < sf.n_sub; ++sub)
        {
            Warp const c = warp_pixel<false>(sf.Mt + sub * 12, x + 0.5,
                y + 0.5, static_cast<double>(dep), 0.0, 0.0);
            int const sw = sf.sub_dims[2 * sub], sh = sf.sub_dims[2 * sub + 1];
            double const cut = 3.0;
            /* written so that a NaN projection is skipped (the reference
             * would index with it) */
            if (!(c.projx >= cut && c.projx < sw - cut
                && c.projy >= cut && c.projy < sh - cut))
                continue;
            int const cx = static_cast<int>(c.projx);
            int const cy = static_cast<int>(c.projy);
            unsigned int const key = float_key(static_cast<float>(c.depth));
            unsigned int* z = a.zbuf + a.zoff[sub];
            for (int dy = -1; dy < 2; ++dy)
                for (int dx = -1; dx < 2; ++dx)
                    atomicMin(z + static_cast<size_t>(cy + dy) * (sw + 1)
                        + (cx + dx), key);
        }
    }
}

/* anisotropy of the warp over a patch: largest ratio of the squared singular
 * values of the 2x2 Jacobian, :555-577 */
__device__ __forceinline__ double
warp_anisotropy_at (double const* cf, double const* __restrict__ Mt, int px0,
    int py0, int ps, int pid)
{
    int const i = pid % ps, j = pid / ps;
    PatchSample const smp = patch_sample<true>(cf, i, j, ps);
    Warp const c = warp_pixel<true>(Mt, px0 + i + 0.5, py0 + j + 0.5,
        smp.w, smp.wx, smp.wy);
    xd const j0(c.jac[0]), j1(c.jac[1]), j2(c.jac[2]), j3(c.jac[3]);
    xd const e = j0 - j3, f = j1 + j2, g = j0 + j3, h = j1 - j2;
    xd const q = xsqrt(e * e + f * f);
    xd const s0 = (q + xsqrt(g * g + h * h)) / xd(2.0);
    double const s1 = fabs((s0 - q).v);
    double const big = (s0.v < s1) ? s1 : s0.v;     /* std::max(S0, S1) */
    double const small = (s1 < s0.v) ? s1 : s0.v;   /* std::min(S0, S1) */
    return (xd(big) * xd(big) / (xd(small) * xd(small))).v;
}

__device__ __forceinline__ double
warp_anisotropy (double const* cf, double const* __restrict__ Mt, int px0,
    int py0, int ps)
{
    double worst = 0.0;
    for (int pid = 0; pid < ps * ps; ++pid)
    {
        double const ratio = warp_anisotropy_at(cf, Mt, px0, py0, ps, pid);
        worst = (worst < ratio) ? ratio : worst;        /* std::max */
    }
    return worst;
}

/* The per-pixel test of the second pass (:520-540): the pixel's projection
 * into neighbour sub lies inside its 3 % border and is not behind its depth
 * cache. */
struct NeighbourTest
{
    unsigned int const* z;
    int sw, sh;
    double cut, hi_x, hi_y;

    __device__ __forceinline__
    NeighbourTest (VisArgs const& a, int sub)
        : z(a.zbuf + a.zoff[sub]), sw(a.s.sub_dims[2 * sub]),
          sh(a.s.sub_dims[2 * sub + 1])
    {
        cut = (xd(0.03) * xd(static_cast<double>(max(sw, sh)))).v;
        hi_x = (xd(static_cast<double>(sw)) - xd(cut)).v;
        hi_y = (xd(static_cast<double>(sh)) - xd(cut)).v;
    }

    __device__ __forceinline__ bool
    passes (Warp const& c) const
    {
        if (!(c.projx >= cut && c.projx < hi_x
            && c.projy >= cut && c.projy < hi_y))
            return false;
        int const cx = static_cast<int>(c.projx);
        int const cy = static_cast<int>(c.projy);
        double const near = (xd(c.depth) * xd(0.95)).v;
        bool visible = true;
        for (int dy = -1; dy < 2; ++dy)
            for (int dx = -1; dx < 2; ++dx)
            {
                int const zx = cx + dx, zy = cy + dy;
                if (zx < 0 || zy < 0 || zx > sw || zy > sh)
                    continue;
                float const zc = key_float(z[static_cast<size_t>(zy)
                    * (sw + 1) + zx]);
                if (near > static_cast<double>(zc))
                    visible = false;
            }
        return visible;
    }
};

/* second pass, :502-583: L lanes per (patch, neighbour). L = 32 serves the
 * coarse scales (patch size 8 .. 64 pixels, a few thousand patches), where
 * one thread per pair would leave the GPU to a handful of threads that each
 * walk up to 4096 pixels. All three tests are order-free (every pixel
 * passes / largest ratio), so the lanes take the pixels in turn. */
template <int L>
__global__ void __launch_bounds__(128)
vis_patch_kernel (VisArgs const a)
{
    SurfaceDev const& sf = a.s;
    int const t = (blockIdx.x * blockDim.x + threadIdx.x) / L;
    int const lane = threadIdx.x % L;
    if (t >= sf.npx * sf.npy * sf.n_sub)
        return;
    int const patch = t / sf.n_sub, sub = t % sf.n_sub;
    if (!sf.patch_valid[patch])
        return;
    int const idx = patch % sf.npx, idy = patch / sf.npx;
    int const ps = sf.ps;
    double theta[16], cf[16];
    load_patch_theta(sf.nodes, sf.npx, idx, idy, theta);
    patch_coefficients(theta, cf);
    double const* Mt = sf.Mt + sub * 12;
    int const px0 = sf.start_x + idx * ps, py0 = sf.start_y + idy * ps;
    NeighbourTest const test(a, sub);
    bool fail = false;
    for (int pid = lane; pid < ps * ps && !fail; pid += L)
    {
        int const i = pid % ps, j = pid / ps;
        PatchSample const smp = patch_sample<false>(cf, i, j, ps);
        fail = !test.passes(warp_pixel<false>(Mt, px0 + i + 0.5,
            py0 + j + 0.5, smp.w, 0.0, 0.0));
    }
    if (L == 1 ? fail : __any_sync(0xffffffffu, fail))
        return;
    double worst = 0.0;
    for (int pid = lane; pid < ps * ps; pid += L)
    {
        double const ratio = warp_anisotropy_at(cf, Mt, px0, py0, ps, pid);
        worst = (worst < ratio) ? ratio : worst;        /* std::max */
    }
    for (int off = L / 2; off > 0; off >>= 1)
    {
        double const other = __shfl_xor_sync(0xffffffffu, worst, off);
        worst = (worst < other) ? other : worst;
    }
    if (worst > 8.0)
        return;
    if (lane == 0)
        atomicOr(a.vis_mask + patch, 1u << sub);
}

/* ---- use_sgm = false: the NCC occlusion filter ----------------------- */

/* mve::Image<float>::linear_at(x, y, channel) on an interleaved 3-channel
 * image: clamped fp32 coordinates, fp32 weights, left-to-right fp32 sum, no
 * contraction (as the reference is built, -ffp-contract=off). */
__device__ __forceinline__ float
linear_at_rgb (float const* __restrict__ img, int w, int h, float x, float y,
    int ch)
{
    x = fmaxf(0.0f, fminf(static_cast<float>(w - 1), x));
    y = fmaxf(0.0f, fminf(static_cast<float>(h - 1), y));
    int const fx = static_cast<int>(x), fy = static_cast<int>(y);
    int const fx1 = min(fx + 1, w - 1), fy1 = min(fy + 1, h - 1);
    float const w1 = __fsub_rn(x, static_cast<float>(fx));
    float const w0 = __fsub_rn(1.0f, w1);
    float const w3 = __fsub_rn(y, static_cast<float>(fy));
    float const w2 = __fsub_rn(1.0f, w3);
    float const v00 = img[(static_cast<size_t>(fy) * w + fx) * 3 + ch];
    float const v10 = img[(static_cast<size_t>(fy) * w + fx1) * 3 + ch];
    float const v01 = img[(static_cast<size_t>(fy1) * w + fx) * 3 + ch];
    float const v11 = img[(static_cast<size_t>(fy1) * w + fx1) * 3 + ch];
    float acc = __fmul_rn(v00, __fmul_rn(w0, w2));
    acc = __fadd_rn(acc, __fmul_rn(v10, __fmul_rn(w1, w2)));
    acc = __fadd_rn(acc, __fmul_rn(v01, __fmul_rn(w0, w3)));
    acc = __fadd_rn(acc, __fmul_rn(v11, __fmul_rn(w1, w3)));
    return acc;
}

/* Entry i of the pixel list ncc_for_patch builds (:803-859): the patch's own
 * pixels, then the rim the growing loop appends. The list's SHAPE depends
 * only on the patch size and on three yes/no conditions of the patch's
 * position, so the host builds the eight lists once (offsets from the patch
 * origin and where each entry's depth is copied from: a patch pixel or a
 * corner node) and the device walks them. */
struct ListEntry
{
    double x, y, depth;
};

__device__ __forceinline__ ListEntry
list_entry (short4 const* __restrict__ rim, int i, int ps,
    double const* cf, double const* theta, int px0, int py0)
{
    int ox, oy, src;
    if (i < ps * ps)
    {
        ox = i % ps; oy = i / ps; src = i;
    }
    else
    {
        short4 const e = rim[i - ps * ps];
        ox = e.x; oy = e.y;
        src = static_cast<int>((static_cast<unsigned>(static_cast<uint16_t>(
            e.w)) << 16) | static_cast<uint16_t>(e.z));
    }
    ListEntry out;
    out.x = static_cast<double>(px0 + ox);
    out.y = static_cast<double>(py0 + oy);
    /* src < 0: corner node -src - 1 (fill_values_at_nodes, :804), else the
     * depth of patch pixel src (fill_values_at_pixels, :807) */
    out.depth = (src < 0) ? theta[(-src - 1) * 4]
        : patch_sample<false>(cf, src % ps, src / ps, ps).w;
    return out;
}

/* DepthOptimizer::ncc_for_patch. Only the sign of the result is used
 * (:579-581). Two passes over the list instead of the reference's two
 * value vectors: the means first, then the three sums, in the order
 * SSEVector::dot adds them. */
__device__ double
ncc_for_patch_dev (VisArgs const& a, int sub, short4 const* rim, int n_list,
    int ps, double const* cf, double const* theta, int px0, int py0)
{
    SurfaceDev const& sf = a.s;
    double const* Mt = sf.Mt + sub * 12;
    int const sw = sf.sub_dims[2 * sub], sh = sf.sub_dims[2 * sub + 1];
    float const* simg = a.color_subs[sub];
    xd means0[3], means1[3], counter[3];
    for (int c = 0; c < 3; ++c)
        means0[c] = means1[c] = counter[c] = xd(0.0);
    double const hi_x = static_cast<double>(sw - 2);
    double const hi_y = static_cast<double>(sh - 2);
    for (int i = 0; i < n_list; ++i)
    {
        ListEntry const e = list_entry(rim, i, ps, cf, theta, px0, py0);
        Warp const c = warp_pixel<false>(Mt, (xd(e.x) + xd(0.5)).v,
            (xd(e.y) + xd(0.5)).v, e.depth, 0.0, 0.0);
        if (c.projx < 1 || c.projx > hi_x || c.projy < 1 || c.projy > hi_y)
            return -1.0;
        size_t const mp = (static_cast<size_t>(static_cast<int>(e.y)) * sf.w
            + static_cast<int>(e.x)) * 3;
        for (int ch = 0; ch < 3; ++ch)
        {
            xd const cm(static_cast<double>(a.color_main[mp + ch]));
            xd const cs(static_cast<double>(linear_at_rgb(simg, sw, sh,
                static_cast<float>(c.projx), static_cast<float>(c.projy),
                ch)));
            counter[ch] += xd(1.0);
            means0[ch] += (cm - means0[ch]) / counter[ch];
            means1[ch] += (cs - means1[ch]) / counter[ch];
        }
    }
    /* SSEVector::dot (lib/sse_vector.cc:19-41, SSE branch): the products of
     * an element pair are added to each other first (_mm_dp_pd), then to the
     * running sum; an odd last element is added on its own */
    xd s00(0.0), s11(0.0), s01(0.0);
    xd p00(0.0), p11(0.0), p01(0.0);
    int k = 0;
    for (int i = 0; i < n_list; ++i)
    {
        ListEntry const e = list_entry(rim, i, ps, cf, theta, px0, py0);
        Warp const c = warp_pixel<false>(Mt, (xd(e.x) + xd(0.5)).v,
            (xd(e.y) + xd(0.5)).v, e.depth, 0.0, 0.0);
        size_t const mp = (static_cast<size_t>(static_cast<int>(e.y)) * sf.w
            + static_cast<int>(e.x)) * 3;
        for (int ch = 0; ch < 3; ++ch, ++k)
        {
            xd const v0 = xd(static_cast<double>(a.color_main[mp + ch]))
                - means0[ch];
            xd const v1 = xd(static_cast<double>(linear_at_rgb(simg, sw, sh,
                static_cast<float>(c.projx), static_cast<float>(c.projy),
                ch))) - means1[ch];
            if ((k & 1) == 0)
            {
                p00 = v0 * v0; p11 = v1 * v1; p01 = v0 * v1;
            }
            else
            {
                s00 += p00 + v0 * v0;
                s11 += p11 + v1 * v1;
                s01 += p01 + v0 * v1;
            }
        }
    }
    if (k & 1)
    {
        s00 += p00; s11 += p11; s01 += p01;
    }
    xd const norm0 = xsqrt(s00), norm1 = xsqrt(s11);
    if ((norm0 + norm1).v < (xd(0.001) * xd(static_cast<double>(n_list))).v)
        return 1.0;
    return (s01 / (norm0 * norm1)).v;
}

/* ncc_for_patch_dev on the 32 lanes of a warp (patch sizes 128 and 256: a
 * list of 16 K / 65 K entries). The lanes evaluate 32 entries at a time --
 * the warp into the neighbour and the bilinear taps, which are the cost --
 * and every lane then folds them into the running means, and in the second
 * pass into the paired sums, one after the other in list order: the result is
 * bitwise the sequential one. The reference returns -1 at the first entry
 * whose projection leaves the image, whatever the entries before it gave, so
 * "any entry leaves" is the same test. */
__device__ double
ncc_for_patch_warp (VisArgs const& a, int sub, short4 const* rim, int n_list,
    int ps, double const* cf, double const* theta, int px0, int py0, int lane)
{
    SurfaceDev const& sf = a.s;
    double const* Mt = sf.Mt + sub * 12;
    int const sw = sf.sub_dims[2 * sub], sh = sf.sub_dims[2 * sub + 1];
    float const* simg = a.color_subs[sub];
    xd means0[3], means1[3], counter[3];
    for (int c = 0; c < 3; ++c)
        means0[c] = means1[c] = counter[c] = xd(0.0);
    double const hi_x = static_cast<double>(sw - 2);
    double const hi_y = static_cast<double>(sh - 2);
    for (int base = 0; base < n_list; base += 32)
    {
        int const i = base + lane;
        bool out = false;
        double cm[3] = {0.0, 0.0, 0.0}, cs[3] = {0.0, 0.0, 0.0};
        if (i < n_list)
        {
            ListEntry const e = list_entry(rim, i, ps, cf, theta, px0, py0);
            Warp const c = warp_pixel<false>(Mt, (xd(e.x) + xd(0.5)).v,
                (xd(e.y) + xd(0.5)).v, e.depth, 0.0, 0.0);
            out = c.projx < 1 || c.projx > hi_x || c.projy < 1
                || c.projy > hi_y;
            if (!out)
            {
                size_t const mp = (static_cast<size_t>(static_cast<int>(e.y))
                    * sf.w + static_cast<int>(e.x)) * 3;
                for (int ch = 0; ch < 3; ++ch)
                {
                    cm[ch] = static_cast<double>(a.color_main[mp + ch]);
                    cs[ch] = static_cast<double>(linear_at_rgb(simg, sw, sh,
                        static_cast<float>(c.projx),
                        static_cast<float>(c.projy), ch));
                }
            }
        }
        if (__any_sync(0xffffffffu, out))
            return -1.0;
        int const m = min(32, n_list - base);
        for (int l = 0; l < m; ++l)
            for (int ch = 0; ch < 3; ++ch)
            {
                xd const vm(__shfl_sync(0xffffffffu, cm[ch], l));
                xd const vs(__shfl_sync(0xffffffffu, cs[ch], l));
                counter[ch] += xd(1.0);
                means0[ch] += (vm - means0[ch]) / counter[ch];
                means1[ch] += (vs - means1[ch]) / counter[ch];
            }
    }
    /* SSEVector::dot pairing as in ncc_for_patch_dev */
    xd s00(0.0), s11(0.0), s01(0.0);
    xd p00(0.0), p11(0.0), p01(0.0);
    int k = 0;
    for (int base = 0; base < n_list; base += 32)
    {
        int const i = base + lane;
        double d0[3] = {0.0, 0.0, 0.0}, d1[3] = {0.0, 0.0, 0.0};
        if (i < n_list)
        {
            ListEntry const e = list_entry(rim, i, ps, cf, theta, px0, py0);
            Warp const c = warp_pixel<false>(Mt, (xd(e.x) + xd(0.5)).v,
                (xd(e.y) + xd(0.5)).v, e.depth, 0.0, 0.0);
            size_t const mp = (static_cast<size_t>(static_cast<int>(e.y))
                * sf.w + static_cast<int>(e.x)) * 3;
            for (int ch = 0; ch < 3; ++ch)
            {
                d0[ch] = (xd(static_cast<double>(a.color_main[mp + ch]))
                    - means0[ch]).v;
                d1[ch] = (xd(static_cast<double>(linear_at_rgb(simg, sw, sh,
                    static_cast<float>(c.projx), static_cast<float>(c.projy),
                    ch))) - means1[ch]).v;
            }
        }
        int const m = min(32, n_list - base);
        for (int l = 0; l < m; ++l)
            for (int ch = 0; ch < 3; ++ch, ++k)
            {
                xd const v0(__shfl_sync(0xffffffffu, d0[ch], l));
                xd const v1(__shfl_sync(0xffffffffu, d1[ch], l));
                if ((k & 1) == 0)
                {
                    p00 = v0 * v0; p11 = v1 * v1; p01 = v0 * v1;
                }
                else
                {
                    s00 += p00 + v0 * v0;
                    s11 += p11 + v1 * v1;
                    s01 += p01 + v0 * v1;
                }
            }
    }
    if (k & 1)
    {
        s00 += p00; s11 += p11; s01 += p01;
    }
    xd const norm0 = xsqrt(s00), norm1 = xsqrt(s11);
    if ((norm0 + norm1).v < (xd(0.001) * xd(static_cast<double>(n_list))).v)
        return 1.0;
    return (s01 / (norm0 * norm1)).v;
}

/* second pass in the use_sgm = false mode: L lanes per PATCH, neighbours
 * in order, because the reference's member vectors `pixels` / `depths` carry
 * state from one neighbour to the next (:508, :514, :551, :579): after
 * ncc_for_patch ran they hold the patch AND its rim, and the next
 * neighbour's border and depth tests run over that longer list until a
 * neighbour passes them (which resets the vectors to the patch's pixels).
 * L = 32 serves patch sizes 128 and 256 (scales 7 and 8), where one thread
 * per patch would leave a few hundred threads to walk 16 K / 65 K pixels per
 * neighbour: the lanes take the list entries in turn for the border / depth
 * test (every entry passes) and the anisotropy (largest ratio), and
 * ncc_for_patch_warp keeps the NCC's sequential sums. */
template <int L>
__global__ void __launch_bounds__(128)
vis_patch_ncc_kernel (VisArgs const a)
{
    SurfaceDev const& sf = a.s;
    int const patch = (blockIdx.x * blockDim.x + threadIdx.x) / L;
    int const lane = threadIdx.x % L;
    if (patch >= sf.npx * sf.npy || !sf.patch_valid[patch])
        return;
    int const idx = patch % sf.npx, idy = patch / sf.npx;
    int const ps = sf.ps;
    double theta[16], cf[16];
    load_patch_theta(sf.nodes, sf.npx, idx, idy, theta);
    patch_coefficients(theta, cf);
    int const px0 = sf.start_x + idx * ps, py0 = sf.start_y + idy * ps;

    /* which of the eight rim lists: corners (:813-824), top (:828), left
     * (:844); the bottom and right conditions (:836, :852) compare pixel
     * coordinates with the patch's far corner and never hold */
    int const min0 = px0, min1 = py0, max0 = px0 + ps, max1 = py0 + ps;
    int shape = 0;
    if (min0 > 1 && max0 < sf.w - 2 && min1 > 1 && max1 < sf.h - 2)
        shape |= 1;
    if (min1 > 2)
        shape |= 2;
    if (min0 > 2)
        shape |= 4;
    short4 const* rim = a.rim + a.rim_off[shape];
    int const n_long = ps * ps + a.rim_off[shape + 1] - a.rim_off[shape];

    unsigned int mask = 0;
    bool extended = false;
    for (int sub = 0; sub < sf.n_sub; ++sub)
    {
        double const* Mt = sf.Mt + sub * 12;
        NeighbourTest const test(a, sub);
        int const n_list = extended ? n_long : ps * ps;
        bool success = true;
        for (int base = 0; base < n_list && success; base += L)
        {
            int const i = base + lane;
            bool pass = true;
            if (i < n_list)
            {
                ListEntry const e = list_entry(rim, i, ps, cf, theta, px0,
                    py0);
                pass = test.passes(warp_pixel<false>(Mt, (xd(e.x)
                    + xd(0.5)).v, (xd(e.y) + xd(0.5)).v, e.depth, 0.0, 0.0));
            }
            success = (L == 1) ? pass : __all_sync(0xffffffffu, pass);
        }
        if (!success)
            continue;
        extended = false;           /* :551 refills the vectors */
        double worst;
        if constexpr (L == 1)
            worst = warp_anisotropy(cf, Mt, px0, py0, ps);
        else
        {
            worst = 0.0;
            for (int pid = lane; pid < ps * ps; pid += L)
            {
                double const ratio = warp_anisotropy_at(cf, Mt, px0, py0, ps,
                    pid);
                worst = (worst < ratio) ? ratio : worst;    /* std::max */
            }
            for (int off = L / 2; off > 0; off >>= 1)
            {
                double const other = __shfl_xor_sync(0xffffffffu, worst, off);
                worst = (worst < other) ? other : worst;
            }
        }
        if (worst > 8.0)
            continue;
        extended = true;            /* ncc_for_patch leaves the rim in them */
        double const ncc = (L == 1)
            ? ncc_for_patch_dev(a, sub, rim, n_long, ps, cf, theta, px0, py0)
            : ncc_for_patch_warp(a, sub, rim, n_long, ps, cf, theta, px0, py0,
                lane);
        if (ncc < 0)
            continue;
        mask |= 1u << sub;
    }
    if (lane == 0)
        a.vis_mask[patch] = mask;
}

/* :585-600: patches no neighbour sees are deleted */
__global__ void
vis_finalize_kernel (VisArgs const a, uint8_t* patch_valid,
    uint32_t* counts)
{
    int const patch = blockIdx.x * blockDim.x + threadIdx.x;
    if (patch >= a.s.npx * a.s.npy)
        return;
    uint32_t n = 0;
    if (patch_valid[patch])
    {
        n = __popc(a.vis_mask[patch]);
        if (n == 0)
        {
            patch_valid[patch] = 0;
            atomicAdd(a.counters, 1ull);
        }
    }
    counts[patch] = n;
}

/* Surface::remove_nodes_without_patch: a node goes when none of the patches
 * around it (those inside the grid) is left */
__global__ void
remove_nodes_kernel (int npx, int npy, uint8_t const* __restrict__ patch_valid,
    uint8_t* __restrict__ node_valid)
{
    int const node = blockIdx.x * blockDim.x + threadIdx.x;
    if (node >= (npx + 1) * (npy + 1) || !node_valid[node])
        return;
    int const ix = node % (npx + 1), iy = node / (npx + 1);
    bool any = false;
    for (int dy = -1; dy <= 0; ++dy)
        for (int dx = -1; dx <= 0; ++dx)
        {
            int const px = ix + dx, py = iy + dy;
            if (px < 0 || py < 0 || px >= npx || py >= npy)
                continue;
            any = any || patch_valid[py * npx + px];
        }
    if (!any)
        node_valid[node] = 0;
}

/* exclusive prefix sum of counts[0..n) into off[0..n), and the total into
 * off[n]; one block */
__global__ void __launch_bounds__(1024)
scan_kernel (uint32_t const* __restrict__ counts, uint32_t* __restrict__ off,
    int n)
{
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry;
    if (threadIdx.x == 0)
        s_carry = 0;
    __syncthreads();
    int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int base = 0; base < n; base += 1024)
    {
        int const i = base + threadIdx.x;
        uint32_t const v = (i < n) ? counts[i] : 0;
        uint32_t inc = v;
        for (int o = 1; o < 32; o <<= 1)
        {
            uint32_t const u = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o)
                inc += u;
        }
        if (lane == 31)
            s_warp[warp] = inc;
        __syncthreads();
        if (warp == 0)
        {
            uint32_t w = s_warp[lane];
            for (int o = 1; o < 32; o <<= 1)
            {
                uint32_t const u = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o)
                    w += u;
            }
            s_warp[lane] = w;
        }
        __syncthreads();
        uint32_t const before = s_carry + (warp > 0 ? s_warp[warp - 1] : 0)
            + inc - v;
        if (i < n)
            off[i] = before;
        __syncthreads();
        if (threadIdx.x == 1023)
            s_carry = before + v;
        __syncthreads();
    }
    if (threadIdx.x == 0)
        off[n] = s_carry;
}

/* the lists themselves, ascending neighbour id like the reference's
 * push_back order */
__global__ void
vis_lists_kernel (int n_patches, unsigned int const* __restrict__ mask,
    uint32_t const* __restrict__ counts, uint32_t const* __restrict__ off,
    uint8_t* __restrict__ ids)
{
    int const patch = blockIdx.x * blockDim.x + threadIdx.x;
    if (patch >= n_patches || counts[patch] == 0)
        return;
    unsigned int m = mask[patch];
    uint32_t o = off[patch];
    while (m)
    {
        int const sub = __ffs(m) - 1;
        ids[o++] = static_cast<uint8_t>(sub);
        m &= m - 1;
    }
}

/* ------------------------------------------------------------------ */

struct CutArgs
{
    SurfaceDev s;
    float inv[9];                   /* inverse calibration of the main view */
    uint8_t* patch_valid;           /* written */
    unsigned long long* counters;
};

/* depth discontinuities, :367-400 */
__global__ void
cut_depth_kernel (CutArgs const a)
{
    SurfaceDev const& sf = a.s;
    int const patch = blockIdx.x * blockDim.x + threadIdx.x;
    if (patch >= sf.npx * sf.npy || !a.patch_valid[patch])
        return;
    int const idx = patch % sf.npx, idy = patch / sf.npx;
    double dep[4];
    for (int nd = 0; nd < 4; ++nd)
    {
        int const node = (idy + (nd >> 1)) * (sf.npx + 1) + idx + (nd & 1);
        dep[nd] = sf.nodes[static_cast<size_t>(node) * 4];
    }
    /* std::multimap ordering: smallest key first, equal keys in insertion
     * order -> first minimum, last maximum */
    int lo = 0, hi = 0;
    for (int i = 1; i < 4; ++i)
    {
        if (dep[i] < dep[lo]) lo = i;
        if (!(dep[i] < dep[hi])) hi = i;
    }
    double dd_factor = 5.0;
    if (lo + hi == 3)
        dd_factor = (xd(dd_factor) * xd(1.41421356237309504880168872420969808)).v;
    /* v = invproj * (x + 0.5, y + 0.5, 1) and its norm, in fp32 */
    float const fx = __fadd_rn(static_cast<float>(
        static_cast<double>(sf.start_x + idx * sf.ps)), 0.5f);
    float const fy = __fadd_rn(static_cast<float>(
        static_cast<double>(sf.start_y + idy * sf.ps)), 0.5f);
    float v[3];
    for (int r = 0; r < 3; ++r)
    {
        float sum = 0.0f;
        sum = __fadd_rn(sum, __fmul_rn(a.inv[r * 3 + 0], fx));
        sum = __fadd_rn(sum, __fmul_rn(a.inv[r * 3 + 1], fy));
        sum = __fadd_rn(sum, __fmul_rn(a.inv[r * 3 + 2], 1.0f));
        v[r] = sum;
    }
    float sq = 0.0f;
    for (int r = 0; r < 3; ++r)
        sq = __fadd_rn(sq, __fmul_rn(v[r], v[r]));
    float const norm = __fsqrt_rn(sq);
    double const threshold = (xd(dd_factor) * xd(dep[lo])
        * xd(static_cast<double>(a.inv[0]))
        * xd(static_cast<double>(sf.ps)) / xd(static_cast<double>(norm))).v;
    double const dist = (xd(dep[hi]) - xd(dep[lo])).v;
    if (dist > threshold)
    {
        a.patch_valid[patch] = 0;
        atomicAdd(a.counters, 1ull);
    }
}

/* a patch at the rim (:402-412): one of its nodes has more than one of its
 * eight neighbours missing (neighbours outside the grid count as missing) */
__device__ __forceinline__ bool
patch_at_rim (SurfaceDev const& sf, int idx, int idy)
{
    int const ns = sf.npx + 1;
    bool rim = false;
    for (int nd = 0; nd < 4 && !rim; ++nd)
    {
        int const nx = idx + (nd & 1), ny = idy + (nd >> 1);
        int present = 0;
        for (int dy = -1; dy < 2; ++dy)
            for (int dx = -1; dx < 2; ++dx)
            {
                if (dx == 0 && dy == 0)
                    continue;
                int const qx = nx + dx, qy = ny + dy;
                if (qx < 0 || qy < 0 || qx > sf.npx || qy > sf.npy)
                    continue;
                present += sf.node_valid[qy * ns + qx] ? 1 : 0;
            }
        rim = (8 - present) > 1;
    }
    return rim;
}

/* one term of mse_for_patch (:760-788): pixel pid of the patch against
 * neighbour sub, |grad_main - J grad_sub| */
__device__ __forceinline__ xd
mse_term (SurfaceDev const& sf, double const* cf, int px0, int py0, int ps,
    int pid, int sub)
{
    int const i = pid % ps, j = pid / ps;
    PatchSample const smp = patch_sample<true>(cf, i, j, ps);
    size_t const pix = static_cast<size_t>(py0 + j) * sf.w + (px0 + i);
    xd const gmx(static_cast<double>(sf.main_grad[2 * pix]));
    xd const gmy(static_cast<double>(sf.main_grad[2 * pix + 1]));
    Warp const c = warp_pixel<true>(sf.Mt + sub * 12, px0 + i + 0.5,
        py0 + j + 0.5, smp.w, smp.wx, smp.wy);
    float tap[5];
    tap_neighbour(sf.sub_texels[sub], sf.sub_dims[2 * sub],
        sf.sub_dims[2 * sub + 1], c.projx, c.projy, tap);
    xd const gx(static_cast<double>(tap[0]));
    xd const gy(static_cast<double>(tap[1]));
    /* diff = grad_main - jac * grad_sub; error += |diff| */
    xd const dx = gmx - (xd(0.0) + xd(c.jac[0]) * gx + xd(c.jac[1]) * gy);
    xd const dy = gmy - (xd(0.0) + xd(c.jac[2]) * gx + xd(c.jac[3]) * gy);
    return xsqrt(xd(0.0) + dx * dx + dy * dy);
}

/* high photometric error at the rim of the surface, :402-428 with
 * mse_for_patch :747-793; L lanes per patch (32 at the coarse scales, see
 * vis_patch_kernel). mse_for_patch is a sequential sum (pixels outer,
 * neighbours inner); the lanes evaluate L terms at a time and the terms are
 * then added one after the other in that order (every lane keeps the same
 * running sum), so the sum is bitwise the one-thread sum. */
template <int L>
__global__ void __launch_bounds__(128)
cut_border_kernel (CutArgs const a)
{
    SurfaceDev const& sf = a.s;
    int const patch = (blockIdx.x * blockDim.x + threadIdx.x) / L;
    int const lane = threadIdx.x % L;
    if (patch >= sf.npx * sf.npy || !a.patch_valid[patch])
        return;
    int const idx = patch % sf.npx, idy = patch / sf.npx;
    if (!patch_at_rim(sf, idx, idy))
        return;
    double theta[16], cf[16];
    load_patch_theta(sf.nodes, sf.npx, idx, idy, theta);
    patch_coefficients(theta, cf);
    int const ps = sf.ps;
    int const px0 = sf.start_x + idx * ps, py0 = sf.start_y + idy * ps;
    uint32_t const v0 = sf.vis_off[patch];
    int const n = static_cast<int>(sf.vis_off[patch + 1] - v0);
    int const total = ps * ps * n;
    xd error(0.0);
    if constexpr (L == 1)
    {
        for (int pid = 0; pid < ps * ps; ++pid)
            for (int k = 0; k < n; ++k)
                error += mse_term(sf, cf, px0, py0, ps, pid,
                    sf.vis_ids[v0 + k]);
    }
    else
    {
        for (int base = 0; base < total; base += L)
        {
            int const t = base + lane;
            double term = 0.0;
            if (t < total)
                term = mse_term(sf, cf, px0, py0, ps, t / n,
                    sf.vis_ids[v0 + t % n]).v;
            for (int l = 0; l < min(L, total - base); ++l)
                error += xd(__shfl_sync(0xffffffffu, term, l));
        }
    }
    double const counter = static_cast<double>(total);
    double const mse = (total == 0) ? 1.0 : (error / xd(counter)).v;
    if (lane == 0 && mse > 0.05)
    {
        a.patch_valid[patch] = 0;
        atomicAdd(a.counters, 1ull);
    }
}

} /* namespace */

/* ------------------------------------------------------------------ */

void
launch_remove_nodes (smvsb_ctx* c)
{
    remove_nodes_kernel<<<(c->n_nodes + 255) / 256, 256, 0, c->stream>>>(
        c->npx, c->npy, c->patch_valid.p, c->node_valid.p);
    CUDA_CHECK(cudaGetLastError());
    smvsb::count_launches(c, 1);
}

void
launch_exclusive_scan (smvsb_ctx* c, uint32_t const* counts, uint32_t* off,
    int n)
{
    scan_kernel<<<1, 1024, 0, c->stream>>>(counts, off, n);
    CUDA_CHECK(cudaGetLastError());
    smvsb::count_launches(c, 1);
}

uint64_t
run_visibility (smvsb_ctx* c, float const* sgm_depth_host)
{
    size_t const npix = static_cast<size_t>(c->w) * c->h;
    c->sgm_depth.reserve(npix);
    CUDA_CHECK(cudaMemcpyAsync(c->sgm_depth.p, sgm_depth_host,
        npix * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    return run_visibility_device(c);
}

/* The pixel lists ncc_for_patch builds (lib/depth_optimizer.cc:803-859),
 * relative to the patch origin: entries beyond the patch's own ps * ps pixels
 * for each of the eight combinations of (corners fit, top rim fits, left rim
 * fits). Run exactly like the reference: the loop walks the list while it
 * grows. Where the depth comes from (patch pixel index, or -1 - corner) is
 * 32 bits, low half in z and high half in w: at patch size 256 a pixel index
 * reaches 65 280. */
static void
build_rim_lists (int ps, std::vector<short4>* out, int* off)
{
    out->clear();
    for (int shape = 0; shape < 8; ++shape)
    {
        off[shape] = static_cast<int>(out->size());
        struct E { int x, y, src; };
        std::vector<E> list;
        for (int i = 0; i < ps * ps; ++i)
            list.push_back(E{ i % ps, i / ps, i });
        int const min0 = 0, min1 = 0, max0 = ps, max1 = ps;
        if (shape & 1)
        {
            list.push_back(E{ min0 - 1, min1 - 1, -1 });
            list.push_back(E{ max0 + 1, min1 - 1, -2 });
            list.push_back(E{ min0 - 1, max1 + 1, -3 });
            list.push_back(E{ max0 + 1, max1 + 1, -4 });
        }
        for (std::size_t i = 0; i < list.size(); ++i)
        {
            E const e = list[i];
            if ((shape & 2) && e.y == min1)
            {
                list.push_back(E{ e.x, e.y - 2, e.src });
                list.push_back(E{ e.x, e.y - 1, e.src });
            }
            /* :836 / :852 compare with the far corner (max = origin + ps);
             * no list entry ever lies on it, whatever the image size */
            if (e.y == max1 || e.x == max0)
                throw smvsb::Error(SMVSB_ERR_INVALID,
                    "rim list: bottom / right rule would fire");
            if ((shape & 4) && e.x == min0)
            {
                list.push_back(E{ e.x - 2, e.y, e.src });
                list.push_back(E{ e.x - 1, e.y, e.src });
            }
        }
        for (std::size_t i = static_cast<std::size_t>(ps) * ps;
            i < list.size(); ++i)
        {
            unsigned const src = static_cast<unsigned>(list[i].src);
            out->push_back(make_short4(static_cast<short>(list[i].x),
                static_cast<short>(list[i].y),
                static_cast<short>(static_cast<uint16_t>(src & 0xffffu)),
                static_cast<short>(static_cast<uint16_t>(src >> 16))));
        }
    }
    off[8] = static_cast<int>(out->size());
}

uint64_t
run_visibility_ncc (smvsb_ctx* c)
{
    if (c->rim_ps != c->ps)
    {
        std::vector<short4> lists;
        build_rim_lists(c->ps, &lists, c->rim_off);
        c->rim_lists.reserve(lists.size() + 1);
        CUDA_CHECK(cudaMemcpyAsync(c->rim_lists.p, lists.data(),
            lists.size() * sizeof(short4), cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));   /* `lists` goes away */
        c->rim_ps = c->ps;
    }
    return run_visibility_device(c, false);
}

uint64_t
run_visibility_device (smvsb_ctx* c, bool use_sgm)
{
    size_t const npix = static_cast<size_t>(c->w) * c->h;
    int const np = c->n_patches;

    /* caches: (w + 1) x (h + 1) per neighbour, :441-450 */
    std::vector<unsigned long long> zoff(c->n_sub + 1, 0);
    for (int s = 0; s < c->n_sub; ++s)
        zoff[s + 1] = zoff[s] + static_cast<unsigned long long>(
            c->subs[s].w + 1) * (c->subs[s].h + 1);
    c->zbuf.reserve(zoff[c->n_sub]);
    c->zoff.reserve(c->n_sub + 1);
    CUDA_CHECK(cudaMemcpyAsync(c->zoff.p, zoff.data(),
        zoff.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice,
        c->stream));
    c->image_out.reserve(npix * 3);
    CUDA_CHECK(cudaMemsetAsync(c->image_out.p, 0, npix * sizeof(float),
        c->stream));
    launch_render_depth(c, c->image_out.p);
    c->vis_mask.reserve(np);
    CUDA_CHECK(cudaMemsetAsync(c->vis_mask.p, 0, np * sizeof(unsigned int),
        c->stream));
    c->vis_counts.reserve(np);
    c->counters.reserve(4);
    CUDA_CHECK(cudaMemsetAsync(c->counters.p, 0,
        4 * sizeof(unsigned long long), c->stream));
    c->vis_ids.reserve(static_cast<size_t>(np) * c->n_sub + 1);
    c->vis_off.reserve(static_cast<size_t>(np) + 1);

    VisArgs a;
    a.s = surface_args(c);
    a.zbuf = c->zbuf.p; a.zoff = c->zoff.p;
    a.surf_depth = c->image_out.p;
    a.sgm_depth = use_sgm ? c->sgm_depth.p : nullptr;
    a.vis_mask = c->vis_mask.p; a.counters = c->counters.p;
    a.color_main = use_sgm ? nullptr : c->color_main.p;
    a.color_subs = use_sgm ? nullptr : c->color_ptrs.p;
    a.rim = use_sgm ? nullptr : c->rim_lists.p;
    for (int i = 0; i < 9; ++i)
        a.rim_off[i] = use_sgm ? 0 : c->rim_off[i];

    zbuf_fill_kernel<<<c->num_sms * 8, 256, 0, c->stream>>>(c->zbuf.p,
        zoff[c->n_sub], float_key(ZBUF_FAR));
    zbuf_scatter_kernel<<<static_cast<unsigned int>((npix + 255) / 256), 256,
        0, c->stream>>>(a);
    int const nt = np * c->n_sub;
    if (use_sgm && c->ps >= 8)
        vis_patch_kernel<32><<<(nt + 3) / 4, 128, 0, c->stream>>>(a);
    else if (use_sgm)
        vis_patch_kernel<1><<<(nt + 127) / 128, 128, 0, c->stream>>>(a);
    else if (c->ps >= 128)
        vis_patch_ncc_kernel<32><<<(np + 3) / 4, 128, 0, c->stream>>>(a);
    else
        vis_patch_ncc_kernel<1><<<(np + 127) / 128, 128, 0, c->stream>>>(a);
    vis_finalize_kernel<<<(np + 255) / 256, 256, 0, c->stream>>>(a,
        c->patch_valid.p, c->vis_counts.p);
    CUDA_CHECK(cudaGetLastError());
    launch_remove_nodes(c);
    launch_exclusive_scan(c, c->vis_counts.p, c->vis_off.p, np);
    vis_lists_kernel<<<(np + 255) / 256, 256, 0, c->stream>>>(np,
        c->vis_mask.p, c->vis_counts.p, c->vis_off.p, c->vis_ids.p);
    smvsb::count_launches(c, 5);
    CUDA_CHECK(cudaGetLastError());

    unsigned long long removed = 0;
    CUDA_CHECK(cudaMemcpyAsync(&removed, c->counters.p, sizeof(removed),
        cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return removed;
}

uint64_t
run_cut_boundaries (smvsb_ctx* c, float const* inv_calib)
{
    c->counters.reserve(4);
    CUDA_CHECK(cudaMemsetAsync(c->counters.p, 0,
        4 * sizeof(unsigned long long), c->stream));
    CutArgs a;
    a.s = surface_args(c);
    for (int i = 0; i < 9; ++i)
        a.inv[i] = inv_calib[i];
    a.patch_valid = c->patch_valid.p;
    a.counters = c->counters.p;
    int const np = c->n_patches;
    cut_depth_kernel<<<(np + 255) / 256, 256, 0, c->stream>>>(a);
    if (c->ps >= 8)
        cut_border_kernel<32><<<(np + 3) / 4, 128, 0, c->stream>>>(a);
    else
        cut_border_kernel<1><<<(np + 127) / 128, 128, 0, c->stream>>>(a);
    CUDA_CHECK(cudaGetLastError());
    launch_remove_nodes(c);
    smvsb::count_launches(c, 2);
    unsigned long long deleted = 0;
    CUDA_CHECK(cudaMemcpyAsync(&deleted, c->counters.p, sizeof(deleted),
        cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return deleted;
}

} /* namespace smvsb */

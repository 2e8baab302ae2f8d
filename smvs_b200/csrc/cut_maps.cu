/*
 * cut_maps.cu -- MeshGenerator::cut_depth_maps (lib/mesh_generator.cc:25-158)
 * on the device: the cross-view consistency cut that follows the per-view
 * optimisation (SURVEY.md section 8f, "next" row 4). For every pixel of every
 * depth map the 3-D point is projected into all other views; the depth is
 * dropped when it faces away from its own camera, when a view that sees the
 * point much better disagrees, or when the views that agree with it do not
 * outweigh those it occludes.
 *
 * Everything is fp32 with the reference's operation order (math::Vector /
 * Matrix operators, mve::geom::pixel_3dpos, ViewProjection::get_proj /
 * get_surface_power, :302-344) and no contraction, the three comparisons the
 * reference makes in double (:118, :121, :123-128) are made in double: the
 * decisions are the CPU's. The camera matrices come from the host (the
 * reference computes them with MVE's CameraInfo; the kernel only consumes
 * them).
 *
 * Scenes larger than one device: each target view i is independent (:60-148)
 * and reads only inputs, so the work is split three ways without changing a
 * bit of the result.
 *  - Workers: one host thread per entry of a device list takes target views
 *    from a shared counter and keeps a *target group* (depth, normals, z-depth,
 *    per-pixel state) resident on its device.
 *  - Source chunks: the source views j the group needs are streamed through a
 *    ring of slots in ascending j. Each target pixel carries its consistency
 *    sum and a hard-cut flag from one chunk launch to the next, so the sum is
 *    accumulated in the reference's order and a pixel that hit the break
 *    (:137-142) takes no further work, however the views are chunked.
 *  - Culling: a 16x16 tile of target pixels gets the world-space box of the
 *    fp32 positions the cut kernel computes; a (tile, j) pair is dropped only
 *    when the box proves that every pixel of the tile would `continue` at the
 *    `proj.z < 0` or the bounds test (pair_culled). The union over tiles is the
 *    view-level list: a source view no target of the group needs is never
 *    uploaded.
 */
#include <algorithm>
#include <atomic>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "common.cuh"

namespace smvsb {

namespace {

constexpr int kTile = 16;            /* target pixels per tile edge = CTA */

struct CutView
{
    int w, h;
    float const* cut;        /* depth as given (MVE convention: along the ray) */
    float const* zdepth;     /* after depthmap_convert_conventions(.., false) */
    float const* normals;    /* world space, w*h*3 */
    float invproj[9], ctw[16], KR[9], t[3];
};

/* What the cull test needs of a source view. */
struct CullCam
{
    float KR[9], t[3];
    int w, h;
};

/* World-space box of the valid pixels of one tile. */
struct TileBox
{
    float lo[3], hi[3];
    unsigned int valid;      /* pixels with depth */
    unsigned int finite;     /* 0: some position is inf / nan: never culled */
};

/* A target view of the group and its state across chunk launches. */
struct CutTarget
{
    CutView v;
    float* acc;              /* consistency; the cut map after finalize */
    uint8_t* done;           /* 1: hard cut (:137-142), no further work */
    uint32_t const* keep;    /* tiles x nwords: source views not culled */
    int nwords, tiles_x;
};

struct f3
{
    float x, y, z;
};

/* std::inner_product(a, a + 3, b, 0.f) */
__device__ __forceinline__ float
dot3 (float const* a, f3 const& b)
{
    float s = __fadd_rn(0.0f, __fmul_rn(a[0], b.x));
    s = __fadd_rn(s, __fmul_rn(a[1], b.y));
    return __fadd_rn(s, __fmul_rn(a[2], b.z));
}

__device__ __forceinline__ float
dot3 (f3 const& a, f3 const& b)
{
    float s = __fadd_rn(0.0f, __fmul_rn(a.x, b.x));
    s = __fadd_rn(s, __fmul_rn(a.y, b.y));
    return __fadd_rn(s, __fmul_rn(a.z, b.z));
}

/* mve::geom::pixel_3dpos, then Matrix4f::mult(pos, 1.0f) with cam-to-world */
__device__ __forceinline__ f3
world_pos (CutView const& v, int x, int y, float depth)
{
    f3 const px = { __fadd_rn(static_cast<float>(x), 0.5f),
        __fadd_rn(static_cast<float>(y), 0.5f), 1.0f };
    f3 ray = { dot3(v.invproj, px), dot3(v.invproj + 3, px),
        dot3(v.invproj + 6, px) };
    float const n = __fsqrt_rn(dot3(ray, ray));
    ray.x = __fmul_rn(__fdiv_rn(ray.x, n), depth);
    ray.y = __fmul_rn(__fdiv_rn(ray.y, n), depth);
    ray.z = __fmul_rn(__fdiv_rn(ray.z, n), depth);
    f3 out;
    out.x = __fadd_rn(dot3(v.ctw, ray), v.ctw[3]);
    out.y = __fadd_rn(dot3(v.ctw + 4, ray), v.ctw[7]);
    out.z = __fadd_rn(dot3(v.ctw + 8, ray), v.ctw[11]);
    return out;
}

/* ViewProjection::get_proj, :314-321 */
__device__ __forceinline__ f3
get_proj (CutView const& v, f3 const& pos)
{
    f3 out;
    out.x = __fsub_rn(dot3(v.KR, pos), v.t[0]);
    out.y = __fsub_rn(dot3(v.KR + 3, pos), v.t[1]);
    out.z = __fsub_rn(dot3(v.KR + 6, pos), v.t[2]);
    return out;
}

/* ViewProjection::get_surface_power, :323-344 */
__device__ __forceinline__ float
surface_power (CutView const& v, f3 const& pos, f3 const& normal)
{
    f3 const p = get_proj(v, pos);
    float const denom = __fmul_rn(p.z, p.z);
    float ud[3], vd[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        ud[k] = __fdiv_rn(__fsub_rn(__fmul_rn(v.KR[k], p.z),
            __fmul_rn(v.KR[6 + k], p.x)), denom);
        vd[k] = __fdiv_rn(__fsub_rn(__fmul_rn(v.KR[3 + k], p.z),
            __fmul_rn(v.KR[6 + k], p.y)), denom);
    }
    f3 c;
    c.x = __fsub_rn(__fmul_rn(ud[1], vd[2]), __fmul_rn(ud[2], vd[1]));
    c.y = __fsub_rn(__fmul_rn(ud[2], vd[0]), __fmul_rn(ud[0], vd[2]));
    c.z = __fsub_rn(__fmul_rn(ud[0], vd[1]), __fmul_rn(ud[1], vd[0]));
    return -dot3(normal, c);
}

/* mve::image::depthmap_convert_conventions<float>(dm, invproj, false) */
__global__ void
to_zdepth_kernel (int w, int h, float const* __restrict__ in, float i0,
    float i1, float i2, float i3, float i4, float i5, float i6, float i7,
    float i8, float* __restrict__ out)
{
    int const x = blockIdx.x * blockDim.x + threadIdx.x;
    int const y = blockIdx.y;
    if (x >= w)
        return;
    float const m[9] = { i0, i1, i2, i3, i4, i5, i6, i7, i8 };
    f3 const px = { __fadd_rn(static_cast<float>(x), 0.5f),
        __fadd_rn(static_cast<float>(y), 0.5f), 1.0f };
    f3 const ray = { dot3(m, px), dot3(m + 3, px), dot3(m + 6, px) };
    double const len = static_cast<double>(__fsqrt_rn(dot3(ray, ray)));
    size_t const i = static_cast<size_t>(y) * w + x;
    out[i] = static_cast<float>(__dmul_rn(static_cast<double>(in[i]),
        __ddiv_rn(1.0, len)));
}

/* Box of the fp32 world positions of one tile's pixels with depth -- the
 * positions cut_chunk_kernel computes, by the same function. */
__global__ void __launch_bounds__(kTile * kTile)
tile_box_kernel (CutView const V, TileBox* __restrict__ boxes,
    unsigned long long* __restrict__ valid_total)
{
    int const x = blockIdx.x * kTile + threadIdx.x;
    int const y = blockIdx.y * kTile + threadIdx.y;
    float lo[3] = { INFINITY, INFINITY, INFINITY };
    float hi[3] = { -INFINITY, -INFINITY, -INFINITY };
    unsigned int valid = 0, bad = 0;
    if (x < V.w && y < V.h)
    {
        float const d = V.cut[static_cast<size_t>(y) * V.w + x];
        if (d != 0.0f)
        {
            f3 const p = world_pos(V, x, y, d);
            valid = 1;
            bad = !(isfinite(p.x) && isfinite(p.y) && isfinite(p.z));
            lo[0] = hi[0] = p.x; lo[1] = hi[1] = p.y; lo[2] = hi[2] = p.z;
        }
    }
    unsigned const full = 0xffffffffu;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            lo[k] = fminf(lo[k], __shfl_xor_sync(full, lo[k], o));
            hi[k] = fmaxf(hi[k], __shfl_xor_sync(full, hi[k], o));
        }
    valid = __reduce_add_sync(full, valid);
    bad = __reduce_or_sync(full, bad);
    __shared__ float s_lo[8][3], s_hi[8][3];
    __shared__ unsigned int s_valid[8], s_bad[8];
    int const t = threadIdx.y * kTile + threadIdx.x;
    int const warp = t >> 5;
    if ((t & 31) == 0)
    {
        for (int k = 0; k < 3; ++k) { s_lo[warp][k] = lo[k]; s_hi[warp][k] = hi[k]; }
        s_valid[warp] = valid;
        s_bad[warp] = bad;
    }
    __syncthreads();
    if (t == 0)
    {
        TileBox b;
        b.valid = 0;
        unsigned int any_bad = 0;
        for (int k = 0; k < 3; ++k) { b.lo[k] = INFINITY; b.hi[k] = -INFINITY; }
        for (int wi = 0; wi < 8; ++wi)
        {
            for (int k = 0; k < 3; ++k)
            {
                b.lo[k] = fminf(b.lo[k], s_lo[wi][k]);
                b.hi[k] = fmaxf(b.hi[k], s_hi[wi][k]);
            }
            b.valid += s_valid[wi];
            any_bad |= s_bad[wi];
        }
        b.finite = any_bad ? 0u : 1u;
        boxes[blockIdx.y * gridDim.x + blockIdx.x] = b;
        if (b.valid)
            atomicAdd(valid_total, static_cast<unsigned long long>(b.valid));
    }
}

/*
 * True when no pixel of the tile can pass the `proj.z < 0` test and the bounds
 * test of source view c (:103-110), i.e. every pixel would `continue` there.
 *
 * Soundness. Every position p the cut kernel computes for a valid pixel of
 * the tile lies in the box [lo, hi] (tile_box_kernel takes min / max of those
 * very fp32 values; a tile with a non-finite position is never culled).
 *  1. get_proj computes each component as fl(fl(fl(fl(a0 p0) + fl(a1 p1))
 *     + fl(a2 p2)) - t): each term passes through at most 4 roundings, so the
 *     result is within gamma_4 * (|a0 p0| + |a1 p1| + |a2 p2| + |t|) of the
 *     exact value (gamma_4 = 4u / (1 - 4u), u = 2^-24), plus at most a few
 *     2^-149 where products underflow. The exact value of a linear function
 *     over a box lies between the sums of the per-term minima / maxima; those
 *     products of two floats are exact in double, their sums are within a
 *     few 2^-53 relative. [s_lo - e, s_hi + e] with e = 8u * magnitude + 1e-30
 *     therefore contains every computed component (magnitudes beyond 1e30 are
 *     not culled: fp32 may overflow there).
 *  2. z: if s_hi + e < 0 every computed proj.z is < 0: culled. proj.z == 0 is
 *     not behind the camera, so a box whose z interval reaches 0 from either
 *     side is never culled beyond this point.
 *  3. With Z0 = z lower bound > 0, x / z over independent intervals X x Z is
 *     monotone in each argument, so its extremes are at interval corners (a
 *     superset of the box's linear-fractional image, whose extremes are at the
 *     box corners). Rounding of the fp32 division is monotone and within u
 *     relative; the double corner quotients are within 2^-53: q_lo / q_hi
 *     widened by 2u relative (and 1e-30 absolute) bound every computed
 *     quotient.
 *  4. static_cast<int> truncates toward zero: a quotient in (-1, 0) lands on
 *     column 0, which is IN bounds. Culled are q_hi < -1 (every index <= -1;
 *     out-of-range conversions give INT_MIN on the CPU, also < 0) and
 *     q_lo >= w (every index >= w; the device saturates to INT_MAX >= w, the
 *     CPU gives INT_MIN < 0: out of bounds either way). The same for y and h.
 */
__device__ bool
pair_culled (TileBox const& b, CullCam const& c)
{
    if (!b.finite || b.valid == 0)
        return b.valid == 0;
    double const u = 0x1p-24;
    double lo[3], hi[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
    {
        double const t = static_cast<double>(c.t[r]);
        double s_lo = -t, s_hi = -t, mag = fabs(t);
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            double const a = static_cast<double>(c.KR[3 * r + k]);
            double const p = a * static_cast<double>(b.lo[k]);
            double const q = a * static_cast<double>(b.hi[k]);
            s_lo += fmin(p, q);
            s_hi += fmax(p, q);
            mag += fmax(fabs(p), fabs(q));
        }
        if (!(mag < 1e30))
            return false;
        double const e = 8.0 * u * mag + 1e-30;
        lo[r] = s_lo - e;
        hi[r] = s_hi + e;
    }
    if (hi[2] < 0.0)
        return true;
    if (!(lo[2] > 0.0))
        return false;
    int const dims[2] = { c.w, c.h };
#pragma unroll
    for (int r = 0; r < 2; ++r)
    {
        double const q_hi = hi[r] >= 0.0 ? hi[r] / lo[2] : hi[r] / hi[2];
        double const q_lo = lo[r] >= 0.0 ? lo[r] / hi[2] : lo[r] / lo[2];
        double const q_hi_w = q_hi + 2.0 * u * fabs(q_hi) + 1e-30;
        double const q_lo_w = q_lo - 2.0 * u * fabs(q_lo) - 1e-30;
        if (q_hi_w < -1.0 || q_lo_w >= static_cast<double>(dims[r]))
            return true;
    }
    return false;
}

/* One warp per (tile, 32 source views): keep bits of the tile, the view-level
 * list of the target (OR over tiles) and the pairs left after culling. */
__global__ void __launch_bounds__(256)
cull_kernel (TileBox const* __restrict__ boxes, int n_tiles,
    CullCam const* __restrict__ cams, int n_views, int vi, int nwords,
    uint32_t* __restrict__ keep, uint32_t* __restrict__ needed,
    unsigned long long* __restrict__ pairs)
{
    int const gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int const lane = threadIdx.x & 31;
    if (gw >= n_tiles * nwords)
        return;
    int const tile = gw / nwords;
    int const word = gw - tile * nwords;
    int const j = word * 32 + lane;
    TileBox const b = boxes[tile];
    bool k = false;
    if (j < n_views && j != vi)
        k = !pair_culled(b, cams[j]);
    uint32_t const m = __ballot_sync(0xffffffffu, k);
    if (lane == 0)
    {
        keep[static_cast<size_t>(tile) * nwords + word] = m;
        if (m)
        {
            atomicOr(needed + word, m);
            atomicAdd(pairs, static_cast<unsigned long long>(__popc(m))
                * b.valid);
        }
    }
}

/*
 * The reference's loop over j (:95-144) for the source views of [j0, j1) that
 * the pixel's tile keeps, in ascending j. One CTA per tile: the list is the
 * same for all its threads, the loop does not diverge on it. The consistency
 * sum and the hard-cut flag carry over from the previous chunk.
 */
__global__ void __launch_bounds__(kTile * kTile)
cut_chunk_kernel (CutTarget const T, CutView const* __restrict__ views,
    int vi, int j0, int j1)
{
    CutView const& V = T.v;
    int const x = blockIdx.x * kTile + threadIdx.x;
    int const y = blockIdx.y * kTile + threadIdx.y;
    if (x >= V.w || y >= V.h)
        return;
    size_t const pix = static_cast<size_t>(y) * V.w + x;
    float const d = V.cut[pix];
    if (d == 0.0f || T.done[pix])
        return;
    f3 const pos = world_pos(V, x, y, d);
    f3 const normal = { V.normals[3 * pix], V.normals[3 * pix + 1],
        V.normals[3 * pix + 2] };
    float const sp = surface_power(V, pos, normal);
    float consistency = T.acc[pix];
    uint32_t const* keep = T.keep
        + static_cast<size_t>(blockIdx.y * T.tiles_x + blockIdx.x) * T.nwords;
    int const w_first = j0 >> 5, w_last = (j1 - 1) >> 5;
    for (int wd = w_first; wd <= w_last; ++wd)
    {
        uint32_t m = keep[wd];
        if (wd == w_first)
            m &= ~0u << (j0 & 31);
        if (wd == w_last && ((j1 - 1) & 31) != 31)
            m &= (1u << (((j1 - 1) & 31) + 1)) - 1u;
        while (m)
        {
            int const j = wd * 32 + __ffs(m) - 1;
            m &= m - 1u;
            if (j == vi)
                continue;
            CutView const& J = views[j];
            f3 const proj = get_proj(J, pos);
            if (proj.z < 0.0f)
                continue;
            int const xj = static_cast<int>(__fdiv_rn(proj.x, proj.z));
            int const yj = static_cast<int>(__fdiv_rn(proj.y, proj.z));
            if (xj < 0 || xj >= J.w || yj < 0 || yj >= J.h)
                continue;
            size_t const pj = static_cast<size_t>(yj) * J.w + xj;
            float const dm_j = J.zdepth[pj];
            if (dm_j == 0.0f)
                continue;
            float const sp_j = surface_power(J, pos, normal);
            f3 const pos_j = world_pos(J, xj, yj, J.cut[pj]);
            f3 const normal_j = { J.normals[3 * pj], J.normals[3 * pj + 1],
                J.normals[3 * pj + 2] };
            float const sp_jj = surface_power(J, pos_j, normal_j);
            double const z = static_cast<double>(proj.z);
            if (__dmul_rn(static_cast<double>(dm_j), 1.01) < z)
                continue;
            if (__dmul_rn(static_cast<double>(dm_j), 0.997) > z)
            {
                if (static_cast<double>(sp_jj) > __dmul_rn(0.5,
                    static_cast<double>(sp)))
                    consistency = __fsub_rn(consistency, sp_jj);
                continue;
            }
            double const twice = __dmul_rn(2.0, static_cast<double>(sp));
            if (static_cast<double>(sp_jj) > twice
                || static_cast<double>(sp_j) > twice)
            {
                T.done[pix] = 1;
                return;
            }
            consistency = __fadd_rn(consistency, sp_jj);
        }
    }
    T.acc[pix] = consistency;
}

/* :87-91 and :145-146: the cut map of the target, written over acc. */
__global__ void __launch_bounds__(kTile * kTile)
cut_finalize_kernel (CutTarget const T)
{
    CutView const& V = T.v;
    int const x = blockIdx.x * kTile + threadIdx.x;
    int const y = blockIdx.y * kTile + threadIdx.y;
    if (x >= V.w || y >= V.h)
        return;
    size_t const pix = static_cast<size_t>(y) * V.w + x;
    float const d = V.cut[pix];
    float result = d;
    if (d != 0.0f)
    {
        f3 const pos = world_pos(V, x, y, d);
        f3 const normal = { V.normals[3 * pix], V.normals[3 * pix + 1],
            V.normals[3 * pix + 2] };
        if (surface_power(V, pos, normal) < 0.0f || T.done[pix]
            || T.acc[pix] <= 0.0f)
            result = 0.0f;
    }
    T.acc[pix] = result;
}

std::mutex g_cut_lock;

constexpr size_t kAlign = 256;

size_t
align_up (size_t n)
{
    return (n + kAlign - 1) / kAlign * kAlign;
}

/* Device memory freed and taken again when a larger size is asked for. */
struct Arena
{
    uint8_t* p = nullptr;
    size_t cap = 0;

    Arena (void) = default;
    Arena (Arena const&) = delete;
    Arena& operator= (Arena const&) = delete;
    ~Arena (void) { release(); }

    void release (void)
    {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }

    void reserve (size_t n)
    {
        if (n <= cap)
            return;
        release();
        cudaError_t const e = cudaMalloc(&p, n);
        if (e != cudaSuccess)
        {
            p = nullptr;
            cudaGetLastError();
            throw Error(SMVSB_ERR_ALLOC, "smvsb_cut_depth_maps: cudaMalloc of "
                + std::to_string(n) + " bytes: " + cudaGetErrorString(e));
        }
        cap = n;
    }
};

/* The call's inputs and the work shared by its workers. */
struct Scene
{
    int n;
    int const* w;
    int const* h;
    float const* const* depth;
    float const* const* normals;
    float const* invproj9;
    float const* ctw16;
    float const* KR9;
    float const* t3;
    float* const* out;
    int nwords;              /* 32-view words of a keep / needed list */
    size_t max_pix;
    int group_cap;           /* targets per group: the workers share the views */
    std::atomic<int> next{0};
    std::atomic<bool> failed{false};
    std::mutex err_lock;
    int err_code = SMVSB_OK;
    std::string err_msg;

    size_t pix (int i) const { return static_cast<size_t>(w[i]) * h[i]; }
    int tiles_x (int i) const { return (w[i] + kTile - 1) / kTile; }
    int tiles (int i) const
    {
        return tiles_x(i) * ((h[i] + kTile - 1) / kTile);
    }

    /* device bytes of one target view of a group */
    size_t target_bytes (int i) const
    {
        size_t const p = pix(i);
        size_t const t = static_cast<size_t>(tiles(i));
        return 3 * align_up(p * 4) + align_up(p * 12) + align_up(p)
            + align_up(t * sizeof(TileBox)) + align_up(t * nwords * 4)
            + align_up(static_cast<size_t>(nwords) * 4);
    }

    /* device bytes of one source slot: cut, z-depth, normals */
    size_t slot_bytes (void) const
    {
        return 2 * align_up(max_pix * 4) + align_up(max_pix * 12);
    }

    /* view tables and counters of a worker */
    size_t fixed_bytes (void) const
    {
        return align_up(n * sizeof(CutView)) + align_up(n * sizeof(CullCam))
            + kAlign;
    }

    void fill_view (int i, CutView* v) const
    {
        v->w = w[i]; v->h = h[i];
        std::copy(invproj9 + 9 * i, invproj9 + 9 * i + 9, v->invproj);
        std::copy(ctw16 + 16 * i, ctw16 + 16 * i + 16, v->ctw);
        std::copy(KR9 + 9 * i, KR9 + 9 * i + 9, v->KR);
        std::copy(t3 + 3 * i, t3 + 3 * i + 3, v->t);
    }

    void fail (Error const& e)
    {
        std::lock_guard<std::mutex> g(err_lock);
        if (err_code == SMVSB_OK)
        {
            err_code = e.code;
            err_msg = e.msg;
        }
        failed = true;
    }
};

struct WorkerStats
{
    uint64_t valid = 0, pairs = 0, bytes = 0, launches = 0;
    int groups = 0, chunks = 0;
    double ms = 0.0;
};

/* One worker: a device, a budget, two streams and two pinned staging buffers
 * through which every map is uploaded. */
class Worker
{
public:
    Worker (Scene& s, int device, size_t budget)
        : S(s), dev(device), budget(budget) {}

    ~Worker (void)
    {
        if (copy) cudaStreamSynchronize(copy);
        if (st) cudaStreamSynchronize(st);
        for (int k = 0; k < 2; ++k)
        {
            if (stage[k]) cudaFreeHost(stage[k]);
            if (staged[k]) cudaEventDestroy(staged[k]);
        }
        for (cudaEvent_t e : slot_free) cudaEventDestroy(e);
        if (h_views) cudaFreeHost(h_views);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
        if (copy) cudaStreamDestroy(copy);
        if (st) cudaStreamDestroy(st);
    }

    void run (void);

    WorkerStats stats;

private:
    struct Target
    {
        int i;
        float* cut; float* z; float* nrm; float* acc;
        uint8_t* done;
        TileBox* boxes;
        uint32_t* keep;
        uint32_t* needed;
        std::vector<uint32_t> h_needed;
    };

    void upload (int v, float* d_cut, float* d_nrm, float* d_z,
        cudaEvent_t wait);
    CutTarget cut_target (Target const& T) const;
    void run_group (std::vector<int> const& group);

    Scene& S;
    int dev;
    size_t budget;
    cudaStream_t st = nullptr, copy = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float* stage[2] = { nullptr, nullptr };
    cudaEvent_t staged[2] = { nullptr, nullptr };
    uint64_t n_staged = 0;
    std::vector<cudaEvent_t> slot_free;
    CutView* h_views = nullptr;          /* pinned copy of the view table */
    Arena fixed, targets, slots;
    CutView* d_views = nullptr;
    CullCam* d_cams = nullptr;
    unsigned long long* d_count = nullptr;    /* valid pixels, pairs kept */
};

/* Host map -> pinned staging -> device on the copy stream (after `wait`, the
 * event that frees the destination); the z-depth on the compute stream. */
void
Worker::upload (int v, float* d_cut, float* d_nrm, float* d_z,
    cudaEvent_t wait)
{
    size_t const n = S.pix(v);
    int const k = static_cast<int>(n_staged++ & 1);
    CUDA_CHECK(cudaEventSynchronize(staged[k]));
    std::memcpy(stage[k], S.depth[v], n * sizeof(float));
    std::memcpy(stage[k] + n, S.normals[v], 3 * n * sizeof(float));
    if (wait)
        CUDA_CHECK(cudaStreamWaitEvent(copy, wait, 0));
    CUDA_CHECK(cudaMemcpyAsync(d_cut, stage[k], n * sizeof(float),
        cudaMemcpyHostToDevice, copy));
    CUDA_CHECK(cudaMemcpyAsync(d_nrm, stage[k] + n, 3 * n * sizeof(float),
        cudaMemcpyHostToDevice, copy));
    CUDA_CHECK(cudaEventRecord(staged[k], copy));
    CUDA_CHECK(cudaStreamWaitEvent(st, staged[k], 0));
    float const* m = S.invproj9 + 9 * v;
    dim3 const grid((S.w[v] + 127) / 128, S.h[v]);
    to_zdepth_kernel<<<grid, 128, 0, st>>>(S.w[v], S.h[v], d_cut,
        m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7], m[8], d_z);
    CUDA_CHECK(cudaGetLastError());
    stats.bytes += 16 * n;
    stats.launches += 1;
}

/* The chunk and finalize kernels' view of a target of the group. */
CutTarget
Worker::cut_target (Target const& T) const
{
    CutTarget ct;
    S.fill_view(T.i, &ct.v);
    ct.v.cut = T.cut; ct.v.zdepth = T.z; ct.v.normals = T.nrm;
    ct.acc = T.acc; ct.done = T.done; ct.keep = T.keep;
    ct.nwords = S.nwords; ct.tiles_x = S.tiles_x(T.i);
    return ct;
}

void
Worker::run (void)
{
    CUDA_CHECK(cudaSetDevice(dev));
    CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
    CUDA_CHECK(cudaEventCreate(&ev0));
    CUDA_CHECK(cudaEventCreate(&ev1));
    for (int k = 0; k < 2; ++k)
    {
        CUDA_CHECK(cudaEventCreateWithFlags(&staged[k],
            cudaEventDisableTiming));
        CUDA_CHECK(cudaMallocHost(&stage[k], 16 * S.max_pix));
    }
    CUDA_CHECK(cudaMallocHost(&h_views, S.n * sizeof(CutView)));
    fixed.reserve(S.fixed_bytes());
    d_views = reinterpret_cast<CutView*>(fixed.p);
    d_cams = reinterpret_cast<CullCam*>(fixed.p
        + align_up(S.n * sizeof(CutView)));
    d_count = reinterpret_cast<unsigned long long*>(fixed.p
        + align_up(S.n * sizeof(CutView)) + align_up(S.n * sizeof(CullCam)));
    std::vector<CullCam> cams(S.n);
    for (int j = 0; j < S.n; ++j)
    {
        std::copy(S.KR9 + 9 * j, S.KR9 + 9 * j + 9, cams[j].KR);
        std::copy(S.t3 + 3 * j, S.t3 + 3 * j + 3, cams[j].t);
        cams[j].w = S.w[j];
        cams[j].h = S.h[j];
    }
    CUDA_CHECK(cudaMemcpyAsync(d_cams, cams.data(), S.n * sizeof(CullCam),
        cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemsetAsync(d_count, 0, 2 * sizeof(unsigned long long),
        st));
    stats.bytes += S.n * sizeof(CullCam);
    CUDA_CHECK(cudaEventRecord(ev0, st));

    /* target groups: views from the shared counter while they fit next to
     * one source slot (none when the group holds every view) */
    size_t const slot = S.slot_bytes();
    int carried = -1;
    while (!S.failed)
    {
        std::vector<int> group;
        size_t bytes = S.fixed_bytes();
        for (;;)
        {
            if (static_cast<int>(group.size()) >= S.group_cap)
                break;
            int const i = carried >= 0 ? carried : S.next.fetch_add(1);
            carried = -1;
            if (i >= S.n)
                break;
            size_t const more = bytes + S.target_bytes(i);
            bool const all = static_cast<int>(group.size()) + 1 == S.n;
            if (more + (all ? 0 : slot) > budget)
            {
                carried = i;      /* fits an empty group (checked up front) */
                break;
            }
            group.push_back(i);
            bytes = more;
        }
        if (group.empty())
            break;
        run_group(group);
    }
    CUDA_CHECK(cudaEventRecord(ev1, st));
    CUDA_CHECK(cudaEventSynchronize(ev1));
    float ms = 0.0f;
    CUDA_CHECK(cudaEventElapsedTime(&ms, ev0, ev1));
    stats.ms = ms;
    unsigned long long cnt[2];
    CUDA_CHECK(cudaMemcpy(cnt, d_count, sizeof(cnt), cudaMemcpyDeviceToHost));
    stats.valid = cnt[0];
    stats.pairs = cnt[1];
}

void
Worker::run_group (std::vector<int> const& group)
{
    int const nw = S.nwords;
    std::vector<char> resident(S.n, 0);
    size_t tbytes = 0;
    for (int i : group)
    {
        tbytes += S.target_bytes(i);
        resident[i] = 1;
    }
    slots.release();
    if (targets.cap > tbytes)
        targets.release();        /* the slots get what the targets leave */
    targets.reserve(tbytes);
    stats.groups += 1;

    /* targets: upload, z-depth, tile boxes, culling */
    std::vector<Target> tg(group.size());
    uint8_t* p = targets.p;
    auto take = [&p] (size_t n) { uint8_t* q = p; p += align_up(n); return q; };
    for (size_t g = 0; g < group.size(); ++g)
    {
        int const i = group[g];
        size_t const n = S.pix(i);
        size_t const t = static_cast<size_t>(S.tiles(i));
        Target& T = tg[g];
        T.i = i;
        T.cut = reinterpret_cast<float*>(take(n * 4));
        T.z = reinterpret_cast<float*>(take(n * 4));
        T.acc = reinterpret_cast<float*>(take(n * 4));
        T.nrm = reinterpret_cast<float*>(take(n * 12));
        T.done = take(n);
        T.boxes = reinterpret_cast<TileBox*>(take(t * sizeof(TileBox)));
        T.keep = reinterpret_cast<uint32_t*>(take(t * nw * 4));
        T.needed = reinterpret_cast<uint32_t*>(take(static_cast<size_t>(nw)
            * 4));
        upload(i, T.cut, T.nrm, T.z, nullptr);
        CUDA_CHECK(cudaMemsetAsync(T.acc, 0, n * 4, st));
        CUDA_CHECK(cudaMemsetAsync(T.done, 0, n, st));
        CUDA_CHECK(cudaMemsetAsync(T.needed, 0, nw * 4, st));
        CutView& v = h_views[i];
        S.fill_view(i, &v);
        v.cut = T.cut; v.zdepth = T.z; v.normals = T.nrm;
        dim3 const grid(S.tiles_x(i), (S.h[i] + kTile - 1) / kTile);
        tile_box_kernel<<<grid, dim3(kTile, kTile), 0, st>>>(v, T.boxes,
            d_count);
        CUDA_CHECK(cudaGetLastError());
        int const warps = static_cast<int>(t) * nw;
        cull_kernel<<<(warps + 7) / 8, 256, 0, st>>>(T.boxes,
            static_cast<int>(t), d_cams, S.n, i, nw, T.keep, T.needed,
            d_count + 1);
        CUDA_CHECK(cudaGetLastError());
        stats.launches += 2;
    }
    std::vector<uint32_t> h_needed(group.size() * nw);
    for (size_t g = 0; g < group.size(); ++g)
        CUDA_CHECK(cudaMemcpyAsync(h_needed.data() + g * nw, tg[g].needed,
            nw * 4, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    std::vector<uint32_t> need_any(nw, 0);
    for (size_t g = 0; g < group.size(); ++g)
    {
        tg[g].h_needed.assign(h_needed.begin() + g * nw,
            h_needed.begin() + (g + 1) * nw);
        for (int k = 0; k < nw; ++k)
            need_any[k] |= tg[g].h_needed[k];
    }
    auto needs = [] (std::vector<uint32_t> const& m, int j) {
        return (m[j >> 5] >> (j & 31)) & 1u;
    };

    /* source slots: as many as the budget leaves, at most the views the
     * group needs from outside; chunks take half of them so that uploads of
     * the next chunk run under the cut of this one */
    int n_stream = 0;
    for (int j = 0; j < S.n; ++j)
        n_stream += needs(need_any, j) && !resident[j];
    size_t const sb = S.slot_bytes();
    size_t const left = budget - std::min(budget, S.fixed_bytes() + tbytes);
    int const n_slots = static_cast<int>(std::min<size_t>(left / sb,
        static_cast<size_t>(n_stream)));
    if (n_stream > 0 && n_slots < 1)
        throw Error(SMVSB_ERR_INVALID, "smvsb_cut_depth_maps: no room for a "
            "source view next to the target group");
    if (n_slots > 0)
        slots.reserve(n_slots * sb);
    while (static_cast<int>(slot_free.size()) < n_slots)
    {
        cudaEvent_t e;
        CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        slot_free.push_back(e);
    }
    int const per_chunk = std::max(1, n_slots / 2);

    int j = 0, next_slot = 0;
    while (j < S.n)
    {
        /* the chunk [j0, j1): needed views in ascending j, at most per_chunk
         * of them streamed */
        while (j < S.n && !needs(need_any, j))
            ++j;
        if (j >= S.n)
            break;
        int const j0 = j;
        int streamed = 0;
        std::vector<int> used;
        for (; j < S.n; ++j)
        {
            if (!needs(need_any, j))
                continue;
            if (!resident[j])
            {
                if (streamed == per_chunk)
                    break;
                int const s = next_slot;
                next_slot = (next_slot + 1) % n_slots;
                uint8_t* base = slots.p + s * sb;
                float* cut = reinterpret_cast<float*>(base);
                float* z = reinterpret_cast<float*>(base
                    + align_up(S.max_pix * 4));
                float* nrm = reinterpret_cast<float*>(base
                    + 2 * align_up(S.max_pix * 4));
                upload(j, cut, nrm, z, slot_free[s]);
                CutView& v = h_views[j];
                S.fill_view(j, &v);
                v.cut = cut; v.zdepth = z; v.normals = nrm;
                used.push_back(s);
                ++streamed;
            }
        }
        int const j1 = j;
        stats.chunks += 1;
        CUDA_CHECK(cudaMemcpyAsync(d_views + j0, h_views + j0,
            (j1 - j0) * sizeof(CutView), cudaMemcpyHostToDevice, st));
        stats.bytes += (j1 - j0) * sizeof(CutView);
        for (Target const& T : tg)
        {
            bool any = false;
            for (int k = j0; k < j1 && !any; ++k)
                any = needs(T.h_needed, k);
            if (!any)
                continue;
            int const i = T.i;
            dim3 const grid(S.tiles_x(i), (S.h[i] + kTile - 1) / kTile);
            cut_chunk_kernel<<<grid, dim3(kTile, kTile), 0, st>>>(
                cut_target(T), d_views, i, j0, j1);
            CUDA_CHECK(cudaGetLastError());
            stats.launches += 1;
        }
        for (int s : used)
            CUDA_CHECK(cudaEventRecord(slot_free[s], st));
    }

    for (Target const& T : tg)
    {
        int const i = T.i;
        dim3 const grid(S.tiles_x(i), (S.h[i] + kTile - 1) / kTile);
        cut_finalize_kernel<<<grid, dim3(kTile, kTile), 0, st>>>(
            cut_target(T));
        CUDA_CHECK(cudaGetLastError());
        stats.launches += 1;
        CUDA_CHECK(cudaMemcpyAsync(S.out[i], T.acc, S.pix(i) * sizeof(float),
            cudaMemcpyDeviceToHost, st));
    }
    CUDA_CHECK(cudaStreamSynchronize(st));
}

} /* namespace */

void
cut_depth_maps_multi (smvsb_cut_options const* opts, int n_views,
    int const* w, int const* h, float const* const* depth,
    float const* const* normals, float const* invproj9,
    float const* cam_to_world16, float const* KR9, float const* t3,
    float* const* depth_out, smvsb_cut_stats* stats)
{
    if (n_views < 1 || !w || !h || !depth || !normals || !invproj9
        || !cam_to_world16 || !KR9 || !t3 || !depth_out || !opts)
        throw Error(SMVSB_ERR_INVALID, "smvsb_cut_depth_maps: arguments");
    if (opts->n_devices < 1 || !opts->devices)
        throw Error(SMVSB_ERR_INVALID,
            "smvsb_cut_depth_maps: empty device list");
    for (int i = 0; i < n_views; ++i)
        if (w[i] < 1 || h[i] < 1 || !depth[i] || !normals[i]
            || !depth_out[i])
            throw Error(SMVSB_ERR_INVALID,
                "smvsb_cut_depth_maps: view without maps");
    std::vector<int> const devs(opts->devices,
        opts->devices + opts->n_devices);
    for (int d : devs)
        check_device(d);
    std::lock_guard<std::mutex> guard(g_cut_lock);
    int caller_dev = 0;
    CUDA_CHECK(cudaGetDevice(&caller_dev));
    struct Restore
    {
        int d;
        ~Restore (void) { cudaSetDevice(d); }
    } restore{ caller_dev };

    Scene S;
    S.n = n_views; S.w = w; S.h = h; S.depth = depth; S.normals = normals;
    S.invproj9 = invproj9; S.ctw16 = cam_to_world16; S.KR9 = KR9;
    S.t3 = t3; S.out = depth_out;
    S.nwords = (n_views + 31) / 32;
    S.max_pix = 0;
    size_t max_target = 0;
    for (int i = 0; i < n_views; ++i)
    {
        S.max_pix = std::max(S.max_pix, S.pix(i));
        max_target = std::max(max_target, S.target_bytes(i));
    }
    int const n_workers = static_cast<int>(devs.size());
    S.group_cap = (n_views + n_workers - 1) / n_workers;
    size_t const least = S.fixed_bytes() + max_target
        + (n_views > 1 ? S.slot_bytes() : 0);

    /* budget per worker: the device's cap (or its free memory less a
     * margin) split among the workers on it */
    std::vector<size_t> budget(n_workers);
    for (int k = 0; k < n_workers; ++k)
    {
        int const d = devs[k];
        int const share = static_cast<int>(std::count(devs.begin(),
            devs.end(), d));
        size_t dev_bytes = opts->device_bytes;
        if (dev_bytes == 0)
        {
            CUDA_CHECK(cudaSetDevice(d));
            dev_bytes = usable_device_bytes();
        }
        budget[k] = dev_bytes / share;
        if (budget[k] < least)
            throw Error(opts->device_bytes ? SMVSB_ERR_INVALID
                : SMVSB_ERR_ALLOC, "smvsb_cut_depth_maps: "
                + std::to_string(budget[k]) + " bytes per worker on "
                "device " + std::to_string(d) + " do not hold the "
                "largest target view and one source view ("
                + std::to_string(least) + " bytes)");
    }

    /* A worker reports through Scene::fail: nothing may leave a thread. The
     * workers are joined at the end of the block, also when a later one
     * could not be started. */
    struct Threads : std::vector<std::thread>
    {
        ~Threads (void) { for (std::thread& t : *this) t.join(); }
    };
    std::vector<WorkerStats> ws(n_workers);
    {
        Threads threads;
        for (int k = 0; k < n_workers; ++k)
            threads.emplace_back([&S, &ws, &devs, &budget, k] {
                try
                {
                    Worker wk(S, devs[k], budget[k]);
                    try
                    {
                        wk.run();
                    }
                    catch (Error const& e)
                    {
                        S.fail(e);
                    }
                    ws[k] = wk.stats;
                    count_device_launches(devs[k],
                        static_cast<int>(wk.stats.launches));
                }
                catch (Error const& e)
                {
                    S.fail(e);
                }
                catch (std::exception const& e)
                {
                    S.fail(Error(SMVSB_ERR_INVALID, e.what()));
                }
            });
    }
    if (S.err_code != SMVSB_OK)
        throw Error(S.err_code, S.err_msg);
    if (stats)
    {
        smvsb_cut_stats out = {};
        for (WorkerStats const& s : ws)
        {
            out.reference_pairs += s.valid
                * static_cast<uint64_t>(n_views - 1);
            out.evaluated_pairs += s.pairs;
            out.bytes_uploaded += s.bytes;
            out.target_groups += s.groups;
            out.source_chunks += s.chunks;
            out.ms_device = std::max(out.ms_device, s.ms);
        }
        *stats = out;
    }
}

} /* namespace smvsb */

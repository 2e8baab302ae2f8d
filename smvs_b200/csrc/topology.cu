/*
 * topology.cu -- the Surface operations between the Newton loops, on the
 * device, so that a view's surface stays resident from the coarsest scale to
 * the output depth map (SURVEY.md section 8f, "next" row 3):
 *
 *   init_nodes_kernel      Surface::initialize_node_from_depth
 *                          (lib/surface.cc:665-760) for every node without a
 *                          value: per quadrant the smallest depth of the
 *                          window, the median of all of them as f
 *   fill_holes_kernel      Surface::fill_holes (:628-649)
 *   (remove_nodes)         Surface::remove_nodes_without_patch (:762-867),
 *                          visibility.cu
 *     -> Surface::Surface(.., init_depth) (:19-53) and
 *        Surface::fill_patches_from_depth (:141-153) are these three in a row
 *   subdivide_kernel       Surface::subdivide_patches (:983-1107): every node
 *                          of the finer grid from the ONE source the
 *                          reference's sequential loop leaves in it (an old
 *                          node, or the patch with the highest id that owns
 *                          the position)
 *   remove_isolated_kernel Surface::remove_isolated_patches (:887-927): the
 *                          reference sweeps x outer / y inner and a deletion
 *                          changes the counts of patches visited later; the
 *                          kernel runs the same recurrence as a wavefront
 *                          over t = 2x + y (a patch depends on (x-1, y-1),
 *                          (x-1, y), (x-1, y+1) and (x, y-1): all earlier
 *                          wavefronts)
 *   expand_round_kernel    Surface::expand (:482-628): two rounds of new rim
 *                          nodes. A round reads only the nodes as they were
 *                          before it (the reference collects the round's nodes
 *                          in a map and commits them after its loop), so a
 *                          round is one thread per node; the up to eight
 *                          offers of a node are taken in the reference's order
 *                          with check_swap_nodes' 0.9 hysteresis (:472-480)
 *
 * No arithmetic here can differ from the CPU: selections (min, median),
 * copies, divisions by 2 and 4, and BicubicPatch::evaluate_* in the
 * reference's expression order (patch_eval.cuh).
 */
#include <cmath>

#include "gn_math.cuh"
#include "patch_eval.cuh"

namespace smvsb {

namespace {

/* The tail of initialize_node_from_depth (lib/surface.cc:716-759) once the
 * window is reduced to its quadrant counts and minima and the median of its
 * n >= 2 depths: f = the median, the derivatives from the minima (a quadrant
 * without depth counts as 0). */
__device__ __forceinline__ void
write_node (int node, int const* cnt, float const* qmin, float med,
    uint8_t* __restrict__ node_valid, double* __restrict__ nodes)
{
    int num_non_zeros = 4;
    double avg[4];
    for (int q = 0; q < 4; ++q)
    {
        if (cnt[q] == 0)
        {
            avg[q] = 0.0;
            num_non_zeros -= 1;
        }
        else
            avg[q] = static_cast<double>(qmin[q]);
    }
    double const f = static_cast<double>(med);
    double dx = 0.0, dy = 0.0, dxy = 0.0;
    if (num_non_zeros == 4)
    {
        dx = __ddiv_rn(__dadd_rn(__dadd_rn(avg[1], avg[3]),
            -__dadd_rn(avg[0], avg[2])), 2.0);
        dy = __ddiv_rn(__dadd_rn(__dadd_rn(avg[2], avg[3]),
            -__dadd_rn(avg[0], avg[1])), 2.0);
        dxy = __dadd_rn(__dadd_rn(avg[3], -avg[2]),
            -__dadd_rn(avg[1], -avg[0]));
    }
    else
    {
        if ((avg[1] == 0 || avg[0] == 0) && avg[3] != 0 && avg[2] != 0)
            dx = __dadd_rn(avg[3], -avg[2]);
        else if ((avg[2] == 0 || avg[3] == 0) && avg[1] != 0
            && avg[0] != 0)
            dx = __dadd_rn(avg[1], -avg[0]);
        if ((avg[0] == 0 || avg[2] == 0) && avg[3] != 0 && avg[1] != 0)
            dy = __dadd_rn(avg[3], -avg[1]);
        else if ((avg[1] == 0 || avg[2] == 0) && avg[0] != 0
            && avg[2] != 0)
            dy = __dadd_rn(avg[2], -avg[0]);
    }
    nodes[static_cast<size_t>(node) * 4 + 0] = f;
    nodes[static_cast<size_t>(node) * 4 + 1] = dx;
    nodes[static_cast<size_t>(node) * 4 + 2] = dy;
    nodes[static_cast<size_t>(node) * 4 + 3] = dxy;
    node_valid[node] = 1;
}

/* One warp per node. Window values (floats) are gathered into shared memory,
 * per-quadrant minima by warp reduction, the median by ranking: the element
 * std::nth_element(all.begin(), all.begin() + n / 2, all.end()) leaves at
 * n / 2 is the one with exactly n / 2 elements ordered before it (ties broken
 * by position -- equal values are interchangeable). */
constexpr int INIT_WARPS = 2;

__global__ void __launch_bounds__(INIT_WARPS * 32)
init_nodes_kernel (int npx, int npy, int ps, int sx, int sy, int w, int h,
    float const* __restrict__ depth, uint8_t* __restrict__ node_valid,
    double* __restrict__ nodes)
{
    extern __shared__ float s_vals[];          /* INIT_WARPS x 4 win^2 */
    int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int const node = blockIdx.x * INIT_WARPS + warp;
    int const ns = npx + 1;
    if (node >= ns * (npy + 1))
        return;
    if (node_valid[node])
        return;
    int const idx = node % ns, idy = node / ns;
    int const x = idx * ps + sx, y = idy * ps + sy;
    int const win = ps / 2;
    int const cap = 4 * win * win;
    float* vals = s_vals + warp * cap;

    /* gather, quadrant by quadrant (order inside `all` does not matter) */
    int n = 0;
    int cnt[4];
    float qmin[4];
    for (int q = 0; q < 4; ++q)
    {
        int const i0 = (q & 1) ? 0 : -win, j0 = (q & 2) ? 0 : -win;
        int c = 0;
        float mn = INFINITY;
        for (int base = 0; base < win * win; base += 32)
        {
            int const e = base + lane;
            bool take = false;
            float v = 0.0f;
            if (e < win * win)
            {
                /* the reference walks i (x) outer, j (y) inner */
                int const i = i0 + e / win, j = j0 + e % win;
                int const gx = x + i, gy = y + j;
                if (gx >= 0 && gx < w && gy >= 0 && gy < h)
                {
                    v = depth[static_cast<size_t>(gy) * w + gx];
                    take = v > 0.0f;
                }
            }
            unsigned const ballot = __ballot_sync(0xffffffffu, take);
            if (take)
            {
                vals[n + c + __popc(ballot & ((1u << lane) - 1u))] = v;
                mn = fminf(mn, v);
            }
            c += __popc(ballot);
        }
        for (int off = 16; off > 0; off >>= 1)
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        cnt[q] = c;
        qmin[q] = mn;
        n += c;
    }
    __syncwarp();

    if (n < 2)          /* n >= 2: some quadrant has depth */
        return;

    /* median: element with rank n / 2 */
    int const k = n / 2;
    float med = 0.0f;
    bool found = false;
    for (int e = lane; e < n; e += 32)
    {
        float const v = vals[e];
        int rank = 0;
        for (int o = 0; o < n; ++o)
        {
            float const u = vals[o];
            rank += (u < v || (u == v && o < e)) ? 1 : 0;
        }
        if (rank == k)
        {
            med = v;
            found = true;
        }
    }
    unsigned const who = __ballot_sync(0xffffffffu, found);
    med = __shfl_sync(0xffffffffu, med, __ffs(who) - 1);

    if (lane == 0)
        write_node(node, cnt, qmin, med, node_valid, nodes);
}

/* The same for windows that do not fit in shared memory (patch size 128 and
 * 256, scales 7 and 8: 16 K and 64 K depths per node): one block per node
 * re-reads the window from the depth image. One pass counts each quadrant's
 * depths and takes its minimum; the median is then found by radix selection
 * over the fp32 bits, eight bits per pass. The depths are positive, so their
 * bits order like their values, and after four passes the selected bits are
 * the value with exactly n / 2 depths below it in the sorted order -- the
 * element std::nth_element leaves at n / 2. Counts, minima and histograms are
 * order-free, so the result does not depend on the thread schedule. */
constexpr int SELECT_THREADS = 256;

__global__ void __launch_bounds__(SELECT_THREADS)
init_nodes_select_kernel (int npx, int npy, int ps, int sx, int sy, int w,
    int h, float const* __restrict__ depth, uint8_t* __restrict__ node_valid,
    double* __restrict__ nodes)
{
    __shared__ unsigned s_hist[256];
    __shared__ int s_cnt[4];
    __shared__ unsigned s_min[4];
    __shared__ unsigned s_prefix;
    __shared__ int s_rank;
    int const tid = threadIdx.x;
    int const node = blockIdx.x;
    int const ns = npx + 1;
    if (node_valid[node])
        return;
    int const idx = node % ns, idy = node / ns;
    int const x = idx * ps + sx, y = idy * ps + sy;
    int const win = ps / 2, side = 2 * win;

    /* depth bits of window entry e (row-major over [-win, win)^2), 0 where
     * the window leaves the image or has no depth */
    auto bits_at = [&](int e) -> unsigned {
        int const gx = x + e % side - win, gy = y + e / side - win;
        if (gx < 0 || gx >= w || gy < 0 || gy >= h)
            return 0u;
        float const v = depth[static_cast<size_t>(gy) * w + gx];
        return (v > 0.0f) ? __float_as_uint(v) : 0u;
    };

    if (tid < 4)
    {
        s_cnt[tid] = 0;
        s_min[tid] = 0xffffffffu;
    }
    for (int i = tid; i < 256; i += SELECT_THREADS)
        s_hist[i] = 0;
    __syncthreads();
    int cnt[4] = {0, 0, 0, 0};
    unsigned mn[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
    for (int e = tid; e < side * side; e += SELECT_THREADS)
    {
        unsigned const b = bits_at(e);
        if (b == 0u)
            continue;
        /* quadrant: bit 0 = right half (i >= 0), bit 1 = lower half */
        int const q = (e % side >= win ? 1 : 0) + (e / side >= win ? 2 : 0);
        cnt[q] += 1;
        mn[q] = min(mn[q], b);
        atomicAdd(&s_hist[b >> 24], 1u);
    }
    for (int q = 0; q < 4; ++q)
    {
        if (cnt[q] == 0)
            continue;
        atomicAdd(&s_cnt[q], cnt[q]);
        atomicMin(&s_min[q], mn[q]);
    }
    __syncthreads();
    int const n = s_cnt[0] + s_cnt[1] + s_cnt[2] + s_cnt[3];
    if (n < 2)
        return;

    unsigned prefix = 0u;
    int rank = n / 2;               /* rank among the depths matching prefix */
    for (int shift = 24; ; shift -= 8)
    {
        if (tid == 0)
        {
            int below = 0, b = 0;
            while (below + static_cast<int>(s_hist[b]) <= rank)
                below += static_cast<int>(s_hist[b++]);
            s_prefix = prefix | (static_cast<unsigned>(b) << shift);
            s_rank = rank - below;
        }
        __syncthreads();
        prefix = s_prefix;
        rank = s_rank;
        if (shift == 0)
            break;
        for (int i = tid; i < 256; i += SELECT_THREADS)
            s_hist[i] = 0;
        __syncthreads();
        unsigned const high = 0xffffffffu << shift;
        for (int e = tid; e < side * side; e += SELECT_THREADS)
        {
            unsigned const b = bits_at(e);
            if (b != 0u && (b & high) == prefix)
                atomicAdd(&s_hist[(b >> (shift - 8)) & 255u], 1u);
        }
        __syncthreads();
    }

    if (tid == 0)
    {
        int c[4];
        float qmin[4];
        for (int q = 0; q < 4; ++q)
        {
            c[q] = s_cnt[q];
            qmin[q] = __uint_as_float(s_min[q]);
        }
        write_node(node, c, qmin, __uint_as_float(prefix), node_valid, nodes);
    }
}

/* a patch wherever its four nodes exist; counter (unless null) counts the
 * new patches, as Surface::expand returns them */
__global__ void
fill_holes_kernel (int npx, int npy, uint8_t const* __restrict__ node_valid,
    uint8_t* __restrict__ patch_valid, unsigned long long* __restrict__ counter)
{
    int const patch = blockIdx.x * blockDim.x + threadIdx.x;
    if (patch >= npx * npy || patch_valid[patch])
        return;
    int const idx = patch % npx, idy = patch / npx;
    int const n0 = idy * (npx + 1) + idx;
    if (node_valid[n0] && node_valid[n0 + 1] && node_valid[n0 + npx + 1]
        && node_valid[n0 + npx + 2])
    {
        patch_valid[patch] = 1;
        if (counter != nullptr)
            atomicAdd(counter, 1ull);
    }
}

/* One round of Surface::expand step 1 (lib/surface.cc:490-616). has_new /
 * new_f carry the nodes the earlier round made (the reference's new_nodes
 * map); nodes / node_valid are read only. */
__global__ void
expand_round_kernel (int npx, int npy, double const* __restrict__ nodes,
    uint8_t const* __restrict__ node_valid, uint8_t* __restrict__ has_new,
    double* __restrict__ new_f)
{
    int const node = blockIdx.x * blockDim.x + threadIdx.x;
    int const ns = npx + 1;
    if (node >= ns * (npy + 1))
        return;
    bool have = has_new[node] != 0;
    if (node_valid[node] && !have)
        return;
    double best = new_f[node];
    int const ix = node % ns, iy = node / ns;
    /* fill_node_neighbors: 0..7 = NW N NE W E SW S SE */
    bool ok[8];
    double f[8], dx[8], dy[8];
    int k = 0;
    for (int oy = -1; oy < 2; ++oy)
        for (int ox = -1; ox < 2; ++ox)
        {
            if (ox == 0 && oy == 0)
                continue;
            int const qx = ix + ox, qy = iy + oy;
            ok[k] = qx >= 0 && qy >= 0 && qx <= npx && qy <= npy
                && node_valid[qy * ns + qx];
            f[k] = dx[k] = dy[k] = 0.0;
            if (ok[k])
            {
                double const* n = nodes + static_cast<size_t>(qy * ns + qx) * 4;
                f[k] = n[0]; dx[k] = n[1]; dy[k] = n[2];
            }
            k += 1;
        }
    /* check_swap_nodes */
    auto offer = [&] (xd value)
    {
        if (!have || (value * xd(0.9)).v > best)
        {
            have = true;
            best = value.v;
        }
    };
    xd const two(2.0), three(3.0);
    auto px = [&] (int i) { return xd(f[i]) + xd(dx[i]) / two; };
    auto mx = [&] (int i) { return xd(f[i]) - xd(dx[i]) / two; };
    auto py = [&] (int i) { return xd(f[i]) + xd(dy[i]) / two; };
    auto my = [&] (int i) { return xd(f[i]) - xd(dy[i]) / two; };
    if (ok[0] && ok[1] && ok[3]) offer((px(3) + py(1)) / two);
    if (ok[1] && ok[2] && ok[4]) offer((mx(4) + py(1)) / two);
    if (ok[3] && ok[5] && ok[6]) offer((px(3) + my(6)) / two);
    if (ok[4] && ok[6] && ok[7]) offer((mx(4) + my(6)) / two);
    if (ok[0] && ok[1] && ok[2]) offer((py(0) + py(1) + py(2)) / three);
    if (ok[0] && ok[3] && ok[5]) offer((px(0) + px(3) + px(5)) / three);
    if (ok[5] && ok[6] && ok[7]) offer((my(5) + my(6) + my(7)) / three);
    if (ok[2] && ok[4] && ok[7]) offer((mx(2) + mx(4) + mx(7)) / three);
    has_new[node] = have ? 1 : 0;
    new_f[node] = best;
}

/* the round's nodes become the surface's (:617-619; dx = dy = dxy = 0) */
__global__ void
expand_commit_kernel (int n_nodes, uint8_t const* __restrict__ has_new,
    double const* __restrict__ new_f, double* __restrict__ nodes,
    uint8_t* __restrict__ node_valid)
{
    int const node = blockIdx.x * blockDim.x + threadIdx.x;
    if (node >= n_nodes || !has_new[node])
        return;
    node_valid[node] = 1;
    double* n = nodes + static_cast<size_t>(node) * 4;
    n[0] = new_f[node]; n[1] = 0.0; n[2] = 0.0; n[3] = 0.0;
}

/* BicubicPatch::evaluate_f / _dx / _dy / _dxy (lib/bicubic_patch.cc:121-187)
 * at (x, y) in [0, 1]^2, bitwise. */
__device__ __forceinline__ void
patch_eval4 (double const* cf, double x, double y, double* out)
{
    xd const sx(x), sy(y);
    xd ex[4], ey[4];
    ex[0] = xd(1.0); ex[1] = sx; ex[2] = sx * sx; ex[3] = ex[2] * sx;
    ey[0] = xd(1.0); ey[1] = sy; ey[2] = sy * sy; ey[3] = ey[2] * sy;
    xd f(0.0), fx(0.0), fy(0.0), fxy(0.0);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            f += xd(cf[i * 4 + j]) * ex[i] * ey[j];
#pragma unroll
    for (int i = 1; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            fx += xd(cf[i * 4 + j]) * xd(double(i)) * ex[i - 1] * ey[j];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 1; j < 4; ++j)
            fy += xd(cf[i * 4 + j]) * ex[i] * xd(double(j)) * ey[j - 1];
#pragma unroll
    for (int i = 1; i < 4; ++i)
#pragma unroll
        for (int j = 1; j < 4; ++j)
            fxy += xd(cf[i * 4 + j]) * xd(double(i)) * ex[i - 1]
                * xd(double(j)) * ey[j - 1];
    out[0] = f.v; out[1] = fx.v; out[2] = fy.v; out[3] = fxy.v;
}

struct SubdivArgs
{
    int npx, npy;               /* old grid */
    int new_npx, new_npy, off_x, off_y;
    double const* nodes;
    uint8_t const* node_valid;
    uint8_t const* patch_valid;
    double* new_nodes;
    uint8_t* new_valid;
};

/* One thread per node of the finer grid. In the coordinates (u, v) = new
 * index - offset, old node (i, j) sits at (2i, 2j); old patch (i, j) writes
 * its five new nodes at (2i+1, 2j), (2i, 2j+1), (2i+1, 2j+1), (2i+2, 2j+1),
 * (2i+1, 2j+2). The reference walks the patches in id order, so where two
 * patches write the same node the one with the higher id stays. */
__global__ void
subdivide_kernel (SubdivArgs const a)
{
    int const nn = blockIdx.x * blockDim.x + threadIdx.x;
    int const new_ns = a.new_npx + 1;
    if (nn >= new_ns * (a.new_npy + 1))
        return;
    int const u = nn % new_ns - a.off_x, v = nn / new_ns - a.off_y;
    double out[4] = {0.0, 0.0, 0.0, 0.0};
    bool valid = false;
    if (u >= 0 && v >= 0 && u <= 2 * a.npx && v <= 2 * a.npy)
    {
        if (!(u & 1) && !(v & 1))
        {
            int const node = (v / 2) * (a.npx + 1) + u / 2;
            if (a.node_valid[node])
            {
                valid = true;
                out[0] = a.nodes[static_cast<size_t>(node) * 4];
                out[1] = a.nodes[static_cast<size_t>(node) * 4 + 1] / 2;
                out[2] = a.nodes[static_cast<size_t>(node) * 4 + 2] / 2;
                out[3] = a.nodes[static_cast<size_t>(node) * 4 + 3] / 4;
            }
        }
        else
        {
            /* candidate patches, the one with the higher id first */
            int pi[2], pj[2];
            double ax[2], ay[2];
            int nc = 0;
            if ((u & 1) && (v & 1))
            {
                pi[0] = (u - 1) / 2; pj[0] = (v - 1) / 2;
                ax[0] = 0.5; ay[0] = 0.5; nc = 1;
            }
            else if (u & 1)           /* v even: top edge of (i, v/2) ...   */
            {
                pi[0] = (u - 1) / 2; pj[0] = v / 2; ax[0] = 0.5; ay[0] = 0.0;
                pi[1] = (u - 1) / 2; pj[1] = v / 2 - 1;      /* ... bottom */
                ax[1] = 0.5; ay[1] = 1.0; nc = 2;
            }
            else                      /* u even: left edge of (u/2, j) ...  */
            {
                pi[0] = u / 2; pj[0] = (v - 1) / 2; ax[0] = 0.0; ay[0] = 0.5;
                pi[1] = u / 2 - 1; pj[1] = (v - 1) / 2;      /* ... right  */
                ax[1] = 1.0; ay[1] = 0.5; nc = 2;
            }
            for (int c = 0; c < nc && !valid; ++c)
            {
                if (pi[c] < 0 || pj[c] < 0 || pi[c] >= a.npx
                    || pj[c] >= a.npy)
                    continue;
                if (!a.patch_valid[pj[c] * a.npx + pi[c]])
                    continue;
                double theta[16], cf[16], e[4];
                load_patch_theta(a.nodes, a.npx, pi[c], pj[c], theta);
                patch_coefficients(theta, cf);
                patch_eval4(cf, ax[c], ay[c], e);
                out[0] = e[0]; out[1] = e[1] / 2; out[2] = e[2] / 2;
                out[3] = e[3] / 4;
                valid = true;
            }
        }
    }
    a.new_valid[nn] = valid ? 1 : 0;
#pragma unroll
    for (int c = 0; c < 4; ++c)
        a.new_nodes[static_cast<size_t>(nn) * 4 + c] = out[c];
}

/* One block; wavefront t = 2x + y. */
__global__ void __launch_bounds__(1024)
remove_isolated_kernel (int npx, int npy, uint8_t* __restrict__ patch_valid)
{
    for (int t = 0; t <= 2 * (npx - 1) + (npy - 1); ++t)
    {
        /* cells (x, y = t - 2x) with 0 <= y < npy */
        int const x_lo = max(0, (t - (npy - 1) + 1) / 2);
        int const x_hi = min(npx - 1, t / 2);
        for (int x = x_lo + threadIdx.x; x <= x_hi; x += blockDim.x)
        {
            int const y = t - 2 * x;
            if (y < 0 || y >= npy || !patch_valid[y * npx + x])
                continue;
            int valid_neighbors = 0;
            for (int dx = -1; dx < 2; ++dx)
                for (int dy = -1; dy < 2; ++dy)
                {
                    if (dx == 0 && dy == 0)
                        continue;
                    int const qx = x + dx, qy = y + dy;
                    if (qx < 0 || qy < 0 || qx > npx - 1 || qy > npy - 1)
                        continue;
                    valid_neighbors += patch_valid[qy * npx + qx] ? 1 : 0;
                }
            if (valid_neighbors < 3)
                patch_valid[y * npx + x] = 0;
        }
        __syncthreads();
    }
}

__global__ void
count_valid_kernel (int n, uint8_t const* __restrict__ flags,
    unsigned long long* out)
{
    int const i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned const m = __ballot_sync(0xffffffffu, i < n && flags[i] != 0);
    if ((threadIdx.x & 31) == 0 && m)
        atomicAdd(out, static_cast<unsigned long long>(__popc(m)));
}

__global__ void
keep_positive_kernel (size_t n, float const* __restrict__ in,
    float* __restrict__ out)
{
    size_t const i = static_cast<size_t>(blockIdx.x) * blockDim.x
        + threadIdx.x;
    if (i < n)
        out[i] = (in[i] > 0.0f) ? in[i] : 0.0f;
}

} /* namespace */

/* Surface::fill_patches_from_depth on the context's grid and init depth. */
void
topo_fill_from_depth (smvsb_ctx* c)
{
    int const nn = c->n_nodes, np = c->n_patches;
    int const win = c->ps / 2;
    if (win > 32)
    {
        init_nodes_select_kernel<<<nn, SELECT_THREADS, 0, c->stream>>>(
            c->npx, c->npy, c->ps, c->start_x, c->start_y, c->w, c->h,
            c->init_depth.p, c->node_valid.p, c->nodes.p);
        CUDA_CHECK(cudaGetLastError());
        count_launches(c, 1);
    }
    else if (win >= 1)
    {
        size_t const smem = static_cast<size_t>(INIT_WARPS) * 4 * win * win
            * sizeof(float);
        if (smem > 48 * 1024)
            CUDA_CHECK(cudaFuncSetAttribute(init_nodes_kernel,
                cudaFuncAttributeMaxDynamicSharedMemorySize,
                static_cast<int>(smem)));
        init_nodes_kernel<<<(nn + INIT_WARPS - 1) / INIT_WARPS,
            INIT_WARPS * 32, smem, c->stream>>>(c->npx, c->npy, c->ps,
            c->start_x, c->start_y, c->w, c->h, c->init_depth.p,
            c->node_valid.p, c->nodes.p);
        CUDA_CHECK(cudaGetLastError());
        count_launches(c, 1);
    }
    fill_holes_kernel<<<(np + 255) / 256, 256, 0, c->stream>>>(c->npx, c->npy,
        c->node_valid.p, c->patch_valid.p, nullptr);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
    launch_remove_nodes(c);
}

/* The init depth a Surface keeps (lib/surface.cc:43-51: values > 0 copied
 * into a zeroed image); src is a device image of the main view's size. */
void
topo_set_init_depth (smvsb_ctx* c, float const* src_dev)
{
    size_t const npix = static_cast<size_t>(c->w) * c->h;
    c->init_depth.reserve(npix);
    keep_positive_kernel<<<static_cast<unsigned>((npix + 255) / 256), 256, 0,
        c->stream>>>(npix, src_dev, c->init_depth.p);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
}

/* Surface::subdivide_patches; the caller re-configures the grid afterwards
 * with the geometry returned here. */
void
topo_subdivide (smvsb_ctx* c, int* new_npx, int* new_npy, int* new_sx,
    int* new_sy)
{
    int const ps = c->ps / 2;
    int nnx = (c->w - 2) / ps, nny = (c->h - 2) / ps;
    int off_x = nnx - c->npx * 2, off_y = nny - c->npy * 2;
    int sx = c->start_x, sy = c->start_y;
    if (off_x >= 2)
    {
        nnx = c->npx * 2 + 2;
        sx = (c->w - nnx * ps) / 2;
        off_x = 1;
    }
    else
    {
        off_x = 0;
        nnx = c->npx * 2;
    }
    if (off_y >= 2)
    {
        nny = c->npy * 2 + 2;
        sy = (c->h - nny * ps) / 2;
        off_y = 1;
    }
    else
    {
        off_y = 0;
        nny = c->npy * 2;
    }
    size_t const new_nodes = static_cast<size_t>(nnx + 1) * (nny + 1);
    c->nodes_tmp.reserve(new_nodes * 4);
    c->node_valid_tmp.reserve(new_nodes);
    SubdivArgs a;
    a.npx = c->npx; a.npy = c->npy;
    a.new_npx = nnx; a.new_npy = nny; a.off_x = off_x; a.off_y = off_y;
    a.nodes = c->nodes.p; a.node_valid = c->node_valid.p;
    a.patch_valid = c->patch_valid.p;
    a.new_nodes = c->nodes_tmp.p; a.new_valid = c->node_valid_tmp.p;
    subdivide_kernel<<<static_cast<unsigned>((new_nodes + 127) / 128), 128, 0,
        c->stream>>>(a);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
    *new_npx = nnx; *new_npy = nny; *new_sx = sx; *new_sy = sy;
}

/* After topo_subdivide + grid reconfiguration: the new nodes become the
 * surface, no patches yet, then fill_holes + remove_nodes_without_patch
 * (lib/surface.cc:1090-1106). */
void
topo_subdivide_finish (smvsb_ctx* c)
{
    size_t const nn = c->n_nodes, np = c->n_patches;
    c->nodes.reserve(nn * 4);
    c->node_valid.reserve(nn);
    c->patch_valid.reserve(np);
    CUDA_CHECK(cudaMemcpyAsync(c->nodes.p, c->nodes_tmp.p,
        nn * 4 * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    CUDA_CHECK(cudaMemcpyAsync(c->node_valid.p, c->node_valid_tmp.p, nn,
        cudaMemcpyDeviceToDevice, c->stream));
    CUDA_CHECK(cudaMemsetAsync(c->patch_valid.p, 0, np, c->stream));
    fill_holes_kernel<<<static_cast<unsigned>((np + 255) / 256), 256, 0,
        c->stream>>>(c->npx, c->npy, c->node_valid.p, c->patch_valid.p,
        nullptr);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
    launch_remove_nodes(c);
}

/* Surface::remove_isolated_patches */
void
topo_remove_isolated (smvsb_ctx* c)
{
    remove_isolated_kernel<<<1, 1024, 0, c->stream>>>(c->npx, c->npy,
        c->patch_valid.p);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
    launch_remove_nodes(c);
}

/* Surface::expand; returns the patches fill_holes created (synchronises) */
uint64_t
topo_expand (smvsb_ctx* c)
{
    int const nn = c->n_nodes, np = c->n_patches;
    c->node_valid_tmp.reserve(nn);
    c->nodes_tmp.reserve(static_cast<size_t>(nn) * 4);
    c->counters.reserve(4);
    CUDA_CHECK(cudaMemsetAsync(c->node_valid_tmp.p, 0, nn, c->stream));
    CUDA_CHECK(cudaMemsetAsync(c->nodes_tmp.p, 0, nn * sizeof(double),
        c->stream));
    CUDA_CHECK(cudaMemsetAsync(c->counters.p, 0, sizeof(unsigned long long),
        c->stream));
    for (int round = 0; round < 2; ++round)
    {
        expand_round_kernel<<<(nn + 127) / 128, 128, 0, c->stream>>>(c->npx,
            c->npy, c->nodes.p, c->node_valid.p, c->node_valid_tmp.p,
            c->nodes_tmp.p);
        expand_commit_kernel<<<(nn + 255) / 256, 256, 0, c->stream>>>(nn,
            c->node_valid_tmp.p, c->nodes_tmp.p, c->nodes.p,
            c->node_valid.p);
    }
    fill_holes_kernel<<<(np + 255) / 256, 256, 0, c->stream>>>(c->npx,
        c->npy, c->node_valid.p, c->patch_valid.p, c->counters.p);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 5);
    launch_remove_nodes(c);
    unsigned long long n = 0;
    CUDA_CHECK(cudaMemcpyAsync(&n, c->counters.p, sizeof(n),
        cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return n;
}

/* number of valid patches (synchronises) */
uint64_t
topo_count_patches (smvsb_ctx* c)
{
    c->counters.reserve(4);
    CUDA_CHECK(cudaMemsetAsync(c->counters.p, 0, sizeof(unsigned long long),
        c->stream));
    count_valid_kernel<<<(c->n_patches + 255) / 256, 256, 0, c->stream>>>(
        c->n_patches, c->patch_valid.p, c->counters.p);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
    unsigned long long n = 0;
    CUDA_CHECK(cudaMemcpyAsync(&n, c->counters.p, sizeof(n),
        cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return n;
}

} /* namespace smvsb */

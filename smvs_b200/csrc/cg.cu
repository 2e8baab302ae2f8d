/*
 * cg.cu -- ConjugateGradient::solve (lib/conjugate_gradient.h:72-202) with
 * BlockSparseMatrix<4>::multiply (lib/block_sparse_matrix.h:276-298) and the
 * SSEVector updates (lib/sse_vector.cc) as ONE persistent kernel -- for one
 * view, or for several independent views (one system each) in the same
 * launch.
 *
 * The Hessian lives in a fixed 3x3-stencil block row format
 * H[node][9][4][4] (a node couples only to its 8 grid neighbours), the
 * preconditioner as P[node][4][4]. Four threads own one node (one per block
 * row); a warp therefore streams 8 complete 1152-byte block rows per pass,
 * every 128-byte line fully used.
 *
 * The whole solve -- SpMV, the dot products, the reference's two stopping
 * tests (residual < tolerance and the Nash/Sofer quadratic-model test),
 * preconditioning and direction update -- runs on the device; grid-wide
 * reductions go through per-block partial sums that every block re-sums in
 * the same fixed order, so the result is deterministic run to run and the
 * stopping decision is taken identically by all blocks without a host
 * round trip. Two grid barriers per iteration: the direction update
 * d = z + beta d is folded into the next SpMV (formed on the fly for the nine
 * neighbours), the block-diagonal preconditioner into the residual update
 * (quad shuffles).
 *
 * All three phases (initialisation, SpMV, vector update) walk the compacted
 * list of the system's block rows (the nodes that are valid and active,
 * lib/gauss_newton_step.cc:91-105), so a system that has shrunk to 10 % of
 * the grid costs 10 % of the vector traffic as well.
 *
 * H does not change during a solve, and a CTA's first pass (its 64 block
 * rows) is the same in every iteration: for a single view the kernel copies
 * those rows into shared memory once per solve (TMA bulk copies at kernel
 * start, waited for before the first SpMV) and reads them from there. With
 * 2 CTAs on each of the H100's 132 SMs that is 16 896 rows held on chip: the
 * full system (119 064 rows at 1920x1080 scale 2) streams 14 % less of H per
 * iteration, and the systems of the last Newton steps of a loop, which fit
 * in one pass, stream none after the copy. (Shared memory, unlike the L2
 * pinning below, takes no space from the vectors; it comes out of L1, 73 KB
 * per CTA.) Where each value of H is read from is all that changes: the
 * arithmetic, and so the result, is bitwise the same.
 *
 * Several views per launch (smvsb_newton_loop_batch; the reference runs one
 * view per pool thread, app/smvsrecon.cc:658-733): what an iteration costs
 * besides the Hessian stream is two grid-wide synchronisations, a fixed
 * cost whatever the system size. With V views in one launch every CTA
 * works through "its" rows of view 0, then of view 1, ... between two
 * barriers, so the fixed cost is paid once per V views. CTA b handles of
 * every view exactly the rows it would handle in a launch of its own, the
 * per-view partial sums are kept apart and re-summed in the same order, and
 * every view takes its stopping decisions for itself: the result of a view
 * is bitwise the one of a single-view launch. Views that have converged are
 * skipped.
 *
 * Alternatives that were tried and not kept: parking what only the owning
 * thread touches (x, r, A d, its row of P) in shared memory for the whole
 * solve (every KB of shared memory is a KB less L1, which the SpMV needs both
 * for the vector entries nine rows share and as landing space for the loads in
 * flight); reading the blocks left of / above the diagonal as transposes of
 * the neighbours' mirror blocks (the second use of a line rarely hits L2, and
 * the assembled H is symmetric only to rounding, so x changes); prefetching
 * the rows a CTA reads first into L2 during the vector-update phase; keeping
 * part of H in L2 from one iteration to the next (the SpMV phase is limited by
 * what the SMs keep in flight through L2, and the vectors lose their place);
 * fetching across the grid barriers (registers live across the barrier change
 * the streaming loop's schedule: fewer loads in flight); the compacted row
 * list in 8 x 8 tiles of the node grid instead of row-major strips (the warps
 * of a CTA then stream separate pieces of H instead of one contiguous piece).
 */
#include <algorithm>

#include "common.cuh"

namespace smvsb {

namespace {

constexpr int CG_THREADS = 256;
constexpr int CG_WARPS = CG_THREADS / 32;
constexpr int CG_QUADS = CG_THREADS / 4;     /* block rows per CTA and pass */
constexpr int CG_MAX_BLOCKS = 1024;
constexpr int CG_UF = 4;          /* rows per thread in flight, update phase */
constexpr int CG_SLOTS = 10;      /* partial-sum slots per view */
constexpr int CG_ROW_CACHE = 16;  /* row-list passes per CTA held in shared
                                     memory, shared out among the NV views */

/* One view's system and vectors. */
struct CgView
{
    int n_nodes, npx;
    int grid;                /* CTAs that work on this view: min(launch grid,
                                ceil(4 n_nodes / 256)) -- what a launch of its
                                own would use */
    int pad;
    double err_tol;          /* < 0: 0.01 * ||g|| (lib/depth_optimizer.cc:247) */
    double const* H;
    double const* P;
    double const* g;         /* b = -g (lib/depth_optimizer.cc:251) */
    uint16_t const* rowmask; /* bit k: block k of the node's row exists */
    uint32_t const* rows;    /* nodes with a non-empty row, ascending */
    unsigned long long const* counts;   /* [0] blocks, [1] rows of the system */
    double* x;               /* zeroed by the host before the launch */
    double* r;
    double* d;               /* search direction, double buffered */
    double* d2;
    double* Ad;
    double* z;
    double* partials;        /* [CG_SLOTS][CG_MAX_BLOCKS] */
    double* result;          /* [0] iterations, [1] info, [2] isnan(x[0]) */
};

struct CgArgs
{
    int n_views;
    int max_iter;
    double q_tol;
    unsigned int* sync;      /* barrier counter */
    CgView v[SMVSB_MAX_BATCH];
};

/* Per-view scalars of the iteration, identical in every CTA. */
struct CgState
{
    double r_dot_r, Q0, beta, alpha, tol;
    double* partials;        /* copy of CgView::partials, see publish() */
    int n_rows, passes, done, iters, info;
    int grid;                /* copy of CgView::grid */
};

__device__ __forceinline__ void
grid_barrier (unsigned int* counter, unsigned int& epoch)
{
    __syncthreads();
    if (threadIdx.x == 0)
    {
        epoch += 1;
        unsigned int const target = epoch * gridDim.x;
        /* arrive: one release reduction (the CTA's stores, ordered before it
         * by the bar.sync above, are visible to whoever observes the count);
         * cheaper than fence + atomicAdd (benchmarks/micro/barrier_probe.cu) */
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;"
            :: "l"(counter) : "memory");
        /* spin with relaxed loads (served by L2) and acquire once at the
         * end: an acquire load in the loop invalidates the SM's L1 on every
         * poll (CCTL.IVALL, ~40 polls per barrier) -- under the other CTA of
         * the SM, which may still be gathering vector entries through L1 */
        unsigned int v;
        do {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];"
                : "=r"(v) : "l"(counter) : "memory");
        } while (v < target);
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];"
            : "=r"(v) : "l"(counter) : "memory");
    }
    __syncthreads();
}

/* L2 evict-first access policy. Not volatile: the compiler may hoist it out
 * of the streaming loop. */
__device__ __forceinline__ unsigned long long
policy_evict_first (void)
{
    unsigned long long pol;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

/* Streaming load of the four Hessian entries of one block row: two 128-bit
 * requests per thread (sm_90 has neither the 256-bit load nor the eviction
 * qualifier on vector loads, so the priority travels as a cache-policy
 * operand), not allocated in L1 -- L1 is left to the vector entries the nine
 * rows around a node share -- and marked evict-first in L2 (H is 148 MB at
 * 1920x1080 scale 2, read once per iteration). */
__device__ __forceinline__ void
ld_stream (double const* p, double2& h01, double2& h23)
{
    unsigned long long const pol = policy_evict_first();
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f64 "
        "{%0, %1}, [%2], %3;"
        : "=d"(h01.x), "=d"(h01.y) : "l"(p), "l"(pol));
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f64 "
        "{%0, %1}, [%2], %3;"
        : "=d"(h23.x), "=d"(h23.y) : "l"(p + 2), "l"(pol));
}

/* 16-byte load of a vector entry pair other rows re-use from L1. */
__device__ __forceinline__ double2
ld_vec (double const* p)
{
    return *reinterpret_cast<double2 const*>(p);
}

/* 16-byte load with an L2 eviction-priority hint (P: keep resident). */
__device__ __forceinline__ double2
ld_hint (double const* p, unsigned long long policy)
{
    double2 v;
    asm volatile("ld.global.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;"
        : "=d"(v.x), "=d"(v.y) : "l"(p), "l"(policy));
    return v;
}

__device__ __forceinline__ unsigned long long
policy_evict_last (void)
{
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;"
        : "=l"(pol));
    return pol;
}

/*
 * Block-wide sums in two stages, each in a fixed order. Stage 1 (flush, once
 * per view and phase): shuffle tree inside every warp, lane 0 parks the
 * warp's value in shared memory. Stage 2 (publish, once per phase): after a
 * __syncthreads one thread per (view, value) adds the warps' results left to
 * right and writes the CTA's partial sum for that view.
 */
template <int NV>
__device__ __forceinline__ void
warp_flush (double (&v)[NV], double* s_red, int view)
{
#pragma unroll
    for (int j = 0; j < NV; ++j)
        for (int off = 16; off > 0; off >>= 1)
            v[j] += __shfl_down_sync(0xffffffffu, v[j], off);
    if ((threadIdx.x & 31) == 0)
    {
#pragma unroll
        for (int j = 0; j < NV; ++j)
            s_red[(view * 3 + j) * CG_WARPS + (threadIdx.x >> 5)] = v[j];
    }
}

/* (The view's grid size and partial-sum array are read from the shared copy:
 * indexing the kernel parameters with a per-thread view number is a divergent
 * constant-bank access -- the compiler hoists it above the branch, every
 * thread of the CTA fetches a different cache line, and the warp replays it
 * 32 times.) */
template <int NV>
__device__ __forceinline__ void
publish (CgArgs const& a, CgState const* s_state, double const* s_red,
    int first_slot, bool init)
{
    __syncthreads();
    int const t = threadIdx.x;
    if (t < a.n_views * NV)
    {
        int const view = t / NV, j = t % NV;
        CgState const& S = s_state[view];
        if (static_cast<int>(blockIdx.x) < S.grid && (init || !S.done))
        {
            /* a view without rows was never flushed */
            double total = 0.0;
            if (S.passes > 0)
                for (int i = 0; i < CG_WARPS; ++i)
                    total += s_red[(view * 3 + j) * CG_WARPS + i];
            S.partials[(first_slot + j) * CG_MAX_BLOCKS + blockIdx.x] = total;
        }
    }
}

/* Every CTA sums, per view, the partials of slots first .. first+NV-1 of all
 * the view's CTAs in the same order: one warp per (view, slot), lane l adds
 * partials l, l+32, ... in sequence (loads issued in batches ahead of the
 * adds), then the shuffle tree. Results in s_bcast[view * 3 + j]. Called
 * right after grid_barrier, whose closing bar.sync orders it. */
template <int NV>
__device__ __forceinline__ void
all_sums (CgArgs const& a, CgState const* s_state, int first_slot,
    double* s_bcast, bool init)
{
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int pair = warp; pair < a.n_views * NV; pair += CG_WARPS)
    {
        int const view = pair / NV, j = pair % NV;
        if (!init && s_state[view].done)
            continue;
        double const* p = s_state[view].partials
            + (first_slot + j) * CG_MAX_BLOCKS;
        int const nb = s_state[view].grid;
        double v = 0.0;
        /* 12 loads per lane in flight: one L2 round trip for up to 384 CTAs
         * (2 x 132 on H100) */
        for (int base = lane; base < nb; base += 32 * 12)
        {
            double t[12];
#pragma unroll
            for (int u = 0; u < 12; ++u)
                t[u] = (base + 32 * u < nb) ? __ldcg(p + base + 32 * u) : 0.0;
#pragma unroll
            for (int u = 0; u < 12; ++u)
                if (base + 32 * u < nb)
                    v += t[u];
        }
        for (int off = 16; off > 0; off >>= 1)
            v += __shfl_down_sync(0xffffffffu, v, off);
        if (lane == 0)
            s_bcast[view * 3 + j] = v;
    }
    __syncthreads();
}

/*
 * Plain (weak, L1-cached) loads are correct for the vectors other CTAs wrote
 * in the previous phase: the grid barrier is a release (red.release.gpu) /
 * acquire (relaxed polls + one ld.acquire.gpu) pair extended to the CTA by
 * bar.sync, so causality order covers them, and the gpu-scope acquire after
 * the spin drops the SM's L1 lines. Each vector entry is used by up to nine rows, most of
 * them in the same CTA pass: L1 serves the re-use instead of L2.
 *
 * VecOp: the vector the matrix is applied to. For CG it is the NEW search
 * direction z + beta * d_old, formed on the fly for the nine neighbours, so
 * the direction update (lib/conjugate_gradient.h:192-198) needs no pass and
 * no grid barrier of its own.
 */
struct PlainVec
{
    double const* v;
    __device__ __forceinline__ void load (int node, double* out) const
    {
        double2 const a = *reinterpret_cast<double2 const*>(
            v + static_cast<size_t>(node) * 4);
        double2 const b = *reinterpret_cast<double2 const*>(
            v + static_cast<size_t>(node) * 4 + 2);
        out[0] = a.x; out[1] = a.y; out[2] = b.x; out[3] = b.y;
    }
};

struct DirVec
{
    double const* z;
    double const* d_old;
    double beta;
    __device__ __forceinline__ void load (int node, double* out) const
    {
        double2 const z0 = ld_vec(z + static_cast<size_t>(node) * 4);
        double2 const z1 = ld_vec(z + static_cast<size_t>(node) * 4 + 2);
        double2 const d0 = ld_vec(d_old + static_cast<size_t>(node) * 4);
        double2 const d1 = ld_vec(d_old + static_cast<size_t>(node) * 4 + 2);
        out[0] = z0.x + d0.x * beta; out[1] = z0.y + d0.y * beta;
        out[2] = z1.x + d1.x * beta; out[3] = z1.y + d1.y * beta;
    }
};

/*
 * Where spmv_row reads a block row of H from. StreamRows: the matrix in HBM,
 * streamed. PinnedRows: the copy of the CTA's pass-0 rows in shared memory
 * (one row per quad, CG_PIN_STRIDE doubles apart), see cg_kernel.
 */
struct StreamRows
{
    double const* H;
    __device__ __forceinline__ double const* row (int node, int rp) const
    {
        return H + static_cast<size_t>(node) * 144 + rp * 4;
    }
    __device__ __forceinline__ void load (double const* p, double2& h01,
        double2& h23) const
    {
        ld_stream(p, h01, h23);
    }
};

/* Row stride 146 doubles (1168 B) rather than 144: with 1152 B the eight
 * quads of a warp hit the same 16 banks and every LDS.128 takes 8 wavefronts;
 * 1168 B moves odd quads onto the other 16 banks, the ideal 4. */
constexpr int CG_PIN_STRIDE = 146;
constexpr size_t CG_PIN_BYTES = sizeof(double) * CG_PIN_STRIDE * CG_QUADS;

struct PinnedRows
{
    double const* s;
    __device__ __forceinline__ double const* row (int, int rp) const
    {
        return s + (threadIdx.x >> 2) * CG_PIN_STRIDE + rp * 4;
    }
    __device__ __forceinline__ void load (double const* p, double2& h01,
        double2& h23) const
    {
        h01 = *reinterpret_cast<double2 const*>(p);
        h23 = *reinterpret_cast<double2 const*>(p + 2);
    }
};

/* (H v)[node, rp] for the thread's node and block row, blocks visited in
 * the reference's order (ascending column block,
 * lib/block_sparse_matrix.h:283-296). own[] receives v[node]. */
template <typename Rows, typename VecOp>
__device__ __forceinline__ double
spmv_row (Rows const& H, int ns, VecOp const& vec, int node, int rp,
    unsigned int mask, double* own)
{
    int const ix = node % ns, iy = node / ns;
    double const* hrow = H.row(node, rp);
    double acc = 0.0;
    own[0] = 0.0; own[1] = 0.0; own[2] = 0.0; own[3] = 0.0;
    /* The reference drops the rows and columns of inactive nodes
     * (lib/gauss_newton_step.cc:91,101,105); here they are zero blocks, which
     * are neither fetched nor multiplied: as the active set shrinks from one
     * Newton step to the next, so does the Hessian traffic. */
    /* The mask (both nodes valid, active and inside the grid) is in a
     * register before the row starts, so the nine loads stay independent. */
    if (mask == 0)
        return 0.0;
#pragma unroll
    for (int k = 0; k < 9; ++k)
    {
        if (!((mask >> k) & 1u))
            continue;
        int const jx = ix + (k % 3) - 1, jy = iy + (k / 3) - 1;
        int const nj = jy * ns + jx;
        double2 h01, h23;
        H.load(hrow + k * 16, h01, h23);
        double v[4];
        vec.load(nj, v);
        if (k == 4)
        {
            own[0] = v[0]; own[1] = v[1]; own[2] = v[2]; own[3] = v[3];
        }
        acc += h01.x * v[0];
        acc += h01.y * v[1];
        acc += h23.x * v[2];
        acc += h23.y * v[3];
    }
    return acc;
}

/* Does CTA b work on view v between the next two barriers? */
__device__ __forceinline__ bool
view_on (CgArgs const& a, CgState const* s_state, int v, bool init)
{
    return static_cast<int>(blockIdx.x) < s_state[v].grid
        && (init || !s_state[v].done) && s_state[v].passes > 0;
}

/* The row this thread's quad handles in pass p of view V: whether there is
 * one is decided from the position alone, so that nothing branches on the
 * loaded index and the load can travel while other work is issued. */
__device__ __forceinline__ bool
pass_row (CgView const& V, int n_rows, int pass, int& node)
{
    int const q = pass * (V.grid * CG_QUADS) + blockIdx.x * CG_QUADS
        + (threadIdx.x >> 2);
    bool const ok = q < n_rows;
    node = ok ? static_cast<int>(V.rows[q]) : 0;
    return ok;
}

/* The row list does not change during a solve: the nodes and masks of the
 * first PASSES passes of every view (per quad of the CTA; node 0 and mask 0
 * past the end of the list) are loaded into shared memory once, so that a
 * phase does not begin with the dependent rows[] -> rowmask[] fetches through
 * L2 (the grid barrier's acquire has just emptied L1). */
template <int NV>
struct RowCache
{
    static constexpr int PASSES = CG_ROW_CACHE / NV;
    uint32_t node[NV][PASSES][CG_QUADS];
    uint16_t mask[NV][PASSES][CG_QUADS];
};

template <int NV>
__device__ __forceinline__ void
fill_rows (RowCache<NV>& c, CgArgs const& a, CgState const* s_state)
{
    constexpr int N = RowCache<NV>::PASSES * CG_QUADS;
#pragma unroll
    for (int v = 0; v < NV; ++v)
    {
#pragma unroll
        for (int k = 0; k < (N + CG_THREADS - 1) / CG_THREADS; ++k)
        {
            int const e = k * CG_THREADS + threadIdx.x;
            if (e >= N)
                break;
            int const p = e / CG_QUADS, qd = e % CG_QUADS;
            int node = 0;
            unsigned int mask = 0u;
            if (v < a.n_views && static_cast<int>(blockIdx.x) < s_state[v].grid)
            {
                int const q = p * (s_state[v].grid * CG_QUADS)
                    + blockIdx.x * CG_QUADS + qd;
                if (q < s_state[v].n_rows)
                {
                    node = static_cast<int>(a.v[v].rows[q]);
                    mask = a.v[v].rowmask[node];
                }
            }
            c.node[v][p][qd] = static_cast<uint32_t>(node);
            c.mask[v][p][qd] = static_cast<uint16_t>(mask);
        }
    }
}

/* pass_row, and the row's mask: from the cache for the first passes. */
template <int NV>
__device__ __forceinline__ bool
cached_row (RowCache<NV> const& c, CgView const& V, int v, int n_rows,
    int pass, int& node, unsigned int& mask)
{
    if (pass < RowCache<NV>::PASSES)
    {
        int const qd = threadIdx.x >> 2;
        node = static_cast<int>(c.node[v][pass][qd]);
        mask = c.mask[v][pass][qd];
        return pass * (V.grid * CG_QUADS) + static_cast<int>(blockIdx.x)
            * CG_QUADS + qd < n_rows;
    }
    bool const ok = pass_row(V, n_rows, pass, node);
    mask = ok ? V.rowmask[node] : 0u;
    return ok;
}

/* 2 CTAs / SM: measured faster than 3 at 80 registers (fewer loads hoisted,
 * more barrier participants).
 *
 * NV = compile-time bound on the number of views (1, 2, 4, 8): the loops over
 * the views are unrolled, so a view's pointers are kernel parameters at fixed
 * offsets (constant-bank operands of the instructions that use them), not
 * values fetched per pass. The kernel is bound by the number of loads a warp
 * has in flight, and every dependent fetch in front of a pass's Hessian loads
 * lengthens the time a warp spends per pass. */
template <int NV>
__global__ void __launch_bounds__(CG_THREADS, 2)
cg_kernel (CgArgs const a)
{
    unsigned long long const keep = policy_evict_last();
    __shared__ double s_red[NV * 3 * CG_WARPS];
    __shared__ double s_bcast[NV * 3];
    __shared__ CgState s_state[NV];
    /* z's address per view, read back from shared memory where it is needed:
     * a value the compiler cannot re-derive from the kernel parameters, so it
     * stays in a register through the SpMV loop. (As a plain parameter it is
     * re-fetched from the constant bank in front of every neighbour's load
     * once registers are tight -- ncu: short-scoreboard stalls 4.0 instead of
     * 0.7 per issue, SpMV phase +20 %.) */
    __shared__ double const* s_zptr[NV];
    /* NV = 1: the H rows of the CTA's pass 0 (CG_PIN_BYTES, dynamic) and the
     * mbarrier their copies complete on */
    extern __shared__ __align__(16) double s_pin[];
    __shared__ __align__(8) unsigned long long s_pin_bar;
    __shared__ RowCache<NV> s_rows;
    unsigned int epoch = 0;
    int const quad = threadIdx.x & 28;      /* first lane of the node's quad */
    int const rp = threadIdx.x & 3;
    unsigned const pin_bar = static_cast<unsigned>(
        __cvta_generic_to_shared(&s_pin_bar));

    if (threadIdx.x < a.n_views)
    {
        CgView const& V = a.v[threadIdx.x];
        CgState& S = s_state[threadIdx.x];
        S.n_rows = static_cast<int>(V.counts[1]);
        int const per_pass = V.grid * CG_QUADS;
        int const passes = (S.n_rows + per_pass - 1) / per_pass;
        S.passes = ((passes + CG_UF - 1) / CG_UF) * CG_UF;
        S.done = 0; S.iters = 0; S.info = SMVSB_CG_MAX_ITERATIONS;
        S.r_dot_r = 0.0; S.Q0 = 0.0; S.beta = 0.0; S.alpha = 0.0; S.tol = 0.0;
        S.partials = V.partials;
        S.grid = V.grid;
        s_zptr[threadIdx.x] = V.z;
        if (NV == 1)
        {
            int const n_pin = static_cast<int>(blockIdx.x) < V.grid
                ? min(max(S.n_rows - static_cast<int>(blockIdx.x) * CG_QUADS,
                  0), CG_QUADS) : 0;
            if (n_pin > 0)
            {
                asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;"
                    :: "r"(pin_bar), "r"(n_pin));
                asm volatile("fence.mbarrier_init.release.cluster;"
                    ::: "memory");
            }
        }
    }
    __syncthreads();

    /* H does not change during the solve: the block rows of the CTA's pass 0
     * are copied into shared memory once, by the TMA engine (one 1152-byte
     * bulk copy per row, issued by the row's first thread), and the SpMV
     * reads them from there in every iteration. The copies travel while the
     * initialisation phase runs; the mbarrier counts one arrival per row
     * plus its bytes. */
    bool const pin = NV == 1 && static_cast<int>(blockIdx.x) < s_state[0].grid
        && static_cast<int>(blockIdx.x) * CG_QUADS < s_state[0].n_rows;
    if (NV == 1 && rp == 0)
    {
        int node;
        if (static_cast<int>(blockIdx.x) < s_state[0].grid
            && pass_row(a.v[0], s_state[0].n_rows, 0, node))
        {
            unsigned const dst = static_cast<unsigned>(__cvta_generic_to_shared(
                s_pin + (threadIdx.x >> 2) * CG_PIN_STRIDE));
            double const* src = a.v[0].H + static_cast<size_t>(node) * 144;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], "
                "%1;" :: "r"(pin_bar), "r"(1152) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global"
                ".mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                :: "r"(dst), "l"(src), "r"(1152), "r"(pin_bar) : "memory");
        }
    }
    /* read from the first SpMV on, behind the initialisation's barriers */
    fill_rows(s_rows, a, s_state);

    /* r = b = -g; x = 0 (host memset); z = P r; r_dot_r = z.r; ||g||^2
     * (lib/conjugate_gradient.h:85-117). d_old = 0 with beta = 0 makes the
     * first direction d = z. P is block diagonal: the four threads of a node
     * exchange their r entries by shuffle. */
#pragma unroll
    for (int v = 0; v < NV; ++v)
    {
        if (v >= a.n_views || !view_on(a, s_state, v, true))
            continue;
        CgView const& V = a.v[v];
        int const n_rows = s_state[v].n_rows, passes = s_state[v].passes;
        double acc[2] = { 0.0, 0.0 };       /* z.r, g.g */
        for (int p = 0; p < passes; ++p)
        {
            int node;
            bool const ok = pass_row(V, n_rows, p, node);
            size_t const i = static_cast<size_t>(node) * 4 + rp;
            double const gi = ok ? V.g[i] : 0.0;
            double const ri = -gi;
            double const r0 = __shfl_sync(0xffffffffu, ri, quad);
            double const r1 = __shfl_sync(0xffffffffu, ri, quad + 1);
            double const r2 = __shfl_sync(0xffffffffu, ri, quad + 2);
            double const r3 = __shfl_sync(0xffffffffu, ri, quad + 3);
            if (ok)
            {
                double const* prow = V.P + static_cast<size_t>(node) * 16
                    + rp * 4;
                double2 const p01 = *reinterpret_cast<double2 const*>(prow);
                double2 const p23 = *reinterpret_cast<double2 const*>(prow + 2);
                double const zi = p01.x * r0 + p01.y * r1 + p23.x * r2
                    + p23.y * r3;
                V.r[i] = ri;
                V.z[i] = zi;
                V.d[i] = 0.0;
                V.d2[i] = 0.0;
                V.Ad[i] = 0.0;
                acc[1] += gi * gi;
                acc[0] += zi * ri;
            }
        }
        warp_flush<2>(acc, s_red, v);
    }
    publish<2>(a, s_state, s_red, 0, true);
    grid_barrier(a.sync, epoch);
    all_sums<2>(a, s_state, 0, s_bcast, true);
    if (threadIdx.x < a.n_views)
    {
        CgState& S = s_state[threadIdx.x];
        S.r_dot_r = s_bcast[threadIdx.x * 3 + 0];
        double const gg = s_bcast[threadIdx.x * 3 + 1];
        double const et = a.v[threadIdx.x].err_tol;
        S.tol = (et < 0.0) ? sqrt(gg) * 0.01 : et;
    }
    __syncthreads();

    int iter = 1;
    if (pin)
    {
        unsigned done = 0;
        while (!done)
            asm volatile("{\n.reg .pred p;\n"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n"
                "selp.u32 %0, 1, 0, p;\n}"
                : "=r"(done) : "r"(pin_bar) : "memory");
    }
    for (; iter < a.max_iter; ++iter)
    {
        /* the direction is double buffered; all views swap in lock-step */
        bool const odd = (iter & 1) != 0;
        int const slot = 2 + 4 * (iter & 1);

        /* d = z + beta d_old (:192-198 of the previous iteration);
         * Ad = A d; alpha = r_dot_r / d.Ad (:126-127). */
        {
            /* One pass = the CTA's 64 block rows; the next pass's row index
             * and mask are fetched while this pass streams (from s_rows, or
             * past its passes from the row list). (A deeper pipeline -- index
             * two passes ahead, mask one -- was slower.) */
#pragma unroll
            for (int v = 0; v < NV; ++v)
            {
                if (v >= a.n_views || !view_on(a, s_state, v, false))
                    continue;
                CgView const& V = a.v[v];
                int const n_rows = s_state[v].n_rows;
                int const quads = V.grid * CG_QUADS;
                int const quad0 = blockIdx.x * CG_QUADS + (threadIdx.x >> 2);
                DirVec dir;
                dir.z = s_zptr[v];
                dir.d_old = odd ? V.d : V.d2;
                dir.beta = s_state[v].beta;
                double* d_new = odd ? V.d2 : V.d;
                double acc[1] = { 0.0 };
                int node;
                unsigned int mask;
                cached_row(s_rows, V, v, n_rows, 0, node, mask);
                auto row_pass = [&](auto const& rows, int p)
                {
                    int node_next;
                    unsigned int mask_next;
                    cached_row(s_rows, V, v, n_rows, p + 1, node_next,
                        mask_next);
                    double own[4];
                    size_t const i = static_cast<size_t>(node) * 4 + rp;
                    double const val = spmv_row(rows, V.npx + 1, dir, node, rp,
                        mask, own);
                    node = node_next;
                    mask = mask_next;
                    double const di = (rp == 0) ? own[0] : (rp == 1) ? own[1]
                        : (rp == 2) ? own[2] : own[3];
                    V.Ad[i] = val;
                    d_new[i] = di;
                    acc[0] += val * di;
                };
                int q = quad0, p = 0;
                if (NV == 1 && q < n_rows)
                {
                    row_pass(PinnedRows{ s_pin }, p);
                    q += quads;
                    ++p;
                }
                for (; q < n_rows; q += quads, ++p)
                    row_pass(StreamRows{ V.H }, p);
                warp_flush<1>(acc, s_red, v);
            }
            publish<1>(a, s_state, s_red, slot, false);
        }
        grid_barrier(a.sync, epoch);
        all_sums<1>(a, s_state, slot, s_bcast, false);
        if (threadIdx.x < a.n_views && !s_state[threadIdx.x].done)
            s_state[threadIdx.x].alpha = s_state[threadIdx.x].r_dot_r
                / s_bcast[threadIdx.x * 3];
        __syncthreads();

        /* x += alpha d; r -= alpha Ad; r.r; Q1 = -x.(b + r); z = P r; z.r
         * (:130-181) */
#pragma unroll
        for (int v = 0; v < NV; ++v)
        {
            if (v >= a.n_views || !view_on(a, s_state, v, false))
                continue;
            CgView const& V = a.v[v];
            int const n_rows = s_state[v].n_rows;
            int const passes = s_state[v].passes;
            double const alpha = s_state[v].alpha;
            double const* d_new = odd ? V.d2 : V.d;
            double acc[3] = { 0.0, 0.0, 0.0 };    /* r.r, x.(r - g), z.r */
            int nodes[CG_UF];
            bool oks[CG_UF];
            unsigned int unused;
#pragma unroll
            for (int u = 0; u < CG_UF; ++u)
                oks[u] = cached_row(s_rows, V, v, n_rows, u, nodes[u], unused);
            /* CG_UF rows per thread in flight: the pass is latency bound */
            for (int p = 0; p < passes; p += CG_UF)
            {
                int nodes_next[CG_UF];
                bool oks_next[CG_UF];
#pragma unroll
                for (int u = 0; u < CG_UF; ++u)
                    oks_next[u] = cached_row(s_rows, V, v, n_rows,
                        p + CG_UF + u, nodes_next[u], unused);

                double xv[CG_UF], rv[CG_UF], gv[CG_UF];
                double2 p01[CG_UF], p23[CG_UF];
#pragma unroll
                for (int u = 0; u < CG_UF; ++u)
                {
                    xv[u] = 0.0; rv[u] = 0.0; gv[u] = 0.0;
                    p01[u] = make_double2(0, 0); p23[u] = p01[u];
                    if (oks[u])
                    {
                        size_t const i = static_cast<size_t>(nodes[u]) * 4 + rp;
                        double const dn = d_new[i], ad = V.Ad[i];
                        gv[u] = V.g[i];
                        xv[u] = V.x[i]; rv[u] = V.r[i];
                        double const* prow = V.P
                            + static_cast<size_t>(nodes[u]) * 16 + rp * 4;
                        p01[u] = ld_hint(prow, keep);
                        p23[u] = ld_hint(prow + 2, keep);
                        xv[u] += dn * alpha; rv[u] -= ad * alpha;
                    }
                }
#pragma unroll
                for (int u = 0; u < CG_UF; ++u)
                {
                    double const q0 = __shfl_sync(0xffffffffu, rv[u], quad);
                    double const q1 = __shfl_sync(0xffffffffu, rv[u], quad + 1);
                    double const q2 = __shfl_sync(0xffffffffu, rv[u], quad + 2);
                    double const q3 = __shfl_sync(0xffffffffu, rv[u], quad + 3);
                    if (oks[u])
                    {
                        size_t const i = static_cast<size_t>(nodes[u]) * 4 + rp;
                        double const zi = p01[u].x * q0 + p01[u].y * q1
                            + p23[u].x * q2 + p23[u].y * q3;
                        V.x[i] = xv[u]; V.r[i] = rv[u];
                        V.z[i] = zi;
                        acc[0] += rv[u] * rv[u];
                        acc[1] += xv[u] * (rv[u] - gv[u]);
                        acc[2] += zi * rv[u];
                    }
                }
#pragma unroll
                for (int u = 0; u < CG_UF; ++u)
                {
                    nodes[u] = nodes_next[u];
                    oks[u] = oks_next[u];
                }
            }
            warp_flush<3>(acc, s_red, v);
        }
        publish<3>(a, s_state, s_red, slot + 1, false);
        grid_barrier(a.sync, epoch);
        all_sums<3>(a, s_state, slot + 1, s_bcast, false);

        /* the reference's two stopping tests, per view (:139, :170-176) */
        if (threadIdx.x < a.n_views && !s_state[threadIdx.x].done)
        {
            CgState& S = s_state[threadIdx.x];
            double const new_rr = s_bcast[threadIdx.x * 3 + 0];
            double const xbr = s_bcast[threadIdx.x * 3 + 1];
            double const new_zr = s_bcast[threadIdx.x * 3 + 2];
            bool stop = false;
            if (new_rr < S.tol)
                stop = true;
            else
            {
                double const Q1 = -1.0 * xbr;
                double const zeta = iter * (Q1 - S.Q0) / Q1;
                if (zeta < a.q_tol)
                    stop = true;
                else
                {
                    S.Q0 = Q1;
                    S.beta = new_zr / S.r_dot_r;
                    S.r_dot_r = new_zr;
                }
            }
            if (stop)
            {
                S.done = 1;
                S.iters = iter;
                S.info = SMVSB_CG_CONVERGENCE;
            }
        }
        __syncthreads();
        bool all_done = true;
        for (int v = 0; v < a.n_views; ++v)
            all_done = all_done && (s_state[v].done != 0);
        if (all_done)
            break;
    }

    if (blockIdx.x == 0 && threadIdx.x < a.n_views)
    {
        CgState const& S = s_state[threadIdx.x];
        double* res = a.v[threadIdx.x].result;
        res[0] = S.done ? S.iters : iter;
        res[1] = S.info;
        /* lib/depth_optimizer.cc:267 looks at the first entry of the solution;
         * the final barrier has made every CTA's x visible */
        res[2] = isnan(__ldcg(a.v[threadIdx.x].x)) ? 1.0 : 0.0;
    }
}

/* bit k of rowmask[node]: block k of the node's 3x3 stencil row exists, i.e.
 * the node and its k-th grid neighbour are both valid and active. */
__global__ void __launch_bounds__(256)
cg_mark_kernel (int npx, int npy, uint8_t const* __restrict__ node_valid,
    uint8_t const* __restrict__ active, uint16_t* __restrict__ rowmask,
    uint32_t* __restrict__ block_rows, unsigned long long* __restrict__ counts)
{
    int const node = blockIdx.x * blockDim.x + threadIdx.x;
    int const ns = npx + 1;
    unsigned int m = 0;
    if (node < ns * (npy + 1) && node_valid[node] && active[node])
    {
        int const ix = node % ns, iy = node / ns;
        for (int k = 0; k < 9; ++k)
        {
            int const jx = ix + (k % 3) - 1, jy = iy + (k / 3) - 1;
            if (jx < 0 || jx > npx || jy < 0 || jy > npy)
                continue;
            int const nj = jy * ns + jx;
            if (node_valid[nj] && active[nj])
                m |= 1u << k;
        }
    }
    if (node < ns * (npy + 1))
        rowmask[node] = static_cast<uint16_t>(m);
    /* counts[0]: blocks of the system, counts[1]: its block rows */
    unsigned int const blocks = __reduce_add_sync(0xffffffffu, __popc(m));
    int const rows = __syncthreads_count(m != 0);
    if ((threadIdx.x & 31) == 0)
        atomicAdd(counts, static_cast<unsigned long long>(blocks));
    if (threadIdx.x == 0)
    {
        block_rows[blockIdx.x] = rows;
        atomicAdd(counts + 1, static_cast<unsigned long long>(rows));
    }
}

/* rows[]: the nodes with a non-empty row in ascending order -- the solver
 * walks this list, so the work is spread evenly over the CTAs however the
 * active set is scattered over the image */
__global__ void __launch_bounds__(256)
cg_list_kernel (int n_nodes, uint16_t const* __restrict__ rowmask,
    uint32_t const* __restrict__ block_off, uint32_t* __restrict__ rows)
{
    __shared__ uint32_t s_warp[8];
    int const node = blockIdx.x * blockDim.x + threadIdx.x;
    bool const on = node < n_nodes && rowmask[node] != 0;
    unsigned int const ballot = __ballot_sync(0xffffffffu, on);
    int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0)
        s_warp[warp] = __popc(ballot);
    __syncthreads();
    uint32_t before = block_off[blockIdx.x];
    for (int w = 0; w < warp; ++w)
        before += s_warp[w];
    before += __popc(ballot & ((1u << lane) - 1u));
    if (on)
        rows[before] = node;
}

__global__ void
spmv_kernel (int n_nodes, int npx, double const* __restrict__ H,
    uint16_t const* __restrict__ rowmask, double const* __restrict__ x,
    double* __restrict__ y)
{
    int const i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes * 4)
        return;
    PlainVec vec;
    vec.v = x;
    StreamRows const rows{ H };
    double own[4];
    y[i] = spmv_row(rows, npx + 1, vec, i >> 2, i & 3, rowmask[i >> 2], own);
}

/* The system's row masks, counts and compacted row list (three small kernels
 * per solve). */
void
mark_system (smvsb_ctx* c)
{
    int const nb = (c->n_nodes + 255) / 256;
    c->cg_rowmask.reserve(c->n_nodes);
    c->cg_row_list.reserve(c->n_nodes);
    /* the per-block row counts, then their prefix sum and its total */
    c->cg_block_rows.reserve(2 * static_cast<size_t>(nb) + 1);
    c->cg_counts.reserve(2);
    CUDA_CHECK(cudaMemsetAsync(c->cg_counts.p, 0,
        2 * sizeof(unsigned long long), c->stream));
    cg_mark_kernel<<<nb, 256, 0, c->stream>>>(c->npx, c->npy,
        c->node_valid.p, c->active.p, c->cg_rowmask.p, c->cg_block_rows.p,
        c->cg_counts.p);
    CUDA_CHECK(cudaGetLastError());
    launch_exclusive_scan(c, c->cg_block_rows.p, c->cg_block_rows.p + nb, nb);
    cg_list_kernel<<<nb, 256, 0, c->stream>>>(c->n_nodes, c->cg_rowmask.p,
        c->cg_block_rows.p + nb, c->cg_row_list.p);
    smvsb::count_launches(c, 2);
    CUDA_CHECK(cudaGetLastError());
}

} /* namespace */

void
launch_spmv (smvsb_ctx* c, double const* x, double* y)
{
    mark_system(c);
    int const n = c->n_nodes * 4;
    spmv_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(c->n_nodes, c->npx,
        c->H.p, c->cg_rowmask.p, x, y);
    smvsb::count_launches(c, 1);
    CUDA_CHECK(cudaGetLastError());
}

/*
 * Enqueues one PCG launch for the systems of `n` contexts (same device; all
 * work goes to the stream of cs[0], which the caller has made the stream of
 * every context of the batch) and the copies of the results into the
 * contexts' pinned scalars. cg_collect() reads them after the caller has
 * synchronised the stream.
 */
void
cg_enqueue (smvsb_ctx* const* cs, int n, int max_iter, double err_tol,
    double q_tol)
{
    if (n < 1 || n > SMVSB_MAX_BATCH)
        throw Error(SMVSB_ERR_INVALID, "batch size out of range");
    smvsb_ctx* lead = cs[0];
    void const* kernel = nullptr;
    if (n == 1)
        kernel = (void const*)cg_kernel<1>;
    else if (n == 2)
        kernel = (void const*)cg_kernel<2>;
    else if (n <= 4)
        kernel = (void const*)cg_kernel<4>;
    else
        kernel = (void const*)cg_kernel<8>;

    /* cg_kernel<1> keeps its pass-0 rows of H in shared memory: ask for a
     * carveout that holds two CTAs and leaves the rest of the SM's 256 KB to
     * L1 */
    size_t const dyn_smem = (n == 1) ? CG_PIN_BYTES : 0;
    if (n == 1)
    {
        cudaFuncAttributes fa;
        CUDA_CHECK(cudaFuncGetAttributes(&fa, kernel));
        int smem_sm = 0, reserved = 0;
        CUDA_CHECK(cudaDeviceGetAttribute(&smem_sm,
            cudaDevAttrMaxSharedMemoryPerMultiprocessor, lead->device));
        CUDA_CHECK(cudaDeviceGetAttribute(&reserved,
            cudaDevAttrReservedSharedMemoryPerBlock, lead->device));
        size_t const need = 2 * (dyn_smem + fa.sharedSizeBytes + reserved);
        int const carveout = static_cast<int>(std::min<size_t>(100,
            (100 * need + smem_sm - 1) / smem_sm));
        CUDA_CHECK(cudaFuncSetAttribute(kernel,
            cudaFuncAttributeMaxDynamicSharedMemorySize,
            static_cast<int>(dyn_smem)));
        CUDA_CHECK(cudaFuncSetAttribute(kernel,
            cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
    }
    int per_sm = 0;
    CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm,
        kernel, CG_THREADS, dyn_smem));
    if (per_sm < 1)
        throw Error(SMVSB_ERR_CUDA, "cg_kernel does not fit on an SM");
    /* the grid size fixes the order of the grid-wide sums: a single view is
     * solved with 2 CTAs/SM or not at all */
    if (n == 1 && per_sm < 2)
        throw Error(SMVSB_ERR_CUDA, "cg_kernel<1> fits only "
            + std::to_string(per_sm) + " CTA per SM, needs 2");
    /* (Two views in flight on one GPU with 1 CTA/SM each, so that one view's
     * SpMV runs under the other's barriers and vector update, was slower end
     * to end than 2 CTAs/SM with the two launches taking turns.) */
    int const grid_max = std::min(lead->num_sms * std::min(per_sm, 2),
        CG_MAX_BLOCKS);

    CgArgs a;
    a.n_views = n; a.max_iter = max_iter; a.q_tol = q_tol;
    lead->cg_sync.reserve(1);
    a.sync = lead->cg_sync.p;
    int grid = 1;
    for (int k = 0; k < n; ++k)
    {
        smvsb_ctx* c = cs[k];
        size_t const nn = static_cast<size_t>(c->n_nodes) * 4;
        c->x.reserve(nn); c->r.reserve(nn); c->d.reserve(nn);
        c->d2.reserve(nn); c->Ad.reserve(nn); c->z.reserve(nn);
        c->cg_partials.reserve(static_cast<size_t>(CG_SLOTS) * CG_MAX_BLOCKS);
        c->cg_result.reserve(16);
        mark_system(c);
        CUDA_CHECK(cudaMemsetAsync(c->x.p, 0, nn * sizeof(double),
            c->stream));
        CgView& V = a.v[k];
        V.n_nodes = c->n_nodes; V.npx = c->npx; V.pad = 0;
        int const need = static_cast<int>((nn + CG_THREADS - 1) / CG_THREADS);
        V.grid = std::max(1, std::min(grid_max, need));
        grid = std::max(grid, V.grid);
        V.err_tol = err_tol;
        V.H = c->H.p; V.P = c->P.p; V.g = c->g.p;
        V.rowmask = c->cg_rowmask.p; V.rows = c->cg_row_list.p;
        V.counts = c->cg_counts.p;
        V.x = c->x.p; V.r = c->r.p; V.d = c->d.p; V.d2 = c->d2.p;
        V.Ad = c->Ad.p; V.z = c->z.p;
        V.partials = c->cg_partials.p; V.result = c->cg_result.p;
    }
    CUDA_CHECK(cudaMemsetAsync(a.sync, 0, sizeof(unsigned int), lead->stream));
    void* params[] = { &a };
    CUDA_CHECK(cudaLaunchCooperativeKernel(kernel, dim3(grid),
        dim3(CG_THREADS), params, dyn_smem, lead->stream));
    smvsb::count_launches(lead, 1);
    CUDA_CHECK(cudaGetLastError());
    for (int k = 0; k < n; ++k)
    {
        smvsb_ctx* c = cs[k];
        CUDA_CHECK(cudaMemcpyAsync(c->pinned->cg, c->cg_result.p,
            3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK(cudaMemcpyAsync(c->pinned->cg_counts, c->cg_counts.p,
            2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
            c->stream));
    }
}

void
cg_collect (smvsb_ctx* c, int* iters, int* info, bool* x0_nan)
{
    double const* res = c->pinned->cg;
    c->cg_blocks = c->pinned->cg_counts[0];
    c->cg_rows = c->pinned->cg_counts[1];
    if (iters) *iters = static_cast<int>(res[0]);
    if (info) *info = static_cast<int>(res[1]);
    if (x0_nan) *x0_nan = (res[2] != 0.0);
}

void
run_cg (smvsb_ctx* c, int max_iter, double err_tol, double q_tol, int* iters,
    int* info, bool* x0_nan)
{
    smvsb_ctx* cs[1] = { c };
    cg_enqueue(cs, 1, max_iter, err_tol, q_tol);
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    cg_collect(c, iters, info, x0_nan);
}

} /* namespace smvsb */

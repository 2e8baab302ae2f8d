/*
 * gn_construct.cu -- GaussNewtonStep::construct on the GPU
 * (reference: lib/gauss_newton_step.cc:33-518).
 *
 *   K1  gn_patch_kernel     per patch: 16-vector gradient + 16x16 Hessian
 *                           (jacobian_entries_for_patch +
 *                           fill_gradient_and_hessian_entries, :145-518)
 *   K2a gn_assemble_kernel  per node: gradient entries and the <= 9 4x4
 *                           blocks of the node's block row (:88-142), fixed
 *                           3x3 stencil layout instead of the reference's
 *                           std::map + two transposes
 *   K2b gn_precond_kernel   per node: LDL^T inverse of the diagonal block
 *                           (BlockSparseMatrix::invert_blocks_inplace)
 *
 * K1 layout: 128 threads per block. Phase 1: one thread per sample computes
 * the 6x6 basis-space normal matrix (gn_math.cuh) into shared memory.
 * Phase 2: one thread per (16-sample group, Hessian row) expands
 * D^T A D row by row using the Hermite tensor-product structure of D, so
 * every output row is produced by one thread in a fixed order (deterministic,
 * no atomics) and written as one 128-byte line.
 */
#include "gn_math.cuh"
#include "patch_eval.cuh"

namespace smvsb {

namespace {

constexpr int K1_THREADS = 128;
constexpr int AS_STRIDE = 27;           /* 21 + 6 doubles per sample, odd */

/* Hermite basis and its derivatives on [0,1]; index = side + 2 * order. */
__host__ __device__ inline void
hermite (double t, double* b0, double* b1, double* b2)
{
    double const t2 = t * t, t3 = t2 * t;
    b0[0] = 2 * t3 - 3 * t2 + 1;    /* value at 0 */
    b0[1] = -2 * t3 + 3 * t2;       /* value at 1 */
    b0[2] = t3 - 2 * t2 + t;        /* slope at 0 */
    b0[3] = t3 - t2;                /* slope at 1 */
    b1[0] = 6 * t2 - 6 * t;
    b1[1] = -6 * t2 + 6 * t;
    b1[2] = 3 * t2 - 4 * t + 1;
    b1[3] = 3 * t2 - 2 * t;
    b2[0] = 12 * t - 6;
    b2[1] = -12 * t + 6;
    b2[2] = 6 * t - 4;
    b2[3] = 6 * t - 2;
}

} /* namespace */

/* Host: tables B[order][position][4], first derivatives already divided by
 * ps, second by ps^2 (lib/surface.cc:929-955, lib/surface_patch.cc:101-108).
 * `step` = sampling for the Gauss-Newton samples, 1 for all pixels. */
void
fill_basis_table (std::vector<double>& tab, int ps, int step)
{
    int const npos = ps / step;
    tab.assign(3 * npos * 4, 0.0);
    for (int a = 0; a < npos; ++a)
    {
        double b0[4], b1[4], b2[4];
        hermite((a * step + 0.5) / ps, b0, b1, b2);
        for (int i = 0; i < 4; ++i)
        {
            tab[(0 * npos + a) * 4 + i] = b0[i];
            tab[(1 * npos + a) * 4 + i] = b1[i] / ps;
            tab[(2 * npos + a) * 4 + i] = b2[i] / (double(ps) * ps);
        }
    }
}

/* ------------------------------------------------------------------ */

__global__ void
pack_subview_kernel (float const* __restrict__ grad,
    float const* __restrict__ hess, float* __restrict__ texels, int n)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    float4 a, b;
    a.x = grad[2 * i]; a.y = grad[2 * i + 1];
    a.z = hess[3 * i]; a.w = hess[3 * i + 1];
    b.x = hess[3 * i + 2]; b.y = 0.f; b.z = 0.f; b.w = 0.f;
    reinterpret_cast<float4*>(texels)[2 * i] = a;
    reinterpret_cast<float4*>(texels)[2 * i + 1] = b;
}

void
launch_pack_subview (smvsb_ctx* c, float const* grad, float const* hess,
    float* texels, int w, int h)
{
    int const n = w * h;
    pack_subview_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(grad, hess,
        texels, n);
    smvsb::count_launches(c, 1);
    CUDA_CHECK(cudaGetLastError());
}

/* ------------------------------------------------------------------ */

struct ConstructArgs
{
    SurfaceDev s;
    double regularization;
    double light_surf_regularization;
    double const* light;      /* 16 doubles or null */
    double* patch_H;          /* n_patches * 256 */
    double* patch_g;          /* n_patches * 16 */
    uint8_t* patch_proc;      /* n_patches */
};

/*
 * S = samples per patch (1 / 4 / 16 / 16 / 64 / 64 / 256 / 1024 / 4096 at
 * scales 0..8; lib/gauss_newton_step.cc:157-161 with
 * lib/surface_patch.cc:57-120).
 * S >= 16: groups of 16 samples; a patch of more than 128 samples takes
 * S / 128 chunks of 128.
 * S < 16: 8 patches per block, 8 * S threads busy in phase 1.
 */
/* 4 CTAs / SM at 128 registers, the best of 3 / 4 / 5 / 6 (168 / 128 / 96 /
 * 80 registers). The kernel is fp64-latency bound (4 warps per scheduler).
 * Giving the in-order scheduler two independent streams -- two neighbours'
 * rows computed side by side, the divisions of two pair terms hoisted -- does
 * not help at this register budget: the streams cost more spills than the
 * overlap gains. */
template <int S, int MINB = 4>
__global__ void __launch_bounds__(K1_THREADS, MINB)
gn_patch_kernel (ConstructArgs const args)
{
    /* samples of one patch per chunk, chunks per patch, patches per block,
     * samples per phase-2 group, groups per patch and chunk */
    constexpr int SPC = (S < K1_THREADS) ? S : K1_THREADS;
    constexpr int CHUNKS = S / SPC;
    constexpr int PPB = (S >= 16) ? K1_THREADS / SPC : 8;
    constexpr int GSZ = (S >= 16) ? 16 : S;
    constexpr int GPP = (S >= 16) ? SPC / 16 : 1;
    /* sample positions per side the basis table holds: 16 up to scale 6,
     * 32 / 64 at scales 7 / 8 */
    constexpr int NPOS_MAX = (S <= 256) ? 16 : (S <= 1024 ? 32 : 64);
    /* above 256 samples the partial rows reuse s_as (free after the last
     * chunk), which keeps the 64-position table within 48 KB */
    constexpr bool PART_IN_AS = S > 256;
    SurfaceDev const& sf = args.s;

    __shared__ double s_theta[PPB][16];
    __shared__ double s_coef[PPB][16];        /* coeffs[i][j] at [i * 4 + j] */
    __shared__ double s_as[K1_THREADS * AS_STRIDE];
    __shared__ double s_basis[3 * NPOS_MAX * 4];
    __shared__ double s_part_own[(GPP > 1 && !PART_IN_AS) ? K1_THREADS * 17
        : 1];
    __shared__ int s_proc[PPB];
    static_assert(K1_THREADS * 17 <= K1_THREADS * AS_STRIDE,
        "partial rows must fit in s_as");
    double* const s_part = PART_IN_AS ? s_as : s_part_own;

    int const tid = threadIdx.x;
    int const npos = sf.npos;

    for (int i = tid; i < 3 * npos * 4; i += K1_THREADS)
        s_basis[i] = sf.basis_s[i];

    /* patch bookkeeping */
    if (tid < PPB)
    {
        int const patch = blockIdx.x * PPB + tid;
        int proc = 0;
        if (patch < sf.n_patches && sf.patch_valid[patch])
        {
            int const idx = patch % sf.npx, idy = patch / sf.npx;
            int const n0 = idy * (sf.npx + 1) + idx;
            proc = sf.active[n0] | sf.active[n0 + 1]
                | sf.active[n0 + sf.npx + 1] | sf.active[n0 + sf.npx + 2];
            proc = proc != 0;
        }
        s_proc[tid] = proc;
        if (patch < sf.n_patches)
            args.patch_proc[patch] = static_cast<uint8_t>(proc);
    }
    if (tid < PPB * 16)
    {
        int const pl = tid / 16, col = tid % 16;
        int const patch = blockIdx.x * PPB + pl;
        double v = 0.0;
        if (patch < sf.n_patches)
        {
            int const idx = patch % sf.npx, idy = patch / sf.npx;
            int const node = (idy + ((col >> 3) & 1)) * (sf.npx + 1)
                + idx + ((col >> 2) & 1);
            v = sf.nodes[node * 4 + (col & 3)];
        }
        s_theta[pl][col] = v;
    }
    __syncthreads();

    /* BicubicPatch::compute_coefficients, lib/bicubic_patch.cc:56-86: a = A x
     * with x = (f x4, dx x4, dy x4, dxy x4), summed in index order exactly
     * like the reference, so that the sample values below are bitwise its */
    if (tid < PPB * 16)
    {
        int const pl = tid / 16, r = tid % 16;
        xd sum(0.0);
#pragma unroll
        for (int k = 0; k < 16; ++k)
        {
            /* x[4 * c + node] = theta[node * 4 + c] */
            double const xv = s_theta[pl][(k & 3) * 4 + (k >> 2)];
            sum += xd(c_hermite[r * 16 + k]) * xd(xv);
        }
        /* a[k = j * 4 + i] -> coeffs[i][j] */
        s_coef[pl][(r & 3) * 4 + (r >> 2)] = sum.v;
    }
    __syncthreads();

    /* phase-2 accumulators live across the chunks of a patch */
    int const q = tid / 16;                  /* group in block */
    int const row = tid % 16;
    int const pl2 = q / GPP;
    int const patch2 = blockIdx.x * PPB + pl2;
    bool const proc2 = s_proc[pl2] != 0;
    double hrow[16];
    double grow = 0.0;
#pragma unroll
    for (int i = 0; i < 16; ++i) hrow[i] = 0.0;

    for (int chunk = 0; chunk < CHUNKS; ++chunk)
    {
    /* ---------------- phase 1: one thread per sample ---------------- */
    if (tid < PPB * SPC)
    {
        int const pl = tid / SPC;
        int const s = chunk * SPC + tid % SPC;
        int const patch = blockIdx.x * PPB + pl;
        double A[21], b[6];
#pragma unroll
        for (int i = 0; i < 21; ++i) A[i] = 0.0;
#pragma unroll
        for (int i = 0; i < 6; ++i) b[i] = 0.0;

        if (s_proc[pl])
        {
            int const ix = s % npos, iy = s / npos;

            /* depth and derivatives at the sample: BicubicPatch::evaluate_*
             * (lib/bicubic_patch.cc:121-187) on the polynomial coefficients,
             * then the 1/ps scaling of lib/surface_patch.cc:93-109 -- exact
             * arithmetic in the reference's order (see xd in gn_math.cuh) */
            double w, wx, wy, wxy, wxx, wyy;
            {
                double const* cf = s_coef[pl];
                /* the patch size is a power of two: dividing by it and
                 * multiplying by its reciprocal are the same exact scaling */
                xd const inv_size(1.0 / static_cast<double>(sf.ps));
                xd const sx = (xd(static_cast<double>(ix * sf.sampling))
                    + xd(0.5)) * inv_size;
                xd const sy = (xd(static_cast<double>(iy * sf.sampling))
                    + xd(0.5)) * inv_size;
                xd ex[4], ey[4];
                ex[0] = xd(1.0); ex[1] = sx; ex[2] = sx * sx; ex[3] = ex[2] * sx;
                ey[0] = xd(1.0); ey[1] = sy; ey[2] = sy * sy; ey[3] = ey[2] * sy;
                xd f(0.0), fx(0.0), fy(0.0), fxy(0.0), fxx(0.0), fyy(0.0);
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        f += xd(cf[i * 4 + j]) * ex[i] * ey[j];
#pragma unroll
                for (int i = 1; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        fx += xd(cf[i * 4 + j]) * xd(double(i)) * ex[i - 1]
                            * ey[j];
#pragma unroll
                for (int i = 2; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        fxx += xd(cf[i * 4 + j]) * xd(double(i))
                            * xd(double(i - 1)) * ex[i - 2] * ey[j];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 1; j < 4; ++j)
                        fy += xd(cf[i * 4 + j]) * ex[i] * xd(double(j))
                            * ey[j - 1];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 2; j < 4; ++j)
                        fyy += xd(cf[i * 4 + j]) * ex[i] * xd(double(j))
                            * xd(double(j - 1)) * ey[j - 2];
#pragma unroll
                for (int i = 1; i < 4; ++i)
#pragma unroll
                    for (int j = 1; j < 4; ++j)
                        fxy += xd(cf[i * 4 + j]) * xd(double(i)) * ex[i - 1]
                            * xd(double(j)) * ey[j - 1];
                xd const inv_size2(1.0 / static_cast<double>(sf.ps * sf.ps));
                w = f.v;
                wx = (fx * inv_size).v;
                wy = (fy * inv_size).v;
                wxy = (fxy * inv_size2).v;
                wxx = (fxx * inv_size2).v;
                wyy = (fyy * inv_size2).v;
            }

            int const idx = patch % sf.npx, idy = patch / sf.npx;
            int const px = sf.start_x + idx * sf.ps + ix * sf.sampling;
            int const py = sf.start_y + idy * sf.ps + iy * sf.sampling;
            size_t const pix = static_cast<size_t>(py) * sf.w + px;
            float2 const gm = __ldg(
                reinterpret_cast<float2 const*>(sf.main_grad) + pix);
            double const gmx = gm.x, gmy = gm.y;

            /* per-neighbour rows, lib/gauss_newton_step.cc:175-208 */
            uint32_t const v0 = sf.vis_off[patch];
            int const n = static_cast<int>(sf.vis_off[patch + 1] - v0);
            NbRow rows[SMVSB_MAX_SUBS];
            for (int j = 0; j < n; ++j)
            {
                int const sub = sf.vis_ids[v0 + j];
                rows[j] = neighbour_row(sf.Mt + sub * 12, sf.sub_texels[sub],
                    sf.sub_dims[2 * sub], sf.sub_dims[2 * sub + 1],
                    px + 0.5, py + 0.5, w, wx, wy);
            }

            /* photometric terms, lib/gauss_newton_step.cc:263-321 */
            for (int j = 0; j < n; ++j)
            {
                NbRow const rj = rows[j];
                double const dx_ = rj.jgx - gmx, dy_ = rj.jgy - gmy;
                add_photo_row<1>(A, b, rj.ax, rj.be, dx_,
                    1.0 / (fabs(dx_) + SMVSB_R_FACTOR));
                add_photo_row<2>(A, b, rj.ay, rj.be, dy_,
                    1.0 / (fabs(dy_) + SMVSB_R_FACTOR));
                for (int j2 = j + 1; j2 < n; ++j2)
                {
                    NbRow const r2 = rows[j2];
                    double const sx_ = rj.jgx - r2.jgx;
                    double const sy_ = rj.jgy - r2.jgy;
                    double const be = rj.be - r2.be;
                    add_photo_row<1>(A, b, rj.ax - r2.ax, be, sx_,
                        1.0 / (fabs(sx_) + SMVSB_R_FACTOR));
                    add_photo_row<2>(A, b, rj.ay - r2.ay, be, sy_,
                        1.0 / (fabs(sy_) + SMVSB_R_FACTOR));
                }
            }

            if (args.regularization > 0.0)
            {
                /* lib/gauss_newton_step.cc:210-240, 388-417 */
                double const num_diffs = double((n * (n + 1)) / 2);
                double const basic = args.regularization * 0.005
                    / fmax(0.03, fabs(gmx) + fabs(gmy)) * num_diffs;
                double const x = px + 0.5 - static_cast<double>(sf.w) / 2.0;
                double const y = py + 0.5 - static_cast<double>(sf.h) / 2.0;
                SurfGeo geo;
                surface_geometry(x, y, sf.flen, w, wx, wy, wxy, wxx, wyy, geo);

                bool const lit = (args.light != nullptr);
                if (!lit || args.light_surf_regularization > 0.0)
                {
                    double geom_weight = 1.0;
                    if (lit)
                        geom_weight *= args.light_surf_regularization / 100;
#pragma unroll
                    for (int v = 0; v < 6; ++v)
                    {
                        double const wgt = geom_weight
                            / (SMVSB_R_FACTOR + fabs(geo.div[v])) * basic;
                        add_full_row(A, b, geo.C[v], geo.div[v], wgt);
                    }
                }

                if (lit)
                {
                    /* shading term, lib/gauss_newton_step.cc:419-515 */
                    double L[16];
#pragma unroll
                    for (int l = 0; l < 16; ++l) L[l] = args.light[l];
                    double nrm[3];
                    fill_normal(x, y, sf.inv_flen, w, wx, wy, nrm);
                    double sh[16];
                    sh_evaluate_4_band(nrm, sh);
                    double shading = 0.0;
#pragma unroll
                    for (int l = 0; l < 16; ++l) shading += L[l] * sh[l];
                    float2 const lg = __ldg(reinterpret_cast<float2 const*>(
                        sf.main_shading_grad) + pix);
                    double ligx = lg.x, ligy = lg.y;
                    double const liv = __ldg(sf.main_shading + pix);
                    double const shading_weight = 0.001 * num_diffs
                        / (SMVSB_R_FACTOR + fabs(ligx) + fabs(ligy));
                    bool ok = !(sqrt(ligx * ligx + ligy * ligy) < 1e-10);
                    ok = ok && !(shading * shading < 1e-10
                        || liv * liv < 1e-10);
                    if (ok)
                    {
                        double G[3];
                        sh_light_gradient(nrm, L, G);
                        double const sgx = G[0] * geo.div[0]
                            + G[1] * geo.div[1] + G[2] * geo.div[2];
                        double const sgy = G[0] * geo.div[3]
                            + G[1] * geo.div[4] + G[2] * geo.div[5];
                        double const inv_s = 1.0 / shading;
                        ligx *= 1.0 / liv;
                        ligy *= 1.0 / liv;
                        double const ex = sgx * inv_s - ligx;
                        double const ey = sgy * inv_s - ligy;
                        double cx[6], cy[6];
                        double const inv_s2 = 1.0 / (shading * shading);
#pragma unroll
                        for (int k = 0; k < 6; ++k)
                        {
                            double const sd = (k < 3) ? G[0] * geo.N[0][k]
                                + G[1] * geo.N[1][k] + G[2] * geo.N[2][k]
                                : 0.0;
                            double const gdx = G[0] * geo.C[0][k]
                                + G[1] * geo.C[1][k] + G[2] * geo.C[2][k];
                            double const gdy = G[0] * geo.C[3][k]
                                + G[1] * geo.C[4][k] + G[2] * geo.C[5][k];
                            cx[k] = (gdx * shading - sgx * sd) * inv_s2;
                            cy[k] = (gdy * shading - sgy * sd) * inv_s2;
                        }
                        add_full_row(A, b, cx, ex, shading_weight
                            / (SMVSB_R_FACTOR + fabs(ex)));
                        add_full_row(A, b, cy, ey, shading_weight
                            / (SMVSB_R_FACTOR + fabs(ey)));
                    }
                }
            }
        }

        double* dst = s_as + tid * AS_STRIDE;
#pragma unroll
        for (int i = 0; i < 21; ++i) dst[i] = A[i];
#pragma unroll
        for (int i = 0; i < 6; ++i) dst[21 + i] = b[i];
    }
    __syncthreads();

    /* ------- phase 2: one thread per (sample group, row) ----------- */
    if (proc2)
    {
        int const rbx = ((row >> 2) & 1) + 2 * (row & 1);
        int const rby = ((row >> 3) & 1) + 2 * ((row >> 1) & 1);
        for (int ss = 0; ss < GSZ; ++ss)
        {
            int const sl = (q % GPP) * GSZ + ss;     /* sample in chunk */
            int const s = chunk * SPC + sl;          /* sample in patch */
            int const ix = s % npos, iy = s / npos;
            double const* as = s_as + (pl2 * SPC + sl) * AS_STRIDE;
            double const* X0 = s_basis + (0 * npos + ix) * 4;
            double const* X1 = s_basis + (1 * npos + ix) * 4;
            double const* X2 = s_basis + (2 * npos + ix) * 4;
            double const* Y0 = s_basis + (0 * npos + iy) * 4;
            double const* Y1 = s_basis + (1 * npos + iy) * 4;
            double const* Y2 = s_basis + (2 * npos + iy) * 4;

            /* D_k[row] */
            double Dr[6];
            Dr[0] = X0[rbx] * Y0[rby];
            Dr[1] = X1[rbx] * Y0[rby];
            Dr[2] = X0[rbx] * Y1[rby];
            Dr[3] = X1[rbx] * Y1[rby];
            Dr[4] = X2[rbx] * Y0[rby];
            Dr[5] = X0[rbx] * Y2[rby];

            /* E = A * D[:, row], gradient entry */
            double E[6];
#pragma unroll
            for (int k = 0; k < 6; ++k)
            {
                double e = 0.0;
#pragma unroll
                for (int l = 0; l < 6; ++l)
                    e += as[(k <= l) ? sym6(k, l) : sym6(l, k)] * Dr[l];
                E[k] = e;
                grow += as[21 + k] * Dr[k];
            }

            /* hrow[(bx,by)] += sum_k E_k X_k[bx] Y_k[by], grouped by X */
            double U0[4], U1[4], U2[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
            {
                U0[j] = E[0] * Y0[j] + E[2] * Y1[j] + E[5] * Y2[j];
                U1[j] = E[1] * Y0[j] + E[3] * Y1[j];
                U2[j] = E[4] * Y0[j];
            }
#pragma unroll
            for (int col = 0; col < 16; ++col)
            {
                int const bx = ((col >> 2) & 1) + 2 * (col & 1);
                int const by = ((col >> 3) & 1) + 2 * ((col >> 1) & 1);
                hrow[col] += X0[bx] * U0[by] + X1[bx] * U1[by]
                    + X2[bx] * U2[by];
            }
        }
    }
    if (CHUNKS > 1)
        __syncthreads();     /* s_as is rewritten by the next chunk */
    } /* chunk */

    if (GPP == 1)
    {
        if (proc2 && patch2 < sf.n_patches)
        {
            double2* dst = reinterpret_cast<double2*>(
                args.patch_H + (static_cast<size_t>(patch2) * 16 + row) * 16);
#pragma unroll
            for (int i = 0; i < 8; ++i)
                dst[i] = make_double2(hrow[2 * i], hrow[2 * i + 1]);
            args.patch_g[static_cast<size_t>(patch2) * 16 + row] = grow;
        }
    }
    else
    {
        /* sum the GPP partial rows of a patch in fixed order */
        double* part = s_part + tid * 17;
#pragma unroll
        for (int i = 0; i < 16; ++i) part[i] = hrow[i];
        part[16] = grow;
        __syncthreads();
        if (tid < PPB * 16)
        {
            int const pl = tid / 16, r = tid % 16;
            int const patch = blockIdx.x * PPB + pl;
            if (s_proc[pl] && patch < sf.n_patches)
            {
                double acc[17];
#pragma unroll
                for (int i = 0; i < 17; ++i) acc[i] = 0.0;
                for (int gq = 0; gq < GPP; ++gq)
                {
                    double const* p = s_part
                        + ((pl * GPP + gq) * 16 + r) * 17;
#pragma unroll
                    for (int i = 0; i < 17; ++i) acc[i] += p[i];
                }
                double* dst = args.patch_H
                    + (static_cast<size_t>(patch) * 16 + r) * 16;
#pragma unroll
                for (int i = 0; i < 16; ++i) dst[i] = acc[i];
                args.patch_g[static_cast<size_t>(patch) * 16 + r] = acc[16];
            }
        }
    }
}

/* ------------------------------------------------------------------ */

/*
 * One thread per (node, stencil block k, block row rp): sums the matching
 * 1x4 row segments of the <= 4 adjacent patches
 * (lib/gauss_newton_step.cc:98-121; rows / columns of inactive nodes are
 * dropped, :91,101,105). H layout: [node][k = (dy+1)*3 + (dx+1)][rp][cp],
 * block(row = node, col = neighbour), so y_node += B * x_neighbour.
 */
__global__ void
gn_assemble_kernel (SurfaceDev const sf, double const* __restrict__ patch_H,
    double const* __restrict__ patch_g,
    uint8_t const* __restrict__ patch_proc, double* __restrict__ H,
    double* __restrict__ g)
{
    int const gid = blockIdx.x * blockDim.x + threadIdx.x;
    int const node = gid / 36;
    int const rem = gid % 36;
    int const k = rem / 4, rp = rem % 4;
    if (node >= sf.n_nodes)
        return;

    int const ns = sf.npx + 1;
    int const ix = node % ns, iy = node / ns;
    int const dx = k % 3 - 1, dy = k / 3 - 1;
    int const jx = ix + dx, jy = iy + dy;

    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    double gacc = 0.0;
    bool const row_on = sf.node_valid[node] && sf.active[node];
    bool col_on = false;
    if (jx >= 0 && jx <= sf.npx && jy >= 0 && jy <= sf.npy)
    {
        int const nj = jy * ns + jx;
        col_on = sf.node_valid[nj] && sf.active[nj];
    }

    if (row_on)
    {
#pragma unroll
        for (int pb = 0; pb < 2; ++pb)
#pragma unroll
            for (int pa = 0; pa < 2; ++pa)
            {
                int const ppx = ix - 1 + pa, ppy = iy - 1 + pb;
                if (ppx < 0 || ppx >= sf.npx || ppy < 0 || ppy >= sf.npy)
                    continue;
                int const patch = ppy * sf.npx + ppx;
                if (!patch_proc[patch])
                    continue;
                int const li = (1 - pa) + 2 * (1 - pb);
                if (k == 4)
                    gacc += patch_g[static_cast<size_t>(patch) * 16
                        + li * 4 + rp];
                int const ljx = dx + 1 - pa, ljy = dy + 1 - pb;
                if (!col_on || ljx < 0 || ljx > 1 || ljy < 0 || ljy > 1)
                    continue;
                int const lj = ljx + 2 * ljy;
                double const* src = patch_H + (static_cast<size_t>(patch) * 16
                    + li * 4 + rp) * 16 + lj * 4;
                double2 const a = *reinterpret_cast<double2 const*>(src);
                double2 const b = *reinterpret_cast<double2 const*>(src + 2);
                acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
            }
    }
    double2* dst = reinterpret_cast<double2*>(
        H + (static_cast<size_t>(node) * 9 + k) * 16 + rp * 4);
    dst[0] = make_double2(acc[0], acc[1]);
    dst[1] = make_double2(acc[2], acc[3]);
    if (k == 4)
        g[static_cast<size_t>(node) * 4 + rp] = gacc;
}

/* BlockSparseMatrix::invert_blocks_inplace, lib/block_sparse_matrix.h:300-316:
 * P = inverse of the diagonal block; a NaN result or a zero pivot keeps the
 * un-inverted block. Nodes without a diagonal block get P = 0. */
__global__ void
gn_precond_kernel (SurfaceDev const sf, double const* __restrict__ H,
    double* __restrict__ P)
{
    int const node = blockIdx.x * blockDim.x + threadIdx.x;
    if (node >= sf.n_nodes)
        return;
    double A[16], out[16];
    bool const on = sf.node_valid[node] && sf.active[node];
    double const* src = H + (static_cast<size_t>(node) * 9 + 4) * 16;
#pragma unroll
    for (int i = 0; i < 16; ++i) A[i] = on ? src[i] : 0.0;
    if (on)
    {
        bool ok = ldl_inverse4(A, out);
        if (ok)
        {
            bool nan = false;
#pragma unroll
            for (int i = 0; i < 16; ++i) nan = nan || isnan(out[i]);
            ok = !nan;
        }
        if (!ok)
        {
#pragma unroll
            for (int i = 0; i < 16; ++i) out[i] = A[i];
        }
    }
    else
    {
#pragma unroll
        for (int i = 0; i < 16; ++i) out[i] = 0.0;
    }
    double* dst = P + static_cast<size_t>(node) * 16;
#pragma unroll
    for (int i = 0; i < 16; ++i) dst[i] = out[i];
}

void
launch_construct (smvsb_ctx* c, bool use_light, double reg, double light_reg)
{
    ConstructArgs a;
    a.s = surface_args(c);
    a.regularization = reg;
    a.light_surf_regularization = light_reg;
    a.light = use_light ? c->light.p : nullptr;
    a.patch_H = c->patch_H.p;
    a.patch_g = c->patch_g.p;
    a.patch_proc = c->patch_proc.p;

    /* samples per patch: 1 (scale 0), 4 (scale 1), 16 (scales 2, 3),
     * 64 (scales 4, 5), 256 (scale 6), 1024 (scale 7), 4096 (scale 8),
     * lib/gauss_newton_step.cc:157-161 */
    int const S = c->npos * c->npos;
    auto blocks = [&](int ppb) { return (c->n_patches + ppb - 1) / ppb; };
    switch (S)
    {
    case 1:
        gn_patch_kernel<1><<<blocks(8), K1_THREADS, 0, c->stream>>>(a); break;
    case 4:
        gn_patch_kernel<4><<<blocks(8), K1_THREADS, 0, c->stream>>>(a); break;
    case 16:
    {
        gn_patch_kernel<16><<<blocks(8), K1_THREADS, 0, c->stream>>>(a);
        break;
    }
    case 64:
        gn_patch_kernel<64><<<blocks(2), K1_THREADS, 0, c->stream>>>(a); break;
    case 256:
        gn_patch_kernel<256><<<blocks(1), K1_THREADS, 0, c->stream>>>(a); break;
    case 1024:
        gn_patch_kernel<1024><<<blocks(1), K1_THREADS, 0, c->stream>>>(a);
        break;
    case 4096:
        gn_patch_kernel<4096><<<blocks(1), K1_THREADS, 0, c->stream>>>(a);
        break;
    default:
        throw Error(SMVSB_ERR_INVALID, "unsupported samples per patch");
    }
    CUDA_CHECK(cudaGetLastError());

    int const n_thr = c->n_nodes * 36;
    gn_assemble_kernel<<<(n_thr + 287) / 288, 288, 0, c->stream>>>(a.s,
        c->patch_H.p, c->patch_g.p, c->patch_proc.p, c->H.p, c->g.p);
    CUDA_CHECK(cudaGetLastError());
    gn_precond_kernel<<<(c->n_nodes + 127) / 128, 128, 0, c->stream>>>(a.s,
        c->H.p, c->P.p);
    CUDA_CHECK(cudaGetLastError());
    smvsb::count_launches(c, 3);
}

} /* namespace smvsb */

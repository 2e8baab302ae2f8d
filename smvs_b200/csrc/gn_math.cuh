/*
 * gn_math.cuh -- per-sample math of the Gauss-Newton step, written for the
 * GPU in "basis space".
 *
 * Every residual row the reference builds (lib/gauss_newton_step.cc:200-207,
 * 220-240, 450-499) is a linear combination of the six node-derivative rows
 *     D_k[col] = d(q_k)/d(theta_col),  q = (w, wx, wy, wxy, wxx, wyy),
 * of the bicubic patch (lib/bicubic_patch.cc:258-316). So instead of carrying
 * 16-column rows per residual, a sample accumulates the 6x6 normal matrix
 * A = sum_rho weight * c c^T and b = sum_rho weight * rho * c of the
 * coefficient vectors c in R^6, and the 16x16 patch block is D^T A D
 * (done cooperatively in gn_construct.cu). D itself is a Hermite tensor
 * product, D_k[col(ix,iy)] = X_k[ix] * Y_k[iy].
 */
#ifndef SMVSB_GN_MATH_CUH
#define SMVSB_GN_MATH_CUH

#include "common.cuh"

namespace smvsb {

#define SMVSB_R_FACTOR 1e-4     /* lib/gauss_newton_step.cc:17 */

/* index of (k,l), k <= l, in the packed upper triangle of a 6x6 */
__host__ __device__ constexpr int
sym6 (int k, int l)
{
    return k * 6 - (k * (k - 1)) / 2 + (l - k);
}

/*
 * "Exact double": arithmetic with explicit round-to-nearest instructions, so
 * the compiler cannot contract a*b+c into an FMA. Several formulas of the
 * path subtract nearly equal products (p*d - r*a, dxx*n - dx*nx, second
 * derivatives of a smooth depth field from Hermite data, ...); at 2 MP their
 * rounding noise is amplified 1e3..1e5 x, so evaluating them in a different
 * order than the CPU costs parity (1e-9 instead of 1e-13 on the Hessian).
 * Code written with xd in the reference's expression order is bitwise equal
 * to the reference built with -ffp-contract=off.
 */
struct xd
{
    double v;
    __device__ __forceinline__ xd (void) {}
    __device__ __forceinline__ xd (double a) : v(a) {}
};
__device__ __forceinline__ xd operator+ (xd a, xd b) { return xd(__dadd_rn(a.v, b.v)); }
__device__ __forceinline__ xd operator- (xd a, xd b) { return xd(__dadd_rn(a.v, -b.v)); }
__device__ __forceinline__ xd operator* (xd a, xd b) { return xd(__dmul_rn(a.v, b.v)); }
__device__ __forceinline__ xd operator/ (xd a, xd b) { return xd(__ddiv_rn(a.v, b.v)); }
__device__ __forceinline__ xd operator- (xd a) { return xd(-a.v); }
__device__ __forceinline__ xd& operator+= (xd& a, xd b) { a = a + b; return a; }
__device__ __forceinline__ xd& operator-= (xd& a, xd b) { a = a - b; return a; }
__device__ __forceinline__ xd& operator/= (xd& a, xd b) { a = a / b; return a; }
__device__ __forceinline__ xd xsqrt (xd a) { return xd(__dsqrt_rn(a.v)); }

/* Division by a divisor that is used many times: r = RN(1 / d) once (a true
 * division), then per quotient q = RN(x r), e = x - d q (exact in an FMA),
 * RN(q + e r) -- Markstein's correction step, which returns the correctly
 * rounded x / d whenever q is within one ulp of it. Three instructions
 * instead of the ~13 of a division; gn_patch_kernel divides 22 times per
 * sample and neighbour by d, d^2 and d^4. (The decision kernels of
 * visibility.cu keep true divisions: there every bit counts; here a rare
 * last-bit difference is far below the 4e-15 of the row sums.) */
struct xrecip
{
    double d, r;
};
__device__ __forceinline__ xrecip xrcp (xd d)
{
    xrecip out;
    out.d = d.v;
    out.r = __ddiv_rn(1.0, d.v);
    return out;
}
__device__ __forceinline__ xd operator/ (xd x, xrecip const& c)
{
    double const q = __dmul_rn(x.v, c.r);
    double const e = __fma_rn(-c.d, q, x.v);
    return xd(__fma_rn(e, c.r, q));
}

/*
 * mve::Image<float>::linear_at on a packed neighbour texel image, restated
 * bit-for-bit: coordinates narrowed to fp32 and clamped to the image, fp32
 * weights, left-to-right fp32 sum without FMA contraction
 * (call sites lib/gauss_newton_step.cc:192-198).
 */
__device__ __forceinline__ void
tap_neighbour (float const* __restrict__ tex, int w, int h, double px,
    double py, float out[5])
{
    float x = static_cast<float>(px);
    float y = static_cast<float>(py);
    x = fmaxf(0.0f, fminf(static_cast<float>(w - 1), x));
    y = fmaxf(0.0f, fminf(static_cast<float>(h - 1), y));
    int const fx = static_cast<int>(x);
    int const fy = static_cast<int>(y);
    int const fx1 = min(fx + 1, w - 1);
    int const fy1 = min(fy + 1, h - 1);
    float const w1 = x - static_cast<float>(fx);
    float const w0 = 1.0f - w1;
    float const w3 = y - static_cast<float>(fy);
    float const w2 = 1.0f - w3;
    float const w00 = __fmul_rn(w0, w2), w10 = __fmul_rn(w1, w2);
    float const w01 = __fmul_rn(w0, w3), w11 = __fmul_rn(w1, w3);

    float4 const* t00 = reinterpret_cast<float4 const*>(
        tex + (static_cast<size_t>(fy) * w + fx) * SMVSB_NB_STRIDE);
    float4 const* t10 = reinterpret_cast<float4 const*>(
        tex + (static_cast<size_t>(fy) * w + fx1) * SMVSB_NB_STRIDE);
    float4 const* t01 = reinterpret_cast<float4 const*>(
        tex + (static_cast<size_t>(fy1) * w + fx) * SMVSB_NB_STRIDE);
    float4 const* t11 = reinterpret_cast<float4 const*>(
        tex + (static_cast<size_t>(fy1) * w + fx1) * SMVSB_NB_STRIDE);
    float4 const a0 = __ldg(t00), a1 = __ldg(t00 + 1);
    float4 const b0 = __ldg(t10), b1 = __ldg(t10 + 1);
    float4 const c0 = __ldg(t01), c1 = __ldg(t01 + 1);
    float4 const d0 = __ldg(t11), d1 = __ldg(t11 + 1);

#define SMVSB_TAP(A, B, C, D) __fadd_rn(__fadd_rn(__fadd_rn(                \
        __fmul_rn(A, w00), __fmul_rn(B, w10)), __fmul_rn(C, w01)),          \
        __fmul_rn(D, w11))
    out[0] = SMVSB_TAP(a0.x, b0.x, c0.x, d0.x);
    out[1] = SMVSB_TAP(a0.y, b0.y, c0.y, d0.y);
    out[2] = SMVSB_TAP(a0.z, b0.z, c0.z, d0.z);
    out[3] = SMVSB_TAP(a0.w, b0.w, c0.w, d0.w);
    out[4] = SMVSB_TAP(a1.x, b1.x, c1.x, d1.x);
#undef SMVSB_TAP
}

/* What one neighbour contributes to a sample: J*grad_sub and the three
 * basis coefficients of its two Jacobian rows
 * (x row = ax*D_w + be*D_wx, y row = ay*D_w + be*D_wy). */
struct NbRow
{
    double jgx, jgy, ax, ay, be;
};

/*
 * Correspondence::update/fill/fill_jacobian/fill_derivative/
 * fill_jacobian_derivative_grad (lib/correspondence.cc:20-187) and the
 * jac_entries assembly (lib/gauss_newton_step.cc:200-207) for one neighbour.
 */
__device__ __forceinline__ NbRow
neighbour_row (double const* __restrict__ Mt, float const* __restrict__ tex,
    int sw, int sh, double u, double v, double w, double wx, double wy)
{
    double const M0 = Mt[0], M1 = Mt[1], M2 = Mt[2];
    double const M3 = Mt[3], M4 = Mt[4], M5 = Mt[5];
    double const M6 = Mt[6], M7 = Mt[7], M8 = Mt[8];
    double const t0 = Mt[9], t1 = Mt[10], t2 = Mt[11];

    /* exact arithmetic in the reference's expression order (see xd) */
    xd const m0(M0), m1(M1), m2(M2), m3(M3), m4(M4), m5(M5), m6(M6), m7(M7),
        m8(M8), T0(t0), T1(t1), T2(t2), W(w), WX(wx), WY(wy), U(u), V(v);
    /* update, lib/correspondence.cc:20-44 */
    xd const p = m0 * U + m1 * V + m2;
    xd const q = m3 * U + m4 * V + m5;
    xd const r = m6 * U + m7 * V + m8;
    xd const a = W * p + T0;
    xd const b = W * q + T1;
    xd const d = W * r + T2;
    xd const d2 = d * d;
    xrecip const rd = xrcp(d), rd2 = xrcp(d2);

    /* fill (:46-51) and the caller's -0.5 (gauss_newton_step.cc:189-190) */
    double const projx = (a / rd - xd(0.5)).v;
    double const projy = (b / rd - xd(0.5)).v;
    /* fill_jacobian, :88-100 */
    xd j0 = (WX * p + W * m0) / rd;
    xd j2 = (WY * p + W * m1) / rd;
    j0 -= a * (WX * r + W * m6) / rd2;
    j2 -= a * (WY * r + W * m7) / rd2;
    xd j1 = (WX * q + W * m3) / rd;
    xd j3 = (WY * q + W * m4) / rd;
    j1 -= b * (WX * r + W * m6) / rd2;
    j3 -= b * (WY * r + W * m7) / rd2;

    float tap[5];
    tap_neighbour(tex, sw, sh, projx, projy, tap);
    xd const GX(tap[0]), GY(tap[1]), H0(tap[2]), H1(tap[3]), H3(tap[4]);
    double const gx = GX.v, gy = GY.v;

    NbRow out;
    /* jac * grad_sub and jac * hess_sub (row times column, left to right) */
    out.jgx = (j0 * GX + j1 * GY).v;
    out.jgy = (j2 * GX + j3 * GY).v;
    double const jh00 = (j0 * H0 + j1 * H1).v;
    double const jh01 = (j0 * H1 + j1 * H3).v;
    double const jh10 = (j2 * H0 + j3 * H1).v;
    double const jh11 = (j2 * H1 + j3 * H3).v;
    /* fill_derivative, :74-86 */
    double const du_w = ((p * d - r * a) / rd2).v;
    double const dv_w = ((q * d - r * b) / rd2).v;

    /* fill_jacobian_derivative_grad, :102-187 */
    xd const d4 = d2 * d2;
    xrecip const rd4 = xrcp(d4);
    xd const d_prime = xd(2.0) * d * r;
    xd const du_c_prime = p * T2 - r * T0;
    xd const dv_c_prime = q * T2 - r * T1;
    xd const du_a_t0 = W * (m0 * r - p * m6), du_a_t1 = W * (m1 * r - p * m7);
    xd const du_b0 = m0 * T2 - m6 * T0, du_b1 = m1 * T2 - m7 * T0;
    xd const dv_a_t0 = W * (m3 * r - q * m6), dv_a_t1 = W * (m4 * r - q * m7);
    xd const dv_b0 = m3 * T2 - m6 * T1, dv_b1 = m4 * T2 - m7 * T1;
    double const A0 = ((xd(2.0) * du_a_t0 + du_b0) / rd2
        - (W * (du_a_t0 + du_b0) + WX * du_c_prime) * d_prime / rd4).v;
    double const A1 = ((xd(2.0) * du_a_t1 + du_b1) / rd2
        - (W * (du_a_t1 + du_b1) + WY * du_c_prime) * d_prime / rd4).v;
    double const B0 = ((xd(2.0) * dv_a_t0 + dv_b0) / rd2
        - (W * (dv_a_t0 + dv_b0) + WX * dv_c_prime) * d_prime / rd4).v;
    double const B1 = ((xd(2.0) * dv_a_t1 + dv_b1) / rd2
        - (W * (dv_a_t1 + dv_b1) + WY * dv_c_prime) * d_prime / rd4).v;
    double const cu = (du_c_prime / rd2).v;
    double const cv = (dv_c_prime / rd2).v;

    out.ax = A0 * gx + B0 * gy + jh00 * du_w + jh01 * dv_w;
    out.ay = A1 * gx + B1 * gy + jh10 * du_w + jh11 * dv_w;
    out.be = cu * gx + cv * gy;
    return out;
}

/* A += wgt * c c^T, b += wgt * rho * c for a row with coefficients on the
 * basis functions 0 (D_w) and K (D_wx: 1, D_wy: 2) only. */
template <int K>
__device__ __forceinline__ void
add_photo_row (double* A, double* b, double c0, double ck, double rho,
    double wgt)
{
    double const w0 = c0 * wgt, wk = ck * wgt;
    A[sym6(0, 0)] += w0 * c0;
    A[sym6(0, K)] += w0 * ck;
    A[sym6(K, K)] += wk * ck;
    b[0] += w0 * rho;
    b[K] += wk * rho;
}

__device__ __forceinline__ void
add_full_row (double* A, double* b, double const* c, double rho, double wgt)
{
#pragma unroll
    for (int k = 0; k < 6; ++k)
    {
        double const wk = c[k] * wgt;
        b[k] += wk * rho;
#pragma unroll
        for (int l = k; l < 6; ++l)
            A[sym6(k, l)] += wk * c[l];
    }
}

/*
 * surfderiv::normal_divergence, normal_divergence_deriv and normal_derivative
 * (lib/surface_derivative.cc:31-190), with the derivative expressed as
 * coefficients on (w', wx', wy', wxy', wxx', wyy').
 *   div[6]      the six entries of d(normal)/d(pixel)
 *   C[v][k]     d(div[v]) / d(q_k)
 *   N[c][k]     d(normal[c]) / d(q_k), k < 3 (the rest is zero)
 */
struct SurfGeo
{
    double div[6];
    double C[6][6];
    double N[3][3];
};

__device__ __forceinline__ void
surface_geometry (double x_, double y_, double f_, double w_, double dx_,
    double dy_, double dxy_, double dxx_, double dyy_, SurfGeo& g)
{
    /* exact arithmetic in the reference's expression order (see xd) */
    xd const x(x_), y(y_), f(f_), w(w_), dx(dx_), dy(dy_), dxy(dxy_),
        dxx(dxx_), dyy(dyy_);
    xd const a = w + x * dx + y * dy;
    xd const ax = xd(2.0) * dx + x * dxx + y * dxy;
    xd const ay = xd(2.0) * dy + y * dyy + x * dxy;

    /* normal_divergence, :69-107 */
    {
        xd t = a / f;
        t = t * t;
        t += dx * dx + dy * dy;
        xd const n = xsqrt(t);
        xd nx = dx * dxx + dy * dxy;
        nx += (xd(1.0) / (f * f)) * (w + x * dx + y * dy)
            * (dx + dx + x * dxx + y * dxy);
        nx /= n;
        xd ny = dx * dxy + dy * dyy;
        ny += (xd(1.0) / (f * f)) * (w + x * dx + y * dy)
            * (dy + dy + x * dxy + y * dyy);
        ny /= n;
        g.div[0] = ((dxx * n - dx * nx) / t).v;
        g.div[1] = (-((dxy * n - dy * nx) / t)).v;
        g.div[2] = ((ax * n - a * nx) / (t * f)).v;
        g.div[3] = ((dxy * n - dx * ny) / t).v;
        g.div[4] = (-((dyy * n - dy * ny) / t)).v;
        g.div[5] = ((ay * n - a * ny) / (t * f)).v;
    }

    /* normal_divergence_deriv, :109-190, and normal_derivative, :31-65,
     * applied to the six unit "prime" vectors. The shared quantities
     * (t, n, b, c, nx, ny) are exact; the coefficients themselves are only
     * ever combined linearly with the basis rows, so ordinary (contracted)
     * double arithmetic is enough for them and much cheaper. */
    xd const f_sqr_inv_x = xd(1.0) / (f * f);
    xd const a_f2_x = a * f_sqr_inv_x;
    xd const t_x = dx * dx + dy * dy + a * a_f2_x;
    xd const n_x = xsqrt(t_x);
    xd const b_x = dx * dxx + dy * dxy
        + a_f2_x * (xd(2.0) * dx + x * dxx + y * dxy);
    xd const c_x = dx * dxy + dy * dyy
        + a_f2_x * (xd(2.0) * dy + x * dxy + y * dyy);
    double const f_sqr_inv = f_sqr_inv_x.v, t = t_x.v, n = n_x.v;
    double const b = b_x.v, c = c_x.v;
    double const nx = (b_x / n_x).v, ny = (c_x / n_x).v;
    double const X = x_, Y = y_, F = f_, A = a.v, AX = ax.v, AY = ay.v;
    double const DX = dx_, DY = dy_, DXY = dxy_, DXX = dxx_, DYY = dyy_;
    double const inv_t = 1.0 / t;
    double const inv_n = 1.0 / n;
    double const inv_tt = inv_t * inv_t;
    double const inv_ttf = inv_tt / F;
    double const inv_tf = inv_t / F;

#pragma unroll
    for (int k = 0; k < 6; ++k)
    {
        double const w_p = (k == 0), dx_p = (k == 1), dy_p = (k == 2);
        double const dxy_p = (k == 3), dxx_p = (k == 4), dyy_p = (k == 5);

        double const a_p = w_p + X * dx_p + Y * dy_p;
        double const ax_p = 2.0 * dx_p + X * dxx_p + Y * dxy_p;
        double const ay_p = 2.0 * dy_p + Y * dyy_p + X * dxy_p;
        double const t_p2 = DX * dx_p + DY * dy_p + f_sqr_inv * A * a_p;
        double const n_p = t_p2 * inv_n;
        double const b_p = (dx_p * DXX + DX * dxx_p)
            + (dy_p * DXY + DY * dxy_p) + f_sqr_inv * (a_p * AX + A * ax_p);
        double const c_p = (dx_p * DXY + DX * dxy_p)
            + (dy_p * DYY + DY * dyy_p) + f_sqr_inv * (a_p * AY + A * ay_p);
        double const nx_p = (b_p * n - b * n_p) * inv_t;
        double const ny_p = (c_p * n - c * n_p) * inv_t;

        double const xx_p = ((dxx_p * n + DXX * n_p - dx_p * nx - DX * nx_p)
            * t - (DXX * n - DX * nx) * t_p2 * 2.0) * inv_tt;
        double const yy_p = ((dyy_p * n + DYY * n_p - dy_p * ny - DY * ny_p)
            * t - (DYY * n - DY * ny) * t_p2 * 2.0) * inv_tt;
        double const xy_p = ((dxy_p * n + DXY * n_p - dx_p * ny - DX * ny_p)
            * t - (DXY * n - DX * ny) * t_p2 * 2.0) * inv_tt;
        double const yx_p = ((dxy_p * n + DXY * n_p - dy_p * nx - DY * nx_p)
            * t - (DXY * n - DY * nx) * t_p2 * 2.0) * inv_tt;
        double const zx_p = ((ax_p * n + AX * n_p - a_p * nx - A * nx_p)
            * t - (AX * n - A * nx) * t_p2 * 2.0) * inv_ttf;
        double const zy_p = ((ay_p * n + AY * n_p - a_p * ny - A * ny_p)
            * t - (AY * n - A * ny) * t_p2 * 2.0) * inv_ttf;

        g.C[0][k] = xx_p;
        g.C[1][k] = -yx_p;
        g.C[2][k] = zx_p;
        g.C[3][k] = xy_p;
        g.C[4][k] = -yy_p;
        g.C[5][k] = zy_p;

        if (k < 3)
        {
            g.N[0][k] = (dx_p * n - DX * n_p) * inv_t;
            g.N[1][k] = (-dy_p * n + DY * n_p) * inv_t;
            g.N[2][k] = (a_p * n - A * n_p) * inv_tf;
        }
    }
}

/* sh::evaluate_4_band, lib/spherical_harmonics.h:62-151 */
__device__ __forceinline__ void
sh_evaluate_4_band (double const* nrm, double* sh)
{
    double const x = nrm[0], y = nrm[1], z = nrm[2];
    double const x2 = x * x, y2 = y * y, z2 = z * z;
    sh[0] = 1.0;
    sh[1] = y;
    sh[2] = z;
    sh[3] = x;
    sh[4] = x * y;
    sh[5] = y * z;
    sh[6] = -x2 - y2 + 2.0 * z2;
    sh[7] = x * z;
    sh[8] = x * x - y * y;
    sh[9] = (3.0 * x2 - y2) * y;
    sh[10] = x * y * z;
    sh[11] = (4.0 * z2 - x2 - y2) * y;
    sh[12] = (2.0 * z2 - 3.0 * x2 - 3.0 * y2) * z;
    sh[13] = (4.0 * z2 - x2 - y2) * x;
    sh[14] = (x2 - y2) * z;
    sh[15] = (x2 - 3.0 * y2) * x;
}

/* G[c] = sum_{l=1..15} L[l] * d(sh_l)/d(n_c), the light-weighted rows of
 * sh::derivative_4_band (lib/spherical_harmonics.h:83-201); sh0 is constant
 * (lib/gauss_newton_step.cc:451). */
__device__ __forceinline__ void
sh_light_gradient (double const* nrm, double const* L, double* G)
{
    double const x = nrm[0], y = nrm[1], z = nrm[2];
    double const x2 = x * x, y2 = y * y, z2 = z * z;
    double d[16][3];
    d[0][0] = 0; d[0][1] = 0; d[0][2] = 0;
    d[1][0] = 0; d[1][1] = 1; d[1][2] = 0;
    d[2][0] = 0; d[2][1] = 0; d[2][2] = 1;
    d[3][0] = 1; d[3][1] = 0; d[3][2] = 0;
    d[4][0] = y; d[4][1] = x; d[4][2] = 0;
    d[5][0] = 0; d[5][1] = z; d[5][2] = y;
    d[6][0] = -2.0 * x; d[6][1] = -2.0 * y; d[6][2] = 4.0 * z;
    d[7][0] = z; d[7][1] = 0; d[7][2] = x;
    d[8][0] = 2.0 * x; d[8][1] = -2.0 * y; d[8][2] = 0;
    d[9][0] = 6.0 * x * y; d[9][1] = 3.0 * (x2 - y2); d[9][2] = 0;
    d[10][0] = y * z; d[10][1] = x * z; d[10][2] = x * y;
    d[11][0] = -2.0 * x * y; d[11][1] = 4.0 * z2 - x2 - 3.0 * y2;
    d[11][2] = 8.0 * y * z;
    d[12][0] = -6.0 * x * z; d[12][1] = -6.0 * y * z;
    d[12][2] = 6.0 * z2 - 3.0 * (x2 + y2);
    d[13][0] = 4.0 * z2 - 3.0 * x2 - y2; d[13][1] = -2.0 * x * y;
    d[13][2] = 8.0 * x * z;
    d[14][0] = 2.0 * x * z; d[14][1] = -2.0 * y * z; d[14][2] = x2 - y2;
    d[15][0] = 3.0 * (x2 - y2); d[15][1] = -6.0 * x * y; d[15][2] = 0;
    G[0] = G[1] = G[2] = 0.0;
#pragma unroll
    for (int l = 1; l < 16; ++l)
    {
        G[0] += L[l] * d[l][0];
        G[1] += L[l] * d[l][1];
        G[2] += L[l] * d[l][2];
    }
}

/* surfderiv::fill_normal, lib/surface_derivative.cc:17-28, rounded after
 * every operation like the CPU (no FMA contraction): the normal map is the
 * reference's bits, and a fused x * dx + y * dy or sum of squares moves it
 * by an ulp. math::Vector::norm sums the squares from 0 in order. */
__device__ __forceinline__ void
fill_normal (double x, double y, double inv_flen, double w, double dx,
    double dy, double* n)
{
    xd const n0(dx), n1(-dy);
    xd const n2 = (xd(x) * xd(dx) + xd(y) * xd(dy) + xd(w)) * xd(inv_flen);
    double const len = sqrt((n0 * n0 + n1 * n1 + n2 * n2).v);
    n[0] = n0.v / len;
    n[1] = n1.v / len;
    n[2] = n2.v / len;
}

/* 4x4 symmetric inverse by LDL^T exactly as ldl_inverse does it
 * (lib/ldl_decomposition.h:43-92): returns false (A untouched) on a zero
 * pivot; the caller applies the NaN rule of
 * lib/block_sparse_matrix.h:300-316. */
__device__ __forceinline__ bool
ldl_inverse4 (double const* A, double* out)
{
    double L[16], D[4];
#pragma unroll
    for (int i = 0; i < 16; ++i) L[i] = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j)
    {
        D[j] = A[j * 4 + j];
        L[j * 4 + j] = 1.0;
#pragma unroll
        for (int k = 0; k < j; ++k)
            D[j] -= (L[j * 4 + k] * L[j * 4 + k]) * D[k];
        if (D[j] == 0.0)
            return false;
#pragma unroll
        for (int i = j + 1; i < 4; ++i)
        {
            L[i * 4 + j] = A[i * 4 + j];
#pragma unroll
            for (int k = 0; k < j; ++k)
                L[i * 4 + j] -= L[i * 4 + k] * D[k] * L[j * 4 + k];
            L[i * 4 + j] /= D[j];
        }
    }
    /* invert L */
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = i + 1; j < 4; ++j)
        {
            double sum = 0.0;
#pragma unroll
            for (int k = i; k < j; ++k)
                sum -= L[j * 4 + k] * L[k * 4 + i];
            L[j * 4 + i] = sum;
        }
#pragma unroll
    for (int i = 0; i < 4; ++i)
        D[i] = 1.0 / D[i];
    /* combine_ldl: out = L^T D L */
#pragma unroll
    for (int i = 0; i < 16; ++i) out[i] = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c1 = 0; c1 < 4; ++c1)
#pragma unroll
            for (int c2 = 0; c2 < 4; ++c2)
                out[c1 * 4 + c2] += L[r * 4 + c2] * L[r * 4 + c1] * D[r];
    return true;
}

} /* namespace smvsb */

#endif

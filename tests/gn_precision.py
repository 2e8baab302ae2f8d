"""Extended-precision restatement of GaussNewtonStep::construct (gn_patch_kernel,
gn_assemble_kernel, gn_precond_kernel in smvs_b200/csrc/gn_construct.cu) and of
the node update (reproj_kernel / update_reduce_*, smvs_b200/csrc/update.cu),
used by tests/test_gn_system_precision.py.

Two stages, as the kernel splits them:

* The quantities the kernel evaluates bitwise like the reference (xd in
  gn_math.cuh) -- the patch coefficients, w ... wyy, neighbour_row's
  projections, Jacobian, A0..B1, cu, cv, the fp32 texture taps,
  surface_geometry's div / t / n / b / c / nx / ny and fill_normal -- are
  evaluated here in numpy float64 (float32 for the taps), one rounded
  operation at a time in the kernel's order. They feed fp32 narrowing, floor
  and clamping, so they must be the kernel's values, not exact ones.
* Everything after that is evaluated in np.longdouble, each value carrying a
  first-order bound on the kernel's rounding error (class T). Sums whose
  order an implementation may choose (the rows of a sample, the samples and
  patches of an entry) are bounded order-independently: a sum of N terms
  gets (N - 1) times the sum of the terms' magnitudes.

The bound and the derivation of K are in tests/test_gn_system_precision.py.
"""
from __future__ import annotations

import numpy as np

LD = np.longdouble
R_FACTOR = 1e-4                 # SMVSB_R_FACTOR, lib/gauss_newton_step.cc:17

# BicubicPatch's Hermite matrix (patch_eval.cuh: c_hermite), the table of
# small integers any bicubic Hermite patch implies
HERMITE = np.array([
    1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
    0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
    -3, 3, 0, 0, -2, -1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
    2, -2, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
    0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0,
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0,
    0, 0, 0, 0, 0, 0, 0, 0, -3, 3, 0, 0, -2, -1, 0, 0,
    0, 0, 0, 0, 0, 0, 0, 0, 2, -2, 0, 0, 1, 1, 0, 0,
    -3, 0, 3, 0, 0, 0, 0, 0, -2, 0, -1, 0, 0, 0, 0, 0,
    0, 0, 0, 0, -3, 0, 3, 0, 0, 0, 0, 0, -2, 0, -1, 0,
    9, -9, -9, 9, 6, 3, -6, -3, 6, -6, 3, -3, 4, 2, 2, 1,
    -6, 6, 6, -6, -3, -3, 3, 3, -4, 4, -2, 2, -2, -2, -1, -1,
    2, 0, -2, 0, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0,
    0, 0, 0, 0, 2, 0, -2, 0, 0, 0, 0, 0, 1, 0, 1, 0,
    -6, 6, 6, -6, -4, -2, 4, 2, -3, 3, -3, 3, -2, -1, -2, -1,
    4, -4, -4, 4, 2, 2, -2, -2, 2, -2, 2, -2, 1, 1, 1, 1], dtype=np.float64).reshape(16, 16)


def sampling_for_scale(scale):
    """lib/gauss_newton_step.cc:157-161"""
    return 1 if scale < 3 else (2 if scale < 5 else 4)


def basis_table(ps, step):
    """fill_basis_table: B[order][position][4], derivatives divided by ps."""
    npos = ps // step
    t = (np.arange(npos) * step + 0.5) / ps
    t2, t3 = t * t, t * t * t
    b0 = np.stack([2 * t3 - 3 * t2 + 1, -2 * t3 + 3 * t2, t3 - 2 * t2 + t, t3 - t2], 1)
    b1 = np.stack([6 * t2 - 6 * t, -6 * t2 + 6 * t, 3 * t2 - 4 * t + 1, 3 * t2 - 2 * t], 1)
    b2 = np.stack([12 * t - 6, -12 * t + 6, 6 * t - 4, 6 * t - 2], 1)
    return np.stack([b0, b1 / ps, b2 / (float(ps) * ps)])


# column c of a patch's 16 parameters: node li = c >> 2 (n00, n10, n01, n11),
# component c & 3 (f, dx, dy, dxy); its Hermite basis indices (side + 2 order)
_COL = np.arange(16)
BX = ((_COL >> 2) & 1) + 2 * (_COL & 1)
BY = ((_COL >> 3) & 1) + 2 * ((_COL >> 1) & 1)
# basis rows of q = (w, wx, wy, wxy, wxx, wyy): (order in x, order in y)
_ORDERS = ((0, 0), (1, 0), (0, 1), (1, 1), (2, 0), (0, 2))


def node_derivatives(ps, step):
    """D[s, k, col] = X_k[ix][bx] * Y_k[iy][by] (rounded once, as the kernel
    forms it), s = iy * npos + ix."""
    B = basis_table(ps, step)
    npos = B.shape[1]
    iy, ix = np.divmod(np.arange(npos * npos), npos)
    D = np.empty((npos * npos, 6, 16))
    for k, (ox, oy) in enumerate(_ORDERS):
        D[:, k, :] = B[ox][ix][:, BX] * B[oy][iy][:, BY]
    return D


# ---------------------------------------------------------------------------
# tracked longdouble values
# ---------------------------------------------------------------------------

class T:
    """A longdouble value and its first-order error bound in units of u:
    |fl(x) - x| <= u e for the kernel's value fl(x), whatever the kernel's
    order of operations within one product or quotient. Exact inputs (the
    bitwise stage's values, python floats) carry e = 0; every operation adds
    its own rounding |result|; errors propagate linearly:
        x + y: e_x + e_y + |x + y|       x y: |x| e_y + |y| e_x + |x y|
        x / y: (e_x + |q| e_y) / |y| + |q|"""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = np.asarray(v, dtype=LD)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, dtype=LD)

    @staticmethod
    def _t(x):
        return x if isinstance(x, T) else T(x)

    def __add__(self, o):
        o = T._t(o)
        s = self.v + o.v
        return T(s, self.e + o.e + np.abs(s))

    __radd__ = __add__

    def __sub__(self, o):
        o = T._t(o)
        s = self.v - o.v
        return T(s, self.e + o.e + np.abs(s))

    def __rsub__(self, o):
        return T._t(o) - self

    def __neg__(self):
        return T(-self.v, self.e)

    # samples that fail the shading test divide by a zero shading image; their
    # rows are masked out, their inf / NaN never reach a sum
    @np.errstate(divide="ignore", invalid="ignore", over="ignore")
    def __mul__(self, o):
        o = T._t(o)
        p = self.v * o.v
        return T(p, np.abs(self.v) * o.e + np.abs(o.v) * self.e + np.abs(p))

    __rmul__ = __mul__

    @np.errstate(divide="ignore", invalid="ignore", over="ignore")
    def __truediv__(self, o):
        o = T._t(o)
        q = self.v / o.v
        return T(q, (self.e + np.abs(q) * o.e) / np.abs(o.v) + np.abs(q))

    def __rtruediv__(self, o):
        return T._t(o) / self

    def __abs__(self):
        return T(np.abs(self.v), self.e)


def tsum(terms):
    out = terms[0]
    for t in terms[1:]:
        out = out + t
    return out


# ---------------------------------------------------------------------------
# the bitwise stage (float64 / float32, the kernel's order, no fusion)
# ---------------------------------------------------------------------------

def patch_coefficients(theta):
    """theta (P, 16) node-major -> coeffs (P, 16) at [i * 4 + j]."""
    x = theta[:, [(k & 3) * 4 + (k >> 2) for k in range(16)]]
    cf = np.empty_like(theta)
    for r in range(16):
        s = np.zeros(len(theta))
        for k in range(16):
            s = s + HERMITE[r, k] * x[:, k]
        cf[:, (r & 3) * 4 + (r >> 2)] = s
    return cf


def sample_values(cf, ix, iy, ps, sampling):
    """w, wx, wy, wxy, wxx, wyy of every (patch, sample): cf (P, 16), ix / iy
    (S,) -> arrays (P, S)."""
    inv = 1.0 / float(ps)
    sx = (ix * sampling + 0.5) * inv
    sy = (iy * sampling + 0.5) * inv
    ex = [np.ones_like(sx), sx, sx * sx, (sx * sx) * sx]
    ey = [np.ones_like(sy), sy, sy * sy, (sy * sy) * sy]
    c = [cf[:, i][:, None] for i in range(16)]
    z = np.zeros((cf.shape[0], len(ix)))
    f, fx, fy, fxy, fxx, fyy = z.copy(), z.copy(), z.copy(), z.copy(), z.copy(), z.copy()
    for i in range(4):
        for j in range(4):
            f = f + (c[i * 4 + j] * ex[i]) * ey[j]
    for i in range(1, 4):
        for j in range(4):
            fx = fx + ((c[i * 4 + j] * float(i)) * ex[i - 1]) * ey[j]
    for i in range(2, 4):
        for j in range(4):
            fxx = fxx + (((c[i * 4 + j] * float(i)) * float(i - 1)) * ex[i - 2]) * ey[j]
    for i in range(4):
        for j in range(1, 4):
            fy = fy + ((c[i * 4 + j] * ex[i]) * float(j)) * ey[j - 1]
    for i in range(4):
        for j in range(2, 4):
            fyy = fyy + (((c[i * 4 + j] * ex[i]) * float(j)) * float(j - 1)) * ey[j - 2]
    for i in range(1, 4):
        for j in range(1, 4):
            fxy = fxy + ((((c[i * 4 + j] * float(i)) * ex[i - 1]) * float(j)) * ey[j - 1])
    inv2 = 1.0 / float(ps * ps)
    return f, fx * inv, fy * inv, fxy * inv2, fxx * inv2, fyy * inv2


def tap(grad, hess, px, py):
    """tap_neighbour: fp32 bilinear taps of (gx, gy, hxx, hxy, hyy)."""
    h, w = grad.shape[:2]
    x = np.maximum(np.float32(0), np.minimum(np.float32(w - 1), px.astype(np.float32)))
    y = np.maximum(np.float32(0), np.minimum(np.float32(h - 1), py.astype(np.float32)))
    fx, fy = x.astype(np.int64), y.astype(np.int64)
    fx1, fy1 = np.minimum(fx + 1, w - 1), np.minimum(fy + 1, h - 1)
    w1 = x - fx.astype(np.float32)
    w0 = np.float32(1) - w1
    w3 = y - fy.astype(np.float32)
    w2 = np.float32(1) - w3
    w00, w10, w01, w11 = w0 * w2, w1 * w2, w0 * w3, w1 * w3
    tex = np.concatenate([grad, hess], axis=2)
    a, b, c, d = tex[fy, fx], tex[fy, fx1], tex[fy1, fx], tex[fy1, fx1]
    return ((a * w00[..., None] + b * w10[..., None]) + c * w01[..., None]) + d * w11[..., None]


def neighbour_row(M, t, u, v, w, wx, wy, grad, hess):
    """The bitwise part of neighbour_row for one neighbour, arrays (M,)."""
    m0, m1, m2, m3, m4, m5, m6, m7, m8 = [float(x) for x in M]
    T0, T1, T2 = [float(x) for x in t]
    p = (m0 * u + m1 * v) + m2
    q = (m3 * u + m4 * v) + m5
    r = (m6 * u + m7 * v) + m8
    a = w * p + T0
    b = w * q + T1
    d = w * r + T2
    d2 = d * d
    projx = a / d - 0.5
    projy = b / d - 0.5
    j0 = (wx * p + w * m0) / d
    j2 = (wy * p + w * m1) / d
    j0 = j0 - (a * (wx * r + w * m6)) / d2
    j2 = j2 - (a * (wy * r + w * m7)) / d2
    j1 = (wx * q + w * m3) / d
    j3 = (wy * q + w * m4) / d
    j1 = j1 - (b * (wx * r + w * m6)) / d2
    j3 = j3 - (b * (wy * r + w * m7)) / d2
    tp = tap(grad, hess, projx, projy).astype(np.float64)
    GX, GY, H0, H1, H3 = (tp[..., i] for i in range(5))
    out = dict(jgx=j0 * GX + j1 * GY, jgy=j2 * GX + j3 * GY, gx=GX, gy=GY,
               jh00=j0 * H0 + j1 * H1, jh01=j0 * H1 + j1 * H3,
               jh10=j2 * H0 + j3 * H1, jh11=j2 * H1 + j3 * H3,
               du_w=(p * d - r * a) / d2, dv_w=(q * d - r * b) / d2,
               projx=projx, projy=projy)
    d4 = d2 * d2
    d_prime = (2.0 * d) * r
    du_c = p * T2 - r * T0
    dv_c = q * T2 - r * T1
    du_a_t0, du_a_t1 = w * (m0 * r - p * m6), w * (m1 * r - p * m7)
    du_b0, du_b1 = m0 * T2 - m6 * T0, m1 * T2 - m7 * T0
    dv_a_t0, dv_a_t1 = w * (m3 * r - q * m6), w * (m4 * r - q * m7)
    dv_b0, dv_b1 = m3 * T2 - m6 * T1, m4 * T2 - m7 * T1
    out["A0"] = (2.0 * du_a_t0 + du_b0) / d2 - ((w * (du_a_t0 + du_b0) + wx * du_c) * d_prime) / d4
    out["A1"] = (2.0 * du_a_t1 + du_b1) / d2 - ((w * (du_a_t1 + du_b1) + wy * du_c) * d_prime) / d4
    out["B0"] = (2.0 * dv_a_t0 + dv_b0) / d2 - ((w * (dv_a_t0 + dv_b0) + wx * dv_c) * d_prime) / d4
    out["B1"] = (2.0 * dv_a_t1 + dv_b1) / d2 - ((w * (dv_a_t1 + dv_b1) + wy * dv_c) * d_prime) / d4
    out["cu"] = du_c / d2
    out["cv"] = dv_c / d2
    return out


def surface_bitwise(x, y, f, w, dx, dy, dxy, dxx, dyy):
    """surface_geometry's exact part: div[6] and the shared quantities."""
    a = (w + x * dx) + y * dy
    ax = (2.0 * dx + x * dxx) + y * dxy
    ay = (2.0 * dy + y * dyy) + x * dxy
    t = a / f
    t = t * t
    t = t + (dx * dx + dy * dy)
    n = np.sqrt(t)
    finv = 1.0 / (f * f)
    nx = dx * dxx + dy * dxy
    nx = nx + (finv * ((w + x * dx) + y * dy)) * (((dx + dx) + x * dxx) + y * dxy)
    nx = nx / n
    ny = dx * dxy + dy * dyy
    ny = ny + (finv * ((w + x * dx) + y * dy)) * (((dy + dy) + x * dxy) + y * dyy)
    ny = ny / n
    div = [(dxx * n - dx * nx) / t, -((dxy * n - dy * nx) / t), (ax * n - a * nx) / (t * f),
           (dxy * n - dx * ny) / t, -((dyy * n - dy * ny) / t), (ay * n - a * ny) / (t * f)]
    a_f2 = a * finv
    t2 = (dx * dx + dy * dy) + a * a_f2
    n2 = np.sqrt(t2)
    b2 = (dx * dxx + dy * dxy) + a_f2 * ((2.0 * dx + x * dxx) + y * dxy)
    c2 = (dx * dxy + dy * dyy) + a_f2 * ((2.0 * dy + x * dxy) + y * dyy)
    return dict(div=div, finv=finv, t=t2, n=n2, b=b2, c=c2, nx=b2 / n2, ny=c2 / n2,
                A=a, AX=ax, AY=ay)


def fill_normal(x, y, inv_flen, w, dx, dy):
    n0, n1 = dx, -dy
    n2 = ((x * dx + y * dy) + w) * inv_flen
    ln = np.sqrt((n0 * n0 + n1 * n1) + n2 * n2)
    return n0 / ln, n1 / ln, n2 / ln


# ---------------------------------------------------------------------------
# the longdouble stage
# ---------------------------------------------------------------------------

def geometry_coefficients(x, y, f, dx, dy, dxy, dxx, dyy, sg):
    """C[v][k] = d div[v] / d q_k and N[c][k] (k < 3), tracked, the kernel's
    formulas (surface_geometry's second half)."""
    X, Y, F = T(x), T(y), T(f)
    DX, DY, DXY, DXX, DYY = T(dx), T(dy), T(dxy), T(dxx), T(dyy)
    fsi, t, n, b, c = T(sg["finv"]), T(sg["t"]), T(sg["n"]), T(sg["b"]), T(sg["c"])
    nx, ny, A, AX, AY = T(sg["nx"]), T(sg["ny"]), T(sg["A"]), T(sg["AX"]), T(sg["AY"])
    inv_t = 1.0 / t
    inv_n = 1.0 / n
    inv_tt = inv_t * inv_t
    inv_ttf = inv_tt / F
    inv_tf = inv_t / F
    C = [[None] * 6 for _ in range(6)]
    N = [[None] * 3 for _ in range(3)]
    for k in range(6):
        w_p, dx_p, dy_p, dxy_p, dxx_p, dyy_p = (float(k == i) for i in range(6))
        a_p = (w_p + X * dx_p) + Y * dy_p
        ax_p = (2.0 * dx_p + X * dxx_p) + Y * dxy_p
        ay_p = (2.0 * dy_p + Y * dyy_p) + X * dxy_p
        t_p2 = (DX * dx_p + DY * dy_p) + (fsi * A) * a_p
        n_p = t_p2 * inv_n
        b_p = ((dx_p * DXX + DX * dxx_p) + (dy_p * DXY + DY * dxy_p)
               + fsi * (a_p * AX + A * ax_p))
        c_p = ((dx_p * DXY + DX * dxy_p) + (dy_p * DYY + DY * dyy_p)
               + fsi * (a_p * AY + A * ay_p))
        nx_p = (b_p * n - b * n_p) * inv_t
        ny_p = (c_p * n - c * n_p) * inv_t

        def dd(e_p, E, g_p, G, h, h_p, scale):
            return ((((e_p * n + E * n_p) - g_p * h) - G * h_p) * t
                    - ((E * n - G * h) * t_p2) * 2.0) * scale
        xx_p = dd(dxx_p, DXX, dx_p, DX, nx, nx_p, inv_tt)
        yy_p = dd(dyy_p, DYY, dy_p, DY, ny, ny_p, inv_tt)
        xy_p = dd(dxy_p, DXY, dx_p, DX, ny, ny_p, inv_tt)
        yx_p = dd(dxy_p, DXY, dy_p, DY, nx, nx_p, inv_tt)
        zx_p = dd(ax_p, AX, a_p, A, nx, nx_p, inv_ttf)
        zy_p = dd(ay_p, AY, a_p, A, ny, ny_p, inv_ttf)
        C[0][k], C[1][k], C[2][k] = xx_p, -yx_p, zx_p
        C[3][k], C[4][k], C[5][k] = xy_p, -yy_p, zy_p
        if k < 3:
            N[0][k] = (dx_p * n - DX * n_p) * inv_t
            N[1][k] = (-dy_p * n + DY * n_p) * inv_t
            N[2][k] = (a_p * n - A * n_p) * inv_tf
    return C, N


def sh_4band(x, y, z):
    x2, y2, z2 = x * x, y * y, z * z
    return [T(np.ones_like(x.v)), y, z, x, x * y, y * z, (-x2 - y2) + 2.0 * z2, x * z,
            x * x - y * y, (3.0 * x2 - y2) * y, (x * y) * z, ((4.0 * z2 - x2) - y2) * y,
            ((2.0 * z2 - 3.0 * x2) - 3.0 * y2) * z, ((4.0 * z2 - x2) - y2) * x,
            (x2 - y2) * z, (x2 - 3.0 * y2) * x]


def sh_light_gradient(x, y, z, L):
    x2, y2, z2 = x * x, y * y, z * z
    zero = T(np.zeros_like(x.v))
    one = T(np.ones_like(x.v))
    d = [(zero, zero, zero), (zero, one, zero), (zero, zero, one), (one, zero, zero),
         (y, x, zero), (zero, z, y), (-2.0 * x, -2.0 * y, 4.0 * z), (z, zero, x),
         (2.0 * x, -2.0 * y, zero), ((6.0 * x) * y, 3.0 * (x2 - y2), zero),
         (y * z, x * z, x * y), ((-2.0 * x) * y, (4.0 * z2 - x2) - 3.0 * y2, (8.0 * y) * z),
         ((-6.0 * x) * z, (-6.0 * y) * z, 6.0 * z2 - 3.0 * (x2 + y2)),
         ((4.0 * z2 - 3.0 * x2) - y2, (-2.0 * x) * y, (8.0 * x) * z),
         ((2.0 * x) * z, (-2.0 * y) * z, x2 - y2), (3.0 * (x2 - y2), (-6.0 * x) * y, zero)]
    return [tsum([float(L[l]) * d[l][c] for l in range(1, 16)]) for c in range(3)]


class Acc:
    """Per-sample 6x6 normal matrix (upper triangle) and right-hand side:
    for every entry the value, the sum of its terms' error bounds and the
    sum of its terms' magnitudes."""

    def __init__(self, m):
        self.A = {(k, l): [np.zeros(m, LD) for _ in range(3)]
                  for k in range(6) for l in range(k, 6)}
        self.b = [[np.zeros(m, LD) for _ in range(3)] for _ in range(6)]
        self.rows = np.zeros(m, dtype=np.int64)

    def photo(self, K, c0, ck, rho, wgt, mask):
        w0, wk = c0 * wgt, ck * wgt
        _add(self.A[(0, 0)], w0 * c0, mask)
        _add(self.A[(0, K)], w0 * ck, mask)
        _add(self.A[(K, K)], wk * ck, mask)
        _add(self.b[0], w0 * rho, mask)
        _add(self.b[K], wk * rho, mask)
        self.rows += mask

    def full(self, c, rho, wgt, mask):
        for k in range(6):
            wk = c[k] * wgt
            _add(self.b[k], wk * rho, mask)
            for l in range(k, 6):
                _add(self.A[(k, l)], wk * c[l], mask)
        self.rows += mask


def _add(acc, t, mask):
    acc[0] += np.where(mask, t.v, 0)
    acc[1] += np.where(mask, t.e, 0)
    acc[2] += np.where(mask, np.abs(t.v), 0)


# ---------------------------------------------------------------------------
# K1 + K2a: the system
# ---------------------------------------------------------------------------

class Inputs:
    """What the context was given (set_views + set_surface)."""

    def __init__(self, main_grad, sub_grads, sub_hess, Mi, ti, flen, inv_flen, shading,
                 shading_grad, scale, npx, npy, start_x, start_y, nodes, node_valid,
                 patch_valid, vis_off, vis_ids):
        self.main_grad = np.asarray(main_grad, np.float32)
        self.sub_grads = [np.asarray(g, np.float32) for g in sub_grads]
        self.sub_hess = [np.asarray(h, np.float32) for h in sub_hess]
        self.Mi, self.ti = np.asarray(Mi, np.float64), np.asarray(ti, np.float64)
        self.flen, self.inv_flen = float(flen), float(inv_flen)
        self.shading = None if shading is None else np.asarray(shading, np.float32)
        self.shading_grad = None if shading_grad is None else np.asarray(shading_grad, np.float32)
        self.scale, self.npx, self.npy = int(scale), int(npx), int(npy)
        self.start_x, self.start_y = int(start_x), int(start_y)
        self.nodes = np.asarray(nodes, np.float64).reshape(-1, 4)
        self.node_valid = np.asarray(node_valid, np.uint8)
        self.patch_valid = np.asarray(patch_valid, np.uint8)
        self.vis_off = np.asarray(vis_off, np.int64)
        self.vis_ids = np.asarray(vis_ids, np.int64)
        self.ps = 1 << self.scale
        self.sampling = sampling_for_scale(self.scale)
        self.npos = self.ps // self.sampling
        self.h, self.w = self.main_grad.shape[:2]

    @classmethod
    def from_golden(cls, G):
        n = int(G["n_sub"])
        return cls(G["main_grad"], [G[f"sub_grad{k}"] for k in range(n)],
                   [G[f"sub_hess{k}"] for k in range(n)], G["Mi"], G["ti"], float(G["flen"]),
                   float(G["inv_flen"]), G["shading"] if "shading" in G else None,
                   G["shading_grad"] if "shading_grad" in G else None, int(G["scale"]),
                   int(G["npx"]), int(G["npy"]), int(G["start_x"]), int(G["start_y"]),
                   G["nodes"], G["node_valid"], G["patch_valid"], G["vis_off"], G["vis_ids"])

    @classmethod
    def from_pair(cls, P):
        R, n = P.R, P.scene.n_sub
        sh, shg = R.shading() if P.scene.shading else (None, None)
        i = P.info
        return cls(R.gradients(0), [R.gradients(k + 1) for k in range(n)],
                   [R.hessian(k + 1) for k in range(n)], P.Mi, P.ti, R.flen(0),
                   R.inverse_flen(0), sh, shg, i["scale"], i["npx"], i["npy"], i["start_x"],
                   i["start_y"], P.nodes, P.node_valid, P.patch_valid, P.vis_off, P.vis_ids)

    def patch_nodes(self):
        """(n_patches, 4) node ids n00, n10, n01, n11."""
        p = np.arange(self.npx * self.npy)
        idy, idx = np.divmod(p, self.npx)
        n0 = idy * (self.npx + 1) + idx
        return np.stack([n0, n0 + 1, n0 + self.npx + 1, n0 + self.npx + 2], 1)

    def processed(self, active):
        act = np.asarray(active).astype(bool)
        return self.patch_valid.astype(bool) & act[self.patch_nodes()].any(1)


class Patches:
    """Per-patch 16x16 H and 16-vector g (tracked) of the processed patches,
    plus what the tests need to know about them."""


def construct_patches(I, active, light=None, reg=0.01, lreg=0.0, patches=None,
                      drop_geometry=None, drop_sample=None, drop_pair=None):
    """K1 for the processed patches (or the given subset). Returns a dict with
    `ids` (patch ids), `H` / `He` (P, 16, 16), `g` / `ge` (P, 16), `rows`
    (residual rows per sample, the largest), `shade` (shading-branch counts)
    and `margin` (smallest relative distance of a shading test from its
    threshold), `clamped` / `taps` (neighbour taps whose projection lies
    outside the neighbour and was clamped, and all taps). drop_geometry /
    drop_sample = (patch index, sample) and drop_pair = (patch index, sample,
    j, j2): mutations for the sensitivity tests (that sample's geometry rows,
    all its rows, or the two rows of its neighbour pair (j, j2))."""
    proc = I.processed(active)
    ids = np.flatnonzero(proc) if patches is None else np.asarray(patches)
    S = I.npos * I.npos
    iy, ix = np.divmod(np.arange(S), I.npos)
    P = len(ids)
    out = dict(ids=ids, S=S, rows=0, shade=[0, 0], margin=np.inf, clamped=0, taps=0)
    if P == 0:
        out.update(H=np.zeros((0, 16, 16), LD), He=np.zeros((0, 16, 16), LD),
                   g=np.zeros((0, 16), LD), ge=np.zeros((0, 16), LD))
        return out
    theta = I.nodes[I.patch_nodes()[ids]].reshape(P, 16)
    cf = patch_coefficients(theta)
    w, wx, wy, wxy, wxx, wyy = (a.reshape(-1) for a in sample_values(cf, ix, iy, I.ps, I.sampling))
    idy, idx = np.divmod(ids, I.npx)
    px = (I.start_x + idx[:, None] * I.ps + ix[None, :] * I.sampling).reshape(-1)
    py = (I.start_y + idy[:, None] * I.ps + iy[None, :] * I.sampling).reshape(-1)
    M = P * S
    gm = I.main_grad[py, px].astype(np.float64)
    gmx, gmy = gm[:, 0], gm[:, 1]

    # neighbour lists, padded: slot j of sample m is neighbour lists[patch][j]
    counts = (I.vis_off[ids + 1] - I.vis_off[ids])
    nmax = int(counts.max()) if P else 0
    n_m = np.repeat(counts, S)
    rows = []
    u, v = px + 0.5, py + 0.5
    for j in range(nmax):
        has = n_m > j
        sub = np.zeros(M, dtype=np.int64)
        pid = np.repeat(np.arange(P), S)
        sel = counts[pid] > j
        sub[sel] = I.vis_ids[I.vis_off[ids[pid[sel]]] + j]
        r = {k: np.zeros(M) for k in ("jgx", "jgy", "ax", "ay", "be")}
        rt = {}
        for s in np.unique(sub[has]):
            m = has & (sub == s)
            nb = neighbour_row(I.Mi[s], I.ti[s], u[m], v[m], w[m], wx[m], wy[m],
                               I.sub_grads[s], I.sub_hess[s])
            for k in ("jgx", "jgy"):
                r[k][m] = nb[k]
            sh_, sw_ = I.sub_grads[s].shape[:2]
            out["clamped"] += int(((nb["projx"] < 0) | (nb["projx"] > sw_ - 1)
                                   | (nb["projy"] < 0) | (nb["projy"] > sh_ - 1)).sum())
            out["taps"] += int(m.sum())
            for k in ("A0", "A1", "B0", "B1", "cu", "cv", "gx", "gy", "jh00", "jh01",
                      "jh10", "jh11", "du_w", "dv_w"):
                rt.setdefault(k, np.zeros(M))[m] = nb[k]
        g_ = {k: T(rt.get(k, np.zeros(M))) for k in rt}
        if not rt:
            z = T(np.zeros(M))
            ax = ay = be = z
        else:
            ax = tsum([g_["A0"] * g_["gx"], g_["B0"] * g_["gy"], g_["jh00"] * g_["du_w"],
                       g_["jh01"] * g_["dv_w"]])
            ay = tsum([g_["A1"] * g_["gx"], g_["B1"] * g_["gy"], g_["jh10"] * g_["du_w"],
                       g_["jh11"] * g_["dv_w"]])
            be = g_["cu"] * g_["gx"] + g_["cv"] * g_["gy"]
        rows.append(dict(jgx=T(r["jgx"]), jgy=T(r["jgy"]), ax=ax, ay=ay, be=be, has=has))

    acc = Acc(M)
    GMX, GMY = T(gmx), T(gmy)
    for j in range(nmax):
        rj = rows[j]
        dx_, dy_ = rj["jgx"] - GMX, rj["jgy"] - GMY
        acc.photo(1, rj["ax"], rj["be"], dx_, 1.0 / (abs(dx_) + R_FACTOR), rj["has"])
        acc.photo(2, rj["ay"], rj["be"], dy_, 1.0 / (abs(dy_) + R_FACTOR), rj["has"])
        for j2 in range(j + 1, nmax):
            r2 = rows[j2]
            both = rj["has"] & r2["has"]
            if drop_pair is not None and drop_pair[2:] == (j, j2):
                both = both.copy()
                both[drop_pair[0] * S + drop_pair[1]] = False
            sx_, sy_ = rj["jgx"] - r2["jgx"], rj["jgy"] - r2["jgy"]
            be = rj["be"] - r2["be"]
            acc.photo(1, rj["ax"] - r2["ax"], be, sx_, 1.0 / (abs(sx_) + R_FACTOR), both)
            acc.photo(2, rj["ay"] - r2["ay"], be, sy_, 1.0 / (abs(sy_) + R_FACTOR), both)

    lit = light is not None
    if reg > 0.0:
        num_diffs = ((n_m * (n_m + 1)) // 2).astype(np.float64)
        basic = (T(reg * 0.005) / T(np.maximum(0.03, np.abs(gmx) + np.abs(gmy)))) * T(num_diffs)
        x = px + 0.5 - I.w / 2.0
        y = py + 0.5 - I.h / 2.0
        sg = surface_bitwise(x, y, I.flen, w, wx, wy, wxy, wxx, wyy)
        C, N = geometry_coefficients(x, y, I.flen, wx, wy, wxy, wxx, wyy, sg)
        div = [T(d) for d in sg["div"]]
        allm = np.ones(M, dtype=bool)
        if not lit or lreg > 0.0:
            gw = 1.0 if not lit else lreg / 100
            gmask = allm.copy()
            if drop_geometry is not None:
                gmask[drop_geometry[0] * S + drop_geometry[1]] = False
            for vv in range(6):
                wgt = (T(gw) / (abs(div[vv]) + R_FACTOR)) * basic
                acc.full(C[vv], div[vv], wgt, gmask)
        if lit:
            nrm = fill_normal(x, y, I.inv_flen, w, wx, wy)
            nx, ny, nz = (T(c) for c in nrm)
            sh = sh_4band(nx, ny, nz)
            shading = tsum([float(light[l]) * sh[l] for l in range(16)])
            # the branch from float64 values, the kernel's order
            x64, y64, z64 = nrm
            sh64 = _sh64(x64, y64, z64)
            s64 = np.zeros(M)
            for l in range(16):
                s64 = s64 + float(light[l]) * sh64[l]
            lg = I.shading_grad[py, px].astype(np.float64)
            liv = I.shading[py, px].astype(np.float64)
            gn = np.sqrt(lg[:, 0] * lg[:, 0] + lg[:, 1] * lg[:, 1])
            ok = ~(gn < 1e-10) & ~((s64 * s64 < 1e-10) | (liv * liv < 1e-10))
            for val, thr in ((gn, 1e-10), (s64 * s64, 1e-10), (liv * liv, 1e-10)):
                out["margin"] = min(out["margin"], float(np.min(np.abs(val - thr) / thr)))
            out["shade"] = [int(ok.sum()), int((~ok).sum())]
            sw = (0.001 * T(num_diffs)) / ((R_FACTOR + abs(T(lg[:, 0]))) + abs(T(lg[:, 1])))
            G = sh_light_gradient(nx, ny, nz, light)
            sgx = tsum([G[0] * div[0], G[1] * div[1], G[2] * div[2]])
            sgy = tsum([G[0] * div[3], G[1] * div[4], G[2] * div[5]])
            inv_s = 1.0 / shading
            ligx = T(lg[:, 0]) * (1.0 / T(liv))
            ligy = T(lg[:, 1]) * (1.0 / T(liv))
            ex = sgx * inv_s - ligx
            ey = sgy * inv_s - ligy
            inv_s2 = 1.0 / (shading * shading)
            cx, cy = [], []
            for k in range(6):
                sd = tsum([G[c] * N[c][k] for c in range(3)]) if k < 3 else T(np.zeros(M))
                gdx = tsum([G[c] * C[c][k] for c in range(3)])
                gdy = tsum([G[c] * C[3 + c][k] for c in range(3)])
                cx.append((gdx * shading - sgx * sd) * inv_s2)
                cy.append((gdy * shading - sgy * sd) * inv_s2)
            acc.full(cx, ex, sw / (abs(ex) + R_FACTOR), ok)
            acc.full(cy, ey, sw / (abs(ey) + R_FACTOR), ok)
    out["rows"] = int(acc.rows.max())

    # D^T A D and D^T b per patch
    D = node_derivatives(I.ps, I.sampling)
    # every entry of H is a sum over <= 4 patches x S samples of (rows of the
    # sample + the 36 terms of D^T A D); of g, rows + 6: the longest chain of
    # additions any order of these sums can make
    out["NH"] = 4 * S * (out["rows"] + 36) + 16
    out["Ng"] = 4 * S * (out["rows"] + 6) + 16
    Av, Ab = np.zeros((M, 6, 6), LD), np.zeros((M, 6, 6), LD)
    for (k, l), (v, e, m) in acc.A.items():
        Av[:, k, l] = Av[:, l, k] = v
        Ab[:, k, l] = Ab[:, l, k] = e + out["NH"] * m
    bv = np.stack([t[0] for t in acc.b], 1)
    bb = np.stack([t[1] + out["Ng"] * t[2] for t in acc.b], 1)
    if drop_sample is not None:
        Av[drop_sample[0] * S + drop_sample[1]] = 0
        bv[drop_sample[0] * S + drop_sample[1]] = 0
    DL, DA = D.astype(LD), np.abs(D).astype(LD)
    out["H"] = _dtad(DL, Av.reshape(P, S, 6, 6))
    out["He"] = _dtad(DA, Ab.reshape(P, S, 6, 6))
    out["g"] = np.einsum("sko,psk->po", DL, bv.reshape(P, S, 6))
    out["ge"] = np.einsum("sko,psk->po", DA, bb.reshape(P, S, 6))
    return out


def _dtad(D, A):
    """sum_s D_s^T A_s D_s, (P, S, 6, 6) -> (P, 16, 16), in chunks of patches."""
    P = A.shape[0]
    out = np.empty((P, 16, 16), LD)
    for p0 in range(0, P, 64):
        E = np.einsum("pskl,slq->pskq", A[p0:p0 + 64], D)
        out[p0:p0 + 64] = np.einsum("sko,pskq->poq", D, E)
    return out


def _sh64(x, y, z):
    x2, y2, z2 = x * x, y * y, z * z
    return [np.ones_like(x), y, z, x, x * y, y * z, -x2 - y2 + 2.0 * z2, x * z, x * x - y * y,
            (3.0 * x2 - y2) * y, x * y * z, (4.0 * z2 - x2 - y2) * y,
            (2.0 * z2 - 3.0 * x2 - 3.0 * y2) * z, (4.0 * z2 - x2 - y2) * x, (x2 - y2) * z,
            (x2 - 3.0 * y2) * x]


def assemble(I, active, pat):
    """K2a: the 3x3 stencil blocks [node, k = (dy+1)*3 + dx+1, 4, 4] (block
    row = node, column = its neighbour) and g [node, 4], value and companion,
    plus the number of patches summed into each node's diagonal block."""
    npx, npy = I.npx, I.npy
    ns = npx + 1
    nn = ns * (npy + 1)
    on = (I.node_valid.astype(bool) & np.asarray(active).astype(bool))
    Hd = np.zeros((npy + 2, npx + 2, 16, 16), LD)
    Hde = np.zeros_like(Hd)
    gd = np.zeros((npy + 2, npx + 2, 16), LD)
    gde = np.zeros_like(gd)
    pid_y, pid_x = np.divmod(pat["ids"], npx)
    Hd[pid_y + 1, pid_x + 1], Hde[pid_y + 1, pid_x + 1] = pat["H"], pat["He"]
    gd[pid_y + 1, pid_x + 1], gde[pid_y + 1, pid_x + 1] = pat["g"], pat["ge"]
    has = np.zeros((npy + 2, npx + 2), bool)
    has[pid_y + 1, pid_x + 1] = True
    iy, ix = np.divmod(np.arange(nn), ns)
    H = np.zeros((nn, 9, 4, 4), LD)
    He = np.zeros_like(H)
    g = np.zeros((nn, 4), LD)
    ge = np.zeros_like(g)
    npatch = np.zeros(nn, np.int64)
    onp = np.pad(on.reshape(npy + 1, ns), 1)
    for pb in (0, 1):
        for pa in (0, 1):
            py, px = iy - 1 + pb + 1, ix - 1 + pa + 1          # padded patch coords
            li = (1 - pa) + 2 * (1 - pb)
            use = on & has[py, px]
            npatch += use
            g[use] += gd[py, px][use][:, li * 4:li * 4 + 4]
            ge[use] += gde[py, px][use][:, li * 4:li * 4 + 4]
            for k in range(9):
                dx, dy = k % 3 - 1, k // 3 - 1
                ljx, ljy = dx + 1 - pa, dy + 1 - pb
                if not (0 <= ljx <= 1 and 0 <= ljy <= 1):
                    continue
                lj = ljx + 2 * ljy
                col_on = onp[iy + dy + 1, ix + dx + 1]
                m = use & col_on
                H[m, k] += Hd[py, px][m][:, li * 4:li * 4 + 4, lj * 4:lj * 4 + 4]
                He[m, k] += Hde[py, px][m][:, li * 4:li * 4 + 4, lj * 4:lj * 4 + 4]
    return dict(H=H, He=He, g=g, ge=ge, npatch=npatch, on=on)


def system_blocks(I, sysd):
    """(row, col, stencil slot) of every BSC block of sysd."""
    outer = sysd["Houter"].astype(np.int64)
    col = np.repeat(np.arange(len(outer) - 1), np.diff(outer))
    row = sysd["Hinner"].astype(np.int64) // 4
    ns = I.npx + 1
    dx = col % ns - row % ns
    dy = col // ns - row // ns
    assert (np.abs(dx) <= 1).all() and (np.abs(dy) <= 1).all()
    return row, col, (dy + 1) * 3 + (dx + 1)


def expected_blocks(I, active, proc):
    """Number of blocks (row i, col j) the reference stores: both valid and
    active, and some processed patch holds both."""
    on = I.node_valid.astype(bool) & np.asarray(active).astype(bool)
    pn = I.patch_nodes()[proc]
    pairs = set()
    for q in pn:
        qq = [n for n in q if on[n]]
        for a in qq:
            for b in qq:
                pairs.add((a, b))
    return pairs


def inverse4(B):
    """Inverse of (n, 4, 4) longdouble blocks by the adjugate (no LDL^T)."""
    B = np.asarray(B, LD)
    n = B.shape[0]
    cof = np.empty_like(B)
    idx = np.arange(4)
    for i in range(4):
        for j in range(4):
            r = idx[idx != i]
            c = idx[idx != j]
            m = B[:, r][:, :, c]
            det3 = (m[:, 0, 0] * (m[:, 1, 1] * m[:, 2, 2] - m[:, 1, 2] * m[:, 2, 1])
                    - m[:, 0, 1] * (m[:, 1, 0] * m[:, 2, 2] - m[:, 1, 2] * m[:, 2, 0])
                    + m[:, 0, 2] * (m[:, 1, 0] * m[:, 2, 1] - m[:, 1, 1] * m[:, 2, 0]))
            cof[:, i, j] = (-1) ** (i + j) * det3
    det = np.einsum("nj,nj->n", B[:, 0, :], cof[:, 0, :])
    with np.errstate(divide="ignore", invalid="ignore"):
        return cof.transpose(0, 2, 1) / det[:, None, None], det


def ldl_branch(B):
    """ldl_inverse4's branch in float64: True where it inverts (no zero pivot
    and no NaN), False where the block is kept."""
    out = np.empty(len(B), bool)
    for n, A in enumerate(np.asarray(B, np.float64)):
        L = np.zeros((4, 4))
        Dg = np.zeros(4)
        ok = True
        for j in range(4):
            Dg[j] = A[j, j]
            L[j, j] = 1.0
            for k in range(j):
                Dg[j] -= (L[j, k] * L[j, k]) * Dg[k]
            if Dg[j] == 0.0:
                ok = False
                break
            for i in range(j + 1, 4):
                L[i, j] = A[i, j]
                for k in range(j):
                    L[i, j] -= L[i, k] * Dg[k] * L[j, k]
                L[i, j] /= Dg[j]
        if ok:
            with np.errstate(all="ignore"):
                for i in range(4):
                    for jj in range(i + 1, 4):
                        L[jj, i] = -sum(L[jj, k] * L[k, i] for k in range(i, jj))
                inv = np.einsum("rb,ra,r->ab", L, L, 1.0 / Dg)
            ok = not np.isnan(inv).any()
        out[n] = ok
    return out


# ---------------------------------------------------------------------------
# K4: the node update
# ---------------------------------------------------------------------------

def update(I, active, delta, thresh=0.15, patches=None):
    """fill_node_reprojections before / after update_nodes, per processed
    patch: the largest difference (value, and its companion), the sum and
    its companion, and the pixel-neighbour count, longdouble."""
    proc = I.processed(active)
    ids = np.flatnonzero(proc) if patches is None else np.asarray(patches)
    ps = I.ps
    B = basis_table(ps, 1)[0]
    j, i = np.divmod(np.arange(ps * ps), ps)
    X0 = (B[i][:, BX] * B[j][:, BY]).astype(LD)       # (npix, 16), rounded once
    Xa = np.abs(X0)
    pn = I.patch_nodes()[ids]
    th = I.nodes[pn].reshape(-1, 16).astype(LD)
    dth = np.asarray(delta, np.float64).reshape(-1, 4)[pn].reshape(-1, 16).astype(LD)
    # a 16-term sum of products theta * (X0 Y0), the basis product itself
    # rounded once: a chain of 15 additions over terms of depth 2
    w1 = T(th @ X0.T, 17 * (np.abs(th) @ Xa.T))
    e = T(dth @ X0.T, 17 * (np.abs(dth) @ Xa.T))
    w2 = w1 + e
    idy, idx = np.divmod(ids, I.npx)
    u = T((I.start_x + idx[:, None] * ps + i[None, :]).astype(np.float64))
    v = T((I.start_y + idy[:, None] * ps + j[None, :]).astype(np.float64))
    counts = I.vis_off[ids + 1] - I.vis_off[ids]
    P = len(ids)
    mx = np.zeros(P, LD)
    mxa = np.zeros(P, LD)
    sm = np.zeros(P, LD)
    sma = np.zeros(P, LD)
    for jn in range(int(counts.max()) if P else 0):
        sel = counts > jn
        sub = np.zeros(P, np.int64)
        sub[sel] = I.vis_ids[I.vis_off[ids[sel]] + jn]
        Mt = np.concatenate([I.Mi, I.ti], 1)[sub].astype(np.float64)
        m = [T(np.broadcast_to(Mt[:, k][:, None], u.v.shape)) for k in range(12)]
        pp = (m[0] * u + m[1] * v) + m[2]
        qq = (m[3] * u + m[4] * v) + m[5]
        rr = (m[6] * u + m[7] * v) + m[8]
        d1, d2 = w1 * rr + m[11], w2 * rr + m[11]
        ex = (w1 * pp + m[9]) / d1 - (w2 * pp + m[9]) / d2
        ey = (w1 * qq + m[10]) / d1 - (w2 * qq + m[10]) / d2
        t = ex * ex + ey * ey
        diff = np.sqrt(t.v)
        with np.errstate(divide="ignore", invalid="ignore"):
            da = np.where(diff > 0, t.e / (2 * diff), np.sqrt(t.e)) + diff
        s = sel[:, None]
        dmax = np.where(s, diff, 0).max(1)
        amax = np.where(s & (diff == dmax[:, None]), da, 0).max(1)
        take = dmax > mx
        mxa = np.where(take, amax, mxa)
        mx = np.maximum(mx, dmax)
        sm += np.where(s, diff, 0).sum(1)
        sma += np.where(s, da, 0).sum(1)
    return dict(ids=ids, max=mx, max_a=mxa, sum=sm, sum_a=sma,
                count=(counts * ps * ps).astype(np.float64), nodes=pn)

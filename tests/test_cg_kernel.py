"""The PCG kernel (cg_kernel, smvs_b200/csrc/cg.cu) against a plain numpy
restatement of ConjugateGradient::solve (lib/conjugate_gradient.h:72-202),
run on the system the device built (smvsb_debug_get_system), so that only the
solver is under test.

The restatement runs in fp64 (scipy's block SpMV) and in extended precision
(np.longdouble, a fixed-order block SpMV). The longdouble run is the yardstick:
the kernel's x after k iterations must be about as close to it as the plain
fp64 run's, err_gpu <= 16 err_fp64 + 1e-15 (max-abs error over max-abs of
the longdouble x). A single wrong row of A d moves alpha by ~1e-4 relative,
far outside that bound, while rounding differences stay inside it.

The kernel can be stopped after exactly k iterations: max_iter = k + 1,
err_tol = 0 (r.r < 0 is never true) and q_tol = -inf (zeta < -inf neither).

Where the kernel reads its data from changes with the system's size: a CTA
handles 64 block rows per pass; the grid is min(2 x 132 SMs, ceil(n_nodes /
64)) CTAs; cg_kernel<1> holds pass 0 of H in shared memory; the row list of
the first 16 / NV passes is held in shared memory and later passes come from
the global list. The sizes below sit on those boundaries, and every test
asserts the boundary it is named for.
"""
import os

import numpy as np
import pytest
import scipy.sparse

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

CG_CONVERGENCE, CG_MAX_ITERATIONS = 0, 1       # include/smvs_b200.h
QUADS = 64              # block rows per CTA and pass (CG_THREADS / 4)
ROW_CACHE = 16          # row-list passes per CTA in shared memory, over NV views
H100_SMS = 132
GRID_MAX = 2 * H100_SMS                         # 2 CTAs per SM
PASS = GRID_MAX * QUADS                         # rows per pass of a capped grid
KS = (1, 2, 3, 5, 10)                           # truncated-iteration checkpoints
RATIO = 16.0
MARGIN = 1e-8
REPORT = []                                     # (case, k, err_gpu, err_fp64)


# ---------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------

class System:
    """H, P and g restricted to the block rows of `rows` (ascending node ids
    of the valid, active nodes), as the reference's system
    (lib/gauss_newton_step.cc:91-105); the kernel walks the same compacted
    row list. Hvals[k] is the row-major 4x4 block at (Hinner[k] // 4, the
    BSC column of k); P has the same layout, one diagonal block per row."""

    def __init__(self, sysd, rows, transpose=False):
        rows = np.asarray(rows, dtype=np.int64)
        n_nodes = len(sysd["Houter"]) - 1
        self.rows, self.n_nodes, self.n = rows, n_nodes, len(rows)
        where = np.full(n_nodes, -1, dtype=np.int64)
        where[rows] = np.arange(self.n)

        col = where[np.repeat(np.arange(n_nodes), np.diff(sysd["Houter"].astype(np.int64)))]
        row = where[sysd["Hinner"].astype(np.int64) // 4]
        assert (row >= 0).all() and (col >= 0).all(), "a block outside the rows"
        order = np.lexsort((col, row))
        self.col = col[order]
        row = row[order]
        self.starts = np.searchsorted(row, np.arange(self.n))
        # every row holds its diagonal block, so no row of the SpMV is empty
        diag = np.zeros(self.n, dtype=bool)
        diag[row[row == self.col]] = True
        assert diag.all(), "a row without its diagonal block"
        blocks = sysd["Hvals"][order].reshape(-1, 4, 4)
        self.H = np.ascontiguousarray(blocks.transpose(0, 2, 1) if transpose else blocks)
        self.bsr = scipy.sparse.bsr_matrix(
            (self.H, self.col, np.append(self.starts, len(self.col))),
            shape=(4 * self.n, 4 * self.n))

        pcol = np.repeat(np.arange(n_nodes), np.diff(sysd["Pouter"].astype(np.int64)))
        assert np.array_equal(pcol, rows), "P blocks are not the rows' diagonal"
        assert np.array_equal(sysd["Pinner"].astype(np.int64) // 4, rows)
        P = sysd["Pvals"].reshape(-1, 4, 4)
        self.P = np.ascontiguousarray(P.transpose(0, 2, 1) if transpose else P)
        self.g = np.ascontiguousarray(sysd["g"].reshape(-1, 4)[rows].reshape(-1))
        self._ld = None

    def _longdouble(self):
        if self._ld is None:
            self._ld = (self.H.astype(np.longdouble), self.P.astype(np.longdouble))
        return self._ld

    def multiply(self, v):
        if v.dtype == np.float64:
            return self.bsr @ v
        if self.n == 0:
            return v.copy()
        H, _ = self._longdouble()
        y = np.einsum("kij,kj->ki", H, v.reshape(-1, 4)[self.col])
        return np.add.reduceat(y, self.starts, axis=0).reshape(-1)

    def precondition(self, v):
        P = self.P if v.dtype == np.float64 else self._longdouble()[1]
        return np.einsum("kij,kj->ki", P, v.reshape(-1, 4)).reshape(-1)

    def scatter(self, x):
        """x of the compacted system as the full-size delta (zeros elsewhere)."""
        full = np.zeros((self.n_nodes, 4), dtype=x.dtype)
        full[self.rows] = x.reshape(-1, 4)
        return full.reshape(-1)


def pcg(S, dtype=np.float64, max_iter=200, err_tol=-1.0, q_tol=1e-3, snapshots=()):
    """ConjugateGradient::solve with the block-diagonal preconditioner, b = -g
    and error_tolerance = 0.01 ||g|| for err_tol < 0 (lib/depth_optimizer.cc:
    245-254), in `dtype`. Returns the full-size x, the iteration count, info,
    the trace (r.r before the first and after every iteration, zeta of every
    iteration that reached the quadratic-model test), the smallest relative
    distance of any stopping test from its threshold, and x after each of the
    iterations in `snapshots`."""
    one = dtype(1.0)
    b = -S.g.astype(dtype)
    x = np.zeros(4 * S.n, dtype=dtype)
    r = b.copy()
    tol = np.sqrt(np.dot(b, b)) * dtype(0.01) if err_tol < 0 else dtype(err_tol)
    z = S.precondition(r)
    r_dot_r = np.dot(z, r)
    d = z
    Q0 = -one * np.dot(x, b + r)
    rr, zetas, margins, snaps = [np.dot(r, r)], [], [], {}

    def margin(value, threshold):
        if not np.isfinite(threshold):
            return np.inf
        if threshold == 0:
            return np.inf if value >= 0 else 0.0
        m = abs(value - threshold) / abs(threshold)
        return 0.0 if np.isnan(m) else float(m)

    info = CG_MAX_ITERATIONS
    it = 1
    with np.errstate(divide="ignore", invalid="ignore"):
        while it < max_iter:
            Ad = S.multiply(d)
            alpha = r_dot_r / np.dot(d, Ad)
            x = x + d * alpha
            if it in snapshots:
                snaps[it] = S.scatter(x)
            r = r - Ad * alpha
            new_r_dot_r = np.dot(r, r)
            rr.append(new_r_dot_r)
            margins.append(margin(new_r_dot_r, tol))
            if new_r_dot_r < tol:
                info = CG_CONVERGENCE
                break
            Q1 = -one * np.dot(x, b + r)
            zeta = it * (Q1 - Q0) / Q1
            zetas.append(zeta)
            margins.append(margin(zeta, q_tol))
            if zeta < q_tol:
                info = CG_CONVERGENCE
                break
            Q0 = Q1
            z = S.precondition(r)
            new_r_dot_r = np.dot(z, r)
            beta = new_r_dot_r / r_dot_r
            d = z + d * beta
            r_dot_r = new_r_dot_r
            it += 1
    return dict(x=S.scatter(x), it=it, info=info, rr=rr, zeta=zetas,
                margin=min(margins, default=np.inf), snaps=snaps)


def err(x, ref):
    """max |x - ref| / max |ref|, evaluated in extended precision."""
    ref = np.asarray(ref, dtype=np.longdouble)
    diff = np.asarray(x, dtype=np.longdouble) - ref
    return float(np.max(np.abs(diff)) / np.max(np.abs(ref)))


# ---------------------------------------------------------------------------
# CPU: the restatement reproduces the compiled reference's golden solves
# ---------------------------------------------------------------------------

def golden_systems():
    for name in ("gn_s2.npz", "gn_s4.npz"):
        G = np.load(os.path.join(GOLD, name), allow_pickle=False)
        for tag in G["variants"]:
            sysd = {k: G[f"{tag}_{k}"] for k in
                    ("g", "Hvals", "Houter", "Hinner", "Pvals", "Pouter", "Pinner")}
            rows = np.flatnonzero(G["node_valid"] & G[f"{tag}_active"])
            yield (f"{name}:{tag}", sysd, rows, int(G[f"{tag}_cg_iters"]),
                   int(G[f"{tag}_cg_info"]), G[f"{tag}_x"])


GOLDEN = {case[0]: case[1:] for case in golden_systems()}


def test_longdouble_is_extended():
    assert np.finfo(np.longdouble).eps < 1e-18


@pytest.mark.parametrize("case", sorted(GOLDEN))
def test_restatement_matches_golden(case):
    """Iteration count and info exactly; x to 1e-13 on short solves, and on
    the long lit solves (85-87 iterations) to 5e-8, the amplified rounding of
    any implementation (the compiled reference's own error against the
    longdouble run is up to 5e-9 there)."""
    sysd, rows, it, info, x_ref = GOLDEN[case]
    S = System(sysd, rows)
    tol = 1e-13 if it <= 20 else 5e-8
    for dtype in (np.float64, np.longdouble):
        res = pcg(S, dtype)
        assert (res["it"], res["info"]) == (it, info), (dtype, res["it"], res["info"])
        assert res["margin"] >= MARGIN
        assert err(res["x"], x_ref) <= tol, (dtype, err(res["x"], x_ref))


def test_golden_iteration_counts():
    assert sorted(c[2] for c in GOLDEN.values()) == [3, 5, 9, 17, 85, 87]


@pytest.mark.parametrize("case", sorted(GOLDEN))
def test_restatement_fp64_tracks_longdouble(case):
    """The yardstick itself: in the first ten iterations plain fp64 stays
    within 1e-13 of the longdouble run."""
    sysd, rows, _, _, _ = GOLDEN[case]
    S = System(sysd, rows)
    kw = dict(max_iter=11, err_tol=0.0, q_tol=-np.inf, snapshots=KS)
    a, b = pcg(S, np.float64, **kw), pcg(S, np.longdouble, **kw)
    assert (a["it"], a["info"]) == (11, CG_MAX_ITERATIONS)
    for k in KS:
        assert 0.0 < err(a["snaps"][k], b["snaps"][k]) < 1e-13, k


def test_transposed_blocks_are_caught():
    """Reading every block transposed changes the iteration counts: the golden
    comparison above pins the block layout."""
    for case, (sysd, rows, it, _, _) in GOLDEN.items():
        if it >= 9:
            assert pcg(System(sysd, rows, transpose=True))["it"] != it, case


def test_empty_system_leaves_x_untouched():
    """alpha = 0 / 0 on an empty system: the compacted restatement (like the
    reference and the kernel) has nothing to update, runs to max_iter and
    leaves x zero."""
    sysd, rows, _, _, _ = GOLDEN[sorted(GOLDEN)[0]]
    n = len(sysd["Houter"]) - 1
    empty = dict(g=np.zeros(4 * n), Hvals=np.zeros((0, 16)), Houter=np.zeros(n + 1, np.uint64),
                 Hinner=np.zeros(0, np.uint64), Pvals=np.zeros((0, 16)),
                 Pouter=np.zeros(n + 1, np.uint64), Pinner=np.zeros(0, np.uint64))
    for dtype in (np.float64, np.longdouble):
        res = pcg(System(empty, []), dtype)
        assert (res["it"], res["info"]) == (200, CG_MAX_ITERATIONS)
        assert res["x"].shape == (4 * n,) and not res["x"].any()


# ---------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------

def kernel_grid(n_nodes):
    return min(GRID_MAX, -(-n_nodes // QUADS))


def kernel_passes(n_rows, n_nodes):
    return -(-n_rows // (kernel_grid(n_nodes) * QUADS))


def check_sms():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert sms == H100_SMS, f"the boundary sizes are chosen for {H100_SMS} SMs, not {sms}"


def construct(ctx, wl, nodes):
    """The system of the valid nodes `nodes`, activated alone."""
    act = np.zeros(ctx.n_nodes, dtype=np.uint8)
    act[nodes] = 1
    assert wl.node_valid[nodes].all()
    ctx.gn_construct(act, None, 0.01, 0.0)
    S = System(ctx.debug_get_system(), nodes)
    assert S.n == len(nodes)        # n_rows: one row per valid, active node
    return S


def truncated(ctx, k):
    it, info = ctx.cg_solve(max_iter=k + 1, err_tol=0.0, q_tol=-np.inf)
    assert (it, info) == (k + 1, CG_MAX_ITERATIONS)
    return ctx.get_delta()


def check_truncated(ctx, S, case, ks=KS):
    """x after k iterations against the longdouble restatement, for every k
    in ks whose fp64 run stays clear of underflow (a system the
    preconditioner solves in one step shrinks its residual by ~1e-16 per
    iteration from then on)."""
    kw = dict(max_iter=max(ks) + 1, err_tol=0.0, q_tol=-np.inf, snapshots=ks)
    ld, f64 = pcg(S, np.longdouble, **kw), pcg(S, np.float64, **kw)
    compared = []
    for k in ks:
        if not np.isfinite(f64["snaps"][k]).all() or min(f64["rr"][:k + 1]) < 1e-200:
            continue
        x = truncated(ctx, k)
        e_gpu, e_64 = err(x, ld["snaps"][k]), err(f64["snaps"][k], ld["snaps"][k])
        REPORT.append((case, k, e_gpu, e_64))
        assert e_gpu <= RATIO * e_64 + 1e-15, (case, k, e_gpu, e_64)
        compared.append(k)
    assert compared[:3] == [1, 2, 3], compared
    return ld


def check_full(ctx, S, case, longdouble=False, **kw):
    """A solve with the reference's stopping rules: iteration count and info
    those of the fp64 restatement (whose every stopping test is at least
    MARGIN from its threshold), x bitwise that of the run truncated at the
    same iteration, and (where affordable) x against longdouble."""
    ref = pcg(S, np.float64, **kw)
    assert ref["margin"] >= MARGIN, (case, ref["margin"])
    it, info = ctx.cg_solve(**kw)
    assert (it, info) == (ref["it"], ref["info"]), (case, it, info, ref["it"], ref["info"])
    x = ctx.get_delta()
    k = it if info == CG_CONVERGENCE else it - 1
    assert np.array_equal(truncated(ctx, k), x), case
    if longdouble:
        ld = pcg(S, np.longdouble, **kw)
        assert (ld["it"], ld["info"]) == (it, info), case
        e_gpu, e_64 = err(x, ld["x"]), err(ref["x"], ld["x"])
        REPORT.append((case, "full", e_gpu, e_64))
        assert e_gpu <= RATIO * e_64 + 1e-15, (case, e_gpu, e_64)
    return ref


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    rows = [r for r in REPORT if r[3] > 0]
    if rows:
        worst = max(rows, key=lambda r: r[2] / r[3])
        print(f"\ncg kernel: {len(REPORT)} comparisons, largest err_gpu / err_fp64 "
              f"{worst[2] / worst[3]:.3g} ({worst[0]}, k={worst[1]}: "
              f"{worst[2]:.3g} vs {worst[3]:.3g})")


# ---------------------------------------------------------------------------
# GPU: one large surface, N rows selected through the active set
# ---------------------------------------------------------------------------

@pytest.fixture(scope="module")
def big():
    """2880x1920 at scale 2: 344 401 nodes (grid capped at 264 CTAs) and about
    312 700 valid ones, 19 passes: past the row cache of every batch width."""
    from smvs_b200 import api, workload
    check_sms()
    wl = workload.build_workload(2880, 1920, 2, scale=2)
    valid = np.flatnonzero(wl.node_valid)
    assert kernel_grid(len(wl.node_valid)) == GRID_MAX
    assert kernel_passes(len(valid), len(wl.node_valid)) > ROW_CACHE
    ctx = api.Context(0)
    wl.push(ctx)
    yield wl, ctx, valid
    ctx.close()


def pick(valid, n, how):
    if how == "prefix":             # row-major: full 3x3 stencils
        return valid[:n]
    rng = np.random.default_rng(n)  # scattered: mostly diagonal-only rows
    return np.sort(rng.choice(valid, size=n, replace=False))


# (rows, passes): 1-65 leave most CTAs without rows (65: CTA 1 holds one);
# PASS +- 1: pass 0 exactly full, then one row alone in pass 1; 4 PASS + 1:
# the first row of the update phase's second CG_UF group; 16 PASS +- 1: the
# NV = 1 row-cache boundary (pass 16 is the first past the cache)
BIG = [(1, 1), (63, 1), (64, 1), (65, 1), (PASS - 1, 1), (PASS, 1), (PASS + 1, 2),
       (4 * PASS + 1, 5), (16 * PASS - 1, 16), (16 * PASS, 16), (16 * PASS + 1, 17)]


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["random", "prefix"])
@pytest.mark.parametrize("n,passes", BIG)
def test_big_surface_rows(big, n, passes, how):
    wl, ctx, valid = big
    assert kernel_passes(n, ctx.n_nodes) == passes
    S = construct(ctx, wl, pick(valid, n, how))
    case = f"big {how} {n}"
    check_truncated(ctx, S, case)
    check_full(ctx, S, case)


@pytest.mark.gpu
def test_big_surface_all_valid(big):
    wl, ctx, valid = big
    assert kernel_passes(len(valid), ctx.n_nodes) == 19
    S = construct(ctx, wl, valid)
    check_truncated(ctx, S, "big all")
    check_full(ctx, S, "big all")


# ---------------------------------------------------------------------------
# GPU: small surfaces (uncapped grids), a long lit solve, the stopping rules
# ---------------------------------------------------------------------------

def small(width, height, shading=False):
    from smvs_b200 import api, workload
    wl = workload.build_workload(width, height, 2, scale=2, shading=shading)
    ctx = api.Context(0)
    wl.push(ctx)
    return wl, ctx


# (width, height, nodes, grid): 8x8 nodes, one CTA; 10x10, two; 128x132 =
# 16 896 nodes, 264 CTAs, one pass; 129x132, the first capped size
SMALL = [(34, 34, 64, 1), (42, 42, 100, 2), (514, 530, 16896, 264), (518, 530, 17028, 264)]


@pytest.mark.gpu
@pytest.mark.parametrize("width,height,nodes,grid", SMALL)
def test_small_surface(width, height, nodes, grid):
    check_sms()
    wl, ctx = small(width, height)
    with ctx:
        assert ctx.n_nodes == nodes and kernel_grid(nodes) == grid
        valid = np.flatnonzero(wl.node_valid)
        assert len(valid) > 0.5 * nodes
        assert kernel_passes(len(valid), nodes) == 1
        assert (-(-nodes // QUADS) > GRID_MAX) == (width == 518)
        S = construct(ctx, wl, valid)
        case = f"small {width}x{height}"
        check_truncated(ctx, S, case)
        check_full(ctx, S, case, longdouble=True)


@pytest.mark.gpu
def test_lit_long_solve():
    """The lit golden inputs with the device's own fit_lighting: a long solve
    (the reference's takes 87 iterations with its lighting)."""
    from smvs_b200 import api
    G = np.load(os.path.join(GOLD, "gn_s2.npz"), allow_pickle=False)
    n = int(G["n_sub"])
    with api.Context(0) as ctx:
        ctx.set_views(G["main_grad"], [G[f"sub_grad{k}"] for k in range(n)],
                      [G[f"sub_hess{k}"] for k in range(n)], G["Mi"], G["ti"],
                      float(G["flen"]), float(G["inv_flen"]), G["shading"], G["shading_grad"])
        ctx.set_surface(int(G["scale"]), int(G["npx"]), int(G["npy"]), int(G["start_x"]),
                        int(G["start_y"]), G["nodes"], G["node_valid"], G["patch_valid"],
                        G["vis_off"], G["vis_ids"])
        light = ctx.fit_lighting()
        act = G["lit_active"]
        ctx.gn_construct(act, light, 0.01, 0.0)
        S = System(ctx.debug_get_system(), np.flatnonzero(G["node_valid"] & act))
        check_truncated(ctx, S, "lit")
        ref = check_full(ctx, S, "lit", longdouble=True)
        assert ref["it"] >= 50, ref["it"]


@pytest.fixture(scope="module")
def one_pass():
    """The 514x530 surface: 16 896 nodes, 264 CTAs, one pass."""
    check_sms()
    wl, ctx = small(514, 530)
    valid = np.flatnonzero(wl.node_valid)
    S = construct(ctx, wl, valid)
    yield wl, ctx, S
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("max_iter", [0, 1, 2])
def test_max_iter_small(one_pass, max_iter):
    """max_iter 0 and 1: no iteration, (1, MAX_ITERATIONS), x = 0; 2: one
    iteration, which returns 1 if it stops and 2 otherwise."""
    _, ctx, S = one_pass
    ref = pcg(S, max_iter=max_iter)
    assert ref["margin"] >= MARGIN
    if max_iter < 2:
        assert (ref["it"], ref["info"]) == (1, CG_MAX_ITERATIONS)
    else:
        assert (ref["it"], ref["info"]) in ((1, CG_CONVERGENCE), (2, CG_MAX_ITERATIONS))
    it, info = ctx.cg_solve(max_iter=max_iter)
    assert (it, info) == (ref["it"], ref["info"])
    x = ctx.get_delta()
    if max_iter < 2:
        assert info == CG_MAX_ITERATIONS and not x.any()
    else:
        ld = pcg(S, np.longdouble, max_iter=max_iter)
        assert err(x, ld["x"]) <= RATIO * err(ref["x"], ld["x"]) + 1e-15


@pytest.mark.gpu
@pytest.mark.parametrize("j", [1, 2, 7])
def test_residual_rule_stops_at(one_pass, j):
    """An explicit err_tol stops the solve by the residual rule, not the
    quadratic-model rule that ends most solves, at the iteration i where r.r
    reaches its j-th new low: err_tol is the geometric mean of r.r at i and
    the smallest r.r of the iterations before i (16 r.r at i for i = 1).
    (r.r is not monotone in PCG: on this system it rises in iteration 1 and
    in iteration 2, so r.r at i - 1 would not do.)"""
    _, ctx, S = one_pass
    rr = pcg(S)["rr"]
    lows = [i for i in range(1, len(rr)) if rr[i] < min(rr[1:i], default=np.inf)]
    assert len(lows) >= 7, lows
    i = lows[j - 1]
    tol = float(np.sqrt(rr[i] * min(rr[1:i], default=16 * rr[i])))
    ref = check_full(ctx, S, f"err_tol low {j}", longdouble=True, err_tol=tol)
    assert (ref["it"], ref["info"]) == (i, CG_CONVERGENCE)
    assert ref["rr"][-1] < tol and len(ref["zeta"]) == i - 1


@pytest.mark.gpu
def test_empty_active_set():
    from smvs_b200 import api, workload
    wl = workload.build_workload(42, 42, 2, scale=2)
    with api.Context(0) as ctx:
        wl.push(ctx)
        S = construct(ctx, wl, np.zeros(0, dtype=np.int64))
        ref = pcg(S)
        it, info = ctx.cg_solve()
        assert (it, info) == (ref["it"], ref["info"]) == (200, CG_MAX_ITERATIONS)
        x = ctx.get_delta()
        assert x.shape == ref["x"].shape and not x.any()
        assert ctx.cg_solve(max_iter=3) == (3, CG_MAX_ITERATIONS)


# ---------------------------------------------------------------------------
# GPU: every batch width against the single-view kernel
# ---------------------------------------------------------------------------

def batch_width(m):
    return 1 if m == 1 else 2 if m == 2 else 4 if m <= 4 else 8


@pytest.mark.gpu
def test_batch_widths_match_single_view(big):
    """One Newton step of the large view in batches of m = 2, 3, 4, 5 and 8
    (one PCG launch with NV = 2, 4, 4, 8, 8; their row caches end at pass 8,
    4, 4, 2, 2 of 19, and they do not hold H in shared memory) against the
    single-view launch (pass 0 of H in shared memory, 16 passes cached)."""
    from smvs_b200 import api
    wl, ctx, valid = big
    n_rows = len(valid)
    ctx.set_nodes(wl.nodes)
    single = ctx.newton_loop(None, 0.01, 0.0, max_steps=1)
    nodes = ctx.get_nodes()
    ctx.set_nodes(wl.nodes)
    assert single["newton_steps"] == 1 and not single["nan"]
    assert single["cg_row_iterations"] == n_rows * single["cg_iterations"]
    ctxs = [ctx] + [api.Context(0) for _ in range(7)]
    try:
        for c in ctxs[1:]:
            wl.push(c)
        for m in (2, 3, 4, 5, 8):
            assert kernel_passes(n_rows, ctx.n_nodes) > ROW_CACHE // batch_width(m)
            for c in ctxs[:m]:
                c.set_nodes(wl.nodes)
            stats = api.newton_loop_batch(ctxs[:m], None, 0.01, 0.0, max_steps=1)
            for v, (c, st) in enumerate(zip(ctxs[:m], stats)):
                for key in ("newton_steps", "cg_iterations", "n_active", "nan",
                            "cg_row_iterations", "cg_block_iterations"):
                    assert st[key] == single[key], (m, v, key, st[key], single[key])
                assert np.array_equal(c.get_nodes(), nodes), (m, v)
    finally:
        ctx.set_nodes(wl.nodes)
        for c in ctxs[1:]:
            c.close()


@pytest.mark.gpu
def test_mixed_batch_matches_single_view(big):
    """One launch (NV = 4) of the large view, a one-CTA view and a window of
    the large workload with 16 900 valid nodes (4 rows in pass 1)."""
    from smvs_b200 import api, workload
    wl, ctx, _ = big
    tiny = workload.build_workload(34, 34, 2, scale=2)
    win = wl.restrict(300, 150, 129, 129)
    assert int(win.node_valid.sum()) == PASS + 4
    assert kernel_grid(len(tiny.node_valid)) == 1
    wls = [wl, tiny, win]
    ctxs = [ctx, api.Context(0), api.Context(0)]
    try:
        single, nodes = [], []
        for w, c in zip(wls, ctxs):
            w.push(c)
            single.append(c.newton_loop(None, 0.01, 0.0, max_steps=1))
            nodes.append(c.get_nodes())
            c.set_nodes(w.nodes)
        win_rows = int(single[2]["cg_row_iterations"]) // single[2]["cg_iterations"]
        assert win_rows == PASS + 4 and kernel_passes(win_rows, ctx.n_nodes) == 2
        stats = api.newton_loop_batch(ctxs, None, 0.01, 0.0, max_steps=1)
        for v, (c, st) in enumerate(zip(ctxs, stats)):
            for key in ("newton_steps", "cg_iterations", "n_active", "nan",
                        "cg_row_iterations"):
                assert st[key] == single[v][key], (v, key, st[key], single[v][key])
            assert np.array_equal(c.get_nodes(), nodes[v]), v
    finally:
        ctx.set_nodes(wl.nodes)
        for c in ctxs[1:]:
            c.close()

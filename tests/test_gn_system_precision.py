"""The Gauss-Newton construct (K1 gn_patch_kernel, K2a gn_assemble_kernel, K2b
gn_precond_kernel) and the node update (K4) against an extended-precision
restatement (tests/gn_precision.py), entry by entry.

The bound. For every entry x of g and of H (all <= 9 blocks of every valid,
active row; the rows of other nodes must be exactly 0):

    |x - x_ld| <= u E,   u = 2^-53,

where x_ld is the longdouble value and E the entry's first-order error bound,
built from the code, not fitted to measured errors:

* the per-sample quantities the kernel computes bitwise like the reference
  (xd) are the restatement's own float64 values: no error;
* every later operation of the per-sample phase (ax, ay, be, the C / N
  coefficients, SH terms, weights, the row products) adds its rounding and
  propagates its operands' bounds to first order (gn_precision.T). This is
  the "non-xd operations per sample" part of K, counted operation by
  operation instead of as one depth for all entries;
* the sums: an entry of H is a sum over at most 4 patches, S samples each,
  of the sample's residual rows (the reference's order) or of the 36 terms of
  D^T A D (the kernel's). Whatever the order, a sum of N terms is off by at
  most (N - 1) u times the sum of their magnitudes, so the chain length
  K_sum = 4 S (rows + 36) + 16 (rows + 6 for g) multiplies the entry's
  magnitude |D|^T |A| |D|. At S = 4096 that is 4 S rows and more, as a
  sequential sum of every row of every sample would need.

The same bound must hold for the compiled reference (oracle/_ref), whose
summation order is different again: that validates both the bound and the
restatement without a GPU.

P: each block against the longdouble inverse (adjugate, no LDL^T) of the
device's own diagonal block, so that only K2b is under test:
|P - B^-1| <= c u kappa_inf(B) max|B^-1| with c = 64 (4 n^2 for the
factorisation, the inversion of L and the product L^T D^-1 L of a 4x4).
Blocks with kappa_inf u > 1e-3, or numerically singular by their float64
SVD condition number (where the adjugate's determinant is rounding noise),
are excluded from the value check; every block, excluded or not, must take
the reference's branch exactly (inverted, or kept un-inverted on a zero
pivot or NaN); inactive nodes get no P block.

The update: the largest reprojection difference per patch decides its flag
(> 0.15 px); the mean shift sum / count is bounded like the sums above.
"""
import os

import numpy as np
import pytest

import gn_precision as gp

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U = 2.0 ** -53
P_C = 64.0
# case -> worst |err| / (u E) of g and H and worst of P, for the device and
# for the reference, with S, rows per sample and the shading branch counts
REPORT = {}


def load(name):
    return np.load(os.path.join(GOLD, name), allow_pickle=False)


# ---------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------

def restate(I, active, light, reg, lreg, **kw):
    pat = gp.construct_patches(I, active, light, reg, lreg, **kw)
    return pat, gp.assemble(I, active, pat)


def worst_ratio(sysd, I, asm):
    """Largest |x - x_ld| / (u E) over g and the stored H blocks, with the
    entry it was found at; the structure of H and zero rows asserted."""
    row, col, k = gp.system_blocks(I, sysd)
    on = asm["on"]
    assert on[row].all() and on[col].all()
    Hv = sysd["Hvals"].astype(gp.LD).reshape(-1, 4, 4)
    err = np.abs(Hv - asm["H"][row, k])
    bound = U * asm["He"][row, k]
    # a block that is stored but has no contribution must be 0 exactly
    assert (err[bound == 0] == 0).all()
    with np.errstate(divide="ignore", invalid="ignore"):
        rH = np.where(bound > 0, err / bound, 0)
    g = sysd["g"].reshape(-1, 4).astype(gp.LD)
    assert not g[~on].any(), "a gradient entry in an inactive row"
    eg = np.abs(g - asm["g"])
    bg = U * asm["ge"]
    assert (eg[bg == 0] == 0).all()
    with np.errstate(divide="ignore", invalid="ignore"):
        rg = np.where(bg > 0, eg / bg, 0)
    wh = np.unravel_index(int(np.argmax(rH)), rH.shape) if rH.size else None
    wg = np.unravel_index(int(np.argmax(rg)), rg.shape)
    where = dict(H_block=(int(row[wh[0]]), int(col[wh[0]])) if wh else None,
                 g_node=int(wg[0]))
    return float(max(rH.max(initial=0), rg.max())), where, len(row)


def check_P(sysd):
    """K2b against the longdouble inverse of the device's own blocks."""
    outer = sysd["Houter"].astype(np.int64)
    col = np.repeat(np.arange(len(outer) - 1), np.diff(outer))
    row = sysd["Hinner"].astype(np.int64) // 4
    diag = row == col
    nodes = col[diag]
    B = sysd["Hvals"][diag].reshape(-1, 4, 4)
    pcol = np.repeat(np.arange(len(outer) - 1), np.diff(sysd["Pouter"].astype(np.int64)))
    assert np.array_equal(pcol, nodes), "P blocks are not the active rows' diagonal"
    P = sysd["Pvals"].reshape(-1, 4, 4)
    inv, det = gp.inverse4(B)
    inverts = gp.ldl_branch(B)
    kept = np.all(P == B, axis=(1, 2))
    assert np.array_equal(kept, ~inverts), "a block took the wrong branch"
    assert not (inverts & ~np.isfinite(P).all(axis=(1, 2))).any()
    Bl = B.astype(gp.LD)
    with np.errstate(invalid="ignore", over="ignore"):
        kappa = np.abs(Bl).sum(2).max(1) * np.abs(inv).sum(2).max(1)
    # a numerically singular block makes the adjugate's determinant rounding
    # noise and its kappa meaningless: the SVD's 2-norm condition number
    # (within a factor 4 of kappa_inf for a 4x4) excludes it as well
    with np.errstate(all="ignore"):
        cond2 = np.linalg.cond(B) if len(B) else np.zeros(0)
    good = (inverts & np.isfinite(kappa) & (kappa * U <= 1e-3)
            & np.isfinite(cond2) & (4 * cond2 * U <= 1e-3))
    worst = 0.0
    if good.any():
        bound = P_C * U * kappa[good] * np.abs(inv[good]).max(axis=(1, 2))
        r = np.abs(P[good].astype(gp.LD) - inv[good]).max(axis=(1, 2)) / bound
        worst = float(r.max())
    return worst, int(good.sum()), int((~inverts).sum())


def check_system(case, who, I, sysd, active, light, reg, lreg, pat_asm=None):
    """sysd (the device's or the reference's system, `who`) against the
    restatement: the bound on g and H, the block structure, and P."""
    pat, asm = pat_asm or restate(I, active, light, reg, lreg)
    assert pat["margin"] > 1e-9, "a shading sample within 1e-9 of its threshold"
    blocks = gp.expected_blocks(I, active, I.processed(active))
    r, where, nblk = worst_ratio(sysd, I, asm)
    assert nblk == len(blocks)
    p, n_good, n_kept = check_P(sysd)
    row = REPORT.setdefault(case, dict(S=pat["S"], rows=pat["rows"], shade=pat["shade"]))
    row[who] = (r, p)
    assert r <= 1.0, (case, who, r, where)
    assert p <= 1.0, (case, who, p)
    return pat, asm, n_kept


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\nworst |err| / (u E)          g,H device  g,H ref  P device    P ref"
              "     S  rows  shading ok/failed")
        nan = (float("nan"), float("nan"))
        for case, r in REPORT.items():
            d, f = r.get("device", nan), r.get("reference", nan)
            print(f"  {case:30s} {d[0]:9.3g} {f[0]:9.3g} {d[1]:9.3g} {f[1]:9.3g} "
                  f"{r['S']:5d} {r['rows']:5d}  {r['shade']}")


# ---------------------------------------------------------------------------
# CPU: the restatement against the golden systems of the compiled reference
# ---------------------------------------------------------------------------

def test_longdouble_is_extended():
    assert np.finfo(np.longdouble).eps < 1e-18


def golden_cases():
    for name in ("gn_s2.npz", "gn_s4.npz"):
        for tag in load(name)["variants"]:
            yield f"{name}:{tag}"


def golden_case(case):
    name, tag = case.split(":")
    G = load(name)
    I = gp.Inputs.from_golden(G)
    light = G["light"] if tag in ("lit", "litR") else None
    sysd = {k: G[f"{tag}_{k}"] for k in
            ("g", "Hvals", "Houter", "Hinner", "Pvals", "Pouter", "Pinner")}
    return G, I, sysd, G[f"{tag}_active"], light, float(G["regularization"]), \
        float(G[f"{tag}_lreg"])


@pytest.mark.parametrize("case", list(golden_cases()))
def test_golden_systems_meet_the_bound(case):
    G, I, sysd, act, light, reg, lreg = golden_case(case)
    pat, _, _ = check_system(f"golden {case}", "reference", I, sysd, act, light, reg, lreg)
    if light is not None:
        ok, failed = pat["shade"]
        assert ok > 0 and failed > 0, pat["shade"]      # both branches taken


@pytest.mark.parametrize("name", ["gn_s2.npz", "gn_s4.npz"])
def test_golden_update(name):
    """upd_*: the reference's update with its own CG step (full_x)."""
    G = load(name)
    I = gp.Inputs.from_golden(G)
    act = G["full_active"]
    res = check_update(I, act, G["full_x"], G["upd_active"], int(G["upd_n_active"]),
                       float(G["upd_mean_shift"]), f"golden {name}")
    valid = I.node_valid.astype(bool)
    assert np.array_equal(G["upd_nodes"][valid], (I.nodes + G["full_x"].reshape(-1, 4))[valid])


def update_expectation(I, act, delta, thresh=0.15):
    r = gp.update(I, act, delta)
    flag = r["max"] > thresh
    amb = np.abs(r["max"] - thresh) <= np.maximum(1e-9 * thresh, U * r["max_a"])
    nn = len(I.node_valid)
    sure = np.zeros(nn, bool)
    maybe = np.zeros(nn, bool)
    for q in range(4):
        np.logical_or.at(sure, r["nodes"][:, q], flag & ~amb)
        np.logical_or.at(maybe, r["nodes"][:, q], amb)
    shift = r["sum"].sum() / r["count"].sum()
    n = r["count"].sum()
    shift_e = (r["sum_a"].sum() + n * r["sum"].sum()) / r["count"].sum() + abs(shift)
    return dict(r=r, sure=sure, unsure=maybe & ~sure, shift=shift, shift_e=shift_e,
                flag=flag, amb=amb)


def check_update(I, act, delta, got_active, got_n, got_shift, case, full_opt=False):
    ex = update_expectation(I, act, delta)
    decided = ~ex["unsure"]
    want = act.astype(bool) if full_opt else ex["sure"]
    got = np.asarray(got_active).astype(bool)
    assert np.array_equal(got[decided], want[decided]), case
    assert ex["unsure"].sum() <= max(2, 0.001 * len(got)), ex["unsure"].sum()
    assert got_n == int(got.sum())
    r = abs(gp.LD(got_shift) - ex["shift"]) / (U * ex["shift_e"])
    REPORT[f"update {case}"] = dict(S=int(I.ps * I.ps), rows=0, shade=[
        int(ex["flag"].sum()), int((~ex["flag"]).sum())], device=(float(r), float("nan")))
    assert r <= 1.0, (case, float(r))
    return dict(flagged=int(ex["flag"].sum()), amb=int(ex["amb"].sum()))


# ---------------------------------------------------------------------------
# CPU: sensitivity -- every mutation of the restatement breaks the bound
# ---------------------------------------------------------------------------

def _mutant_ratio(I, sysd, asm):
    try:
        r, _, _ = worst_ratio(sysd, I, asm)
    except AssertionError:
        return np.inf
    return r


def test_sensitivity_golden():
    G, I, sysd, act, light, reg, lreg = golden_case("gn_s2.npz:full")
    pat, asm = restate(I, act, light, reg, lreg)
    assert _mutant_ratio(I, sysd, asm) <= 1.0
    proc = np.flatnonzero(I.processed(act))
    # one sample of one patch dropped
    m = gp.construct_patches(I, act, light, reg, lreg, drop_sample=(5, 3))
    assert _mutant_ratio(I, sysd, gp.assemble(I, act, m)) > 1.0
    # the last patch of a partial CTA missing (8 patches per CTA at S = 16)
    assert len(proc) % 8 != 0
    m = gp.construct_patches(I, act, light, reg, lreg, patches=proc[:-1])
    assert _mutant_ratio(I, sysd, gp.assemble(I, act, m)) > 1.0
    # one off-diagonal block transposed
    a2 = dict(asm)
    a2["H"] = asm["H"].copy()
    node = int(np.flatnonzero(asm["on"])[len(proc) // 2])
    a2["H"][node, 5] = asm["H"][node, 5].T.copy()
    assert _mutant_ratio(I, sysd, a2) > 1.0
    # the geometry rows of one sample dropped (regularization > 0)
    m = gp.construct_patches(I, act, light, reg, lreg, drop_geometry=(7, 2))
    assert _mutant_ratio(I, sysd, gp.assemble(I, act, m)) > 1.0
    # a g contribution from a patch whose only active node is another one
    G2, I2, sysd2, act2, l2, reg2, lreg2 = golden_case("gn_s2.npz:part")
    pat2, asm2 = restate(I2, act2, l2, reg2, lreg2)
    assert _mutant_ratio(I2, sysd2, asm2) <= 1.0
    on = asm2["on"]
    pn = I2.patch_nodes()
    lone = [p for p in np.flatnonzero(I2.processed(act2)) if on[pn[p]].sum() == 1]
    assert lone
    p = lone[0]
    li_on = int(np.flatnonzero(on[pn[p]])[0])
    other = pn[p][(li_on + 1) % 4]
    k = list(pat2["ids"]).index(p)
    a3 = dict(asm2)
    a3["g"] = asm2["g"].copy()
    j = (li_on + 1) % 4
    a3["g"][other] += pat2["g"][k, j * 4:j * 4 + 4]
    assert _mutant_ratio(I2, sysd2, a3) > 1.0


# ---------------------------------------------------------------------------
# K1 / K2a / K2b at every samples-per-patch instantiation: the compiled
# reference on CPU, the kernels on the GPU, the same scenes and restatements
# ---------------------------------------------------------------------------

# scale -> (width, height): scales 0-5 with a patch count that is not a
# multiple of the patches per CTA (8 up to S = 16, 2 at S = 64); scales 7-8
# as in test_gpu_high_scales (9 x 7 and 4 x 3 patches)
SCENES = {0: (45, 33), 1: (70, 50), 2: (164, 120), 3: (200, 150), 4: (362, 262),
          5: (417, 343), 6: (640, 480), 7: (1300, 1060), 8: (1300, 1060)}
SAMPLES = {0: 1, 1: 4, 2: 16, 3: 16, 4: 64, 5: 64, 6: 256, 7: 1024, 8: 4096}
CASES = ("full", "full reg 0", "25%", "single", "lit", "lit lreg 5")
_SCENES, _RESTATED = {}, {}


def needs_ref():
    from oracle import ref as oref
    if not oref.available():
        pytest.skip("oracle/_ref not built")


def patches_per_cta(S):
    return 8 if S < 64 else (2 if S == 64 else 1)


def _single_node(I):
    """One valid node whose eight neighbours are all inactive."""
    on = np.zeros(len(I.node_valid), np.uint8)
    ns = I.npx + 1
    cand = [n for n in np.flatnonzero(I.node_valid)
            if 0 < n % ns < I.npx and 0 < n // ns < I.npy]
    on[cand[len(cand) // 2] if cand else np.flatnonzero(I.node_valid)[0]] = 1
    return on


def scene(scale):
    """The scale's reference scene (shared by the CPU and GPU tests): a
    shading scene whose shading image is 0 over the left quarter and whose
    shading gradient is 0 over a further block, so that the lit construct
    takes both branches of the shading `ok` test; the lighting is fitted
    before that."""
    if scale not in _SCENES:
        from util_scene import Pair
        w, h = SCENES[scale]
        P = Pair(w, h, 2, scale, seed_index=200 + scale, shading=True, gpu=False)
        light = P.R.fit_lighting()
        img, grad = P.R.shading()
        img[:, :w // 4] = 0.0
        grad[h // 2:, w // 4:w // 2] = 0.0
        P.R.set_shading(img, grad)
        I = gp.Inputs.from_pair(P)
        assert I.npos * I.npos == SAMPLES[scale]
        if scale <= 5:
            assert (I.npx * I.npy) % patches_per_cta(SAMPLES[scale]) != 0
        full = P.node_valid.copy()
        rng = np.random.default_rng(scale)
        part = (full & (rng.random(full.shape) < 0.25)).astype(np.uint8)
        cases = {"full": (full, None, 0.01, 0.0), "full reg 0": (full, None, 0.0, 0.0),
                 "25%": (part, None, 0.01, 0.0), "single": (_single_node(I), None, 0.01, 0.0),
                 "lit": (full, light, 0.01, 0.0), "lit lreg 5": (full, light, 0.01, 5.0)}
        _SCENES[scale] = (P, I, cases)
    return _SCENES[scale]


def restated(key, I, case):
    if key not in _RESTATED:
        _RESTATED[key] = restate(I, *case)
    return _RESTATED[key]


def _check_scale(scale, who, system):
    P, I, cases = scene(scale)
    for name in CASES:
        act, light, reg, lreg = cases[name]
        pat, asm = restated((scale, name), I, cases[name])
        check_system(f"s{scale} {name}", who, I, system(act, light, reg, lreg), act, light,
                     reg, lreg, pat_asm=(pat, asm))
        if name == "single":
            assert 1 <= len(pat["ids"]) <= 4
        if light is not None:
            ok, failed = pat["shade"]
            assert ok > 0 and failed > 0, pat["shade"]     # both branches taken


def _ref_system(P):
    def system(act, light, reg, lreg):
        P.R.gn_construct(act, light, reg, lreg)
        return P.R.get_system()
    return system


def _device_system(ctx):
    def system(act, light, reg, lreg):
        ctx.gn_construct(act, light, reg, lreg)
        return ctx.debug_get_system()
    return system


def _with_context(P):
    """A GPU context fed with the pair's (shading-modified) arrays."""
    from smvs_b200 import api
    P.ctx = api.Context(0)
    P.push_views()
    P.push_surface()
    return P.ctx


@pytest.mark.parametrize("scale", sorted(SCENES))
def test_reference_every_instantiation(scale):
    """The compiled reference meets the bound at every S, lit and unlit."""
    needs_ref()
    _check_scale(scale, "reference", _ref_system(scene(scale)[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("scale", sorted(SCENES))
def test_construct_every_instantiation(scale):
    needs_ref()
    P = scene(scale)[0]
    ctx = _with_context(P)
    try:
        _check_scale(scale, "device", _device_system(ctx))
    finally:
        ctx.close()
        P.ctx = None


def _n32():
    """32 neighbours, 496 pair rows per sample (uniform_scene of
    test_mixed_views), its restatement and the reference's system."""
    if "n32" not in _SCENES:
        from util_scene import Pair
        from test_mixed_views import uniform_scene
        P = Pair(160, 120, 32, 2, scene=uniform_scene(32), gpu=False)
        I = gp.Inputs.from_pair(P)
        assert np.diff(I.vis_off.astype(np.int64)).max() == 32
        _SCENES["n32"] = (P, I, {"full": (P.node_valid, None, 0.01, 0.0)})
    P, I, cases = _SCENES["n32"]
    return P, I, cases["full"], restated("n32", I, cases["full"])


def test_reference_32_neighbours():
    needs_ref()
    P, I, case, pa = _n32()
    pat, _, _ = check_system("32 neighbours", "reference", I, _ref_system(P)(*case), *case,
                             pat_asm=pa)
    assert pat["rows"] == 32 * 33 + 6


@pytest.mark.gpu
def test_construct_32_neighbours():
    needs_ref()
    P, I, case, pa = _n32()
    ctx = _with_context(P)
    try:
        check_system("32 neighbours", "device", I, _device_system(ctx)(*case), *case,
                     pat_asm=pa)
    finally:
        ctx.close()
        P.ctx = None


# ---------------------------------------------------------------------------
# CPU: sensitivity at S = 1, S = 4096 and 32 neighbours, on reference systems
# ---------------------------------------------------------------------------

def _mutants_break(I, sysd, case, pat, p, **mutation):
    """Restates patch index p alone with the mutation (its index within that
    one-patch run is 0), puts it in place of the patch's correct restatement
    and asks whether the system then breaks the bound."""
    act, light, reg, lreg = case
    mutation = {k: (0,) + tuple(v[1:]) for k, v in mutation.items()}
    one = gp.construct_patches(I, act, light, reg, lreg, patches=pat["ids"][p:p + 1], **mutation)
    mut = dict(pat)
    for key in ("H", "He", "g", "ge"):
        mut[key] = pat[key].copy()
        mut[key][p] = one[key][0]
    return _mutant_ratio(I, sysd, gp.assemble(I, act, mut)) > 1.0


@pytest.mark.parametrize("scale", [0, 8])
def test_sensitivity_dropped_sample(scale):
    """One sample of one patch dropped, with S = 1 (the patch's only sample)
    and with S = 4096 (one of 4 S (rows + 36) summands, the largest chain
    multiplier of the bound)."""
    needs_ref()
    P, I, cases = scene(scale)
    case = cases["full"]
    pat, asm = restated((scale, "full"), I, case)
    sysd = _ref_system(P)(*case)
    assert _mutant_ratio(I, sysd, asm) <= 1.0
    S = SAMPLES[scale]
    p = len(pat["ids"]) // 2
    s = S // 2 + 3 if S > 1 else 0
    assert not _mutants_break(I, sysd, case, pat, p)         # the unmutated patch
    assert _mutants_break(I, sysd, case, pat, p, drop_sample=(p, s))


def test_sensitivity_dropped_pair_term():
    """The two rows of one neighbour pair of one sample dropped, among 496
    pairs per sample."""
    needs_ref()
    P, I, case, (pat, asm) = _n32()
    sysd = _ref_system(P)(*case)
    assert _mutant_ratio(I, sysd, asm) <= 1.0
    counts = np.diff(I.vis_off.astype(np.int64))[pat["ids"]]
    p = int(np.flatnonzero(counts == 32)[0])
    assert _mutants_break(I, sysd, case, pat, p, drop_pair=(p, 5, 11, 29))


# ---------------------------------------------------------------------------
# GPU: thinned lists and the zero pivot, mixed neighbour sizes
# ---------------------------------------------------------------------------

@pytest.mark.gpu
def test_construct_thinned_lists_and_zero_pivot():
    """Visibility lists thinned to 0..n per patch; one active node whose
    adjacent patches all have empty lists: with regularization 0 its
    diagonal block is exactly 0, so P keeps it (the zero-pivot branch)."""
    needs_ref()
    from util_scene import Pair
    P = Pair(164, 120, 2, 2, seed_index=202)
    try:
        rng = np.random.default_rng(7)
        npx, npy = P.info["npx"], P.info["npy"]
        I = gp.Inputs.from_pair(P)
        pn = I.patch_nodes()
        ns = npx + 1
        node = (npy // 2) * ns + npx // 2
        assert P.node_valid[node]
        empty = set(np.flatnonzero((pn == node).any(1)))
        off, ids = [0], []
        for p in range(npx * npy):
            lst = list(P.vis_ids[P.vis_off[p]:P.vis_off[p + 1]])
            lst = [] if p in empty else lst[:int(rng.integers(0, len(lst) + 1))]
            ids += lst
            off.append(len(ids))
        P.vis_off, P.vis_ids = np.array(off, np.uint32), np.array(ids, np.uint8)
        P.R.set_visibility(P.vis_off, P.vis_ids)
        P.push_surface()
        I = gp.Inputs.from_pair(P)
        counts = np.diff(I.vis_off.astype(np.int64))
        assert {0, 1, 2} <= set(counts[P.patch_valid.astype(bool)])
        for reg in (0.01, 0.0):
            case = (P.node_valid, None, reg, 0.0)
            pa = restate(I, *case)
            check_system(f"thinned reg {reg}", "reference", I, _ref_system(P)(*case), *case,
                         pat_asm=pa)
            gs = _device_system(P.ctx)(*case)
            _, _, kept = check_system(f"thinned reg {reg}", "device", I, gs, *case, pat_asm=pa)
        # reg 0: the node's diagonal block is 0 and P is that block
        outer = gs["Houter"].astype(np.int64)
        blk = [k for k in range(outer[node], outer[node + 1])
               if int(gs["Hinner"][k]) // 4 == node]
        assert len(blk) == 1 and not gs["Hvals"][blk[0]].any()
        prow = int(np.searchsorted(np.repeat(np.arange(len(outer) - 1),
                                             np.diff(gs["Pouter"].astype(np.int64))), node))
        assert not gs["Pvals"][prow].any() and kept >= 1
    finally:
        P.close()


@pytest.mark.gpu
def test_construct_mixed_sizes_clamped():
    """Neighbours of other sizes, each listed for every patch: some of the
    processed samples project outside a neighbour, where tap_neighbour
    clamps."""
    needs_ref()
    from util_scene import MIXED_SUBS, Pair, make_mixed_scene
    sc = make_mixed_scene(400, 300, MIXED_SUBS, seed_index=80)
    P = Pair(400, 300, sc.n_sub, 2, scene=sc)
    try:
        # every neighbour in every valid patch's list: the visibility test
        # would drop the ones a patch projects outside of
        pv = P.patch_valid.astype(bool)
        n = sc.n_sub
        P.vis_off = np.concatenate([[0], np.cumsum(np.where(pv, n, 0))]).astype(np.uint32)
        P.vis_ids = np.tile(np.arange(n, dtype=np.uint8), int(pv.sum()))
        P.R.set_visibility(P.vis_off, P.vis_ids)
        P.push_surface()
        I = gp.Inputs.from_pair(P)
        case = (P.node_valid, None, 0.01, 0.0)
        pa = restate(I, *case)
        assert 0.01 < pa[0]["clamped"] / pa[0]["taps"] < 0.9, (pa[0]["clamped"], pa[0]["taps"])
        check_system("mixed sizes", "reference", I, _ref_system(P)(*case), *case, pat_asm=pa)
        check_system("mixed sizes", "device", I, _device_system(P.ctx)(*case), *case,
                     pat_asm=pa)
    finally:
        P.close()


# ---------------------------------------------------------------------------
# GPU: K4, the node update
# ---------------------------------------------------------------------------

def _step(I, act, rng):
    """d = alpha * noise, alpha by bisection so that about half the processed
    patches have a largest reprojection difference above 0.15 px; NaN in the
    invalid nodes."""
    noise = rng.standard_normal((len(I.node_valid), 4)) * np.array([1.0, 0.05, 0.05, 0.01])
    noise *= np.abs(I.nodes[:, :1]).mean()
    # the differences grow about linearly with alpha: start from the median
    # patch at alpha = 1e-3, then bisect on the restatement
    m0 = gp.update(I, act, (1e-3 * noise).reshape(-1))["max"]
    a0 = 1e-3 * 0.15 / float(np.median(m0))

    def frac(alpha):
        return (gp.update(I, act, (alpha * noise).reshape(-1))["max"] > 0.15).mean()
    lo, hi = a0 / 8, a0 * 8
    assert frac(lo) < 0.5 < frac(hi)
    for _ in range(4):          # a factor 64 narrowed to 1.3
        mid = np.sqrt(lo * hi)
        lo, hi = (lo, mid) if frac(mid) > 0.5 else (mid, hi)
    d = hi * noise
    d[~I.node_valid.astype(bool)] = np.nan
    return d.reshape(-1)


# (scale, size): G = 1, 4, 16, 64 and PS_MAX = 256; 240x180 at scale 0 has
# 42 364 patches, more than update_reduce_kernel's 32 768 threads
UPDATE = [(0, (45, 33)), (0, (240, 180)), (1, (70, 50)), (2, (164, 120)), (3, (200, 150)),
          (7, (1300, 1060)), (8, (1300, 1060))]


@pytest.mark.gpu
@pytest.mark.parametrize("scale,size", UPDATE)
def test_update(scale, size):
    needs_ref()
    from util_scene import Pair
    P = Pair(size[0], size[1], 2, scale, seed_index=300 + scale)
    try:
        # invalid nodes: a block of nodes in the middle of the grid, and every
        # patch that touches one of them
        npx, npy = P.info["npx"], P.info["npy"]
        nv = P.node_valid.reshape(npy + 1, npx + 1).copy()
        nv[npy // 3:npy // 3 + max(1, npy // 6), npx // 3:npx // 3 + max(1, npx // 6)] = 0
        pv = P.patch_valid.reshape(npy, npx) & nv[:-1, :-1] & nv[1:, :-1] & nv[:-1, 1:] \
            & nv[1:, 1:]
        P.node_valid, P.patch_valid = nv.reshape(-1), pv.reshape(-1).astype(np.uint8)
        P.push_surface()
        I = gp.Inputs.from_pair(P)
        invalid = ~I.node_valid.astype(bool)
        assert invalid.any()
        G = min(I.ps * I.ps, 64)
        n_patches = I.npx * I.npy
        if size == (240, 180):
            assert n_patches > 32768
        if G < 16:
            assert n_patches % (64 // G) != 0
        rng = np.random.default_rng(scale)
        act = P.node_valid.copy()
        d = _step(I, act, rng)
        for full_opt in (False, True):
            ex = update_expectation(I, act, d)
            frac = ex["flag"].mean()
            assert 0.2 <= frac <= 0.8, frac
            P.ctx.set_nodes(P.nodes)
            P.ctx.gn_construct(act, None, 0.01, 0.0)
            P.ctx.set_delta(d)
            got, n, shift = P.ctx.update_nodes(full_opt=full_opt)
            check_update(I, act, d, got, n, shift, f"s{scale} {size} full_opt={full_opt}",
                         full_opt=full_opt)
            nodes = P.ctx.get_nodes()
            assert np.array_equal(nodes[~invalid], (I.nodes + d.reshape(-1, 4))[~invalid])
            assert np.array_equal(nodes[invalid], I.nodes[invalid])     # NaN steps unused
            assert np.isnan(d.reshape(-1, 4)[invalid]).all() and np.isfinite(shift)
    finally:
        P.close()

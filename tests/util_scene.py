"""Shared helpers of the parity tests: drive the compiled-verbatim reference
(oracle/_ref) and the CUDA library (through the C ABI) with identical arrays.

The oracle is used here only as the checker."""
from __future__ import annotations

import numpy as np

from smvs_b200 import api, synth
from oracle import ref as oref


def colour_scene(width, height, n_sub, seed_index, shading=False):
    """Three different channels per view (the NCC filter works on colour)."""
    import copy
    sc = synth.make_scene(width, height, n_sub, seed_index=seed_index, shading=shading)
    col = copy.copy(sc)
    rng = np.random.default_rng(seed_index)
    imgs = []
    for im in sc.images:
        f = im.astype(np.float32)
        chans = [np.clip(f * g + o + rng.normal(0, 2.0, f.shape), 0, 255)
                 for g, o in ((1.0, 0.0), (0.8, 20.0), (1.1, -10.0))]
        imgs.append(np.stack(chans, axis=2).astype(np.uint8))
    col.images = imgs
    return col


# Neighbours of a mixed scene as (width, height, flen): the smallest in both
# dimensions first, a portrait view, one between, and an odd-sized one that is
# wider and taller than the 400x300 main view. Widths 256, 352 take the TMA
# set_scale (row pitch a multiple of 16 bytes), 300 and 417 the three kernels.
MIXED_SUBS = ((256, 192, 1.3), (300, 400, 1.0), (352, 264, 1.15), (417, 311, 0.85))


def make_mixed_scene(width, height, subs, seed_index=0, main_flen=1.0,
                     init_noise=0.02, shading=False):
    """synth.make_scene with neighbours of their own size and focal length:
    neighbour k is rendered at subs[k] = (w_k, h_k, flen_k) with its own
    calibration K_k, through M_k = K_k R_k K_0^-1 and t_k = K_k t_k. The
    returned synth.Scene holds per-view image shapes and per-view flen."""
    import concurrent.futures
    seed = synth.BASE_SEED + int(seed_index)
    rng = np.random.default_rng(seed)
    n_sub = len(subs)
    rot, trans = synth.make_cameras(n_sub)
    flen = np.array([main_flen] + [f for _, _, f in subs], dtype=np.float32)
    K0inv = np.linalg.inv(synth.calibration(float(flen[0]), width, height))
    depth = synth.DepthField(width, height)
    tex = synth.Texture(width, rng)
    pert = synth.Perturbation(width, height, rng, amp=init_noise)
    f_px = float(flen[0]) * max(width, height)

    def radiance(u, v):
        val = tex(u, v)
        if shading:
            n = synth._surface_normal(u, v, depth, width, height, f_px)
            val = val * (synth.sh_basis(n) @ synth.SH_LIGHT) / 1.9
        return np.clip(np.rint(255.0 * val), 0, 255).astype(np.uint8)

    def render(k):
        w, h = (width, height) if k == 0 else subs[k - 1][:2]
        ys, xs = np.mgrid[0:h, 0:w]
        pu, pv = xs.astype(np.float64) + 0.5, ys.astype(np.float64) + 0.5
        if k == 0:
            return radiance(pu, pv)
        K = synth.calibration(float(flen[k]), w, h)
        M = K @ rot[k].astype(np.float64).reshape(3, 3) @ K0inv
        t = K @ trans[k].astype(np.float64)
        return radiance(*synth._invert_warp(M, t, depth, pu, pv))

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, 1 + n_sub)) as ex:
        images = list(ex.map(render, range(1 + n_sub)))
    ys, xs = np.mgrid[0:height, 0:width]
    pu, pv = xs.astype(np.float64) + 0.5, ys.astype(np.float64) + 0.5
    sc = synth.Scene(width, height, n_sub, flen, rot, trans, images,
                     depth(pu, pv).astype(np.float32),
                     (depth(pu, pv) * pert(pu, pv)).astype(np.float32), seed, shading)
    sc._depth_fn = depth
    sc._pert_fn = pert
    return sc


class Pair:
    """Reference scene + (optionally) a GPU context fed with the reference's
    own prepared arrays at one scale."""

    def __init__(self, width, height, n_sub, scale, seed_index=0, shading=False,
                 gpu=True, init_noise=0.02, scene=None):
        self.scene = scene if scene is not None else synth.make_scene(
            width, height, n_sub, seed_index=seed_index, shading=shading,
            init_noise=init_noise)
        self.R = oref.RefScene(self.scene, init_linear=shading)
        self.scale = scale
        self.R.set_scale(scale)
        if scale == 0:
            # a scale-0 surface only ever arises by subdividing a scale-1 one
            # (initialize_node_from_depth has an empty window at patch size 1)
            self.R.surface_create(1, self.scene.init_depth)
            self.R.surface_subdivide()
        else:
            self.R.surface_create(scale, self.scene.init_depth)
        self.R.compute_visibility()
        self.info = self.R.surface_info()
        self.nodes, self.node_valid, self.patch_valid = self.R.surface_get()
        self.vis_off, self.vis_ids = self.R.get_visibility()
        self.Mi, self.ti = self.R.Mt()
        self.ctx = None
        if gpu:
            self.ctx = api.Context(0)
            self.push_views()
            self.push_surface()

    def push_views(self):
        R, n = self.R, self.scene.n_sub
        sh_img, sh_grad = R.shading() if self.scene.shading else (None, None)
        self.ctx.set_views(R.gradients(0),
                           [R.gradients(k + 1) for k in range(n)],
                           [R.hessian(k + 1) for k in range(n)],
                           self.Mi, self.ti, R.flen(0), R.inverse_flen(0),
                           sh_img, sh_grad)

    def push_surface(self, nodes=None):
        i = self.info
        self.ctx.set_surface(i["scale"], i["npx"], i["npy"], i["start_x"],
                             i["start_y"], self.nodes if nodes is None else nodes,
                             self.node_valid, self.patch_valid, self.vis_off,
                             self.vis_ids)

    def close(self):
        if self.ctx is not None:
            self.ctx.close()
        self.R.close()


def bsc_to_dict(sysd):
    """{(block_row, block_col): 4x4} from the reference BSC arrays."""
    out = {}
    outer, inner, vals = sysd["Houter"], sysd["Hinner"], sysd["Hvals"]
    for col in range(len(outer) - 1):
        for k in range(int(outer[col]), int(outer[col + 1])):
            out[(int(inner[k]) // 4, col)] = vals[k].reshape(4, 4)
    return out


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))

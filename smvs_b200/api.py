"""ctypes host-side mirror of include/smvs_b200.h.

Python plumbing for the tests and the benchmark: it calls the C ABI of
smvs_b200/libsmvs_b200.so (hand-written sm_90a kernels) with numpy host
buffers, exactly as the patched reference C++ would (INTEGRATION.md).
There is no fallback: a missing library or a missing GPU raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsmvs_b200.so")

EXPORTS = [
    "smvsb_create", "smvsb_destroy", "smvsb_last_error", "smvsb_version",
    "smvsb_launch_count", "smvsb_global_launch_count", "smvsb_set_views",
    "smvsb_set_views_u8", "smvsb_debug_get_view", "smvsb_set_surface",
    "smvsb_set_nodes", "smvsb_gn_construct", "smvsb_cg_solve",
    "smvsb_get_delta", "smvsb_set_delta", "smvsb_update_nodes",
    "smvsb_newton_loop", "smvsb_get_nodes", "smvsb_get_depth",
    "smvsb_get_normals", "smvsb_debug_get_system", "smvsb_debug_spmv",
    "smvsb_fit_lighting", "smvsb_sgm", "smvsb_visibility",
    "smvsb_cut_boundaries", "smvsb_get_surface_state", "smvsb_view_set_scale",
    "smvsb_bilateral_filter", "smvsb_debug_expf", "smvsb_device_count", "smvsb_cut_depth_maps", "smvsb_surface_create", "smvsb_surface_subdivide",
    "smvsb_surface_fill_from_depth", "smvsb_surface_remove_isolated", "smvsb_surface_expand", "smvsb_surface_info",
    "smvsb_set_color_images",
    "smvsb_optimize", "smvsb_optimize_rgb_f32", "smvsb_view_set_scale_c", "smvsb_measure_fp64_peak", "smvsb_sgm_reconstruct", "smvsb_newton_loop_batch", "smvsb_device_launch_count",
    "smvsb_cut_depth_maps_multi", "smvsb_sgm_ex", "smvsb_sgm_reconstruct_ex",
]


class SmvsbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"smvs_b200 error {code}: {msg}")
        self.code = code


class NewtonStats(C.Structure):
    _fields_ = [("newton_steps", C.c_int32), ("cg_iterations", C.c_int32),
                ("nan_break", C.c_int32), ("reserved", C.c_int32),
                ("n_active", C.c_uint64), ("pixel_iterations", C.c_double),
                ("ms_construct", C.c_double), ("ms_solve", C.c_double),
                ("ms_update", C.c_double), ("ms_total", C.c_double),
                ("cg_block_iterations", C.c_double), ("cg_row_iterations", C.c_double)]


_lib = None


def lib():
    """Loads libsmvs_b200.so; raises if it was not built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SmvsbError(-100, f"{LIB_PATH} missing: run "
                             "`python -m smvs_b200.build` (or __graft_entry__.build())")
        L = C.CDLL(LIB_PATH)
        L.smvsb_last_error.restype = C.c_char_p
        L.smvsb_last_error.argtypes = [C.c_void_p]
        L.smvsb_version.restype = C.c_char_p
        L.smvsb_launch_count.restype = C.c_uint64
        L.smvsb_launch_count.argtypes = [C.c_void_p]
        L.smvsb_global_launch_count.restype = C.c_uint64
        L.smvsb_device_launch_count.restype = C.c_uint64
        L.smvsb_device_launch_count.argtypes = [C.c_int]
        L.smvsb_destroy.argtypes = [C.c_void_p]
        L.smvsb_destroy.restype = None
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


def _u8(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.uint8)


class Context:
    """One smvsb_ctx: device memory + stream of one reference view."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        rc = lib().smvsb_create(int(device), C.byref(self._h))
        if rc != 0:
            raise SmvsbError(rc, lib().smvsb_last_error(None).decode())
        self.device = device
        self.n_nodes = 0
        self.n_patches = 0
        self.w = self.h = 0

    def close(self):
        if self._h:
            lib().smvsb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, rc):
        if rc != 0:
            raise SmvsbError(rc, lib().smvsb_last_error(self._h).decode())

    @property
    def launches(self):
        return int(lib().smvsb_launch_count(self._h))

    # -- inputs ----------------------------------------------------------
    def set_views(self, main_grad, sub_grads, sub_hess, Mi, ti, flen_px,
                  inv_flen, main_shading=None, main_shading_grad=None):
        main_grad = _f32(main_grad)
        h, w = main_grad.shape[:2]
        n = len(sub_grads)
        sg = [_f32(a) for a in sub_grads]
        sh = [_f32(a) for a in sub_hess]
        sw = (C.c_int * max(n, 1))(*[a.shape[1] for a in sg])
        shh = (C.c_int * max(n, 1))(*[a.shape[0] for a in sg])
        gp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in sg])
        hp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in sh])
        Mi = _f64(Mi)
        ti = _f64(ti)
        ms, msg = _f32(main_shading), _f32(main_shading_grad)
        self._check(lib().smvsb_set_views(
            self._h, w, h, C.c_double(flen_px), C.c_double(inv_flen), _p(main_grad),
            _p(ms), _p(msg), n, sw, shh, gp, hp, _p(Mi), _p(ti)))
        self.w, self.h = w, h

    def set_views_u8(self, scale, main_img, sub_imgs, Mi, ti, flen_px, inv_flen,
                     with_shading=False):
        """StereoView::set_scale on the device from the byte images."""
        main_img = _u8(main_img)
        h, w = main_img.shape
        n = len(sub_imgs)
        si = [_u8(a) for a in sub_imgs]
        sw = (C.c_int * max(n, 1))(*[a.shape[1] for a in si])
        shh = (C.c_int * max(n, 1))(*[a.shape[0] for a in si])
        ip = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in si])
        Mi, ti = _f64(Mi), _f64(ti)
        self._check(lib().smvsb_set_views_u8(
            self._h, int(scale), w, h, C.c_double(flen_px), C.c_double(inv_flen),
            _p(main_img), int(with_shading), n, sw, shh, ip, _p(Mi), _p(ti)))
        self.w, self.h = w, h
        self._sub_shapes = [a.shape for a in si]

    def debug_get_view(self, view):
        if view == 0:
            g = np.empty((self.h, self.w, 2), dtype=np.float32)
            self._check(lib().smvsb_debug_get_view(self._h, 0, _p(g), None))
            return g, None
        hh, ww = self._sub_shapes[view - 1]
        g = np.empty((hh, ww, 2), dtype=np.float32)
        hs = np.empty((hh, ww, 3), dtype=np.float32)
        self._check(lib().smvsb_debug_get_view(self._h, int(view), _p(g), _p(hs)))
        return g, hs

    def set_surface(self, scale, npx, npy, start_x, start_y, nodes, node_valid,
                    patch_valid, vis_off, vis_ids):
        nodes = _f64(nodes)
        nv, pv = _u8(node_valid), _u8(patch_valid)
        if vis_off is None:
            vo, vi = None, None          # no lists yet: smvsb_visibility makes them
        else:
            vo = np.ascontiguousarray(vis_off, dtype=np.uint32)
            vi = _u8(vis_ids)
            if vi.size == 0:
                vi = np.zeros(1, dtype=np.uint8)
        self._check(lib().smvsb_set_surface(
            self._h, int(scale), int(npx), int(npy), int(start_x), int(start_y),
            _p(nodes), _p(nv), _p(pv), _p(vo), _p(vi)))
        self.n_nodes = (npx + 1) * (npy + 1)
        self.n_patches = npx * npy

    def view_set_scale(self, image, scale):
        """StereoView::set_scale of one float image, (h, w) single channel or
        (h, w, 3) colour: (scaleimage, gradients, hessian) as host arrays."""
        img = np.ascontiguousarray(image, dtype=np.float32)
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else img.shape[2]
        blur = np.empty(img.shape, dtype=np.float32)
        grad = np.empty((h, w, 2), dtype=np.float32)
        hess = np.empty((h, w, 3), dtype=np.float32)
        self._check(lib().smvsb_view_set_scale_c(self._h, w, h, ch, _p(img), int(scale),
                                                 _p(blur), _p(grad), _p(hess)))
        return blur, grad, hess

    def bilateral_filter(self, guide, depth, sigma=5.0, kernel_size=5):
        """DepthOptimizer::depthmap_bilateral_filter: guide (h, w[, C]) float
        image, depth (dm_h, dm_w) -> filtered (h, w) depth."""
        g = np.ascontiguousarray(guide, dtype=np.float32)
        d = np.ascontiguousarray(depth, dtype=np.float32)
        h, w = g.shape[:2]
        ch = 1 if g.ndim == 2 else g.shape[2]
        out = np.empty((h, w), dtype=np.float32)
        self._check(lib().smvsb_bilateral_filter(
            self._h, w, h, ch, _p(g), d.shape[1], d.shape[0], _p(d),
            C.c_float(sigma), int(kernel_size), _p(out)))
        return out

    # -- visibility / boundary cutting --------------------------------------
    def set_color_images(self, main_rgb, sub_rgbs):
        """StereoView::get_image() of every view at the current scale
        ((h, w, 3) floats) for the use_sgm = false visibility."""
        m = _f32(main_rgb)
        subs = [_f32(a) for a in sub_rgbs]
        assert m.shape == (self.h, self.w, 3)
        ptrs = (C.c_void_p * max(len(subs), 1))(*[a.ctypes.data for a in subs])
        self._check(lib().smvsb_set_color_images(self._h, _p(m), len(subs), ptrs))

    def visibility(self, sgm_depth):
        """DepthOptimizer::create_subview_surfaces on the context's surface;
        sgm_depth None = the use_sgm = false mode (needs set_color_images).
        Returns the number of patches it deleted."""
        d = None if sgm_depth is None else np.ascontiguousarray(sgm_depth, dtype=np.float32)
        removed = C.c_uint64(0)
        self._check(lib().smvsb_visibility(self._h, _p(d), C.byref(removed)))
        return removed.value

    def cut_boundaries(self, inv_calib9):
        """One DepthOptimizer::cut_boundaries(); returns the patches deleted."""
        k = np.ascontiguousarray(inv_calib9, dtype=np.float32).reshape(9)
        deleted = C.c_int(0)
        self._check(lib().smvsb_cut_boundaries(self._h, _p(k), C.byref(deleted)))
        return deleted.value

    def surface_state(self):
        """(node_valid, patch_valid, vis_off, vis_ids) as the context holds them."""
        nv = np.empty(self.n_nodes, dtype=np.uint8)
        pv = np.empty(self.n_patches, dtype=np.uint8)
        vo = np.empty(self.n_patches + 1, dtype=np.uint32)
        cap = self.n_patches * 32 + 1
        vi = np.empty(cap, dtype=np.uint8)
        self._check(lib().smvsb_get_surface_state(self._h, _p(nv), _p(pv), _p(vo), _p(vi),
                                                  C.c_uint64(cap)))
        return nv, pv, vo, vi[:vo[-1]].copy()

    # -- surface topology on the device ---------------------------------------
    def _sync_surface_info(self):
        info = (C.c_int * 6)()
        self._check(lib().smvsb_surface_info(self._h, info))
        self.n_nodes = (info[1] + 1) * (info[2] + 1)
        self.n_patches = info[1] * info[2]
        return dict(scale=info[0], npx=info[1], npy=info[2], start_x=info[3],
                    start_y=info[4], patchsize=info[5])

    def surface_info(self):
        return self._sync_surface_info()

    def surface_create(self, scale, init_depth):
        """Surface::create(bundle, view, scale, init_depth) on the device."""
        d = np.ascontiguousarray(init_depth, dtype=np.float32)
        self._check(lib().smvsb_surface_create(self._h, int(scale), _p(d)))
        return self._sync_surface_info()

    def surface_subdivide(self):
        self._check(lib().smvsb_surface_subdivide(self._h))
        return self._sync_surface_info()

    def surface_fill_from_depth(self, init_depth=None):
        d = None if init_depth is None else np.ascontiguousarray(init_depth, dtype=np.float32)
        self._check(lib().smvsb_surface_fill_from_depth(self._h, _p(d)))

    def surface_remove_isolated(self):
        self._check(lib().smvsb_surface_remove_isolated(self._h))

    def surface_expand(self):
        """Surface::expand; returns the patches it created."""
        filled = C.c_int(0)
        self._check(lib().smvsb_surface_expand(self._h, C.byref(filled)))
        return filled.value

    def set_nodes(self, nodes):
        nodes = _f64(nodes)
        self._check(lib().smvsb_set_nodes(self._h, _p(nodes)))

    # -- Gauss-Newton ----------------------------------------------------
    def gn_construct(self, active=None, light16=None, regularization=0.01,
                     light_surf_regularization=0.0):
        a, l = _u8(active), _f64(light16)
        self._check(lib().smvsb_gn_construct(
            self._h, _p(a), _p(l), C.c_double(regularization),
            C.c_double(light_surf_regularization)))

    def cg_solve(self, max_iter=200, err_tol=-1.0, q_tol=1e-3):
        it, info = C.c_int(0), C.c_int(0)
        self._check(lib().smvsb_cg_solve(self._h, int(max_iter), C.c_double(err_tol),
                                         C.c_double(q_tol), C.byref(it), C.byref(info)))
        return it.value, info.value

    def get_delta(self):
        x = np.empty(self.n_nodes * 4, dtype=np.float64)
        self._check(lib().smvsb_get_delta(self._h, _p(x)))
        return x

    def set_delta(self, delta):
        d = _f64(delta)
        self._check(lib().smvsb_set_delta(self._h, _p(d)))

    def update_nodes(self, reproj_thresh=0.15, full_opt=False):
        act = np.empty(self.n_nodes, dtype=np.uint8)
        n_active, shift = C.c_uint64(0), C.c_double(0)
        self._check(lib().smvsb_update_nodes(
            self._h, C.c_double(reproj_thresh), int(full_opt), _p(act),
            C.byref(n_active), C.byref(shift)))
        return act, int(n_active.value), float(shift.value)

    def newton_loop(self, light16=None, regularization=0.01,
                    light_surf_regularization=0.0, max_steps=200, full_opt=False):
        l = _f64(light16)
        st = NewtonStats()
        self._check(lib().smvsb_newton_loop(
            self._h, _p(l), C.c_double(regularization),
            C.c_double(light_surf_regularization), int(max_steps), int(full_opt),
            C.byref(st)))
        return dict(newton_steps=st.newton_steps, cg_iterations=st.cg_iterations,
                    nan=bool(st.nan_break), n_active=int(st.n_active),
                    pixel_iterations=float(st.pixel_iterations),
                    ms_construct=st.ms_construct, ms_solve=st.ms_solve,
                    ms_update=st.ms_update, ms_total=st.ms_total,
                    cg_block_iterations=st.cg_block_iterations,
                    cg_row_iterations=st.cg_row_iterations)

    # -- outputs ---------------------------------------------------------
    def get_nodes(self, out=None):
        """Node parameters (n_nodes, 4). `out`: a caller-owned C-contiguous
        float64 array to read into (e.g. page-locked memory, so that the
        device-to-host copy is one DMA transfer)."""
        if out is None:
            out = np.empty((self.n_nodes, 4), dtype=np.float64)
        else:
            if (out.dtype != np.float64 or not out.flags.c_contiguous
                    or out.size != self.n_nodes * 4):
                raise ValueError("out must be C-contiguous float64 with n_nodes * 4 entries")
        self._check(lib().smvsb_get_nodes(self._h, _p(out)))
        return out

    def get_depth(self):
        out = np.empty((self.h, self.w), dtype=np.float32)
        self._check(lib().smvsb_get_depth(self._h, _p(out)))
        return out

    def get_normals(self):
        out = np.empty((self.h, self.w, 3), dtype=np.float32)
        self._check(lib().smvsb_get_normals(self._h, _p(out)))
        return out

    def debug_get_system(self):
        nh, npc = C.c_uint64(0), C.c_uint64(0)
        self._check(lib().smvsb_debug_get_system(
            self._h, None, None, None, None, C.byref(nh), None, None, None,
            C.byref(npc)))
        n = self.n_nodes
        g = np.empty(n * 4, dtype=np.float64)
        Hv = np.empty((int(nh.value), 16), dtype=np.float64)
        Ho = np.empty(n + 1, dtype=np.uint64)
        Hi = np.empty(int(nh.value), dtype=np.uint64)
        Pv = np.empty((int(npc.value), 16), dtype=np.float64)
        Po = np.empty(n + 1, dtype=np.uint64)
        Pi = np.empty(int(npc.value), dtype=np.uint64)
        self._check(lib().smvsb_debug_get_system(
            self._h, _p(g), _p(Hv), _p(Ho), _p(Hi), C.byref(nh), _p(Pv), _p(Po),
            _p(Pi), C.byref(npc)))
        return dict(g=g, Hvals=Hv, Houter=Ho, Hinner=Hi, Pvals=Pv, Pouter=Po, Pinner=Pi)

    def debug_spmv(self, x):
        x = _f64(x)
        y = np.empty_like(x)
        self._check(lib().smvsb_debug_spmv(self._h, _p(x), _p(y)))
        return y

    def fit_lighting(self, nccl_comm=None):
        out = np.zeros(16, dtype=np.float64)
        comm = C.c_void_p(nccl_comm) if nccl_comm else None
        self._check(lib().smvsb_fit_lighting(self._h, _p(out), comm))
        return out


def _stats_dict(st):
    return dict(newton_steps=st.newton_steps, cg_iterations=st.cg_iterations,
                nan=bool(st.nan_break), n_active=int(st.n_active),
                pixel_iterations=float(st.pixel_iterations),
                ms_construct=st.ms_construct, ms_solve=st.ms_solve,
                ms_update=st.ms_update, ms_total=st.ms_total,
                cg_block_iterations=st.cg_block_iterations,
                cg_row_iterations=st.cg_row_iterations)


def newton_loop_batch(ctxs, lights=None, regularization=0.01,
                      light_surf_regularization=0.0, max_steps=200, full_opt=False):
    """smvsb_newton_loop_batch: the inner Newton loops of several contexts of
    one device in lock-step (one PCG launch per step for all of them).
    Returns one stats dict per context; the ms_* fields are the batch's."""
    n = len(ctxs)
    handles = (C.c_void_p * n)(*[c._h for c in ctxs])
    keep, lp = [], None
    if lights is not None and any(l is not None for l in lights):
        keep = [None if l is None else _f64(l) for l in lights]
        lp = (C.c_void_p * n)(*[None if l is None else l.ctypes.data for l in keep])
    st = (NewtonStats * n)()
    rc = lib().smvsb_newton_loop_batch(handles, n, lp, C.c_double(regularization),
                                       C.c_double(light_surf_regularization),
                                       int(max_steps), int(full_opt), st)
    if rc != 0:
        raise SmvsbError(rc, lib().smvsb_last_error(ctxs[0]._h).decode())
    return [_stats_dict(s) for s in st]


class SgmOptions(C.Structure):
    _fields_ = [("device_bytes", C.c_uint64), ("reserved", C.c_uint64 * 3)]


class SgmStats(C.Structure):
    _fields_ = [("banded", C.c_int32), ("bands", C.c_int32),
                ("peak_device_bytes", C.c_uint64), ("host_bytes", C.c_uint64),
                ("ms_device", C.c_double)]


def _sgm_ex_args(device_bytes):
    """The stats and the (options, stats) arguments of smvsb_sgm_ex /
    smvsb_sgm_reconstruct_ex."""
    st = SgmStats()
    return st, (C.byref(SgmOptions(int(device_bytes))), C.byref(st))


def _sgm_stats(st):
    return {f: getattr(st, f) for f, _ in SgmStats._fields_}


def sgm(main_lum, neigh_lum, M, t, min_depth, max_depth, num_steps=128,
        penalty1=6, penalty2=96, device=0, volumes=False, *, device_bytes=0,
        return_stats=False):
    """SGMStereo::run_sgm for one luminance pair (smvsb_sgm).
    device_bytes (a cap on the device's SGM workspace; 0 = the default budget)
    or return_stats select smvsb_sgm_ex; with return_stats the result is
    (dict, stats dict)."""
    main_lum, neigh_lum = _u8(main_lum), _u8(neigh_lum)
    h, w = main_lum.shape
    nh, nw = neigh_lum.shape
    M, t = _f32(M), _f32(t)
    depth = np.empty((h, w), dtype=np.float32)
    cost = np.empty((h, w, num_steps), dtype=np.uint16) if volumes else None
    S = np.empty((h, w, num_steps), dtype=np.uint16) if volumes else None
    ms = np.zeros(3, dtype=np.float64)
    args = (int(device), w, h, _p(main_lum), nw, nh, _p(neigh_lum),
            _p(M), _p(t), C.c_float(min_depth), C.c_float(max_depth),
            int(num_steps), C.c_uint16(penalty1), C.c_uint16(penalty2),
            _p(depth), _p(cost), _p(S), _p(ms))
    if not device_bytes and not return_stats:
        rc = lib().smvsb_sgm(*args)
    else:
        st, ex = _sgm_ex_args(device_bytes)
        rc = lib().smvsb_sgm_ex(*args, *ex)
    if rc != 0:
        raise SmvsbError(rc, lib().smvsb_last_error(None).decode())
    out = dict(depth=depth, cost=cost, sgm=S, ms=ms)
    return (out, _sgm_stats(st)) if return_stats else out


def sgm_reconstruct(main_lum, neigh_lum, M_mn, t_mn, M_nm, t_nm, range_main, range_neigh,
                    num_steps=128, penalty1=6, penalty2=96, merge_with=None, device=0, *,
                    device_bytes=0, return_stats=False):
    """SGMStereo::reconstruct for one luminance pair (smvsb_sgm_reconstruct):
    both directions, consistency check and optional merge on the device.
    device_bytes or return_stats select smvsb_sgm_reconstruct_ex, as in sgm()."""
    main_lum, neigh_lum = _u8(main_lum), _u8(neigh_lum)
    h, w = main_lum.shape
    nh, nw = neigh_lum.shape
    arrs = [_f32(a) for a in (M_mn, t_mn, M_nm, t_nm, range_main, range_neigh)]
    prev = _f32(merge_with)
    depth = np.empty((h, w), dtype=np.float32)
    ms = np.zeros(2, dtype=np.float64)
    args = (int(device), w, h, _p(main_lum), nw, nh, _p(neigh_lum), *[_p(a) for a in arrs],
            int(num_steps), C.c_uint16(penalty1), C.c_uint16(penalty2), _p(prev), _p(depth),
            _p(ms))
    if not device_bytes and not return_stats:
        rc = lib().smvsb_sgm_reconstruct(*args)
    else:
        st, ex = _sgm_ex_args(device_bytes)
        rc = lib().smvsb_sgm_reconstruct_ex(*args, *ex)
    if rc != 0:
        raise SmvsbError(rc, lib().smvsb_last_error(None).decode())
    out = dict(depth=depth, ms=ms)
    return (out, _sgm_stats(st)) if return_stats else out


def measure_fp64_peak(device=0):
    """Measured dense fp64 FMA throughput in TFLOP/s (smvsb_measure_fp64_peak)."""
    out = C.c_double(0)
    rc = lib().smvsb_measure_fp64_peak(int(device), C.byref(out))
    if rc != 0:
        raise SmvsbError(rc, lib().smvsb_last_error(None).decode())
    return float(out.value)


class OptimizeOptions(C.Structure):
    _fields_ = [("regularization", C.c_double), ("light_surf_regularization", C.c_double),
                ("num_iterations", C.c_int32), ("min_scale", C.c_int32),
                ("use_shading", C.c_int32), ("full_optimization", C.c_int32),
                ("no_sgm", C.c_int32), ("reserved", C.c_int32)]


class OptimizeStats(C.Structure):
    _fields_ = [("scales", C.c_int32), ("final_scale", C.c_int32),
                ("newton_loops", C.c_int32), ("newton_steps", C.c_int32),
                ("cg_iterations", C.c_int32), ("reserved", C.c_int32),
                ("patches", C.c_uint64), ("pixel_iterations", C.c_double),
                ("ms_newton", C.c_double)]


def optimize(ctx, main_img, sub_imgs, Mi, ti, flen_px, inv_flen, inv_calib9, sgm_depth,
             regularization=0.01, num_iterations=5, min_scale=2, shading=None,
             shading_grad=None, light_surf_regularization=0.0, full_optimization=False,
             use_sgm=True):
    """smvsb_optimize / smvsb_optimize_rgb_f32: DepthOptimizer::optimize() of
    one view, resident on the device. Images: (h, w) bytes, or (h, w, 3) float
    RGB in [0, 1] for colour views. use_sgm=False (colour views only): sgm_depth
    is the sparse initial depth of the bundle's features, (h, w). Returns (depth,
    normals, light16, stats dict)."""
    colour = np.asarray(main_img).ndim == 3
    conv = _f32 if colour else _u8          # colour: float RGB as get_image() holds it
    main_img = conv(main_img)
    h, w = main_img.shape[:2]
    n = len(sub_imgs)
    si = [conv(a) for a in sub_imgs]
    sw = (C.c_int * n)(*[a.shape[1] for a in si])
    shh = (C.c_int * n)(*[a.shape[0] for a in si])
    ip = (C.c_void_p * n)(*[a.ctypes.data for a in si])
    Mi, ti = _f64(Mi), _f64(ti)
    k = _f32(inv_calib9).reshape(9)
    sgm = _f32(sgm_depth)
    sh, shg = _f32(shading), _f32(shading_grad)
    opts = OptimizeOptions(regularization, light_surf_regularization, num_iterations,
                           min_scale, int(shading is not None), int(full_optimization),
                           int(not use_sgm), 0)
    depth = np.empty((h, w), dtype=np.float32)
    normals = np.empty((h, w, 3), dtype=np.float32)
    light = np.zeros(16, dtype=np.float64)
    st = OptimizeStats()
    fn = lib().smvsb_optimize_rgb_f32 if colour else lib().smvsb_optimize
    ctx._check(fn(
        ctx._h, w, h, C.c_double(flen_px), C.c_double(inv_flen), _p(k), _p(main_img), n,
        sw, shh, ip, _p(Mi), _p(ti), _p(sh), _p(shg), sgm.shape[1], sgm.shape[0], _p(sgm),
        C.byref(opts), _p(depth), _p(normals), _p(light), C.byref(st)))
    ctx.w, ctx.h = w, h
    ctx._sync_surface_info()
    stats = {f: getattr(st, f) for f, _ in OptimizeStats._fields_ if f != "reserved"}
    return depth, normals, light, stats


class CutOptions(C.Structure):
    _fields_ = [("devices", C.POINTER(C.c_int)), ("n_devices", C.c_int32),
                ("reserved0", C.c_int32), ("device_bytes", C.c_uint64),
                ("reserved", C.c_uint64 * 2)]


class CutStats(C.Structure):
    _fields_ = [("reference_pairs", C.c_uint64), ("evaluated_pairs", C.c_uint64),
                ("bytes_uploaded", C.c_uint64), ("target_groups", C.c_int32),
                ("source_chunks", C.c_int32), ("ms_device", C.c_double)]


def cut_depth_maps(depths, normals, invproj, cam_to_world, KR, t, device=0, *,
                   devices=None, device_bytes=0, return_stats=False):
    """smvsb_cut_depth_maps: lists of (h, w) depth maps (MVE convention) and
    (h, w, 3) world-space normal maps, per-view matrices as (n, 9) / (n, 16) /
    (n, 9) / (n, 3) float arrays -> list of cut depth maps.
    devices (a list of ids, one worker each, repeats allowed), device_bytes (a
    per-device memory cap) or return_stats select smvsb_cut_depth_maps_multi;
    with return_stats the result is (maps, stats dict)."""
    n = len(depths)
    d = [_f32(a) for a in depths]
    nr = [_f32(a) for a in normals]
    outs = [np.empty_like(a) for a in d]
    w = (C.c_int * n)(*[a.shape[1] for a in d])
    h = (C.c_int * n)(*[a.shape[0] for a in d])
    dp = (C.c_void_p * n)(*[a.ctypes.data for a in d])
    npp = (C.c_void_p * n)(*[a.ctypes.data for a in nr])
    op = (C.c_void_p * n)(*[a.ctypes.data for a in outs])
    m = [_f32(a).reshape(-1) for a in (invproj, cam_to_world, KR, t)]
    args = (n, w, h, dp, npp, _p(m[0]), _p(m[1]), _p(m[2]), _p(m[3]), op)
    if devices is None and not device_bytes and not return_stats:
        rc = lib().smvsb_cut_depth_maps(int(device), *args)
        if rc != 0:
            raise SmvsbError(rc, lib().smvsb_last_error(None).decode())
        return outs
    devs = [int(device)] if devices is None else [int(x) for x in devices]
    dv = (C.c_int * max(len(devs), 1))(*devs)
    opts = CutOptions(dv, len(devs), 0, int(device_bytes))
    st = CutStats()
    rc = lib().smvsb_cut_depth_maps_multi(C.byref(opts), *args, C.byref(st))
    if rc != 0:
        raise SmvsbError(rc, lib().smvsb_last_error(None).decode())
    if not return_stats:
        return outs
    return outs, {f: getattr(st, f) for f, _ in CutStats._fields_}

"""ctypes front-end of the CPU oracle (oracle/glic_oracle.c).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  gaussian_lic_b200/ must never import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def build(force=False):
    """Compile both oracle variants with the committed Makefile (gcc only, no GPU needed)."""
    libs = [os.path.join(HERE, "libglic_oracle_f32.so"), os.path.join(HERE, "libglic_oracle_f64.so")]
    src = os.path.join(HERE, "glic_oracle.c")
    stale = force or any((not os.path.isfile(l)) or os.path.getmtime(l) < os.path.getmtime(src) for l in libs)
    if stale:
        subprocess.check_call(["make", "-C", HERE, "-s", "-B"], stdout=subprocess.DEVNULL)
    return libs


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Oracle:
    """dtype float32 = bit-pattern-faithful restatement, float64 = finite-difference variant."""

    def __init__(self, dtype=np.float32):
        build()
        self.dtype = np.dtype(dtype)
        name = "libglic_oracle_f32.so" if self.dtype == np.float32 else "libglic_oracle_f64.so"
        self.lib = C.CDLL(os.path.join(HERE, name))
        self.real = C.c_float if self.dtype == np.float32 else C.c_double
        assert self.lib.glic_oracle_real_bytes() == self.dtype.itemsize
        self.lib.glic_oracle_forward.restype = C.c_void_p
        self.lib.glic_oracle_loss.restype = C.c_double
        self.lib.glic_oracle_emit_keys.restype = C.c_int64
        self.lib.glic_oracle_higher_msb.restype = C.c_uint32
        self.lib.glic_oracle_ranges.restype = C.c_uint32

    def set_threads(self, n):
        """Override OMP_NUM_THREADS (torchrun exports 1) for the timed CPU legs."""
        self.lib.glic_oracle_set_threads(C.c_int(int(n)))

    def max_threads(self):
        return int(self.lib.glic_oracle_max_threads())

    def _a(self, x, shape=None):
        a = np.ascontiguousarray(np.asarray(x, dtype=self.dtype))
        if shape is not None:
            a = a.reshape(shape)
        return a

    # ---- camera (A.1) -------------------------------------------------------------------
    def camera(self, W, H, fx, fy, cx, cy, R_wc=None, t_wc=None):
        R_wc = np.eye(3) if R_wc is None else np.asarray(R_wc, dtype=np.float64)
        t_wc = np.zeros(3) if t_wc is None else np.asarray(t_wc, dtype=np.float64)
        R_wc = np.ascontiguousarray(R_wc)
        t_wc = np.ascontiguousarray(t_wc)
        view = np.zeros(16, np.float32)
        proj = np.zeros(16, np.float32)
        campos = np.zeros(3, np.float32)
        tanfov = np.zeros(2, np.float32)
        lims = np.zeros(4, np.float32)
        self.lib.glic_oracle_camera(C.c_int(W), C.c_int(H), C.c_double(fx), C.c_double(fy), C.c_double(cx),
                                    C.c_double(cy), _ptr(R_wc), _ptr(t_wc), _ptr(view), _ptr(proj), _ptr(campos),
                                    _ptr(tanfov), _ptr(lims))
        return dict(W=W, H=H, view=view, proj=proj, campos=campos, tanfovx=float(tanfov[0]), tanfovy=float(tanfov[1]),
                    lims=lims)

    # ---- forward / backward of the boundary functions -------------------------------------
    def forward(self, g, cam, no_color=False, scale_modifier=1.0):
        """g: dict(means[P,3], scales[P,3] (activated), rots[P,4] (normalised), opacity[P] (activated),
        dc[P,3], sh[P,M,3], degree).  Returns dict with outputs + opaque state."""
        P = int(g["means"].shape[0])
        M = int(g["sh"].shape[1]) if g["sh"].size else 0
        W, H = cam["W"], cam["H"]
        a = {k: self._a(g[k]) for k in ("means", "scales", "rots", "opacity", "dc", "sh")}
        view, proj, campos, lims = (self._a(cam[k]) for k in ("view", "proj", "campos", "lims"))
        color = np.zeros((3, H, W), self.dtype)
        final_T = np.zeros((H, W), self.dtype)
        radii = np.zeros(max(P, 1), np.int32)
        R = C.c_int64(0)
        B = C.c_uint32(0)
        st = self.lib.glic_oracle_forward(
            C.c_int(P), C.c_int(int(g["degree"])), C.c_int(M), _ptr(a["means"]), _ptr(a["scales"]),
            self.real(scale_modifier), _ptr(a["rots"]), _ptr(a["opacity"]), _ptr(a["dc"]), _ptr(a["sh"]),
            _ptr(view), _ptr(proj), _ptr(campos), C.c_int(W), C.c_int(H), self.real(cam["tanfovx"]),
            self.real(cam["tanfovy"]), _ptr(lims), C.c_int(int(no_color)), _ptr(color), _ptr(final_T), _ptr(radii),
            C.byref(R), C.byref(B))
        out = dict(color=color, final_T=final_T, radii=radii[:P], R=int(R.value), B=int(B.value), state=st, P=P, M=M,
                   W=W, H=H, inputs=a, cam=(view, proj, campos, lims, cam["tanfovx"], cam["tanfovy"]),
                   scale_modifier=scale_modifier)
        return out

    def state(self, fwd):
        P, R, W, H = fwd["P"], fwd["R"], fwd["W"], fwd["H"]
        T = ((W + 15) // 16) * ((H + 15) // 16)
        d = dict(depth=np.zeros(P, self.dtype), xy=np.zeros((P, 2), self.dtype),
                 conic_opacity=np.zeros((P, 4), self.dtype), rgb=np.zeros((P, 3), self.dtype),
                 tiles_touched=np.zeros(P, np.uint32), point_list=np.zeros(R, np.uint32),
                 keys_sorted=np.zeros(R, np.uint64), ranges=np.zeros((T, 2), np.uint32),
                 bucket_offsets=np.zeros(T, np.uint32), n_contrib=np.zeros(H * W, np.uint32),
                 max_contrib=np.zeros(T, np.uint32), clamped=np.zeros((P, 3), np.uint8))
        self.lib.glic_oracle_state_get(C.c_void_p(fwd["state"]), *[_ptr(d[k]) for k in (
            "depth", "xy", "conic_opacity", "rgb", "tiles_touched", "point_list", "keys_sorted", "ranges",
            "bucket_offsets", "n_contrib", "max_contrib", "clamped")])
        return d

    def backward(self, fwd, dL_dpix, lambda_erank=0.0):
        P, M = fwd["P"], fwd["M"]
        a = fwd["inputs"]
        view, proj, campos, lims, tfx, tfy = fwd["cam"]
        g = self._a(dL_dpix)
        o = dict(dL_dmeans2D=np.zeros((P, 3), self.dtype), dL_dcolors=np.zeros((P, 3), self.dtype),
                 dL_dopacity=np.zeros((P, 1), self.dtype), dL_dmeans3D=np.zeros((P, 3), self.dtype),
                 dL_dcov3D=np.zeros((P, 6), self.dtype), dL_ddc=np.zeros((P, 1, 3), self.dtype),
                 dL_dsh=np.zeros((P, M, 3), self.dtype), dL_dscales=np.zeros((P, 3), self.dtype),
                 dL_drots=np.zeros((P, 4), self.dtype), dL_dconic=np.zeros((P, 4), self.dtype))
        self.lib.glic_oracle_backward(
            C.c_void_p(fwd["state"]), _ptr(a["means"]), _ptr(a["scales"]), self.real(fwd["scale_modifier"]),
            _ptr(a["rots"]), _ptr(a["dc"]), _ptr(a["sh"]) if a["sh"].size else None, _ptr(view), _ptr(proj), _ptr(campos), self.real(tfx),
            self.real(tfy), _ptr(lims), _ptr(g), self.real(lambda_erank), _ptr(o["dL_dmeans2D"]),
            _ptr(o["dL_dcolors"]), _ptr(o["dL_dopacity"]), _ptr(o["dL_dmeans3D"]), _ptr(o["dL_dcov3D"]),
            _ptr(o["dL_ddc"]), _ptr(o["dL_dsh"]), _ptr(o["dL_dscales"]), _ptr(o["dL_drots"]), _ptr(o["dL_dconic"]))
        return o

    def preprocess_backward(self, g, cam, radii, clamped, dL_dmeans2D, dL_dconic, dL_dcolors, scale_modifier=1.0,
                            lambda_erank=0.0):
        """The per-Gaussian backward alone (A.7 + A.8) on given 2-D gradients: dL_dmeans2D [P,>=2], dL_dconic [P,3]
        (xx, xy, yy), dL_dcolors [P,3], with the forward's radii [P] and clamp bits clamped [P,3].  g as for forward()
        (an empty sh: no colour backward).  Returns dL_dmeans3D, dL_dcov3D, dL_ddc, dL_dsh, dL_dscales, dL_drots."""
        P = int(np.asarray(g["means"]).shape[0])
        M = int(g["sh"].shape[1]) if g["sh"].size else 0
        a = {k: self._a(g[k]) for k in ("means", "scales", "rots", "dc", "sh")}
        view, proj, campos, lims = (self._a(cam[k]) for k in ("view", "proj", "campos", "lims"))
        o = dict(dL_dmeans3D=np.zeros((P, 3), self.dtype), dL_dcov3D=np.zeros((P, 6), self.dtype),
                 dL_ddc=np.zeros((P, 3), self.dtype), dL_dsh=np.zeros((P, M, 3), self.dtype),
                 dL_dscales=np.zeros((P, 3), self.dtype), dL_drots=np.zeros((P, 4), self.dtype))
        r = np.ascontiguousarray(np.asarray(radii).reshape(-1)[:P], np.int32)
        cl = np.ascontiguousarray(np.asarray(clamped).reshape(P, 3), np.uint8)
        dm2 = self._a(np.asarray(dL_dmeans2D).reshape(P, -1)[:, :2])
        dco, dcol = self._a(dL_dconic, (P, 3)), self._a(dL_dcolors, (P, 3))
        self.lib.glic_oracle_preprocess_backward(
            C.c_int(P), C.c_int(int(g["degree"])), C.c_int(M), _ptr(a["means"]), _ptr(a["scales"]), self.real(scale_modifier),
            _ptr(a["rots"]), _ptr(a["dc"]), _ptr(a["sh"]) if M else None, _ptr(view), _ptr(proj), _ptr(campos),
            C.c_int(cam["W"]), C.c_int(cam["H"]), self.real(cam["tanfovx"]), self.real(cam["tanfovy"]), _ptr(lims), _ptr(r),
            _ptr(cl), _ptr(dm2), _ptr(dco), _ptr(dcol), self.real(lambda_erank), _ptr(o["dL_dmeans3D"]), _ptr(o["dL_dcov3D"]),
            _ptr(o["dL_ddc"]), _ptr(o["dL_dsh"]), _ptr(o["dL_dscales"]), _ptr(o["dL_drots"]))
        return o

    def render(self, W, H, ranges, point_list, xy, conic_opacity, rgb):
        """The render forward alone (A.5) on a given state: ranges [T,2], point_list [R], xy [P,2], conic_opacity [P,4],
        rgb [P,3].  Returns color [3,H,W], final_T [H,W], n_contrib [H*W], max_contrib [T]."""
        T = ((W + 15) // 16) * ((H + 15) // 16)
        rg = np.ascontiguousarray(np.asarray(ranges).reshape(T, 2), np.uint32)
        pl = np.ascontiguousarray(point_list, np.uint32)
        xy, co, rgb = self._a(xy), self._a(conic_opacity), self._a(rgb)
        color, final_T = np.zeros((3, H, W), self.dtype), np.zeros((H, W), self.dtype)
        n_contrib, max_contrib = np.zeros(H * W, np.uint32), np.zeros(T, np.uint32)
        self.lib.glic_oracle_render(C.c_int(W), C.c_int(H), _ptr(rg), _ptr(pl), _ptr(xy), _ptr(co), _ptr(rgb), None, C.c_int(0),
                                    _ptr(color), _ptr(final_T), _ptr(n_contrib), _ptr(max_contrib), None, None)
        return color, final_T, n_contrib, max_contrib

    def render_backward(self, W, H, ranges, point_list, xy, conic_opacity, rgb, n_contrib, color, dL_dpix):
        """The render backward alone (A.6) on a given state and the forward's n_contrib [H*W] and color [3,H,W].  Returns the
        2-D gradients dmean2D [P,2] (NDC-scaled), dconic [P,3] (x, y, w), dopacity [P], dcolor [P,3]."""
        T = ((W + 15) // 16) * ((H + 15) // 16)
        rg = np.ascontiguousarray(np.asarray(ranges).reshape(T, 2), np.uint32)
        pl = np.ascontiguousarray(point_list, np.uint32)
        nc = np.ascontiguousarray(np.asarray(n_contrib).reshape(-1), np.uint32)
        xy, co, rgb, col, g = (self._a(a) for a in (xy, conic_opacity, rgb, color, dL_dpix))
        P = xy.shape[0]
        o = dict(dmean2D=np.zeros((P, 2), self.dtype), dconic=np.zeros((P, 3), self.dtype), dopacity=np.zeros(P, self.dtype),
                 dcolor=np.zeros((P, 3), self.dtype))
        self.lib.glic_oracle_render_backward(C.c_int(P), C.c_int(W), C.c_int(H), _ptr(rg), _ptr(pl), _ptr(xy), _ptr(co), _ptr(rgb),
                                             _ptr(nc), _ptr(col), _ptr(g), _ptr(o["dmean2D"]), _ptr(o["dconic"]),
                                             _ptr(o["dopacity"]), _ptr(o["dcolor"]))
        return o

    def free(self, fwd):
        if fwd.get("state"):
            self.lib.glic_oracle_state_free(C.c_void_p(fwd["state"]))
            fwd["state"] = None

    # ---- loss (A.9) ---------------------------------------------------------------------
    def ssim(self, img1, img2, train=True, C1=0.01 ** 2, C2=0.03 ** 2):
        a, b = self._a(img1), self._a(img2)
        CH, H, W = a.shape[-3:]
        m = np.zeros_like(a)
        d1, d2, d3 = (np.zeros_like(a) for _ in range(3)) if train else (None, None, None)
        self.lib.glic_oracle_ssim(C.c_int(CH), C.c_int(H), C.c_int(W), self.real(np.float32(C1)),
                                  self.real(np.float32(C2)), _ptr(a), _ptr(b), _ptr(m), _ptr(d1), _ptr(d2), _ptr(d3))
        return m, d1, d2, d3

    def ssim_backward(self, img1, img2, dL_dmap, d1, d2, d3):
        a, b, g = self._a(img1), self._a(img2), self._a(dL_dmap)
        CH, H, W = a.shape[-3:]
        out = np.zeros_like(a)
        self.lib.glic_oracle_ssim_backward(C.c_int(CH), C.c_int(H), C.c_int(W), _ptr(a), _ptr(b), _ptr(g),
                                           _ptr(self._a(d1)), _ptr(self._a(d2)), _ptr(self._a(d3)), _ptr(out))
        return out

    def loss(self, img, gt, lambda_dssim=0.2, grad=True):
        a, b = self._a(img), self._a(gt)
        CH, H, W = a.shape
        g = np.zeros_like(a) if grad else None
        L = self.lib.glic_oracle_loss(C.c_int(CH), C.c_int(H), C.c_int(W), self.real(lambda_dssim), _ptr(a), _ptr(b),
                                      _ptr(g))
        return float(L), g

    # ---- Adam (A.10), knn (A.11), sort (A.4) ------------------------------------------------
    def adam(self, param, grad, m, v, visible, lr, b1=0.9, b2=0.999, eps=1e-15):
        p, g, m, v = (self._a(x).copy() for x in (param, grad, m, v))
        vis = np.ascontiguousarray(np.asarray(visible, dtype=np.uint8))
        N = vis.shape[0]
        Mm = p.size // N
        self.lib.glic_oracle_adam(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(vis), self.real(lr), self.real(b1),
                                  self.real(b2), self.real(eps), C.c_uint32(N), C.c_uint32(Mm))
        return p, m, v

    def adam_packed(self, params, grads, m, v, visible, lr6, M, b1=0.9, b2=0.999, eps=1e-15):
        """SparseGaussianAdam over the planar model (buffer order rotation, xyz, scaling, opacity, f_dc, f_rest):
        six per-group applications of A.10 -- the oracle of glic_adam_update_packed."""
        p, mm, vv = (self._a(x).copy().reshape(-1) for x in (params, m, v))
        g = self._a(grads).reshape(-1)
        P = np.asarray(visible).shape[0]
        off = 0
        for k, lr in zip((4, 3, 3, 1, 3, 3 * M), lr6):
            n = P * k
            if n:
                p[off:off + n], mm[off:off + n], vv[off:off + n] = (
                    x.reshape(-1) for x in self.adam(p[off:off + n], g[off:off + n], mm[off:off + n], vv[off:off + n], visible, lr, b1, b2, eps))
            off += n
        return p, mm, vv

    def activations(self, logits, log_scales, rots_raw):
        a, b, c = self._a(logits).reshape(-1), self._a(log_scales), self._a(rots_raw)
        P = a.shape[0]
        op, sc, rot = np.zeros(P, self.dtype), np.zeros((P, 3), self.dtype), np.zeros((P, 4), self.dtype)
        self.lib.glic_oracle_activations(C.c_int(P), _ptr(a), _ptr(b), _ptr(c), _ptr(op), _ptr(sc), _ptr(rot))
        return op, sc, rot

    def activations_backward(self, opacity, scales, rots_raw, dL_dopacity, dL_dscales, dL_drots):
        op, sc, rr = self._a(opacity).reshape(-1), self._a(scales), self._a(rots_raw)
        g1, g2, g3 = self._a(dL_dopacity).copy().reshape(-1), self._a(dL_dscales).copy(), self._a(dL_drots).copy()
        self.lib.glic_oracle_activations_backward(C.c_int(op.shape[0]), _ptr(op), _ptr(sc), _ptr(rr), _ptr(g1), _ptr(g2), _ptr(g3))
        return g1, g2, g3

    def extend_select(self, points, depth_rsp, R_cw, t_cw, fx, fy, cx, cy, W, H, final_T):
        """Indices (ascending) of the LiDAR points extend() turns into Gaussians (gaussian.cpp:499-607)."""
        p, d = self._a(points), self._a(depth_rsp).reshape(-1)
        R, t, T = self._a(R_cw), self._a(t_cw).reshape(-1), self._a(final_T)
        keep = np.zeros(max(p.shape[0], 1), np.int32)
        self.lib.glic_oracle_extend_select.restype = C.c_int
        m = self.lib.glic_oracle_extend_select(C.c_int(p.shape[0]), _ptr(p), _ptr(d), _ptr(R), _ptr(t), self.real(fx), self.real(fy),
                                               self.real(cx), self.real(cy), C.c_int(W), C.c_int(H), _ptr(T), _ptr(keep))
        return keep[:m].copy()

    def extend_init(self, keep, points, colors, depth_rsp, scaling_scale, fx, fy):
        """Initial raw parameters of the inserted Gaussians (gaussian.cpp:610-631)."""
        k = np.ascontiguousarray(keep, np.int32)
        m = k.shape[0]
        p, c, d = self._a(points), self._a(colors), self._a(depth_rsp).reshape(-1)
        out = dict(xyz=np.zeros((m, 3), self.dtype), f_dc=np.zeros((m, 3), self.dtype), log_scale=np.zeros((m, 3), self.dtype),
                   rot=np.zeros((m, 4), self.dtype), opacity_logit=np.zeros(m, self.dtype))
        self.lib.glic_oracle_extend_init(C.c_int(m), _ptr(k), _ptr(p), _ptr(c), _ptr(d), self.real(scaling_scale), self.real(fx),
                                         self.real(fy), _ptr(out["xyz"]), _ptr(out["f_dc"]), _ptr(out["log_scale"]), _ptr(out["rot"]),
                                         _ptr(out["opacity_logit"]))
        return out

    def knn(self, pts):
        p = self._a(pts)
        out = np.zeros(p.shape[0], self.dtype)
        self.lib.glic_oracle_knn(C.c_int(p.shape[0]), _ptr(p), _ptr(out))
        return out

    def sort_pairs(self, keys, vals, nbits):
        k = np.ascontiguousarray(keys, dtype=np.uint64)
        v = np.ascontiguousarray(vals, dtype=np.uint32)
        ko, vo = np.zeros_like(k), np.zeros_like(v)
        self.lib.glic_oracle_sort_pairs(C.c_int64(k.size), C.c_int(nbits), _ptr(k), _ptr(v), _ptr(ko), _ptr(vo))
        return ko, vo

    def higher_msb(self, n):
        return int(self.lib.glic_oracle_higher_msb(C.c_uint32(n)))

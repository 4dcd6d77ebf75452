"""ctypes face of the native mapping host (include/glic_b200.h "Native mapping host", csrc/mapper.cu).

Plumbing for tests and bench.py only: the host of the loop is the C++ object; this class converts numpy arrays to
pointers and keeps the host memory it handed over alive.  The mapper mirrors GaussianModel + extend() + optimize() +
evaluateVisualQuality() + saveMap() of the reference (gaussian.cpp:113-830).
"""
import ctypes as C

import numpy as np

from . import capi

FASTLIVO = dict(position_lr=1.6e-4, feature_lr=2.5e-3, opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001,
                lambda_dssim=0.2, scaling_scale=1.0)                  # config/fastlivo.yaml:15-24
DEAD_OPACITY = float(np.float32(1.0) / np.float32(255.0))             # GLIC_MAPPER_DEAD_OPACITY: the preprocess's o < 1/255 cull
DENSIFY_GRAD_THRESHOLD = float(np.float32(0.0002))                   # GLIC_MAPPER_DENSIFY_GRAD_THRESHOLD (Inria's default)
PERCENT_DENSE = float(np.float32(0.01))                              # GLIC_MAPPER_PERCENT_DENSE
RESET_OPACITY = float(np.float32(0.01))                              # GLIC_MAPPER_RESET_OPACITY
# glic_density_schedule's fields at Inria's defaults (GLIC_MAPPER_DENSIFY_FROM ... ; scene_extent 0: derived at each step)
DENSITY_SCHEDULE = dict(densify_from=500, densify_until=15000, densify_interval=100, opacity_reset_interval=3000,
                        grad_threshold=DENSIFY_GRAD_THRESHOLD, percent_dense=PERCENT_DENSE, min_opacity=float(np.float32(0.005)),
                        reset_opacity=RESET_OPACITY, screen_radius=20, world_scale_factor=float(np.float32(0.1)), scene_extent=0.0)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return None if a is None or a.size == 0 else a.ctypes.data_as(C.c_void_p)


def camera_block(W, H, fx, fy, cx, cy, R_wc, t_wc):
    """camera.h:38-110 as the mapper evaluates it -> dict shaped like synthetic.make_camera's."""
    R = (C.c_float * 9)(*[float(x) for x in np.asarray(R_wc, np.float64).reshape(9)])
    t = (C.c_float * 3)(*[float(x) for x in np.asarray(t_wc, np.float64).reshape(3)])
    out = (C.c_float * 41)()
    capi.check(capi.lib.glic_camera_block(int(W), int(H), fx, fy, cx, cy, R, t, out), "camera_block")
    o = np.array(out[:], np.float32)
    return dict(W=int(W), H=int(H), view=o[:16].copy(), proj=o[16:32].copy(), campos=o[32:35].copy(), tanfovx=float(o[35]),
                tanfovy=float(o[36]), lims=o[37:41].copy())


def _f32x(a, n):
    return (C.c_float * n)(*[float(x) for x in np.asarray(a, np.float32).reshape(n)])


def _sh_blocks(sh, degree):
    """the band matrices A_1 .. A_degree of a record's sh[83], as float64 arrays"""
    out, off = [], 0
    for l in range(1, 4):
        n = 2 * l + 1
        if l <= degree:
            out.append(np.array(sh[off:off + n * n], np.float64).reshape(n, n))
        off += n * n
    return out


def pose_correction_record(R_old, t_old, R_new, t_new, degree=3):
    """glic_pose_correction_record: the rigid correction from a keyframe's old pose to its new one (R_wc [3,3], t_wc [3], taken
    as float32).  Returns dict R [3,3], t [3], q [4] (r, x, y, z) float64 and sh, the list of band matrices A_1 .. A_degree."""
    r = capi.RigidCorrection()
    capi.check(capi.lib.glic_pose_correction_record(_f32x(R_old, 9), _f32x(t_old, 3), _f32x(R_new, 9), _f32x(t_new, 3), int(degree),
                                                    C.byref(r)), "pose_correction_record")
    return dict(R=np.array(r.R[:], np.float64).reshape(3, 3), t=np.array(r.t[:], np.float64), q=np.array(r.q[:], np.float64),
                sh=_sh_blocks(r.sh, degree))


def sh_rotation(q, degree=3):
    """glic_sh_rotation: the band matrices A_1 .. A_degree of R(q) for a unit quaternion q = (r, x, y, z) (float64)."""
    qq = (C.c_double * 4)(*[float(x) for x in np.asarray(q, np.float64).reshape(4)])
    out = (C.c_double * 83)()
    capi.check(capi.lib.glic_sh_rotation(qq, int(degree), out), "sh_rotation")
    return _sh_blocks(out, degree)


def checkpoint_config(path):
    """The configuration (capi.MapperConfig, capacity = the saved arena capacity) of a checkpoint file; host only."""
    cfg = capi.MapperConfig()
    capi.check(capi.lib.glic_mapper_checkpoint_config(str(path).encode(), C.byref(cfg)), "mapper_checkpoint_config")
    return cfg


class Mapper:
    def __init__(self, W, H, fx, fy, cx, cy, sh_degree=3, capacity=0, max_iters=100, seed=0, rank=0, world=1, views_per_rank=1,
                 **lrs):
        cfg = capi.MapperConfig()
        cfg.width, cfg.height, cfg.fx, cfg.fy, cfg.cx, cfg.cy = int(W), int(H), fx, fy, cx, cy
        cfg.sh_degree = int(sh_degree)
        for k, v in dict(FASTLIVO, **lrs).items():
            setattr(cfg, k, float(v))
        cfg.capacity, cfg.max_iters, cfg.seed = int(capacity), int(max_iters), int(seed)
        cfg.rank, cfg.world, cfg.views_per_rank = int(rank), int(world), int(views_per_rank)
        self._create(cfg)

    def _create(self, cfg):
        self.cfg = cfg
        self.M = (cfg.sh_degree + 1) ** 2 - 1
        self.W, self.H = int(cfg.width), int(cfg.height)
        self._h = C.c_void_p()
        self._keep = []                                   # host arrays the C++ side points into
        capi.check(capi.lib.glic_mapper_create(C.byref(cfg), C.byref(self._h)), "mapper_create")

    @classmethod
    def from_checkpoint(cls, path, lpips=None):
        """A new mapper that continues from a file of save_checkpoint(): created with the file's configuration (checkpoint_config),
        with the LPIPS weights of `lpips` (a glic_lpips weight file; they are not in the checkpoint) loaded, then restored.  The
        restored mapper owns its keyframe images.  With world > 1, export_handle() / connect() follow."""
        m = cls.__new__(cls)
        m._h = C.c_void_p()
        m._create(checkpoint_config(path))
        try:
            if lpips is not None:
                m.load_lpips(lpips)
            m.load_checkpoint(path)
        except Exception:
            m.close()
            raise
        return m

    def close(self):
        if self._h:
            capi.lib.glic_mapper_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def initialize(self, g):
        """g: raw parameters as synthetic.make_gaussians returns them (means, dc, sh, opacity_logits, log_scales, rots)."""
        P = int(g["means"].shape[0])
        a = [_f32(g["means"]), _f32(g["dc"]).reshape(P, 3), _f32(g["sh"]), _f32(g["opacity_logits"]), _f32(g["log_scales"]), _f32(g["rots"])]
        capi.check(capi.lib.glic_mapper_initialize(self._h, P, *[_p(x) for x in a]), "mapper_initialize")

    def initialize_lidar(self, points, colors, depth_rsp, focal, sky_points=0, sky_radius=0):
        """initialize() (gaussian.cpp:212-304) on the GPU: sky_points sky rows keyed by the seed, then the first scan's LiDAR
        points in order.  colors are the Dataset's doubles (rgb / 255.0); focal = (fx + fy) / 2 of the configuration."""
        pts, dep = _f32(points), _f32(depth_rsp)
        col = np.ascontiguousarray(colors, dtype=np.float64)
        n = int(pts.shape[0])
        capi.check(capi.lib.glic_mapper_initialize_lidar(self._h, n, _p(pts), _p(col), _p(dep), float(focal), int(sky_points),
                                                         int(sky_radius)), "mapper_initialize_lidar")

    def sky_rows(self):
        """How many leading rows are the skybox (save_map leaves them out)."""
        out = C.c_uint32()
        capi.check(capi.lib.glic_mapper_sky_rows(self._h, C.byref(out)), "mapper_sky_rows")
        return int(out.value)

    def add_keyframe(self, R_wc, t_wc, image, train=True, pinned=None):
        """image: [3,H,W] float32 numpy array, or a pinned torch tensor (kept alive here)."""
        kf = capi.Keyframe()
        kf.R_wc[:] = [float(x) for x in np.asarray(R_wc, np.float64).reshape(9)]
        kf.t_wc[:] = [float(x) for x in np.asarray(t_wc, np.float64).reshape(3)]
        if hasattr(image, "data_ptr"):
            self._keep.append(image)
            kf.image = image.data_ptr()
        else:
            img = _f32(image)
            self._keep.append(img)
            kf.image = img.ctypes.data
        capi.check(capi.lib.glic_mapper_add_keyframe(self._h, C.byref(kf), int(bool(train))), "mapper_add_keyframe")

    def enable_frames(self, select_every_k_frame=5, sky_points=0, sky_radius=0):
        """Accept raw frames through add_frame (config/*.yaml: select_every_k_frame, skybox_points_num, skybox_radius)."""
        capi.check(capi.lib.glic_mapper_enable_frames(self._h, int(select_every_k_frame), int(sky_points), int(sky_radius)),
                   "mapper_enable_frames")

    def add_frame(self, q_wc, t_wc, bgr, xyz, rgb, mask=None):
        """Dataset::addFrame (gaussian.cpp:41-111) and the keyframe hand-off of mapping.cpp:158-174 on the GPU.  q_wc: (x, y, z, w)
        odometry orientation; t_wc: position; bgr: [H,W,3] uint8 BGR8 image (a row-padded view such as a[:, :W] of a wider
        array is passed with its row stride); xyz: [n,3] float32 world points; rgb: [n,3] uint8; mask (optional): the frame's
        [H,W] valid-pixel map (nonzero / True = used, see set_mask), set before the hand-off so that its extend() seeds
        nothing at a masked pixel.  Returns True for a training keyframe, False for a held-out one."""
        f = capi.Frame()
        f.q_wc[:] = [float(x) for x in np.asarray(q_wc, np.float64).reshape(4)]
        f.t_wc[:] = [float(x) for x in np.asarray(t_wc, np.float64).reshape(3)]
        img = np.asarray(bgr)
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape != (self.H, self.W, 3) or img.strides[1:] != (3, 1):
            raise ValueError("bgr must be a [%d,%d,3] uint8 array with packed pixels" % (self.H, self.W))
        f.bgr, f.row_bytes = img.ctypes.data, int(img.strides[0])
        pts = _f32(xyz).reshape(-1, 3)
        col = np.ascontiguousarray(rgb, dtype=np.uint8).reshape(-1, 3)
        if pts.shape[0] != col.shape[0]:
            raise ValueError("xyz and rgb must have the same number of points")
        f.n_points, f.xyz, f.rgb = int(pts.shape[0]), _p(pts), _p(col)
        out = C.c_int()
        if mask is None:
            capi.check(capi.lib.glic_mapper_add_frame(self._h, C.byref(f), C.byref(out)), "mapper_add_frame")
        else:
            valid = self._mask_bytes(mask)
            capi.check(capi.lib.glic_mapper_add_frame_masked(self._h, C.byref(f), _p(valid), C.byref(out)), "mapper_add_frame_masked")
        return bool(out.value)

    def _mask_bytes(self, mask):
        m = np.asarray(mask)
        if m.shape != (self.H, self.W):
            raise ValueError("mask must be a [%d,%d] array" % (self.H, self.W))
        return np.ascontiguousarray(m != 0, dtype=np.uint8)

    def set_mask(self, is_train, index, valid):
        """Set (valid: [H,W] array, nonzero / True = the pixel is used) or clear (valid=None) a keyframe's valid-pixel mask.  The
        loss, evaluate / evaluate_lpips, align and extend() leave masked pixels out (include/glic_b200.h, "Per-keyframe
        valid-pixel masks"); a mask with no used pixel is refused."""
        v = None if valid is None else self._mask_bytes(valid)
        capi.check(capi.lib.glic_mapper_set_keyframe_mask(self._h, int(bool(is_train)), int(index), _p(v)), "mapper_set_keyframe_mask")

    def mask(self, is_train, index):
        """-> (the stored [H,W] uint8 0/1 mask, or None when the keyframe has none; the number of used pixels)"""
        n = C.c_uint32()
        out = np.empty((self.H, self.W), np.uint8)
        capi.check(capi.lib.glic_mapper_keyframe_mask(self._h, int(bool(is_train)), int(index), _p(out), C.byref(n)), "mapper_keyframe_mask")
        return (out if n.value else None), int(n.value)

    def keyframe_image(self, index, train=True):
        """The [3,H,W] float32 image the loss sees for a keyframe (decoded from 8 bits for add_frame keyframes)."""
        out = np.empty((3, self.H, self.W), np.float32)
        capi.check(capi.lib.glic_mapper_keyframe_image(self._h, int(bool(train)), int(index), _p(out)), "mapper_keyframe_image")
        return out

    def frames_get(self):
        st = capi.FrameStats()
        capi.check(capi.lib.glic_mapper_frames_get(self._h, C.byref(st)), "mapper_frames_get")
        return st

    def extend(self, points, colors, depth_rsp):
        pts, col, dep = _f32(points), _f32(colors), _f32(depth_rsp)
        capi.check(capi.lib.glic_mapper_extend(self._h, int(pts.shape[0]), _p(pts), _p(col), _p(dep)), "mapper_extend")
        return self.stats().last_inserted

    def optimize(self, views=None):
        if views is None:
            capi.check(capi.lib.glic_mapper_optimize(self._h, None, 0), "mapper_optimize")
        else:
            arr = (C.c_int * len(views))(*[int(v) for v in views])
            capi.check(capi.lib.glic_mapper_optimize(self._h, arr, len(views)), "mapper_optimize")
        return self.stats()

    def sample_views(self):
        buf = (C.c_int * max(1, self.cfg.max_iters))()
        n = C.c_int()
        capi.check(capi.lib.glic_mapper_sample_views(self._h, buf, C.byref(n)), "mapper_sample_views")
        return list(buf[:n.value])

    def evaluate(self, index, train=True):
        a, b = C.c_float(), C.c_float()
        capi.check(capi.lib.glic_mapper_evaluate(self._h, int(bool(train)), int(index), C.byref(a), C.byref(b)), "mapper_evaluate")
        return a.value, b.value

    def load_lpips(self, path):
        """Load a glic_lpips weight file (gaussian_lic_b200.lpips_weights.convert makes one from lpips_alex.pt)."""
        capi.check(capi.lib.glic_mapper_load_lpips(self._h, str(path).encode()), "mapper_load_lpips")

    def evaluate_lpips(self, index, train=True):
        """(PSNR, SSIM, LPIPS) of one keyframe from one render; PSNR and SSIM are evaluate()'s, bit for bit."""
        a, b, c = C.c_float(), C.c_float(), C.c_float()
        capi.check(capi.lib.glic_mapper_evaluate_lpips(self._h, int(bool(train)), int(index), C.byref(a), C.byref(b), C.byref(c)),
                   "mapper_evaluate_lpips")
        return a.value, b.value, c.value

    def render(self, index, train=True):
        """The [3,H,W] float32 image evaluation scores: drawn at the keyframe's current pose, a training keyframe's exposure
        applied, clamped to [0,1]."""
        out = np.empty((3, self.H, self.W), np.float32)
        capi.check(capi.lib.glic_mapper_render(self._h, int(bool(train)), int(index), _p(out)), "mapper_render")
        return out

    def save_map(self, path):
        capi.check(capi.lib.glic_mapper_save_map(self._h, str(path).encode()), "mapper_save_map")

    def save_checkpoint(self, path):
        """Write the whole mapper state to `path` (include/glic_b200.h "Checkpoints"): via <path>.tmp, renamed over path once
        complete, so an existing file survives a failed save.  Changes nothing in the mapper."""
        capi.check(capi.lib.glic_mapper_save_checkpoint(self._h, str(path).encode()), "mapper_save_checkpoint")

    def load_checkpoint(self, path):
        """Restore a checkpoint into this mapper, which must be fresh (created, with no rows, keyframes or features) and have the
        file's configuration but for the capacity (see from_checkpoint)."""
        capi.check(capi.lib.glic_mapper_load_checkpoint(self._h, str(path).encode()), "mapper_load_checkpoint")

    def stats(self):
        st = capi.MapperStats()
        capi.check(capi.lib.glic_mapper_stats_get(self._h, C.byref(st)), "mapper_stats")
        return st

    def set_optimizer(self, on):
        capi.check(capi.lib.glic_mapper_set_option(self._h, 1, int(bool(on))), "mapper_set_option")

    def set_binning_pairs(self, pairs):
        capi.check(capi.lib.glic_mapper_set_option(self._h, 2, int(pairs)), "mapper_set_option")

    def set_deterministic(self, on):
        """GLIC_MAPPER_OPT_DETERMINISTIC: fixed-order render backward, loss and evaluation sums (bit-reproducible training)"""
        capi.check(capi.lib.glic_mapper_set_option(self._h, 3, int(bool(on))), "mapper_set_option")

    def enable_exposure(self, exposure_lr=0.001):
        """Train a 3x4 affine exposure per training keyframe from now on (config/fastlivo.yaml:25-26: exposure_lr 0.001)."""
        capi.check(capi.lib.glic_mapper_enable_exposure(self._h, float(exposure_lr)), "mapper_enable_exposure")

    def exposure(self, index):
        """E of training keyframe `index` as a [3,4] float32 array (out_c = E[0][c] r + E[1][c] g + E[2][c] b + E[c][3])."""
        out = (C.c_float * 12)()
        capi.check(capi.lib.glic_mapper_exposure_get(self._h, int(index), out), "mapper_exposure_get")
        return np.array(out[:], np.float32).reshape(3, 4)

    def set_exposure(self, index, E):
        """Overwrite E of training keyframe `index`; its Adam state is kept."""
        e = np.asarray(E, np.float32).reshape(12)
        capi.check(capi.lib.glic_mapper_exposure_set(self._h, int(index), (C.c_float * 12)(*[float(x) for x in e])), "mapper_exposure_set")

    def exposure_state(self, index):
        """(E [3,4], exp_avg [3,4], exp_avg_sq [3,4], step count) of training keyframe `index`"""
        m1, m2, t = (C.c_float * 12)(), (C.c_float * 12)(), C.c_int()
        capi.check(capi.lib.glic_mapper_exposure_adam_state(self._h, int(index), m1, m2, C.byref(t)), "mapper_exposure_adam_state")
        return self.exposure(index), np.array(m1[:], np.float32).reshape(3, 4), np.array(m2[:], np.float32).reshape(3, 4), int(t.value)

    def enable_pose_refinement(self, lr_translation, lr_rotation):
        """Refine every training keyframe's pose from now on: T_cw <- Exp(u) T_cw, u from Adam on dL/d(rho, omega)."""
        capi.check(capi.lib.glic_mapper_enable_pose_refinement(self._h, float(lr_translation), float(lr_rotation)),
                   "mapper_enable_pose_refinement")

    def pose(self, index, camera=False):
        """(R_wc [3,3], t_wc [3]) float32 of training keyframe `index`; camera=True adds its device camera block as a dict
        shaped like camera_block()'s."""
        R, t, cam = (C.c_float * 9)(), (C.c_float * 3)(), (C.c_float * 41)()
        capi.check(capi.lib.glic_mapper_pose_get(self._h, int(index), R, t, cam if camera else None), "mapper_pose_get")
        out = (np.array(R[:], np.float32).reshape(3, 3), np.array(t[:], np.float32))
        if not camera:
            return out
        o = np.array(cam[:], np.float32)
        return out + (dict(W=self.W, H=self.H, view=o[:16].copy(), proj=o[16:32].copy(), campos=o[32:35].copy(),
                           tanfovx=float(o[35]), tanfovy=float(o[36]), lims=o[37:41].copy()),)

    def set_pose(self, index, R_wc, t_wc):
        """Overwrite the pose of training keyframe `index`; its Adam state is kept."""
        R = (C.c_float * 9)(*[float(x) for x in np.asarray(R_wc, np.float32).reshape(9)])
        t = (C.c_float * 3)(*[float(x) for x in np.asarray(t_wc, np.float32).reshape(3)])
        capi.check(capi.lib.glic_mapper_pose_set(self._h, int(index), R, t), "mapper_pose_set")

    def pose_state(self, index):
        """(exp_avg [6], exp_avg_sq [6], step count) of training keyframe `index`'s pose (rho then omega)"""
        m1, m2, t = (C.c_float * 6)(), (C.c_float * 6)(), C.c_int()
        capi.check(capi.lib.glic_mapper_pose_adam_state(self._h, int(index), m1, m2, C.byref(t)), "mapper_pose_adam_state")
        return np.array(m1[:], np.float32), np.array(m2[:], np.float32), int(t.value)

    def anchors(self):
        """anchor [P] int32: the training keyframe each row moves with under correct_poses, or -1 (never moves)."""
        P = int(self.stats().num_gaussians)
        out = np.zeros(max(P, 1), np.int32)
        capi.check(capi.lib.glic_mapper_anchors(self._h, out.ctypes.data_as(C.c_void_p)), "mapper_anchors")
        return out[:P]

    def set_anchors(self, anchors):
        """Overwrite every row's anchor (-1, or a training keyframe index); anything else is refused and nothing changes."""
        a = np.ascontiguousarray(anchors, dtype=np.int32).reshape(-1)
        if a.shape[0] != int(self.stats().num_gaussians):
            raise ValueError("set_anchors needs one anchor per row")
        capi.check(capi.lib.glic_mapper_set_anchors(self._h, a.ctypes.data_as(C.c_void_p)), "mapper_set_anchors")

    def correct_poses(self, corrections):
        """Move keyframes to corrected poses and the rows anchored to them with them (glic_mapper_correct_poses).
        corrections: a list of (is_train, index, R_wc [3,3], t_wc [3]).  Returns the number of rows moved."""
        arr = (capi.PoseCorrection * max(len(corrections), 1))()
        for e, (is_train, index, R, t) in zip(arr, corrections):
            e.is_train, e.index = int(bool(is_train)), int(index)
            e.R_wc[:] = [float(x) for x in np.asarray(R, np.float32).reshape(9)]
            e.t_wc[:] = [float(x) for x in np.asarray(t, np.float32).reshape(3)]
        moved = C.c_uint32()
        capi.check(capi.lib.glic_mapper_correct_poses(self._h, len(corrections), arr, C.byref(moved)), "mapper_correct_poses")
        return int(moved.value)

    def align(self, index, train=False, iterations=100, lr_translation=1e-3, lr_rotation=1e-3, exposure_lr=0.0, split=False,
              image=False):
        """Fit keyframe `index`'s pose (and with exposure_lr > 0 its exposure) to its image against the frozen map, then score it
        there (glic_mapper_align).  split=True fits on the left half and scores on the right half.  Returns a dict of the
        result fields: R_wc [3,3], t_wc [3], E [3,4], psnr, ssim, lpips (NaN without load_lpips), first_loss, last_loss, the
        Adam moments (pose_exp_avg [6], pose_exp_avg_sq [6], expo_exp_avg [3,4], expo_exp_avg_sq [3,4]), steps, skipped; and
        with image=True the [3,H,W] clamped, exposed frame at the fitted camera under "image"."""
        p = capi.AlignParams(int(iterations), float(lr_translation), float(lr_rotation), float(exposure_lr), int(bool(split)))
        r = capi.AlignResult()
        img = np.empty((3, self.H, self.W), np.float32) if image else None
        capi.check(capi.lib.glic_mapper_align(self._h, int(bool(train)), int(index), C.byref(p), C.byref(r), _p(img)), "mapper_align")
        shapes = dict(R_wc=(3, 3), E=(3, 4), expo_exp_avg=(3, 4), expo_exp_avg_sq=(3, 4))
        out = {}
        for k, _ in capi.AlignResult._fields_:
            v = getattr(r, k)
            if isinstance(v, C.Array):
                out[k] = np.array(v[:], np.float32).reshape(shapes.get(k, (-1,)))
            else:
                out[k] = v
        if image:
            out["image"] = img
        return out

    def render_camera(self, R_wc, t_wc, width=None, height=None, fx=None, fy=None, cx=None, cy=None, exposure=-1, sky=True,
                      outputs=("rgb", "final_T", "depth", "median_depth")):
        """Draw the current map from a camera of the caller's choosing (glic_mapper_render_camera).  R_wc [3,3], t_wc [3] as
        add_keyframe takes them; the intrinsics and frame size left as None are the configuration's.  exposure: a training
        keyframe index whose E colours the image (exposure enabled), or -1 for the identity; sky=False leaves the skybox rows
        out.  Returns a dict of float32 numpy arrays for the requested outputs: rgb [3,H,W] (exposed, clamped to [0,1]),
        final_T [H,W], depth [H,W] (expected depth, unnormalised: divide by 1 - final_T) and median_depth [H,W]."""
        c = self.cfg
        cam = capi.RenderCamera()
        cam.R_wc[:] = [float(x) for x in np.asarray(R_wc, np.float32).reshape(9)]
        cam.t_wc[:] = [float(x) for x in np.asarray(t_wc, np.float32).reshape(3)]
        cam.fx, cam.fy = c.fx if fx is None else float(fx), c.fy if fy is None else float(fy)
        cam.cx, cam.cy = c.cx if cx is None else float(cx), c.cy if cy is None else float(cy)
        W, H = self.W if width is None else int(width), self.H if height is None else int(height)
        cam.width, cam.height = W, H
        shapes = dict(rgb=(3, H, W), final_T=(H, W), depth=(H, W), median_depth=(H, W))
        unknown = set(outputs) - set(shapes)
        if unknown:
            raise ValueError("unknown outputs: %s" % sorted(unknown))
        out = {k: np.empty(shapes[k], np.float32) for k in shapes if k in outputs}
        capi.check(capi.lib.glic_mapper_render_camera(self._h, C.byref(cam), int(exposure), int(bool(sky)),
                                                      *[_p(out.get(k)) for k in shapes]), "mapper_render_camera")
        return out

    def extract_mesh(self, origin, voxel_size, dims, trunc, max_depth=0.0, views=None):
        """A coloured triangle mesh of the map (glic_mapper_extract_mesh): the median depth and the colour of the map without
        its sky rows, drawn at each of training keyframes `views` (None: all of them) and fused into a dense TSDF grid of dims
        (nx, ny, nz) lattice points from origin with spacing voxel_size (truncation trunc; depths beyond max_depth > 0 left
        out), then naive surface nets.  Returns a dict of numpy arrays vertices [V,3] float32, colors [V,3] uint8 and faces
        [F,3] int32 (outward winding), and the counts vertices, faces and observed_voxels.  The mesh also stays in the mapper
        for save_mesh()."""
        p = capi.MeshParams()
        keep = None
        if views is not None:
            keep = (C.c_int * max(len(views), 1))(*[int(v) for v in views])
            p.views, p.n_views = C.cast(keep, C.c_void_p), len(views)
        p.origin[:] = [float(x) for x in np.asarray(origin, np.float32).reshape(3)]
        p.voxel_size = float(voxel_size)
        p.dims[:] = [int(x) for x in dims]
        p.trunc, p.max_depth = float(trunc), float(max_depth)
        counts = capi.MeshCounts()
        capi.check(capi.lib.glic_mapper_extract_mesh(self._h, C.byref(p), C.byref(counts)), "mapper_extract_mesh")
        del keep
        return self.mesh()

    def extract_mesh_sparse(self, origin, voxel_size, trunc, max_depth=0.0, views=None, max_blocks=0):
        """extract_mesh() over a sparse block grid (glic_mapper_extract_mesh_sparse): only the 8^3-voxel blocks near some view's
        observed surface are stored, on a lattice aligned to origin with spacing voxel_size and no box, so a map of any extent can
        be meshed; the mesh equals extract_mesh()'s with a box holding those blocks.  max_blocks > 0 refuses a map that needs more
        blocks (GlicError) before the grid is allocated.  Returns the counts as a dict (vertices, faces, observed_voxels, blocks,
        clipped_pixels, lattice_lo, lattice_hi: the inclusive lattice box of the blocks); the mesh itself is read with mesh()."""
        p = capi.SparseMeshParams()
        keep = None
        if views is not None:
            keep = (C.c_int * max(len(views), 1))(*[int(v) for v in views])
            p.views, p.n_views = C.cast(keep, C.c_void_p), len(views)
        p.origin[:] = [float(x) for x in np.asarray(origin, np.float32).reshape(3)]
        p.voxel_size, p.trunc, p.max_depth, p.max_blocks = float(voxel_size), float(trunc), float(max_depth), int(max_blocks)
        c = capi.SparseMeshCounts()
        capi.check(capi.lib.glic_mapper_extract_mesh_sparse(self._h, C.byref(p), C.byref(c)), "mapper_extract_mesh_sparse")
        del keep
        return dict(vertices=int(c.vertices), faces=int(c.faces), observed_voxels=int(c.observed_voxels), blocks=int(c.blocks),
                    clipped_pixels=int(c.clipped_pixels), lattice_lo=tuple(c.lattice_lo), lattice_hi=tuple(c.lattice_hi))

    def mesh(self):
        """The last extracted mesh as extract_mesh() returns it (empty arrays before any)."""
        c = capi.MeshCounts()
        capi.check(capi.lib.glic_mapper_mesh_get(self._h, C.byref(c), None, None, None), "mapper_mesh_get")
        V, F = int(c.vertices), int(c.faces)
        xyz, rgb, faces = np.empty((V, 3), np.float32), np.empty((V, 3), np.uint8), np.empty((F, 3), np.int32)
        capi.check(capi.lib.glic_mapper_mesh_get(self._h, None, _p(xyz), _p(rgb), _p(faces)), "mapper_mesh_get")
        return dict(vertices=xyz, colors=rgb, faces=faces, n_vertices=V, n_faces=F, observed_voxels=int(c.observed_voxels))

    def save_mesh(self, path):
        """Write the last extracted mesh as a binary little-endian PLY (x y z float, red green blue uchar, vertex_indices)."""
        capi.check(capi.lib.glic_mapper_save_mesh(self._h, str(path).encode()), "mapper_save_mesh")

    def synchronize(self):
        capi.check(capi.lib.glic_mapper_synchronize(self._h), "mapper_synchronize")

    def download(self, moments=False):
        P, M = int(self.stats().num_gaussians), self.M
        out = dict(means=np.zeros((P, 3), np.float32), dc=np.zeros((P, 3), np.float32), sh=np.zeros((P, M, 3), np.float32),
                   opacity_logits=np.zeros(P, np.float32), log_scales=np.zeros((P, 3), np.float32), rots=np.zeros((P, 4), np.float32))
        m1 = np.zeros(P * (14 + 3 * M), np.float32) if moments else None
        m2 = np.zeros(P * (14 + 3 * M), np.float32) if moments else None
        capi.check(capi.lib.glic_mapper_download(self._h, _p(out["means"]), _p(out["dc"]), _p(out["sh"]), _p(out["opacity_logits"]),
                                                 _p(out["log_scales"]), _p(out["rots"]), _p(m1), _p(m2)), "mapper_download")
        if moments:
            out["exp_avg"], out["exp_avg_sq"] = m1, m2
        return out

    def prune(self, min_opacity=DEAD_OPACITY, dry_run=False):
        """Remove every row whose activated opacity is below min_opacity (stable: survivors keep their order, parameters and
        Adam moments; the surviving sky rows stay in front).  The default removes exactly the rows the preprocess culls in every
        view.  dry_run only counts.  Returns the number of rows removed (or that would be)."""
        out = C.c_uint32()
        capi.check(capi.lib.glic_mapper_prune(self._h, float(min_opacity), int(bool(dry_run)), C.byref(out)), "mapper_prune")
        return int(out.value)

    def contribution(self, views=None):
        """The contribution scores of every row, sky rows included, over training keyframes `views` (None: all of them), each
        drawn at its current pose (glic_mapper_contribution).  Returns numpy arrays (max_weight [P] float32: the largest
        T * alpha of any pixel that takes the row; hits [P] uint64: the number of (view, pixel) pairs that take it; ends [P]
        uint64: the number of (view, pixel) pairs whose blend it ends without being taken)."""
        P = int(self.stats().num_gaussians)
        mw, hits, ends = np.zeros(max(P, 1), np.float32), np.zeros(max(P, 1), np.uint64), np.zeros(max(P, 1), np.uint64)
        arr, n = (None, 0) if views is None else ((C.c_int * len(views))(*[int(v) for v in views]), len(views))
        capi.check(capi.lib.glic_mapper_contribution(self._h, arr, n, _p(mw), _p(hits), _p(ends)), "mapper_contribution")
        return mw[:P], hits[:P], ends[:P]

    def prune_unseen(self, min_hits=1, min_weight=0.0, sky=False, views=None, dry_run=False):
        """Remove every row (sky rows only with sky=True) whose scores over training keyframes `views` (None: all) fall short:
        hits + ends < min_hits or max_weight < min_weight (glic_mapper_prune_unseen).  The defaults remove exactly the rows that
        neither take nor end a pixel of any scored view, which changes none of those views' pixels.  The compaction is
        prune()'s.  dry_run only counts.  Returns the number of rows removed (or that would be)."""
        p = capi.UnseenParams()
        keep = None
        if views is not None:
            keep = (C.c_int * max(len(views), 1))(*[int(v) for v in views])
            p.views, p.n_views = C.cast(keep, C.c_void_p), len(views)
        p.min_weight, p.min_hits, p.sky = float(min_weight), int(min_hits), int(sky)
        out = C.c_uint32()
        capi.check(capi.lib.glic_mapper_prune_unseen(self._h, C.byref(p), int(bool(dry_run)), C.byref(out)), "mapper_prune_unseen")
        del keep
        return int(out.value)

    def enable_densification(self):
        """Gather the view-space gradient statistics densify() selects on, from the next iteration on (world > 1: before
        export_handle())."""
        capi.check(capi.lib.glic_mapper_enable_densification(self._h), "mapper_enable_densification")

    def densify(self, scene_extent, grad_threshold=DENSIFY_GRAD_THRESHOLD, percent_dense=PERCENT_DENSE, dry_run=False):
        """Clone the selected small rows and split the selected large ones into two children (Inria's densify_and_clone /
        densify_and_split); the statistics start again.  dry_run only counts.  Returns (cloned, split)."""
        c, s = C.c_uint32(), C.c_uint32()
        capi.check(capi.lib.glic_mapper_densify(self._h, float(grad_threshold), float(percent_dense), float(scene_extent),
                                                int(bool(dry_run)), C.byref(c), C.byref(s)), "mapper_densify")
        return int(c.value), int(s.value)

    def densify_stats(self):
        """(accum [P], denom [P]) float32: the summed view-space gradient norms and the number of views that saw each row."""
        P = int(self.stats().num_gaussians)
        acc, den = np.zeros(P, np.float32), np.zeros(P, np.float32)
        capi.check(capi.lib.glic_mapper_densify_stats(self._h, _p(acc) if P else acc.ctypes.data_as(C.c_void_p),
                                                      _p(den) if P else den.ctypes.data_as(C.c_void_p)), "mapper_densify_stats")
        return acc, den

    def screen_radii(self):
        """maxr [P] int32: the largest screen radius each row has had in a stepped view since the statistics last restarted."""
        P = int(self.stats().num_gaussians)
        out = np.zeros(max(P, 1), np.int32)
        capi.check(capi.lib.glic_mapper_screen_radii(self._h, out.ctypes.data_as(C.c_void_p)), "mapper_screen_radii")
        return out[:P]

    def reset_opacity(self, max_opacity=RESET_OPACITY):
        """Inria's reset_opacity on the non-sky rows: logits above max_opacity drop to it, the opacity moments become zero."""
        capi.check(capi.lib.glic_mapper_reset_opacity(self._h, float(max_opacity)), "mapper_reset_opacity")

    def densify_and_prune(self, scene_extent, grad_threshold=DENSIFY_GRAD_THRESHOLD, percent_dense=PERCENT_DENSE, min_opacity=0.0,
                          max_screen_radius=0, max_world_scale=0.0, dry_run=False):
        """densify() and then the removal of the result's rows with act(logit) < min_opacity, or (non-sky) maxr >
        max_screen_radius > 0, or largest scale > max_world_scale > 0, in one compaction.  dry_run only counts.  Returns
        {cloned, split, pruned, rows}."""
        p = capi.DensityParams(float(grad_threshold), float(percent_dense), float(scene_extent), float(min_opacity), int(max_screen_radius),
                               float(max_world_scale))
        out = capi.DensityCounts()
        capi.check(capi.lib.glic_mapper_densify_and_prune(self._h, C.byref(p), int(bool(dry_run)), C.byref(out)), "mapper_densify_and_prune")
        return {k: int(getattr(out, k)) for k, _ in capi.DensityCounts._fields_}

    def set_density_schedule(self, **fields):
        """Run density control inside optimize(): densify_and_prune every densify_interval iterations in (densify_from,
        densify_until), reset_opacity every opacity_reset_interval.  Fields not given take Inria's defaults (DENSITY_SCHEDULE)."""
        unknown = set(fields) - set(DENSITY_SCHEDULE)
        if unknown:
            raise TypeError("unknown schedule fields: %s" % sorted(unknown))
        s = capi.DensitySchedule(**dict(DENSITY_SCHEDULE, **fields))
        capi.check(capi.lib.glic_mapper_set_density_schedule(self._h, C.byref(s)), "mapper_set_density_schedule")

    def clear_density_schedule(self):
        capi.check(capi.lib.glic_mapper_set_density_schedule(self._h, None), "mapper_set_density_schedule")

    def scene_extent(self):
        """getNerfppNorm's radius over the training keyframes' current camera centres."""
        out = C.c_float()
        capi.check(capi.lib.glic_mapper_scene_extent(self._h, C.byref(out)), "mapper_scene_extent")
        return out.value

    def density_totals(self):
        """What the schedule has done since it was set: {cloned, split, pruned, rows, steps, resets}."""
        out, steps, resets = capi.DensityCounts(), C.c_uint32(), C.c_uint32()
        capi.check(capi.lib.glic_mapper_density_totals(self._h, C.byref(out), C.byref(steps), C.byref(resets)), "mapper_density_totals")
        d = {k: int(getattr(out, k)) for k, _ in capi.DensityCounts._fields_}
        d.update(steps=int(steps.value), resets=int(resets.value))
        return d

    # ---- multi-GPU wiring: torch.distributed (or anything else) only carries the 64-byte handles --------------------------
    def export_handle(self):
        h = C.create_string_buffer(64)
        capi.check(capi.lib.glic_mapper_export(self._h, h), "mapper_export")
        return h.raw

    def connect(self, handles):
        blob = b"".join(handles)
        assert len(blob) == 64 * self.cfg.world
        capi.check(capi.lib.glic_mapper_connect(self._h, blob), "mapper_connect")

"""Host-side mirror of the reference's operator interface for the rasterizer hot path.

Two faces, both plumbing over libglic_b200.so (no compute here, no fallback):

* the LibTorch shim (csrc/torch_shim.cpp -> glic_b200_torch.so) exports the reference's C++ symbols
  RasterizeGaussiansCUDA / RasterizeGaussiansBackwardCUDA / adamUpdate / fusedssim /
  fusedssim_backward / distCUDA2 (reference rasterizer/rasterize_points.h:25-96,
  fused-ssim/ssim.h:7-26, simple-knn/spatial.h:14); the functions of the same names below call them;
* `GaussianRasterizerFunction`, `GaussianRasterizer`, `FusedSSIMMap`, `fused_ssim`, `l1_loss`,
  `SparseGaussianAdam` restate, in Python, the reference's C++ callers (rasterizer/rasterizer.cpp:21-216,
  loss_utils.h:30-33,135-193, optim_utils.h:69-137) so that tests read like uses of the reference;
* `CRasterizer` drives the C ABI directly through ctypes with persistent workspaces (bench / parity tests).
"""
import ctypes as C
import importlib.util
import os

import torch

from . import capi

PKG = os.path.dirname(os.path.abspath(__file__))
_SHIM = None


def shim():
    """The pybind face of glic_b200_torch.so (the reference-symbol LibTorch shim)."""
    global _SHIM
    if _SHIM is None:
        path = os.path.join(PKG, "glic_b200_torch.so")
        if not os.path.isfile(path):
            raise ImportError("gaussian_lic_b200: %s is missing; build it with "
                              "`python gaussian_lic_b200/build.py --torch`. No fallback exists." % path)
        spec = importlib.util.spec_from_file_location("glic_b200_torch", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _SHIM = mod
    return _SHIM


# ---- the six boundary functions (same names, argument order and meaning as the reference) ------
def RasterizeGaussiansCUDA(*args):
    return shim().RasterizeGaussiansCUDA(*args)


def RasterizeGaussiansBackwardCUDA(*args):
    return shim().RasterizeGaussiansBackwardCUDA(*args)


def adamUpdate(param, param_grad, exp_avg, exp_avg_sq, visible, lr, b1, b2, eps, N, M):
    return shim().adamUpdate(param, param_grad, exp_avg, exp_avg_sq, visible, lr, b1, b2, eps, N, M)


def fusedssim(C1, C2, img1, img2, train):
    return shim().fusedssim(C1, C2, img1, img2, train)


def fusedssim_backward(C1, C2, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12):
    return shim().fusedssim_backward(C1, C2, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)


def distCUDA2(points):
    return shim().distCUDA2(points)


# ---- reference callers restated (rasterizer.h:27-73, rasterizer.cpp:21-216) -----------------------
class GaussianRasterizationSettings:
    def __init__(self, image_height, image_width, tanfovx, tanfovy, limx_neg, limx_pos, limy_neg, limy_pos, bg,
                 scale_modifier, viewmatrix, projmatrix, sh_degree, campos, prefiltered=False, debug=False,
                 no_color=False, lambda_erank=0.0):
        self.image_height, self.image_width = int(image_height), int(image_width)
        self.tanfovx, self.tanfovy = float(tanfovx), float(tanfovy)
        self.limx_neg, self.limx_pos, self.limy_neg, self.limy_pos = map(float, (limx_neg, limx_pos, limy_neg, limy_pos))
        self.bg, self.scale_modifier = bg, float(scale_modifier)
        self.viewmatrix, self.projmatrix, self.campos = viewmatrix, projmatrix, campos
        self.sh_degree, self.prefiltered, self.debug, self.no_color = int(sh_degree), prefiltered, debug, no_color
        self.lambda_erank = float(lambda_erank)


class GaussianRasterizerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, dc, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs):
        (num_rendered, num_buckets, color, final_T, radii, geomBuffer, binningBuffer, imgBuffer,
         sampleBuffer) = RasterizeGaussiansCUDA(
            rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
            rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, rs.limx_neg,
            rs.limx_pos, rs.limy_neg, rs.limy_pos, dc, sh, rs.sh_degree, rs.campos, rs.prefiltered, rs.debug, rs.no_color)
        ctx.rs, ctx.num_rendered, ctx.num_buckets = rs, num_rendered, num_buckets
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, dc, sh, geomBuffer,
                              binningBuffer, imgBuffer, sampleBuffer)
        ctx.mark_non_differentiable(radii, final_T)
        return color, radii, final_T

    @staticmethod
    def backward(ctx, dL_dcolor, _dradii, _dfinal_T):
        rs = ctx.rs
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, dc, sh, geomBuffer, binningBuffer, imgBuffer,
         sampleBuffer) = ctx.saved_tensors
        (dL_dmeans2D, dL_dcolors_precomp, dL_dopacities, dL_dmeans3D, dL_dcov3Ds_precomp, dL_ddc, dL_dsh, dL_dscales,
         dL_drotations) = RasterizeGaussiansBackwardCUDA(
            rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix,
            rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.limx_neg, rs.limx_pos, rs.limy_neg, rs.limy_pos,
            dL_dcolor.contiguous(), dc, sh, rs.sh_degree, rs.campos, geomBuffer, ctx.num_rendered, binningBuffer,
            imgBuffer, ctx.num_buckets, sampleBuffer, rs.lambda_erank, False)
        # rasterizer.cpp:171-182 (grads of the two *_precomp inputs are dropped: they are empty tensors)
        return dL_dmeans3D, dL_dmeans2D, dL_ddc, dL_dsh, None, dL_dopacities, dL_dscales, dL_drotations, None, None


class GaussianRasterizer(torch.nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def forward(self, means3D, means2D, opacities, dc, shs, scales, rotations):
        empty = torch.empty(0, device=means3D.device)                       # rasterizer.cpp:200-201
        return GaussianRasterizerFunction.apply(means3D, means2D, dc, shs, empty, opacities, scales, rotations, empty,
                                                self.raster_settings)


# ---- loss (loss_utils.h:30-33,130-193) ---------------------------------------------------------------
SSIM_C1 = 0.01 ** 2
SSIM_C2 = 0.03 ** 2


def l1_loss(network_output, gt):
    return torch.abs(network_output - gt).mean()


class FusedSSIMMap(torch.autograd.Function):
    @staticmethod
    def forward(ctx, C1, C2, img1, img2):
        ssim_map, dm_dmu1, dm_dsigma1_sq, dm_dsigma12 = fusedssim(C1, C2, img1, img2, True)
        ctx.save_for_backward(img1.detach(), img2, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)
        ctx.C1, ctx.C2 = C1, C2
        return ssim_map

    @staticmethod
    def backward(ctx, dL_dmap):
        img1, img2, dm_dmu1, dm_dsigma1_sq, dm_dsigma12 = ctx.saved_tensors
        grad = fusedssim_backward(ctx.C1, ctx.C2, img1, img2, dL_dmap.contiguous(), dm_dmu1, dm_dsigma1_sq, dm_dsigma12)
        return None, None, grad, None


def fused_ssim(img1, img2):
    return FusedSSIMMap.apply(SSIM_C1, SSIM_C2, img1, img2).mean()


def l1_ssim_loss_exposure(img, gt, E, lambda_dssim=0.2, grad=True, scratch=None, stream=None):
    """The photometric loss on the exposed image out_c = E[0][c] r + E[1][c] g + E[2][c] b + E[c][3] (glic_l1_ssim_loss_exposure).
    img, gt: [3,H,W] float32 CUDA tensors; E: [3,4] (or 12) float32 CUDA tensor.  Returns (loss[1], dL_dimg[3,H,W], dL_dE[3,4]);
    the two gradients are None when grad is False.  dL_dE is deterministic (fixed-order float64 sums)."""
    _, H, W = img.shape
    assert img.shape[0] == 3 and gt.shape == img.shape and E.numel() == 12
    need = capi.lib.glic_loss_exposure_scratch_bytes(H, W)
    if scratch is None or scratch.numel() < need:
        scratch = torch.empty(need, dtype=torch.uint8, device=img.device)
    f32 = dict(dtype=torch.float32, device=img.device)
    loss = torch.empty(1, **f32)
    dL_dimg = torch.empty(3, H, W, **f32) if grad else None
    dL_dE = torch.empty(3, 4, **f32) if grad else None
    capi.check(capi.lib.glic_l1_ssim_loss_exposure(H, W, lambda_dssim, capi.ptr(img), capi.ptr(gt), capi.ptr(E.contiguous()),
                                                   capi.ptr(loss), capi.ptr(dL_dimg), capi.ptr(dL_dE), capi.ptr(scratch),
                                                   scratch.numel(), stream), "l1_ssim_loss_exposure")
    return loss, dL_dimg, dL_dE


def lpips(img, gt, weights, scratch=None, stream=None):
    """LPIPS (AlexNet) of two [3,H,W] float32 CUDA tensors (glic_lpips; both are clamped to [0,1] inside).  weights: the float32
    CUDA payload of a weight file (lpips_weights.read).  Returns a [1] tensor; no host synchronisation."""
    _, H, W = img.shape
    assert img.shape[0] == 3 and gt.shape == img.shape
    need = capi.lib.glic_lpips_scratch_bytes(H, W)
    if scratch is None or scratch.numel() < need:
        scratch = torch.empty(max(need, 1), dtype=torch.uint8, device=img.device)
    out = torch.empty(1, dtype=torch.float32, device=img.device)
    capi.check(capi.lib.glic_lpips(H, W, capi.ptr(img.contiguous()), capi.ptr(gt.contiguous()), capi.ptr(weights), capi.ptr(out),
                                   capi.ptr(scratch), scratch.numel(), stream), "lpips")
    return out


def lidar_init(points, colors, depth_rsp, scaling_scale, focal, stream=None):
    """initialize()'s LiDAR rows (glic_lidar_init).  points [n,3] float32, colors [n,3] float64 (rgb / 255.0), depth_rsp [n]
    float32, all CUDA tensors; scaling_scale and focal = (fx + fy) / 2 are doubles.  Returns the raw parameters
    dict(xyz [n,3], f_dc [n,3], log_scale [n,3], rot [n,4], opacity_logit [n]); f_rest is zero and not returned."""
    n = int(points.shape[0])
    assert points.dtype == torch.float32 and colors.dtype == torch.float64 and depth_rsp.dtype == torch.float32
    f32 = dict(dtype=torch.float32, device=points.device)
    out = dict(xyz=torch.empty(n, 3, **f32), f_dc=torch.empty(n, 3, **f32), log_scale=torch.empty(n, 3, **f32),
               rot=torch.empty(n, 4, **f32), opacity_logit=torch.empty(n, **f32))
    capi.check(capi.lib.glic_lidar_init(n, capi.ptr(points.contiguous()), capi.ptr(colors.contiguous()), capi.ptr(depth_rsp.contiguous()),
                                        float(scaling_scale), float(focal), *[capi.ptr(out[k]) for k in ("xyz", "f_dc", "log_scale", "rot",
                                                                                                          "opacity_logit")], stream),
               "lidar_init")
    return out


def skybox_init(n, radius, seed, device="cuda:0", uniforms=False, stream=None):
    """initialize()'s n sky rows (glic_skybox_init) keyed by seed, as the raw-parameter dict lidar_init returns; uniforms=True
    adds the generator's draws as uv [n,2] (u1, u2 per row)."""
    f32 = dict(dtype=torch.float32, device=device)
    out = dict(xyz=torch.empty(n, 3, **f32), f_dc=torch.empty(n, 3, **f32), log_scale=torch.empty(n, 3, **f32),
               rot=torch.empty(n, 4, **f32), opacity_logit=torch.empty(n, **f32))
    if uniforms:
        out["uv"] = torch.empty(n, 2, **f32)
    need = capi.lib.glic_skybox_init_bytes(int(n))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
    capi.check(capi.lib.glic_skybox_init(int(n), int(radius), int(seed), capi.ptr(ws), need,
                                         *[capi.ptr(out[k]) for k in ("xyz", "f_dc", "log_scale", "rot", "opacity_logit")],
                                         capi.ptr(out.get("uv")), stream), "skybox_init")
    return out


# ---- meshing (include/glic_b200.h "Meshing") -------------------------------------------------------------------------
def tsdf_grid(origin, voxel_size, dims, device="cuda:0", stream=None):
    """A cleared TSDF grid: returns (capi.TsdfGrid, its data tensor).  The data is planar tsdf[N] | weight[N] | colour[3][N]
    float32, N = nx ny nz, lattice point (i, j, k) at index i + nx (j + ny k); view it with tsdf_planes()."""
    d = (C.c_int * 3)(*[int(x) for x in dims])
    nbytes = capi.lib.glic_tsdf_bytes(d)
    if not nbytes:
        raise capi.GlicError("tsdf_grid: every dimension must be in [2, 2048], with fewer than 2^31 lattice points")
    data = torch.empty(nbytes // 4, dtype=torch.float32, device=device)
    g = capi.TsdfGrid()
    g.origin[:] = [float(x) for x in origin]
    g.voxel_size, g.dims[:], g.data = float(voxel_size), [int(x) for x in dims], data.data_ptr()
    capi.check(capi.lib.glic_tsdf_clear(C.byref(g), stream), "tsdf_clear")
    return g, data


def tsdf_planes(data, dims):
    """(tsdf [nz,ny,nx], weight [nz,ny,nx], colour [3,nz,ny,nx]) views of a grid's data tensor"""
    nx, ny, nz = (int(x) for x in dims)
    N = nx * ny * nz
    return data[:N].view(nz, ny, nx), data[N:2 * N].view(nz, ny, nx), data[2 * N:].view(3, nz, ny, nx)


def tsdf_integrate(grid, viewmatrix, W, H, fx, fy, cx, cy, depth, rgb=None, mask_words=None, words_per_row=0, trunc=0.1, max_depth=0.0,
                   stream=None):
    """Fuse one view into grid (glic_tsdf_integrate).  viewmatrix: 16 column-major float32 CUDA values of a camera block;
    depth [H,W], rgb [3,H,W] (None: colour untouched) float32 CUDA tensors; mask_words (optional) a glic_pack_mask int32 CUDA
    tensor of words_per_row words per row.  Asynchronous."""
    capi.check(capi.lib.glic_tsdf_integrate(C.byref(grid), capi.ptr(viewmatrix.contiguous()), int(W), int(H), float(fx), float(fy),
                                            float(cx), float(cy), capi.ptr(depth.contiguous()),
                                            capi.ptr(None if rgb is None else rgb.contiguous()), capi.ptr(mask_words),
                                            int(words_per_row), float(trunc), float(max_depth), stream), "tsdf_integrate")


def mesh_extract(grid, device="cuda:0", stream=None):
    """Surface nets of grid (glic_mesh_count + glic_mesh_extract): returns CUDA tensors (xyz [V,3] float32, rgb [V,3] uint8,
    faces [F,3] int32).  Synchronises once, for the counts."""
    dev = torch.device(device)
    need = capi.lib.glic_mesh_scratch_bytes(grid.dims)
    scratch = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    counts = (C.c_uint64 * 2)()
    capi.check(capi.lib.glic_mesh_count(C.byref(grid), capi.ptr(scratch), need, counts, stream), "mesh_count")
    V, F = int(counts[0]), int(counts[1])
    xyz = torch.empty(max(V, 1), 3, dtype=torch.float32, device=dev)
    rgb = torch.empty(max(V, 1), 3, dtype=torch.uint8, device=dev)
    faces = torch.empty(max(F, 1), 3, dtype=torch.int32, device=dev)
    capi.check(capi.lib.glic_mesh_extract(C.byref(grid), capi.ptr(scratch), need, capi.ptr(xyz), capi.ptr(rgb), capi.ptr(faces), stream),
               "mesh_extract")
    return xyz[:V], rgb[:V], faces[:F]


# ---- sparse meshing (include/glic_b200.h "Sparse meshing") ----------------------------------------------------------
def block_set(capacity, device="cuda:0", stream=None):
    """An empty block set of `capacity` blocks: returns (capi.BlockSet, its data tensor)."""
    nbytes = capi.lib.glic_block_set_bytes(int(capacity))
    if not nbytes:
        raise capi.GlicError("block_set: capacity must be in [1, 2^24]")
    data = torch.empty(nbytes, dtype=torch.uint8, device=device)
    s = capi.BlockSet(int(capacity), data.data_ptr())
    capi.check(capi.lib.glic_block_set_clear(C.byref(s), stream), "block_set_clear")
    return s, data


def block_set_copy(src, dst, stream=None):
    """Rehash src into dst (a set of at least twice src's capacity; glic_block_set_copy).  Asynchronous."""
    capi.check(capi.lib.glic_block_set_copy(C.byref(src), C.byref(dst), stream), "block_set_copy")


def block_set_insert(set_, origin, voxel_size, viewmatrix, W, H, fx, fy, cx, cy, depth, mask_words=None, words_per_row=0, trunc=0.1,
                     max_depth=0.0, stream=None):
    """Add one view's blocks to set_ (glic_block_set_insert); arguments as tsdf_integrate takes them.  Synchronises and returns
    (blocks in the set, clipped pixels of this call, overflow)."""
    o = (C.c_float * 3)(*[float(x) for x in origin])
    cnt = (C.c_int64 * 3)()
    capi.check(capi.lib.glic_block_set_insert(C.byref(set_), o, float(voxel_size), capi.ptr(viewmatrix.contiguous()), int(W), int(H),
                                              float(fx), float(fy), float(cx), float(cy), capi.ptr(depth.contiguous()), capi.ptr(mask_words),
                                              int(words_per_row), float(trunc), float(max_depth), cnt, stream), "block_set_insert")
    torch.cuda.synchronize()
    return int(cnt[0]), int(cnt[1]), int(cnt[2])


def sparse_tsdf(origin, voxel_size, set_, n_blocks, device="cuda:0", stream=None):
    """The sparse grid of set_'s n_blocks blocks (its block count), cleared: returns (capi.SparseTsdf, its data tensor)."""
    nbytes = capi.lib.glic_sparse_tsdf_bytes(int(n_blocks))
    if not nbytes and n_blocks:
        raise capi.GlicError("sparse_tsdf: more than 2^23 - 1 blocks")
    data = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)
    g = capi.SparseTsdf()
    g.origin[:] = [float(x) for x in origin]
    g.voxel_size, g.n_blocks, g.data = float(voxel_size), int(n_blocks), data.data_ptr()
    capi.check(capi.lib.glic_sparse_tsdf_init(C.byref(g), C.byref(set_), stream), "sparse_tsdf_init")
    return g, data


def sparse_tsdf_integrate(grid, viewmatrix, W, H, fx, fy, cx, cy, depth, rgb=None, mask_words=None, words_per_row=0, trunc=0.1,
                          max_depth=0.0, stream=None):
    """Fuse one view into a sparse grid (glic_sparse_tsdf_integrate), as tsdf_integrate takes it.  Asynchronous."""
    capi.check(capi.lib.glic_sparse_tsdf_integrate(C.byref(grid), capi.ptr(viewmatrix.contiguous()), int(W), int(H), float(fx), float(fy),
                                                   float(cx), float(cy), capi.ptr(depth.contiguous()),
                                                   capi.ptr(None if rgb is None else rgb.contiguous()), capi.ptr(mask_words),
                                                   int(words_per_row), float(trunc), float(max_depth), stream), "sparse_tsdf_integrate")


def sparse_tsdf_planes(grid, device="cuda:0", stream=None):
    """(sorted block keys [n] int64, pool [n, 5, 512] float32: tsdf, weight, colour x3) of a sparse grid (glic_debug_sparse_tsdf)"""
    n = int(grid.n_blocks)
    keys = torch.empty(max(n, 1), dtype=torch.int64, device=device)
    pool = torch.empty(max(n, 1), 5, 512, dtype=torch.float32, device=device)
    capi.check(capi.lib.glic_debug_sparse_tsdf(C.byref(grid), capi.ptr(keys), capi.ptr(pool), stream), "debug_sparse_tsdf")
    return keys[:n], pool[:n]


def sparse_mesh_extract(grid, device="cuda:0", stream=None):
    """Surface nets of a sparse grid (glic_sparse_mesh_count + glic_sparse_mesh_extract): returns CUDA tensors (xyz [V,3] float32,
    rgb [V,3] uint8, faces [F,3] int32) and the capi.SparseMeshCounts.  Synchronises once, for the counts."""
    dev = torch.device(device)
    need = capi.lib.glic_sparse_mesh_scratch_bytes(grid.n_blocks)
    scratch = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    counts = capi.SparseMeshCounts()
    capi.check(capi.lib.glic_sparse_mesh_count(C.byref(grid), capi.ptr(scratch), need, C.byref(counts), stream), "sparse_mesh_count")
    V, F = int(counts.vertices), int(counts.faces)
    ws_bytes = capi.lib.glic_sparse_mesh_extract_bytes(V, F)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    xyz = torch.empty(max(V, 1), 3, dtype=torch.float32, device=dev)
    rgb = torch.empty(max(V, 1), 3, dtype=torch.uint8, device=dev)
    faces = torch.empty(max(F, 1), 3, dtype=torch.int32, device=dev)
    capi.check(capi.lib.glic_sparse_mesh_extract(C.byref(grid), capi.ptr(scratch), need, C.byref(counts), capi.ptr(ws), ws_bytes,
                                                 capi.ptr(xyz), capi.ptr(rgb), capi.ptr(faces), stream), "sparse_mesh_extract")
    return xyz[:V], rgb[:V], faces[:F], counts


# ---- render() and the model getters it uses (rasterizer/renderer.cpp:21-88; gaussian.cpp:147-175) ------------------
class GaussianParams:
    """The six raw parameter tensors of GaussianModel with its activation getters (sigmoid / exp / normalize)."""

    def __init__(self, xyz, features_dc, features_rest, opacity, scaling, rotation, sh_degree, lambda_erank=0.0):
        self.xyz_, self.features_dc_, self.features_rest_ = xyz, features_dc, features_rest
        self.opacity_, self.scaling_, self.rotation_ = opacity, scaling, rotation
        self.sh_degree_, self.lambda_erank_ = int(sh_degree), float(lambda_erank)

    def getXYZ(self):
        return self.xyz_

    def getOpacity(self):
        return torch.sigmoid(self.opacity_)

    def getScaling(self):
        return torch.exp(self.scaling_)

    def getRotation(self):
        return torch.nn.functional.normalize(self.rotation_)

    def getFeaturesDc(self):
        return self.features_dc_

    def getFeaturesRest(self):
        return self.features_rest_


def render(viewpoint_camera, pc, bg_color, no_color=False, scaling_modifier=1.0):
    """renderer.cpp:21-88.  viewpoint_camera: mapping with W, H, tanfovx, tanfovy, lims[4] and DEVICE tensors view[16|4x4],
    proj[16|4x4], campos[3] (column-major, as Camera stores the transposed matrices).  Returns the reference's tuple
    (rendered_image, rendered_final_T, screenspace_points, radii > 0, radii)."""
    xyz = pc.getXYZ()
    screenspace_points = torch.zeros_like(xyz, requires_grad=True)
    cam = viewpoint_camera
    lims = [float(x) for x in cam["lims"]]
    rs = GaussianRasterizationSettings(cam["H"], cam["W"], cam["tanfovx"], cam["tanfovy"], lims[0], lims[1], lims[2], lims[3],
                                       bg_color, scaling_modifier, cam["view"].view(4, 4), cam["proj"].view(4, 4),
                                       pc.sh_degree_, cam["campos"], False, False, no_color, pc.lambda_erank_)
    rendered_image, radii, rendered_final_T = GaussianRasterizer(rs)(xyz, screenspace_points, pc.getOpacity(), pc.getFeaturesDc(),
                                                                     pc.getFeaturesRest(), pc.getScaling(), pc.getRotation())
    return rendered_image, rendered_final_T, screenspace_points, radii > 0, radii


# ---- optimiser (optim_utils.h:69-137; gaussian.cpp:399-424) ---------------------------------------------
class SparseGaussianAdam:
    """One tensor per group, visibility-masked, no bias correction, eps = 1e-15."""

    def __init__(self, params_and_lrs, eps=1e-15):
        self.groups = [dict(param=p, lr=float(lr), exp_avg=None, exp_avg_sq=None, step=0) for p, lr in params_and_lrs]
        self.eps = eps
        self.visibility, self.N = None, 0

    def set_visibility_and_N(self, visibility, N):
        self.visibility, self.N = visibility, int(N)

    @torch.no_grad()
    def step(self):
        for g in self.groups:
            p = g["param"]
            if p.grad is None:
                continue
            if g["exp_avg"] is None:
                g["exp_avg"], g["exp_avg_sq"] = torch.zeros_like(p), torch.zeros_like(p)
            M = p.numel() // self.N
            adamUpdate(p, p.grad, g["exp_avg"], g["exp_avg_sq"], self.visibility, g["lr"], 0.9, 0.999, self.eps, self.N, M)
            g["step"] += 1

    def zero_grad(self):
        for g in self.groups:
            g["param"].grad = None


# ---- direct C-ABI driver (ctypes) ------------------------------------------------------------------------
class CRasterizer:
    """Persistent-workspace driver of the C ABI for one image size.  Device memory = torch tensors."""

    def __init__(self, W, H, device="cuda:0"):
        self.W, self.H, self.dev = int(W), int(H), torch.device(device)
        self.lib = capi.lib
        u8 = dict(dtype=torch.uint8, device=self.dev)
        self.image_ws = torch.empty(self.lib.glic_image_bytes(self.W, self.H), **u8)
        self.geom_ws = torch.empty(0, **u8)
        self.binning_ws = torch.empty(0, **u8)
        self.sample_ws = torch.empty(0, **u8)
        self.det_ws = torch.empty(0, **u8)       # glic_backward_deterministic's workspace, grown on first use
        self.loss_scratch = torch.empty(self.lib.glic_loss_scratch_bytes(3, self.H, self.W), **u8)
        self.R = 0
        self.B = 0
        self.P = 0
        self.cap = 0            # capacity (pairs) the binning / sample workspaces are carved with
        self.cap_target = 0
        self.stream = None      # cudaStream_t handle (int) or None = legacy default stream
        self.counters = torch.zeros(3, dtype=torch.int64).pin_memory() if torch.cuda.is_available() else torch.zeros(3, dtype=torch.int64)
        self._view_keep = []    # device tensors behind every View handed out (a View only holds raw pointers)

    def _grow(self, name, nbytes, slack=1.25):
        t = getattr(self, name)
        if t.numel() < nbytes:
            setattr(self, name, torch.empty(int(nbytes * slack) + 256, dtype=torch.uint8, device=self.dev))
        return getattr(self, name)

    def make_view(self, cam):
        """cam: dict from synthetic.make_camera (numpy) or tensors already on the device."""
        def dev(x):
            return x if isinstance(x, torch.Tensor) else torch.as_tensor(x, dtype=torch.float32).to(self.dev)
        v, p, c = dev(cam["view"]), dev(cam["proj"]), dev(cam["campos"])
        lims = [float(x) for x in cam["lims"]]
        view = capi.View(v.data_ptr(), p.data_ptr(), c.data_ptr(), cam["tanfovx"], cam["tanfovy"], lims[0], lims[1],
                         lims[2], lims[3], self.W, self.H)
        self._view_keep.append((v, p, c))
        return view

    def forward(self, g, view, no_color=False, scale_modifier=1.0, out_color=None, out_T=None, radii=None, sync=True):
        """One asynchronous glic_forward call.  g: dict of device tensors means[P,3] scales[P,3] rots[P,4] opacity[P]
        dc[P,3] sh[P,M,3] + degree.  The binning / sample workspaces are sized by a capacity that grows on overflow;
        with sync=False nothing blocks (call finish() before trusting R/B or after a scene change)."""
        lib = self.lib
        P = int(g["means"].shape[0])
        M = int(g["sh"].shape[1]) if g["sh"].numel() else 0
        self.P, self.M, self.D = P, M, int(g["degree"])
        f32 = dict(dtype=torch.float32, device=self.dev)
        out_color = torch.empty(3, self.H, self.W, **f32) if out_color is None else out_color
        out_T = torch.empty(self.H, self.W, **f32) if out_T is None else out_T
        radii = torch.empty(max(P, 1), dtype=torch.int32, device=self.dev) if radii is None else radii
        self._grow("geom_ws", lib.glic_geom_bytes(P))
        if self.cap_target == 0:
            self.cap_target = max(8 * P, 1 << 16)
        while True:
            self._grow("binning_ws", lib.glic_binning_bytes(self.cap_target), slack=1.0)
            if not no_color:
                self._grow("sample_ws", lib.glic_sample_bytes(self.cap_target, self.W, self.H), slack=1.0)
            self.cap = int(lib.glic_binning_capacity(self.binning_ws.numel(), self.sample_ws.numel(), self.W, self.H, int(no_color)))
            capi.check(lib.glic_forward(
                P, self.D, M, capi.ptr(g["means"]), capi.ptr(g["scales"]), scale_modifier, capi.ptr(g["rots"]),
                capi.ptr(g["opacity"]), capi.ptr(g["dc"]), capi.ptr(g["sh"]) if M else None, C.byref(view), int(no_color),
                capi.ptr(radii), capi.ptr(self.geom_ws), self.geom_ws.numel(), capi.ptr(self.image_ws),
                self.image_ws.numel(), capi.ptr(self.binning_ws), self.binning_ws.numel(),
                None if no_color else capi.ptr(self.sample_ws), self.sample_ws.numel(), capi.ptr(out_color), capi.ptr(out_T),
                capi.ptr(self.counters), self.stream), "forward")
            if not sync:
                break
            if not self.finish():
                break
        return out_color, out_T, radii[:P]

    def render(self, g, view, scale_modifier=1.0, depth=True, median_depth=True, radii=None):
        """One glic_render call (the inference form of the forward: no sample workspace, nothing saved for a backward) at
        this rasterizer's size, synchronised; an overflow grows the binning workspace and draws again.  It draws into the
        workspaces forward() saves its state in, so a backward() belongs to the forward() before any render().  Returns a dict of
        device tensors: color [3,H,W], final_T [H,W], depth [H,W] (unnormalised expected depth) and median_depth [H,W] when
        asked for, radii [P], and counters (R, B = 0, overflow) of the last call."""
        lib = self.lib
        P = int(g["means"].shape[0])
        M = int(g["sh"].shape[1]) if g["sh"].numel() else 0
        f32 = dict(dtype=torch.float32, device=self.dev)
        out = dict(color=torch.empty(3, self.H, self.W, **f32), final_T=torch.empty(self.H, self.W, **f32),
                   depth=torch.empty(self.H, self.W, **f32) if depth else None,
                   median_depth=torch.empty(self.H, self.W, **f32) if median_depth else None)
        radii = torch.empty(max(P, 1), dtype=torch.int32, device=self.dev) if radii is None else radii
        self._grow("geom_ws", lib.glic_geom_bytes(P))
        if self.cap_target == 0:
            self.cap_target = max(8 * P, 1 << 16)
        while True:
            self._grow("binning_ws", lib.glic_binning_bytes(self.cap_target), slack=1.0)
            capi.check(lib.glic_render(
                P, int(g["degree"]), M, capi.ptr(g["means"]), capi.ptr(g["scales"]), scale_modifier, capi.ptr(g["rots"]),
                capi.ptr(g["opacity"]), capi.ptr(g["dc"]), capi.ptr(g["sh"]) if M else None, C.byref(view), capi.ptr(radii),
                capi.ptr(self.geom_ws), self.geom_ws.numel(), capi.ptr(self.image_ws), self.image_ws.numel(),
                capi.ptr(self.binning_ws), self.binning_ws.numel(), capi.ptr(out["color"]), capi.ptr(out["final_T"]),
                capi.ptr(out["depth"]), capi.ptr(out["median_depth"]), capi.ptr(self.counters), self.stream), "render")
            torch.cuda.synchronize(self.dev)
            R, B, ovf = (int(x) for x in self.counters.tolist())
            if not ovf:
                break
            self.cap_target = int(R * 1.25) + 4096
        out["radii"], out["counters"] = radii[:P], (R, B, ovf)
        return out

    def contribution(self, g, view, max_weight, hits, ends=None, scale_modifier=1.0, final_T=False, radii=None):
        """One glic_contribution call at this rasterizer's size, synchronised: the view's contribution scores ADDED to max_weight
        [P] float32 (max), hits [P] int64 (sum of taken pixels) and, when given, ends [P] int64 (sum of pixels the row ends)
        device tensors; an overflow grows the binning workspace and
        draws again (the overflowed call added nothing).  It draws into the workspaces forward() uses and publishes R as finish()
        does, so debug_state() shows this call's lists.  Returns final_T [H,W] (a device tensor) when asked for, else None."""
        lib = self.lib
        P = int(g["means"].shape[0])
        out_T = torch.empty(self.H, self.W, dtype=torch.float32, device=self.dev) if final_T else None
        radii = torch.empty(max(P, 1), dtype=torch.int32, device=self.dev) if radii is None else radii
        self._grow("geom_ws", lib.glic_geom_bytes(P))
        if self.cap_target == 0:
            self.cap_target = max(8 * P, 1 << 16)
        while True:
            self._grow("binning_ws", lib.glic_binning_bytes(self.cap_target), slack=1.0)
            self.cap = int(lib.glic_binning_capacity(self.binning_ws.numel(), 0, self.W, self.H, 1))
            capi.check(lib.glic_contribution(
                P, capi.ptr(g["means"]), capi.ptr(g["scales"]), scale_modifier, capi.ptr(g["rots"]), capi.ptr(g["opacity"]),
                C.byref(view), capi.ptr(radii), capi.ptr(self.geom_ws), self.geom_ws.numel(), capi.ptr(self.image_ws),
                self.image_ws.numel(), capi.ptr(self.binning_ws), self.binning_ws.numel(), capi.ptr(max_weight), capi.ptr(hits),
                capi.ptr(ends), capi.ptr(out_T), capi.ptr(self.counters), self.stream), "contribution")
            self.P = P
            if not self.finish():
                break
        return out_T

    def finish(self):
        """Synchronise, publish R / B, and grow the capacity if the last forward overflowed (returns True then)."""
        torch.cuda.synchronize(self.dev)
        R, B, ovf = (int(x) for x in self.counters.tolist())
        self.R, self.B = R, B
        if ovf:
            self.cap_target = int(R * 1.25) + 4096
            return True
        return False

    def alloc_grads(self, P=None, M=None):
        P = self.P if P is None else P
        M = self.M if M is None else M
        f32 = dict(dtype=torch.float32, device=self.dev)
        return dict(dL_dmeans2D=torch.empty(P, 3, **f32), dL_dconic=torch.empty(P, 4, **f32),
                    dL_dopacity=torch.empty(P, 1, **f32), dL_dcolors=torch.empty(P, 3, **f32),
                    dL_dmeans3D=torch.empty(P, 3, **f32), dL_dcov3D=torch.empty(P, 6, **f32),
                    dL_ddc=torch.empty(P, 1, 3, **f32), dL_dsh=torch.empty(P, M, 3, **f32),
                    dL_dscales=torch.empty(P, 3, **f32), dL_drots=torch.empty(P, 4, **f32))

    def backward(self, g, view, radii, dL_dpix, grads=None, scale_modifier=1.0, lambda_erank=0.0, deterministic=False):
        """glic_backward on the saved state of the last forward; deterministic=True: glic_backward_deterministic (bit-identical
        outputs across calls on the same state, contributions added in ascending tile order)."""
        grads = self.alloc_grads() if grads is None else grads
        args = [self.P, self.D, self.M, capi.ptr(g["means"]), capi.ptr(g["scales"]), scale_modifier, capi.ptr(g["rots"]),
                capi.ptr(g["dc"]), capi.ptr(g["sh"]) if self.M else None, C.byref(view), capi.ptr(radii), self.cap,
                capi.ptr(self.geom_ws), capi.ptr(self.binning_ws), capi.ptr(self.image_ws), capi.ptr(self.sample_ws),
                capi.ptr(dL_dpix), lambda_erank, capi.ptr(grads["dL_dmeans2D"]), capi.ptr(grads["dL_dconic"]),
                capi.ptr(grads["dL_dopacity"]), capi.ptr(grads["dL_dcolors"]), capi.ptr(grads["dL_dmeans3D"]),
                capi.ptr(grads["dL_dcov3D"]), capi.ptr(grads["dL_ddc"]), capi.ptr(grads["dL_dsh"]) if self.M else None,
                capi.ptr(grads["dL_dscales"]), capi.ptr(grads["dL_drots"])]
        if deterministic:
            ws = self._grow("det_ws", self.lib.glic_deterministic_bytes(self.cap, self.W, self.H), slack=1.0)
            capi.check(self.lib.glic_backward_deterministic(*args, capi.ptr(ws), ws.numel(), self.stream), "backward_deterministic")
        else:
            capi.check(self.lib.glic_backward(*args, self.stream), "backward")
        return grads

    def loss(self, img, gt, lambda_dssim=0.2, loss_out=None, dL_dimg=None):
        f32 = dict(dtype=torch.float32, device=self.dev)
        loss_out = torch.empty(1, **f32) if loss_out is None else loss_out
        dL_dimg = torch.empty_like(img) if dL_dimg is None else dL_dimg
        capi.check(self.lib.glic_l1_ssim_loss(3, self.H, self.W, lambda_dssim, capi.ptr(img), capi.ptr(gt),
                                              capi.ptr(loss_out), capi.ptr(dL_dimg), capi.ptr(self.loss_scratch),
                                              self.loss_scratch.numel(), self.stream), "l1_ssim_loss")
        return loss_out, dL_dimg

    BWD_COUNTERS = ("live_buckets", "splats", "splats_taken", "visits", "visits_taken", "candidate_pixels", "taken_pixels",
                    "fallback_pixels")

    def render_backward(self, view, dL_dpix, grads, exact=False, counters=None):
        """The render backward alone on the saved state of the last forward (glic_debug_render_backward), accumulating into
        grads' four 2-D gradient tensors (zero them first).  exact=True: the former kernel body.  counters: a zeroed [8]
        int64 device tensor selects the counting form, which adds BWD_COUNTERS to it."""
        capi.check(self.lib.glic_debug_render_backward(
            self.P, C.byref(view), self.cap, capi.ptr(self.geom_ws), capi.ptr(self.binning_ws), capi.ptr(self.image_ws),
            capi.ptr(self.sample_ws), capi.ptr(dL_dpix), capi.ptr(grads["dL_dmeans2D"]), capi.ptr(grads["dL_dconic"]),
            capi.ptr(grads["dL_dopacity"]), capi.ptr(grads["dL_dcolors"]), int(exact), capi.ptr(counters), self.stream),
            "debug_render_backward")

    def deterministic_entries(self, view, dL_dpix, grads):
        """The deterministic render backward alone on the saved state of the last forward (glic_debug_deterministic_entries):
        writes grads' four 2-D gradient tensors and returns the ordered entry list as device tensors gid [n] int32, tile [n]
        int32 and values [n, 9] float32 (mean.x, mean.y, conic.x, conic.y, conic.w, colour r, g, b, opacity), in the order the
        reduction adds them."""
        ws = self._grow("det_ws", self.lib.glic_deterministic_bytes(self.cap, self.W, self.H), slack=1.0)
        cap = 32 * max(int(self.lib.glic_max_buckets(self.cap, self.W, self.H)), 1)
        gid = torch.empty(cap, dtype=torch.int32, device=self.dev)
        tile = torch.empty(cap, dtype=torch.int32, device=self.dev)
        values = torch.empty(cap, 9, dtype=torch.float32, device=self.dev)
        n = C.c_int64(0)
        capi.check(self.lib.glic_debug_deterministic_entries(
            self.P, C.byref(view), self.cap, capi.ptr(self.geom_ws), capi.ptr(self.binning_ws), capi.ptr(self.image_ws),
            capi.ptr(self.sample_ws), capi.ptr(dL_dpix), capi.ptr(ws), ws.numel(), capi.ptr(grads["dL_dmeans2D"]),
            capi.ptr(grads["dL_dconic"]), capi.ptr(grads["dL_dopacity"]), capi.ptr(grads["dL_dcolors"]), C.byref(n), capi.ptr(gid),
            capi.ptr(tile), capi.ptr(values), self.stream), "debug_deterministic_entries")
        n = int(n.value)
        return gid[:n], tile[:n], values[:n]

    # ---- introspection for parity tests -------------------------------------------------------------------
    def debug_state(self):
        lib, P, R, W, H = self.lib, self.P, self.R, self.W, self.H
        T = ((W + 15) // 16) * ((H + 15) // 16)
        dev = self.dev
        d = dict(depth=torch.empty(P, device=dev), xy=torch.empty(P, 2, device=dev),
                 conic_opacity=torch.empty(P, 4, device=dev), rgb=torch.empty(P, 3, device=dev),
                 tiles_touched=torch.empty(P, dtype=torch.int32, device=dev),
                 offsets=torch.empty(P, dtype=torch.int32, device=dev),
                 clamped=torch.empty(P, 3, dtype=torch.uint8, device=dev),
                 point_list=torch.empty(R, dtype=torch.int32, device=dev),
                 keys_sorted=torch.empty(R, dtype=torch.int64, device=dev),
                 ranges=torch.empty(T, 2, dtype=torch.int32, device=dev),
                 bucket_offsets=torch.empty(T, dtype=torch.int32, device=dev),
                 n_contrib=torch.empty(H * W, dtype=torch.int32, device=dev),
                 max_contrib=torch.empty(T, dtype=torch.int32, device=dev))
        capi.check(lib.glic_debug_geom(P, capi.ptr(self.geom_ws), capi.ptr(d["depth"]), capi.ptr(d["xy"]),
                                       capi.ptr(d["conic_opacity"]), capi.ptr(d["rgb"]), capi.ptr(d["tiles_touched"]),
                                       capi.ptr(d["offsets"]), capi.ptr(d["clamped"]), None), "debug_geom")
        capi.check(lib.glic_debug_binning(P, capi.ptr(self.geom_ws), self.cap, R, capi.ptr(self.binning_ws), capi.ptr(d["point_list"]),
                                          capi.ptr(d["keys_sorted"]), None), "debug_binning")
        cnt = (C.c_int64 * 2)()
        capi.check(lib.glic_debug_image(W, H, capi.ptr(self.image_ws), capi.ptr(d["ranges"]),
                                        capi.ptr(d["bucket_offsets"]), capi.ptr(d["n_contrib"]),
                                        capi.ptr(d["max_contrib"]), cnt, None), "debug_image")
        spans = (C.c_uint32 * 2)()
        capi.check(lib.glic_debug_spans(P, capi.ptr(self.geom_ws), spans, None), "debug_spans")
        torch.cuda.synchronize(dev)
        d["R"], d["B"] = int(cnt[0]), int(cnt[1])
        d["span_count"], d["span_cap"] = int(spans[0]), int(spans[1])
        return d

    def debug_render_state(self, R):
        """debug_state() of the lists the last render() drew, R = its counters[0]: glic_render carves the binning workspace
        with the capacity glic_binning_capacity(binning_bytes, 0, W, H, 1), which need not be the forward's.  The rasterizer's
        own R and capacity (those of the last forward, which backward() uses) are left as they were."""
        saved = self.R, self.cap
        self.R, self.cap = int(R), int(self.lib.glic_binning_capacity(self.binning_ws.numel(), 0, self.W, self.H, 1))
        try:
            return self.debug_state()
        finally:
            self.R, self.cap = saved


def sort_pairs(keys, vals, end_bit):
    """Stable sort of (int64-viewed u64 keys, int32-viewed u32 values) device tensors on bits [0,end_bit)."""
    n = keys.numel()
    lib = capi.lib
    k_in, v_in = keys.clone(), vals.clone()
    k_out, v_out = torch.empty_like(keys), torch.empty_like(vals)
    temp = torch.empty(lib.glic_sort_temp_bytes(n), dtype=torch.uint8, device=keys.device)
    capi.check(lib.glic_sort_pairs_u64_u32(n, end_bit, capi.ptr(k_in), capi.ptr(v_in), capi.ptr(k_out), capi.ptr(v_out),
                                           capi.ptr(temp), temp.numel(), None), "sort_pairs")
    return k_out, v_out


def scene_to_device(g, device="cuda:0"):
    """numpy scene dict (synthetic.make_gaussians) -> dict of contiguous float32 device tensors."""
    out = {}
    for k in ("means", "scales", "rots", "opacity", "dc", "sh"):
        out[k] = torch.as_tensor(g[k], dtype=torch.float32).contiguous().to(device)
    out["degree"] = int(g["degree"])
    return out

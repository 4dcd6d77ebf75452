"""ctypes bindings of the C ABI (include/glic_b200.h) -- plumbing only.

Device memory comes from torch tensors (`tensor.data_ptr()`); every byte of compute happens in
libglic_b200.so.  There is no fallback: if the library is missing, import fails loudly.
"""
import ctypes as C
import os

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "libglic_b200.so")

GLIC_OK = 0


class GlicError(RuntimeError):
    pass


class View(C.Structure):
    _fields_ = [("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float),
                ("limx_neg", C.c_float), ("limx_pos", C.c_float), ("limy_neg", C.c_float), ("limy_pos", C.c_float),
                ("width", C.c_int), ("height", C.c_int)]


class MapperConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("sh_degree", C.c_int), ("position_lr", C.c_float), ("feature_lr", C.c_float), ("opacity_lr", C.c_float),
                ("scaling_lr", C.c_float), ("rotation_lr", C.c_float), ("lambda_dssim", C.c_float), ("scaling_scale", C.c_float),
                ("capacity", C.c_uint32), ("max_iters", C.c_int), ("seed", C.c_uint64), ("rank", C.c_int), ("world", C.c_int),
                ("views_per_rank", C.c_int)]


class Keyframe(C.Structure):
    _fields_ = [("R_wc", C.c_float * 9), ("t_wc", C.c_float * 3), ("image", C.c_void_p)]


class Frame(C.Structure):
    _fields_ = [("q_wc", C.c_double * 4), ("t_wc", C.c_double * 3), ("bgr", C.c_void_p), ("row_bytes", C.c_size_t), ("n_points", C.c_int),
                ("xyz", C.c_void_p), ("rgb", C.c_void_p)]


class FrameStats(C.Structure):
    _fields_ = [("frames", C.c_uint32), ("train", C.c_uint32), ("test", C.c_uint32), ("pending_points", C.c_uint32),
                ("image_bytes", C.c_uint64)]


class MapperStats(C.Structure):
    _fields_ = [("num_gaussians", C.c_uint32), ("capacity", C.c_uint32), ("iterations", C.c_uint64), ("last_inserted", C.c_uint32),
                ("last_loss", C.c_float), ("mean_visible", C.c_double), ("overflow_regrows", C.c_uint32), ("ms_extend", C.c_float),
                ("ms_optimize", C.c_float)]


class DensityParams(C.Structure):
    _fields_ = [("grad_threshold", C.c_float), ("percent_dense", C.c_float), ("scene_extent", C.c_float), ("min_opacity", C.c_float),
                ("max_screen_radius", C.c_int32), ("max_world_scale", C.c_float)]


class DensityCounts(C.Structure):
    _fields_ = [("cloned", C.c_uint32), ("split", C.c_uint32), ("pruned", C.c_uint32), ("rows", C.c_uint32)]


class DensitySchedule(C.Structure):
    _fields_ = [("densify_from", C.c_uint32), ("densify_until", C.c_uint32), ("densify_interval", C.c_uint32),
                ("opacity_reset_interval", C.c_uint32), ("grad_threshold", C.c_float), ("percent_dense", C.c_float),
                ("min_opacity", C.c_float), ("reset_opacity", C.c_float), ("screen_radius", C.c_int32),
                ("world_scale_factor", C.c_float), ("scene_extent", C.c_float)]


class AlignParams(C.Structure):
    _fields_ = [("iterations", C.c_int), ("lr_translation", C.c_float), ("lr_rotation", C.c_float), ("exposure_lr", C.c_float),
                ("split", C.c_int)]


class AlignResult(C.Structure):
    _fields_ = [("R_wc", C.c_float * 9), ("t_wc", C.c_float * 3), ("E", C.c_float * 12), ("psnr", C.c_float), ("ssim", C.c_float),
                ("lpips", C.c_float), ("first_loss", C.c_float), ("last_loss", C.c_float), ("pose_exp_avg", C.c_float * 6),
                ("pose_exp_avg_sq", C.c_float * 6), ("expo_exp_avg", C.c_float * 12), ("expo_exp_avg_sq", C.c_float * 12),
                ("steps", C.c_int), ("skipped", C.c_int)]


class RenderCamera(C.Structure):
    _fields_ = [("R_wc", C.c_float * 9), ("t_wc", C.c_float * 3), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float),
                ("cy", C.c_float), ("width", C.c_int), ("height", C.c_int)]


class UnseenParams(C.Structure):
    _fields_ = [("views", C.c_void_p), ("n_views", C.c_int), ("min_weight", C.c_float), ("min_hits", C.c_uint64), ("sky", C.c_int)]


class TsdfGrid(C.Structure):
    _fields_ = [("origin", C.c_float * 3), ("voxel_size", C.c_float), ("dims", C.c_int * 3), ("data", C.c_void_p)]


class MeshParams(C.Structure):
    _fields_ = [("views", C.c_void_p), ("n_views", C.c_int), ("origin", C.c_float * 3), ("voxel_size", C.c_float), ("dims", C.c_int * 3),
                ("trunc", C.c_float), ("max_depth", C.c_float)]


class MeshCounts(C.Structure):
    _fields_ = [("vertices", C.c_uint32), ("faces", C.c_uint32), ("observed_voxels", C.c_uint64)]


class BlockSet(C.Structure):
    _fields_ = [("capacity", C.c_uint32), ("data", C.c_void_p)]


class SparseTsdf(C.Structure):
    _fields_ = [("origin", C.c_float * 3), ("voxel_size", C.c_float), ("n_blocks", C.c_uint32), ("data", C.c_void_p)]


class SparseMeshCounts(C.Structure):
    _fields_ = [("vertices", C.c_uint32), ("faces", C.c_uint32), ("observed_voxels", C.c_uint64), ("blocks", C.c_uint32),
                ("clipped_pixels", C.c_uint32), ("lattice_lo", C.c_int32 * 3), ("lattice_hi", C.c_int32 * 3)]


class SparseMeshParams(C.Structure):
    _fields_ = [("views", C.c_void_p), ("n_views", C.c_int), ("origin", C.c_float * 3), ("voxel_size", C.c_float), ("trunc", C.c_float),
                ("max_depth", C.c_float), ("max_blocks", C.c_uint32)]


class RigidCorrection(C.Structure):
    _fields_ = [("R", C.c_double * 9), ("t", C.c_double * 3), ("q", C.c_double * 4), ("sh", C.c_double * 83)]


class PoseCorrection(C.Structure):
    _fields_ = [("is_train", C.c_int), ("index", C.c_int), ("R_wc", C.c_float * 9), ("t_wc", C.c_float * 3)]


def _load():
    if not os.path.isfile(LIB_PATH):
        raise ImportError(
            "gaussian_lic_b200: %s is missing. Build it with `python gaussian_lic_b200/build.py` "
            "(or __graft_entry__.build()); there is no CPU or PyTorch fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, sz, i64, i32, f32, u32 = C.c_void_p, C.c_size_t, C.c_int64, C.c_int, C.c_float, C.c_uint32
    sig = {
        "glic_last_error": (C.c_char_p, []),
        "glic_abi_version": (i32, []),
        "glic_launch_count": (C.c_uint64, []),
        "glic_profile_enable": (i32, [i32]),
        "glic_profile_read": (i32, [C.POINTER(C.c_float), C.POINTER(i32)]),
        "glic_geom_bytes": (sz, [i32]),
        "glic_image_bytes": (sz, [i32, i32]),
        "glic_binning_bytes": (sz, [i64]),
        "glic_sample_bytes": (sz, [i64, i32, i32]),
        "glic_max_buckets": (i64, [i64, i32, i32]),
        "glic_sort_temp_bytes": (sz, [i64]),
        "glic_loss_scratch_bytes": (sz, [i32, i32, i32]),
        "glic_knn_temp_bytes": (sz, [i32]),
        "glic_forward_preprocess": (i32, [i32, i32, i32, vp, vp, f32, vp, vp, vp, vp, C.POINTER(View), i32, vp, vp, sz,
                                          vp, sz, C.POINTER(i64), vp]),
        "glic_binning_capacity": (i64, [sz, sz, i32, i32, i32]),
        "glic_forward": (i32, [i32, i32, i32, vp, vp, f32, vp, vp, vp, vp, C.POINTER(View), i32, vp, vp, sz, vp, sz, vp, sz, vp, sz, vp, vp,
                               vp, vp]),
        "glic_render": (i32, [i32, i32, i32, vp, vp, f32, vp, vp, vp, vp, C.POINTER(View), vp, vp, sz, vp, sz, vp, sz, vp, vp, vp, vp,
                              vp, vp]),
        "glic_contribution": (i32, [i32, vp, vp, f32, vp, vp, C.POINTER(View), vp, vp, sz, vp, sz, vp, sz, vp, vp, vp, vp, vp, vp]),
        "glic_forward_render": (i32, [i32, C.POINTER(View), i32, i64, vp, vp, vp, sz, vp, sz, vp, vp, C.POINTER(i64), vp]),
        "glic_backward": (i32, [i32, i32, i32, vp, vp, f32, vp, vp, vp, C.POINTER(View), vp, i64, vp, vp, vp, vp, vp, f32,
                                vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "glic_deterministic_bytes": (sz, [i64, i32, i32]),
        "glic_backward_deterministic": (i32, [i32, i32, i32, vp, vp, f32, vp, vp, vp, C.POINTER(View), vp, i64, vp, vp, vp, vp, vp,
                                              f32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]),
        "glic_sort_pairs_u64_u32": (i32, [i64, i32, vp, vp, vp, vp, vp, sz, vp]),
        "glic_debug_sort_pairs_u32": (i32, [i64, i32, vp, vp, vp, vp, vp, vp, sz, vp]),
        "glic_adam_update": (i32, [vp, vp, vp, vp, vp, f32, f32, f32, f32, u32, u32, vp]),
        "glic_fused_ssim": (i32, [i32, i32, i32, i32, f32, f32, vp, vp, vp, vp, vp, vp, vp]),
        "glic_fused_ssim_backward": (i32, [i32, i32, i32, i32, f32, f32, vp, vp, vp, vp, vp, vp, vp, vp]),
        "glic_l1_ssim_loss": (i32, [i32, i32, i32, f32, vp, vp, vp, vp, vp, sz, vp]),
        "glic_loss_exposure_scratch_bytes": (sz, [i32, i32]),
        "glic_l1_ssim_loss_exposure": (i32, [i32, i32, f32, vp, vp, vp, vp, vp, vp, vp, sz, vp]),
        "glic_knn_mean_dist2": (i32, [i32, vp, vp, vp, sz, vp]),
        "glic_extend_bytes": (sz, [i32, i32, i32]),
        "glic_extend": (i32, [i32, vp, vp, vp, C.POINTER(f32), C.POINTER(f32), f32, f32, f32, f32, i32, i32, vp, f32, vp, sz, vp, vp,
                              vp, vp, vp, vp, C.POINTER(i32), vp]),
        "glic_lidar_init": (i32, [i32, vp, vp, vp, C.c_double, C.c_double, vp, vp, vp, vp, vp, vp]),
        "glic_skybox_init_bytes": (sz, [i32]),
        "glic_skybox_init": (i32, [i32, i32, C.c_uint64, vp, sz, vp, vp, vp, vp, vp, vp, vp]),
        "glic_decode_bgr8": (i32, [i32, i32, vp, vp, vp]),
        "glic_ply_bytes": (sz, [u32, u32]),
        "glic_ply_write": (i32, [C.c_char_p, u32, u32, vp, vp, vp, vp, vp, vp]),
        "glic_ply_write_packed": (i32, [C.c_char_p, u32, u32, vp]),
        "glic_ply_read_header": (i32, [C.c_char_p, C.POINTER(u32), C.POINTER(u32), C.POINTER(sz)]),
        "glic_ply_read": (i32, [C.c_char_p, u32, u32, vp, vp, vp, vp, vp, vp]),
        "glic_packed_floats": (sz, [u32, u32]),
        "glic_packed_offsets": (i32, [u32, u32, C.POINTER(sz)]),
        "glic_activations_forward": (i32, [i32, vp, vp, vp, vp, vp, vp, vp]),
        "glic_activations_backward": (i32, [i32, vp, vp, vp, vp, vp, vp, vp]),
        "glic_adam_update_packed": (i32, [vp, vp, vp, vp, vp, C.POINTER(f32), f32, f32, f32, u32, u32, vp]),
        "glic_p2p_buffer_bytes": (sz, [sz, sz]),
        "glic_p2p_model_bytes": (sz, [sz, sz]),
        "glic_p2p_reduce_adam": (i32, [i32, i32, C.POINTER(vp), u32, u32, vp, vp, C.POINTER(f32), f32, f32, f32, vp]),
        "glic_p2p_slice": (i32, [i32, i32, sz, sz, C.POINTER(sz)]),
        "glic_p2p_alloc": (i32, [sz, C.POINTER(vp), C.c_char_p]),
        "glic_p2p_open": (i32, [C.c_char_p, C.POINTER(vp)]),
        "glic_p2p_close": (i32, [vp]),
        "glic_p2p_free": (i32, [vp]),
        "glic_p2p_allreduce_mean": (i32, [i32, i32, C.POINTER(vp), sz, sz, vp]),
        "glic_p2p_check": (i32, [vp, sz, sz, vp]),
        "glic_eval_scratch_bytes": (sz, [i32, i32, i32]),
        "glic_eval_psnr_ssim": (i32, [i32, i32, i32, vp, vp, vp, vp, sz, vp]),
        "glic_mask_words_per_row": (i32, [i32]),
        "glic_pack_mask": (i32, [i32, i32, vp, vp, vp, vp]),
        "glic_loss_masked_scratch_bytes": (sz, [i32, i32]),
        "glic_l1_ssim_loss_masked": (i32, [i32, i32, f32, vp, vp, vp, vp, i32, i32, u32, i32, vp, vp, vp, vp, sz, vp]),
        "glic_eval_masked_scratch_bytes": (sz, [i32, i32, i32]),
        "glic_eval_psnr_ssim_masked": (i32, [i32, i32, i32, vp, vp, vp, vp, i32, i32, u32, i32, vp, vp, sz, vp]),
        "glic_lpips_weight_floats": (sz, []),
        "glic_lpips_read_weights": (i32, [C.c_char_p, vp]),
        "glic_lpips_scratch_bytes": (sz, [i32, i32]),
        "glic_lpips": (i32, [i32, i32, vp, vp, vp, vp, vp, sz, vp]),
        "glic_arena_append": (i32, [vp, vp, vp, u32, u32, u32, u32, vp, vp, vp, vp, vp, vp]),
        "glic_arena_regrow": (i32, [vp, u32, vp, u32, u32, u32, vp]),
        "glic_camera_block": (i32, [i32, i32, f32, f32, f32, f32, C.POINTER(f32), C.POINTER(f32), C.POINTER(f32)]),
        "glic_mapper_create": (i32, [C.POINTER(MapperConfig), C.POINTER(vp)]),
        "glic_mapper_destroy": (i32, [vp]),
        "glic_mapper_initialize": (i32, [vp, u32, vp, vp, vp, vp, vp, vp]),
        "glic_mapper_initialize_lidar": (i32, [vp, i32, vp, vp, vp, C.c_double, i32, i32]),
        "glic_mapper_sky_rows": (i32, [vp, C.POINTER(u32)]),
        "glic_mapper_add_keyframe": (i32, [vp, C.POINTER(Keyframe), i32]),
        "glic_mapper_extend": (i32, [vp, i32, vp, vp, vp]),
        "glic_mapper_optimize": (i32, [vp, C.POINTER(i32), i32]),
        "glic_mapper_sample_views": (i32, [vp, C.POINTER(i32), C.POINTER(i32)]),
        "glic_mapper_evaluate": (i32, [vp, i32, i32, C.POINTER(f32), C.POINTER(f32)]),
        "glic_mapper_load_lpips": (i32, [vp, C.c_char_p]),
        "glic_mapper_evaluate_lpips": (i32, [vp, i32, i32, C.POINTER(f32), C.POINTER(f32), C.POINTER(f32)]),
        "glic_mapper_render": (i32, [vp, i32, i32, vp]),
        "glic_mapper_save_map": (i32, [vp, C.c_char_p]),
        "glic_mapper_stats_get": (i32, [vp, C.POINTER(MapperStats)]),
        "glic_mapper_download": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "glic_mapper_prune": (i32, [vp, f32, i32, C.POINTER(u32)]),
        "glic_mapper_enable_densification": (i32, [vp]),
        "glic_mapper_densify": (i32, [vp, f32, f32, f32, i32, C.POINTER(u32), C.POINTER(u32)]),
        "glic_mapper_densify_stats": (i32, [vp, vp, vp]),
        "glic_densify_split": (i32, [i32, vp, vp, vp, C.c_uint64, C.c_uint64, u32, vp, vp, vp]),
        "glic_mapper_screen_radii": (i32, [vp, vp]),
        "glic_mapper_reset_opacity": (i32, [vp, f32]),
        "glic_mapper_densify_and_prune": (i32, [vp, C.POINTER(DensityParams), i32, C.POINTER(DensityCounts)]),
        "glic_mapper_set_density_schedule": (i32, [vp, C.POINTER(DensitySchedule)]),
        "glic_mapper_scene_extent": (i32, [vp, C.POINTER(f32)]),
        "glic_mapper_density_totals": (i32, [vp, C.POINTER(DensityCounts), C.POINTER(u32), C.POINTER(u32)]),
        "glic_mapper_export": (i32, [vp, C.c_char_p]),
        "glic_mapper_connect": (i32, [vp, C.c_char_p]),
        "glic_mapper_synchronize": (i32, [vp]),
        "glic_mapper_set_option": (i32, [vp, i32, i32]),
        "glic_mapper_enable_exposure": (i32, [vp, f32]),
        "glic_mapper_exposure_get": (i32, [vp, i32, C.POINTER(f32)]),
        "glic_mapper_exposure_set": (i32, [vp, i32, C.POINTER(f32)]),
        "glic_mapper_exposure_adam_state": (i32, [vp, i32, C.POINTER(f32), C.POINTER(f32), C.POINTER(i32)]),
        "glic_mapper_enable_pose_refinement": (i32, [vp, f32, f32]),
        "glic_mapper_pose_get": (i32, [vp, i32, C.POINTER(f32), C.POINTER(f32), C.POINTER(f32)]),
        "glic_mapper_pose_set": (i32, [vp, i32, C.POINTER(f32), C.POINTER(f32)]),
        "glic_mapper_pose_adam_state": (i32, [vp, i32, C.POINTER(f32), C.POINTER(f32), C.POINTER(i32)]),
        "glic_mapper_align": (i32, [vp, i32, i32, C.POINTER(AlignParams), C.POINTER(AlignResult), vp]),
        "glic_mapper_render_camera": (i32, [vp, C.POINTER(RenderCamera), i32, i32, vp, vp, vp, vp]),
        "glic_mapper_contribution": (i32, [vp, C.POINTER(i32), i32, vp, vp, vp]),
        "glic_mapper_prune_unseen": (i32, [vp, C.POINTER(UnseenParams), i32, C.POINTER(u32)]),
        "glic_mapper_enable_frames": (i32, [vp, i32, i32, i32]),
        "glic_mapper_add_frame": (i32, [vp, C.POINTER(Frame), C.POINTER(i32)]),
        "glic_mapper_keyframe_image": (i32, [vp, i32, i32, vp]),
        "glic_mapper_add_frame_masked": (i32, [vp, C.POINTER(Frame), vp, C.POINTER(i32)]),
        "glic_mapper_set_keyframe_mask": (i32, [vp, i32, i32, vp]),
        "glic_mapper_keyframe_mask": (i32, [vp, i32, i32, vp, C.POINTER(u32)]),
        "glic_mapper_frames_get": (i32, [vp, C.POINTER(FrameStats)]),
        "glic_tsdf_bytes": (sz, [C.POINTER(i32)]),
        "glic_tsdf_clear": (i32, [C.POINTER(TsdfGrid), vp]),
        "glic_tsdf_integrate": (i32, [C.POINTER(TsdfGrid), vp, i32, i32, f32, f32, f32, f32, vp, vp, vp, i32, f32, f32, vp]),
        "glic_mesh_scratch_bytes": (sz, [C.POINTER(i32)]),
        "glic_mesh_count": (i32, [C.POINTER(TsdfGrid), vp, sz, C.POINTER(C.c_uint64), vp]),
        "glic_mesh_extract": (i32, [C.POINTER(TsdfGrid), vp, sz, vp, vp, vp, vp]),
        "glic_mesh_ply_write": (i32, [C.c_char_p, u32, vp, vp, u32, vp]),
        "glic_mapper_extract_mesh": (i32, [vp, C.POINTER(MeshParams), C.POINTER(MeshCounts)]),
        "glic_mapper_mesh_get": (i32, [vp, C.POINTER(MeshCounts), vp, vp, vp]),
        "glic_mapper_save_mesh": (i32, [vp, C.c_char_p]),
        "glic_block_set_bytes": (sz, [u32]),
        "glic_block_set_clear": (i32, [C.POINTER(BlockSet), vp]),
        "glic_block_set_copy": (i32, [C.POINTER(BlockSet), C.POINTER(BlockSet), vp]),
        "glic_block_set_insert": (i32, [C.POINTER(BlockSet), C.POINTER(f32), f32, vp, i32, i32, f32, f32, f32, f32, vp, vp, i32, f32, f32,
                                        C.POINTER(C.c_int64), vp]),
        "glic_sparse_tsdf_bytes": (sz, [u32]),
        "glic_sparse_tsdf_init": (i32, [C.POINTER(SparseTsdf), C.POINTER(BlockSet), vp]),
        "glic_sparse_tsdf_integrate": (i32, [C.POINTER(SparseTsdf), vp, i32, i32, f32, f32, f32, f32, vp, vp, vp, i32, f32, f32, vp]),
        "glic_sparse_mesh_scratch_bytes": (sz, [u32]),
        "glic_sparse_mesh_extract_bytes": (sz, [u32, u32]),
        "glic_sparse_mesh_count": (i32, [C.POINTER(SparseTsdf), vp, sz, C.POINTER(SparseMeshCounts), vp]),
        "glic_sparse_mesh_extract": (i32, [C.POINTER(SparseTsdf), vp, sz, C.POINTER(SparseMeshCounts), vp, sz, vp, vp, vp, vp]),
        "glic_debug_sparse_tsdf": (i32, [C.POINTER(SparseTsdf), vp, vp, vp]),
        "glic_mapper_extract_mesh_sparse": (i32, [vp, C.POINTER(SparseMeshParams), C.POINTER(SparseMeshCounts)]),
        "glic_pose_correction_record": (i32, [C.POINTER(f32), C.POINTER(f32), C.POINTER(f32), C.POINTER(f32), i32,
                                              C.POINTER(RigidCorrection)]),
        "glic_sh_rotation": (i32, [C.POINTER(C.c_double), i32, C.POINTER(C.c_double)]),
        "glic_mapper_anchors": (i32, [vp, vp]),
        "glic_mapper_set_anchors": (i32, [vp, vp]),
        "glic_mapper_correct_poses": (i32, [vp, i32, C.POINTER(PoseCorrection), C.POINTER(u32)]),
        "glic_mapper_save_checkpoint": (i32, [vp, C.c_char_p]),
        "glic_mapper_checkpoint_config": (i32, [C.c_char_p, C.POINTER(MapperConfig)]),
        "glic_mapper_load_checkpoint": (i32, [vp, C.c_char_p]),
        "glic_debug_geom": (i32, [i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "glic_debug_binning": (i32, [i32, vp, i64, i64, vp, vp, vp, vp]),
        "glic_debug_image": (i32, [i32, i32, vp, vp, vp, vp, vp, C.POINTER(i64), vp]),
        "glic_debug_spans": (i32, [i32, vp, C.POINTER(u32), vp]),
        "glic_debug_render_backward": (i32, [i32, C.POINTER(View), i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp]),
        "glic_debug_deterministic_entries": (i32, [i32, C.POINTER(View), i64, vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp,
                                                   C.POINTER(i64), vp, vp, vp, vp]),
        "glic_debug_pose_backward": (i32, [i32, i32, i32, vp, vp, vp, vp, vp, vp, C.POINTER(View), vp, vp, vp, vp, vp, vp, i32, vp,
                                           vp, vp, vp]),
        "glic_debug_fail_allocation": (i32, [i32]),
        "glic_debug_mapper_allocations": (i64, []),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib, sorted(sig)


lib, SYMBOLS = _load()


def check(status, what):
    if status != GLIC_OK:
        raise GlicError("glic_b200 %s failed (%d): %s" % (what, status, lib.glic_last_error().decode()))


def ptr(t):
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def launch_count():
    return int(lib.glic_launch_count())


STAGES = ["preprocess", "emit", "sort", "ranges", "render_fwd", "loss_fwd", "loss_bwd", "render_bwd", "preprocess_bwd",
          "adam", "zero", "allreduce"]


def profile_enable(on=True):
    check(lib.glic_profile_enable(int(on)), "profile_enable")


def profile_read():
    """-> {stage: (total_ms, count)} since the last profile_enable(True)."""
    ms = (C.c_float * len(STAGES))()
    cnt = (C.c_int * len(STAGES))()
    check(lib.glic_profile_read(ms, cnt), "profile_read")
    return {n: (float(ms[i]), int(cnt[i])) for i, n in enumerate(STAGES)}

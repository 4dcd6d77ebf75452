// mapper_mesh.cu -- the native mapper's meshing: TSDF fusion of rendered median depth over a dense or a sparse block grid,
// and the last mesh (glic_mapper_extract_mesh, glic_mapper_extract_mesh_sparse, glic_mapper_mesh_get).
#include "mapper_state.cuh"
#include "mesh.cuh"
#include <algorithm>
#include <cmath>

namespace mapper_impl {

// ---- meshing (glic_mapper_extract_mesh) ------------------------------------------------------------------------------------
// the grid of p's geometry over `data`
glic_tsdf_grid mesh_grid(const glic_mesh_params& p, void* data) {
    glic_tsdf_grid g;
    for (int a = 0; a < 3; ++a) { g.origin[a] = p.origin[a]; g.dims[a] = p.dims[a]; }
    g.voxel_size = p.voxel_size;
    g.data = data;
    return g;
}

// keyframe kf drawn as glic_mapper_extract_mesh draws it, without the sky rows: its median depth into r.median and, with rgb,
// its clamped colour into r.rgb
int draw_mesh_view(glic_mapper* m, const Keyframe& kf, const RenderPlanes& r, bool rgb, const char* what) {
    const int W = m->cfg.width, H = m->cfg.height;
    MAP_TRY(draw_rows(m, m->n_sky, kf.view, r, nullptr, r.median));
    if (m->counters_host[2]) { set_error(std::string(what) + ": a view still overflows the binning workspace after regrowing it"); return GLIC_ERR_WORKSPACE; }
    if (rgb) MAP_TRY(launch_scored_image(H, W, r.color, nullptr, r.rgb, m->stream));
    return GLIC_OK;
}

// the checks both meshing entry points make of their grid and volume arguments (glic_mesh_params or glic_sparse_mesh_params) and of
// the map, each message led by the entry point's name `what`
template <typename Params>
int mesh_check(const glic_mapper* m, const Params& p, const char* what) {
    if (!(std::isfinite(p.voxel_size) && p.voxel_size > 0.0f) || !std::isfinite(p.origin[0]) || !std::isfinite(p.origin[1]) ||
        !std::isfinite(p.origin[2])) {
        set_error(std::string(what) + ": voxel_size must be finite and > 0, the origin finite"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!(std::isfinite(p.trunc) && p.trunc > 0.0f)) { set_error(std::string(what) + ": trunc must be finite and > 0"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!(std::isfinite(p.max_depth) && p.max_depth >= 0.0f)) {
        set_error(std::string(what) + ": max_depth must be finite and >= 0"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    MAP_TRY(views_check(m, p.views, p.n_views, what));
    if (m->P <= m->n_sky) { set_error(std::string(what) + ": the mapper has no non-sky rows"); return GLIC_ERR_INVALID_ARGUMENT; }
    return GLIC_OK;
}

// the new mesh of V vertices and F faces replaces the last one once `extract` has filled it
template <typename Extract>
int replace_mesh(glic_mapper* m, const glic_mesh_counts& c, Extract extract) {
    Dev<float> xyz;
    Dev<uint8_t> rgb;
    Dev<int32_t> faces;
    MAP_TRY(xyz.allocate(12 * (size_t)c.vertices));
    MAP_TRY(rgb.allocate(3 * (size_t)c.vertices));
    MAP_TRY(faces.allocate(12 * (size_t)c.faces));
    MAP_TRY(extract((float*)xyz, (uint8_t*)rgb, (int32_t*)faces));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    m->mesh_xyz = std::move(xyz);
    m->mesh_rgb = std::move(rgb);
    m->mesh_faces = std::move(faces);
    m->mesh_counts = c;
    m->mesh_ready = true;
    return GLIC_OK;
}

// glic_mapper_extract_mesh after its checks.  The grid and the scratch are this call's own; the render workspace is
// glic_mapper_render_camera's; the new mesh replaces the previous one only once it is complete.
int extract_mesh(glic_mapper* m, const glic_mesh_params& p, glic_mesh_counts* out) {
    const int W = m->cfg.width, H = m->cfg.height;
    cudaStream_t s = m->stream;
    MAP_TRY(poll_ring(m, true));
    MAP_TRY(reserve(m, m->render_ws, render_carve(nullptr, W, H, nullptr)));
    Buf grid_buf, scratch;
    MAP_TRY(grid_buf.allocate(glic_tsdf_bytes(p.dims)));
    MAP_TRY(scratch.allocate(glic_mesh_scratch_bytes(p.dims)));
    const glic_tsdf_grid grid = mesh_grid(p, grid_buf.raw());
    MAP_TRY(glic_tsdf_clear(&grid, s));
    RenderPlanes r;
    render_carve(m->render_ws, W, H, &r);
    MAP_TRY(activate(m));
    const int count = p.views ? p.n_views : (int)m->train.size();
    for (int q = 0; q < count; ++q) {
        const Keyframe& kf = m->train[p.views ? p.views[q] : q];
        MAP_TRY(draw_mesh_view(m, kf, r, true, "mapper_extract_mesh"));
        MAP_TRY(glic_tsdf_integrate(&grid, kf.cam_dev, W, H, m->cfg.fx, m->cfg.fy, m->cfg.cx, m->cfg.cy, r.median, r.rgb,
                                    kf.mask_valid ? (const uint32_t*)kf.mask : nullptr, mask_words_per_row(W), p.trunc, p.max_depth, s));
    }
    uint64_t t[3];
    MAP_TRY(mesh_count(grid, scratch.raw(), scratch.bytes(), t, s));
    if (t[1] > 0xFFFFFFFFull) { set_error("mapper_extract_mesh: more than 2^32 - 1 faces"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(replace_mesh(m, glic_mesh_counts{(uint32_t)t[0], (uint32_t)t[1], t[2]}, [&](float* xyz, uint8_t* rgb, int32_t* faces) {
        return glic_mesh_extract(&grid, scratch.raw(), scratch.bytes(), xyz, rgb, faces, s);
    }));
    if (out) *out = m->mesh_counts;
    return GLIC_OK;
}

// glic_mapper_extract_mesh_sparse after its checks: pass 1 builds the block set (grown and the insertion repeated on overflow),
// then the grid, pass 2 integrates, then count and extract.  The set, the grid and the scratch are this call's own.
constexpr uint32_t SPARSE_FIRST_CAPACITY = 1u << 16;
constexpr uint32_t SPARSE_MAX_BLOCKS = (1u << 23) - 1;  // glic_sparse_tsdf_bytes' largest grid; sets double up to 2^24

int extract_mesh_sparse(glic_mapper* m, const glic_sparse_mesh_params& p, glic_sparse_mesh_counts* out) {
    const int W = m->cfg.width, H = m->cfg.height;
    cudaStream_t s = m->stream;
    MAP_TRY(poll_ring(m, true));
    MAP_TRY(reserve(m, m->render_ws, render_carve(nullptr, W, H, nullptr)));
    Buf set_buf;
    MAP_TRY(set_buf.allocate(glic_block_set_bytes(SPARSE_FIRST_CAPACITY)));
    glic_block_set set{SPARSE_FIRST_CAPACITY, set_buf.raw()};
    MAP_TRY(glic_block_set_clear(&set, s));
    RenderPlanes r;
    render_carve(m->render_ws, W, H, &r);
    MAP_TRY(activate(m));
    const int count = p.views ? p.n_views : (int)m->train.size();
    const int words = mask_words_per_row(W);
    const uint64_t limit = p.max_blocks ? std::min(p.max_blocks, SPARSE_MAX_BLOCKS) : SPARSE_MAX_BLOCKS;
    uint64_t clipped = 0, blocks = 0;
    for (int q = 0; q < count; ++q) {
        const Keyframe& kf = m->train[p.views ? p.views[q] : q];
        MAP_TRY(draw_mesh_view(m, kf, r, false, "mapper_extract_mesh_sparse"));
        for (;;) {
            const int64_t* c = (const int64_t*)m->counters_host.raw();
            MAP_TRY(glic_block_set_insert(&set, p.origin, p.voxel_size, kf.cam_dev, W, H, m->cfg.fx, m->cfg.fy, m->cfg.cx, m->cfg.cy, r.median,
                                          kf.mask_valid ? (const uint32_t*)kf.mask : nullptr, words, p.trunc, p.max_depth,
                                          (int64_t*)m->counters_host.raw(), s));
            GLIC_CUDA_TRY(cudaStreamSynchronize(s));
            // the count is exact, and an overflow means more blocks than the capacity
            const bool over = c[2] != 0;
            blocks = (uint64_t)c[0];
            if ((over && set.capacity >= limit) || (!over && blocks > limit)) {
                set_error("mapper_extract_mesh_sparse: the map needs more than " + std::to_string(limit) + " blocks" +
                          (p.max_blocks ? " (max_blocks)" : ""));
                return GLIC_ERR_WORKSPACE;
            }
            if (!over) { clipped += (uint64_t)c[1]; break; }
            Buf bigger;
            MAP_TRY(bigger.allocate(glic_block_set_bytes(2 * set.capacity)));
            const glic_block_set next{2 * set.capacity, bigger.raw()};
            MAP_TRY(glic_block_set_copy(&set, &next, s));
            GLIC_CUDA_TRY(cudaStreamSynchronize(s));       // the old set is read until the copy ends
            set_buf = std::move(bigger);
            set = next;
        }
    }
    Buf grid_buf, scratch;
    MAP_TRY(grid_buf.allocate(glic_sparse_tsdf_bytes((uint32_t)blocks)));
    MAP_TRY(scratch.allocate(glic_sparse_mesh_scratch_bytes((uint32_t)blocks)));
    glic_sparse_tsdf grid;
    for (int a = 0; a < 3; ++a) grid.origin[a] = p.origin[a];
    grid.voxel_size = p.voxel_size;
    grid.n_blocks = (uint32_t)blocks;
    grid.data = grid_buf.raw();
    MAP_TRY(glic_sparse_tsdf_init(&grid, &set, s));
    for (int q = 0; q < count; ++q) {
        const Keyframe& kf = m->train[p.views ? p.views[q] : q];
        MAP_TRY(draw_mesh_view(m, kf, r, true, "mapper_extract_mesh_sparse"));
        MAP_TRY(glic_sparse_tsdf_integrate(&grid, kf.cam_dev, W, H, m->cfg.fx, m->cfg.fy, m->cfg.cx, m->cfg.cy, r.median, r.rgb,
                                           kf.mask_valid ? (const uint32_t*)kf.mask : nullptr, words, p.trunc, p.max_depth, s));
    }
    glic_sparse_mesh_counts c;
    MAP_TRY(glic_sparse_mesh_count(&grid, scratch.raw(), scratch.bytes(), &c, s));
    c.clipped_pixels = (uint32_t)std::min<uint64_t>(clipped, 0xFFFFFFFFull);
    Buf ws;
    MAP_TRY(ws.allocate(glic_sparse_mesh_extract_bytes(c.vertices, c.faces)));
    MAP_TRY(replace_mesh(m, glic_mesh_counts{c.vertices, c.faces, c.observed_voxels}, [&](float* xyz, uint8_t* rgb, int32_t* faces) {
        return glic_sparse_mesh_extract(&grid, scratch.raw(), scratch.bytes(), &c, ws.raw(), ws.bytes(), xyz, rgb, faces, s);
    }));
    if (out) *out = c;
    return GLIC_OK;
}

}  // namespace mapper_impl

extern "C" {

int glic_mapper_extract_mesh(glic_mapper* m, const glic_mesh_params* p, glic_mesh_counts* out) {
    if (!m || !p) { set_error("mapper_extract_mesh: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!glic_tsdf_bytes(p->dims)) {
        set_error("mapper_extract_mesh: every grid dimension must be in [2, 2048], with fewer than 2^31 lattice points"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    MAP_TRY(mesh_check(m, *p, "mapper_extract_mesh"));
    return extract_mesh(m, *p, out);
}

int glic_mapper_extract_mesh_sparse(glic_mapper* m, const glic_sparse_mesh_params* p, glic_sparse_mesh_counts* out) {
    if (!m || !p) { set_error("mapper_extract_mesh_sparse: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(mesh_check(m, *p, "mapper_extract_mesh_sparse"));
    return extract_mesh_sparse(m, *p, out);
}

int glic_mapper_mesh_get(glic_mapper* m, glic_mesh_counts* counts, float* xyz, uint8_t* rgb, int32_t* faces) {
    if (!m) { set_error("mapper_mesh_get: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (counts) *counts = m->mesh_counts;
    const size_t V = m->mesh_counts.vertices, F = m->mesh_counts.faces;
    if (xyz && V) GLIC_CUDA_TRY(cudaMemcpyAsync(xyz, m->mesh_xyz, 12 * V, cudaMemcpyDefault, m->stream));
    if (rgb && V) GLIC_CUDA_TRY(cudaMemcpyAsync(rgb, m->mesh_rgb, 3 * V, cudaMemcpyDefault, m->stream));
    if (faces && F) GLIC_CUDA_TRY(cudaMemcpyAsync(faces, m->mesh_faces, 12 * F, cudaMemcpyDefault, m->stream));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

int glic_mapper_save_mesh(glic_mapper* m, const char* path) {
    if (!m || !path) { set_error("mapper_save_mesh: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!m->mesh_ready) { set_error("mapper_save_mesh: no mesh extracted yet (glic_mapper_extract_mesh)"); return GLIC_ERR_INVALID_ARGUMENT; }
    const glic_mesh_counts c = m->mesh_counts;
    std::vector<float> xyz(3 * (size_t)c.vertices);
    std::vector<uint8_t> rgb(3 * (size_t)c.vertices);
    std::vector<int32_t> faces(3 * (size_t)c.faces);
    MAP_TRY(glic_mapper_mesh_get(m, nullptr, xyz.data(), rgb.data(), faces.data()));
    return glic_mesh_ply_write(path, c.vertices, xyz.data(), rgb.data(), c.faces, faces.data());
}

}  // extern "C"

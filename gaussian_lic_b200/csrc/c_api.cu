// c_api.cu -- extern "C" entry points of libglic_b200.so (include/glic_b200.h): argument
// validation, workspace carving, stage sequencing.  No torch types, no allocation, no exceptions.
#include "common.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

namespace glic {

static thread_local std::string g_error;
unsigned long long g_launches = 0;

void set_error(const std::string& s) { g_error = s; }

// ---- stage profiling ----------------------------------------------------------------------
namespace {
struct EvPair { cudaEvent_t a, b; };
bool g_prof = false;
std::vector<EvPair> g_pairs[GLIC_STAGE_COUNT];
std::vector<EvPair> g_pool;
}
bool profiling_on() { return g_prof; }
void profile_mark(int stage, bool begin, cudaStream_t s) {
    if (stage < 0 || stage >= GLIC_STAGE_COUNT) return;
    if (begin) {
        EvPair p;
        if (!g_pool.empty()) { p = g_pool.back(); g_pool.pop_back(); }
        else { cudaEventCreate(&p.a); cudaEventCreate(&p.b); }
        cudaEventRecord(p.a, s);
        g_pairs[stage].push_back(p);
    } else if (!g_pairs[stage].empty()) {
        cudaEventRecord(g_pairs[stage].back().b, s);
    }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static int check_view(const glic_view* v) {
    if (!v || !v->viewmatrix || !v->projmatrix || !v->campos) { set_error("view: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (v->width <= 0 || v->height <= 0) { set_error("view: non-positive image size"); return GLIC_ERR_INVALID_ARGUMENT; }
    const int64_t T = (int64_t)((v->width + TILE - 1) / TILE) * ((v->height + TILE - 1) / TILE);
    if (T > GLIC_MAX_TILES) {
        set_error("view: " + std::to_string(v->width) + "x" + std::to_string(v->height) + " has " + std::to_string(T) +
                  " tiles of 16x16, more than GLIC_MAX_TILES = " + std::to_string(GLIC_MAX_TILES));
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    return GLIC_OK;
}

static int fail(int status, const char* name, const char* what) {
    set_error(std::string(name) + ": " + what);
    return status;
}

// ---- debug copy-out kernels ---------------------------------------------------------------
__global__ void debug_geom_kernel(int P, GeomState g, float* depth, float* xy, float* conic_opacity, float* rgb,
                                  uint32_t* tiles, uint32_t* offsets, uint8_t* clamped) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float4 r0 = g.rec[3 * i], r1 = g.rec[3 * i + 1], r2 = g.rec[3 * i + 2];
    if (depth) depth[i] = r2.y;
    if (xy) { xy[2 * i] = r0.x; xy[2 * i + 1] = r0.y; }
    if (conic_opacity) { conic_opacity[4 * i] = r0.z; conic_opacity[4 * i + 1] = r0.w; conic_opacity[4 * i + 2] = r1.x; conic_opacity[4 * i + 3] = r1.y; }
    if (rgb) { rgb[3 * i] = r1.z; rgb[3 * i + 1] = r1.w; rgb[3 * i + 2] = r2.x; }
    if (tiles) tiles[i] = g.tiles[i];
    if (offsets) offsets[i] = g.offsets[i];
    if (clamped) { const unsigned c = g.clamped[i]; clamped[3 * i] = c & 1u; clamped[3 * i + 1] = (c >> 1) & 1u; clamped[3 * i + 2] = (c >> 2) & 1u; }
}

struct ZeroSpans {
    static constexpr int MAX = 5;
    uint32_t* p[MAX];
    size_t words[MAX];
};

__global__ void __launch_bounds__(256) fill_kernel(size_t n, float v, float* __restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) out[i] = v;
}

__global__ void __launch_bounds__(256) zero_spans_kernel(ZeroSpans z) {
    pdl_enter();
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (int k = 0; k < ZeroSpans::MAX; ++k)
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < z.words[k]; i += stride) z.p[k][i] = 0u;
}

__global__ void debug_keys_kernel(long long R, GeomState g, const uint32_t* tile_keys, const uint32_t* point_list, uint64_t* out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R) return;
    const uint32_t gid = point_list[i];
    out[i] = ((uint64_t)tile_keys[i] << 32) | (uint64_t)__float_as_uint(g.rec[3 * (size_t)gid + 2].y);
}

// the deterministic backward's entries in reduction order: sorted positions i < n whose key is a gid (the sentinels sort last)
__global__ void debug_det_entries_kernel(unsigned n, uint32_t P, const uint32_t* keys, const uint32_t* idx, const float* vals,
                                         const uint32_t* live_offsets, int T, uint32_t* gid, uint32_t* tile, float* values,
                                         unsigned int* n_valid) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || keys[i] >= P) return;
    const uint32_t e = idx[i], live = e / BUCKET;
    int lo = 0, hi = T - 1;                                  // first tile t with live_offsets[t] > live
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (live_offsets[mid] > live) hi = mid; else lo = mid + 1; }
    gid[i] = keys[i];
    tile[i] = (uint32_t)lo;
    for (int j = 0; j < 9; ++j) values[9 * (size_t)i + j] = vals[9 * (size_t)e + j];
    atomicAdd(n_valid, 1u);
}

int launch_zero_spans(std::initializer_list<ZeroSpan> spans, cudaStream_t s) {
    if (spans.size() > (size_t)ZeroSpans::MAX) { set_error("zero_spans: too many spans"); return GLIC_ERR_INVALID_ARGUMENT; }
    ZeroSpans z = {};
    size_t most = 0;
    int k = 0;
    for (const ZeroSpan& sp : spans) {
        z.p[k] = static_cast<uint32_t*>(sp.p);
        z.words[k] = sp.bytes / sizeof(uint32_t);
        most = std::max(most, z.words[k++]);
    }
    if (most == 0) return GLIC_OK;
    GLIC_LAUNCH_PDL(zero_spans_kernel, (unsigned)std::min<size_t>((most + 255) / 256, (size_t)NUM_SMS * 8), 256, 0, s, z);
    return GLIC_OK;
}

// The stages of glic_forward and glic_render up to the blend, on workspaces carved for `cap` pairs: preprocess, depth sort and scan,
// key emission, tile sort, tile ranges and, with `buckets`, the bucket offsets of the checkpoints.  Returns the ping-pong half that
// holds the sorted list, < 0 on error.
int bin_view(int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier, const float* rotations,
             const float* opacities, const float* dc, const float* sh, const ViewParams& vp, bool no_color, int* radii, GeomState g,
             BinningState bin, ImageState img, int64_t cap, bool buckets, cudaStream_t s) {
    const int T = vp.grid_x * vp.grid_y, bit = tile_sort_bits(T);
    // every word the binning counts into or reads as empty, in one launch: the geometry header, the look-back status words,
    // both sorts' histograms, tickets and status words, and the tile ranges
    if (int e = launch_zero_spans({{g.hdr, sizeof(GeomHeader)}, {g.scan_status, GeomState::scan_status_bytes(P)},
                                   {g.sort_temp, sort_prepare_bytes(P, 32)}, {bin.sort_temp, sort_prepare_bytes(cap, bit)},
                                   {img.ranges, sizeof(uint2) * (size_t)T}}, s)) return e;
    { StageTimer _t(GLIC_STAGE_PREPROCESS, s);
      if (int e = launch_preprocess_forward(P, sh_degree, M, means3D, scales, scale_modifier, rotations, opacities, dc, sh, vp,
                                            no_color, radii, g, s)) return e; }
    { StageTimer _t(GLIC_STAGE_SORT, s);
      const int cur0 = launch_sort_pairs32(P, 32, g.depth_keys, g.order, g.sort_temp, g.sort_temp_size, s, nullptr, /*hist_ready=*/true);
      if (cur0 < 0) return cur0;
      if (int e = launch_depth_scan(P, g, g.order[cur0], cap, s)) return e; }
    { StageTimer _t(GLIC_STAGE_EMIT, s);
      if (int e = launch_emit_keys(P, vp, g, bin.keys[0], bin.vals[0], cap, sort_hist(bin.sort_temp), bit, s)) return e; }
    int cur;
    { StageTimer _t(GLIC_STAGE_SORT, s);
      cur = launch_sort_pairs32(cap, bit, bin.keys, bin.vals, bin.sort_temp, bin.sort_temp_size, s, &g.hdr->r_eff, true);
      if (cur < 0) return cur; }
    { StageTimer _t(GLIC_STAGE_RANGES, s);
      if (int e = launch_tile_ranges(cap, g.hdr, bin.keys[cur], T, img, buckets, &bin.hdr->sorted_in_b, cur, s)) return e; }
    return cur;
}

// The Gaussians one draw preprocesses.  With no_color, dc and sh are not read.
struct Scene {
    int P, sh_degree, M;
    const float *means3D, *scales; float scale_modifier; const float *rotations, *opacities, *dc, *sh;
    bool no_color; int* radii;
};

// The scene checks of a draw, in the order they fire: the view and the sizes; then the SH coefficients and the image workspace;
// then, for P > 0 only, the inputs and the geometry workspace.  `name` prefixes every message.
static int check_sizes(const char* name, const glic_view* view, const Scene& sc) {
    if (int e = check_view(view)) return e;
    if (sc.P < 0 || sc.sh_degree < 0 || sc.sh_degree > 3 || sc.M < 0) return fail(GLIC_ERR_INVALID_ARGUMENT, name, "bad P / sh_degree / M");
    return GLIC_OK;
}
static int check_image(const char* name, const glic_view* view, const Scene& sc, const void* image_ws, size_t image_bytes) {
    if (!sc.no_color && (sc.sh_degree + 1) * (sc.sh_degree + 1) - 1 > sc.M)
        return fail(GLIC_ERR_INVALID_ARGUMENT, name, "sh has fewer coefficients than sh_degree needs");
    if (!image_ws || image_bytes < glic_image_bytes(view->width, view->height)) return fail(GLIC_ERR_WORKSPACE, name, "image workspace too small");
    return GLIC_OK;
}
static int check_inputs(const char* name, const Scene& sc, const void* geom_ws, size_t geom_bytes) {
    if (!sc.means3D || !sc.scales || !sc.rotations || !sc.opacities || !sc.radii ||
        (!sc.no_color && (!sc.dc || (sc.M > 0 && sc.sh_degree > 0 && !sc.sh)))) return fail(GLIC_ERR_INVALID_ARGUMENT, name, "null input pointer");
    if (!aligned16(sc.rotations)) return fail(GLIC_ERR_INVALID_ARGUMENT, name, "rotations must be 16-byte aligned");
    if (!geom_ws || geom_bytes < glic_geom_bytes(sc.P)) return fail(GLIC_ERR_WORKSPACE, name, "geometry workspace too small");
    return GLIC_OK;
}

// The blend form of a draw, as render_forward_kernel's FORM: training (glic_forward: with colour, the checkpoints into the sample
// workspace and the bucket offsets), inference (glic_render: colour and depth planes) or scoring (glic_contribution)
enum DrawForm { DRAW_TRAIN, DRAW_INFER, DRAW_SCORE };

// What one draw writes.  Null planes are not written.
struct Draw {
    const char* name;
    DrawForm form;
    float empty_T;                  // every pixel's T in an empty scene
    bool missing_output;            // the caller's own output check failed
    float *color, *final_T, *depth, *median_depth, *max_weight;
    uint64_t *hits, *ends;
    void* sample_ws;                // DRAW_TRAIN with colour only: the checkpoints
    size_t sample_bytes;
};

// The planes of an empty scene: T = d.empty_T, every other plane 0
static int write_empty(const Draw& d, size_t HW, cudaStream_t s) {
    if (d.final_T && d.empty_T == 0.f) {
        GLIC_CUDA_TRY(cudaMemsetAsync(d.final_T, 0, sizeof(float) * HW, s));
    } else if (d.final_T) {
        fill_kernel<<<(unsigned)std::min<size_t>((HW + 255) / 256, (size_t)NUM_SMS * 8), 256, 0, s>>>(HW, d.empty_T, d.final_T);
        GLIC_LAUNCH_CHECK();
    }
    if (d.color) GLIC_CUDA_TRY(cudaMemsetAsync(d.color, 0, sizeof(float) * 3 * HW, s));
    if (d.depth) GLIC_CUDA_TRY(cudaMemsetAsync(d.depth, 0, sizeof(float) * HW, s));
    if (d.median_depth) GLIC_CUDA_TRY(cudaMemsetAsync(d.median_depth, 0, sizeof(float) * HW, s));
    return GLIC_OK;
}

// glic_forward, glic_render and glic_contribution: the scene checks, then bin_view on workspaces carved for the largest capacity
// they hold, one blend and the counters {R, B, overflow} copied to counters_host
static int draw(const Draw& d, const Scene& sc, const glic_view* view, void* geom_ws, size_t geom_bytes, void* image_ws,
                size_t image_bytes, void* binning_ws, size_t binning_bytes, int64_t* counters_host, cudaStream_t s) {
    if (int e = check_sizes(d.name, view, sc)) return e;
    if (int e = check_image(d.name, view, sc, image_ws, image_bytes)) return e;
    if (d.missing_output) return fail(GLIC_ERR_INVALID_ARGUMENT, d.name, "null output");
    const ViewParams vp = make_view_params(view);
    ImageState img = ImageState::carve(image_ws, vp.W, vp.H);
    if (sc.P == 0) {
        if (int e = write_empty(d, (size_t)vp.W * vp.H, s)) return e;
        GLIC_CUDA_TRY(cudaMemsetAsync(img.hdr, 0, sizeof(ImageHeader), s));
    } else {
        if (int e = check_inputs(d.name, sc, geom_ws, geom_bytes)) return e;
        const bool samples = d.form == DRAW_TRAIN && !sc.no_color;
        const int64_t cap = glic_binning_capacity(binning_bytes, samples ? d.sample_bytes : 0, vp.W, vp.H, !samples);
        if (!binning_ws || cap < 1 || (samples && !d.sample_ws))
            return fail(GLIC_ERR_WORKSPACE, d.name, d.form == DRAW_TRAIN ? "binning / sample workspace missing or too small"
                                                                         : "binning workspace missing or too small");
        GeomState g = GeomState::carve(geom_ws, sc.P);
        BinningState bin = BinningState::carve(binning_ws, cap);
        SampleState smp = SampleState::carve(samples ? d.sample_ws : nullptr, samples ? glic_max_buckets(cap, vp.W, vp.H) : 0);
        const int cur = bin_view(sc.P, sc.sh_degree, sc.M, sc.means3D, sc.scales, sc.scale_modifier, sc.rotations, sc.opacities, sc.dc,
                                 sc.sh, vp, sc.no_color, sc.radii, g, bin, img, cap, samples, s);
        if (cur < 0) return cur;
        StageTimer _t(GLIC_STAGE_RENDER_FWD, s);
        const uint32_t* list = bin.vals[cur];
        const int e = d.form == DRAW_TRAIN ? launch_render_forward(vp, sc.no_color, list, g, img, smp, d.color, d.final_T, s)
                    : d.form == DRAW_INFER ? launch_render_infer(vp, list, g, img, d.color, d.final_T, d.depth, d.median_depth, s)
                                           : launch_render_score(vp, list, g, img, d.max_weight, d.hits, d.ends, d.final_T, s);
        if (e) return e;
    }
    if (counters_host) GLIC_CUDA_TRY(cudaMemcpyAsync(counters_host, img.hdr->counters, 3 * sizeof(long long), cudaMemcpyDeviceToHost, s));
    return GLIC_OK;
}

// The state a forward left for its backward in the caller's workspaces, carved for R pairs; the sorted list is bin.vals[cur]
struct Saved { GeomState g; ImageState img; BinningState bin; SampleState smp; int64_t max_buckets; int cur; };
static Saved carve_saved(int P, const ViewParams& vp, int64_t R, const void* geom_ws, const void* image_ws, const void* binning_ws,
                         const void* sample_ws) {
    const int64_t max_buckets = glic_max_buckets(R, vp.W, vp.H);
    return {GeomState::carve(const_cast<void*>(geom_ws), P), ImageState::carve(const_cast<void*>(image_ws), vp.W, vp.H),
            BinningState::carve(const_cast<void*>(binning_ws), R), SampleState::carve(const_cast<void*>(sample_ws), max_buckets),
            max_buckets, tile_sort_passes(vp.grid_x * vp.grid_y) & 1};
}

// The render backward of a saved forward: deterministic with det_ws (glic_deterministic_bytes), atomic without
static int render_backward(int P, const ViewParams& vp, const Saved& sv, void* det_ws, const float* dL_dpix, float* dL_dmeans2D,
                           float* dL_dconic, float* dL_dopacity, float* dL_dcolors, cudaStream_t s) {
    StageTimer _t(GLIC_STAGE_RENDER_BWD, s);
    const uint32_t* list = sv.bin.vals[sv.cur];
    if (det_ws)
        return launch_render_backward_det(P, vp, sv.max_buckets, list, sv.g, sv.img, sv.smp, DetState::carve(det_ws, sv.max_buckets),
                                          dL_dpix, dL_dmeans2D, dL_dconic, dL_dopacity, dL_dcolors, s);
    return launch_render_backward(P, vp, sv.max_buckets, list, sv.g, sv.img, sv.smp, dL_dpix, dL_dmeans2D, dL_dconic, dL_dopacity,
                                  dL_dcolors, s);
}

int backward_compact(int P, int sh_degree, int M, const float* means3D, const float* scales, const float* rotations, const float* sh,
                     const glic_view* view, const int* radii, int64_t R, const void* geom_ws, const void* binning_ws,
                     const void* image_ws, const void* sample_ws, const float* dL_dpix, float* dL_dmeans2D, float* dL_dconic,
                     float* dL_dopacity, float* dL_dcolors, const CompactGrads& cg, cudaEvent_t after_render, cudaStream_t s,
                     void* det_ws) {
    if (int e = check_view(view)) return e;
    if (P <= 0) return GLIC_OK;
    const ViewParams vp = make_view_params(view);
    const Saved sv = carve_saved(P, vp, R, geom_ws, image_ws, binning_ws, sample_ws);
    if (!cg.grads_zeroed) { StageTimer _t(GLIC_STAGE_ZERO, s);
    // conic | mean2D | opacity carved from ONE block (the mapper's capacity layout): one memset over the span when the slack
    // between the live prefixes is small, three otherwise
    const ptrdiff_t span = dL_dconic < dL_dmeans2D && dL_dmeans2D < dL_dopacity ? (dL_dopacity + P) - dL_dconic : -1;
    if (span > 0 && span <= 10 * (ptrdiff_t)P) {
        GLIC_CUDA_TRY(cudaMemsetAsync(dL_dconic, 0, sizeof(float) * (size_t)span, s));
    } else {
        GLIC_CUDA_TRY(cudaMemsetAsync(dL_dmeans2D, 0, sizeof(float) * 3 * (size_t)P, s));
        GLIC_CUDA_TRY(cudaMemsetAsync(dL_dconic, 0, sizeof(float) * 4 * (size_t)P, s));
        GLIC_CUDA_TRY(cudaMemsetAsync(dL_dopacity, 0, sizeof(float) * (size_t)P, s));
    }
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dcolors, 0, sizeof(float) * 3 * (size_t)P, s)); }
    if (R > 0)
        if (int e = render_backward(P, vp, sv, det_ws, dL_dpix, dL_dmeans2D, dL_dconic, dL_dopacity, dL_dcolors, s)) return e;
    // the colour gradients are final here: the multi-GPU push may start while the per-Gaussian backward still runs
    if (after_render) GLIC_CUDA_TRY(cudaEventRecord(after_render, s));
    StageTimer _t(GLIC_STAGE_PREPROCESS_BWD, s);
    return launch_preprocess_backward_compact(P, sh_degree, M, means3D, scales, 1.0f, rotations, sh, vp, radii, sv.g, dL_dmeans2D,
                                              dL_dconic, dL_dcolors, cg, s);
}

}  // namespace glic

using namespace glic;

extern "C" {

const char* glic_last_error(void) { return g_error.c_str(); }
int glic_abi_version(void) { return GLIC_ABI_VERSION; }
uint64_t glic_launch_count(void) { return g_launches; }

int glic_profile_enable(int on) {
    for (int i = 0; i < GLIC_STAGE_COUNT; ++i) { for (auto& p : g_pairs[i]) g_pool.push_back(p); g_pairs[i].clear(); }
    g_prof = on != 0;
    return GLIC_OK;
}
int glic_profile_read(float* ms_host, int* count_host) {
    if (!ms_host || !count_host) { set_error("profile_read: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    for (int i = 0; i < GLIC_STAGE_COUNT; ++i) {
        float tot = 0.f; int n = 0;
        for (auto& p : g_pairs[i]) {
            if (cudaEventSynchronize(p.b) != cudaSuccess) { cudaGetLastError(); continue; }
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) { tot += ms; ++n; } else cudaGetLastError();
        }
        ms_host[i] = tot; count_host[i] = n;
    }
    return GLIC_OK;
}

size_t glic_geom_bytes(int P) { size_t b = 0; GeomState::carve(nullptr, P > 0 ? P : 0, &b); return b; }
size_t glic_image_bytes(int width, int height) { size_t b = 0; ImageState::carve(nullptr, width, height, &b); return b; }
size_t glic_binning_bytes(int64_t R) { size_t b = 0; BinningState::carve(nullptr, R, &b); return b; }
int64_t glic_max_buckets(int64_t R, int width, int height) {
    // B = sum_t ceil(n_t/32) <= floor(R/32) + min(T, R): at most one partial bucket per non-empty tile
    const int64_t T = (int64_t)((width + TILE - 1) / TILE) * ((height + TILE - 1) / TILE);
    return R / BUCKET + std::min<int64_t>(T, R);
}
size_t glic_sample_bytes(int64_t R, int width, int height) {
    size_t b = 0;
    SampleState::carve(nullptr, glic_max_buckets(R, width, height), &b);
    return b;
}
size_t glic_sort_temp_bytes(int64_t n) { return sort_temp_bytes(n); }

int glic_forward_preprocess(int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier,
                            const float* rotations, const float* opacities, const float* dc, const float* sh,
                            const glic_view* view, int no_color, int* radii, void* geom_ws, size_t geom_bytes,
                            void* image_ws, size_t image_bytes, int64_t* num_rendered_host, void* stream) {
    const char* name = "forward_preprocess";
    const Scene sc{P, sh_degree, M, means3D, scales, scale_modifier, rotations, opacities, dc, sh, no_color != 0, radii};
    if (int e = check_sizes(name, view, sc)) return e;
    if (!num_rendered_host) return fail(GLIC_ERR_INVALID_ARGUMENT, name, "num_rendered_host is NULL");
    *num_rendered_host = 0;
    if (int e = check_image(name, view, sc, image_ws, image_bytes)) return e;
    if (P == 0) return GLIC_OK;
    if (int e = check_inputs(name, sc, geom_ws, geom_bytes)) return e;
    cudaStream_t s = (cudaStream_t)stream;
    GeomState g = GeomState::carve(geom_ws, P);
    const ViewParams vp = make_view_params(view);
    if (int e = launch_zero_spans({{g.hdr, sizeof(GeomHeader)}, {g.scan_status, GeomState::scan_status_bytes(P)},
                                   {g.sort_temp, sort_prepare_bytes(P, 32)}}, s)) return e;
    { StageTimer _t(GLIC_STAGE_PREPROCESS, s);
    if (int e = launch_preprocess_forward(P, sh_degree, M, means3D, scales, scale_modifier, rotations, opacities, dc, sh, vp,
                                          no_color != 0, radii, g, s)) return e; }
    // R is complete as soon as the preprocess kernel is: ship it to pinned host memory NOW and keep the GPU busy with the
    // depth sort while the host waits for exactly that copy (the reference blocks here too, rasterizer_impl.cu:398, but
    // with an idle GPU).
    struct RChannel { unsigned int* pinned; cudaEvent_t ready, done; cudaStream_t stream; };
    static thread_local RChannel r_channels[64] = {};        // one per device: streams and events are device-bound
    int dev = 0;
    GLIC_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) { set_error("forward_preprocess: device index out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    RChannel& rc = r_channels[dev];
    if (!rc.pinned) {
        GLIC_CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&rc.pinned), sizeof(unsigned int), cudaHostAllocDefault));
        GLIC_CUDA_TRY(cudaEventCreateWithFlags(&rc.ready, cudaEventDisableTiming));
        GLIC_CUDA_TRY(cudaEventCreateWithFlags(&rc.done, cudaEventDisableTiming));
        GLIC_CUDA_TRY(cudaStreamCreateWithFlags(&rc.stream, cudaStreamNonBlocking));   // the 4-byte copy must not sit in front of the depth sort
    }
    unsigned int* r_pinned = rc.pinned;
    cudaEvent_t r_ready = rc.ready, r_event = rc.done;
    cudaStream_t r_stream = rc.stream;
    GLIC_CUDA_TRY(cudaEventRecord(r_ready, s));
    GLIC_CUDA_TRY(cudaStreamWaitEvent(r_stream, r_ready, 0));
    GLIC_CUDA_TRY(cudaMemcpyAsync(r_pinned, &g.hdr->total, sizeof(unsigned int), cudaMemcpyDeviceToHost, r_stream));
    GLIC_CUDA_TRY(cudaEventRecord(r_event, r_stream));
    {   // depth-first binning: order the Gaussians by (depth, index) once, then prefix-sum their tile counts in that order
        StageTimer _t(GLIC_STAGE_SORT, s);
        const int cur = launch_sort_pairs32(P, 32, g.depth_keys, g.order, g.sort_temp, g.sort_temp_size, s, nullptr, /*hist_ready=*/true);
        if (cur < 0) return cur;
        if (int e = launch_depth_scan(P, g, g.order[cur], 0xFFFFFFFFll, s)) return e;
    }
    GLIC_CUDA_TRY(cudaEventSynchronize(r_event));
    const unsigned int total = *r_pinned;
    *num_rendered_host = (int64_t)total;
    return GLIC_OK;
}

int glic_forward_render(int P, const glic_view* view, int no_color, int64_t R, void* geom_ws, void* image_ws,
                        void* binning_ws, size_t binning_bytes, void* sample_ws, size_t sample_bytes, float* out_color,
                        float* out_final_T, int64_t* num_buckets_host, void* stream) {
    if (int e = check_view(view)) return e;
    const char* name = "forward_render";
    if (P < 0 || R < 0 || !image_ws || !out_final_T || (!no_color && !out_color)) return fail(GLIC_ERR_INVALID_ARGUMENT, name, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    const ViewParams vp = make_view_params(view);
    const int T = vp.grid_x * vp.grid_y;
    const size_t HW = (size_t)vp.W * vp.H;
    if (num_buckets_host) *num_buckets_host = 0;
    if (P == 0) {   // rasterize_points.cu:110: zero outputs
        Draw d{name, DRAW_TRAIN, 0.f};
        d.color = out_color; d.final_T = out_final_T;
        return write_empty(d, HW, s);
    }
    if (!geom_ws) return fail(GLIC_ERR_WORKSPACE, name, "geometry workspace is NULL");
    if (!binning_ws || binning_bytes < glic_binning_bytes(R)) return fail(GLIC_ERR_WORKSPACE, name, "binning workspace too small");
    const int64_t max_buckets = no_color ? 0 : glic_max_buckets(R, vp.W, vp.H);
    if (!no_color && (!sample_ws || sample_bytes < glic_sample_bytes(R, vp.W, vp.H))) return fail(GLIC_ERR_WORKSPACE, name, "sample workspace too small");
    GeomState g = GeomState::carve(geom_ws, P);
    ImageState img = ImageState::carve(image_ws, vp.W, vp.H);
    BinningState bin = BinningState::carve(binning_ws, R);
    SampleState smp = SampleState::carve(no_color ? nullptr : sample_ws, max_buckets);

    int cur = 0;
    if (R > 0) {
        const int bit = tile_sort_bits(T);                                  // rasterizer_impl.cu:417
        { StageTimer _t(GLIC_STAGE_EMIT, s);
          if (int e = sort_prepare(R, bit, bin.sort_temp, s)) return e;      // emit builds the tile sort's digit histograms
          if (int e = launch_emit_keys(P, vp, g, bin.keys[0], bin.vals[0], R, sort_hist(bin.sort_temp), bit, s)) return e; }
        // pairs arrive ordered by (depth, index): a stable sort on the tile bits alone finishes the job
        { StageTimer _t(GLIC_STAGE_SORT, s); cur = launch_sort_pairs32(R, bit, bin.keys, bin.vals, bin.sort_temp, bin.sort_temp_size, s, nullptr, true); }
        if (cur < 0) return cur;
    }
    GLIC_CUDA_TRY(cudaMemsetAsync(img.ranges, 0, sizeof(uint2) * (size_t)T, s));
    { StageTimer _t(GLIC_STAGE_RANGES, s);
      if (int e = launch_tile_ranges(R, nullptr, bin.keys[cur], T, img, !no_color, &bin.hdr->sorted_in_b, cur, s)) return e; }
    { StageTimer _t(GLIC_STAGE_RENDER_FWD, s); if (int e = launch_render_forward(vp, no_color != 0, bin.vals[cur], g, img, smp, out_color, out_final_T, s)) return e; }
    if (num_buckets_host) {
        unsigned int nb = 0;
        GLIC_CUDA_TRY(cudaMemcpyAsync(&nb, &img.hdr->num_buckets, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
        GLIC_CUDA_TRY(cudaStreamSynchronize(s));
        *num_buckets_host = nb;
    }
    return GLIC_OK;
}

int64_t glic_binning_capacity(size_t binning_bytes, size_t sample_bytes, int width, int height, int no_color) {
    // largest R whose workspaces fit: both size functions are monotone in R
    int64_t lo = 0, hi = (int64_t)1 << 31;
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo + 1) / 2;
        const bool fits = glic_binning_bytes(mid) <= binning_bytes && (no_color || glic_sample_bytes(mid, width, height) <= sample_bytes);
        if (fits) lo = mid; else hi = mid - 1;
    }
    return lo;
}

int glic_forward(int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier,
                 const float* rotations, const float* opacities, const float* dc, const float* sh, const glic_view* view,
                 int no_color, int* radii, void* geom_ws, size_t geom_bytes, void* image_ws, size_t image_bytes, void* binning_ws,
                 size_t binning_bytes, void* sample_ws, size_t sample_bytes, float* out_color, float* out_final_T,
                 int64_t* counters_host, void* stream) {
    Draw d{"forward", DRAW_TRAIN, 0.f, !out_final_T || (!no_color && !out_color)};
    d.color = out_color; d.final_T = out_final_T; d.sample_ws = sample_ws; d.sample_bytes = sample_bytes;
    const Scene sc{P, sh_degree, M, means3D, scales, scale_modifier, rotations, opacities, dc, sh, no_color != 0, radii};
    return draw(d, sc, view, geom_ws, geom_bytes, image_ws, image_bytes, binning_ws, binning_bytes, counters_host, (cudaStream_t)stream);
}

int glic_render(int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier,
                const float* rotations, const float* opacities, const float* dc, const float* sh, const glic_view* view,
                int* radii, void* geom_ws, size_t geom_bytes, void* image_ws, size_t image_bytes, void* binning_ws,
                size_t binning_bytes, float* out_color, float* out_final_T, float* out_depth, float* out_median_depth,
                int64_t* counters_host, void* stream) {
    // glic_forward's stages up to the blend, so the tile lists are its lists; no checkpoints, so no bucket offsets.  An empty
    // scene has T = 1 (nothing covers a pixel)
    Draw d{"render", DRAW_INFER, 1.f, !out_color || !out_final_T};
    d.color = out_color; d.final_T = out_final_T; d.depth = out_depth; d.median_depth = out_median_depth;
    const Scene sc{P, sh_degree, M, means3D, scales, scale_modifier, rotations, opacities, dc, sh, false, radii};
    return draw(d, sc, view, geom_ws, geom_bytes, image_ws, image_bytes, binning_ws, binning_bytes, counters_host, (cudaStream_t)stream);
}

int glic_contribution(int P, const float* means3D, const float* scales, float scale_modifier, const float* rotations,
                      const float* opacities, const glic_view* view, int* radii, void* geom_ws, size_t geom_bytes, void* image_ws,
                      size_t image_bytes, void* binning_ws, size_t binning_bytes, float* max_weight, uint64_t* hits,
                      uint64_t* ends, float* out_final_T, int64_t* counters_host, void* stream) {
    if (int e = check_view(view)) return e;
    if (P < 0) return fail(GLIC_ERR_INVALID_ARGUMENT, "contribution", "P must be >= 0");
    // glic_forward's stages with no_color = 1, so the lists are its lists; an overflow leaves every range empty (r_eff = 0), so
    // the blend takes no pair and adds nothing.  An empty scene has glic_forward's outputs and nothing to score
    Draw d{"contribution", DRAW_SCORE, 0.f, P > 0 && (!max_weight || !hits)};
    d.final_T = out_final_T; d.max_weight = max_weight; d.hits = hits; d.ends = ends;
    const Scene sc{P, 0, 0, means3D, scales, scale_modifier, rotations, opacities, nullptr, nullptr, true, radii};
    return draw(d, sc, view, geom_ws, geom_bytes, image_ws, image_bytes, binning_ws, binning_bytes, counters_host, (cudaStream_t)stream);
}

size_t glic_deterministic_bytes(int64_t num_rendered, int width, int height) {
    size_t b = 0;
    DetState::carve(nullptr, glic_max_buckets(num_rendered > 0 ? num_rendered : 0, width, height), &b);
    return b;
}

// glic_backward and glic_backward_deterministic: det_ws == NULL selects the atomic render backward.  2-D gradient accumulators
// are filled by atomics (or, deterministic, written for the rows with a contribution): zero them here (11 floats / Gaussian)
static int backward_impl(const char* what, int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier,
                         const float* rotations, const float* sh, const glic_view* view, const int* radii, int64_t R,
                         const void* geom_ws, const void* binning_ws, const void* image_ws, const void* sample_ws,
                         const float* dL_dpix, float lambda_erank, float* dL_dmeans2D, float* dL_dconic, float* dL_dopacity,
                         float* dL_dcolors, float* dL_dmeans3D, float* dL_dcov3D, float* dL_ddc, float* dL_dsh, float* dL_dscales,
                         float* dL_drotations, void* det_ws, cudaStream_t s) {
    if (int e = check_view(view)) return e;
    if (P < 0 || R < 0 || sh_degree < 0 || sh_degree > 3 || M < 0) return fail(GLIC_ERR_INVALID_ARGUMENT, what, "bad sizes");
    if (P == 0) return GLIC_OK;
    if (!means3D || !scales || !rotations || !radii || !dL_dpix || !dL_dmeans2D || !dL_dconic || !dL_dopacity || !dL_dcolors ||
        !dL_dmeans3D || !dL_dcov3D || !dL_ddc || !dL_dscales || !dL_drotations || (M > 0 && (!sh || !dL_dsh)))
        return fail(GLIC_ERR_INVALID_ARGUMENT, what, "null pointer");
    if (!aligned16(rotations) || !aligned16(dL_drotations)) return fail(GLIC_ERR_INVALID_ARGUMENT, what, "rotations / dL_drotations must be 16-byte aligned");
    if (!geom_ws || !image_ws || (R > 0 && (!binning_ws || !sample_ws))) return fail(GLIC_ERR_WORKSPACE, what, "missing saved workspace");
    const ViewParams vp = make_view_params(view);
    const Saved sv = carve_saved(P, vp, R, geom_ws, image_ws, binning_ws, sample_ws);
    { StageTimer _t(GLIC_STAGE_ZERO, s);
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dmeans2D, 0, sizeof(float) * 3 * (size_t)P, s));
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dconic, 0, sizeof(float) * 4 * (size_t)P, s));
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dopacity, 0, sizeof(float) * (size_t)P, s));
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dcolors, 0, sizeof(float) * 3 * (size_t)P, s)); }
    if (R > 0)
        if (int e = render_backward(P, vp, sv, det_ws, dL_dpix, dL_dmeans2D, dL_dconic, dL_dopacity, dL_dcolors, s)) return e;
    StageTimer _t(GLIC_STAGE_PREPROCESS_BWD, s);
    return launch_preprocess_backward(P, sh_degree, M, means3D, scales, scale_modifier, rotations, sh, vp, radii, sv.g,
                                      lambda_erank, dL_dmeans2D, dL_dconic, dL_dcolors, dL_dmeans3D, dL_dcov3D, dL_ddc,
                                      dL_dsh, dL_dscales, dL_drotations, s);
}

int glic_backward_deterministic(int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier,
                                const float* rotations, const float* dc, const float* sh, const glic_view* view, const int* radii,
                                int64_t R, const void* geom_ws, const void* binning_ws, const void* image_ws, const void* sample_ws,
                                const float* dL_dpix, float lambda_erank, float* dL_dmeans2D, float* dL_dconic, float* dL_dopacity,
                                float* dL_dcolors, float* dL_dmeans3D, float* dL_dcov3D, float* dL_ddc, float* dL_dsh,
                                float* dL_dscales, float* dL_drotations, void* det_ws, size_t det_bytes, void* stream) {
    (void)dc;
    if (int e = check_view(view)) return e;
    if (P > 0 && R > 0 && (!det_ws || det_bytes < glic_deterministic_bytes(R, view->width, view->height)))
        return fail(GLIC_ERR_WORKSPACE, "backward_deterministic", "deterministic workspace too small");
    return backward_impl("backward_deterministic", P, sh_degree, M, means3D, scales, scale_modifier, rotations, sh, view, radii, R,
                         geom_ws, binning_ws, image_ws, sample_ws, dL_dpix, lambda_erank, dL_dmeans2D, dL_dconic, dL_dopacity,
                         dL_dcolors, dL_dmeans3D, dL_dcov3D, dL_ddc, dL_dsh, dL_dscales, dL_drotations, det_ws, (cudaStream_t)stream);
}

int glic_backward(int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier,
                  const float* rotations, const float* dc, const float* sh, const glic_view* view, const int* radii,
                  int64_t R, const void* geom_ws, const void* binning_ws, const void* image_ws, const void* sample_ws,
                  const float* dL_dpix, float lambda_erank, float* dL_dmeans2D, float* dL_dconic, float* dL_dopacity,
                  float* dL_dcolors, float* dL_dmeans3D, float* dL_dcov3D, float* dL_ddc, float* dL_dsh, float* dL_dscales,
                  float* dL_drotations, void* stream) {
    (void)dc;
    return backward_impl("backward", P, sh_degree, M, means3D, scales, scale_modifier, rotations, sh, view, radii, R, geom_ws,
                         binning_ws, image_ws, sample_ws, dL_dpix, lambda_erank, dL_dmeans2D, dL_dconic, dL_dopacity, dL_dcolors,
                         dL_dmeans3D, dL_dcov3D, dL_ddc, dL_dsh, dL_dscales, dL_drotations, nullptr, (cudaStream_t)stream);
}

int glic_debug_pose_backward(int P, int sh_degree, int M, const float* means3D, const float* scales, const float* rotations,
                             const float* rot_raw, const float* opacity, const float* sh, const glic_view* view, const int* radii,
                             const void* geom_ws, const float* dL_dmeans2D, const float* dL_dconic, const float* dL_dopacity,
                             const float* dL_dcolors, int pose_only, float* g_geo, void* partials, float* pose6, void* stream) {
    if (int e = check_view(view)) return e;
    if (P <= 0 || !means3D || !scales || !rotations || !radii || !geom_ws || !dL_dmeans2D || !dL_dconic || !dL_dcolors || !partials ||
        !pose6 || (!pose_only && (!g_geo || !rot_raw || !opacity || !dL_dopacity))) return fail(GLIC_ERR_INVALID_ARGUMENT, "debug_pose_backward", "bad arguments");
    CompactGrads cg{};
    if (!pose_only) {                                   // the mapper's compact block: rotation | xyz | log-scale | opacity logit
        cg.g_rot = reinterpret_cast<float4*>(g_geo);
        cg.g_xyz = g_geo + 4 * (size_t)P;
        cg.g_scale = g_geo + 7 * (size_t)P;
        cg.g_opacity = g_geo + 10 * (size_t)P;
        cg.opacity = opacity; cg.dL_dopacity = dL_dopacity; cg.rot_raw = reinterpret_cast<const float4*>(rot_raw);
    }
    cg.pose_partials = static_cast<double*>(partials);
    cg.pose_grad = pose6;
    StageTimer _t(GLIC_STAGE_PREPROCESS_BWD, (cudaStream_t)stream);
    return launch_preprocess_backward_compact(P, sh_degree, M, means3D, scales, 1.0f, rotations, sh, make_view_params(view), radii,
                                              GeomState::carve(const_cast<void*>(geom_ws), P), dL_dmeans2D, dL_dconic, dL_dcolors, cg,
                                              (cudaStream_t)stream);
}

int glic_sort_pairs_u64_u32(int64_t n, int end_bit, uint64_t* keys_in, uint32_t* vals_in, uint64_t* keys_out,
                            uint32_t* vals_out, void* temp, size_t temp_bytes, void* stream) {
    if (n < 0 || (n > 0 && (!keys_in || !vals_in || !keys_out || !vals_out || !temp))) { set_error("sort_pairs: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (n == 0) return GLIC_OK;
    cudaStream_t s = (cudaStream_t)stream;
    uint64_t* k[2] = {keys_in, keys_out};
    uint32_t* v[2] = {vals_in, vals_out};
    const int cur = launch_sort_pairs(n, end_bit, k, v, temp, temp_bytes, s);
    if (cur < 0) return cur;
    if (cur == 0) {   // even number of passes: result sits in the input buffers
        GLIC_CUDA_TRY(cudaMemcpyAsync(keys_out, keys_in, sizeof(uint64_t) * (size_t)n, cudaMemcpyDeviceToDevice, s));
        GLIC_CUDA_TRY(cudaMemcpyAsync(vals_out, vals_in, sizeof(uint32_t) * (size_t)n, cudaMemcpyDeviceToDevice, s));
    }
    return GLIC_OK;
}

int glic_debug_sort_pairs_u32(int64_t n, int end_bit, uint32_t* keys, uint32_t* vals, uint32_t* keys_alt, uint32_t* vals_alt,
                              const unsigned int* n_dev, void* temp, size_t temp_bytes, void* stream) {
    if (n < 0 || (n > 0 && (!keys || !vals || !keys_alt || !vals_alt || !temp))) { set_error("debug_sort_pairs_u32: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    uint32_t* k[2] = {keys, keys_alt};
    uint32_t* v[2] = {vals, vals_alt};
    return launch_sort_pairs32(n, end_bit, k, v, temp, temp_bytes, (cudaStream_t)stream, n_dev, false);
}

int glic_debug_render_backward(int P, const glic_view* view, int64_t R, const void* geom_ws, const void* binning_ws,
                               const void* image_ws, const void* sample_ws, const float* dL_dpix, float* dL_dmeans2D,
                               float* dL_dconic, float* dL_dopacity, float* dL_dcolors, int exact, unsigned long long* counters,
                               void* stream) {
    if (int e = check_view(view)) return e;
    const char* name = "debug_render_backward";
    if (P < 0 || R < 0) return fail(GLIC_ERR_INVALID_ARGUMENT, name, "bad sizes");
    if (P == 0 || R == 0) return GLIC_OK;
    if (!dL_dpix || !dL_dmeans2D || !dL_dconic || !dL_dopacity || !dL_dcolors) return fail(GLIC_ERR_INVALID_ARGUMENT, name, "null pointer");
    if (!geom_ws || !image_ws || !binning_ws || !sample_ws) return fail(GLIC_ERR_WORKSPACE, name, "missing saved workspace");
    const ViewParams vp = make_view_params(view);
    const Saved sv = carve_saved(P, vp, R, geom_ws, image_ws, binning_ws, sample_ws);
    return launch_render_backward(P, vp, sv.max_buckets, sv.bin.vals[sv.cur], sv.g, sv.img, sv.smp, dL_dpix, dL_dmeans2D, dL_dconic,
                                  dL_dopacity, dL_dcolors, (cudaStream_t)stream, exact != 0, counters);
}

int glic_debug_deterministic_entries(int P, const glic_view* view, int64_t R, const void* geom_ws, const void* binning_ws,
                                     const void* image_ws, const void* sample_ws, const float* dL_dpix, void* det_ws, size_t det_bytes,
                                     float* dL_dmeans2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolors, int64_t* count_host,
                                     uint32_t* gid, uint32_t* tile, float* values, void* stream) {
    if (int e = check_view(view)) return e;
    const char* name = "debug_deterministic_entries";
    if (P < 0 || R < 0 || !count_host) return fail(GLIC_ERR_INVALID_ARGUMENT, name, "bad arguments");
    *count_host = 0;
    if (P == 0) return GLIC_OK;
    if (!dL_dpix || !dL_dmeans2D || !dL_dconic || !dL_dopacity || !dL_dcolors || !gid || !tile || !values)
        return fail(GLIC_ERR_INVALID_ARGUMENT, name, "null pointer");
    if (!geom_ws || !image_ws || (R > 0 && (!binning_ws || !sample_ws))) return fail(GLIC_ERR_WORKSPACE, name, "missing saved workspace");
    if (R > 0 && (!det_ws || det_bytes < glic_deterministic_bytes(R, view->width, view->height)))
        return fail(GLIC_ERR_WORKSPACE, name, "deterministic workspace too small");
    cudaStream_t s = (cudaStream_t)stream;
    const ViewParams vp = make_view_params(view);
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dmeans2D, 0, sizeof(float) * 3 * (size_t)P, s));
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dconic, 0, sizeof(float) * 4 * (size_t)P, s));
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dopacity, 0, sizeof(float) * (size_t)P, s));
    GLIC_CUDA_TRY(cudaMemsetAsync(dL_dcolors, 0, sizeof(float) * 3 * (size_t)P, s));
    if (R == 0) return GLIC_OK;
    const Saved sv = carve_saved(P, vp, R, geom_ws, image_ws, binning_ws, sample_ws);
    DetState det = DetState::carve(det_ws, sv.max_buckets);
    if (int e = launch_render_backward_det(P, vp, sv.max_buckets, sv.bin.vals[sv.cur], sv.g, sv.img, sv.smp, det, dL_dpix, dL_dmeans2D,
                                           dL_dconic, dL_dopacity, dL_dcolors, s)) return e;
    unsigned int* n_valid = det.count;       // reused: the entry count is read by the launches above only
    const int half = det_sorted_half(P);
    unsigned int n = 0;
    GLIC_CUDA_TRY(cudaMemcpyAsync(&n, det.count, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    GLIC_CUDA_TRY(cudaMemsetAsync(n_valid, 0, sizeof(unsigned int), s));
    if (n > 0) {
        debug_det_entries_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, (uint32_t)P, det.keys[half], det.idx[half], det.vals, sv.img.live_offsets,
                                                                 vp.grid_x * vp.grid_y, gid, tile, values, n_valid);
        GLIC_LAUNCH_CHECK();
    }
    unsigned int valid = 0;
    GLIC_CUDA_TRY(cudaMemcpyAsync(&valid, n_valid, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    *count_host = valid;
    return GLIC_OK;
}

int glic_debug_geom(int P, const void* geom_ws, float* depth, float* xy, float* conic_opacity, float* rgb,
                    uint32_t* tiles_touched, uint32_t* offsets, uint8_t* clamped, void* stream) {
    if (P <= 0) return GLIC_OK;
    if (!geom_ws) { set_error("debug_geom: null workspace"); return GLIC_ERR_WORKSPACE; }
    GeomState g = GeomState::carve(const_cast<void*>(geom_ws), P);
    debug_geom_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(P, g, depth, xy, conic_opacity, rgb, tiles_touched, offsets, clamped);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int glic_debug_spans(int P, const void* geom_ws, uint32_t* count_cap_host, void* stream) {
    if (!count_cap_host) { set_error("debug_spans: null output"); return GLIC_ERR_INVALID_ARGUMENT; }
    count_cap_host[0] = count_cap_host[1] = 0;
    if (P <= 0) return GLIC_OK;
    if (!geom_ws) { set_error("debug_spans: null workspace"); return GLIC_ERR_WORKSPACE; }
    cudaStream_t s = (cudaStream_t)stream;
    GeomState g = GeomState::carve(const_cast<void*>(geom_ws), P);
    unsigned int count = 0;
    GLIC_CUDA_TRY(cudaMemcpyAsync(&count, &g.hdr->span_count, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    count_cap_host[0] = count;
    count_cap_host[1] = g.span_cap;
    return GLIC_OK;
}

int glic_debug_binning(int P, const void* geom_ws, int64_t R, int64_t count, const void* binning_ws, uint32_t* point_list,
                       uint64_t* keys_sorted, void* stream) {
    if (R <= 0 || count <= 0) return GLIC_OK;
    if (count > R) { set_error("debug_binning: count exceeds the carve size"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!binning_ws || !geom_ws) { set_error("debug_binning: null workspace"); return GLIC_ERR_WORKSPACE; }
    cudaStream_t s = (cudaStream_t)stream;
    BinningState bin = BinningState::carve(const_cast<void*>(binning_ws), R);
    GeomState g = GeomState::carve(const_cast<void*>(geom_ws), P);
    unsigned int cur = 0;
    GLIC_CUDA_TRY(cudaMemcpyAsync(&cur, &bin.hdr->sorted_in_b, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    cur &= 1u;
    if (point_list) GLIC_CUDA_TRY(cudaMemcpyAsync(point_list, bin.vals[cur], sizeof(uint32_t) * (size_t)count, cudaMemcpyDeviceToDevice, s));
    if (keys_sorted) {   // the 64-bit (tile|depth) key of the reference, rebuilt from the tile key and the record's depth
        debug_keys_kernel<<<(unsigned)((count + 255) / 256), 256, 0, s>>>((long long)count, g, bin.keys[cur], bin.vals[cur], keys_sorted);
        GLIC_LAUNCH_CHECK();
    }
    return GLIC_OK;
}

int glic_debug_image(int width, int height, const void* image_ws, uint32_t* ranges, uint32_t* bucket_offsets,
                     uint32_t* n_contrib, uint32_t* max_contrib, int64_t* counters2_host, void* stream) {
    if (!image_ws || width <= 0 || height <= 0) { set_error("debug_image: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    cudaStream_t s = (cudaStream_t)stream;
    ImageState img = ImageState::carve(const_cast<void*>(image_ws), width, height);
    const size_t T = (size_t)((width + TILE - 1) / TILE) * ((height + TILE - 1) / TILE);
    if (ranges) GLIC_CUDA_TRY(cudaMemcpyAsync(ranges, img.ranges, sizeof(uint2) * T, cudaMemcpyDeviceToDevice, s));
    if (bucket_offsets) GLIC_CUDA_TRY(cudaMemcpyAsync(bucket_offsets, img.bucket_offsets, sizeof(uint32_t) * T, cudaMemcpyDeviceToDevice, s));
    if (n_contrib) GLIC_CUDA_TRY(cudaMemcpyAsync(n_contrib, img.n_contrib, sizeof(uint32_t) * (size_t)width * height, cudaMemcpyDeviceToDevice, s));
    if (max_contrib) GLIC_CUDA_TRY(cudaMemcpyAsync(max_contrib, img.max_contrib, sizeof(uint32_t) * T, cudaMemcpyDeviceToDevice, s));
    if (counters2_host) {
        ImageHeader h;
        GLIC_CUDA_TRY(cudaMemcpyAsync(&h, img.hdr, sizeof(ImageHeader), cudaMemcpyDeviceToHost, s));
        GLIC_CUDA_TRY(cudaStreamSynchronize(s));
        counters2_host[0] = h.num_rendered;
        counters2_host[1] = h.num_buckets;
    }
    return GLIC_OK;
}

}  // extern "C"

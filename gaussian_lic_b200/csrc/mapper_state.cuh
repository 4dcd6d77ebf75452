// mapper_state.cuh -- the native mapper's state (struct glic_mapper), the types it is made of and the helpers its translation
// units share.  Private to mapper.cu (camera and pose math, growth, keyframes and frames, the iteration, evaluation, options),
// mapper_density.cu (density control and contribution scores), mapper_views.cu (alignment, rendering from a caller's camera),
// mapper_mesh.cu (meshing) and mapper_checkpoint.cu (checkpoints).
#pragma once
#include "common.cuh"
#include "checkpoint.h"

#include <array>
#include <atomic>
#include <functional>
#include <random>
#include <string>
#include <utility>
#include <vector>

// The helpers live in one namespace of their own; the build's -fvisibility=hidden keeps them out of the library's symbols.
namespace mapper_impl {

using namespace glic;

constexpr int MAX_SLOTS = 32;        // world * views_per_rank
static_assert(MAX_SLOTS <= EXPO_MAX_SLOTS, "the exposure step takes every slot of a batch");
constexpr int RING = 8;              // pinned result ring (loss, binning counters)

struct CamBlock {                    // what the rasterizer gets per view (camera.h:38-110, renderer.cpp:31-54)
    float view[16], proj[16], campos[4];
    float tanfovx, tanfovy, lim[4];
};

// ---- ownership: every CUDA resource of a mapper is a member of one of the two types below, and only they allocate or release
// one.  The members release themselves, so destroying a mapper is a drain and a delete, and a failed create needs no cleanup.
extern std::atomic<int> fail_countdown;          // glic_debug_fail_allocation
extern std::atomic<int64_t> live_allocations;    // glic_debug_mapper_allocations

// One device (or pinned host) allocation of a known size, move-only, released by its destructor
class Buf {
public:
    Buf() = default;
    Buf(Buf&& o) noexcept { *this = std::move(o); }
    Buf& operator=(Buf&& o) noexcept {
        if (this != &o) { release(); p_ = std::exchange(o.p_, nullptr); bytes_ = std::exchange(o.bytes_, 0); pinned_ = o.pinned_; }
        return *this;
    }
    ~Buf() { release(); }
    void* raw() const { return p_; }
    size_t bytes() const { return bytes_; }
    // on an empty Buf: `bytes` of device memory (of pinned host memory with `pinned`), not initialised
    int allocate(size_t bytes, bool pinned = false) {
        int n = fail_countdown.load();
        while (n > 0 && !fail_countdown.compare_exchange_weak(n, n - 1)) {}
        const cudaError_t e = n == 1 ? cudaErrorMemoryAllocation
                            : pinned ? cudaHostAlloc(&p_, bytes, cudaHostAllocDefault) : cudaMalloc(&p_, bytes ? bytes : 256);
        if (e != cudaSuccess) {
            p_ = nullptr;
            cudaGetLastError();                      // not left for the next launch check to report
            set_error("mapper: allocation of " + std::to_string(bytes) + " bytes failed: " + cudaGetErrorString(e));
            return GLIC_ERR_CUDA;
        }
        bytes_ = bytes; pinned_ = pinned; ++live_allocations;
        return GLIC_OK;
    }
private:
    void release() {
        if (!p_) return;
        if (pinned_) cudaFreeHost(p_); else cudaFree(p_);
        --live_allocations; p_ = nullptr; bytes_ = 0;
    }
    void* p_ = nullptr;
    size_t bytes_ = 0;
    bool pinned_ = false;
};
// a Buf of T that converts to T*, so the launches take it as they would a raw pointer
template <typename T>
struct Dev : Buf {
    operator T*() const { return static_cast<T*>(raw()); }
};

// a stream, an event or an IPC mapping, move-only, destroyed by its destructor
template <typename H, cudaError_t (*Destroy)(H)>
class Handle {
public:
    Handle() = default;
    explicit Handle(H h) : h_(h) {}
    Handle(Handle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    Handle& operator=(Handle&& o) noexcept { std::swap(h_, o.h_); return *this; }
    ~Handle() { if (h_) Destroy(h_); }
    operator H() const { return h_; }
private:
    H h_ = nullptr;
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using IpcMapping = Handle<void*, cudaIpcCloseMemHandle>;

struct Keyframe {                    // move-only: it owns its device camera block
    float R_wc[9], t_wc[3];
    const float* image = nullptr;
    bool image_on_device = false;    // `image` is memory of the mapper's device: the loss reads it in place
    Buf owned_image;                 // a float image restored from a checkpoint (device or pinned host memory): `image` points here
    const uint8_t* bgr = nullptr;    // add_frame keyframes: packed HWC BGR8 in the frame store, decoded where `image` is copied
    CamBlock cam;
    Dev<float> cam_dev;              // view16 | proj16 | campos4
    glic_view view;
    // valid-pixel mask (glic_mapper_set_keyframe_mask): the packed bits, the number of used pixels (0: no mask) and how many
    // of them lie in columns [0, W/2) (glic_mapper_align's split fit region)
    Dev<uint32_t> mask;
    uint32_t mask_valid = 0, mask_valid_left = 0;
};

struct PoseBatch {
    int kf[MAX_SLOTS];                // keyframe of each slot
    float* cam[MAX_SLOTS];            // its device camera block
    float Pm[16];                     // the pose-independent projection (row-major)
};

constexpr size_t FRAME_CHUNK = ckpt::FRAME_CHUNK;    // frames per device allocation of the 8-bit image store

// Regions of the exchange block that hold one slot per (parity, view slot), in layout order
enum SlotRegion { COLOUR, FLAGS, EXPOSURE, POSE, RADII, N_REGIONS };

// Adam state of a per-training-keyframe parameter of `width` floats: moments [cap][width], step counts [cap]
struct KeyframeAdam {
    int width;
    Dev<float> m, v;
    Dev<int> t;
};

// The exchange block: geo[11*Pcap + 4 (+ 2*Pcap)] | flags words | one region [2][S] of slots per SlotRegion.  With densification
// on, the reduced region ends in the batch's statistics rows: norms [Pcap] | view counts [Pcap], at 11*Pcap + 4.
struct XLayout {
    size_t n_geo = 0;                // floats in the reduced region (11*Pcap + 4; the tail holds the collective overflow word)
    size_t bytes = 0, slot_off[N_REGIONS] = {}, slot_bytes[N_REGIONS] = {};
};

}  // namespace mapper_impl

using namespace mapper_impl;

struct glic_mapper {
    glic_mapper_config cfg{};
    int dev = 0, D = 0, M = 0, S = 1, k = 1;
    Stream stream, copy_stream, push_stream;
    // ---- arenas (capacity Pcap) ----
    uint32_t P = 0, Pcap = 0;
    uint32_t n_sky = 0;                   // rows [0, n_sky) are the skybox (glic_mapper_initialize_lidar): left out of save_map
    Dev<float> params, m1, m2;
    Dev<int32_t> anchor;                  // [Pcap]: the training keyframe each row moves with (glic_mapper_correct_poses), or -1
    Dev<float> act_opacity, act_scales, act_rots;
    Dev<int> radii;
    Dev<float> g_conic;                   // the render backward's 2-D gradient accumulators: conic [4 Pcap] | mean2D [3 Pcap] | opacity
    float *g_mean2D = nullptr, *g_opacity = nullptr;
    Dev<void> geom_ws;
    Dev<char> xblock;
    XLayout x;
    void* peers[8] = {nullptr};
    bool connected = false;
    std::vector<IpcMapping> opened;
    // ---- per-image buffers ----
    Dev<void> image_ws, binning_ws, sample_ws, loss_scratch, eval_scratch, extend_ws;
    int64_t bin_cap = 0;
    // GLIC_MAPPER_OPT_DETERMINISTIC: the fixed-order render backward's workspace (glic_deterministic_bytes(bin_cap, W, H), grown
    // with the binning capacity while the option is on) and the partials of the fixed-order loss and evaluation sums
    bool deterministic = false;
    Dev<void> det_ws, det_sums;
    Dev<float> color, final_T, dL_dpix, gt_dev[2], loss_dev, eval_out;
    Dev<unsigned int> vis_acc;
    Event gt_free[2], gt_ready[2], ev_flags, ev_col, ev_push, ring_ev[RING], t0, t1;
    Dev<long long> counters_host;         // pinned [RING][4]
    Dev<float> loss_host;                 // pinned [RING]
    bool ring_used[RING] = {false};
    // ---- keyframes ----
    std::vector<Keyframe> train, test;
    std::mt19937_64 rng;
    uint64_t view_counter = 0;
    glic_mapper_stats st{};
    bool run_optimizer = true;            // GLIC_MAPPER_OPT_OPTIMIZER (benchmarks time the rasterization step alone with it off)
    // ---- per-training-keyframe rows of the exposure and the pose refinement, kf_cap of each, allocated for both features
    //      once either is enabled (enabling one initialises its rows of the existing keyframes) ----
    size_t kf_cap = 0;
    // exposure (glic_mapper_enable_exposure): E [kf_cap][12] and its Adam state
    bool expo_on = false;
    float expo_lr = 0.f;
    Dev<float> expo_E;
    KeyframeAdam expo_adam{12};
    // pose refinement (glic_mapper_enable_pose_refinement): float64 T_cw [kf_cap][12] (R_cw row-major | t_cw), the float pose
    // [kf_cap][12] (R_wc | t_wc) and the Adam state of the 6-vector
    bool pose_on = false;
    float pose_lr_rho = 0.f, pose_lr_omega = 0.f;
    Dev<double> pose_T;
    Dev<float> pose_f;
    KeyframeAdam pose_adam{6};
    Dev<double> pose_part;                // per-CTA partials of the pose-gradient reduction (pose_partials_count(Pcap))
    Event ev_pose;
    // ---- LPIPS of the evaluation (glic_mapper_load_lpips): weight payload and glic_lpips's scratch, sized on first use ----
    Dev<float> lpips_w;
    Dev<void> lpips_scratch;
    // ---- test-time alignment (glic_mapper_align): its workspace (align_carve), sized on first use ----
    Dev<char> align_ws;
    // ---- rendering from a caller's camera (glic_mapper_render_camera): its workspace (render_carve) for the largest frame so far
    Dev<char> render_ws;
    // ---- contribution scores (glic_mapper_contribution / prune_unseen): hits [Pcap] u64 | max_weight [Pcap] f32, sized on first use
    Dev<char> score_ws;
    // ---- the last mesh of glic_mapper_extract_mesh: xyz [V,3] f32, rgb [V,3] u8, faces [F,3] i32 (empty until the first call)
    bool mesh_ready = false;
    glic_mesh_counts mesh_counts{};
    Dev<float> mesh_xyz;
    Dev<uint8_t> mesh_rgb;
    Dev<int32_t> mesh_faces;
    // ---- raw frames (glic_mapper_enable_frames / add_frame): the 8-bit image store, chunks of FRAME_CHUNK frames of
    //      frame_stride bytes that never move, and the scan of the frames since the last training keyframe (device arrays
    //      of scan_cap points, grown by doubling) ----
    bool initialized = false;             // initialize or initialize_lidar has run (the next scan extends the map)
    bool frames_on = false;
    int frame_k = 1, frame_sky_points = 0, frame_sky_radius = 0;
    std::vector<Dev<uint8_t>> frame_chunks;
    size_t frame_stride = 0;
    Dev<float> scan_xyz, scan_depth;
    Dev<uint8_t> scan_rgb;
    size_t scan_cap = 0;
    glic_frame_stats fst{};
    // ---- densification (glic_mapper_enable_densification): per-row statistics [Pcap] each, and the number of real densify
    //      calls so far (the key of the split children's generator) ----
    bool dens_on = false;
    bool exported = false;                // glic_mapper_export has run: the exchange block can no longer move
    Dev<float> dens_accum, dens_denom;
    Dev<int> dens_maxr;                   // the largest screen radius of each row since the statistics last restarted
    uint64_t dens_calls = 0;
    // ---- the density-control schedule of optimize() (glic_mapper_set_density_schedule) and what it has done since it was set
    bool sched_on = false;
    glic_density_schedule sched{};
    glic_density_counts sched_totals{};
    uint32_t sched_steps = 0, sched_resets = 0;
};

namespace mapper_impl {

#define MAP_TRY(expr) do { int _e = (expr); if (_e != GLIC_OK) return _e; } while (0)

// One buffer of a growth: its new size, the prefix of its old contents it keeps, and whether it starts zeroed
struct Grow { Buf& buf; size_t bytes, keep = 0; bool zero = false; };

// ---- the per-row buffer groups: each is one table of {buffer, bytes per row}, in its checkpoint section's order (the widths are
// checkpoint.h's).  Growth, zeroing, the compaction's gathers, the save and the load iterate these tables; a new per-row buffer
// is declared here and nowhere else.
struct Rows { Buf& buf; size_t bytes; };

// per training keyframe, kf_cap rows: the exposure E and its Adam state
inline std::vector<Rows> exposure_rows(glic_mapper* m) {
    const auto& w = ckpt::EXPOSURE_ROW;
    return {{m->expo_E, w[0]}, {m->expo_adam.m, w[1]}, {m->expo_adam.v, w[2]}, {m->expo_adam.t, w[3]}};
}
// per training keyframe, kf_cap rows: the float64 and float poses and the Adam state of the pose refinement
inline std::vector<Rows> pose_rows(glic_mapper* m) {
    const auto& w = ckpt::POSE_ROW;
    return {{m->pose_T, w[0]}, {m->pose_f, w[1]}, {m->pose_adam.m, w[2]}, {m->pose_adam.v, w[3]}, {m->pose_adam.t, w[4]}};
}
// per Gaussian, Pcap rows (with densification on): the densification statistics
inline std::vector<Rows> densification_rows(glic_mapper* m) {
    const auto& w = ckpt::DENSIFICATION_ROW;
    return {{m->dens_accum, w[0]}, {m->dens_denom, w[1]}, {m->dens_maxr, w[2]}};
}
// per point, scan_cap rows: the pending scan of add_frame
inline std::vector<Rows> scan_rows(glic_mapper* m) {
    const auto& w = ckpt::SCAN_ROW;
    return {{m->scan_xyz, w[0]}, {m->scan_rgb, w[1]}, {m->scan_depth, w[2]}};
}

// appends the growth of a group to `rows` rows, keeping rows [0, keep)
inline void grow_rows(std::vector<Grow>& list, const std::vector<Rows>& group, size_t rows, size_t keep, bool zero) {
    for (const Rows& r : group) list.push_back({r.buf, rows * r.bytes, keep * r.bytes, zero});
}

XLayout xblock_layout(int S, uint32_t cap, bool dens);
size_t arena_floats(const glic_mapper* m, uint32_t cap);

// Every buffer whose size follows the Gaussian capacity, at capacity cap (densification statistics with dens).  params, m1 and m2
// come first (set_capacity's regrow fills entries 0-2); the anchors and the statistics keep their live rows; every buffer but
// pose_part and the anchors starts zeroed, so rows [P, cap) of the arenas are zero.
inline std::vector<Grow> capacity_buffers(glic_mapper* m, uint32_t cap, bool dens) {
    const size_t arena = arena_floats(m, cap) * sizeof(float);
    std::vector<Grow> list = {{m->params, arena, 0, true}, {m->m1, arena, 0, true}, {m->m2, arena, 0, true},
                              {m->act_opacity, (size_t)cap * 4, 0, true}, {m->act_scales, (size_t)cap * 12, 0, true},
                              {m->act_rots, (size_t)cap * 16, 0, true}, {m->radii, (size_t)cap * 4, 0, true},
                              {m->g_conic, (size_t)cap * (16 + 12 + 4), 0, true}, {m->geom_ws, glic_geom_bytes((int)cap), 0, true},
                              {m->xblock, xblock_layout(m->S, cap, dens).bytes, 0, true},
                              {m->pose_part, pose_partials_count(cap) * sizeof(double)}, {m->anchor, (size_t)cap * 4, (size_t)m->P * 4}};
    if (dens) grow_rows(list, densification_rows(m), cap, m->P, true);
    return list;
}

// after the capacity-sized buffers or the exchange block changed: the pointers into them, the exchange layout x and capacity cap
inline void adopt_capacity(glic_mapper* m, uint32_t cap, const XLayout& x) {
    m->g_mean2D = m->g_conic + (size_t)cap * 4;           // conic first: float4-aligned
    m->g_opacity = m->g_mean2D + (size_t)cap * 3;
    m->x = x;
    m->peers[m->cfg.rank] = m->xblock;
    m->Pcap = cap;
    m->st.capacity = cap;
}

// The six row groups of a packed block of capacity cap (an arena, or with M = 0 the exchange block's gradients), in
// glic_packed_offsets order; rest is null without SH rest (M = 0)
struct ArenaRows {
    float *rot, *xyz, *log_scale, *opacity, *dc, *rest;
    std::array<float*, 6> groups() const { return {rot, xyz, log_scale, opacity, dc, rest}; }
};

// draw(counters), then a synchronisation; a binning overflow grows the workspace by regrow(pairs needed), counts the regrow and
// draws again, up to 4 attempts.  The caller has drained the ring (poll_ring(wait)), so ring slot 0's pinned counters are free.
template <typename Draw, typename Regrow>
int draw_settled(glic_mapper* m, Draw draw, Regrow regrow) {
    for (int attempt = 0; attempt < 4; ++attempt) {
        long long* cnt = m->counters_host;
        MAP_TRY(draw(cnt));
        GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
        if (!cnt[2]) break;
        MAP_TRY(regrow(cnt[0] + cnt[0] / 4));
        ++m->st.overflow_regrows;
    }
    return GLIC_OK;
}

// ---- helpers defined in mapper.cu ----------------------------------------------------------------------------------------------
void camera_block(int W, int H, double fx, double fy, double cx, double cy, const float* R_wc, const float* t_wc, CamBlock& o,
                  double* T12 = nullptr);
glic_view make_view(const CamBlock& c, const float* cam, int W, int H);
const MaskView* keyframe_mask(const Keyframe& kf, int W, MaskView& mv, int x0 = 0);
int grow(glic_mapper* m, const std::vector<Grow>& list, const std::function<int(Buf*)>& fill = nullptr);
int reserve(glic_mapper* m, Buf& b, size_t need);
ArenaRows arena_rows(float* base, uint32_t cap, int M);
std::array<size_t, 6> group_widths(int M);
void config_camera_block(const glic_mapper* m, const float* R_wc, const float* t_wc, CamBlock& o, double* T12 = nullptr);
int keyframe_at(glic_mapper* m, int is_train, int index, const char* what, const Keyframe*& out);
int set_capacity(glic_mapper* m, uint32_t cap);
int dens_reset(glic_mapper* m);
int launch_pose_kernel(glic_mapper* m, int S, PoseBatch b, const float* slot_grads, double* T, float* pose_f, float* adam_m, float* adam_v,
                       int* adam_t, float lr_rho, float lr_omega, const unsigned int* skip);
int grow_render_binning(glic_mapper* m, int64_t pairs);
int regrow_after_skip(glic_mapper* m, int64_t pairs);
int poll_ring(glic_mapper* m, bool wait);
int activate(glic_mapper* m, float* zero4 = nullptr);
int forward_view(glic_mapper* m, const glic_view& v, int no_color, long long* counters);
int forward_settled(glic_mapper* m, const glic_view& v, int no_color);
int load_gt(glic_mapper* m, const Keyframe& kf, float* dst, cudaMemcpyKind kind, cudaStream_t s);
int photometric_loss(glic_mapper* m, int H, int W, const float* img, const float* gt, const float* E, float* loss, float* dL_dimg, float* dL_dE,
                     bool loss_zeroed = false, const MaskView* mask = nullptr, uint32_t valid = 0);
int backward_view(glic_mapper* m, const glic_view& v, float* col, const CompactGrads& cg, cudaEvent_t after_render);
int pose_check(const float* R_wc9, const float* t_wc3, const char* what);
int scored_image_to_host(glic_mapper* m, float* rgb_host);
int scored_lpips(glic_mapper* m, int W);
int read_eval_out(glic_mapper* m, float* out, int n);

// ---- mapper_density.cu ----------------------------------------------------------------------------------------------------------
int scheduled_density_step(glic_mapper* m);    // optimize()'s density control
int views_check(const glic_mapper* m, const int* views, int n, const char* what);

// ---- mapper_views.cu ------------------------------------------------------------------------------------------------------------
bool finite_at_least_zero(float x);
// The workspace of glic_mapper_render_camera and the meshing (render_carve)
struct RenderPlanes { float* cam; void* image_ws; float *color, *T, *depth, *median, *rgb; };
size_t render_carve(void* ws, int W, int H, RenderPlanes* out);
int draw_rows(glic_mapper* m, size_t first, const glic_view& v, const RenderPlanes& r, float* depth, float* median);

}  // namespace mapper_impl

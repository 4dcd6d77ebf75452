// common.cuh -- shared declarations of the glic_b200 CUDA library (sm_90a only).
//
// Workspace layouts (all opaque to callers; see DESIGN.md "HBM layout"):
//   geom_ws   : GeomHeader | rec[3P] float4 (48 B AoS splat record) | depth_keys[2][P] u32 + order[2][P] u32
//               (depth sort ping-pong) | offsets[P] u32 (inclusive scan of tiles_touched in DEPTH order) |
//               clamped[P] u8 | look-back status u64[blocks] | depth-sort temp
//   image_ws  : ImageHeader | ranges[T] uint2 | bucket_offsets[T] u32 | max_contrib[T] u32 |
//               n_contrib[HW] u32 | pixel_colors[3HW] f32
//   binning_ws: BinHeader | tile keys[2][R] u32 | vals[2][R] u32 | sort temp
//   sample_ws : bucket_to_tile[Bmax] u32 | ckpt[Bmax*256] float4 (T, C.r, C.g, C.b)
//   det_ws    : DetState (the deterministic render backward's entries, 32 per bucket)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <string>
#include <initializer_list>
#include <utility>

#include "../../include/glic_b200.h"

namespace glic {

constexpr int TILE = GLIC_TILE;
constexpr int TILE_PIX = TILE * TILE;   // 256 pixels, one CTA
constexpr int BUCKET = GLIC_BUCKET;     // 32 splats per checkpoint bucket
constexpr int PRE_THREADS = 256;        // Gaussians per preprocess CTA
constexpr int NUM_SMS = 132;            // H100 SXM: sizes the grid-stride launches (a grid cap, never a correctness bound)

// torch::sigmoid of an opacity logit (GaussianModel::getOpacity, gaussian.cpp:147-150) as the activation kernel evaluates it;
// glic_mapper_prune decides with the same expression, so its 1/255 cut is the preprocess's o < 1/255 test bit for bit
__device__ __forceinline__ float opacity_activation(float logit) { return 1.0f / (1.0f + expf(-logit)); }
// the SplitMix64 finaliser (Steele, Lea, Flood, OOPSLA 2014): the counter-based generators of the skybox and the split children
__device__ __forceinline__ uint64_t splitmix64_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
// torch::exp of a log-scale and normalize (p = 2, eps = 1e-12) of a raw rotation (getScaling / getRotation) as the activation
// kernel evaluates them; glic_mapper_densify decides and places the split children with the same expressions
__device__ __forceinline__ float scale_activation(float log_scale) { return expf(log_scale); }
__device__ __forceinline__ float4 rotation_activation(float4 q) {
    const float n = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);
    return make_float4(q.x / n, q.y / n, q.z / n, q.w / n);
}

// ---- error plumbing --------------------------------------------------------------------
void set_error(const std::string& s);
extern unsigned long long g_launches;

#define GLIC_CUDA_TRY(expr)                                                                   \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            glic::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));             \
            return GLIC_ERR_CUDA;                                                             \
        }                                                                                     \
    } while (0)

#define GLIC_LAUNCH_CHECK()                                                                   \
    do {                                                                                      \
        ++glic::g_launches;                                                                   \
        cudaError_t _e = cudaGetLastError();                                                  \
        if (_e != cudaSuccess) {                                                              \
            glic::set_error(std::string("kernel launch: ") + cudaGetErrorString(_e));       \
            return GLIC_ERR_CUDA;                                                             \
        }                                                                                     \
    } while (0)

// ---- programmatic dependent launch (PDL) ------------------------------------------------
// A kernel launched by GLIC_LAUNCH_PDL may start while the stream's previous kernel is still running.  Every such kernel
// calls pdl_enter() before anything else: it lets the stream's next kernel launch (that kernel cannot run ahead, it waits
// the same way), then waits for the previous kernel to complete and its writes to be visible.  Only kernels that call
// pdl_enter() on every path may be launched this way.  Launched without the attribute, both instructions do nothing.
__device__ __forceinline__ void pdl_enter() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// launch_pdl(kernel, grid, block, smem, stream, args...), counted and checked like GLIC_LAUNCH_CHECK
#define GLIC_LAUNCH_PDL(...)                                                                  \
    do {                                                                                      \
        ++glic::g_launches;                                                                   \
        cudaError_t _e = glic::launch_pdl(__VA_ARGS__);                                       \
        if (_e != cudaSuccess) {                                                              \
            glic::set_error(std::string("kernel launch: ") + cudaGetErrorString(_e));       \
            return GLIC_ERR_CUDA;                                                             \
        }                                                                                     \
    } while (0)

// ---- optional per-stage cudaEvent timing (glic_profile_*) ---------------------------------
bool profiling_on();
void profile_mark(int stage, bool begin, cudaStream_t s);
struct StageTimer {
    int stage; cudaStream_t s; bool on;
    StageTimer(int st, cudaStream_t stream) : stage(st), s(stream), on(profiling_on()) { if (on) profile_mark(stage, true, s); }
    ~StageTimer() { if (on) profile_mark(stage, false, s); }
};

// ---- arena carving (128-byte aligned sub-arrays) ----------------------------------------
struct Carver {
    char* base;
    size_t off;
    __host__ explicit Carver(void* p) : base(static_cast<char*>(p)), off(0) {}
    template <typename T>
    __host__ T* take(size_t count) {
        off = (off + 127) & ~size_t(127);
        T* p = reinterpret_cast<T*>(base + off);
        off += count * sizeof(T);
        return p;
    }
    __host__ size_t total() const { return (off + 127) & ~size_t(127); }
};

// Splat record, 48 bytes: three float4 per Gaussian (AoS so one gather = 1.5 sectors).
//   r0 = (x, y, conic.x, conic.y)   r1 = (conic.z, opacity, red, green)
//   r2 = (blue, depth, radius as int bits, hy = conservative vertical half-extent of the alpha >= 1/255 ellipse)
struct GeomHeader {
    unsigned int ticket;        // dynamic CTA id of the emit kernel's fused scan
    unsigned int total;         // R = sum of tiles_touched
    unsigned int visible;       // #Gaussians with radius > 0
    unsigned int order_cur;     // which ping-pong half holds the depth-sorted order
    unsigned int r_eff;         // R when it fits the binning workspace, else 0: what the sort / ranges / render use
    unsigned int overflow;      // 1 when R exceeded the capacity (frame invalid, caller re-runs with more room)
    unsigned int span_count;    // bump allocator of the row-span arena (preprocess -> emit)
    unsigned int pad[25];
};

size_t sort_temp_bytes(int64_t n);

struct GeomState {
    GeomHeader* hdr;
    float4* rec;
    uint32_t* depth_keys[2];    // float bits of depth (0xFFFFFFFF for culled Gaussians), sort ping-pong
    uint32_t* order[2];         // Gaussian indices, sorted by (depth, index) after the depth sort
    uint32_t* tiles;            // tiles_touched per Gaussian (index order)
    uint32_t* offsets;          // per Gaussian: END of its slot range = inclusive scan of tiles over the depth order
    uint32_t* tmask;            // per Gaussian: accept mask of a <= 32-tile rect, or first row-span entry of a bigger one
    uint32_t* spans;            // row spans (xa | xb << 16) of the big rects, bump-allocated per frame
    uint32_t span_cap;
    uint8_t* clamped;
    unsigned long long* scan_status;
    void* sort_temp;
    size_t sort_temp_size;
    __host__ static GeomState carve(void* ws, int P, size_t* bytes = nullptr) {
        const size_t n = P > 0 ? size_t(P) : 1;
        Carver c(ws);
        GeomState g;
        g.hdr = c.take<GeomHeader>(1);
        g.rec = c.take<float4>(size_t(3) * n);
        g.depth_keys[0] = c.take<uint32_t>(n);
        g.depth_keys[1] = c.take<uint32_t>(n);
        g.order[0] = c.take<uint32_t>(n);
        g.order[1] = c.take<uint32_t>(n);
        g.tiles = c.take<uint32_t>(n);
        g.offsets = c.take<uint32_t>(n);
        g.tmask = c.take<uint32_t>(n);
        g.span_cap = (uint32_t)(4 * n);
        g.spans = c.take<uint32_t>(4 * n);
        g.clamped = c.take<uint8_t>(n);
        g.scan_status = c.take<unsigned long long>((n + PRE_THREADS - 1) / PRE_THREADS + 1);
        g.sort_temp_size = sort_temp_bytes((int64_t)n);
        g.sort_temp = c.take<char>(g.sort_temp_size);
        if (bytes) *bytes = c.total();
        return g;
    }
    // the look-back status words preprocess_forward_kernel's P / PRE_THREADS CTAs use (zeroed before it runs)
    __host__ static size_t scan_status_bytes(int P) { return sizeof(unsigned long long) * ((P + PRE_THREADS - 1) / PRE_THREADS + 1); }
};

// Function attributes (opt-in dynamic shared memory) are per device: run `fn` once per (call site, device).
// `flags` is the call site's own static array.
inline bool first_use_on_device(bool (&flags)[64]) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    if (flags[dev]) return false;
    flags[dev] = true;
    return true;
}

struct ImageHeader {
    long long num_rendered;     // R
    unsigned int num_buckets;   // B
    unsigned int num_live_buckets;   // buckets some pixel reached (backward work list)
    unsigned int bwd_ticket;    // dynamic work counter of the backward's persistent warps (reset by live_scan_kernel)
    long long counters[4];      // {R, B, overflow, 0}: copied to the host asynchronously by glic_forward
    unsigned int pad[20];
};

struct ImageState {
    ImageHeader* hdr;
    uint2* ranges;
    uint32_t* bucket_offsets;
    uint32_t* max_contrib;
    uint32_t* live_offsets;     // inclusive scan of ceil(max_contrib/32) (backward's live-bucket list)
    uint32_t* n_contrib;
    float* pixel_colors;
    __host__ static ImageState carve(void* ws, int W, int H, size_t* bytes = nullptr) {
        const size_t T = size_t((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
        const size_t HW = size_t(W) * H;
        Carver c(ws);
        ImageState s;
        s.hdr = c.take<ImageHeader>(1);
        s.ranges = c.take<uint2>(T);
        s.bucket_offsets = c.take<uint32_t>(T);
        s.max_contrib = c.take<uint32_t>(T);
        s.live_offsets = c.take<uint32_t>(T);
        s.n_contrib = c.take<uint32_t>(HW);
        s.pixel_colors = c.take<float>(3 * HW);
        if (bytes) *bytes = c.total();
        return s;
    }
};

struct BinHeader {
    unsigned int sorted_in_b;   // 1 when the sorted list lives in keys[1]/vals[1]
    unsigned int pad[31];
};

struct BinningState {
    BinHeader* hdr;
    uint32_t* keys[2];          // tile ids
    uint32_t* vals[2];
    void* sort_temp;
    size_t sort_temp_size;
    __host__ static BinningState carve(void* ws, int64_t R, size_t* bytes = nullptr) {
        const size_t n = R > 0 ? size_t(R) : 1;
        Carver c(ws);
        BinningState b;
        b.hdr = c.take<BinHeader>(1);
        b.keys[0] = c.take<uint32_t>(n);
        b.keys[1] = c.take<uint32_t>(n);
        b.vals[0] = c.take<uint32_t>(n);
        b.vals[1] = c.take<uint32_t>(n);
        b.sort_temp_size = sort_temp_bytes(R);
        b.sort_temp = c.take<char>(b.sort_temp_size);
        if (bytes) *bytes = c.total();
        return b;
    }
};

struct SampleState {
    uint32_t* bucket_to_tile;
    float4* ckpt;               // [Bmax][256] (T, C.r, C.g, C.b) per pixel per bucket
    __host__ static SampleState carve(void* ws, int64_t max_buckets, size_t* bytes = nullptr) {
        const size_t n = max_buckets > 0 ? size_t(max_buckets) : 1;
        Carver c(ws);
        SampleState s;
        s.bucket_to_tile = c.take<uint32_t>(n);
        s.ckpt = c.take<float4>(n * TILE_PIX);
        if (bytes) *bytes = c.total();
        return s;
    }
};

// Deterministic render backward (render.cu, launch_render_backward_det): 32 entries per bucket of the sample workspace, each the
// nine values of one (tile, Gaussian) pair, keyed by gid; the keys and entry indices ping-pong through the stable tile sort.
//   det_ws: count u32 | keys[2][n] u32 | idx[2][n] u32 | vals[n][9] f32 | sort temp, n = 32 * max_buckets
struct DetState {
    unsigned int* count;
    uint32_t* keys[2];
    uint32_t* idx[2];
    float* vals;
    void* sort_temp;
    size_t sort_temp_size;
    int64_t cap;                // entries
    __host__ static DetState carve(void* ws, int64_t max_buckets, size_t* bytes = nullptr) {
        const int64_t n = (max_buckets > 0 ? max_buckets : 1) * BUCKET;
        Carver c(ws);
        DetState d;
        d.cap = n;
        d.count = c.take<unsigned int>(1);
        d.keys[0] = c.take<uint32_t>(n);
        d.keys[1] = c.take<uint32_t>(n);
        d.idx[0] = c.take<uint32_t>(n);
        d.idx[1] = c.take<uint32_t>(n);
        d.vals = c.take<float>(9 * (size_t)n);
        d.sort_temp_size = sort_temp_bytes(n);
        d.sort_temp = c.take<char>(d.sort_temp_size);
        if (bytes) *bytes = c.total();
        return d;
    }
};

// getHigherMsb (rasterizer_impl.cu:42-57): number of tile-id bits included in the sort.
inline uint32_t higher_msb(uint32_t n) {
    uint32_t msb = sizeof(n) * 4, step = msb;
    while (step > 1) {
        step /= 2;
        if (n >> msb) msb += step; else msb -= step;
    }
    if (n >> msb) msb++;
    return msb;
}

// Key bits of the tile sort.  Tile ids 0 .. T-1 need higher_msb(T - 1) bits; the reference's higher_msb(T) is one bit more
// when T is a power of two, which at T = GLIC_MAX_TILES would exceed the 16 bits the key emission histograms.  The sorted
// order is the same either way (a stable sort on a bit every key has clear).
inline int tile_sort_bits(int T) { return (int)higher_msb((uint32_t)(T - 1)); }

// Digit split of the LSD radix sorts (radix_sort.cu): ceil(end_bit / 8) passes, the key bits spread evenly over them
// (the wider digits first), so that no pass carries digits no key can have: 13 tile bits -> 7 + 6, 16 -> 8 + 8, 32 -> 4 x 8,
// 45 -> 8,8,8,7,7,7.  Producer kernels that build the sort's histograms count the same digits.
__host__ __device__ inline int sort_passes(int end_bit) { return (end_bit + 7) / 8; }
__host__ __device__ inline int sort_pass_bits(int end_bit, int pass) {
    const int p = sort_passes(end_bit);
    return end_bit / p + (pass < end_bit % p ? 1 : 0);
}
__host__ __device__ inline int sort_pass_shift(int end_bit, int pass) {
    const int p = sort_passes(end_bit);
    return pass * (end_bit / p) + (pass < end_bit % p ? pass : end_bit % p);
}
// Passes of the tile sort: its sorted pairs end in buffer (passes & 1) of the ping-pong pair.
inline int tile_sort_passes(int T) { return sort_passes(tile_sort_bits(T)); }
// key bits of the entry sort: gids 0 .. P-1 and the sentinel P
inline int det_key_bits(int P) { return 32 - __builtin_clz((unsigned)(P > 0 ? P : 1)); }
// the ping-pong half that holds the sorted entries (32-bit keys sort with 8-bit digits)
inline int det_sorted_half(int P) { return sort_passes(det_key_bits(P)) & 1; }

// View parameters passed by value to kernels (pointers stay device pointers).
struct ViewParams {
    const float* view;
    const float* proj;
    const float* campos;
    float tan_fovx, tan_fovy, focal_x, focal_y;
    float limx_neg, limx_pos, limy_neg, limy_pos;
    int W, H, grid_x, grid_y;
};

inline ViewParams make_view_params(const glic_view* v) {
    ViewParams p;
    p.view = v->viewmatrix; p.proj = v->projmatrix; p.campos = v->campos;
    p.tan_fovx = v->tan_fovx; p.tan_fovy = v->tan_fovy;
    p.focal_y = v->height / (2.0f * v->tan_fovy);     // rasterizer_impl.cu:348-349
    p.focal_x = v->width / (2.0f * v->tan_fovx);
    p.limx_neg = v->limx_neg; p.limx_pos = v->limx_pos; p.limy_neg = v->limy_neg; p.limy_pos = v->limy_pos;
    p.W = v->width; p.H = v->height;
    p.grid_x = (v->width + TILE - 1) / TILE; p.grid_y = (v->height + TILE - 1) / TILE;
    return p;
}

// Compact gradient outputs of the per-Gaussian backward (the mapper's form, see preprocess_backward.cu).  Null row pointers
// (g_xyz == NULL) with the two pose pointers set select the pose-only form: the view's pose gradient and nothing per row (the
// other row inputs and the densification pointers are then not read and must be NULL).
struct CompactGrads {
    float4* g_rot;            // [P] dL/d(raw rotation)
    float* g_xyz;             // [P,3]
    float* g_scale;           // [P,3] dL/d(log-scale)
    float* g_opacity;         // [P]   dL/d(opacity logit)
    const float* opacity;     // [P]   activated opacity (sigmoid output)
    const float* dL_dopacity; // [P]   dL/d(activated opacity) from the render backward
    const float4* rot_raw;    // [P]   raw (un-normalised) rotation
    int accumulate;           // 0: overwrite the geometric gradients, 1: add to them (second and later views of a rank)
    // camera-pose gradient of the view (preprocess_backward.cu, POSE); both NULL: not computed
    double* pose_partials;    // [ceil(P/128)][6] per-CTA float64 partial sums (pose_partials_count(capacity) doubles)
    float* pose_grad;         // [6] dL/d(rho, omega) of the view, written by the finish kernel
    // densification statistics of the view (glic_mapper_enable_densification); both NULL: not computed.  Written or accumulated
    // like the geometric gradients: |(dL/dmean2D.x, .y)| and 1 for a visible row, 0 and 0 for a culled one
    float* dens_norm;         // [P]
    float* dens_count;        // [P]
    // 1: the render backward's accumulators (dL_dmeans2D, dL_dconic, dL_dopacity, dL_dcolors) are zero in rows [0, P) already
    // (launch_view_flags zeroed them), so backward_compact does not
    int grads_zeroed = 0;
};
// doubles of the pose-gradient scratch for up to Pcap Gaussians
size_t pose_partials_count(uint32_t Pcap);

// out[j] = the G per-CTA float64 partials [G][N] summed in a fixed order (no atomics: two runs give the same bits).  One CTA of
// N warps, <<<1, 32 * N>>>: warp j sums component j lane-strided, then an xor butterfly.
template <int N>
__global__ void __launch_bounds__(32 * N)
partials_finish_kernel(unsigned G, const double* __restrict__ partials, float* __restrict__ out) {
    const int j = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double s = 0.0;
    for (unsigned b = lane; b < G; b += 32) s += partials[N * (size_t)b + j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[j] = (float)s;
}

// ---- stage launchers (defined in the .cu files) ------------------------------------------
// One launch that zeroes up to five spans (bytes a multiple of 4): a chain of dependent launches continues through it, where a
// memset would end it
struct ZeroSpan { void* p; size_t bytes; };
int launch_zero_spans(std::initializer_list<ZeroSpan> spans, cudaStream_t s);
// The caller zeroes g.hdr, the look-back status words (scan_status_bytes) and the depth sort's temp block
// (sort_prepare_bytes(P, 32)) first: the kernel counts into all three
int launch_preprocess_forward(int P, int D, int M, const float* means, const float* scales, float mod,
                              const float* rots, const float* opac, const float* dc, const float* sh,
                              const ViewParams& vp, bool no_color, int* radii, GeomState g, cudaStream_t s);
int launch_depth_scan(int P, GeomState g, const uint32_t* order, int64_t capacity, cudaStream_t s);
int launch_emit_keys(int P, const ViewParams& vp, GeomState g, uint32_t* tile_keys, uint32_t* vals, int64_t capacity, uint32_t* sort_hist_out,
                     int end_bit, cudaStream_t s);
// Sorts on bits [0,end_bit); returns 0/1 = index of the ping-pong buffer holding the result, <0 on error.
int launch_sort_pairs(int64_t n, int end_bit, uint64_t* keys[2], uint32_t* vals[2], void* temp, size_t temp_bytes,
                      cudaStream_t s);
// n_dev (optional): device-side true count <= n; kernels are launched for n (a capacity) and clip to *n_dev.
int launch_sort_pairs32(int64_t n, int end_bit, uint32_t* keys[2], uint32_t* vals[2], void* temp, size_t temp_bytes,
                        cudaStream_t s, const unsigned int* n_dev = nullptr, bool hist_ready = false);
// A producer kernel may build the digit histograms itself: sort_prepare() zeroes the temp block, the producer adds one count
// per key and pass into sort_hist(temp)[pass * 256 + digit] (digit = bits [sort_pass_shift, + sort_pass_bits) of the key),
// and the sort is launched with hist_ready = true.
int sort_prepare(int64_t n, int end_bit, void* temp, cudaStream_t s);
size_t sort_prepare_bytes(int64_t n, int end_bit);     // the bytes sort_prepare zeroes
uint32_t* sort_hist(void* temp);
// R: host-side count or capacity; r_dev (optional): device-side true count.  img.ranges must be zero; *sorted_in_b is set to cur
int launch_tile_ranges(int64_t R, const GeomHeader* ghdr, const uint32_t* tile_keys_sorted, int T, ImageState img, bool buckets,
                       unsigned int* sorted_in_b, int cur, cudaStream_t s);
int launch_render_forward(const ViewParams& vp, bool no_color, const uint32_t* point_list, GeomState g, ImageState img,
                          SampleState smp, float* out_color, float* out_final_T, cudaStream_t s);
// the inference form of the blend (glic_render): colour, final T and, when non-null, expected and median depth; nothing else
int launch_render_infer(const ViewParams& vp, const uint32_t* point_list, GeomState g, ImageState img, float* out_color,
                        float* out_final_T, float* out_depth, float* out_median, cudaStream_t s);
// the scoring form of the blend (glic_contribution): accumulates every taken pair's weight into max_weight (max) and hits (count)
// of its Gaussian, and every pixel it ends into ends (may be null); out_final_T (may be null) as launch_render_forward writes it
// with no_color
int launch_render_score(const ViewParams& vp, const uint32_t* point_list, GeomState g, ImageState img, float* max_weight,
                        uint64_t* hits, uint64_t* ends, float* out_final_T, cudaStream_t s);
int launch_render_backward(int P, const ViewParams& vp, int64_t max_buckets, const uint32_t* point_list, GeomState g,
                           ImageState img, SampleState smp, const float* dL_dpix, float* dL_dmean2D /*[P,3]*/,
                           float* dL_dconic /*[P,4]*/, float* dL_dopacity, float* dL_dcolors, cudaStream_t s,
                           bool exact = false /* expf for every pixel, no visit skip (tests) */,
                           unsigned long long* counters = nullptr /* [8], device: the counting form (render.cu BwdCount) */);
// The deterministic form of launch_render_backward (RP = 8 body, render.cu DetOut): WRITES the four 2-D gradients of every
// Gaussian with a contribution (rows without one keep what they held: the callers' zeros); independent of grid size and scheduling.
int launch_render_backward_det(int P, const ViewParams& vp, int64_t max_buckets, const uint32_t* point_list, GeomState g,
                               ImageState img, SampleState smp, DetState det, const float* dL_dpix, float* dL_dmean2D,
                               float* dL_dconic, float* dL_dopacity, float* dL_dcolors, cudaStream_t s);
int launch_preprocess_backward(int P, int D, int M, const float* means, const float* scales, float mod,
                               const float* rots, const float* sh, const ViewParams& vp, const int* radii, GeomState g,
                               float lambda_erank, const float* dL_dmean2D, const float* dL_dconic,
                               const float* dL_dcolors, float* dL_dmeans3D, float* dL_dcov3D, float* dL_ddc,
                               float* dL_dsh, float* dL_dscales, float* dL_drots, cudaStream_t s);

int launch_preprocess_backward_compact(int P, int D, int M, const float* means, const float* scales, float mod,
                                       const float* rots, const float* sh, const ViewParams& vp, const int* radii, GeomState g,
                                       const float* dL_dmean2D, const float* dL_dconic, const float* dL_dcolors,
                                       const CompactGrads& cg, cudaStream_t s);

// The backward of the last forward into the compact gradient form of preprocess_backward.cu (the mapper's).  dL_dcolors is zeroed
// and accumulated like the other 2-D gradients but may live anywhere (the mapper points it into its exchange block).
// after_render (optional) is recorded once the colour gradients are final; det_ws: NULL for the atomic render backward, else
// glic_deterministic_bytes(R, W, H) for the deterministic one.
int backward_compact(int P, int sh_degree, int M, const float* means3D, const float* scales, const float* rotations, const float* sh,
                     const glic_view* view, const int* radii, int64_t R, const void* geom_ws, const void* binning_ws,
                     const void* image_ws, const void* sample_ws, const float* dL_dpix, float* dL_dmeans2D, float* dL_dconic,
                     float* dL_dopacity, float* dL_dcolors, const CompactGrads& cg, cudaEvent_t after_render, cudaStream_t s,
                     void* det_ws);
int launch_adam_compact(uint32_t P, uint32_t Pcap, int D, int M, float* params, float* exp_avg, float* exp_avg_sq, const float* g_geo,
                        uint32_t Pcap_geo, const float* lr6, const float* g_color, const uint8_t* flags, const float* const* campos_dev,
                        int n_slots, float grad_scale, float color_scale, float b1, float b2, float eps, const unsigned int* skip_flag,
                        unsigned int* visible_count, cudaStream_t s, const float* g_dens = nullptr, float* dens_accum = nullptr,
                        float* dens_denom = nullptr, float dens_scale = 1.0f, const int* radii = nullptr, int* dens_maxr = nullptr);
// g_dens (optional): the densification statistics of the batch in the gradient block, norms [Pcap_geo] | counts [Pcap_geo]; the
// Adam launch adds dens_scale times them to dens_accum / dens_denom for every row visible in some slot, unless skip_flag is set.
// radii (with g_dens): [n_slots][Pcap_geo] each slot's screen radii; dens_maxr takes their max over the slots that see the row
// campos_dev: n_slots host-held device pointers, each slot's camera centre (read on the device)
// radii_out (optional): the view's radii copied next to its flags (the densification's screen-radius slot)
// what one view's loss and render backward accumulate into: the loss word and the per-Gaussian rows (conic [P,4], 16-byte aligned)
struct ViewZero { float *conic, *mean2D, *opacity, *colors, *loss; };
int launch_view_flags(int P, const int* radii, const GeomState& g, uint8_t* flags, cudaStream_t s, int* radii_out, float* overflow_word,
                      const ViewZero& z);
// glic_activations_forward with zero4[0..3] (optional) zeroed by the same kernel
int launch_activations_forward(int P, const float* opacity_logit, const float* log_scale, const float* rot_raw, float* opacity,
                               float* scale, float* rot, float* zero4, cudaStream_t stream);
// per-keyframe exposure (ssim.cu): one Adam step of every keyframe of a batch of S <= EXPO_MAX_SLOTS slots; slot_grads[S][12]
constexpr int EXPO_MAX_SLOTS = 32;
int launch_exposure_adam(int S, const int* kf_of_slot_host, const float* slot_grads, float* E, float* exp_avg, float* exp_avg_sq,
                         int* steps, float lr, const unsigned int* skip_flag, cudaStream_t s);
// A view of a bit-packed valid-pixel mask (glic_pack_mask): pixel (y, x) of the viewed H x W region is used when bit c & 31 of
// words[y * words_per_row + (c >> 5)] is set, c = x0 + x.  x0 lets a column crop read its frame's mask in place.
struct MaskView {
    const uint32_t* words;
    int words_per_row, x0;
};
__device__ __forceinline__ bool mask_bit(const MaskView& m, int y, int x) {
    const int c = m.x0 + x;
    return (m.words[(size_t)y * m.words_per_row + (c >> 5)] >> (c & 31)) & 1u;
}
// glic_eval_psnr_ssim with an optional exposure E (3 channels) applied to img before the clamp
// fixed (optional, fixed_order_sums_bytes(H, W)): the two sums in a fixed order instead of float64 atomics
// mask (optional, `valid` > 0 pixels set): both clamped images are 0 at masked pixels, and MSE and the SSIM mean are taken over
// the CH * valid used elements
int eval_psnr_ssim(int CH, int H, int W, const float* img, const float* gt, const float* E, float* out2, void* scratch,
                   size_t scratch_bytes, void* stream, void* fixed = nullptr, const MaskView* mask = nullptr, uint32_t valid = 0);
// the native mapper's photometric loss: glic_l1_ssim_loss (3 channels) or, with E, glic_l1_ssim_loss_exposure; partials (optional,
// fixed_order_sums_bytes(H, W)) sums the loss value in a fixed order instead of with float atomics; loss_zeroed: *loss is zero
// already (the float atomics add into it without a memset first); mask (optional, `valid` > 0 pixels set): the masked loss of
// glic_l1_ssim_loss_masked
int photometric_loss_sum(int H, int W, float lambda_dssim, const float* img, const float* gt, const float* E, float* loss, float* dL_dimg,
                         float* dL_dE, void* scratch, size_t scratch_bytes, void* partials, cudaStream_t s, bool loss_zeroed = false,
                         const MaskView* mask = nullptr, uint32_t valid = 0);
// glic_pack_mask: bits and count of a device byte mask [H][W], on stream s
int launch_pack_mask(int H, int W, const uint8_t* valid, uint32_t* words, uint32_t* count, cudaStream_t s);
inline int mask_words_per_row(int W) { return (W + 31) / 32; }
size_t fixed_order_sums_bytes(int H, int W);
// out[3][H][W] = img exposed by E (optional) and clamped to [0,1], element for element the image eval_psnr_ssim scores
int launch_scored_image(int H, int W, const float* img, const float* E, float* out, cudaStream_t s);
// the clamped (and exposed) images eval_psnr_ssim scored, left in its scratch: which = 0 the image, 1 the ground truth
const float* eval_clamped(const void* scratch, int CH, int H, int W, int which);
// stable compaction of the arenas (prune.cu): glic_mapper_densify_and_prune, glic_mapper_densify (nothing removed) and
// glic_mapper_prune (nothing selected) select once and gather every arena by the selection's index map.
// The selection's inputs (device pointers of rows [0, P)) and parameters, as the header states them
struct DensitySelect {
    uint32_t P, n_sky;
    const float *accum, *denom;      // both null: no row is selected (class 0 for every row), and neither is read
    const float *log_scale, *logit;  // log_scale is read only for a selected row, or when max_world_scale > 0
    const int* maxr;                 // read only when max_screen_radius > 0
    float grad_threshold, clone_max, min_opacity, max_world_scale;
    int max_screen_radius;
    // glic_mapper_prune_unseen's test: both null (the default), no row goes by it and neither is read
    const float* score_max = nullptr;
    const uint64_t* score_hits = nullptr;
    const uint64_t* score_ends = nullptr;   // pixels the row ends: they count towards min_hits with its hits
    float min_weight = 0.0f;
    uint64_t min_hits = 0;
    int score_sky = 0;               // 1: sky rows can go by it too
};
// select: the fate of every row; result_host[6] = {clones, splits, surviving kept rows, surviving clones, surviving split rows,
// surviving sky rows}, synchronises s; the scratch then holds the index map of the surviving rows (density_index: idx[new] = old)
// and the children's keys.  children: rows [first, first + 2 n) of the arena, copies of the n surviving split rows' parents,
// become their children in place (xyz and log-scale); P_select is the P the selection ran on, n_split its splits.
size_t density_scratch_bytes(uint32_t P);
int launch_density_select(const DensitySelect& a, void* scratch, uint32_t* result_host, cudaStream_t s);
const uint32_t* density_index(const void* scratch, uint32_t P);
int launch_densify_children(float* params, uint32_t Pcap, int M, uint32_t first, uint32_t n, const void* scratch, uint32_t P_select,
                            uint32_t n_split, uint64_t seed, uint64_t call, cudaStream_t s);
// output rows [0, rows_out) of every group of dst: row r < rows_valid takes row idx[r] of src, the others are zero; src and dst
// are arenas of capacity Pcap
int launch_gather_rows(const float* src, float* dst, uint32_t Pcap, int M, uint32_t rows_out, uint32_t rows_valid, const uint32_t* idx,
                       cudaStream_t s);
// dst[r] = r < rows_valid ? src[idx[r]] : 0 for r < rows_out (one 32-bit word per row)
int launch_gather_words(const void* src, void* dst, uint32_t rows_out, uint32_t rows_valid, const uint32_t* idx, cudaStream_t s);
// glic_mapper_reset_opacity on rows [first, P) of the opacity group of the three arenas
int launch_reset_opacity(uint32_t first, uint32_t P, uint32_t Pcap, int M, float* params, float* m1, float* m2, float max_opacity,
                         float reset_logit, cudaStream_t s);
}  // namespace glic

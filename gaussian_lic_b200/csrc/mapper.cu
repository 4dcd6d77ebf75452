// mapper.cu -- the native mapping host (include/glic_b200.h "Native mapping host"; SURVEY 8f ranks 1-4).
//
// C++ counterpart of the reference's GaussianModel + extend() + optimize() + evaluateVisualQuality() + saveMap()
// (/root/reference/src/gaussian.cpp:113-830, camera.h:38-110) on top of this library's kernels: one object per GPU, plain
// CUDA runtime, no torch, no Python.  What is different from the reference loop, by design:
//   * the model, its Adam moments and every per-Gaussian buffer live in capacity-sized arenas: extend() appends in place
//     (densificationPostfix re-allocates and copies all six parameter tensors and both moment tensors per keyframe);
//   * an iteration enqueues ~25 asynchronous launches and never blocks the host (the reference synchronises 5x per
//     iteration, gaussian.cpp:679,692,698,704,713); the pinned keyframe image travels on a copy stream into a
//     double buffer; binning overflow is detected with a lag through pinned counters and skipped on the device;
//   * gradients never exist as [P,59]: see the header comment of preprocess_backward.cu / adam_compact_kernel;
//   * multi-GPU (view-sharded): per-view colour gradients + flag bytes are PUSHED to every peer's exchange block by the
//     copy engines over NVLink as soon as the render backward has produced them (overlapping the per-Gaussian backward),
//     the 11 geometric floats are mean-reduced in place by the two-shot kernel of p2p.cu; every replica then runs the same
//     Adam launch on the same bytes.  With densification on, the view's statistics ride along as two more rows (13 floats).
#include "mapper_state.cuh"
#include "adam_math.cuh"
#include "pose_correction.cuh"

#include <algorithm>
#include <array>
#include <atomic>
#include <cmath>
#include <cstring>
#include <functional>
#include <initializer_list>
#include <memory>
#include <nv/target>
#include <utility>
#include <vector>

namespace mapper_impl {

// the pose-independent projection P of camera.h (row-major), with the FoV from the intrinsics (float members)
void proj_matrix(int W, int H, double fx, double fy, double cx, double cy, float* Pm, float* fov2) {
    const float fovx = (float)(2.0 * std::atan(W / (2.0 * fx))), fovy = (float)(2.0 * std::atan(H / (2.0 * fy)));
    const float znear = 0.01f, zfar = 100.0f;
    for (int i = 0; i < 16; ++i) Pm[i] = 0.0f;
    Pm[0] = (float)(1.0 / std::tan((double)fovx / 2));
    Pm[5] = (float)(1.0 / std::tan((double)fovy / 2));
    Pm[2] = (2.0f * (float)cx - (float)W) / (float)W;
    Pm[6] = (2.0f * (float)cy - (float)H) / (float)H;
    Pm[14] = 1.0f;
    Pm[10] = zfar / (zfar - znear);
    Pm[11] = -(zfar * znear) / (zfar - znear);
    fov2[0] = fovx; fov2[1] = fovy;
}

// One IEEE double / float operation each, on the device and on the host alike: the _rn intrinsics keep nvcc from contracting
// them into FMAs, and x86-64 host code is compiled without FMA.
__host__ __device__ inline double dmul(double a, double b) { NV_IF_ELSE_TARGET(NV_IS_DEVICE, (return __dmul_rn(a, b);), (return a * b;)) }
__host__ __device__ inline double dadd(double a, double b) { NV_IF_ELSE_TARGET(NV_IS_DEVICE, (return __dadd_rn(a, b);), (return a + b;)) }
__host__ __device__ inline float fmul(float a, float b) { NV_IF_ELSE_TARGET(NV_IS_DEVICE, (return __fmul_rn(a, b);), (return a * b;)) }
__host__ __device__ inline float fadd(float a, float b) { NV_IF_ELSE_TARGET(NV_IS_DEVICE, (return __fadd_rn(a, b);), (return a + b;)) }
__host__ __device__ inline float d2f(double a) { NV_IF_ELSE_TARGET(NV_IS_DEVICE, (return __double2float_rn(a);), (return (float)a;)) }

// The pose-dependent part of camera.h:38-110 from a float pose: the world->view matrix Rt and the full projection P Rt, both
// handed to the kernels transposed (column-major), and the camera centre -R_cw^T t_cw, into cam36 = view16 | proj16 | campos4;
// T12 (optional) = the float64 T_cw = R_cw (row-major) | t_cw they are formed from.  The host (camera_block) and the pose step
// on the device both build the block here, so a refined keyframe's block equals glic_camera_block of its float pose bit for bit.
__host__ __device__ void pose_camera(const float* R_wc, const float* t_wc, const float* Pm, float* cam36, double* T12) {
    double Rcw[9], tcw[3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rcw[3 * i + j] = (double)R_wc[3 * j + i];
    for (int i = 0; i < 3; ++i)
        tcw[i] = -dadd(dadd(dmul(Rcw[3 * i], (double)t_wc[0]), dmul(Rcw[3 * i + 1], (double)t_wc[1])), dmul(Rcw[3 * i + 2], (double)t_wc[2]));
    float Rt[16];
    for (int e = 0; e < 16; ++e) Rt[e] = 0.0f;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) Rt[4 * i + j] = d2f(Rcw[3 * i + j]);
        Rt[4 * i + 3] = d2f(tcw[i]);
    }
    Rt[15] = 1.0f;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float acc = 0.f;
            for (int k = 0; k < 4; ++k) acc = fadd(acc, fmul(Pm[4 * i + k], Rt[4 * k + j]));
            cam36[16 + 4 * j + i] = acc;                                   // proj, column-major
        }
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) cam36[4 * c + r] = Rt[4 * r + c];      // view, column-major
    for (int i = 0; i < 3; ++i)
        cam36[32 + i] = d2f(-dadd(dadd(dmul(Rcw[i], tcw[0]), dmul(Rcw[3 + i], tcw[1])), dmul(Rcw[6 + i], tcw[2])));
    cam36[35] = 0.f;
    if (T12) {
        for (int e = 0; e < 9; ++e) T12[e] = Rcw[e];
        for (int i = 0; i < 3; ++i) T12[9 + i] = tcw[i];
    }
}

// camera.h:38-110 in closed form: FoV from the intrinsics (float members), pose_camera, the asymmetric clamp limits of :63-66
void camera_block(int W, int H, double fx, double fy, double cx, double cy, const float* R_wc, const float* t_wc, CamBlock& o,
                  double* T12) {
    float Pm[16], fov2[2];
    proj_matrix(W, H, fx, fy, cx, cy, Pm, fov2);
    pose_camera(R_wc, t_wc, Pm, o.view, T12);                         // view | proj | campos are contiguous
    o.tanfovx = std::tan(fov2[0] * 0.5f);
    o.tanfovy = std::tan(fov2[1] * 0.5f);
    const float ffx = (float)fx, ffy = (float)fy, fcx = (float)cx, fcy = (float)cy;
    o.lim[0] = -0.15f * W / ffx - fcx / ffx; o.lim[1] = 1.15f * W / ffx - fcx / ffx;
    o.lim[2] = -0.15f * H / ffy - fcy / ffy; o.lim[3] = 1.15f * H / ffy - fcy / ffy;
}

// the rasterizer's view of a W x H frame from c's scalars and cam, the 36 device floats of c's view | proj | campos
glic_view make_view(const CamBlock& c, const float* cam, int W, int H) {
    return glic_view{cam, cam + 16, cam + 32, c.tanfovx, c.tanfovy, c.lim[0], c.lim[1], c.lim[2], c.lim[3], W, H};
}

std::atomic<int> fail_countdown{0};          // glic_debug_fail_allocation
std::atomic<int64_t> live_allocations{0};    // glic_debug_mapper_allocations

// the view of kf's whole mask from column x0 on, or nullptr when kf has none
const MaskView* keyframe_mask(const Keyframe& kf, int W, MaskView& mv, int x0) {
    if (!kf.mask_valid) return nullptr;
    mv = MaskView{kf.mask, mask_words_per_row(W), x0};
    return &mv;
}

// final_T = 0 at the masked pixels of an H x W frame: extend() then takes them as covered and seeds nothing there
__global__ void __launch_bounds__(256) mask_final_T_kernel(int H, int W, MaskView mk, float* __restrict__ T) {
    const size_t n = (size_t)H * W;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        if (!mask_bit(mk, (int)(i / W), (int)(i % W))) T[i] = 0.0f;
}

inline uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }

// ---- pose refinement (glic_mapper_enable_pose_refinement) ---------------------------------------------------------------
// Keyframe k's pose is T_cw = [R_cw | t_cw] (float64 master, R_cw row-major), perturbed as Exp(delta) T_cw with
// delta = (rho, omega) in the camera frame.  Each step: torch::optim::Adam on the 6-vector (as the exposure step), then
// T_cw <- Exp(u) T_cw, the float pose (R_wc = R_cw^T, t_wc = -R_cw^T t_cw) re-derived from it, and the device camera block
// (view16 | proj16 | campos4) rebuilt from those floats by pose_camera.

// SE(3) exponential of u = (rho, omega): R = I + A K + B K^2, V = I + B K + C K^2, K = [omega]_x; t = V rho
__device__ void se3_exp(const double u[6], double R[9], double t[3]) {
    const double wx = u[3], wy = u[4], wz = u[5];
    const double th2 = wx * wx + wy * wy + wz * wz;
    double A, B, C;
    if (th2 < 1e-4) {                     // theta < 1e-2: Taylor series to theta^6 (the next terms are below 1e-21)
        A = 1.0 - th2 / 6.0 * (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0));
        B = 0.5 * (1.0 - th2 / 12.0 * (1.0 - th2 / 30.0 * (1.0 - th2 / 56.0)));
        C = (1.0 / 6.0) * (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0 * (1.0 - th2 / 72.0)));
    } else {
        const double th = sqrt(th2), s = sin(th), sh = sin(0.5 * th);
        A = s / th;
        B = 2.0 * sh * sh / th2;
        C = (th - s) / (th2 * th);
    }
    const double K[9] = {0.0, -wz, wy, wz, 0.0, -wx, -wy, wx, 0.0};
    double K2[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) K2[3 * i + j] = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
    double V[9];
    for (int e = 0; e < 9; ++e) {
        const double I = (e % 4 == 0) ? 1.0 : 0.0;
        R[e] = I + A * K[e] + B * K2[e];
        V[e] = I + B * K[e] + C * K2[e];
    }
    for (int i = 0; i < 3; ++i) t[i] = V[3 * i] * u[0] + V[3 * i + 1] * u[1] + V[3 * i + 2] * u[2];
}

// The float pose (R_wc = R_cw^T, t_wc = -R_cw^T t_cw) of the float64 T_cw = Rn (row-major) | tn into f (R_wc | t_wc), and the
// camera block of that float pose into cam: the pose step and glic_mapper_correct_poses re-derive a refined keyframe here
__device__ __forceinline__ void pose_derive(const double* Rn, const double* tn, const float* Pm, float* f, float* cam) {
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) f[3 * i + j] = (float)Rn[3 * j + i];
        f[9 + i] = (float)(-(Rn[i] * tn[0] + Rn[3 + i] * tn[1] + Rn[6 + i] * tn[2]));
    }
    pose_camera(f, f + 9, Pm, cam, nullptr);
}

// One thread per slot; the first slot that holds a keyframe steps it with the batch gradient of keyframe_batch_grad and
// torch_adam_delta, as the exposure step does.  A set overflow word leaves the pose, m, v and t unchanged; an update of
// exactly zero leaves the pose and its camera block unchanged.
__global__ void __launch_bounds__(MAX_SLOTS)
pose_step_kernel(int S, PoseBatch b, const float* __restrict__ slot_grads /* [S][8] */, double* __restrict__ T /* [kf][12] */,
                 float* __restrict__ pose_f /* [kf][12] */, float* __restrict__ m, float* __restrict__ v, int* __restrict__ t,
                 float lr_rho, float lr_omega, const unsigned int* __restrict__ skip) {
    if (*skip) return;
    const int s = threadIdx.x;
    if (s >= S || !first_slot_of_keyframe(b.kf, s)) return;
    const int kf = b.kf[s];
    const int step = t[kf] + 1;
    double u[6];
    bool moved = false;
    for (int j = 0; j < 6; ++j) {
        const float g = keyframe_batch_grad(b.kf, S, s, slot_grads, 8, j);
        const size_t i = 6 * (size_t)kf + j;
        const float uj = torch_adam_delta(g, m[i], v[i], j < 3 ? lr_rho : lr_omega, step);
        u[j] = (double)uj;
        moved |= uj != 0.0f;
    }
    t[kf] = step;
    if (!moved) return;
    double R[9], tu[3];
    se3_exp(u, R, tu);
    double* Tk = T + 12 * (size_t)kf;
    double Rn[9], tn[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) Rn[3 * i + j] = R[3 * i] * Tk[j] + R[3 * i + 1] * Tk[3 + j] + R[3 * i + 2] * Tk[6 + j];
        tn[i] = R[3 * i] * Tk[9] + R[3 * i + 1] * Tk[10] + R[3 * i + 2] * Tk[11] + tu[i];
    }
    for (int e = 0; e < 9; ++e) Tk[e] = Rn[e];
    for (int i = 0; i < 3; ++i) Tk[9 + i] = tn[i];
    pose_derive(Rn, tn, b.Pm, pose_f + 12 * (size_t)kf, b.cam[s]);
}

// glic_mapper_correct_poses under pose refinement: slot s < S moves keyframe b.kf[s] by its record dT = [R | t]:
// T_cw <- T_cw dT^-1 = R_cw R^T | t_cw - (R_cw R^T) t, then the float pose and the camera block as the pose step derives them
__global__ void __launch_bounds__(MAX_SLOTS)
pose_correct_kernel(int S, PoseBatch b, const glic_rigid_correction* __restrict__ table, double* __restrict__ T, float* __restrict__ pose_f) {
    const int s = threadIdx.x;
    if (s >= S) return;
    const int kf = b.kf[s];
    const double* R = table[kf].R;
    const double* t = table[kf].t;
    double* Tk = T + 12 * (size_t)kf;
    double Rn[9], tn[3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rn[3 * i + j] = dadd(dadd(dmul(Tk[3 * i], R[3 * j]), dmul(Tk[3 * i + 1], R[3 * j + 1])), dmul(Tk[3 * i + 2], R[3 * j + 2]));
    for (int i = 0; i < 3; ++i) tn[i] = dadd(Tk[9 + i], -dadd(dadd(dmul(Rn[3 * i], t[0]), dmul(Rn[3 * i + 1], t[1])), dmul(Rn[3 * i + 2], t[2])));
    for (int e = 0; e < 9; ++e) Tk[e] = Rn[e];
    for (int i = 0; i < 3; ++i) Tk[9 + i] = tn[i];
    pose_derive(Rn, tn, b.Pm, pose_f + 12 * (size_t)kf, b.cam[s]);
}

// ---- raw frames (glic_mapper_add_frame; Dataset::addFrame, gaussian.cpp:41-111) -------------------------------------------

// Eigen::Quaterniond(w, x, y, z).toRotationMatrix() in Eigen's operation order, without normalisation; q = (x, y, z, w).
// Host code: x86-64 is compiled without FMA, so every operation rounds once.
void quat_rotation(const double q[4], double R[9]) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz;         R[2] = txz + twy;
    R[3] = txy + twz;         R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;         R[7] = tyz + twx;         R[8] = 1.0 - (txx + tyy);
}

// gaussian.cpp:66-70: each new point's depth in its own frame's camera, Eigen's fixed-size product without FMA,
// (float)(((Rcw20 p0 + Rcw21 p1) + Rcw22 p2) + tcw2) with p the point in double
__global__ void __launch_bounds__(256)
scan_depth_kernel(int n, const float* __restrict__ xyz, double r0, double r1, double r2, double t2, float* __restrict__ depth) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = xyz + 3 * (size_t)i;
    const double d = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r0, (double)p[0]), __dmul_rn(r1, (double)p[1])), __dmul_rn(r2, (double)p[2])), t2);
    depth[i] = __double2float_rn(d);
}

// the Dataset's colours, rgb / 255.0 in double (gaussian.cpp:65): initialize() reads the doubles, extend() floats of them
// (gaussian.cpp:517-519)
template <typename T>
__global__ void __launch_bounds__(256) scan_colour_kernel(int n3, const uint8_t* __restrict__ rgb, T* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n3) out[i] = (T)__ddiv_rn((double)rgb[i], 255.0);
}

// The one way a mapper's buffers grow: allocate every new buffer; on the mapper's stream zero those that start zeroed and copy the
// kept prefixes (then `fill`, which set_capacity uses to regrow the arenas into the new buffers); synchronise; only then swap the
// new buffers in and release the old.  A failed allocation leaves every buffer as it was.
int grow(glic_mapper* m, const std::vector<Grow>& list, const std::function<int(Buf*)>& fill) {
    std::vector<Buf> fresh(list.size());
    Buf* b = fresh.data();
    for (const Grow& g : list) MAP_TRY((b++)->allocate(g.bytes));
    b = fresh.data();
    for (const Grow& g : list) {
        if (g.zero) GLIC_CUDA_TRY(cudaMemsetAsync(b->raw(), 0, g.bytes, m->stream));
        if (g.keep) GLIC_CUDA_TRY(cudaMemcpyAsync(b->raw(), g.buf.raw(), g.keep, cudaMemcpyDeviceToDevice, m->stream));
        ++b;
    }
    if (fill) MAP_TRY(fill(fresh.data()));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    b = fresh.data();
    for (const Grow& g : list) g.buf = std::move(*b++);
    return GLIC_OK;
}

// grows b to at least `need` bytes without keeping its contents
int reserve(glic_mapper* m, Buf& b, size_t need) { return need <= b.bytes() ? GLIC_OK : grow(m, {Grow{b, need}}); }

size_t arena_floats(const glic_mapper* m, uint32_t cap) { return glic_packed_floats(cap, (uint32_t)m->M); }

ArenaRows arena_rows(float* base, uint32_t cap, int M) {
    size_t off[6];
    glic_packed_offsets(cap, (uint32_t)M, off);
    return {base + off[0], base + off[1], base + off[2], base + off[3], base + off[4], M ? base + off[5] : nullptr};
}
// floats per row of each group, in the same order
std::array<size_t, 6> group_widths(int M) { return {4, 3, 3, 1, 3, (size_t)3 * M}; }

float* geo_ptr(const glic_mapper* m) { return static_cast<float*>(m->xblock.raw()); }

void config_camera_block(const glic_mapper* m, const float* R_wc, const float* t_wc, CamBlock& o, double* T12) {
    camera_block(m->cfg.width, m->cfg.height, m->cfg.fx, m->cfg.fy, m->cfg.cx, m->cfg.cy, R_wc, t_wc, o, T12);
}

int keyframe_at(glic_mapper* m, int is_train, int index, const char* what, const Keyframe*& out) {
    const auto& list = is_train ? m->train : m->test;
    if (index < 0 || index >= (int)list.size()) { set_error(std::string(what) + ": keyframe index out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    out = &list[index];
    return GLIC_OK;
}

// view slot s of parity `parity` in region r of the exchange block
template <typename T = float>
T* slot(const glic_mapper* m, SlotRegion r, int parity, int s) {
    return reinterpret_cast<T*>(m->xblock + m->x.slot_off[r] + ((size_t)parity * m->S + s) * m->x.slot_bytes[r]);
}

// The slot regions follow the flags words, each [2][S] slots rounded up to 256 bytes: colour gradients [cap][3] floats, flag
// bytes [cap], dL/dE [12] floats, dL/d(rho, omega) [8] floats (2 unused), and with densification on the screen radii [cap]
// int32 (empty otherwise).
XLayout xblock_layout(int S, uint32_t cap, bool dens) {
    XLayout x;
    x.n_geo = (size_t)(dens ? 13 : 11) * cap + 4;
    size_t sl[6];
    glic_p2p_slice(0, 1, x.n_geo, 0, sl);
    const size_t bytes[N_REGIONS] = {(size_t)cap * 3 * sizeof(float), cap, 12 * sizeof(float), 8 * sizeof(float),
                                     dens ? (size_t)cap * sizeof(int) : 0};
    x.bytes = sl[5] + 256;
    for (int r = 0; r < N_REGIONS; ++r) {
        x.slot_off[r] = x.bytes;
        x.slot_bytes[r] = bytes[r];
        x.bytes += ((size_t)2 * S * bytes[r] + 255) & ~size_t(255);
    }
    return x;
}

// copies [local, local + bytes) of this rank's exchange block to the same offset in every peer's, on the push stream
int push_to_peers(glic_mapper* m, const void* local, size_t bytes) {
    const size_t off = static_cast<const char*>(local) - m->xblock;
    for (int q = 0; q < m->cfg.world; ++q) {
        if (q == m->cfg.rank) continue;
        GLIC_CUDA_TRY(cudaMemcpyAsync(static_cast<char*>(m->peers[q]) + off, local, bytes, cudaMemcpyDeviceToDevice, m->push_stream));
    }
    return GLIC_OK;
}

// grows everything whose size depends on the Gaussian capacity (capacity_buffers), all of it allocated before any old buffer is
// released
int set_capacity(glic_mapper* m, uint32_t cap) {
    cap = round_up(std::max<uint32_t>(cap, 256), 256);
    if (cap <= m->Pcap) return GLIC_OK;
    if (m->connected) { set_error("mapper: the arena capacity is fixed once the exchange blocks are connected (world > 1); create the mapper with a larger capacity"); return GLIC_ERR_WORKSPACE; }
    auto regrow = [&](Buf* fresh) -> int {
        const float* old[3] = {m->params, m->m1, m->m2};
        for (int a = 0; a < 3 && m->P; ++a)
            MAP_TRY(glic_arena_regrow(old[a], m->Pcap, static_cast<float*>(fresh[a].raw()), cap, (uint32_t)m->M, m->P, m->stream));
        return GLIC_OK;
    };
    MAP_TRY(grow(m, capacity_buffers(m, cap, m->dens_on), regrow));
    adopt_capacity(m, cap, xblock_layout(m->S, cap, m->dens_on));
    return GLIC_OK;
}

// room for the exposure and pose rows of n training keyframes: existing rows are kept, new rows are zero
int reserve_keyframe_rows(glic_mapper* m, size_t n) {
    if (n <= m->kf_cap) return GLIC_OK;
    const size_t cap = std::max<size_t>({n, 2 * m->kf_cap, 64}), old = m->kf_cap;
    std::vector<Grow> list;
    grow_rows(list, exposure_rows(m), cap, old, true);
    grow_rows(list, pose_rows(m), cap, old, true);
    MAP_TRY(grow(m, list));
    m->kf_cap = cap;
    return GLIC_OK;
}

// zero moments and step counts of keyframes [first, last), on the mapper's stream
int adam_reset(glic_mapper* m, const KeyframeAdam& a, size_t first, size_t last) {
    const size_t row = a.width * sizeof(float);
    GLIC_CUDA_TRY(cudaMemsetAsync(a.m + a.width * first, 0, (last - first) * row, m->stream));
    GLIC_CUDA_TRY(cudaMemsetAsync(a.v + a.width * first, 0, (last - first) * row, m->stream));
    GLIC_CUDA_TRY(cudaMemsetAsync(a.t + first, 0, (last - first) * sizeof(int), m->stream));
    return GLIC_OK;
}

// keyframes [first, last): E = [I | 0], zero moments and step counts (on the mapper's stream, which is then drained: the
// legacy-stream cudaMemcpy / cudaMemset would not be ordered before the iterations that read these rows)
int expo_reset(glic_mapper* m, size_t first, size_t last) {
    if (last <= first) return GLIC_OK;
    std::vector<float> id(12 * (last - first), 0.0f);
    for (size_t k = 0; k < last - first; ++k) id[12 * k] = id[12 * k + 5] = id[12 * k + 10] = 1.0f;
    GLIC_CUDA_TRY(cudaMemcpyAsync(m->expo_E + 12 * first, id.data(), id.size() * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    MAP_TRY(adam_reset(m, m->expo_adam, first, last));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

// writes keyframe k's float pose (host copy, master pose, device float pose, camera block); `reset` also zeroes its Adam
// state.  Drains the mapper's stream (see expo_reset).
int pose_write(glic_mapper* m, size_t k, const float* R_wc, const float* t_wc, bool reset) {
    Keyframe& kf = m->train[k];
    float R[9], t[3];
    std::memcpy(R, R_wc, sizeof(R)); std::memcpy(t, t_wc, sizeof(t));
    std::memcpy(kf.R_wc, R, sizeof(R)); std::memcpy(kf.t_wc, t, sizeof(t));
    double T12[12];
    config_camera_block(m, kf.R_wc, kf.t_wc, kf.cam, T12);
    float f12[12];
    std::memcpy(f12, kf.R_wc, 36); std::memcpy(f12 + 9, kf.t_wc, 12);
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    GLIC_CUDA_TRY(cudaMemcpyAsync(kf.cam_dev, kf.cam.view, 36 * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    GLIC_CUDA_TRY(cudaMemcpyAsync(m->pose_T + 12 * k, T12, sizeof(T12), cudaMemcpyHostToDevice, m->stream));
    GLIC_CUDA_TRY(cudaMemcpyAsync(m->pose_f + 12 * k, f12, sizeof(f12), cudaMemcpyHostToDevice, m->stream));
    if (reset) MAP_TRY(adam_reset(m, m->pose_adam, k, k + 1));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

// zero statistics for every row, on the mapper's stream (a no-op with densification off)
int dens_reset(glic_mapper* m) {
    if (!m->dens_on) return GLIC_OK;
    for (const Rows& r : densification_rows(m)) GLIC_CUDA_TRY(cudaMemsetAsync(r.buf.raw(), 0, (size_t)m->Pcap * r.bytes, m->stream));
    return GLIC_OK;
}

// pose_step_kernel on the first S slots of b, with the configuration's projection, on the mapper's stream
int launch_pose_kernel(glic_mapper* m, int S, PoseBatch b, const float* slot_grads, double* T, float* pose_f, float* adam_m, float* adam_v,
                       int* adam_t, float lr_rho, float lr_omega, const unsigned int* skip) {
    float fov2[2];
    proj_matrix(m->cfg.width, m->cfg.height, m->cfg.fx, m->cfg.fy, m->cfg.cx, m->cfg.cy, b.Pm, fov2);
    pose_step_kernel<<<1, MAX_SLOTS, 0, m->stream>>>(S, b, slot_grads, T, pose_f, adam_m, adam_v, adam_t, lr_rho, lr_omega, skip);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_pose_step(glic_mapper* m, const int* views, int parity) {
    PoseBatch b{};
    for (int sl = 0; sl < m->S; ++sl) { b.kf[sl] = views[sl]; b.cam[sl] = m->train[views[sl]].cam_dev; }
    StageTimer _t(GLIC_STAGE_ADAM, m->stream);
    const KeyframeAdam& a = m->pose_adam;
    return launch_pose_kernel(m, m->S, b, slot(m, POSE, parity, 0), m->pose_T, m->pose_f, a.m, a.v, a.t, m->pose_lr_rho, m->pose_lr_omega,
                              reinterpret_cast<const unsigned int*>(geo_ptr(m) + (size_t)11 * m->Pcap));
}

int set_bin_capacity(glic_mapper* m, int64_t pairs, bool exact = false) {
    if (!exact && pairs <= m->bin_cap) return GLIC_OK;
    const size_t binning_bytes = glic_binning_bytes(pairs), sample_bytes = glic_sample_bytes(pairs, m->cfg.width, m->cfg.height);
    const int64_t cap = glic_binning_capacity(binning_bytes, sample_bytes, m->cfg.width, m->cfg.height, 0);
    if (m->deterministic)     // the deterministic workspace follows the capacity, in the same growth
        MAP_TRY(grow(m, {{m->binning_ws, binning_bytes}, {m->sample_ws, sample_bytes},
                         {m->det_ws, glic_deterministic_bytes(cap, m->cfg.width, m->cfg.height)}}));
    else
        MAP_TRY(grow(m, {{m->binning_ws, binning_bytes}, {m->sample_ws, sample_bytes}}));
    m->bin_cap = cap;
    return GLIC_OK;
}

// room for `pairs` in the binning workspace alone, for glic_render (which has no sample workspace); the sample workspace is left
// as it is.  The training capacity is re-derived from both workspaces exactly as glic_forward derives it, so the backward keeps
// carving the binning workspace with the capacity the forward used.
int grow_render_binning(glic_mapper* m, int64_t pairs) {
    if (!m->deterministic) {
        MAP_TRY(reserve(m, m->binning_ws, glic_binning_bytes(pairs)));
        m->bin_cap = glic_binning_capacity(m->binning_ws.bytes(), m->sample_ws.bytes(), m->cfg.width, m->cfg.height, 0);
        return GLIC_OK;
    }
    // a larger training capacity needs a larger deterministic workspace: both grow together or neither does
    const size_t bb = std::max(glic_binning_bytes(pairs), m->binning_ws.bytes());
    const int64_t cap = glic_binning_capacity(bb, m->sample_ws.bytes(), m->cfg.width, m->cfg.height, 0);
    const size_t db = glic_deterministic_bytes(cap, m->cfg.width, m->cfg.height);
    std::vector<Grow> list;
    if (bb > m->binning_ws.bytes()) list.push_back(Grow{m->binning_ws, bb});
    if (db > m->det_ws.bytes()) list.push_back(Grow{m->det_ws, db});
    if (!list.empty()) MAP_TRY(grow(m, list));
    m->bin_cap = cap;
    return GLIC_OK;
}

// after draws skipped on the device for want of room for up to `pairs` pairs: that with a quarter to spare, and at least 1.5x as much
int regrow_after_skip(glic_mapper* m, int64_t pairs) {
    MAP_TRY(set_bin_capacity(m, std::max<int64_t>(pairs + pairs / 4, m->bin_cap * 3 / 2)));
    ++m->st.overflow_regrows;
    return GLIC_OK;
}

// lagged, non-blocking look at the pinned binning counters of finished iterations
int poll_ring(glic_mapper* m, bool wait) {
    for (int r = 0; r < RING; ++r) {
        if (!m->ring_used[r]) continue;
        cudaError_t q = wait ? cudaEventSynchronize(m->ring_ev[r]) : cudaEventQuery(m->ring_ev[r]);
        if (q == cudaErrorNotReady) { cudaGetLastError(); continue; }
        if (q != cudaSuccess) { set_error(std::string("mapper: ") + cudaGetErrorString(q)); return GLIC_ERR_CUDA; }
        m->ring_used[r] = false;
        const long long* c = m->counters_host + 4 * r;
        m->st.last_loss = m->loss_host[r];
        if (c[2]) MAP_TRY(regrow_after_skip(m, c[0]));     // this frame overflowed the binning workspace: it was skipped on the device
    }
    return GLIC_OK;
}

// the activated parameters; zero4[0..3] (optional) zeroed by the same kernel
int activate(glic_mapper* m, float* zero4) {
    const ArenaRows a = arena_rows(m->params, m->Pcap, m->M);
    return launch_activations_forward((int)m->P, a.opacity, a.log_scale, a.rot, m->act_opacity, m->act_scales, m->act_rots, zero4, m->stream);
}

int forward_view(glic_mapper* m, const glic_view& v, int no_color, long long* counters) {
    const ArenaRows a = arena_rows(m->params, m->Pcap, m->M);
    return glic_forward((int)m->P, m->D, m->M, a.xyz, m->act_scales, 1.0f, m->act_rots, m->act_opacity, a.dc, a.rest, &v, no_color, m->radii,
                        m->geom_ws, m->geom_ws.bytes(), m->image_ws, m->image_ws.bytes(), m->binning_ws, m->binning_ws.bytes(), m->sample_ws,
                        m->sample_ws.bytes(), m->color, m->final_T, (int64_t*)counters, m->stream);
}

// activations and a settled forward of v with the training workspaces
int forward_settled(glic_mapper* m, const glic_view& v, int no_color) {
    MAP_TRY(activate(m));
    return draw_settled(m, [&](long long* cnt) { return forward_view(m, v, no_color, cnt); },
                        [&](int64_t pairs) { return set_bin_capacity(m, pairs); });
}

// keyframe kf's float image [3,H,W] into dst on stream s: an add_frame keyframe's 8-bit image decoded from the frame store,
// any other keyframe's float image copied with `kind`
int load_gt(glic_mapper* m, const Keyframe& kf, float* dst, cudaMemcpyKind kind, cudaStream_t s) {
    const int W = m->cfg.width, H = m->cfg.height;
    if (kf.bgr) return glic_decode_bgr8(H, W, kf.bgr, dst, s);
    GLIC_CUDA_TRY(cudaMemcpyAsync(dst, kf.image, sizeof(float) * 3 * (size_t)W * H, kind, s));
    return GLIC_OK;
}

// the L1 + D-SSIM loss of an H x W image against gt, and its dL/dimg; with E (device, 3x4) the loss of the exposed image, and dL/dE;
// loss_zeroed: *loss is zero already
// mask (optional, `valid` used pixels): the masked loss
int photometric_loss(glic_mapper* m, int H, int W, const float* img, const float* gt, const float* E, float* loss, float* dL_dimg, float* dL_dE,
                     bool loss_zeroed, const MaskView* mask, uint32_t valid) {
    return photometric_loss_sum(H, W, m->cfg.lambda_dssim, img, gt, E, loss, dL_dimg, dL_dE, m->loss_scratch, m->loss_scratch.bytes(),
                                m->deterministic ? m->det_sums.raw() : nullptr, m->stream, loss_zeroed, mask, valid);
}

// the backward of the last forward_view of v from dL_dpix: colour gradients into col, after_render (optional) recorded, then cg's
int backward_view(glic_mapper* m, const glic_view& v, float* col, const CompactGrads& cg, cudaEvent_t after_render) {
    const ArenaRows a = arena_rows(m->params, m->Pcap, m->M);
    return glic::backward_compact((int)m->P, m->D, m->M, a.xyz, m->act_scales, m->act_rots, a.rest, &v, m->radii, m->bin_cap, m->geom_ws,
                                  m->binning_ws, m->image_ws, m->sample_ws, m->dL_dpix, m->g_mean2D, m->g_conic, m->g_opacity, col, cg,
                                  after_render, m->stream, m->deterministic ? m->det_ws.raw() : nullptr);
}

// one optimiser step over the view batch `views` (S keyframe indices, slot-major); this rank renders slots [rank*k, rank*k + k)
int iteration(glic_mapper* m, const int* views) {
    if (m->P == 0) return GLIC_OK;
    if (m->cfg.world > 1 && !m->connected) { set_error("mapper: world > 1 needs glic_mapper_connect before the first iteration"); return GLIC_ERR_INVALID_ARGUMENT; }
    for (int sl = 0; sl < m->S; ++sl)
        if (views[sl] < 0 || views[sl] >= (int)m->train.size()) { set_error("mapper: view index out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(poll_ring(m, false));
    const int r = (int)(m->st.iterations % RING);
    if (m->ring_used[r]) { GLIC_CUDA_TRY(cudaEventSynchronize(m->ring_ev[r])); MAP_TRY(poll_ring(m, false)); }
    cudaStream_t s = m->stream;
    const int parity = (int)(m->st.iterations & 1);
    const int W = m->cfg.width, H = m->cfg.height;
    float* geo = geo_ptr(m);
    const ArenaRows a = arena_rows(m->params, m->Pcap, m->M), ga = arena_rows(geo, m->Pcap, 0);
    float* geo_tail = geo + (size_t)11 * m->Pcap;
    MAP_TRY(activate(m, geo_tail));
    for (int j = 0; j < m->k; ++j) {
        const int sl = m->cfg.rank * m->k + j;
        const Keyframe& kf = m->train[views[sl]];
        // keyframe image H2D (gaussian.cpp:678), or the 8-bit frame's decode, on the copy stream, overlapping the previous
        // view's backward / Adam; an image already in device memory is read where it is
        const int buf = kf.image_on_device ? -1 : (int)(m->view_counter++ & 1);
        if (buf >= 0) {
            GLIC_CUDA_TRY(cudaStreamWaitEvent(m->copy_stream, m->gt_free[buf], 0));
            MAP_TRY(load_gt(m, kf, m->gt_dev[buf], cudaMemcpyDefault, m->copy_stream));
            GLIC_CUDA_TRY(cudaEventRecord(m->gt_ready[buf], m->copy_stream));
        }
        MAP_TRY(forward_view(m, kf.view, 0, j == m->k - 1 ? m->counters_host + 4 * r : nullptr));
        uint8_t* fl = slot<uint8_t>(m, FLAGS, parity, sl);
        float* col = slot(m, COLOUR, parity, sl);
        int* rad = m->dens_on ? slot<int>(m, RADII, parity, sl) : nullptr;           // this view's radii for the screen-size statistic
        MAP_TRY(launch_view_flags((int)m->P, m->radii, GeomState::carve(m->geom_ws, (int)m->P), fl, s, rad, geo_tail,
                                  ViewZero{m->g_conic, m->g_mean2D, m->g_opacity, col, m->loss_dev + 1}));
        if (m->cfg.world > 1) {
            GLIC_CUDA_TRY(cudaEventRecord(m->ev_flags, s));
            GLIC_CUDA_TRY(cudaStreamWaitEvent(m->push_stream, m->ev_flags, 0));
            MAP_TRY(push_to_peers(m, fl, m->P));
            if (rad) MAP_TRY(push_to_peers(m, rad, sizeof(int) * (size_t)m->P));
        }
        if (buf >= 0) GLIC_CUDA_TRY(cudaStreamWaitEvent(s, m->gt_ready[buf], 0));
        // loss of this view (the pinned ring keeps the last local view's value for the statistics), under its keyframe's mask
        MaskView mv;
        MAP_TRY(photometric_loss(m, H, W, m->color, buf >= 0 ? m->gt_dev[buf] : kf.image, m->expo_on ? m->expo_E + 12 * (size_t)views[sl] : nullptr,
                                 m->loss_dev + 1, m->dL_dpix, slot(m, EXPOSURE, parity, sl), /*loss_zeroed=*/true, keyframe_mask(kf, W, mv),
                                 kf.mask_valid));
        if (buf >= 0) GLIC_CUDA_TRY(cudaEventRecord(m->gt_free[buf], s));
        CompactGrads cg;
        cg.g_rot = reinterpret_cast<float4*>(ga.rot); cg.g_xyz = ga.xyz; cg.g_scale = ga.log_scale; cg.g_opacity = ga.opacity;
        cg.opacity = m->act_opacity; cg.dL_dopacity = m->g_opacity; cg.rot_raw = reinterpret_cast<const float4*>(a.rot);
        cg.accumulate = j > 0;
        cg.grads_zeroed = 1;
        cg.pose_partials = m->pose_on ? (double*)m->pose_part : nullptr;        // this view's dL/d(rho, omega), fused into the backward
        cg.pose_grad = m->pose_on ? slot(m, POSE, parity, sl) : nullptr;
        cg.dens_norm = m->dens_on ? geo_tail + 4 : nullptr;                        // this view's statistics, summed over the rank's views
        cg.dens_count = m->dens_on ? geo_tail + 4 + m->Pcap : nullptr;
        MAP_TRY(backward_view(m, kf.view, col, cg, m->cfg.world > 1 ? (cudaEvent_t)m->ev_col : nullptr));
        if (m->cfg.world > 1 && m->pose_on) GLIC_CUDA_TRY(cudaEventRecord(m->ev_pose, s));   // after the pose finish kernel
        if (m->cfg.world > 1) {
            GLIC_CUDA_TRY(cudaStreamWaitEvent(m->push_stream, m->ev_col, 0));
            MAP_TRY(push_to_peers(m, col, sizeof(float) * 3 * (size_t)m->P));
            // this slot's dL/dE (the loss wrote it before the render backward ran)
            if (m->expo_on) MAP_TRY(push_to_peers(m, slot(m, EXPOSURE, parity, sl), sizeof(float) * 12));
            if (m->pose_on) {                      // this slot's dL/d(rho, omega): ev_col fired before the per-Gaussian backward
                GLIC_CUDA_TRY(cudaStreamWaitEvent(m->push_stream, m->ev_pose, 0));
                MAP_TRY(push_to_peers(m, slot(m, POSE, parity, sl), sizeof(float) * 6));
            }
        }
    }
    if (m->cfg.world > 1) {
        GLIC_CUDA_TRY(cudaEventRecord(m->ev_push, m->push_stream));
        GLIC_CUDA_TRY(cudaStreamWaitEvent(s, m->ev_push, 0));
        MAP_TRY(glic_p2p_allreduce_mean(m->cfg.rank, m->cfg.world, m->peers, m->x.n_geo, 0, s));
    }
    float lr6[6] = {m->cfg.rotation_lr, m->cfg.position_lr, m->cfg.scaling_lr, m->cfg.opacity_lr, m->cfg.feature_lr, m->cfg.feature_lr / 20.0f};
    // Reference quirk kept for parity (backward.cu:352 `if (shs)`): with no SH-rest tensor bound (degree 0, M = 0) the whole
    // colour backward is skipped, dL/ddc included, so dc never trains.
    const float color_scale = m->M ? 1.0f / (float)m->S : 0.0f;
    // the SH rebuild reads each slot's camera centre from its device camera block (pose refinement moves the blocks there)
    const float* campos[MAX_SLOTS];
    for (int sl = 0; sl < m->S; ++sl) campos[sl] = m->train[views[sl]].cam_dev + 32;
    if (m->run_optimizer)
    MAP_TRY(launch_adam_compact(m->P, m->Pcap, m->D, m->M, m->params, m->m1, m->m2, geo, m->Pcap, lr6, slot(m, COLOUR, parity, 0),
                                slot<uint8_t>(m, FLAGS, parity, 0), campos, m->S, 1.0f / (float)m->k, color_scale, 0.9f, 0.999f, 1e-15f,
                                reinterpret_cast<const unsigned int*>(geo_tail), m->vis_acc, s, m->dens_on ? geo_tail + 4 : nullptr,
                                m->dens_accum, m->dens_denom, (float)m->cfg.world, m->dens_on ? slot<int>(m, RADII, parity, 0) : nullptr,
                                m->dens_maxr));
    // every replica steps the batch's exposures from the same S slot gradients, in slot order
    if (m->run_optimizer && m->expo_on)
        MAP_TRY(launch_exposure_adam(m->S, views, slot(m, EXPOSURE, parity, 0), m->expo_E, m->expo_adam.m, m->expo_adam.v, m->expo_adam.t, m->expo_lr,
                                     reinterpret_cast<const unsigned int*>(geo_tail), s));
    // ... and their poses, after the Gaussians (whose SH rebuild above used the centres the batch was rendered from)
    if (m->run_optimizer && m->pose_on) MAP_TRY(launch_pose_step(m, views, parity));
    GLIC_CUDA_TRY(cudaMemcpyAsync(m->loss_host + r, m->loss_dev + 1, sizeof(float), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaEventRecord(m->ring_ev[r], s));
    m->ring_used[r] = true;
    ++m->st.iterations;
    return GLIC_OK;
}

// glic_mapper_pose_set's test of a float pose: finite entries, R_wc a rotation (R^T R = I to float precision and det R = +1)
int pose_check(const float* R_wc9, const float* t_wc3, const char* what) {
    for (int j = 0; j < 9; ++j) if (!std::isfinite(R_wc9[j])) { set_error(std::string(what) + ": non-finite entry"); return GLIC_ERR_INVALID_ARGUMENT; }
    for (int j = 0; j < 3; ++j) if (!std::isfinite(t_wc3[j])) { set_error(std::string(what) + ": non-finite entry"); return GLIC_ERR_INVALID_ARGUMENT; }
    double R[9], err = 0.0;
    for (int j = 0; j < 9; ++j) R[j] = R_wc9[j];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) err = std::max(err, std::fabs(R[a] * R[b] + R[3 + a] * R[3 + b] + R[6 + a] * R[6 + b] - (a == b ? 1.0 : 0.0)));
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (err > 1e-5 || det < 0.0) { set_error(std::string(what) + ": R_wc is not a rotation (orthonormal, det +1)"); return GLIC_ERR_INVALID_ARGUMENT; }
    return GLIC_OK;
}

// the checks of the per-keyframe getters and setters: a mapper and a buffer, the feature (pose or exposure) enabled, a training
// keyframe index in range
int keyframe_index_check(glic_mapper* m, bool pose, int index, const void* buf, const char* what) {
    if (!m || !buf) { set_error(std::string(what) + ": null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!(pose ? m->pose_on : m->expo_on)) {
        set_error(std::string(what) + (pose ? ": pose refinement is not enabled (glic_mapper_enable_pose_refinement)"
                                            : ": exposure is not enabled (glic_mapper_enable_exposure)"));
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (index < 0 || index >= (int)m->train.size()) { set_error(std::string(what) + ": training keyframe index out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    return GLIC_OK;
}

// moments and step count of a training keyframe's pose or exposure
int keyframe_adam_state(glic_mapper* m, bool pose, int index, float* exp_avg, float* exp_avg_sq, int* step, const char* what) {
    MAP_TRY(keyframe_index_check(m, pose, index, step, what));
    if (!exp_avg || !exp_avg_sq) { set_error(std::string(what) + ": null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const KeyframeAdam& a = pose ? m->pose_adam : m->expo_adam;
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    GLIC_CUDA_TRY(cudaMemcpy(exp_avg, a.m + a.width * (size_t)index, a.width * sizeof(float), cudaMemcpyDeviceToHost));
    GLIC_CUDA_TRY(cudaMemcpy(exp_avg_sq, a.v + a.width * (size_t)index, a.width * sizeof(float), cudaMemcpyDeviceToHost));
    GLIC_CUDA_TRY(cudaMemcpy(step, a.t + index, sizeof(int), cudaMemcpyDeviceToHost));
    return GLIC_OK;
}

// renders keyframe `index` and scores it (evaluateVisualQuality, gaussian.cpp:754-760): PSNR / SSIM land in eval_out[0..1], and
// the clamped image (a training keyframe's E applied first; held-out views: identity) and the clamped ground truth stay in the
// evaluation scratch (eval_clamped).  masked: under the keyframe's mask (if it has one), the masked scores of eval_psnr_ssim and a
// clamped pair that is 0 at masked pixels.  Asynchronous after the settled forward.
int render_scored(glic_mapper* m, int is_train, int index, const char* what, bool masked) {
    const Keyframe* kf = nullptr;
    MAP_TRY(keyframe_at(m, is_train, index, what, kf));
    MAP_TRY(poll_ring(m, true));
    cudaStream_t s = m->stream;
    const int W = m->cfg.width, H = m->cfg.height;
    MAP_TRY(forward_settled(m, kf->view, 0));
    MAP_TRY(load_gt(m, *kf, m->gt_dev[0], cudaMemcpyHostToDevice, s));
    const float* E = (is_train && m->expo_on) ? m->expo_E + 12 * (size_t)index : nullptr;
    MaskView mv;
    return eval_psnr_ssim(3, H, W, m->color, m->gt_dev[0], E, m->eval_out, m->eval_scratch, m->eval_scratch.bytes(), s,
                          m->deterministic ? m->det_sums.raw() : nullptr, masked ? keyframe_mask(*kf, W, mv) : nullptr, kf->mask_valid);
}

// the whole clamped image eval_psnr_ssim last scored (eval_clamped) into rgb_host, on the mapper's stream
int scored_image_to_host(glic_mapper* m, float* rgb_host) {
    const int W = m->cfg.width, H = m->cfg.height;
    GLIC_CUDA_TRY(cudaMemcpyAsync(rgb_host, eval_clamped(m->eval_scratch, 3, H, W, 0), sizeof(float) * 3 * (size_t)W * H,
                                  cudaMemcpyDeviceToHost, m->stream));
    return GLIC_OK;
}

// LPIPS of the clamped pair eval_psnr_ssim last scored, W columns wide, into eval_out[2]
int scored_lpips(glic_mapper* m, int W) {
    const int H = m->cfg.height;
    return glic_lpips(H, W, eval_clamped(m->eval_scratch, 3, H, W, 0), eval_clamped(m->eval_scratch, 3, H, W, 1), m->lpips_w, m->eval_out + 2,
                      m->lpips_scratch, m->lpips_scratch.bytes(), m->stream);
}

// copies n floats of eval_out to the host and waits for them
int read_eval_out(glic_mapper* m, float* out, int n) {
    GLIC_CUDA_TRY(cudaMemcpyAsync(out, m->eval_out, sizeof(float) * n, cudaMemcpyDeviceToHost, m->stream));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

// a new map of P rows: the binning room for it, reserved before the map is replaced (a failure leaves it as it was), then zero
// arenas and (with densification on) zero statistics, on the mapper's stream
int start_map(glic_mapper* m, uint32_t P) {
    MAP_TRY(set_bin_capacity(m, (int64_t)16 * P));
    const size_t nfl = arena_floats(m, m->Pcap);
    GLIC_CUDA_TRY(cudaMemsetAsync(m->params, 0, nfl * 4, m->stream));
    GLIC_CUDA_TRY(cudaMemsetAsync(m->m1, 0, nfl * 4, m->stream));
    GLIC_CUDA_TRY(cudaMemsetAsync(m->m2, 0, nfl * 4, m->stream));
    return dens_reset(m);
}

// once the mapper's stream has drained: the map is the P rows written since start_map, the first n_sky of them the skybox
int install_map(glic_mapper* m, uint32_t P, uint32_t n_sky) {
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    m->P = P;
    m->n_sky = n_sky;
    m->st.num_gaussians = P;
    m->initialized = true;
    return GLIC_OK;
}

// initialize() (gaussian.cpp:212-304) from device arrays: the sky rows, then the n LiDAR rows.  The caller has validated the
// arguments, sized the arena for sky_points + n rows and hands sky_ws of glic_skybox_init_bytes(sky_points) bytes.
// anchor: the LiDAR rows' (the sky rows take -1)
int initialize_lidar_core(glic_mapper* m, int n, const float* d_pts, const double* d_col, const float* d_dep, double focal, int sky_points,
                          int sky_radius, void* sky_ws, int32_t anchor) {
    const uint32_t S = (uint32_t)sky_points, P = S + (uint32_t)n;
    MAP_TRY(start_map(m, P));
    cudaStream_t s = m->stream;
    const ArenaRows a = arena_rows(m->params, m->Pcap, m->M);
    MAP_TRY(glic_skybox_init(sky_points, sky_radius, m->cfg.seed, sky_ws, glic_skybox_init_bytes(sky_points), a.xyz, a.dc, a.log_scale, a.rot,
                             a.opacity, nullptr, s));
    MAP_TRY(glic_lidar_init(n, d_pts, d_col, d_dep, (double)m->cfg.scaling_scale, focal, a.xyz + 3 * (size_t)S, a.dc + 3 * (size_t)S,
                            a.log_scale + 3 * (size_t)S, a.rot + 4 * (size_t)S, a.opacity + S, s));
    MAP_TRY(launch_fill_anchors(m->anchor, 0, S, P, anchor, s));
    return install_map(m, P, S);
}

// extend()'s workspace after its inputs: outputs (keep_idx, xyz, f_dc, log_scale, rot, opacity) | glic_extend's own
size_t extend_core_carve(void* ws, int n, int W, int H, int** keep, float** out5, void** ext_ws) {
    Carver c(ws);
    int* k = c.take<int>(n);
    const size_t width[5] = {3, 3, 3, 4, 1};
    for (int q = 0; q < 5; ++q) {
        float* p = c.take<float>(width[q] * n);
        if (out5) out5[q] = p;
    }
    void* e = c.take<char>(glic_extend_bytes(n, W, H));
    if (keep) *keep = k;
    if (ext_ws) *ext_ws = e;
    return c.total();
}

// extend() (gaussian.cpp:499-638) on training keyframe kf, the newest, from device arrays of n > 0 points; the new rows take
// anchor `anchor`.  The caller has drained the ring, sized the arena for P + n rows, recorded m->t0 before staging its inputs and
// hands ws of extend_core_carve(nullptr, n, W, H, ...) bytes.
int extend_core(glic_mapper* m, const Keyframe& kf, int n, const float* d_pts, const float* d_col, const float* d_dep, void* ws,
                int32_t anchor) {
    cudaStream_t s = m->stream;
    const int W = m->cfg.width, H = m->cfg.height;
    int* d_keep = nullptr;
    float* o[5];
    void* d_ws = nullptr;
    extend_core_carve(ws, n, W, H, &d_keep, o, &d_ws);
    float *d_xyz = o[0], *d_dc = o[1], *d_ls = o[2], *d_rot = o[3], *d_op = o[4];
    // alpha-only render of the newest keyframe (gaussian.cpp:506-507); the binning capacity is settled synchronously here
    if (m->P) {
        MAP_TRY(forward_settled(m, kf.view, 1));
    } else {
        std::vector<float> ones((size_t)W * H, 1.0f);                                       // empty model: alpha = 1 - T = 0
        GLIC_CUDA_TRY(cudaMemcpyAsync(m->final_T, ones.data(), sizeof(float) * ones.size(), cudaMemcpyHostToDevice, s));
        GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    }
    MaskView mv;
    if (const MaskView* mk = keyframe_mask(kf, W, mv)) {           // no point is seeded at a masked pixel
        mask_final_T_kernel<<<(unsigned)std::min<size_t>(((size_t)W * H + 255) / 256, (size_t)NUM_SMS * 8), 256, 0, s>>>(H, W, *mk, m->final_T);
        GLIC_LAUNCH_CHECK();
    }
    float view[16];
    std::memcpy(view, kf.cam.view, sizeof(view));
    if (m->pose_on) {                               // the keyframe's current (possibly refined) pose: its device camera block
        GLIC_CUDA_TRY(cudaStreamSynchronize(s));
        GLIC_CUDA_TRY(cudaMemcpy(view, kf.cam_dev, sizeof(view), cudaMemcpyDeviceToHost));
    }
    float Rcw[9], tcw[3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rcw[3 * i + j] = view[4 * j + i];   // view is column-major Rt
    for (int i = 0; i < 3; ++i) tcw[i] = view[12 + i];
    int count = 0;
    MAP_TRY(glic_extend(n, d_pts, d_col, d_dep, Rcw, tcw, m->cfg.fx, m->cfg.fy, m->cfg.cx, m->cfg.cy, W, H, m->final_T, m->cfg.scaling_scale,
                        d_ws, glic_extend_bytes(n, W, H), d_keep, d_xyz, d_dc, d_ls, d_rot, d_op, &count, s));
    MAP_TRY(glic_arena_append(m->params, m->m1, m->m2, m->P, m->Pcap, (uint32_t)m->M, (uint32_t)count, d_xyz, d_dc, d_ls, d_rot, d_op, s));
    MAP_TRY(launch_fill_anchors(m->anchor, m->P, m->P, m->P + (uint32_t)count, anchor, s));
    GLIC_CUDA_TRY(cudaEventRecord(m->t1, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    cudaEventElapsedTime(&m->st.ms_extend, m->t0, m->t1);
    m->P += (uint32_t)count;
    m->st.num_gaussians = m->P;
    m->st.last_inserted = (uint32_t)count;
    return GLIC_OK;
}

// room in the extend() staging for n points and the arena for P + n rows (ring drained first)
int extend_prepare(glic_mapper* m, int n, size_t input_bytes) {
    MAP_TRY(poll_ring(m, true));
    MAP_TRY(set_capacity(m, std::max<uint32_t>(m->P + (uint32_t)n, m->Pcap < m->P + (uint32_t)n ? 2 * m->Pcap : 0)));
    return reserve(m, m->extend_ws, input_bytes + extend_core_carve(nullptr, n, m->cfg.width, m->cfg.height, nullptr, nullptr, nullptr));
}

// a keyframe at pose (R_wc, t_wc) with its device camera block, not yet in a list; a keyframe of add_frame has image = nullptr
// and its 8-bit image in the frame store
int make_keyframe(glic_mapper* m, const float* R_wc, const float* t_wc, const float* image, const uint8_t* bgr, Keyframe& kf) {
    std::memcpy(kf.R_wc, R_wc, sizeof(kf.R_wc)); std::memcpy(kf.t_wc, t_wc, sizeof(kf.t_wc));
    kf.image = image;
    kf.bgr = bgr;
    if (image) {
        cudaPointerAttributes pa = {};
        int dev = 0;
        GLIC_CUDA_TRY(cudaPointerGetAttributes(&pa, image));
        GLIC_CUDA_TRY(cudaGetDevice(&dev));
        kf.image_on_device = pa.type == cudaMemoryTypeDevice && pa.device == dev;
    }
    config_camera_block(m, kf.R_wc, kf.t_wc, kf.cam);
    MAP_TRY(kf.cam_dev.allocate(36 * sizeof(float)));
    // view | proj | campos are contiguous; ordered before every use of the block, all of which are on the mapper's stream or after
    // a synchronisation of it
    GLIC_CUDA_TRY(cudaMemcpyAsync(kf.cam_dev, kf.cam.view, 36 * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    kf.view = make_view(kf.cam, kf.cam_dev, m->cfg.width, m->cfg.height);
    return GLIC_OK;
}

// appends kf to its list.  A training keyframe's rows (reserve_keyframe_rows, by the caller) start at E = [I | 0] and at its
// given pose, with zero Adam state, for the features that are enabled.
int push_keyframe(glic_mapper* m, Keyframe&& kf, int is_train) {
    (is_train ? m->train : m->test).push_back(std::move(kf));
    if (!is_train) return GLIC_OK;
    const size_t k = m->train.size() - 1;
    if (m->expo_on) MAP_TRY(expo_reset(m, k, k + 1));
    if (m->pose_on) MAP_TRY(pose_write(m, k, m->train[k].R_wc, m->train[k].t_wc, true));
    return GLIC_OK;
}

// Reserves what the hand-off of n scan points will need: the arena for the first map's sky and LiDAR rows, or for n more rows
// of extend(), and the staging of their colours and workspace
int handoff_reserve(glic_mapper* m, int n) {
    Carver c(nullptr);
    if (m->initialized) {
        if (n == 0) return GLIC_OK;
        c.take<float>((size_t)3 * n);
        return extend_prepare(m, n, c.total());
    }
    MAP_TRY(set_capacity(m, (uint32_t)m->frame_sky_points + (uint32_t)n));
    c.take<double>((size_t)3 * n); c.take<char>(glic_skybox_init_bytes(m->frame_sky_points));
    return reserve(m, m->extend_ws, c.total());
}

// mapping.cpp:158-174 at training keyframe kf: the n accumulated scan points initialize the map, or extend it.  kf joins the
// training list right after, so its rows are anchored to index train.size().  Everything is
// reserved (handoff_reserve); the one allocation left is a binning regrow, which comes before the map changes.
int scan_handoff(glic_mapper* m, const Keyframe& kf, int n) {
    cudaStream_t s = m->stream;
    const unsigned blocks = (unsigned)((3 * (size_t)n + 255) / 256);
    Carver c(m->extend_ws);
    if (!m->initialized) {
        const int S = m->frame_sky_points;
        double* d_col = c.take<double>((size_t)3 * n);
        void* sky_ws = c.take<char>(glic_skybox_init_bytes(S));
        scan_colour_kernel<double><<<blocks, 256, 0, s>>>(3 * n, m->scan_rgb, d_col);
        GLIC_LAUNCH_CHECK();
        const double focal = ((double)m->cfg.fx + (double)m->cfg.fy) / 2;
        return initialize_lidar_core(m, n, m->scan_xyz, d_col, m->scan_depth, focal, S, m->frame_sky_radius, sky_ws, (int32_t)m->train.size());
    }
    if (n == 0) { m->st.last_inserted = 0; return GLIC_OK; }
    float* d_col = c.take<float>((size_t)3 * n);
    void* ws = c.take<char>(0);
    GLIC_CUDA_TRY(cudaEventRecord(m->t0, s));
    scan_colour_kernel<float><<<blocks, 256, 0, s>>>(3 * n, m->scan_rgb, d_col);
    GLIC_LAUNCH_CHECK();
    return extend_core(m, kf, n, m->scan_xyz, d_col, m->scan_depth, ws, (int32_t)m->train.size());
}

// the mask checks of set_keyframe_mask and add_frame_masked, before anything is reserved: a mask with no used pixel is refused
int mask_check(const glic_mapper* m, const uint8_t* valid, const char* what) {
    const size_t n = (size_t)m->cfg.width * m->cfg.height;
    if (std::find_if(valid, valid + n, [](uint8_t v) { return v != 0; }) == valid + n) {
        set_error(std::string(what) + ": the mask has no valid pixel"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    return GLIC_OK;
}

// packs the host byte mask `valid` (checked by mask_check) into kf's mask: a new bit buffer and a staging buffer are allocated
// first, so a failure leaves kf's mask as it was; the bits and the count are made on the device, and the mapper's stream is drained
// before the new buffer replaces the old one (which iterations in flight may still read)
int pack_keyframe_mask(glic_mapper* m, Keyframe& kf, const uint8_t* valid) {
    const int W = m->cfg.width, H = m->cfg.height;
    const size_t n = (size_t)W * H, words = (size_t)H * mask_words_per_row(W);
    Dev<uint32_t> bits;
    Dev<uint8_t> staging;                                  // the bytes | the count
    MAP_TRY(bits.allocate(words * sizeof(uint32_t)));
    MAP_TRY(staging.allocate(((n + 255) & ~size_t(255)) + 256));
    uint32_t* d_count = reinterpret_cast<uint32_t*>(staging + ((n + 255) & ~size_t(255)));
    cudaStream_t s = m->stream;
    uint32_t count = 0;
    GLIC_CUDA_TRY(cudaMemcpyAsync(staging, valid, n, cudaMemcpyHostToDevice, s));
    MAP_TRY(launch_pack_mask(H, W, staging, bits, d_count, s));
    GLIC_CUDA_TRY(cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    uint32_t left = 0;
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W / 2; ++x) left += valid[(size_t)y * W + x] != 0;
    kf.mask = std::move(bits);
    kf.mask_valid = count;
    kf.mask_valid_left = left;
    return GLIC_OK;
}

}  // namespace mapper_impl

extern "C" {

int glic_camera_block(int width, int height, float fx, float fy, float cx, float cy, const float* R_wc, const float* t_wc, float* out41) {
    if (!R_wc || !t_wc || !out41 || width <= 0 || height <= 0) { set_error("camera_block: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    CamBlock c;
    camera_block(width, height, fx, fy, cx, cy, R_wc, t_wc, c);
    std::memcpy(out41, c.view, 64); std::memcpy(out41 + 16, c.proj, 64); std::memcpy(out41 + 32, c.campos, 12);
    out41[35] = c.tanfovx; out41[36] = c.tanfovy; std::memcpy(out41 + 37, c.lim, 16);
    return GLIC_OK;
}

int glic_mapper_create(const glic_mapper_config* cfg, glic_mapper** out) {
    if (!cfg || !out) { set_error("mapper_create: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (cfg->width <= 0 || cfg->height <= 0 || cfg->sh_degree < 0 || cfg->sh_degree > 3 || cfg->world < 1 || cfg->world > 8 || cfg->rank < 0 ||
        cfg->rank >= cfg->world || cfg->views_per_rank < 1 || cfg->world * cfg->views_per_rank > MAX_SLOTS) {
        set_error("mapper_create: bad configuration"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    std::unique_ptr<glic_mapper> m(new glic_mapper());     // on a failure its members release whatever was made
    m->cfg = *cfg;
    if (m->cfg.max_iters <= 0) m->cfg.max_iters = 100;
    m->D = cfg->sh_degree; m->M = (m->D + 1) * (m->D + 1) - 1;
    m->k = cfg->views_per_rank; m->S = cfg->world * cfg->views_per_rank;
    m->rng.seed(cfg->seed);
    if (cudaGetDevice(&m->dev) != cudaSuccess) { set_error("mapper_create: no CUDA device"); return GLIC_ERR_NO_DEVICE; }
    cudaStream_t sh = nullptr;
    cudaEvent_t eh = nullptr;
    for (Stream* s : {&m->stream, &m->copy_stream, &m->push_stream}) { GLIC_CUDA_TRY(cudaStreamCreateWithFlags(&sh, cudaStreamNonBlocking)); *s = Stream(sh); }
    std::vector<Event*> evs = {&m->gt_free[0], &m->gt_free[1], &m->gt_ready[0], &m->gt_ready[1], &m->ev_flags, &m->ev_col, &m->ev_push, &m->ev_pose};
    for (Event& e : m->ring_ev) evs.push_back(&e);
    for (Event* e : evs) { GLIC_CUDA_TRY(cudaEventCreateWithFlags(&eh, cudaEventDisableTiming)); *e = Event(eh); }
    for (Event* e : {&m->t0, &m->t1}) { GLIC_CUDA_TRY(cudaEventCreate(&eh)); *e = Event(eh); }
    const int W = cfg->width, H = cfg->height;
    const size_t HW = (size_t)W * H;
    MAP_TRY(set_capacity(m.get(), cfg->capacity ? cfg->capacity : 1u << 20));
    MAP_TRY(grow(m.get(), {{m->image_ws, glic_image_bytes(W, H), 0, true}, {m->loss_scratch, glic_loss_scratch_bytes(3, H, W)},
                           {m->eval_scratch, glic_eval_scratch_bytes(3, H, W)}, {m->color, HW * 12, 0, true}, {m->final_T, HW * 4, 0, true},
                           {m->dL_dpix, HW * 12, 0, true}, {m->gt_dev[0], HW * 12, 0, true}, {m->gt_dev[1], HW * 12, 0, true},
                           {m->loss_dev, 64, 0, true}, {m->eval_out, 64, 0, true}, {m->vis_acc, 64, 0, true}}));
    MAP_TRY(m->counters_host.allocate(sizeof(long long) * 4 * RING, true));
    MAP_TRY(m->loss_host.allocate(sizeof(float) * RING, true));
    std::memset(m->counters_host, 0, sizeof(long long) * 4 * RING);
    std::memset(m->loss_host, 0, sizeof(float) * RING);
    MAP_TRY(set_bin_capacity(m.get(), std::max<int64_t>((int64_t)16 * m->Pcap, (int64_t)1 << 22)));
    cudaEventRecord(m->gt_free[0], m->stream); cudaEventRecord(m->gt_free[1], m->stream);
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));       // the copy and push streams and the peers see the zeroed buffers
    *out = m.release();
    return GLIC_OK;
}

int glic_mapper_destroy(glic_mapper* m) {
    if (!m) return GLIC_OK;
    cudaDeviceSynchronize();                               // nothing in flight may still use what the members release
    delete m;
    cudaGetLastError();
    return GLIC_OK;
}

int glic_mapper_initialize(glic_mapper* m, uint32_t P, const float* xyz, const float* f_dc, const float* f_rest, const float* opacity_logit,
                           const float* log_scale, const float* rot) {
    if (!m || (P && (!xyz || !f_dc || !opacity_logit || !log_scale || !rot))) { set_error("mapper_initialize: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(set_capacity(m, P));
    MAP_TRY(start_map(m, P));
    const auto g = arena_rows(m->params, m->Pcap, m->M).groups();
    const auto kk = group_widths(m->M);
    const float* src[6] = {rot, xyz, log_scale, opacity_logit, f_dc, f_rest};
    for (int q = 0; q < 6; ++q)
        if (P && kk[q] && src[q]) GLIC_CUDA_TRY(cudaMemcpyAsync(g[q], src[q], sizeof(float) * kk[q] * P, cudaMemcpyHostToDevice, m->stream));
    MAP_TRY(launch_fill_anchors(m->anchor, 0, P, P, -1, m->stream));
    return install_map(m, P, 0);
}

int glic_mapper_initialize_lidar(glic_mapper* m, int n, const float* points, const double* colors, const float* depth_rsp, double focal,
                                 int sky_points, int sky_radius) {
    if (!m || !points || !colors || !depth_rsp) { set_error("mapper_initialize_lidar: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    // n > 0 is the reference's assert(num > 0) (gaussian.cpp:216)
    if (n < 1 || sky_points < 0 || (sky_points > 0 && sky_radius <= 0) || (int64_t)n + sky_points > INT32_MAX / 4) {
        set_error("mapper_initialize_lidar: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    MAP_TRY(set_capacity(m, (uint32_t)sky_points + (uint32_t)n));
    cudaStream_t s = m->stream;
    // staging: points | colors | depth | the sky's dist2 and knn workspace
    Carver c(nullptr);
    c.take<float>((size_t)3 * n); c.take<double>((size_t)3 * n); c.take<float>(n); c.take<char>(glic_skybox_init_bytes(sky_points));
    MAP_TRY(reserve(m, m->extend_ws, c.total()));
    c = Carver(m->extend_ws);
    float* d_pts = c.take<float>((size_t)3 * n); double* d_col = c.take<double>((size_t)3 * n); float* d_dep = c.take<float>(n);
    void* d_sky = c.take<char>(glic_skybox_init_bytes(sky_points));
    GLIC_CUDA_TRY(cudaMemcpyAsync(d_pts, points, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, s));
    GLIC_CUDA_TRY(cudaMemcpyAsync(d_col, colors, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, s));
    GLIC_CUDA_TRY(cudaMemcpyAsync(d_dep, depth_rsp, sizeof(float) * n, cudaMemcpyHostToDevice, s));
    return initialize_lidar_core(m, n, d_pts, d_col, d_dep, focal, sky_points, sky_radius, d_sky, (int32_t)m->train.size() - 1);
}

int glic_mapper_sky_rows(glic_mapper* m, uint32_t* out) {
    if (!m || !out) { set_error("mapper_sky_rows: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    *out = m->n_sky;
    return GLIC_OK;
}

int glic_mapper_add_keyframe(glic_mapper* m, const glic_keyframe* kfi, int is_train) {
    if (!m || !kfi || !kfi->image) { set_error("mapper_add_keyframe: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    Keyframe kf;
    MAP_TRY(make_keyframe(m, kfi->R_wc, kfi->t_wc, kfi->image, nullptr, kf));
    if (is_train && (m->expo_on || m->pose_on)) MAP_TRY(reserve_keyframe_rows(m, m->train.size() + 1));
    return push_keyframe(m, std::move(kf), is_train);
}

int glic_mapper_extend(glic_mapper* m, int n, const float* points, const float* colors, const float* depth_rsp) {
    if (!m || n < 0 || (n && (!points || !colors || !depth_rsp))) { set_error("mapper_extend: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (n == 0) { m->st.last_inserted = 0; return GLIC_OK; }
    if (m->train.empty()) { set_error("mapper_extend: no training keyframe yet"); return GLIC_ERR_INVALID_ARGUMENT; }
    // staging: points | colors | depth | extend_core's workspace
    Carver c(nullptr);
    c.take<float>((size_t)3 * n); c.take<float>((size_t)3 * n); c.take<float>(n);
    MAP_TRY(extend_prepare(m, n, c.total()));
    c = Carver(m->extend_ws);
    float* d_pts = c.take<float>((size_t)3 * n); float* d_col = c.take<float>((size_t)3 * n); float* d_dep = c.take<float>(n);
    void* ws = c.take<char>(0);
    cudaStream_t s = m->stream;
    GLIC_CUDA_TRY(cudaEventRecord(m->t0, s));
    GLIC_CUDA_TRY(cudaMemcpyAsync(d_pts, points, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, s));
    GLIC_CUDA_TRY(cudaMemcpyAsync(d_col, colors, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, s));
    GLIC_CUDA_TRY(cudaMemcpyAsync(d_dep, depth_rsp, sizeof(float) * n, cudaMemcpyHostToDevice, s));
    return extend_core(m, m->train.back(), n, d_pts, d_col, d_dep, ws, (int32_t)m->train.size() - 1);
}

int glic_mapper_enable_frames(glic_mapper* m, int select_every_k_frame, int sky_points, int sky_radius) {
    if (!m) { set_error("mapper_enable_frames: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (m->frames_on) { set_error("mapper_enable_frames: frames are already enabled"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (select_every_k_frame < 1 || sky_points < 0 || (sky_points > 0 && sky_radius <= 0) || sky_points > INT32_MAX / 4) {
        set_error("mapper_enable_frames: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    m->frames_on = true;
    m->frame_k = select_every_k_frame;
    m->frame_sky_points = sky_points;
    m->frame_sky_radius = sky_radius;
    m->frame_stride = ckpt::frame_stride(m->cfg.width, m->cfg.height);
    return GLIC_OK;
}

int glic_mapper_add_frame(glic_mapper* m, const glic_frame* f, int* is_keyframe) { return glic_mapper_add_frame_masked(m, f, nullptr, is_keyframe); }

int glic_mapper_add_frame_masked(glic_mapper* m, const glic_frame* f, const uint8_t* valid, int* is_keyframe) {
    if (!m || !f || !f->bgr || (f->n_points > 0 && (!f->xyz || !f->rgb))) { set_error("mapper_add_frame: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (valid) MAP_TRY(mask_check(m, valid, "mapper_add_frame_masked"));
    if (!m->frames_on) { set_error("mapper_add_frame: frames are not enabled (glic_mapper_enable_frames)"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (f->row_bytes < 3 * (size_t)m->cfg.width || f->n_points < 0) { set_error("mapper_add_frame: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t pending = (size_t)m->fst.pending_points + (size_t)f->n_points;
    if (pending + (size_t)m->frame_sky_points > INT32_MAX / 4) { set_error("mapper_add_frame: too many scan points before a keyframe"); return GLIC_ERR_INVALID_ARGUMENT; }
    const int train = (m->fst.frames + 1) % (uint32_t)m->frame_k == 0;
    // the reference's assert(num > 0) of initialize() (gaussian.cpp:216)
    if (train && !m->initialized && pending == 0) { set_error("mapper_add_frame: the first keyframe has no scan points"); return GLIC_ERR_INVALID_ARGUMENT; }
    double R[9];
    quat_rotation(f->q_wc, R);
    float R_wc[9], t_wc[3];
    for (int e = 0; e < 9; ++e) R_wc[e] = (float)R[e];
    for (int i = 0; i < 3; ++i) t_wc[i] = (float)f->t_wc[i];
    // Reserve everything first: the frame store's next slot (a new chunk when the last one is full), room in the scan buffers
    // (grown by doubling), the keyframe and, at a training keyframe, its rows and what the hand-off needs
    const size_t idx = m->fst.frames, have = m->fst.pending_points, n = (size_t)f->n_points;
    if (idx / FRAME_CHUNK >= m->frame_chunks.size()) {
        Dev<uint8_t> chunk;
        MAP_TRY(chunk.allocate(FRAME_CHUNK * m->frame_stride));
        m->frame_chunks.push_back(std::move(chunk));
    }
    if (pending > m->scan_cap) {
        const size_t cap = std::max<size_t>({pending, 2 * m->scan_cap, 4096});
        std::vector<Grow> list;
        grow_rows(list, scan_rows(m), cap, have, false);
        MAP_TRY(grow(m, list));
        m->scan_cap = cap;
    }
    uint8_t* dst = m->frame_chunks[idx / FRAME_CHUNK] + (idx % FRAME_CHUNK) * m->frame_stride;
    Keyframe kf;
    MAP_TRY(make_keyframe(m, R_wc, t_wc, nullptr, dst, kf));
    if (valid) MAP_TRY(pack_keyframe_mask(m, kf, valid));  // before the hand-off: its extend() leaves the masked pixels out
    if (train) {
        if (m->expo_on || m->pose_on) MAP_TRY(reserve_keyframe_rows(m, m->train.size() + 1));
        MAP_TRY(handoff_reserve(m, (int)pending));
    }
    // the image without its row padding, and the points after the pending ones with their depths in the frame's camera
    cudaStream_t s = m->stream;
    const size_t W3 = 3 * (size_t)m->cfg.width;
    GLIC_CUDA_TRY(cudaMemcpy2DAsync(dst, W3, f->bgr, f->row_bytes, W3, (size_t)m->cfg.height, cudaMemcpyHostToDevice, s));
    if (n) {
        GLIC_CUDA_TRY(cudaMemcpyAsync(m->scan_xyz + 3 * have, f->xyz, n * 3 * sizeof(float), cudaMemcpyHostToDevice, s));
        GLIC_CUDA_TRY(cudaMemcpyAsync(m->scan_rgb + 3 * have, f->rgb, n * 3, cudaMemcpyHostToDevice, s));
        // R_cw = R^T; t_cw = -R_cw t_wc in the product's order (gaussian.cpp:66-67)
        const double* t = f->t_wc;
        const double tcw2 = -(((R[2] * t[0]) + (R[5] * t[1])) + (R[8] * t[2]));
        scan_depth_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((int)n, m->scan_xyz + 3 * have, R[2], R[5], R[8], tcw2, m->scan_depth + have);
        GLIC_LAUNCH_CHECK();
    }
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));              // the caller's buffers are free again
    // The hand-off runs before the keyframe joins its list, so that its one possible allocation failure (a binning regrow, before
    // the map changes) leaves nothing to undo.  It draws the keyframe as it will be pushed: the pose it starts at.
    if (train) MAP_TRY(scan_handoff(m, kf, (int)pending));
    MAP_TRY(push_keyframe(m, std::move(kf), train));
    m->fst.pending_points = train ? 0 : (uint32_t)pending;
    ++m->fst.frames;
    ++(train ? m->fst.train : m->fst.test);
    m->fst.image_bytes = m->frame_chunks.size() * FRAME_CHUNK * m->frame_stride;
    if (is_keyframe) *is_keyframe = train;
    return GLIC_OK;
}

int glic_mapper_keyframe_image(glic_mapper* m, int is_train, int index, float* rgb_host) {
    if (!m || !rgb_host) { set_error("mapper_keyframe_image: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const Keyframe* kf = nullptr;
    MAP_TRY(keyframe_at(m, is_train, index, "mapper_keyframe_image", kf));
    const size_t bytes = sizeof(float) * 3 * (size_t)m->cfg.width * m->cfg.height;
    if (!kf->bgr) {
        GLIC_CUDA_TRY(cudaMemcpy(rgb_host, kf->image, bytes, cudaMemcpyDefault));
        return GLIC_OK;
    }
    MAP_TRY(poll_ring(m, true));                          // the iterations' use of gt_dev[0] has finished (see render_scored)
    MAP_TRY(load_gt(m, *kf, m->gt_dev[0], cudaMemcpyHostToDevice, m->stream));
    GLIC_CUDA_TRY(cudaMemcpyAsync(rgb_host, m->gt_dev[0], bytes, cudaMemcpyDeviceToHost, m->stream));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

int glic_mapper_set_keyframe_mask(glic_mapper* m, int is_train, int index, const uint8_t* valid) {
    if (!m) { set_error("mapper_set_keyframe_mask: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    const Keyframe* kf = nullptr;
    MAP_TRY(keyframe_at(m, is_train, index, "mapper_set_keyframe_mask", kf));
    Keyframe& k = (is_train ? m->train : m->test)[index];
    if (!valid) {                                          // clear: the iterations in flight may still read the old bits
        GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
        k.mask = Dev<uint32_t>();
        k.mask_valid = k.mask_valid_left = 0;
        return GLIC_OK;
    }
    MAP_TRY(mask_check(m, valid, "mapper_set_keyframe_mask"));
    return pack_keyframe_mask(m, k, valid);
}

int glic_mapper_keyframe_mask(glic_mapper* m, int is_train, int index, uint8_t* out, uint32_t* valid_count) {
    if (!m || !valid_count) { set_error("mapper_keyframe_mask: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const Keyframe* kf = nullptr;
    MAP_TRY(keyframe_at(m, is_train, index, "mapper_keyframe_mask", kf));
    *valid_count = kf->mask_valid;
    if (!out || !kf->mask_valid) return GLIC_OK;
    const int W = m->cfg.width, H = m->cfg.height, wpr = mask_words_per_row(W);
    std::vector<uint32_t> bits((size_t)H * wpr);
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    GLIC_CUDA_TRY(cudaMemcpy(bits.data(), kf->mask, bits.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) out[(size_t)y * W + x] = (bits[(size_t)y * wpr + (x >> 5)] >> (x & 31)) & 1u;
    return GLIC_OK;
}

int glic_mapper_frames_get(glic_mapper* m, glic_frame_stats* out) {
    if (!m || !out) { set_error("mapper_frames_get: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    *out = m->fst;
    return GLIC_OK;
}

int glic_mapper_sample_views(glic_mapper* m, int* views, int* count) {
    if (!m || !views || !count) { set_error("mapper_sample_views: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    // gaussian.cpp:645-662: every training camera when there are <= max_iters of them, otherwise a uniform subset of
    // max_iters without replacement; then a shuffle.  (Fisher-Yates on an explicit seed: identical on every rank.)
    const int n = (int)m->train.size();
    std::vector<int> all(n);
    for (int i = 0; i < n; ++i) all[i] = i;
    const int take = std::min(n, m->cfg.max_iters);
    for (int i = 0; i < take; ++i) {
        const int j = i + (int)(m->rng() % (uint64_t)(n - i));
        std::swap(all[i], all[j]);
    }
    for (int i = 0; i < take; ++i) views[i] = all[i];
    *count = take;
    return GLIC_OK;
}

int glic_mapper_optimize(glic_mapper* m, const int* views_host, int n_views) {
    if (!m) { set_error("mapper_optimize: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    std::vector<int> list;
    if (views_host && n_views > 0) list.assign(views_host, views_host + n_views);
    else {
        list.resize((size_t)std::max(1, m->cfg.max_iters));
        int cnt = 0;
        MAP_TRY(glic_mapper_sample_views(m, list.data(), &cnt));
        list.resize((size_t)cnt);
    }
    // every index is checked before the first batch is enqueued: a bad index in a later batch (say slot 31 of the second
    // batch of 32) would otherwise return the error with the earlier batches already stepped
    for (int v : list)
        if (v < 0 || v >= (int)m->train.size()) { set_error("mapper_optimize: view index out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (list.empty() || m->P == 0) return GLIC_OK;
    GLIC_CUDA_TRY(cudaMemsetAsync(m->vis_acc, 0, sizeof(unsigned int), m->stream));
    GLIC_CUDA_TRY(cudaEventRecord(m->t0, m->stream));
    const size_t iters = (list.size() + m->S - 1) / m->S;
    std::vector<int> batch((size_t)m->S);
    for (size_t it = 0; it < iters; ++it) {
        for (int sl = 0; sl < m->S; ++sl) batch[sl] = list[(it * m->S + sl) % list.size()];     // the last batch wraps around
        MAP_TRY(iteration(m, batch.data()));
        if (m->sched_on && m->run_optimizer) MAP_TRY(scheduled_density_step(m));
    }
    GLIC_CUDA_TRY(cudaEventRecord(m->t1, m->stream));
    unsigned int vis = 0;
    GLIC_CUDA_TRY(cudaMemcpyAsync(&vis, m->vis_acc, sizeof(vis), cudaMemcpyDeviceToHost, m->stream));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    MAP_TRY(poll_ring(m, true));
    cudaEventElapsedTime(&m->st.ms_optimize, m->t0, m->t1);
    m->st.mean_visible = (double)vis / (double)iters;
    if (m->connected) MAP_TRY(glic_p2p_check(m->xblock, m->x.n_geo, 0, m->stream));
    return GLIC_OK;
}

int glic_mapper_evaluate(glic_mapper* m, int is_train, int index, float* psnr, float* ssim) {
    if (!m || !psnr || !ssim) { set_error("mapper_evaluate: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(render_scored(m, is_train, index, "mapper_evaluate", true));
    float out2[2] = {0.f, 0.f};
    MAP_TRY(read_eval_out(m, out2, 2));
    *psnr = out2[0]; *ssim = out2[1];
    return GLIC_OK;
}

int glic_mapper_load_lpips(glic_mapper* m, const char* path) {
    if (!m || !path) { set_error("mapper_load_lpips: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    std::vector<float> w(glic_lpips_weight_floats());
    MAP_TRY(glic_lpips_read_weights(path, w.data()));
    MAP_TRY(reserve(m, m->lpips_w, w.size() * sizeof(float)));
    GLIC_CUDA_TRY(cudaMemcpyAsync(m->lpips_w, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

int glic_mapper_evaluate_lpips(glic_mapper* m, int is_train, int index, float* psnr, float* ssim, float* lpips) {
    if (!m || !psnr || !ssim || !lpips) { set_error("mapper_evaluate_lpips: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!m->lpips_w) { set_error("mapper_evaluate_lpips: no LPIPS weights loaded (glic_mapper_load_lpips)"); return GLIC_ERR_INVALID_ARGUMENT; }
    const int W = m->cfg.width, H = m->cfg.height;
    const size_t need = glic_lpips_scratch_bytes(H, W);
    if (!need) { set_error("mapper_evaluate_lpips: LPIPS needs a frame of at least 31x31"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(reserve(m, m->lpips_scratch, need));
    MAP_TRY(render_scored(m, is_train, index, "mapper_evaluate_lpips", true));
    MAP_TRY(scored_lpips(m, W));
    float out3[3] = {0.f, 0.f, 0.f};
    MAP_TRY(read_eval_out(m, out3, 3));
    *psnr = out3[0]; *ssim = out3[1]; *lpips = out3[2];
    return GLIC_OK;
}

int glic_mapper_render(glic_mapper* m, int is_train, int index, float* rgb_host) {
    if (!m || !rgb_host) { set_error("mapper_render: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(render_scored(m, is_train, index, "mapper_render", false));
    MAP_TRY(scored_image_to_host(m, rgb_host));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

int glic_mapper_download(glic_mapper* m, float* xyz, float* f_dc, float* f_rest, float* opacity_logit, float* log_scale, float* rot,
                         float* exp_avg_packed, float* exp_avg_sq_packed) {
    if (!m) { set_error("mapper_download: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    const auto g = arena_rows(m->params, m->Pcap, m->M).groups();
    const auto kk = group_widths(m->M);
    float* dst[6] = {rot, xyz, log_scale, opacity_logit, f_dc, f_rest};
    for (int q = 0; q < 6; ++q)
        if (dst[q] && kk[q] && m->P) GLIC_CUDA_TRY(cudaMemcpy(dst[q], g[q], sizeof(float) * kk[q] * m->P, cudaMemcpyDeviceToHost));
    float* mom[2] = {exp_avg_packed, exp_avg_sq_packed};
    float* srcm[2] = {m->m1, m->m2};
    for (int a = 0; a < 2; ++a) {
        if (!mom[a] || !m->P) continue;
        const auto gm = arena_rows(srcm[a], m->Pcap, m->M).groups();
        size_t off = 0;                                     // packed (capacity = P) layout: glic_packed_offsets(P, M)
        for (int q = 0; q < 6; ++q) {
            if (kk[q]) GLIC_CUDA_TRY(cudaMemcpy(mom[a] + off, gm[q], sizeof(float) * kk[q] * m->P, cudaMemcpyDeviceToHost));
            off += kk[q] * m->P;
        }
    }
    return GLIC_OK;
}

}  // extern "C"

namespace mapper_impl {

// ---- pose corrections (glic_mapper_correct_poses) ----------------------------------------------------------------------------
// After the checks: the records, one allocation (a failure changes nothing), the row pass, the keyframes.
int correct_poses(glic_mapper* m, int n, const glic_pose_correction* c, uint32_t* moved) {
    cudaStream_t s = m->stream;
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    MAP_TRY(poll_ring(m, true));
    const size_t nt = m->train.size();
    std::vector<glic_rigid_correction> table(nt);
    for (glic_rigid_correction& r : table) r.q[0] = CORRECTION_NONE;
    std::vector<int> corrected;                          // the listed training keyframes, in list order
    for (int i = 0; i < n; ++i) {
        if (!c[i].is_train) continue;
        const Keyframe& kf = m->train[c[i].index];
        MAP_TRY(glic_pose_correction_record(kf.R_wc, kf.t_wc, c[i].R_wc, c[i].t_wc, m->D, &table[c[i].index]));
        corrected.push_back(c[i].index);
    }
    // device: the table indexed by keyframe | the moved-row count
    Carver cv(nullptr);
    cv.take<glic_rigid_correction>(nt); cv.take<uint32_t>(1);
    Buf buf;
    MAP_TRY(buf.allocate(cv.total()));
    cv = Carver(buf.raw());
    glic_rigid_correction* d_table = cv.take<glic_rigid_correction>(nt);
    uint32_t* d_moved = cv.take<uint32_t>(1);
    if (nt) GLIC_CUDA_TRY(cudaMemcpyAsync(d_table, table.data(), nt * sizeof(glic_rigid_correction), cudaMemcpyHostToDevice, s));
    GLIC_CUDA_TRY(cudaMemsetAsync(d_moved, 0, sizeof(uint32_t), s));
    if (!corrected.empty()) MAP_TRY(launch_correct_rows(m->D, m->P, m->Pcap, m->params, m->anchor, d_table, (int)nt, d_moved, s));
    if (m->pose_on) {                                    // the refined masters move with their keyframes, MAX_SLOTS per launch
        for (size_t first = 0; first < corrected.size(); first += MAX_SLOTS) {
            PoseBatch b{};
            const int S = (int)std::min<size_t>(MAX_SLOTS, corrected.size() - first);
            for (int sl = 0; sl < S; ++sl) { b.kf[sl] = corrected[first + sl]; b.cam[sl] = m->train[b.kf[sl]].cam_dev; }
            float fov2[2];
            proj_matrix(m->cfg.width, m->cfg.height, m->cfg.fx, m->cfg.fy, m->cfg.cx, m->cfg.cy, b.Pm, fov2);
            pose_correct_kernel<<<1, MAX_SLOTS, 0, s>>>(S, b, d_table, m->pose_T, m->pose_f);
            GLIC_LAUNCH_CHECK();
        }
    }
    // the given poses; the camera blocks of keyframes without a refined master are rebuilt from them as make_keyframe builds them
    for (int i = 0; i < n; ++i) {
        Keyframe& kf = (c[i].is_train ? m->train : m->test)[c[i].index];
        std::memcpy(kf.R_wc, c[i].R_wc, sizeof(kf.R_wc)); std::memcpy(kf.t_wc, c[i].t_wc, sizeof(kf.t_wc));
        config_camera_block(m, kf.R_wc, kf.t_wc, kf.cam);
        if (!(c[i].is_train && m->pose_on)) GLIC_CUDA_TRY(cudaMemcpyAsync(kf.cam_dev, kf.cam.view, 36 * sizeof(float), cudaMemcpyHostToDevice, s));
    }
    uint32_t count = 0;
    GLIC_CUDA_TRY(cudaMemcpyAsync(&count, d_moved, sizeof(count), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    if (moved) *moved = count;
    return GLIC_OK;
}

}  // namespace mapper_impl

extern "C" {

int glic_mapper_save_map(glic_mapper* m, const char* path) {
    if (!m || !path) { set_error("mapper_save_map: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t P = m->P, M = (size_t)m->M, S = m->n_sky;
    std::vector<float> xyz(3 * P), dc(3 * P), rest(3 * M * P), op(P), ls(3 * P), rot(4 * P);
    MAP_TRY(glic_mapper_download(m, xyz.data(), dc.data(), M ? rest.data() : nullptr, op.data(), ls.data(), rot.data(), nullptr, nullptr));
    // rows [S, P): saveMap slices the sky off every tensor (gaussian.cpp:310-316).  It hands tinyply the unsliced row count
    // for f_dc and f_rest, but tinyply keeps the count of the element's first property (xyz, sliced), so the reference's file
    // is the consistently sliced one.
    return glic_ply_write(path, (uint32_t)(P - S), (uint32_t)M, xyz.data() + 3 * S, dc.data() + 3 * S, rest.data() + 3 * M * S, op.data() + S,
                          ls.data() + 3 * S, rot.data() + 4 * S);
}

int glic_mapper_stats_get(glic_mapper* m, glic_mapper_stats* out) {
    if (!m || !out) { set_error("mapper_stats: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    *out = m->st;
    return GLIC_OK;
}

int glic_mapper_set_option(glic_mapper* m, int option, int value) {
    if (!m) { set_error("mapper_set_option: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    switch (option) {
        case GLIC_MAPPER_OPT_OPTIMIZER: m->run_optimizer = value != 0; return GLIC_OK;
        case GLIC_MAPPER_OPT_BINNING_PAIRS:            // start from a chosen (possibly too small) binning capacity: exercises the overflow path
            if (value < 1) { set_error("mapper_set_option: binning capacity must be positive"); return GLIC_ERR_INVALID_ARGUMENT; }
            MAP_TRY(poll_ring(m, true));
            return set_bin_capacity(m, value, /*exact=*/true);
        case GLIC_MAPPER_OPT_DETERMINISTIC: {
            MAP_TRY(poll_ring(m, true));
            GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
            if (value) {                                 // both workspaces first, in one growth: a failure changes nothing
                const int W = m->cfg.width, H = m->cfg.height;
                const size_t db = glic_deterministic_bytes(m->bin_cap, W, H), sb = fixed_order_sums_bytes(H, W);
                std::vector<Grow> list;
                if (db > m->det_ws.bytes()) list.push_back(Grow{m->det_ws, db});
                if (sb > m->det_sums.bytes()) list.push_back(Grow{m->det_sums, sb});
                if (!list.empty()) MAP_TRY(grow(m, list));
            }
            m->deterministic = value != 0;
            return GLIC_OK;
        }
        default: set_error("mapper_set_option: unknown option"); return GLIC_ERR_INVALID_ARGUMENT;
    }
}

int glic_mapper_enable_exposure(glic_mapper* m, float exposure_lr) {
    if (!m) { set_error("mapper_enable_exposure: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!(exposure_lr >= 0.0f) || !std::isfinite(exposure_lr)) { set_error("mapper_enable_exposure: exposure_lr must be finite and >= 0"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!m->expo_on) {
        MAP_TRY(reserve(m, m->loss_scratch, glic_loss_exposure_scratch_bytes(m->cfg.height, m->cfg.width)));
        MAP_TRY(reserve_keyframe_rows(m, m->train.size()));
        MAP_TRY(expo_reset(m, 0, m->train.size()));
        m->expo_on = true;
    }
    m->expo_lr = exposure_lr;
    return GLIC_OK;
}

int glic_mapper_exposure_get(glic_mapper* m, int index, float* out12) {
    MAP_TRY(keyframe_index_check(m, false, index, out12, "mapper_exposure_get"));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    GLIC_CUDA_TRY(cudaMemcpy(out12, m->expo_E + 12 * (size_t)index, 12 * sizeof(float), cudaMemcpyDeviceToHost));
    return GLIC_OK;
}

int glic_mapper_exposure_set(glic_mapper* m, int index, const float* in12) {
    MAP_TRY(keyframe_index_check(m, false, index, in12, "mapper_exposure_set"));
    for (int j = 0; j < 12; ++j)
        if (!std::isfinite(in12[j])) { set_error("mapper_exposure_set: non-finite entry"); return GLIC_ERR_INVALID_ARGUMENT; }
    GLIC_CUDA_TRY(cudaMemcpyAsync(m->expo_E + 12 * (size_t)index, in12, 12 * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

int glic_mapper_exposure_adam_state(glic_mapper* m, int index, float* exp_avg12, float* exp_avg_sq12, int* step) {
    return keyframe_adam_state(m, false, index, exp_avg12, exp_avg_sq12, step, "mapper_exposure_adam_state");
}

int glic_mapper_enable_pose_refinement(glic_mapper* m, float lr_translation, float lr_rotation) {
    if (!m) { set_error("mapper_enable_pose_refinement: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!(lr_translation >= 0.0f) || !std::isfinite(lr_translation) || !(lr_rotation >= 0.0f) || !std::isfinite(lr_rotation)) {
        set_error("mapper_enable_pose_refinement: the learning rates must be finite and >= 0"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!m->pose_on) {                               // every training keyframe starts at its given pose with zero state
        MAP_TRY(reserve_keyframe_rows(m, m->train.size()));
        for (size_t k = 0; k < m->train.size(); ++k) MAP_TRY(pose_write(m, k, m->train[k].R_wc, m->train[k].t_wc, true));
        m->pose_on = true;
    }
    m->pose_lr_rho = lr_translation;
    m->pose_lr_omega = lr_rotation;
    return GLIC_OK;
}

int glic_mapper_pose_get(glic_mapper* m, int index, float* R_wc9, float* t_wc3, float* cam41) {
    MAP_TRY(keyframe_index_check(m, true, index, R_wc9, "mapper_pose_get"));
    if (!t_wc3) { set_error("mapper_pose_get: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    float f12[12];
    GLIC_CUDA_TRY(cudaMemcpy(f12, m->pose_f + 12 * (size_t)index, sizeof(f12), cudaMemcpyDeviceToHost));
    std::memcpy(R_wc9, f12, 36); std::memcpy(t_wc3, f12 + 9, 12);
    if (cam41) {
        const Keyframe& kf = m->train[index];
        GLIC_CUDA_TRY(cudaMemcpy(cam41, kf.cam_dev, 35 * sizeof(float), cudaMemcpyDeviceToHost));   // view | proj | campos[3]
        cam41[35] = kf.cam.tanfovx; cam41[36] = kf.cam.tanfovy; std::memcpy(cam41 + 37, kf.cam.lim, 16);
    }
    return GLIC_OK;
}

int glic_mapper_pose_set(glic_mapper* m, int index, const float* R_wc9, const float* t_wc3) {
    MAP_TRY(keyframe_index_check(m, true, index, R_wc9, "mapper_pose_set"));
    if (!t_wc3) { set_error("mapper_pose_set: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(pose_check(R_wc9, t_wc3, "mapper_pose_set"));
    return pose_write(m, (size_t)index, R_wc9, t_wc3, false);
}

int glic_mapper_pose_adam_state(glic_mapper* m, int index, float* exp_avg6, float* exp_avg_sq6, int* step) {
    return keyframe_adam_state(m, true, index, exp_avg6, exp_avg_sq6, step, "mapper_pose_adam_state");
}

int glic_mapper_anchors(glic_mapper* m, int32_t* out) {
    if (!m || !out) { set_error("mapper_anchors: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    if (m->P) GLIC_CUDA_TRY(cudaMemcpy(out, m->anchor, (size_t)m->P * 4, cudaMemcpyDeviceToHost));
    return GLIC_OK;
}

int glic_mapper_set_anchors(glic_mapper* m, const int32_t* in) {
    if (!m || (!in && m->P)) { set_error("mapper_set_anchors: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const int32_t n = (int32_t)m->train.size();
    for (uint32_t i = 0; i < m->P; ++i)
        if (in[i] < -1 || in[i] >= n) { set_error("mapper_set_anchors: an anchor is neither -1 nor a training keyframe index"); return GLIC_ERR_INVALID_ARGUMENT; }
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    if (m->P) GLIC_CUDA_TRY(cudaMemcpy(m->anchor, in, (size_t)m->P * 4, cudaMemcpyHostToDevice));
    return GLIC_OK;
}

int glic_mapper_correct_poses(glic_mapper* m, int n, const glic_pose_correction* c, uint32_t* moved) {
    if (!m || n < 0 || (n > 0 && !c)) { set_error("mapper_correct_poses: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    std::vector<char> seen_train(m->train.size(), 0), seen_test(m->test.size(), 0);
    for (int i = 0; i < n; ++i) {
        const Keyframe* kf = nullptr;
        MAP_TRY(keyframe_at(m, c[i].is_train, c[i].index, "mapper_correct_poses", kf));
        MAP_TRY(pose_check(c[i].R_wc, c[i].t_wc, "mapper_correct_poses"));
        char& seen = (c[i].is_train ? seen_train : seen_test)[c[i].index];
        if (seen) { set_error("mapper_correct_poses: a keyframe is listed twice"); return GLIC_ERR_INVALID_ARGUMENT; }
        seen = 1;
    }
    if (moved) *moved = 0;
    if (n == 0) return GLIC_OK;
    return correct_poses(m, n, c, moved);
}

int glic_mapper_synchronize(glic_mapper* m) {
    if (!m) return GLIC_OK;
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return poll_ring(m, true);
}

int glic_mapper_export(glic_mapper* m, unsigned char* handle64) {
    if (!m || !handle64) { set_error("mapper_export: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    cudaIpcMemHandle_t h;
    GLIC_CUDA_TRY(cudaIpcGetMemHandle(&h, m->xblock));
    std::memcpy(handle64, &h, 64);
    m->exported = true;
    return GLIC_OK;
}

int glic_mapper_connect(glic_mapper* m, const unsigned char* handles) {
    if (!m || !handles) { set_error("mapper_connect: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    for (int q = 0; q < m->cfg.world; ++q) {
        if (q == m->cfg.rank) { m->peers[q] = m->xblock; continue; }
        cudaIpcMemHandle_t h;
        std::memcpy(&h, handles + 64 * (size_t)q, 64);
        void* p = nullptr;
        GLIC_CUDA_TRY(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        m->peers[q] = p;
        m->opened.emplace_back(p);
    }
    m->connected = true;
    return GLIC_OK;
}

int glic_debug_fail_allocation(int n) {
    if (n < 0) { set_error("debug_fail_allocation: n must be >= 0"); return GLIC_ERR_INVALID_ARGUMENT; }
    fail_countdown = n;
    return GLIC_OK;
}

int64_t glic_debug_mapper_allocations(void) { return live_allocations; }

}  // extern "C"

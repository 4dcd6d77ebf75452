// model_step.cu -- the optimiser side of a mapping iteration on the packed model (SURVEY 8f rank 1).
//
// The reference keeps six parameter tensors, derives the rasterizer inputs with three elementwise torch ops
// (GaussianModel::getOpacity / getScaling / getRotation, gaussian.cpp:147-175: sigmoid, exp, normalize), lets autograd
// run their three backward ops, clones every gradient and launches adamUpdateCUDA six times (optim_utils.h:102-137).
// Here the model lives in ONE planar buffer in the layout of the packed gradient buffer
//     rotation[4P] | xyz[3P] | log-scale[3P] | opacity logit[P] | dc[3P] | sh-rest[3MP]
// so that: the activations are one kernel (8 floats in, 8 out per Gaussian), their chain rule is applied IN PLACE on
// the gradient buffer the backward just wrote, and the visibility-masked Adam of all six groups is a single launch
// that consumes that buffer (and, multi-GPU, exactly the bytes the exchange step just reduced).
#include "common.cuh"
#include "adam_math.cuh"
#include "sh_math.cuh"
#include "warp_rows.cuh"
#include <algorithm>

namespace glic {
namespace {

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// torch::sigmoid / torch::exp / torch::nn::functional::normalize (p = 2, eps = 1e-12) of the raw parameters; zero4 (optional) is
// zeroed on the way: the mapper's step starts here, and a memset would end its chain of dependent launches
__global__ void __launch_bounds__(256)
activations_forward_kernel(int P, const float* __restrict__ opacity_logit, const float* __restrict__ log_scale,
                           const float4* __restrict__ rot_raw, float* __restrict__ opacity, float* __restrict__ scale,
                           float4* __restrict__ rot, float* __restrict__ zero4) {
    pdl_enter();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (zero4 && i < 4) zero4[i] = 0.0f;
    if (i >= P) return;
    opacity[i] = opacity_activation(opacity_logit[i]);
#pragma unroll
    for (int c = 0; c < 3; ++c) scale[3 * (size_t)i + c] = scale_activation(log_scale[3 * (size_t)i + c]);
    rot[i] = rotation_activation(rot_raw[i]);
}

// dL/d(activated) -> dL/d(raw), in place: sigmoid' = s(1-s); exp' = exp; normalize: (g - q (q.g)) / |r| (|r| > eps)
__global__ void __launch_bounds__(256)
activations_backward_kernel(int P, const float* __restrict__ opacity, const float* __restrict__ scale,
                            const float4* __restrict__ rot_raw, float* __restrict__ dL_dopacity, float* __restrict__ dL_dscale,
                            float4* __restrict__ dL_drot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float s = opacity[i];
    dL_dopacity[i] = dL_dopacity[i] * (s * (1.0f - s));
#pragma unroll
    for (int c = 0; c < 3; ++c) dL_dscale[3 * (size_t)i + c] *= scale[3 * (size_t)i + c];
    const float4 r = rot_raw[i];
    const float4 g = dL_drot[i];
    const float nn = sqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
    if (nn > 1e-12f) {
        const float inv = 1.0f / nn;
        const float4 q = make_float4(r.x * inv, r.y * inv, r.z * inv, r.w * inv);
        const float qg = q.x * g.x + q.y * g.y + q.z * g.z + q.w * g.w;
        dL_drot[i] = make_float4((g.x - q.x * qg) * inv, (g.y - q.y * qg) * inv, (g.z - q.z * qg) * inv, (g.w - q.w * qg) * inv);
    } else {
        const float inv = 1.0f / 1e-12f;                    // clamped branch of normalize: plain scaling
        dL_drot[i] = make_float4(g.x * inv, g.y * inv, g.z * inv, g.w * inv);
    }
}

struct PackedLayout {
    size_t end[6];       // exclusive end offset (in floats) of each group inside the planar buffer
    size_t begin[6];
    uint32_t k[6];       // floats per Gaussian
    float lr[6];
};

// same arithmetic, element by element, as adam_kernel (adamUpdateCUDA, adam.cu:9-38): only the launch count changes
__global__ void __launch_bounds__(256)
adam_packed_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ exp_avg,
                   float* __restrict__ exp_avg_sq, const uint8_t* __restrict__ visible, PackedLayout L, float b1, float b2,
                   float eps, size_t total) {
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < total; j += (size_t)gridDim.x * blockDim.x) {
        int grp = 0;
#pragma unroll
        for (int q = 0; q < 5; ++q) grp += j >= L.end[q];
        const size_t gaussian = (j - L.begin[grp]) / L.k[grp];
        if (!visible[gaussian]) continue;
        float p = param[j], m = exp_avg[j], v = exp_avg_sq[j];
        adam_element(p, m, v, grad[j], L.lr[grp], b1, b2, eps);
        param[j] = p;
        exp_avg[j] = m;
        exp_avg_sq[j] = v;
    }
}


// ---- the mapper's Adam: compact gradients in, all six groups out (include/glic_b200.h "Native mapping host") -----------
// One warp owns 32 consecutive Gaussians.  Phase 1 (lane = Gaussian): the union of the per-view visibility bytes decides
// whether the Gaussian steps at all; the dc and sh-rest gradients -- never materialised by the backward -- are rebuilt as
// sum_views b_k(dir_view) * g_view (b_k: sh_math.cuh, dir from the PRE-update xyz) into a shared-memory slab.  Phase 2
// (warp-cooperative): all six groups of the warp's visible rows stream through once with coalesced accesses, the geometric
// gradients (already summed over the rank's views and mean-reduced over the ranks) read from the arena-shaped gradient block,
// dc / sh-rest from the slab.
// Densification (g_dens set): lane = Gaussian, every row visible in some slot adds dens_scale times the batch's statistics
// (norm sum, view count; dens_scale = world undoes the exchange's mean) to its running sums, and raises its screen-radius
// statistic to the largest radius of the slots that see it (vs.radii: each slot's radii, next to its flags).  A set skip flag
// leaves them.
struct ArenaLayout {
    size_t off[6];       // float offset of each group in the arena: rotation, xyz, log-scale, opacity, dc, sh-rest
    float lr[6];
};

struct ViewSlots {
    const float* g_color;    // [n_slots][stride][3] dL/dcolour per view as the render backward left it (before the clamp mask)
    const uint8_t* visible;  // [n_slots][stride] per-view flags: 0x80 = radii > 0, bits 0..2 = colour channel clamped (forward.cu:70-75)
    const float* campos[32]; // [n_slots] camera centre of each slot's view, in its device camera block (n_slots <= 32)
    const int* radii;        // [n_slots][stride] per-view screen radii (densification only)
    size_t stride;           // Gaussians per slot (the arena capacity)
    int n_slots;
};

constexpr int ADAM_WARPS = 4;

__global__ void __launch_bounds__(ADAM_WARPS * 32)
adam_compact_kernel(uint32_t P, int D, int M, float* __restrict__ params, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                    const float* __restrict__ g_geo /* arena-shaped: rotation | xyz | log-scale | opacity */, ArenaLayout L,
                    ArenaLayout Lg, ViewSlots vs, float grad_scale, float color_scale, float b1, float b2, float eps,
                    const unsigned int* __restrict__ skip_flag, unsigned int* __restrict__ visible_count,
                    const float* __restrict__ g_dens, float* __restrict__ dens_accum, float* __restrict__ dens_denom, float dens_scale,
                    int* __restrict__ dens_maxr) {
    __shared__ float s_g[ADAM_WARPS][32 * (SH_ROW_MAX + 3)];      // rebuilt gradients of the warp's 32 Gaussians: dc[32][3] | sh-rest[32][K]
    __shared__ uint8_t s_row[ADAM_WARPS][32];                      // compacted list of the warp's visible rows
    if (skip_flag && *skip_flag) return;                          // binning overflow: the frame was empty, do not step (ADVICE r1)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t wfirst = (blockIdx.x * ADAM_WARPS + warp) * 32u;
    if (wfirst >= P) return;
    const uint32_t i = wfirst + lane;
    const int K = 3 * M;
    float* s_dc = s_g[warp];
    float* s_sh = s_g[warp] + 32 * 3;
    bool vis = false;
    if (i < P) {
        for (int v = 0; v < vs.n_slots; ++v) vis |= (vs.visible[(size_t)v * vs.stride + i] & 0x80u) != 0;
    }
    if (g_dens && vis) {
        dens_accum[i] = __fadd_rn(dens_accum[i], __fmul_rn(g_dens[i], dens_scale));
        dens_denom[i] = __fadd_rn(dens_denom[i], __fmul_rn(g_dens[vs.stride + i], dens_scale));
        int r = dens_maxr[i];
        for (int v = 0; v < vs.n_slots; ++v)
            if (vs.visible[(size_t)v * vs.stride + i] & 0x80u) r = max(r, vs.radii[(size_t)v * vs.stride + i]);
        dens_maxr[i] = r;
    }
    const unsigned any = __ballot_sync(0xffffffffu, vis);
    if (!any) return;
    const int nvis = __popc(any);
    if (visible_count && lane == 0) atomicAdd(visible_count, (unsigned)nvis);
    if (vis) s_row[warp][__popc(any & ((1u << lane) - 1u))] = (uint8_t)lane;
    // ---- phase 1 (lane = Gaussian): dL/d(dc, sh-rest) from the per-view colour gradients, into shared memory ----
    if (vis) {
        const float px = params[L.off[1] + 3 * (size_t)i], py = params[L.off[1] + 3 * (size_t)i + 1], pz = params[L.off[1] + 3 * (size_t)i + 2];
        float gdc[3] = {0.f, 0.f, 0.f};
        const int nb = D > 0 ? sh_rest_count(D) : 0;
        float acc[SH_ROW_MAX];
#pragma unroll
        for (int k = 0; k < SH_ROW_MAX; ++k) acc[k] = 0.f;
        for (int v = 0; v < vs.n_slots; ++v) {
            const unsigned fl = vs.visible[(size_t)v * vs.stride + i];
            if (!(fl & 0x80u)) continue;
            const float* gc = vs.g_color + ((size_t)v * vs.stride + i) * 3;
            const float g0 = (fl & 1u) ? 0.f : gc[0], g1 = (fl & 2u) ? 0.f : gc[1], g2 = (fl & 4u) ? 0.f : gc[2];
            gdc[0] += kSH0 * g0; gdc[1] += kSH0 * g1; gdc[2] += kSH0 * g2;
            if (nb > 0) {
                const float cx = vs.campos[v][0], cy = vs.campos[v][1], cz = vs.campos[v][2];
                const float ox = px - cx, oy = py - cy, oz = pz - cz;
                const float inv = 1.0f / sqrtf(ox * ox + oy * oy + oz * oz);
                float bs[15];
                sh_basis(D, ox * inv, oy * inv, oz * inv, bs);
#pragma unroll
                for (int k = 0; k < 15; ++k) {
                    if (k < nb) { acc[3 * k] += bs[k] * g0; acc[3 * k + 1] += bs[k] * g1; acc[3 * k + 2] += bs[k] * g2; }
                }
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) s_dc[3 * lane + c] = gdc[c] * color_scale;
#pragma unroll
        for (int k = 0; k < SH_ROW_MAX; ++k) if (k < K) s_sh[lane * K + k] = acc[k] * color_scale;
    }
    __syncwarp();
    // ---- phase 2 (warp-cooperative, coalesced): every group's rows of the warp's visible Gaussians stream through once.  The
    // 32 lanes walk the (visible row, column) pairs of a group 32 at a time; (row, column) advance incrementally (no division).
    // Element arithmetic = adam_element (adam_math.cuh), i.e. adamUpdateCUDA's.
    // Four 32-element steps are in flight per lane (12 independent loads issued before the first use; eight measured slower): the loop is latency-bound
    // otherwise (one dependent global round trip per 32 elements).
    auto run_group = [&](int grp, int kk, const float* grad_global, size_t goff, float gscale, const float* grad_smem) {
        if (kk == 0) return;
        constexpr int U = 4;
        int r = 0, c = lane;
        while (c >= kk) { c -= kk; ++r; }
        const int step_r = 32 / kk, step_c = 32 % kk;
        while (r < nvis) {
            size_t e[U];
            float g[U], p[U], m[U], vv[U];
            bool ok[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                ok[u] = r < nvis;
                const int row = ok[u] ? s_row[warp][r] : 0;
                e[u] = L.off[grp] + ((size_t)wfirst + row) * kk + c;
                g[u] = 0.f;
                if (ok[u]) {
                    g[u] = grad_global ? grad_global[goff + ((size_t)wfirst + row) * kk + c] * gscale : grad_smem[row * kk + c];
                    p[u] = params[e[u]]; m[u] = exp_avg[e[u]]; vv[u] = exp_avg_sq[e[u]];
                }
                r += step_r; c += step_c;
                if (c >= kk) { c -= kk; ++r; }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (ok[u]) {
                    adam_element(p[u], m[u], vv[u], g[u], L.lr[grp], b1, b2, eps);
                    params[e[u]] = p[u]; exp_avg[e[u]] = m[u]; exp_avg_sq[e[u]] = vv[u];
                }
            }
        }
    };
    run_group(0, 4, g_geo, Lg.off[0], grad_scale, nullptr);
    run_group(1, 3, g_geo, Lg.off[1], grad_scale, nullptr);
    run_group(2, 3, g_geo, Lg.off[2], grad_scale, nullptr);
    run_group(3, 1, g_geo, Lg.off[3], grad_scale, nullptr);
    run_group(4, 3, nullptr, 0, 0.f, s_dc);
    run_group(5, K, nullptr, 0, 0.f, s_sh);
}

// rows [P, P+n) of the arena <- the new Gaussians; their sh-rest rows and Adam moments are zero (densificationPostfix)
__global__ void __launch_bounds__(256)
arena_append_kernel(uint32_t P, uint32_t n, int K, ArenaLayout L, float* __restrict__ params, float* __restrict__ exp_avg,
                    float* __restrict__ exp_avg_sq, const float* __restrict__ xyz, const float* __restrict__ f_dc,
                    const float* __restrict__ log_scale, const float4* __restrict__ rot, const float* __restrict__ opacity_logit) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const size_t i = (size_t)P + t;
    reinterpret_cast<float4*>(params + L.off[0])[i] = rot[t];
    reinterpret_cast<float4*>(exp_avg + L.off[0])[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    reinterpret_cast<float4*>(exp_avg_sq + L.off[0])[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        params[L.off[1] + 3 * i + c] = xyz[3 * (size_t)t + c];
        params[L.off[2] + 3 * i + c] = log_scale[3 * (size_t)t + c];
        params[L.off[4] + 3 * i + c] = f_dc[3 * (size_t)t + c];
        exp_avg[L.off[1] + 3 * i + c] = 0.f; exp_avg_sq[L.off[1] + 3 * i + c] = 0.f;
        exp_avg[L.off[2] + 3 * i + c] = 0.f; exp_avg_sq[L.off[2] + 3 * i + c] = 0.f;
        exp_avg[L.off[4] + 3 * i + c] = 0.f; exp_avg_sq[L.off[4] + 3 * i + c] = 0.f;
    }
    params[L.off[3] + i] = opacity_logit[t];
    exp_avg[L.off[3] + i] = 0.f; exp_avg_sq[L.off[3] + i] = 0.f;
    for (int k = 0; k < K; ++k) {
        params[L.off[5] + i * K + k] = 0.f; exp_avg[L.off[5] + i * K + k] = 0.f; exp_avg_sq[L.off[5] + i * K + k] = 0.f;
    }
}

}  // namespace

int launch_activations_forward(int P, const float* opacity_logit, const float* log_scale, const float* rot_raw, float* opacity,
                               float* scale, float* rot, float* zero4, cudaStream_t stream) {
    if (P < 0) { set_error("activations_forward: bad P"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (P == 0) return GLIC_OK;
    if (!opacity_logit || !log_scale || !rot_raw || !opacity || !scale || !rot) { set_error("activations_forward: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!aligned16(rot_raw) || !aligned16(rot)) { set_error("activations_forward: rotations must be 16-byte aligned"); return GLIC_ERR_INVALID_ARGUMENT; }
    StageTimer _t(GLIC_STAGE_ADAM, stream);
    GLIC_LAUNCH_PDL(activations_forward_kernel, (P + 255) / 256, 256, 0, stream, P, opacity_logit, log_scale,
                    reinterpret_cast<const float4*>(rot_raw), opacity, scale, reinterpret_cast<float4*>(rot), zero4);
    return GLIC_OK;
}
}  // namespace glic

using namespace glic;

extern "C" {

size_t glic_packed_floats(uint32_t P, uint32_t M) { return (size_t)P * (4 + 3 + 3 + 1 + 3 + 3 * (size_t)M); }

int glic_packed_offsets(uint32_t P, uint32_t M, size_t* offsets6) {
    if (!offsets6) { set_error("packed_offsets: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const uint32_t k[6] = {4, 3, 3, 1, 3, 3 * M};
    size_t off = 0;
    for (int q = 0; q < 6; ++q) { offsets6[q] = off; off += (size_t)P * k[q]; }
    return GLIC_OK;
}

int glic_activations_forward(int P, const float* opacity_logit, const float* log_scale, const float* rot_raw, float* opacity,
                             float* scale, float* rot, void* stream) {
    return glic::launch_activations_forward(P, opacity_logit, log_scale, rot_raw, opacity, scale, rot, nullptr, (cudaStream_t)stream);
}

int glic_activations_backward(int P, const float* opacity, const float* scale, const float* rot_raw, float* dL_dopacity,
                              float* dL_dscale, float* dL_drot, void* stream) {
    if (P < 0) { set_error("activations_backward: bad P"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (P == 0) return GLIC_OK;
    if (!opacity || !scale || !rot_raw || !dL_dopacity || !dL_dscale || !dL_drot) { set_error("activations_backward: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!aligned16(rot_raw) || !aligned16(dL_drot)) { set_error("activations_backward: rotations must be 16-byte aligned"); return GLIC_ERR_INVALID_ARGUMENT; }
    StageTimer _t(GLIC_STAGE_ADAM, (cudaStream_t)stream);
    activations_backward_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
        P, opacity, scale, reinterpret_cast<const float4*>(rot_raw), dL_dopacity, dL_dscale, reinterpret_cast<float4*>(dL_drot));
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int glic_adam_update_packed(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const uint8_t* visible,
                            const float* lr6_host, float b1, float b2, float eps, uint32_t P, uint32_t M, void* stream) {
    if (P == 0) return GLIC_OK;
    if (!params || !grads || !exp_avg || !exp_avg_sq || !visible || !lr6_host) { set_error("adam_update_packed: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    PackedLayout L;
    const uint32_t k[6] = {4, 3, 3, 1, 3, 3 * M};
    size_t off = 0;
    for (int q = 0; q < 6; ++q) {
        L.begin[q] = off; L.k[q] = k[q] ? k[q] : 1; L.lr[q] = lr6_host[q];
        off += (size_t)P * k[q];
        L.end[q] = off;
    }
    const size_t total = off;
    const unsigned blocks = (unsigned)std::min<size_t>((total + 255) / 256, (size_t)NUM_SMS * 16);
    StageTimer _t(GLIC_STAGE_ADAM, (cudaStream_t)stream);
    adam_packed_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(params, grads, exp_avg, exp_avg_sq, visible, L, b1, b2, eps, total);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int glic_arena_append(float* params, float* exp_avg, float* exp_avg_sq, uint32_t P, uint32_t Pcap, uint32_t M, uint32_t n_new,
                      const float* xyz, const float* f_dc, const float* log_scale, const float* rot, const float* opacity_logit,
                      void* stream) {
    if (n_new == 0) return GLIC_OK;
    if (!params || !exp_avg || !exp_avg_sq || !xyz || !f_dc || !log_scale || !rot || !opacity_logit) { set_error("arena_append: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if ((Pcap & 3u) != 0 || !aligned16(params) || !aligned16(exp_avg) || !aligned16(exp_avg_sq) || !aligned16(rot)) {
        set_error("arena_append: capacity must be a multiple of 4 and the buffers 16-byte aligned"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if ((uint64_t)P + n_new > Pcap) { set_error("arena_append: capacity exceeded (grow the arena with glic_arena_regrow first)"); return GLIC_ERR_WORKSPACE; }
    ArenaLayout L;
    size_t off6[6];
    glic_packed_offsets(Pcap, M, off6);
    for (int q = 0; q < 6; ++q) { L.off[q] = off6[q]; L.lr[q] = 0.f; }
    arena_append_kernel<<<(n_new + 255) / 256, 256, 0, (cudaStream_t)stream>>>(P, n_new, (int)(3 * M), L, params, exp_avg, exp_avg_sq, xyz, f_dc,
                                                                              log_scale, reinterpret_cast<const float4*>(rot), opacity_logit);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int glic_arena_regrow(const float* src, uint32_t Pcap_src, float* dst, uint32_t Pcap_dst, uint32_t M, uint32_t P, void* stream) {
    if (!src || !dst || P > Pcap_src || P > Pcap_dst) { set_error("arena_regrow: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    size_t a[6], b[6];
    glic_packed_offsets(Pcap_src, M, a);
    glic_packed_offsets(Pcap_dst, M, b);
    const uint32_t k[6] = {4, 3, 3, 1, 3, 3 * M};
    for (int q = 0; q < 6; ++q) {
        if (!k[q] || !P) continue;
        GLIC_CUDA_TRY(cudaMemcpyAsync(dst + b[q], src + a[q], sizeof(float) * (size_t)P * k[q], cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    }
    return GLIC_OK;
}

}  // extern "C"

// ---- launcher used by the mapper (mapper.cu) ---------------------------------------------------------------------
namespace glic {
namespace {
__global__ void __launch_bounds__(256)
view_flags_kernel(int P, const int* __restrict__ radii, const uint8_t* __restrict__ clamped, uint8_t* __restrict__ flags,
                  int* __restrict__ radii_out, const GeomHeader* __restrict__ ghdr, float* __restrict__ overflow_word, ViewZero z) {
    pdl_enter();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        if (ghdr->overflow) *overflow_word = 1.0f;
        *z.loss = 0.0f;
    }
    if (i >= P) return;
    const int r = radii[i];
    flags[i] = r > 0 ? (uint8_t)(0x80u | (clamped[i] & 7u)) : (uint8_t)0;
    if (radii_out) radii_out[i] = r;
    reinterpret_cast<float4*>(z.conic)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int c = 0; c < 3; ++c) { z.mean2D[3 * (size_t)i + c] = 0.0f; z.colors[3 * (size_t)i + c] = 0.0f; }
    z.opacity[i] = 0.0f;
}
}  // namespace

// per-view flags byte of the compact exchange: visibility + the forward's colour-clamp bits; also sets *overflow_word to 1 when the
// forward overflowed its binning workspace, and zeroes what the view's loss and backward accumulate into (z)
int launch_view_flags(int P, const int* radii, const GeomState& g, uint8_t* flags, cudaStream_t s, int* radii_out, float* overflow_word,
                      const ViewZero& z) {
    if (P <= 0) return GLIC_OK;
    GLIC_LAUNCH_PDL(view_flags_kernel, (P + 255) / 256, 256, 0, s, P, radii, g.clamped, flags, radii_out, g.hdr, overflow_word, z);
    return GLIC_OK;
}

int launch_adam_compact(uint32_t P, uint32_t Pcap, int D, int M, float* params, float* exp_avg, float* exp_avg_sq, const float* g_geo,
                        uint32_t Pcap_geo, const float* lr6, const float* g_color, const uint8_t* flags, const float* const* campos_dev,
                        int n_slots, float grad_scale, float color_scale, float b1, float b2, float eps, const unsigned int* skip_flag,
                        unsigned int* visible_count, cudaStream_t s, const float* g_dens, float* dens_accum, float* dens_denom,
                        float dens_scale, const int* radii, int* dens_maxr) {
    if (P == 0) return GLIC_OK;
    ArenaLayout L, Lg;
    size_t off6[6];
    glic_packed_offsets(Pcap, (uint32_t)M, off6);
    for (int q = 0; q < 6; ++q) { L.off[q] = off6[q]; L.lr[q] = lr6[q]; }
    glic_packed_offsets(Pcap_geo, 0, off6);                         // geometric arena: rotation | xyz | log-scale | opacity
    for (int q = 0; q < 6; ++q) { Lg.off[q] = off6[q]; Lg.lr[q] = 0.f; }
    ViewSlots vs;
    if (n_slots < 1 || n_slots > 32 || !campos_dev) { set_error("adam_compact: 1..32 view slots"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (g_dens && (!radii || !dens_maxr)) { set_error("adam_compact: the densification statistics need the radii"); return GLIC_ERR_INVALID_ARGUMENT; }
    vs.g_color = g_color; vs.visible = flags; vs.radii = radii; vs.stride = Pcap_geo; vs.n_slots = n_slots;
    for (int i = 0; i < n_slots; ++i) vs.campos[i] = campos_dev[i];
    const unsigned warps = (P + 31) / 32;
    StageTimer _t(GLIC_STAGE_ADAM, s);
    adam_compact_kernel<<<(warps + ADAM_WARPS - 1) / ADAM_WARPS, ADAM_WARPS * 32, 0, s>>>(
        P, D, M, params, exp_avg, exp_avg_sq, g_geo, L, Lg, vs, grad_scale, color_scale, b1, b2, eps, skip_flag, visible_count, g_dens,
        dens_accum, dens_denom, dens_scale, dens_maxr);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}
}  // namespace glic

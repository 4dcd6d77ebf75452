// initialize.cu -- GPU form of initialize() (/root/reference/src/gaussian.cpp:212-304): the first map, from the first LiDAR
// scan and the skybox, written straight into the caller's rows.  The reference fills its foreground tensors with seven
// indexed GPU writes per LiDAR point from a host loop, draws the sky from torch's global generator and concatenates
// sky | foreground; here one launch writes the LiDAR rows and three write the sky rows (positions, simple-knn over the sky
// alone, the remaining fields).  Checker: the CPU restatement tests/initialize_oracle.py (test infrastructure).
//
// Sky sampling: the reference's two torch.rand draws cannot be reproduced, so the sky is keyed by (seed, row) with a
// counter-based generator instead.  Row i takes the i-th output of SplitMix64 started at `seed`,
//     r = mix64(seed + (i + 1) * 0x9E3779B97F4A7C15),  mix64 = the SplitMix64 finaliser (Steele, Lea, Flood, OOPSLA 2014),
// and splits it into two uniforms on torch.rand's float grid: u1 = (r >> 40) * 2^-24, u2 = ((r >> 16) & 0xFFFFFF) * 2^-24,
// both in [0, 1).  Every device and every rank draws the same sky for the same seed.
#include "common.cuh"

namespace glic {
namespace {

__device__ __forceinline__ void sky_uniforms(uint64_t seed, uint32_t row, float& u1, float& u2) {
    const uint64_t r = splitmix64_mix(seed + ((uint64_t)row + 1) * 0x9E3779B97F4A7C15ull);
    u1 = __fmul_rn((float)(uint32_t)(r >> 40), 5.9604644775390625e-08f);               // * 2^-24: exact
    u2 = __fmul_rn((float)(uint32_t)((r >> 16) & 0xFFFFFFu), 5.9604644775390625e-08f);
}

// gaussian.cpp:214-240.  colors are the Dataset's doubles (rgb / 255.0); RGB2SH and the log-scale are evaluated in double as
// the reference's host loop does (gaussian.h:46-47), then stored as float.
__global__ void __launch_bounds__(256)
lidar_init_kernel(int n, const float* __restrict__ points, const double* __restrict__ colors, const float* __restrict__ depth_rsp,
                  double scaling_scale, double focal, float* __restrict__ xyz, float* __restrict__ f_dc, float* __restrict__ log_scale,
                  float* __restrict__ rot, float* __restrict__ opacity_logit) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float ls = __double2float_rn(log(__ddiv_rn(__dmul_rn(scaling_scale, (double)depth_rsp[i]), focal)));
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        xyz[3 * (size_t)i + c] = points[3 * (size_t)i + c];
        f_dc[3 * (size_t)i + c] = __double2float_rn(__ddiv_rn(__dsub_rn(colors[3 * (size_t)i + c], 0.5), 0.28209479177387814));
        log_scale[3 * (size_t)i + c] = ls;
    }
    reinterpret_cast<float4*>(rot)[i] = make_float4(1.0f, 0.0f, 0.0f, 0.0f);
    opacity_logit[i] = logf(__fdiv_rn(0.1f, __fsub_rn(1.0f, 0.1f)));                  // the bits of extend_init_kernel's
}

// gaussian.cpp:247-253 in torch's float order: theta = (2 * pi) * u1, phi = acos(1 - 1.4 * u2), x = ((10 R) * cos theta) * sin phi
__global__ void __launch_bounds__(256)
sky_xyz_kernel(int n, float r10, uint64_t seed, float* __restrict__ xyz, float* __restrict__ uv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float u1, u2;
    sky_uniforms(seed, (uint32_t)i, u1, u2);
    if (uv) { uv[2 * (size_t)i] = u1; uv[2 * (size_t)i + 1] = u2; }
    const float pi = acosf(-1.0f);
    const float theta = __fmul_rn(__fmul_rn(2.0f, pi), u1);
    const float phi = acosf(__fsub_rn(1.0f, __fmul_rn(1.4f, u2)));
    const float sp = sinf(phi);
    xyz[3 * (size_t)i + 0] = __fmul_rn(__fmul_rn(r10, cosf(theta)), sp);
    xyz[3 * (size_t)i + 1] = __fmul_rn(__fmul_rn(r10, sinf(theta)), sp);
    xyz[3 * (size_t)i + 2] = __fmul_rn(r10, cosf(phi));
}

// gaussian.cpp:255-266: raw colour (0.7, 0.8, 0.95) -- not through RGB2SH --, log(sqrt(clamp_min(dist2, 1e-7))), identity
// rotation, inverse_sigmoid(0.7)
__global__ void __launch_bounds__(256)
sky_fields_kernel(int n, const float* __restrict__ dist2, float* __restrict__ f_dc, float* __restrict__ log_scale,
                  float* __restrict__ rot, float* __restrict__ opacity_logit) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float ls = logf(sqrtf(fmaxf(dist2[i], 1e-7f)));
    const float dc[3] = {0.7f, 0.8f, 0.95f};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        f_dc[3 * (size_t)i + c] = dc[c];
        log_scale[3 * (size_t)i + c] = ls;
    }
    reinterpret_cast<float4*>(rot)[i] = make_float4(1.0f, 0.0f, 0.0f, 0.0f);
    opacity_logit[i] = logf(__fdiv_rn(0.7f, __fsub_rn(1.0f, 0.7f)));
}

// workspace of glic_skybox_init: dist2[n] | glic_knn_mean_dist2's temp
size_t skybox_carve(void* ws, int n, float** dist2, void** knn, size_t* knn_bytes) {
    Carver c(ws);
    float* d = c.take<float>((size_t)(n > 0 ? n : 1));
    const size_t kb = glic_knn_temp_bytes(n);
    void* k = c.take<char>(kb);
    if (dist2) *dist2 = d;
    if (knn) *knn = k;
    if (knn_bytes) *knn_bytes = kb;
    return c.total();
}

bool rot_aligned(const float* rot) { return (reinterpret_cast<uintptr_t>(rot) & 15u) == 0; }

}  // namespace
}  // namespace glic

using namespace glic;

extern "C" {

int glic_lidar_init(int n, const float* points, const double* colors, const float* depth_rsp, double scaling_scale, double focal,
                    float* xyz, float* f_dc, float* log_scale, float* rot, float* opacity_logit, void* stream) {
    if (n < 0) { set_error("lidar_init: n < 0"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (n == 0) return GLIC_OK;
    if (!points || !colors || !depth_rsp || !xyz || !f_dc || !log_scale || !rot || !opacity_logit) {
        set_error("lidar_init: null pointer"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!rot_aligned(rot)) { set_error("lidar_init: rot must be 16-byte aligned"); return GLIC_ERR_INVALID_ARGUMENT; }
    lidar_init_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, points, colors, depth_rsp, scaling_scale, focal, xyz, f_dc,
                                                                          log_scale, rot, opacity_logit);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

size_t glic_skybox_init_bytes(int n) { return skybox_carve(nullptr, n, nullptr, nullptr, nullptr); }

int glic_skybox_init(int n, int radius, uint64_t seed, void* ws, size_t ws_bytes, float* xyz, float* f_dc, float* log_scale, float* rot,
                     float* opacity_logit, float* uv, void* stream) {
    if (n < 0 || (n > 0 && radius <= 0)) { set_error("skybox_init: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (n == 0) return GLIC_OK;
    if (!xyz || !f_dc || !log_scale || !rot || !opacity_logit) { set_error("skybox_init: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!rot_aligned(rot)) { set_error("skybox_init: rot must be 16-byte aligned"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!ws || ws_bytes < glic_skybox_init_bytes(n)) { set_error("skybox_init: workspace too small"); return GLIC_ERR_WORKSPACE; }
    cudaStream_t s = (cudaStream_t)stream;
    float* dist2 = nullptr;
    void* knn = nullptr;
    size_t knn_bytes = 0;
    skybox_carve(ws, n, &dist2, &knn, &knn_bytes);
    const int blocks = (n + 255) / 256;
    // `radius * 10` is a double product in the reference, handed to torch as a float scalar
    sky_xyz_kernel<<<blocks, 256, 0, s>>>(n, (float)((double)radius * 10.0), seed, xyz, uv);
    GLIC_LAUNCH_CHECK();
    if (int e = glic_knn_mean_dist2(n, xyz, dist2, knn, knn_bytes, stream)) return e;
    sky_fields_kernel<<<blocks, 256, 0, s>>>(n, dist2, f_dc, log_scale, rot, opacity_logit);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

}  // extern "C"

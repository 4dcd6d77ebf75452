// extend.cu -- GPU form of extend() (/root/reference/src/gaussian.cpp:499-638, SURVEY 8f rank 2): which LiDAR points of the newest
// frame become Gaussians and with which initial parameters.  The reference projects on the GPU, copies every pixel
// coordinate to the host, de-duplicates through an unordered_map<std::string, ...> and copies the survivors back.
// Here: one 64-bit atomicMin per in-image point on a (orderable depth bits << 32 | index) word per pixel -- the
// smallest camera depth wins a pixel, the earlier index on ties, exactly the reference's strict `<` rule; points
// outside the image cannot shadow in-image ones (different map keys) and are dropped by the filter anyway, so the
// W x H word buffer is the whole map.  Survivors (winner, depth_in_rsp_frame > 0, rendered alpha < 0.99) are compacted in
// ascending index order by a single-CTA scan and initialised in place.  Checkers: tests/extend_oracle.py (exact NumPy
// restatement of the selection), the CPU oracle's restatement, and torch's own device arithmetic (tests/test_gpu_extend_edges.py).
#include "common.cuh"

namespace glic {
namespace {

struct ExtendCam { float r[9]; float t[3]; float fx, fy, cx, cy; int W, H; };

__device__ __forceinline__ bool extend_pixel(const ExtendCam& c, const float* __restrict__ p, int& px, int& py, float& z) {
    // ((p0 r0 + p1 r1) + p2 r2) + t, then (x * fx) / z + cx, every step rounded on its own (no contraction).  The reference's
    // torch.matmul(points, R_cw^T) + t is not one fixed order: measured on an H100 (torch 2.11, TF32 off), its float32 GEMM
    // gives exactly this order for n <= 16 points and the fma chain fmaf(p2, r2, fmaf(p1, r1, p0 r0)) for every n from 17 to
    // 4 194 307 tested, so the two round differently on about half the points of a frame.  A point then falls on another
    // pixel only when an integer lies between its two pixel coordinates, and wins differently only when its depth and its
    // pixel winner's are within that rounding: 3 of 200 000 and 9 of 1 048 577 random points survive differently
    // (tests/test_gpu_extend_edges.py prints the counts per case).
    float cam[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        cam[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p[0], c.r[3 * r + 0]), __fmul_rn(p[1], c.r[3 * r + 1])), __fmul_rn(p[2], c.r[3 * r + 2])), c.t[r]);
    z = cam[2];
    const float fxp = floorf(__fadd_rn(__fdiv_rn(__fmul_rn(cam[0], c.fx), z), c.cx));
    const float fyp = floorf(__fadd_rn(__fdiv_rn(__fmul_rn(cam[1], c.fy), z), c.cy));
    // Non-finite coordinates are rejected.  z = +-0 gives +-inf (x != 0) or NaN (x = 0); z = +-inf gives cx for a finite x.
    // torch's floor().to(int32) on the device saturates +-inf to INT_MAX / INT_MIN, outside the image like here, but turns NaN
    // into 0: in the reference a NaN coordinate lands on column (or row) 0, where a NaN depth wins the pixel if it comes first
    // and then blocks every real point (a NaN scan point has a NaN depth_rsp and is not inserted itself), and a point exactly
    // at the camera centre lands on pixel (0, 0) with depth 0.  Rejecting NaN keeps real points on their pixels.
    // A zero depth never reaches the z-buffer, so every depth that does is finite or +-inf and non-zero.
    if (!(fxp >= 0.0f && fxp < (float)c.W && fyp >= 0.0f && fyp < (float)c.H)) return false;
    px = (int)fxp; py = (int)fyp;
    return true;
}

__device__ __forceinline__ unsigned int orderable(float f) {       // monotone float -> uint (negative depths included)
    f = __fadd_rn(f, 0.0f);                                        // -0.0f -> +0.0f: the reference's float `<` treats them as equal
                                                                   // (extend_pixel passes no zero depth: monotone for every float anyway)
    const unsigned int b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__global__ void __launch_bounds__(256)
extend_zbuffer_kernel(int n, ExtendCam cam, const float* __restrict__ points, unsigned long long* __restrict__ pix) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int px, py; float z;
    if (!extend_pixel(cam, points + 3 * (size_t)i, px, py, z)) return;
    atomicMin(&pix[(size_t)py * cam.W + px], ((unsigned long long)orderable(z) << 32) | (unsigned int)i);
}

__global__ void __launch_bounds__(256)
extend_flag_kernel(int n, ExtendCam cam, const float* __restrict__ points, const float* __restrict__ depth_rsp,
                   const float* __restrict__ final_T, const unsigned long long* __restrict__ pix, unsigned int* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int px, py; float z;
    unsigned int keep = 0;
    if (extend_pixel(cam, points + 3 * (size_t)i, px, py, z)) {
        const size_t q = (size_t)py * cam.W + px;
        const bool winner = (unsigned int)(pix[q] & 0xFFFFFFFFull) == (unsigned int)i;
        const float alpha = __fsub_rn(1.0f, final_T[q]);
        keep = winner && depth_rsp[i] > 0.0f && alpha < 0.99f;
    }
    flag[i] = keep;
}

// exclusive scan of the flags by one CTA (n is a LiDAR frame: 1e4..1e6 points), count out
__global__ void __launch_bounds__(1024)
extend_scan_kernel(int n, unsigned int* __restrict__ flag_to_pos, unsigned int* __restrict__ count) {
    __shared__ unsigned int warp_tot[32];
    __shared__ unsigned int carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + tid;
        const unsigned int f = i < n ? flag_to_pos[i] : 0u;
        unsigned int incl = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const unsigned int w = warp_tot[lane];
            unsigned int wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned int t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            warp_tot[lane] = wi - w;
        }
        __syncthreads();
        const unsigned int excl = carry + warp_tot[warp] + incl - f;
        // position in the low 31 bits, the flag itself in the top bit
        if (i < n) flag_to_pos[i] = excl | (f << 31);
        __syncthreads();
        if (tid == 1023) carry = excl + f;
        __syncthreads();
    }
    if (tid == 0) *count = carry;
}

// the reference's tensor ops on the survivors: RGB2SH (rgb - 0.5f) / C0 and scaling_scale * d / focal divide by a scalar, which
// torch's CUDA division carries out as a multiplication by the scalar's reciprocal, 1.0 / C0 rounded to float once
__global__ void __launch_bounds__(256)
extend_init_kernel(int n, const unsigned int* __restrict__ flag_pos, const float* __restrict__ points,
                   const float* __restrict__ colors, const float* __restrict__ depth_rsp, float scaling_scale, float inv_focal,
                   int* __restrict__ keep_idx, float* __restrict__ xyz, float* __restrict__ f_dc, float* __restrict__ log_scale,
                   float* __restrict__ rot, float* __restrict__ opacity_logit) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned int fp = flag_pos[i];
    if (!(fp >> 31)) return;
    const size_t k = fp & 0x7FFFFFFFu;
    keep_idx[k] = i;
    const float ls = logf(__fmul_rn(__fmul_rn(scaling_scale, depth_rsp[i]), inv_focal));
    constexpr float inv_C0 = (float)(1.0 / 0.28209479177387814);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        xyz[3 * k + c] = points[3 * (size_t)i + c];
        f_dc[3 * k + c] = __fmul_rn(__fsub_rn(colors[3 * (size_t)i + c], 0.5f), inv_C0);
        log_scale[3 * k + c] = ls;
    }
    reinterpret_cast<float4*>(rot)[k] = make_float4(1.0f, 0.0f, 0.0f, 0.0f);
    opacity_logit[k] = logf(__fdiv_rn(0.1f, __fsub_rn(1.0f, 0.1f)));
}

}  // namespace
}  // namespace glic

using namespace glic;

extern "C" {

size_t glic_extend_bytes(int n, int width, int height) {
    const size_t pix = ((size_t)width * height * sizeof(unsigned long long) + 255) & ~size_t(255);
    const size_t flags = ((size_t)(n > 0 ? n : 0) * sizeof(unsigned int) + 255) & ~size_t(255);
    return pix + flags + 256;
}

// All pointers are device pointers except R_cw_host[9] (row-major) / t_cw_host[3] and
// count_host (pinned or pageable; valid after the stream is synchronised by this call).  Output arrays have room for n rows.
int glic_extend(int n, const float* points, const float* colors, const float* depth_rsp, const float* R_cw_host,
                const float* t_cw_host, float fx, float fy, float cx, float cy, int width, int height, const float* final_T,
                float scaling_scale, void* ws, size_t ws_bytes, int* keep_idx, float* xyz, float* f_dc, float* log_scale,
                float* rot, float* opacity_logit, int* count_host, void* stream) {
    if (n < 0 || width <= 0 || height <= 0 || !count_host) { set_error("extend: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    *count_host = 0;
    if (n == 0) return GLIC_OK;
    if (!points || !colors || !depth_rsp || !R_cw_host || !t_cw_host || !final_T || !keep_idx || !xyz || !f_dc || !log_scale || !rot || !opacity_logit) {
        set_error("extend: null pointer"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!ws || ws_bytes < glic_extend_bytes(n, width, height)) { set_error("extend: workspace too small"); return GLIC_ERR_WORKSPACE; }
    if ((reinterpret_cast<uintptr_t>(rot) & 15u) != 0) { set_error("extend: rot must be 16-byte aligned"); return GLIC_ERR_INVALID_ARGUMENT; }
    cudaStream_t s = (cudaStream_t)stream;
    ExtendCam cam;
    for (int i = 0; i < 9; ++i) cam.r[i] = R_cw_host[i];
    for (int i = 0; i < 3; ++i) cam.t[i] = t_cw_host[i];
    cam.fx = fx; cam.fy = fy; cam.cx = cx; cam.cy = cy; cam.W = width; cam.H = height;
    const size_t pix_bytes = ((size_t)width * height * sizeof(unsigned long long) + 255) & ~size_t(255);
    const size_t flag_bytes = ((size_t)n * sizeof(unsigned int) + 255) & ~size_t(255);
    unsigned long long* pix = static_cast<unsigned long long*>(ws);
    unsigned int* flag = reinterpret_cast<unsigned int*>(static_cast<char*>(ws) + pix_bytes);
    unsigned int* count = reinterpret_cast<unsigned int*>(static_cast<char*>(ws) + pix_bytes + flag_bytes);
    GLIC_CUDA_TRY(cudaMemsetAsync(pix, 0xFF, (size_t)width * height * sizeof(unsigned long long), s));
    const int blocks = (n + 255) / 256;
    extend_zbuffer_kernel<<<blocks, 256, 0, s>>>(n, cam, points, pix);
    GLIC_LAUNCH_CHECK();
    extend_flag_kernel<<<blocks, 256, 0, s>>>(n, cam, points, depth_rsp, final_T, pix, flag);
    GLIC_LAUNCH_CHECK();
    extend_scan_kernel<<<1, 1024, 0, s>>>(n, flag, count);
    GLIC_LAUNCH_CHECK();
    const float focal = (fx + fy) / 2.0f;
    extend_init_kernel<<<blocks, 256, 0, s>>>(n, flag, points, colors, depth_rsp, scaling_scale, (float)(1.0 / (double)focal), keep_idx,
                                              xyz, f_dc, log_scale, rot, opacity_logit);
    GLIC_LAUNCH_CHECK();
    unsigned int m = 0;
    GLIC_CUDA_TRY(cudaMemcpyAsync(&m, count, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    *count_host = (int)m;
    return GLIC_OK;
}

}  // extern "C"

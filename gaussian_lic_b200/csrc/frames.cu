// frames.cu -- the 8-bit camera frame as the loss sees it (Dataset::addFrame, /root/reference/src/gaussian.cpp:44-49):
// cv_bridge's BGR8 image, cv::cvtColor(BGR2RGB) and convertTo(CV_32FC3, 1.0f / 255.0f), which evaluates one float product
// x * fl32(1/255) per byte.  The native mapper keeps every frame as packed HWC BGR8 in HBM and decodes it into the [3,H,W]
// float ground truth right before the loss or the evaluation needs it.
#include "common.cuh"

namespace glic {
namespace {

constexpr int DEC_THREADS = 256;
constexpr int DEC_PIX = 16 * DEC_THREADS;            // pixels per CTA: 48 bytes in, 3 x 64 bytes out per thread

__device__ __forceinline__ float dec8(uint32_t word, int shift) {
    return __fmul_rn((float)((word >> shift) & 0xFFu), 1.0f / 255.0f);
}

// One CTA per DEC_PIX pixels.  Full tiles (vec: 16-byte aligned input and output, H*W a multiple of 4): the tile's
// 12288 bytes are read with coalesced 16-byte loads into shared memory, then each thread turns 4 pixels (3 words, stride 3
// words: no bank conflicts) into one float4 per plane, so every warp stores 512 contiguous bytes of each plane.  A partial
// last tile, or unaligned buffers, take the byte-by-byte path.  Both paths compute the same value per byte.
__global__ void __launch_bounds__(DEC_THREADS)
decode_bgr8_kernel(int64_t N, const uint8_t* __restrict__ bgr, float* __restrict__ rgb, int vec) {
    __shared__ uint4 tile[3 * DEC_THREADS];
    const int64_t base = (int64_t)blockIdx.x * DEC_PIX;
    float* r = rgb;
    float* g = rgb + N;
    float* b = rgb + 2 * N;
    if (vec && base + DEC_PIX <= N) {
        const uint4* src = reinterpret_cast<const uint4*>(bgr + 3 * base);
#pragma unroll
        for (int k = 0; k < 3; ++k) tile[threadIdx.x + k * DEC_THREADS] = __ldg(src + threadIdx.x + k * DEC_THREADS);
        __syncthreads();
        const uint32_t* w = reinterpret_cast<const uint32_t*>(tile);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int q = threadIdx.x + j * DEC_THREADS;  // pixels 4q .. 4q+3 of the tile: b0 g0 r0 b1 | g1 r1 b2 g2 | r2 b3 g3 r3
            const uint32_t u0 = w[3 * q], u1 = w[3 * q + 1], u2 = w[3 * q + 2];
            const int64_t p = base + 4 * q;
            *reinterpret_cast<float4*>(r + p) = make_float4(dec8(u0, 16), dec8(u1, 8), dec8(u2, 0), dec8(u2, 24));
            *reinterpret_cast<float4*>(g + p) = make_float4(dec8(u0, 8), dec8(u1, 0), dec8(u1, 24), dec8(u2, 16));
            *reinterpret_cast<float4*>(b + p) = make_float4(dec8(u0, 0), dec8(u0, 24), dec8(u1, 16), dec8(u2, 8));
        }
        return;
    }
    const int64_t end = base + DEC_PIX < N ? base + DEC_PIX : N;
    for (int64_t p = base + threadIdx.x; p < end; p += DEC_THREADS) {
        r[p] = __fmul_rn((float)bgr[3 * p + 2], 1.0f / 255.0f);
        g[p] = __fmul_rn((float)bgr[3 * p + 1], 1.0f / 255.0f);
        b[p] = __fmul_rn((float)bgr[3 * p], 1.0f / 255.0f);
    }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace
}  // namespace glic

using namespace glic;

extern "C" {

int glic_decode_bgr8(int H, int W, const uint8_t* bgr, float* rgb, void* stream) {
    if (H <= 0 || W <= 0) { set_error("decode_bgr8: bad frame size"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!bgr || !rgb) { set_error("decode_bgr8: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const int64_t N = (int64_t)H * W;
    const int vec = aligned16(bgr) && aligned16(rgb) && N % 4 == 0;
    decode_bgr8_kernel<<<(unsigned)((N + DEC_PIX - 1) / DEC_PIX), DEC_THREADS, 0, (cudaStream_t)stream>>>(N, bgr, rgb, vec);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

}  // extern "C"

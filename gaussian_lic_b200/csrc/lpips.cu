// lpips.cu -- LPIPS with the AlexNet trunk, as evaluateVisualQuality scores it (/root/reference/src/gaussian.cpp:741-800 through
// the TorchScript module src/lpips/lpips_alex.pt, traced from lpipsPyTorch/modules/{lpips,networks,utils}.py):
//   x = (clamp(img, 0, 1) - mean) / std                                           (no rescaling to [-1, 1], as the reference)
//   conv0 64x3x11x11 /4 p2 +ReLU -> tap 1 -> maxpool 3/2 -> conv3 192x64x5x5 p2 +ReLU -> tap 2 -> maxpool 3/2 ->
//   conv6 384x192x3x3 p1 +ReLU -> tap 3 -> conv8 256x384x3x3 p1 +ReLU -> tap 4 -> conv10 256x256x3x3 p1 +ReLU -> tap 5
//   LPIPS = sum over taps of mean_px sum_c lin_c * (f_x / (|f_x| + 1e-10) - f_y / (|f_y| + 1e-10))^2
// Both images go through each layer in one launch, as a batch of 2.  The convolutions are one implicit-GEMM kernel (M = output
// pixels of both images, N = output channels, K = Cin*k*k in OIHW order) on mma.sync m16n8k8 TF32 with every operand split
// into hi + lo TF32 parts and hi*hi + hi*lo + lo*hi accumulated in fp32: fp32-class accuracy on the tensor cores (a single
// TF32 pass moves LPIPS by ~3e-4).  Bias and ReLU are fused into the epilogue, the input normalisation into conv0's load.
// Per tap one head kernel writes per-CTA float64 partial sums and one fixed-order finish adds them: no atomics, so two
// identical calls give identical bits.
#include "common.cuh"

#include <algorithm>
#include <cstdio>
#include <string>

namespace glic {
namespace {

constexpr uint32_t LPIPS_MAGIC = 0x5049504Cu;     // "LPIP" as little-endian bytes
constexpr uint32_t LPIPS_VERSION = 1;
constexpr size_t LPIPS_HEADER_BYTES = 16;         // magic | version | float count | 0
constexpr int LPIPS_MIN_SIDE = 31;                // smallest frame with a non-empty tap 5
constexpr int LPIPS_MAX_SIDE = 8192;              // keeps every index of the network inside int32

struct ConvSpec { int cin, cout, k, stride, pad; };
constexpr ConvSpec CONVS[5] = {{3, 64, 11, 4, 2}, {64, 192, 5, 1, 2}, {192, 384, 3, 1, 1}, {384, 256, 3, 1, 1}, {256, 256, 3, 1, 1}};

// float offsets into the weight payload: mean[3] std[3] | (OIHW weight, bias) x 5 | lin 0..4
struct WeightOffsets { size_t w[5], b[5], lin[5], total; };
WeightOffsets weight_offsets() {
    WeightOffsets o{};
    size_t off = 6;
    for (int l = 0; l < 5; ++l) {
        o.w[l] = off; off += (size_t)CONVS[l].cout * CONVS[l].cin * CONVS[l].k * CONVS[l].k;
        o.b[l] = off; off += CONVS[l].cout;
    }
    for (int l = 0; l < 5; ++l) { o.lin[l] = off; off += CONVS[l].cout; }
    o.total = off;
    return o;
}

// spatial size of every tap (h[l] x w[l]) and of the two pooled maps
struct Shapes { int h[5], w[5], ph[2], pw[2]; };
Shapes shapes(int H, int W) {
    Shapes s{};
    s.h[0] = (H + 2 * 2 - 11) / 4 + 1; s.w[0] = (W + 2 * 2 - 11) / 4 + 1;
    s.ph[0] = (s.h[0] - 3) / 2 + 1;    s.pw[0] = (s.w[0] - 3) / 2 + 1;
    s.h[1] = s.ph[0];                  s.w[1] = s.pw[0];
    s.ph[1] = (s.h[1] - 3) / 2 + 1;    s.pw[1] = (s.w[1] - 3) / 2 + 1;
    for (int l = 2; l < 5; ++l) { s.h[l] = s.ph[1]; s.w[l] = s.pw[1]; }
    return s;
}

constexpr int HEAD_THREADS = 256;
inline unsigned head_blocks(int hw) { return (unsigned)((hw + HEAD_THREADS - 1) / HEAD_THREADS); }

struct Scratch { float* tap[5]; float* pool[2]; double* partials[5]; };
Scratch carve(void* ws, int H, int W, size_t* bytes) {
    const Shapes s = shapes(H, W);
    Carver c(ws);
    Scratch r{};
    for (int l = 0; l < 5; ++l) r.tap[l] = c.take<float>((size_t)2 * CONVS[l].cout * s.h[l] * s.w[l]);
    for (int p = 0; p < 2; ++p) r.pool[p] = c.take<float>((size_t)2 * CONVS[p].cout * s.ph[p] * s.pw[p]);
    for (int l = 0; l < 5; ++l) r.partials[l] = c.take<double>(head_blocks(s.h[l] * s.w[l]));
    if (bytes) *bytes = c.total();
    return r;
}

// ---- implicit-GEMM convolution, split-TF32 mma.sync ------------------------------------------------------------------------
constexpr int BM = 64, BN = 64, BK = 32, CONV_THREADS = 128;   // 4 warps, 2 x 2, 32 x 32 outputs each
constexpr int AS_STRIDE = BM + 8;                               // As[k][m]: fragment loads hit 32 distinct banks
constexpr int BS_STRIDE = BK + 4;                               // Bs[n][k]: k-contiguous stores and fragment loads conflict-free

struct ConvArgs {
    const float* in0; const float* in1;   // [Cin][Hi][Wi] of image 0 and image 1
    int Cin, Hi, Wi;
    const float* w; const float* bias;    // OIHW, [Cout]
    int Cout;
    float* out;                           // [2][Cout][Ho][Wo]
    int Ho, Wo;
    const float* norm;                    // NORM: mean[3] std[3]
};

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = to_tf32(x);
    lo = to_tf32(x - __uint_as_float(hi));           // exact in fp32
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// out = ReLU(conv(in) + bias).  NORM: in is the raw image; it is clamped to [0,1] and normalised as it is loaded, and the
// zero padding is applied after the normalisation, as conv2d pads its (normalised) input.
template <int KS, int STRIDE, int PAD, bool NORM>
__global__ void __launch_bounds__(CONV_THREADS)
lpips_conv_kernel(ConvArgs a) {
    __shared__ float As[BK][AS_STRIDE];
    __shared__ float Bs[BN][BS_STRIDE];
    constexpr int KK = KS * KS;
    const int HWo = a.Ho * a.Wo, Mtot = 2 * HWo, K = a.Cin * KK;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int tid = threadIdx.x;

    // A loader: one output pixel (column am of the tile), rows ak0 + 2j of the k block
    const int am = tid & (BM - 1), ak0 = tid >> 6;
    const int mg = m0 + am;
    const bool mvalid = mg < Mtot;
    const float* src = a.in0;
    int iy0 = 0, ix0 = 0;
    if (mvalid) {
        const int n = mg / HWo, r = mg - n * HWo, oy = r / a.Wo, ox = r - oy * a.Wo;
        src = n ? a.in1 : a.in0;
        iy0 = oy * STRIDE - PAD; ix0 = ox * STRIDE - PAD;
    }
    // B loader: k = bk (lane), output channels bn0 + 4j
    const int bk = tid & (BK - 1), bn0 = tid >> 5;
    constexpr int AJ = BM * BK / CONV_THREADS, BJ = BN * BK / CONV_THREADS;   // 16, 16
    float ra[AJ], rb[BJ];

    auto load_tile = [&](int k0) {
#pragma unroll
        for (int j = 0; j < AJ; ++j) {
            const int kk = k0 + ak0 + 2 * j;
            float v = 0.f;
            if (mvalid && kk < K) {
                const int ci = kk / KK, r = kk - ci * KK, ky = r / KS, kx = r - ky * KS;
                const int iy = iy0 + ky, ix = ix0 + kx;
                if (iy >= 0 && iy < a.Hi && ix >= 0 && ix < a.Wi) {
                    v = __ldg(src + ((size_t)ci * a.Hi + iy) * a.Wi + ix);
                    if (NORM) v = __fdiv_rn(__fsub_rn(fminf(fmaxf(v, 0.f), 1.f), __ldg(a.norm + ci)), __ldg(a.norm + 3 + ci));
                }
            }
            ra[j] = v;
        }
#pragma unroll
        for (int j = 0; j < BJ; ++j) {
            const int kk = k0 + bk, co = n0 + bn0 + 4 * j;
            rb[j] = (kk < K && co < a.Cout) ? __ldg(a.w + (size_t)co * K + kk) : 0.f;
        }
    };
    auto store_tile = [&]() {
#pragma unroll
        for (int j = 0; j < AJ; ++j) As[ak0 + 2 * j][am] = ra[j];
#pragma unroll
        for (int j = 0; j < BJ; ++j) Bs[bn0 + 4 * j][bk] = rb[j];
    };

    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

    const int nk = (K + BK - 1) / BK;
    load_tile(0);
    store_tile();
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        if (kt + 1 < nk) load_tile((kt + 1) * BK);
#pragma unroll
        for (int k8 = 0; k8 < BK; k8 += 8) {
            uint32_t ahi[2][4], alo[2][4], bhi[4][2], blo[4][2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int mr = wm + 16 * i + g;
                split_tf32(As[k8 + t][mr], ahi[i][0], alo[i][0]);
                split_tf32(As[k8 + t][mr + 8], ahi[i][1], alo[i][1]);
                split_tf32(As[k8 + t + 4][mr], ahi[i][2], alo[i][2]);
                split_tf32(As[k8 + t + 4][mr + 8], ahi[i][3], alo[i][3]);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int nc = wn + 8 * j + g;
                split_tf32(Bs[nc][k8 + t], bhi[j][0], blo[j][0]);
                split_tf32(Bs[nc][k8 + t + 4], bhi[j][1], blo[j][1]);
            }
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {        // the two small cross terms first, then the main product
                    mma_tf32(acc[i][j], alo[i], bhi[j]);
                    mma_tf32(acc[i][j], ahi[i], blo[j]);
                    mma_tf32(acc[i][j], ahi[i], bhi[j]);
                }
        }
        __syncthreads();
        if (kt + 1 < nk) {
            store_tile();
            __syncthreads();
        }
    }

    // epilogue: c0 (g, 2t), c1 (g, 2t+1), c2 (g+8, 2t), c3 (g+8, 2t+1) of each 16 x 8 tile
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int r2 = 0; r2 < 2; ++r2) {
            const int row = m0 + wm + 16 * i + g + 8 * r2;
            if (row >= Mtot) continue;
            const int n = row / HWo, rem = row - n * HWo;
            float* o = a.out + (size_t)n * a.Cout * HWo + rem;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int c1 = 0; c1 < 2; ++c1) {
                    const int col = n0 + wn + 8 * j + 2 * t + c1;
                    if (col < a.Cout) o[(size_t)col * HWo] = fmaxf(acc[i][j][2 * r2 + c1] + __ldg(a.bias + col), 0.f);
                }
        }
}

// 3x3 / stride 2 max pool without padding (floor mode) over [2*C][h][w]
__global__ void __launch_bounds__(256)
lpips_maxpool_kernel(const float* __restrict__ in, int h, int w, float* __restrict__ out, int ph, int pw, size_t total) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % pw);
        const size_t r = i / pw;
        const int y = (int)(r % ph);
        const size_t plane = r / ph;
        const float* p = in + (plane * h + 2 * y) * w + 2 * x;
        float v = p[0];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) v = fmaxf(v, p[dy * w + dx]);
        out[i] = v;
    }
}

// steps 4-5 for one tap f = [2][C][hw] (image 0 = x, image 1 = y): per pixel sum_c lin_c (x_c/(|x|+eps) - y_c/(|y|+eps))^2,
// summed over the CTA's pixels in float64 in a fixed order -> partials[blockIdx.x]
__global__ void __launch_bounds__(HEAD_THREADS)
lpips_head_kernel(const float* __restrict__ f, int C, int hw, const float* __restrict__ lin, double* __restrict__ partials) {
    __shared__ double red[HEAD_THREADS / 32];
    const int p = blockIdx.x * HEAD_THREADS + threadIdx.x;
    double v = 0.0;
    if (p < hw) {
        const float* fx = f + p;
        const float* fy = f + (size_t)C * hw + p;
        float sx = 0.f, sy = 0.f;
        for (int c = 0; c < C; ++c) {
            const float x = fx[(size_t)c * hw], y = fy[(size_t)c * hw];
            sx = fmaf(x, x, sx); sy = fmaf(y, y, sy);
        }
        const float nx = sqrtf(sx) + 1e-10f, ny = sqrtf(sy) + 1e-10f;
        float d = 0.f;
        for (int c = 0; c < C; ++c) {
            const float e = __fdiv_rn(fx[(size_t)c * hw], nx) - __fdiv_rn(fy[(size_t)c * hw], ny);
            d = fmaf(__ldg(lin + c), e * e, d);
        }
        v = (double)d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int q = 0; q < HEAD_THREADS / 32; ++q) s += red[q];
        partials[blockIdx.x] = s;
    }
}

struct FinishArgs { const double* partials[5]; unsigned blocks[5]; int hw[5]; };

// <<<1, 160>>>: warp l adds tap l's partials lane-strided and takes the spatial mean; thread 0 sums the five taps in order
__global__ void __launch_bounds__(160) lpips_finish_kernel(FinishArgs a, float* __restrict__ out1) {
    __shared__ double tap[5];
    const int l = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double s = 0.0;
    for (unsigned b = lane; b < a.blocks[l]; b += 32) s += a.partials[l][b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) tap[l] = s / (double)a.hw[l];
    __syncthreads();
    if (threadIdx.x == 0) out1[0] = (float)((((tap[0] + tap[1]) + tap[2]) + tap[3]) + tap[4]);
}

template <int KS, int STRIDE, int PAD, bool NORM>
int launch_conv(const ConvArgs& a, cudaStream_t s) {
    const int Mtot = 2 * a.Ho * a.Wo;
    const dim3 grid((unsigned)((Mtot + BM - 1) / BM), (unsigned)((a.Cout + BN - 1) / BN));
    lpips_conv_kernel<KS, STRIDE, PAD, NORM><<<grid, CONV_THREADS, 0, s>>>(a);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_pool(const float* in, int C, int h, int w, float* out, int ph, int pw, cudaStream_t s) {
    const size_t total = (size_t)2 * C * ph * pw;
    const unsigned blocks = (unsigned)std::min<size_t>((total + 255) / 256, (size_t)NUM_SMS * 16);
    lpips_maxpool_kernel<<<blocks, 256, 0, s>>>(in, h, w, out, ph, pw, total);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

#define LPIPS_TRY(...) do { int _e = (__VA_ARGS__); if (_e != GLIC_OK) return _e; } while (0)

bool lpips_frame_ok(int H, int W) {
    return H >= LPIPS_MIN_SIDE && W >= LPIPS_MIN_SIDE && H <= LPIPS_MAX_SIDE && W <= LPIPS_MAX_SIDE;
}

}  // namespace
}  // namespace glic

using namespace glic;

extern "C" {

size_t glic_lpips_weight_floats(void) { return weight_offsets().total; }

int glic_lpips_read_weights(const char* path, float* host) {
    if (!path || !host) { set_error("lpips_read_weights: null argument"); return GLIC_ERR_INVALID_ARGUMENT; }
    FILE* f = std::fopen(path, "rb");
    if (!f) { set_error(std::string("lpips_read_weights: cannot open ") + path); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t n = weight_offsets().total;
    uint32_t hdr[4] = {0, 0, 0, 0};
    std::string err;
    if (std::fread(hdr, 1, LPIPS_HEADER_BYTES, f) != LPIPS_HEADER_BYTES) err = "truncated header";
    else if (hdr[0] != LPIPS_MAGIC) err = "bad magic (not an LPIPS AlexNet weight file)";
    else if (hdr[1] != LPIPS_VERSION) err = "unsupported version " + std::to_string(hdr[1]);
    else if (hdr[2] != n || hdr[3] != 0) err = "header counts " + std::to_string(hdr[2]) + " floats, expected " + std::to_string(n);
    else if (std::fread(host, sizeof(float), n, f) != n) err = "truncated file";
    else if (std::fgetc(f) != EOF) err = "trailing bytes after the weights";
    std::fclose(f);
    if (!err.empty()) { set_error("lpips_read_weights: " + err + ": " + path); return GLIC_ERR_INVALID_ARGUMENT; }
    return GLIC_OK;
}

size_t glic_lpips_scratch_bytes(int H, int W) {
    if (!lpips_frame_ok(H, W)) return 0;
    size_t bytes = 0;
    carve(nullptr, H, W, &bytes);
    return bytes;
}

int glic_lpips(int H, int W, const float* img, const float* gt, const float* weights, float* out1, void* scratch,
               size_t scratch_bytes, void* stream) {
    if (!lpips_frame_ok(H, W)) {
        set_error("lpips: frame " + std::to_string(W) + "x" + std::to_string(H) + " outside 31x31 .. 8192x8192 (AlexNet needs at least 31x31)");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!img || !gt || !weights || !out1 || !scratch) { set_error("lpips: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    size_t need = 0;
    const Scratch sc = carve(scratch, H, W, &need);
    if (scratch_bytes < need) { set_error("lpips: scratch smaller than glic_lpips_scratch_bytes"); return GLIC_ERR_WORKSPACE; }
    cudaStream_t s = (cudaStream_t)stream;
    const Shapes sh = shapes(H, W);
    const WeightOffsets wo = weight_offsets();
    auto args = [&](int l, const float* in0, const float* in1, int hi, int wi) {
        ConvArgs a{};
        a.in0 = in0; a.in1 = in1; a.Cin = CONVS[l].cin; a.Hi = hi; a.Wi = wi;
        a.w = weights + wo.w[l]; a.bias = weights + wo.b[l]; a.Cout = CONVS[l].cout;
        a.out = sc.tap[l]; a.Ho = sh.h[l]; a.Wo = sh.w[l]; a.norm = weights;
        return a;
    };
    auto second = [&](int l_in, const float* buf, int h, int w) { return buf + (size_t)CONVS[l_in].cout * h * w; };
    LPIPS_TRY(launch_conv<11, 4, 2, true>(args(0, img, gt, H, W), s));
    LPIPS_TRY(launch_pool(sc.tap[0], 64, sh.h[0], sh.w[0], sc.pool[0], sh.ph[0], sh.pw[0], s));
    LPIPS_TRY(launch_conv<5, 1, 2, false>(args(1, sc.pool[0], second(0, sc.pool[0], sh.ph[0], sh.pw[0]), sh.ph[0], sh.pw[0]), s));
    LPIPS_TRY(launch_pool(sc.tap[1], 192, sh.h[1], sh.w[1], sc.pool[1], sh.ph[1], sh.pw[1], s));
    LPIPS_TRY(launch_conv<3, 1, 1, false>(args(2, sc.pool[1], second(1, sc.pool[1], sh.ph[1], sh.pw[1]), sh.ph[1], sh.pw[1]), s));
    for (int l = 3; l < 5; ++l)
        LPIPS_TRY(launch_conv<3, 1, 1, false>(args(l, sc.tap[l - 1], second(l - 1, sc.tap[l - 1], sh.h[l - 1], sh.w[l - 1]),
                                                       sh.h[l - 1], sh.w[l - 1]), s));
    FinishArgs fa{};
    for (int l = 0; l < 5; ++l) {
        const int hw = sh.h[l] * sh.w[l];
        fa.partials[l] = sc.partials[l]; fa.blocks[l] = head_blocks(hw); fa.hw[l] = hw;
        lpips_head_kernel<<<fa.blocks[l], HEAD_THREADS, 0, s>>>(sc.tap[l], CONVS[l].cout, hw, weights + wo.lin[l], sc.partials[l]);
        GLIC_LAUNCH_CHECK();
    }
    lpips_finish_kernel<<<1, 160, 0, s>>>(fa, out1);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

}  // extern "C"

// ssim.cu -- fused 11x11 separable-Gaussian SSIM map (+ partial-derivative maps), its backward,
// and the whole L1 + D-SSIM photometric loss of one mapping iteration.
//
// Replaces fusedssimCUDA / fusedssim_backwardCUDA (reference fused-ssim/ssim.cu:186-365) and, for
// glic_l1_ssim_loss, the chain l1_loss + fused_ssim + loss-combine + their autograd backward
// (gaussian.cpp:685-697, loss_utils.h:30-33,135-193).
//
// Design: one CTA (256 threads) = one 32x32 output tile of one channel.  Both 42x42 halo tiles are loaded
// once; the horizontal pass produces all five moment rows (x, y, xx, yy, xy) into shared memory in one
// register-tiled sweep (4 outputs per item) and the vertical pass finishes 4 rows per thread: 3 barriers
// per tile instead of the reference's 18 per channel, ~3x fewer shared-memory loads than one-output-per-
// thread, no scratch-buffer re-zeroing.  Zero ("same") padding as the reference.
// The convolutions are pure multiply-add streams; in the FORWARD kernel the moments travel in PAIRS (f32x2.cuh): (x, y) and
// (xx, yy) are updated together per tap, xy separately, and the pairs sit interleaved in shared memory so one 64-bit load
// fetches both.  Each half is the same fmaf(g, v, acc) chain as the scalar form: bit-identical results.  The backward
// (3 maps) stays scalar: its 64-bit shared-memory traffic would cost more than pairing saves.
#include "common.cuh"
#include "adam_math.cuh"
#include "f32x2.cuh"
#include <algorithm>

namespace glic {

namespace {

constexpr int SB = 32;              // output tile edge
constexpr int HALO = 5;
constexpr int SH_ = SB + 2 * HALO;  // 42
constexpr int ST = 256;             // threads per CTA: 32 columns x 8 row groups, 4 outputs per thread
constexpr int RPT = 4;              // rows (vertical pass) / columns (horizontal pass) per thread

__device__ __constant__ float kG[11] = {0.001028380123898387f, 0.0075987582094967365f, 0.036000773310661316f,
                                        0.10936068743467331f,  0.21300552785396576f,   0.26601171493530273f,
                                        0.21300552785396576f,  0.10936068743467331f,   0.036000773310661316f,
                                        0.0075987582094967365f, 0.001028380123898387f};

__device__ __forceinline__ float pix_or_zero(const float* __restrict__ img, int y, int x, int H, int W) {
    return (x >= 0 && y >= 0 && x < W && y < H) ? img[(size_t)y * W + x] : 0.0f;
}

// Per-image affine exposure (glic_l1_ssim_loss_exposure): E is 3x4 row-major and output channel c is
//   out_c = E[0][c]*r + E[1][c]*g + E[2][c]*b + E[c][3]
// (Inria 3DGS: matmul(img_hwc, E[:3,:3]) + E[:3,3]), evaluated in this fixed fma order so that E = [I | 0] gives out == img
// exactly for finite non-negative images.
struct ExpoCoef { float e0, e1, e2, e3; };

__device__ __forceinline__ ExpoCoef expo_coef(const float* __restrict__ E, int c) { return {E[c], E[4 + c], E[8 + c], E[4 * c + 3]}; }

// i: pixel index within a plane; img: the three planes of the rendered image, HW floats apart
__device__ __forceinline__ float expose(const float* __restrict__ img, size_t HW, size_t i, ExpoCoef e) {
    float acc = e.e3;
    acc = fmaf(img[i], e.e0, acc);
    acc = fmaf(img[HW + i], e.e1, acc);
    return fmaf(img[2 * HW + i], e.e2, acc);
}

// Register-tiled separable 11-tap convolution.  Horizontal pass: one work item = 4 consecutive outputs
// of one halo row (14 loads per image instead of 44); vertical pass: one thread = 4 consecutive rows of
// one column (14 loads per moment instead of 44).  Row strides 43 / 33 keep both passes bank-conflict free.
// LOSS = true: additionally accumulates (1-lambda)*|a-b| - lambda*ssim, scaled by 1/N, into *loss.
// EXPO = true: img1 is the three planes of the rendered image and the tile's channel of the exposed image is formed in the
// halo load (it never exists in global memory); SSIM, its partial maps and the L1 term are those of the exposed image.
// FIXED (fixed-order sums, the native mapper's deterministic option): the CTA's loss term goes to loss[linear block id] instead of
// an atomicAdd into loss[0]; loss_finish_kernel sums those partials in a fixed order.
// MASK (glic_l1_ssim_loss_masked): a pixel whose bit in mk is clear loads as 0 in both images (a select: nothing read there can
// leak), exactly like the zero padding outside the frame, and adds no L1 / SSIM term to the loss.
template <bool LOSS, bool EXPO, bool FIXED = false, bool MASK = false>
__device__ __forceinline__ void
ssim_forward_tile(int H, int W, float C1, float C2, const float* __restrict__ img1, const float* __restrict__ img2,
                  float* __restrict__ ssim_map, float* __restrict__ dm_dmu1, float* __restrict__ dm_dsigma1_sq,
                  float* __restrict__ dm_dsigma12, float lambda_dssim, float inv_n, float* __restrict__ loss,
                  const float* __restrict__ E, MaskView mk = MaskView{nullptr, 0, 0}) {
    __shared__ float s1[SH_][SH_ + 1];
    __shared__ float s2[SH_][SH_ + 1];
    __shared__ float2 h01[SH_][SB + 1];          // horizontal pass of (x, y)
    __shared__ float2 h23[SH_][SB + 1];          // horizontal pass of (xx, yy)
    __shared__ float h4[SH_][SB + 1];            // horizontal pass of xy
    __shared__ float red[ST / 32];
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const size_t plane = (size_t)blockIdx.z * H * W;
    const float* a = img1 + (EXPO ? 0 : plane);
    const float* b = img2 + plane;
    const int x0 = blockIdx.x * SB, y0 = blockIdx.y * SB;
    const uint32_t* vbits = nullptr;

    if (MASK) {
        // the centre rows' mask bits, columns x0 .. x0 + 31 of row y0 + r in bit r of vrow: the loss term reads them here
        // rather than through the view's pointer, which would otherwise stay live across the convolutions
        __shared__ uint32_t vrow[SB];
        if (tid < SB) {
            const int y = y0 + tid, c = mk.x0 + x0, w = c >> 5, sh = c & 31;
            uint32_t bits = 0u;
            if (y < H) {
                const uint32_t* row = mk.words + (size_t)y * mk.words_per_row;
                bits = __funnelshift_r(row[w], (sh && w + 1 < mk.words_per_row) ? row[w + 1] : 0u, sh);
            }
            vrow[tid] = bits;
        }
        vbits = vrow;
        const ExpoCoef e = EXPO ? expo_coef(E, blockIdx.z) : ExpoCoef{};
        for (int i = tid; i < SH_ * SH_; i += ST) {
            const int ly = i / SH_, lx = i % SH_;
            const int y = y0 + ly - HALO, x = x0 + lx - HALO;
            const bool use = x >= 0 && y >= 0 && x < W && y < H && mask_bit(mk, y, x);
            const size_t p = (size_t)y * W + x;
            s1[ly][lx] = use ? (EXPO ? expose(a, (size_t)H * W, p, e) : a[p]) : 0.0f;
            s2[ly][lx] = use ? b[p] : 0.0f;
        }
    } else if (EXPO) {
        const ExpoCoef e = expo_coef(E, blockIdx.z);
        for (int i = tid; i < SH_ * SH_; i += ST) {
            const int ly = i / SH_, lx = i % SH_;
            const int y = y0 + ly - HALO, x = x0 + lx - HALO;
            s1[ly][lx] = (x >= 0 && y >= 0 && x < W && y < H) ? expose(a, (size_t)H * W, (size_t)y * W + x, e) : 0.0f;
            s2[ly][lx] = pix_or_zero(b, y, x, H, W);
        }
    } else {
        for (int i = tid; i < SH_ * SH_; i += ST) {
            const int ly = i / SH_, lx = i % SH_;
            s1[ly][lx] = pix_or_zero(a, y0 + ly - HALO, x0 + lx - HALO, H, W);
            s2[ly][lx] = pix_or_zero(b, y0 + ly - HALO, x0 + lx - HALO, H, W);
        }
    }
    __syncthreads();
    for (int i = tid; i < SH_ * (SB / RPT); i += ST) {
        const int ly = i % SH_, lx = (i / SH_) * RPT;     // consecutive lanes = consecutive rows: conflict-free for the 64-bit pair arrays
        f2 pq[RPT + 10], sq[RPT + 10];
        float xy[RPT + 10];
#pragma unroll
        for (int k = 0; k < RPT + 10; ++k) {
            const float pp = s1[ly][lx + k], qq = s2[ly][lx + k];
            pq[k] = f2_pack(pp, qq);
            sq[k] = f2_mul(pq[k], pq[k]);
            xy[k] = pp * qq;
        }
#pragma unroll
        for (int j = 0; j < RPT; ++j) {
            f2 m = f2_bcast(0.f), q = m;
            float q12 = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                const float g = kG[k];
                m = f2_fma(pq[j + k], g, m);
                q = f2_fma(sq[j + k], g, q);
                q12 = fmaf(g, xy[j + k], q12);
            }
            float lo, hi;
            f2_unpack(m, lo, hi); h01[ly][lx + j] = make_float2(lo, hi);
            f2_unpack(q, lo, hi); h23[ly][lx + j] = make_float2(lo, hi);
            h4[ly][lx + j] = q12;
        }
    }
    __syncthreads();
    float v[5][RPT];
    {
        f2 c01[RPT + 10], c23[RPT + 10];
        float c4[RPT + 10];
#pragma unroll
        for (int k = 0; k < RPT + 10; ++k) {
            const float2 u = h01[ty * RPT + k][tx], w = h23[ty * RPT + k][tx];
            c01[k] = f2_pack(u.x, u.y); c23[k] = f2_pack(w.x, w.y);
            c4[k] = h4[ty * RPT + k][tx];
        }
#pragma unroll
        for (int j = 0; j < RPT; ++j) {
            f2 m = f2_bcast(0.f), q = m;
            float q12 = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                const float g = kG[k];
                m = f2_fma(c01[j + k], g, m);
                q = f2_fma(c23[j + k], g, q);
                q12 = fmaf(g, c4[j + k], q12);
            }
            f2_unpack(m, v[0][j], v[1][j]);
            f2_unpack(q, v[2][j], v[3][j]);
            v[4][j] = q12;
        }
    }
    float part = 0.f;
    const int px = x0 + tx;
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
        const float mu1 = v[0][j], mu2 = v[1][j];
        const float sigma1_sq = v[2][j] - mu1 * mu1, sigma2_sq = v[3][j] - mu2 * mu2, sigma12 = v[4][j] - mu1 * mu2;
        const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu1_mu2 = mu1 * mu2;
        const float Cq = 2.0f * mu1_mu2 + C1, Dq = 2.0f * sigma12 + C2;
        const float A = mu1_sq + mu2_sq + C1, B = sigma1_sq + sigma2_sq + C2;
        const float m = (Cq * Dq) / (A * B);
        const int ry = ty * RPT + j, py = y0 + ry;
        if (px < W && py < H) {
            const size_t gi = plane + (size_t)py * W + px;
            if (ssim_map) ssim_map[gi] = m;
            if (dm_dmu1) {
                dm_dmu1[gi] = ((mu2 * 2.0f * Dq) / (A * B) - (mu2 * 2.0f * Cq) / (A * B) - (mu1 * 2.0f * Cq * Dq) / (A * A * B) +
                               (mu1 * 2.0f * Cq * Dq) / (A * B * B));
                dm_dsigma1_sq[gi] = ((-Cq * Dq) / (A * B * B));
                dm_dsigma12[gi] = ((2.0f * Cq) / (A * B));
            }
            if (LOSS && (!MASK || ((vbits[ry] >> tx) & 1u)))
                part += (1.0f - lambda_dssim) * fabsf(s1[ry + HALO][tx + HALO] - s2[ry + HALO][tx + HALO]) - lambda_dssim * m;
        }
    }
    if (LOSS) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        if (tx == 0) red[ty] = part;
        __syncthreads();
        if (tid == 0) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < ST / 32; ++w) t += red[w];
            if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) t = fmaf(t, inv_n, lambda_dssim);
            else t *= inv_n;
            if (FIXED) loss[(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = t;
            else atomicAdd(loss, t);
        }
    }
}

template <bool LOSS, bool FIXED = false>
__global__ void __launch_bounds__(ST)
ssim_forward_kernel(int H, int W, float C1, float C2, const float* __restrict__ img1, const float* __restrict__ img2,
                    float* __restrict__ ssim_map, float* __restrict__ dm_dmu1, float* __restrict__ dm_dsigma1_sq,
                    float* __restrict__ dm_dsigma12, float lambda_dssim, float inv_n, float* __restrict__ loss) {
    pdl_enter();
    ssim_forward_tile<LOSS, false, FIXED>(H, W, C1, C2, img1, img2, ssim_map, dm_dmu1, dm_dsigma1_sq, dm_dsigma12, lambda_dssim, inv_n,
                                   loss, nullptr);
}

// forward of the exposed loss: the partial maps of SSIM(out, gt) and the loss of out
template <bool FIXED = false>
__global__ void __launch_bounds__(ST)
ssim_loss_exposure_forward_kernel(int H, int W, float C1, float C2, const float* __restrict__ img, const float* __restrict__ gt,
                                  const float* __restrict__ E, float* __restrict__ dm_dmu1, float* __restrict__ dm_dsigma1_sq,
                                  float* __restrict__ dm_dsigma12, float lambda_dssim, float inv_n, float* __restrict__ loss) {
    pdl_enter();
    ssim_forward_tile<true, true, FIXED>(H, W, C1, C2, img, gt, nullptr, dm_dmu1, dm_dsigma1_sq, dm_dsigma12, lambda_dssim, inv_n, loss, E);
}

// dL/dimg1 = conv(dL*dm_dmu1) + 2*img1*conv(dL*dm_dsigma1_sq) + img2*conv(dL*dm_dsigma12)
// CONST_DL: dL_dmap is the constant `dl_const` (fused loss) and the L1 sign term is added.
// EXPO: img1 is the three planes of the rendered image; the result is dL/dout at the exposed image out (see expose()).
// MASK: a masked pixel carries no SSIM term (its dL/dmap is 0 as a halo pixel) and gets dL/dimg1 = +0 (a select).
template <bool CONST_DL, bool EXPO, bool MASK = false>
__device__ __forceinline__ void
ssim_backward_tile(int H, int W, const float* __restrict__ img1, const float* __restrict__ img2,
                   const float* __restrict__ dL_dmap, const float* __restrict__ dm_dmu1,
                   const float* __restrict__ dm_dsigma1_sq, const float* __restrict__ dm_dsigma12,
                   float* __restrict__ dL_dimg1, float dl_const, float l1_scale, const float* __restrict__ E,
                   MaskView mk = MaskView{nullptr, 0, 0}) {
    __shared__ float s[3][SH_][SH_ + 1];
    __shared__ float h[3][SH_][SB + 1];
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const size_t plane = (size_t)blockIdx.z * H * W;
    const int x0 = blockIdx.x * SB, y0 = blockIdx.y * SB;
    for (int i = tid; i < SH_ * SH_; i += ST) {
        const int ly = i / SH_, lx = i % SH_;
        const int y = y0 + ly - HALO, x = x0 + lx - HALO;
        float v0 = 0.f, v1 = 0.f, v2 = 0.f;
        if (x >= 0 && y >= 0 && x < W && y < H && (!MASK || mask_bit(mk, y, x))) {
            const size_t gi = plane + (size_t)y * W + x;
            const float dl = CONST_DL ? dl_const : dL_dmap[gi];
            v0 = dm_dmu1[gi] * dl; v1 = dm_dsigma1_sq[gi] * dl; v2 = dm_dsigma12[gi] * dl;
        }
        s[0][ly][lx] = v0; s[1][ly][lx] = v1; s[2][ly][lx] = v2;
    }
    __syncthreads();
    for (int i = tid; i < SH_ * (SB / RPT); i += ST) {
        const int ly = i / (SB / RPT), lx = (i % (SB / RPT)) * RPT;
#pragma unroll
        for (int qn = 0; qn < 3; ++qn) {
            float p[RPT + 10];
#pragma unroll
            for (int k = 0; k < RPT + 10; ++k) p[k] = s[qn][ly][lx + k];
#pragma unroll
            for (int j = 0; j < RPT; ++j) {
                float acc = 0.f;
#pragma unroll
                for (int k = 0; k < 11; ++k) acc = fmaf(kG[k], p[j + k], acc);
                h[qn][ly][lx + j] = acc;
            }
        }
    }
    __syncthreads();
    float c[3][RPT];
#pragma unroll
    for (int qn = 0; qn < 3; ++qn) {
        float col[RPT + 10];
#pragma unroll
        for (int k = 0; k < RPT + 10; ++k) col[k] = h[qn][ty * RPT + k][tx];
#pragma unroll
        for (int j = 0; j < RPT; ++j) {
            float acc = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) acc = fmaf(kG[k], col[j + k], acc);
            c[qn][j] = acc;
        }
    }
    const int px = x0 + tx;
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
        const int py = y0 + ty * RPT + j;
        if (px < W && py < H) {
            const size_t gi = plane + (size_t)py * W + px;
            const float p1 = EXPO ? expose(img1, (size_t)H * W, (size_t)py * W + px, expo_coef(E, blockIdx.z)) : img1[gi];
            const float p2 = img2[gi];
            float out = c[0][j];
            out += p1 * 2.0f * c[1][j];
            out += p2 * c[2][j];
            if (CONST_DL) {
                const float d = p1 - p2;
                out += l1_scale * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
            }
            dL_dimg1[gi] = (MASK && !mask_bit(mk, py, px)) ? 0.0f : out;
        }
    }
}

template <bool CONST_DL>
__global__ void __launch_bounds__(ST)
ssim_backward_kernel(int H, int W, const float* __restrict__ img1, const float* __restrict__ img2,
                     const float* __restrict__ dL_dmap, const float* __restrict__ dm_dmu1,
                     const float* __restrict__ dm_dsigma1_sq, const float* __restrict__ dm_dsigma12,
                     float* __restrict__ dL_dimg1, float dl_const, float l1_scale) {
    pdl_enter();
    ssim_backward_tile<CONST_DL, false>(H, W, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12, dL_dimg1, dl_const, l1_scale,
                                        nullptr);
}

// backward of the exposed loss: dL/dout (3 planes) into dL_dout
__global__ void __launch_bounds__(ST)
ssim_loss_exposure_backward_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                                   const float* __restrict__ E, const float* __restrict__ dm_dmu1,
                                   const float* __restrict__ dm_dsigma1_sq, const float* __restrict__ dm_dsigma12,
                                   float* __restrict__ dL_dout, float dl_const, float l1_scale) {
    pdl_enter();
    ssim_backward_tile<true, true>(H, W, img, gt, nullptr, dm_dmu1, dm_dsigma1_sq, dm_dsigma12, dL_dout, dl_const, l1_scale, E);
}

// the masked loss (glic_l1_ssim_loss_masked): forward of the 3-plane image (EXPO: exposed by E) against gt, with the
// fixed-order (FIXED) or atomic loss sum, and its backward (dL/dimg, or with EXPO dL/dout for exposure_mix_kernel)
template <bool EXPO, bool FIXED>
__global__ void __launch_bounds__(ST)
ssim_loss_masked_forward_kernel(int H, int W, float C1, float C2, const float* __restrict__ img, const float* __restrict__ gt,
                                const float* __restrict__ E, MaskView mk, float* __restrict__ dm_dmu1, float* __restrict__ dm_dsigma1_sq,
                                float* __restrict__ dm_dsigma12, float lambda_dssim, float inv_n, float* __restrict__ loss) {
    pdl_enter();
    ssim_forward_tile<true, EXPO, FIXED, true>(H, W, C1, C2, img, gt, nullptr, dm_dmu1, dm_dsigma1_sq, dm_dsigma12, lambda_dssim, inv_n,
                                               loss, E, mk);
}

template <bool EXPO>
__global__ void __launch_bounds__(ST)
ssim_loss_masked_backward_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt, const float* __restrict__ E,
                                 MaskView mk, const float* __restrict__ dm_dmu1, const float* __restrict__ dm_dsigma1_sq,
                                 const float* __restrict__ dm_dsigma12, float* __restrict__ dL_dout, float dl_const, float l1_scale) {
    pdl_enter();
    ssim_backward_tile<true, EXPO, true>(H, W, img, gt, nullptr, dm_dmu1, dm_dsigma1_sq, dm_dsigma12, dL_dout, dl_const, l1_scale, E, mk);
}

// glic_pack_mask: one warp per 32-column word of a row, its bits by ballot; the valid pixels counted in integers (exact)
__global__ void __launch_bounds__(256)
pack_mask_kernel(int H, int W, int wpr, const uint8_t* __restrict__ valid, uint32_t* __restrict__ words, unsigned int* __restrict__ count) {
    const int lane = threadIdx.x & 31;
    const size_t n = (size_t)H * wpr, warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    unsigned int c = 0;
    for (size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n; w += warps) {   // warp-uniform
        const int y = (int)(w / wpr), x = (int)(w % wpr) * 32 + lane;
        const unsigned int bits = __ballot_sync(0xffffffffu, x < W && valid[(size_t)y * W + x] != 0);
        if (lane == 0) { words[w] = bits; c += __popc(bits); }
    }
    if (lane == 0 && c) atomicAdd(count, c);
}

constexpr int XT = 256;             // threads of the exposure mix kernel

// CTAs of the exposure mix kernel: a function of the frame size alone, so the partial sums (and their fixed-order total)
// are the same on every call and every replica
inline unsigned expo_blocks(size_t HW) { return (unsigned)std::min<size_t>((HW + XT - 1) / XT, (size_t)NUM_SMS * 4); }

// In place, per pixel: dL/dimg_k = sum_c E[k][c] * dL/dout_c.  Also the CTA's partial sums (float64, fixed order) of
//   dL/dE[k][c] = sum_px img_k * dL/dout_c (k < 3),   dL/dE[c][3] = sum_px dL/dout_c,
// stored at partials[12 * blockIdx.x + (4k + c)] (the layout of E).
__global__ void __launch_bounds__(XT)
exposure_mix_kernel(size_t HW, const float* __restrict__ img, const float* __restrict__ E, float* __restrict__ dL,
                    double* __restrict__ partials) {
    pdl_enter();
    __shared__ double red[XT / 32][12];
    float e[12];
#pragma unroll
    for (int j = 0; j < 12; ++j) e[j] = E[j];
    double acc[12];
#pragma unroll
    for (int j = 0; j < 12; ++j) acc[j] = 0.0;
    for (size_t i = (size_t)blockIdx.x * XT + threadIdx.x; i < HW; i += (size_t)gridDim.x * XT) {
        const float x[3] = {img[i], img[HW + i], img[2 * HW + i]};
        const float d[3] = {dL[i], dL[HW + i], dL[2 * HW + i]};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float g = e[4 * k] * d[0];
            g = fmaf(e[4 * k + 1], d[1], g);
            dL[k * HW + i] = fmaf(e[4 * k + 2], d[2], g);
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[4 * k + c] = fma((double)x[k], (double)d[c], acc[4 * k + c]);
            acc[4 * k + 3] += (double)d[k];
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < 12; ++j) {
        double v = acc[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[warp][j] = v;
    }
    __syncthreads();
    if (threadIdx.x < 12) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < XT / 32; ++w) t += red[w][threadIdx.x];
        partials[12 * (size_t)blockIdx.x + threadIdx.x] = t;
    }
}

struct ExpoBatch { int kf[EXPO_MAX_SLOTS]; };

// One exposure step per batch (torch_adam_delta, bias correction from the keyframe's own step count).  Thread (slot s,
// entry j); the first slot that holds a keyframe steps it with the batch gradient of keyframe_batch_grad.
// A set overflow word (the batch was skipped on the device) leaves E, m, v and t as they are.
__global__ void __launch_bounds__(EXPO_MAX_SLOTS * 12)
exposure_adam_kernel(int S, ExpoBatch batch, const float* __restrict__ slot_grads, float* __restrict__ E, float* __restrict__ m,
                     float* __restrict__ v, int* __restrict__ t, float lr, const unsigned int* __restrict__ skip) {
    if (*skip) return;
    const int s = threadIdx.x / 12, j = threadIdx.x % 12;
    const bool first = s < S && first_slot_of_keyframe(batch.kf, s);
    const int kf = first ? batch.kf[s] : 0;
    int step = 0;
    if (first) step = t[kf] + 1;
    __syncthreads();                                     // every thread has read its keyframe's old step count
    if (!first) return;
    const float g = keyframe_batch_grad(batch.kf, S, s, slot_grads, 12, j);
    const size_t i = 12 * (size_t)kf + j;
    E[i] = __fadd_rn(E[i], torch_adam_delta(g, m[i], v[i], lr, step));
    if (j == 0) t[kf] = step;
}

// out[0] = the G per-CTA loss partials summed in a fixed order (float64, lane-strided, then an xor butterfly): one warp
__global__ void __launch_bounds__(32) loss_finish_kernel(unsigned G, const float* __restrict__ partials, float* __restrict__ out) {
    pdl_enter();
    double s = 0.0;
    for (unsigned b = threadIdx.x; b < G; b += 32) s += (double)partials[b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) out[0] = (float)s;
}

}  // namespace

}  // namespace glic

using namespace glic;

// The planes of one launch run as gridDim.z, which is at most 65535: a larger B*CH (or one that overflows int) is refused
// before anything is enqueued, rather than failing at the launch after validation has passed.
static constexpr long long MAX_PLANES = 65535;

static bool planes_ok(long long planes, const char* what) {
    if (planes <= MAX_PLANES) return true;
    set_error(std::string(what) + ": " + std::to_string(planes) + " planes; at most 65535 per call");
    return false;
}

extern "C" int glic_fused_ssim(int B, int CH, int H, int W, float C1, float C2, const float* img1, const float* img2,
                               float* ssim_map, float* dm_dmu1, float* dm_dsigma1_sq, float* dm_dsigma12, void* stream) {
    if (B < 0 || CH < 0 || H <= 0 || W <= 0 || !img1 || !img2 || !ssim_map) { set_error("fused_ssim: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    if ((dm_dmu1 != nullptr) != (dm_dsigma1_sq != nullptr) || (dm_dmu1 != nullptr) != (dm_dsigma12 != nullptr)) {
        set_error("fused_ssim: partial maps must be all NULL or all non-NULL"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!planes_ok((long long)B * CH, "fused_ssim")) return GLIC_ERR_INVALID_ARGUMENT;
    if (B * CH == 0) return GLIC_OK;
    dim3 grid((W + SB - 1) / SB, (H + SB - 1) / SB, B * CH), block(ST);
    GLIC_LAUNCH_PDL(ssim_forward_kernel<false>, grid, block, 0, (cudaStream_t)stream, H, W, C1, C2, img1, img2, ssim_map, dm_dmu1,
                    dm_dsigma1_sq, dm_dsigma12, 0.f, 0.f, nullptr);
    return GLIC_OK;
}

extern "C" int glic_fused_ssim_backward(int B, int CH, int H, int W, float C1, float C2, const float* img1,
                                        const float* img2, const float* dL_dmap, const float* dm_dmu1,
                                        const float* dm_dsigma1_sq, const float* dm_dsigma12, float* dL_dimg1, void* stream) {
    (void)C1; (void)C2;
    if (B < 0 || CH < 0 || H <= 0 || W <= 0 || !img1 || !img2 || !dL_dmap || !dm_dmu1 || !dm_dsigma1_sq || !dm_dsigma12 || !dL_dimg1) {
        set_error("fused_ssim_backward: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!planes_ok((long long)B * CH, "fused_ssim_backward")) return GLIC_ERR_INVALID_ARGUMENT;
    if (B * CH == 0) return GLIC_OK;
    dim3 grid((W + SB - 1) / SB, (H + SB - 1) / SB, B * CH), block(ST);
    GLIC_LAUNCH_PDL(ssim_backward_kernel<false>, grid, block, 0, (cudaStream_t)stream, H, W, img1, img2, dL_dmap, dm_dmu1,
                    dm_dsigma1_sq, dm_dsigma12, dL_dimg1, 0.f, 0.f);
    return GLIC_OK;
}

extern "C" size_t glic_loss_scratch_bytes(int CH, int H, int W) { return sizeof(float) * 3 * (size_t)CH * H * W + 256; }

// partials == NULL: the loss term of every CTA is added atomically into loss_out; otherwise (G floats, G = the forward grid) it
// is stored per CTA and summed in a fixed order, so the loss value has the same bits on every run
// mask (3 planes, `valid` > 0 pixels set): the masked loss of glic_l1_ssim_loss_masked
static int l1_ssim_loss_impl(int CH, int H, int W, float lambda_dssim, const float* img, const float* gt, float* loss_out, float* dL_dimg,
                             void* scratch, size_t scratch_bytes, float* partials, cudaStream_t s, bool loss_zeroed = false,
                             const MaskView* mask = nullptr, uint32_t valid = 0) {
    if (CH <= 0 || H <= 0 || W <= 0 || !img || !gt || !loss_out || !scratch) { set_error("l1_ssim_loss: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!planes_ok(CH, "l1_ssim_loss")) return GLIC_ERR_INVALID_ARGUMENT;
    if (scratch_bytes < glic_loss_scratch_bytes(CH, H, W)) { set_error("l1_ssim_loss: scratch too small"); return GLIC_ERR_WORKSPACE; }
    const size_t N = (size_t)CH * H * W;
    float* d1 = static_cast<float*>(scratch);
    float* d2 = d1 + N;
    float* d3 = d2 + N;
    const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;     // loss_utils.h:130-131
    const float inv_n = (float)(1.0 / (double)(mask ? (size_t)CH * valid : N));     // N_w = CH * valid: today's 1/N when all are set
    dim3 grid((W + SB - 1) / SB, (H + SB - 1) / SB, CH), block(ST);
    if (!partials && !loss_zeroed) GLIC_CUDA_TRY(cudaMemsetAsync(loss_out, 0, sizeof(float), s));
    if (mask) {
        { StageTimer _t(GLIC_STAGE_LOSS_FWD, s);
        if (partials) GLIC_LAUNCH_PDL(ssim_loss_masked_forward_kernel<false, true>, grid, block, 0, s, H, W, C1, C2, img, gt, nullptr, *mask, d1, d2, d3, lambda_dssim, inv_n, partials);
        else GLIC_LAUNCH_PDL(ssim_loss_masked_forward_kernel<false, false>, grid, block, 0, s, H, W, C1, C2, img, gt, nullptr, *mask, d1, d2, d3, lambda_dssim, inv_n, loss_out); }
        if (partials) GLIC_LAUNCH_PDL(loss_finish_kernel, 1, 32, 0, s, grid.x * grid.y * grid.z, partials, loss_out);
        if (dL_dimg) {
            StageTimer _t(GLIC_STAGE_LOSS_BWD, s);
            GLIC_LAUNCH_PDL(ssim_loss_masked_backward_kernel<false>, grid, block, 0, s, H, W, img, gt, nullptr, *mask, d1, d2, d3, dL_dimg,
                            -lambda_dssim * inv_n, (1.0f - lambda_dssim) * inv_n);
        }
        return GLIC_OK;
    }
    { StageTimer _t(GLIC_STAGE_LOSS_FWD, s);
    if (partials) GLIC_LAUNCH_PDL(ssim_forward_kernel<true, true>, grid, block, 0, s, H, W, C1, C2, img, gt, nullptr, d1, d2, d3, lambda_dssim, inv_n, partials);
    else GLIC_LAUNCH_PDL(ssim_forward_kernel<true>, grid, block, 0, s, H, W, C1, C2, img, gt, nullptr, d1, d2, d3, lambda_dssim, inv_n, loss_out); }
    if (partials) GLIC_LAUNCH_PDL(loss_finish_kernel, 1, 32, 0, s, grid.x * grid.y * grid.z, partials, loss_out);
    if (dL_dimg) {
        StageTimer _t(GLIC_STAGE_LOSS_BWD, s);
        GLIC_LAUNCH_PDL(ssim_backward_kernel<true>, grid, block, 0, s, H, W, img, gt, nullptr, d1, d2, d3, dL_dimg, -lambda_dssim * inv_n,
                        (1.0f - lambda_dssim) * inv_n);
    }
    return GLIC_OK;
}

extern "C" int glic_l1_ssim_loss(int CH, int H, int W, float lambda_dssim, const float* img, const float* gt, float* loss_out,
                                 float* dL_dimg, void* scratch, size_t scratch_bytes, void* stream) {
    return l1_ssim_loss_impl(CH, H, W, lambda_dssim, img, gt, loss_out, dL_dimg, scratch, scratch_bytes, nullptr, (cudaStream_t)stream);
}

// scratch: the three partial maps (9 HW floats) | the mix kernel's float64 partial sums (12 per CTA)
static size_t expo_partials_offset(int H, int W) { return ((sizeof(float) * 9 * (size_t)H * W) + 255) & ~size_t(255); }

extern "C" size_t glic_loss_exposure_scratch_bytes(int H, int W) {
    if (H <= 0 || W <= 0) return 0;
    return expo_partials_offset(H, W) + sizeof(double) * 12 * (size_t)expo_blocks((size_t)H * W) + 256;
}

static int loss_exposure_impl(int H, int W, float lambda_dssim, const float* img, const float* gt, const float* E, float* loss_out,
                              float* dL_dimg, float* dL_dE, void* scratch, size_t scratch_bytes, float* partials, cudaStream_t s,
                              bool loss_zeroed = false, const MaskView* mask = nullptr, uint32_t valid = 0) {
    if (H <= 0 || W <= 0 || !img || !gt || !E || !loss_out || !scratch) { set_error("l1_ssim_loss_exposure: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    if ((dL_dimg == nullptr) != (dL_dE == nullptr)) {
        set_error("l1_ssim_loss_exposure: dL_dimg and dL_dE must be both NULL (loss only) or both non-NULL"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (scratch_bytes < glic_loss_exposure_scratch_bytes(H, W)) { set_error("l1_ssim_loss_exposure: scratch too small"); return GLIC_ERR_WORKSPACE; }
    const size_t HW = (size_t)H * W, N = 3 * HW;
    float* d1 = static_cast<float*>(scratch);
    float* d2 = d1 + N;
    float* d3 = d2 + N;
    double* expo_partials = reinterpret_cast<double*>(static_cast<char*>(scratch) + expo_partials_offset(H, W));
    const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
    const float inv_n = (float)(1.0 / (double)(mask ? 3 * (size_t)valid : N));
    dim3 grid((W + SB - 1) / SB, (H + SB - 1) / SB, 3), block(ST);
    if (!partials && !loss_zeroed) GLIC_CUDA_TRY(cudaMemsetAsync(loss_out, 0, sizeof(float), s));
    { StageTimer _t(GLIC_STAGE_LOSS_FWD, s);
    if (mask && partials) GLIC_LAUNCH_PDL(ssim_loss_masked_forward_kernel<true, true>, grid, block, 0, s, H, W, C1, C2, img, gt, E, *mask, d1, d2, d3, lambda_dssim, inv_n, partials);
    else if (mask) GLIC_LAUNCH_PDL(ssim_loss_masked_forward_kernel<true, false>, grid, block, 0, s, H, W, C1, C2, img, gt, E, *mask, d1, d2, d3, lambda_dssim, inv_n, loss_out);
    else if (partials) GLIC_LAUNCH_PDL(ssim_loss_exposure_forward_kernel<true>, grid, block, 0, s, H, W, C1, C2, img, gt, E, d1, d2, d3, lambda_dssim, inv_n, partials);
    else GLIC_LAUNCH_PDL(ssim_loss_exposure_forward_kernel<false>, grid, block, 0, s, H, W, C1, C2, img, gt, E, d1, d2, d3, lambda_dssim, inv_n, loss_out); }
    if (partials) GLIC_LAUNCH_PDL(loss_finish_kernel, 1, 32, 0, s, grid.x * grid.y * grid.z, partials, loss_out);
    if (dL_dimg) {
        StageTimer _t(GLIC_STAGE_LOSS_BWD, s);
        // under a mask dL/dout is +0 at masked pixels, so the mix below and dL/dE need no mask of their own
        if (mask) GLIC_LAUNCH_PDL(ssim_loss_masked_backward_kernel<true>, grid, block, 0, s, H, W, img, gt, E, *mask, d1, d2, d3, dL_dimg,
                                  -lambda_dssim * inv_n, (1.0f - lambda_dssim) * inv_n);
        else GLIC_LAUNCH_PDL(ssim_loss_exposure_backward_kernel, grid, block, 0, s, H, W, img, gt, E, d1, d2, d3, dL_dimg, -lambda_dssim * inv_n,
                             (1.0f - lambda_dssim) * inv_n);
        const unsigned G = expo_blocks(HW);
        GLIC_LAUNCH_PDL(exposure_mix_kernel, G, XT, 0, s, HW, img, E, dL_dimg, expo_partials);
        partials_finish_kernel<12><<<1, 12 * 32, 0, s>>>(G, expo_partials, dL_dE);
        GLIC_LAUNCH_CHECK();
    }
    return GLIC_OK;
}

extern "C" int glic_l1_ssim_loss_exposure(int H, int W, float lambda_dssim, const float* img, const float* gt, const float* E,
                                          float* loss_out, float* dL_dimg, float* dL_dE, void* scratch, size_t scratch_bytes,
                                          void* stream) {
    return loss_exposure_impl(H, W, lambda_dssim, img, gt, E, loss_out, dL_dimg, dL_dE, scratch, scratch_bytes, nullptr, (cudaStream_t)stream);
}

namespace glic {
// the native mapper's photometric loss (glic_l1_ssim_loss on 3 channels, or glic_l1_ssim_loss_exposure with E); partials
// (fixed_order_sums_bytes(H, W)) selects the fixed-order loss sum
int photometric_loss_sum(int H, int W, float lambda_dssim, const float* img, const float* gt, const float* E, float* loss, float* dL_dimg,
                         float* dL_dE, void* scratch, size_t scratch_bytes, void* partials, cudaStream_t s, bool loss_zeroed,
                         const MaskView* mask, uint32_t valid) {
    float* p = static_cast<float*>(partials);
    if (E) return loss_exposure_impl(H, W, lambda_dssim, img, gt, E, loss, dL_dimg, dL_dE, scratch, scratch_bytes, p, s, loss_zeroed, mask, valid);
    return l1_ssim_loss_impl(3, H, W, lambda_dssim, img, gt, loss, dL_dimg, scratch, scratch_bytes, p, s, loss_zeroed, mask, valid);
}

int launch_pack_mask(int H, int W, const uint8_t* valid, uint32_t* words, uint32_t* count, cudaStream_t s) {
    const size_t n = (size_t)H * mask_words_per_row(W);
    GLIC_CUDA_TRY(cudaMemsetAsync(count, 0, sizeof(uint32_t), s));
    pack_mask_kernel<<<(unsigned)std::min<size_t>((n + 7) / 8, (size_t)NUM_SMS * 8), 256, 0, s>>>(H, W, mask_words_per_row(W), valid, words,
                                                                                                  count);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}
}  // namespace glic

extern "C" int glic_mask_words_per_row(int W) { return W > 0 ? mask_words_per_row(W) : 0; }

extern "C" int glic_pack_mask(int H, int W, const uint8_t* valid, uint32_t* words, uint32_t* count, void* stream) {
    if (H <= 0 || W <= 0 || !valid || !words || !count) { set_error("pack_mask: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    return launch_pack_mask(H, W, valid, words, count, (cudaStream_t)stream);
}

// the masked loss's scratch: the exposed loss's | the fixed-order loss partials
extern "C" size_t glic_loss_masked_scratch_bytes(int H, int W) {
    if (H <= 0 || W <= 0) return 0;
    return glic_loss_exposure_scratch_bytes(H, W) + fixed_order_sums_bytes(H, W);
}

extern "C" int glic_l1_ssim_loss_masked(int H, int W, float lambda_dssim, const float* img, const float* gt, const float* E,
                                        const uint32_t* mask_words, int words_per_row, int mask_x0, uint32_t valid_count,
                                        int fixed_order, float* loss_out, float* dL_dimg, float* dL_dE, void* scratch,
                                        size_t scratch_bytes, void* stream) {
    if (H <= 0 || W <= 0 || !scratch || (E && ((dL_dimg == nullptr) != (dL_dE == nullptr)))) {
        set_error("l1_ssim_loss_masked: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (mask_words && (valid_count == 0 || (uint64_t)valid_count > (uint64_t)H * W || mask_x0 < 0 || words_per_row < 1 ||
                       (int64_t)mask_x0 + W > 32 * (int64_t)words_per_row)) {
        set_error("l1_ssim_loss_masked: bad mask view, or a mask with no valid pixel"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (scratch_bytes < glic_loss_masked_scratch_bytes(H, W)) { set_error("l1_ssim_loss_masked: scratch too small"); return GLIC_ERR_WORKSPACE; }
    const size_t lb = glic_loss_exposure_scratch_bytes(H, W);
    void* partials = fixed_order ? static_cast<char*>(scratch) + lb : nullptr;
    const MaskView mv{mask_words, words_per_row, mask_x0};
    return photometric_loss_sum(H, W, lambda_dssim, img, gt, E, loss_out, dL_dimg, dL_dE, scratch, lb, partials, (cudaStream_t)stream, false,
                                mask_words ? &mv : nullptr, valid_count);
}

namespace glic {
int launch_exposure_adam(int S, const int* kf_of_slot, const float* slot_grads, float* E, float* m, float* v, int* t, float lr,
                         const unsigned int* skip_flag, cudaStream_t s) {
    if (S < 1 || S > EXPO_MAX_SLOTS) { set_error("exposure_adam: bad batch size"); return GLIC_ERR_INVALID_ARGUMENT; }
    ExpoBatch b{};
    for (int q = 0; q < S; ++q) b.kf[q] = kf_of_slot[q];
    StageTimer _t(GLIC_STAGE_ADAM, s);
    exposure_adam_kernel<<<1, EXPO_MAX_SLOTS * 12, 0, s>>>(S, b, slot_grads, E, m, v, t, lr, skip_flag);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}
}  // namespace glic


// ---- evaluation metrics (evaluateVisualQuality, gaussian.cpp:756-760,795-799; loss_utils.h:35-39,84-127) --------------
namespace glic {
namespace {

// element i of the scored image: img exposed by E (optional, 3 channels; see expose()) and clamped to [0,1]
// (gaussian.cpp:756-757); HW = pixels per plane.  Evaluation and glic_mapper_render_camera both draw their images through it.
__device__ __forceinline__ float scored_pixel(const float* __restrict__ img, const float* __restrict__ E, size_t HW, size_t i) {
    float x = img[i];
    if (E) {
        const int c = (int)(i / HW);
        x = expose(img, HW, i - (size_t)c * HW, expo_coef(E, c));
    }
    return fminf(fmaxf(x, 0.f), 1.f);
}

// clamp both images to [0,1] (the image exposed first, scored_pixel) into scratch copies and accumulate the squared error.
// FIXED (the native mapper's deterministic option): each warp stores its float64 sum to acc2[global warp id] instead of adding it
// atomically; eval_finish_fixed_kernel sums the warps in a fixed order.
template <bool FIXED = false>
__global__ void __launch_bounds__(256)
eval_clamp_mse_kernel(size_t N, const float* __restrict__ img, const float* __restrict__ gt, float* __restrict__ a,
                      float* __restrict__ b, double* __restrict__ acc2, const float* __restrict__ E, size_t HW) {
    double se = 0.0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (size_t)gridDim.x * blockDim.x) {
        const float x = scored_pixel(img, E, HW, i);
        const float y = fminf(fmaxf(gt[i], 0.f), 1.f);
        a[i] = x; b[i] = y;
        const float d = x - y;
        se += (double)(d * d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    if (FIXED) { if ((threadIdx.x & 31) == 0) acc2[blockIdx.x * 8 + (threadIdx.x >> 5)] = se; }
    else if ((threadIdx.x & 31) == 0 && se != 0.0) atomicAdd(&acc2[0], se);
}

__global__ void __launch_bounds__(256)
scored_image_kernel(size_t N, const float* __restrict__ img, const float* __restrict__ E, size_t HW, float* __restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (size_t)gridDim.x * blockDim.x)
        out[i] = scored_pixel(img, E, HW, i);
}

template <bool FIXED = false>
__global__ void __launch_bounds__(256)
eval_sum_kernel(size_t N, const float* __restrict__ map, double* __restrict__ acc2) {
    double s = 0.0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (size_t)gridDim.x * blockDim.x) s += (double)map[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (FIXED) { if ((threadIdx.x & 31) == 0) acc2[blockIdx.x * 8 + (threadIdx.x >> 5)] = s; }
    else if ((threadIdx.x & 31) == 0) atomicAdd(&acc2[1], s);
}

// The masked evaluation (eval_psnr_ssim with a mask): the clamped pair is written with 0 in both images at masked pixels, and only
// used pixels enter the two sums (a masked one adds +0.0, which leaves a float64 sum's bits as they are).  W: the row length of
// the planes, HW = H * W.
template <bool FIXED>
__global__ void __launch_bounds__(256)
eval_clamp_mse_masked_kernel(size_t N, const float* __restrict__ img, const float* __restrict__ gt, float* __restrict__ a,
                             float* __restrict__ b, double* __restrict__ acc2, const float* __restrict__ E, size_t HW, int W, MaskView mk) {
    double se = 0.0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (size_t)gridDim.x * blockDim.x) {
        const size_t p = i % HW;
        const bool use = mask_bit(mk, (int)(p / W), (int)(p % W));
        const float x = use ? scored_pixel(img, E, HW, i) : 0.f;
        const float y = use ? fminf(fmaxf(gt[i], 0.f), 1.f) : 0.f;
        a[i] = x; b[i] = y;
        const float d = x - y;
        se += (double)(d * d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    if (FIXED) { if ((threadIdx.x & 31) == 0) acc2[blockIdx.x * 8 + (threadIdx.x >> 5)] = se; }
    else if ((threadIdx.x & 31) == 0 && se != 0.0) atomicAdd(&acc2[0], se);
}

template <bool FIXED>
__global__ void __launch_bounds__(256)
eval_sum_masked_kernel(size_t N, const float* __restrict__ map, double* __restrict__ acc2, size_t HW, int W, MaskView mk) {
    double s = 0.0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (size_t)gridDim.x * blockDim.x) {
        const size_t p = i % HW;
        s += mask_bit(mk, (int)(p / W), (int)(p % W)) ? (double)map[i] : 0.0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (FIXED) { if ((threadIdx.x & 31) == 0) acc2[blockIdx.x * 8 + (threadIdx.x >> 5)] = s; }
    else if ((threadIdx.x & 31) == 0) atomicAdd(&acc2[1], s);
}

// eval_finish_kernel on the per-warp partials of the FIXED forms: warps [0, n) of mse and of ssim, summed in a fixed order
__global__ void __launch_bounds__(32)
eval_finish_fixed_kernel(size_t N, unsigned n, const double* __restrict__ mse_part, const double* __restrict__ ssim_part, float* __restrict__ out2) {
    double a = 0.0, b = 0.0;
    for (unsigned i = threadIdx.x; i < n; i += 32) { a += mse_part[i]; b += ssim_part[i]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
    if (threadIdx.x == 0) {
        const float mse = (float)(a / (double)N);
        out2[0] = 10.0f * log10f(1.0f / mse);
        out2[1] = (float)(b / (double)N);
    }
}

__global__ void eval_finish_kernel(size_t N, const double* __restrict__ acc2, float* __restrict__ out2) {
    const float mse = (float)(acc2[0] / (double)N);
    out2[0] = 10.0f * log10f(1.0f / mse);          // loss_utils.h:35-39
    out2[1] = (float)(acc2[1] / (double)N);        // ssim_map.mean(), loss_utils.h:107
}

}  // namespace
}  // namespace glic

extern "C" size_t glic_eval_scratch_bytes(int CH, int H, int W) { return sizeof(float) * 3 * (size_t)CH * H * W + 256; }

namespace glic {
namespace {
// eval_psnr_ssim under a mask, after its checks: the masked clamp, the SSIM map of the masked pair, its masked sum; both means
// over the Nw = CH * valid used elements
int eval_psnr_ssim_masked(int CH, int H, int W, const float* img, const float* gt, const float* E, float* out2, void* scratch, void* stream,
                          void* fixed, MaskView mk, size_t Nw) {
    const size_t N = (size_t)CH * H * W, HW = (size_t)H * W;
    cudaStream_t s = (cudaStream_t)stream;
    double* acc2 = static_cast<double*>(scratch);
    float* a = reinterpret_cast<float*>(static_cast<char*>(scratch) + 256);
    float* b = a + N;
    float* map = b + N;
    const unsigned blocks = (unsigned)std::min<size_t>((N + 255) / 256, (size_t)NUM_SMS * 8);
    double* mse_part = fixed ? static_cast<double*>(fixed) : acc2;
    double* ssim_part = fixed ? mse_part + (size_t)NUM_SMS * 8 * 8 : acc2;
    if (!fixed) GLIC_CUDA_TRY(cudaMemsetAsync(acc2, 0, 2 * sizeof(double), s));
    if (fixed) eval_clamp_mse_masked_kernel<true><<<blocks, 256, 0, s>>>(N, img, gt, a, b, mse_part, E, HW, W, mk);
    else eval_clamp_mse_masked_kernel<false><<<blocks, 256, 0, s>>>(N, img, gt, a, b, acc2, E, HW, W, mk);
    GLIC_LAUNCH_CHECK();
    if (int e = glic_fused_ssim(1, CH, H, W, 0.01f * 0.01f, 0.03f * 0.03f, a, b, map, nullptr, nullptr, nullptr, stream)) return e;
    if (fixed) eval_sum_masked_kernel<true><<<blocks, 256, 0, s>>>(N, map, ssim_part, HW, W, mk);
    else eval_sum_masked_kernel<false><<<blocks, 256, 0, s>>>(N, map, acc2, HW, W, mk);
    GLIC_LAUNCH_CHECK();
    if (fixed) eval_finish_fixed_kernel<<<1, 32, 0, s>>>(Nw, blocks * 8, mse_part, ssim_part, out2);
    else eval_finish_kernel<<<1, 1, 0, s>>>(Nw, acc2, out2);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}
}  // namespace

int eval_psnr_ssim(int CH, int H, int W, const float* img, const float* gt, const float* E, float* out2, void* scratch,
                   size_t scratch_bytes, void* stream, void* fixed, const MaskView* mask, uint32_t valid) {
    if (CH <= 0 || H <= 0 || W <= 0 || !img || !gt || !out2 || !scratch || (E && CH != 3)) { set_error("eval_psnr_ssim: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (scratch_bytes < glic_eval_scratch_bytes(CH, H, W)) { set_error("eval_psnr_ssim: scratch too small"); return GLIC_ERR_WORKSPACE; }
    if (mask && valid == 0) { set_error("eval_psnr_ssim: a mask with no valid pixel"); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t N = (size_t)CH * H * W;
    if (mask) return eval_psnr_ssim_masked(CH, H, W, img, gt, E, out2, scratch, stream, fixed, *mask, (size_t)CH * valid);
    cudaStream_t s = (cudaStream_t)stream;
    double* acc2 = static_cast<double*>(scratch);                     // first 256 bytes: the two accumulators
    float* a = reinterpret_cast<float*>(static_cast<char*>(scratch) + 256);
    float* b = a + N;
    float* map = b + N;
    const unsigned blocks = (unsigned)std::min<size_t>((N + 255) / 256, (size_t)NUM_SMS * 8);
    if (fixed) {                                                      // per-warp partials, summed in a fixed order
        double* mse_part = static_cast<double*>(fixed);
        double* ssim_part = mse_part + (size_t)NUM_SMS * 8 * 8;
        eval_clamp_mse_kernel<true><<<blocks, 256, 0, s>>>(N, img, gt, a, b, mse_part, E, (size_t)H * W);
        GLIC_LAUNCH_CHECK();
        if (int e = glic_fused_ssim(1, CH, H, W, 0.01f * 0.01f, 0.03f * 0.03f, a, b, map, nullptr, nullptr, nullptr, stream)) return e;
        eval_sum_kernel<true><<<blocks, 256, 0, s>>>(N, map, ssim_part);
        GLIC_LAUNCH_CHECK();
        eval_finish_fixed_kernel<<<1, 32, 0, s>>>(N, blocks * 8, mse_part, ssim_part, out2);
        GLIC_LAUNCH_CHECK();
        return GLIC_OK;
    }
    GLIC_CUDA_TRY(cudaMemsetAsync(acc2, 0, 2 * sizeof(double), s));
    eval_clamp_mse_kernel<<<blocks, 256, 0, s>>>(N, img, gt, a, b, acc2, E, (size_t)H * W);
    GLIC_LAUNCH_CHECK();
    if (int e = glic_fused_ssim(1, CH, H, W, 0.01f * 0.01f, 0.03f * 0.03f, a, b, map, nullptr, nullptr, nullptr, stream)) return e;
    eval_sum_kernel<<<blocks, 256, 0, s>>>(N, map, acc2);
    GLIC_LAUNCH_CHECK();
    eval_finish_kernel<<<1, 1, 0, s>>>(N, acc2, out2);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_scored_image(int H, int W, const float* img, const float* E, float* out, cudaStream_t s) {
    const size_t N = (size_t)3 * H * W;
    scored_image_kernel<<<(unsigned)std::min<size_t>((N + 255) / 256, (size_t)NUM_SMS * 8), 256, 0, s>>>(N, img, E, (size_t)H * W, out);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

const float* eval_clamped(const void* scratch, int CH, int H, int W, int which) {
    return reinterpret_cast<const float*>(static_cast<const char*>(scratch) + 256) + (size_t)which * CH * H * W;
}
}  // namespace glic

extern "C" int glic_eval_psnr_ssim(int CH, int H, int W, const float* img, const float* gt, float* out2, void* scratch,
                                   size_t scratch_bytes, void* stream) {
    return eval_psnr_ssim(CH, H, W, img, gt, nullptr, out2, scratch, scratch_bytes, stream);
}

extern "C" size_t glic_eval_masked_scratch_bytes(int CH, int H, int W) {
    if (CH <= 0 || H <= 0 || W <= 0) return 0;
    return ((glic_eval_scratch_bytes(CH, H, W) + 255) & ~size_t(255)) + fixed_order_sums_bytes(H, W);
}

extern "C" int glic_eval_psnr_ssim_masked(int CH, int H, int W, const float* img, const float* gt, const float* E,
                                          const uint32_t* mask_words, int words_per_row, int mask_x0, uint32_t valid_count,
                                          int fixed_order, float* out2, void* scratch, size_t scratch_bytes, void* stream) {
    if (CH <= 0 || H <= 0 || W <= 0 || !scratch) { set_error("eval_psnr_ssim_masked: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (mask_words && (valid_count == 0 || (uint64_t)valid_count > (uint64_t)H * W || mask_x0 < 0 || words_per_row < 1 ||
                       (int64_t)mask_x0 + W > 32 * (int64_t)words_per_row)) {
        set_error("eval_psnr_ssim_masked: bad mask view, or a mask with no valid pixel"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (scratch_bytes < glic_eval_masked_scratch_bytes(CH, H, W)) { set_error("eval_psnr_ssim_masked: scratch too small"); return GLIC_ERR_WORKSPACE; }
    const size_t eb = (glic_eval_scratch_bytes(CH, H, W) + 255) & ~size_t(255);
    const MaskView mv{mask_words, words_per_row, mask_x0};
    return eval_psnr_ssim(CH, H, W, img, gt, E, out2, scratch, eb, stream, fixed_order ? static_cast<char*>(scratch) + eb : nullptr,
                          mask_words ? &mv : nullptr, valid_count);
}

namespace glic {
// the scratch of the fixed-order sums at H x W (3 channels): the loss's per-CTA partials or the evaluation's per-warp partials
size_t fixed_order_sums_bytes(int H, int W) {
    const size_t loss = sizeof(float) * 3 * (size_t)((W + SB - 1) / SB) * ((H + SB - 1) / SB);
    const size_t eval = sizeof(double) * 2 * (size_t)NUM_SMS * 8 * 8;
    return std::max(loss, eval) + 256;
}
}  // namespace glic

// preprocess_backward.cu -- per-Gaussian backward: 2-D gradients -> dL/d{mean3D, cov3D, dc, sh,
// scale, rotation}.
//
// Replaces computeCov2DCUDA + preprocessCUDA(bwd) + computeColorFromSH(bwd) + computeCov3D(bwd)
// (reference backward.cu:27-377) in ONE kernel, and the ten torch::zeros of
// rasterize_points.cu:192-201: every output row is written here (exact zeros for culled
// Gaussians).  Forward intermediates (cov3D, T) are recomputed from scale/rotation instead of
// being stored (24 B/Gaussian less state, and the inputs are read anyway).
//
// Two output forms (template COMPACT):
//   false: the reference's nine gradient tensors w.r.t. the ACTIVATED inputs (RasterizeGaussiansBackwardCUDA's contract);
//   true : the mapper's compact form (include/glic_b200.h "Native mapping host"): 11 geometric floats per Gaussian
//          w.r.t. the RAW parameters -- the sigmoid / exp / normalize chain rule (gaussian.cpp:147-175) applied here, with the
//          expressions of activations_backward_kernel -- written or ACCUMULATED over a rank's views.  dL/d(dc, sh-rest) are
//          not materialised: they are linear in the clamp-masked dL/dcolour (the render backward's output + the forward's
//          clamp bits) and are rebuilt inside the Adam kernel (model_step.cu).
//
// POSE (only with COMPACT; glic_mapper_enable_pose_refinement): the same pass also reduces the view's camera-pose gradient
// g = dL/d(rho, omega) of T_cw(delta) = Exp(delta) T_cw at delta = 0 (delta in the camera frame, translation first).  With
// W the rotation block of `view`, per visible Gaussian i
//     g_view,i = dL/dp_view through J (dtx, dty, dtz) + W * (the projection adjoint, a world-frame vector),
//     G_i      = J_i^T dL/dT_i  (= dL/dW through T = J W),
//     d_i      = the SH view-direction adjoint (world frame; zero when M = 0, as the colour backward is skipped then),
//     dL/drho   = sum_i g_view,i + W d_i                        (the camera centre moves by -W^T rho)
//     dL/domega = sum_i p_view,i x g_view,i + sum_c W[:,c] x G_i[:,c]   (the camera centre does not move under omega).
// Each Gaussian forms its six terms in fp32; the CTA adds them in float64 in a fixed order (warp shuffles, then the four
// warps in order) and writes one partial per CTA; partials_finish_kernel adds the partials in a fixed order.  No atomics:
// two runs give the same bits.
//
// POSE_ONLY (with POSE, without DENS; glic_mapper_align): the six pose floats and nothing per row.  The same pass, the same
// fp32 expressions for pose6 and the same fixed-order reduction, but no row of the compact block is written, the scale /
// rotation chain rule and the opacity activation are not formed, and neither their inputs (opacity, dL/dopacity, the raw
// rotation) nor the densification statistics are touched.  Given the same render-backward outputs its pose gradient is the
// POSE form's, bit for bit.  Chosen by CompactGrads with null row pointers (g_xyz == NULL) and pose partials.
//
// DENS (only with COMPACT; glic_mapper_enable_densification): the same pass writes (or, for the later views of a rank, adds)
// the view's densification statistics of each row: |(dL/dmean2D.x, dL/dmean2D.y)| and 1 when it is visible, 0 and 0 when it is
// culled.  One thread owns a row, so there are no atomics.
#include "geom_math.cuh"
#include "sh_math.cuh"
#include "warp_rows.cuh"

namespace glic {

constexpr int PB_THREADS = 128;

template <bool COMPACT, bool POSE = false, bool DENS = false, bool POSE_ONLY = false>
__global__ void __launch_bounds__(PB_THREADS)
preprocess_backward_kernel(int P, int D, int M, const float* __restrict__ means, const float* __restrict__ scales,
                           float mod, const float4* __restrict__ rots, const float* __restrict__ sh, ViewParams vp,
                           const int* __restrict__ radii, const uint8_t* __restrict__ clamped, float lambda_erank,
                           const float* __restrict__ dL_dmean2D, const float* __restrict__ dL_dconic,
                           const float* __restrict__ dL_dcolors, float* __restrict__ dL_dmeans3D,
                           float* __restrict__ dL_dcov3D, float* __restrict__ dL_ddc, float* __restrict__ dL_dsh,
                           float* __restrict__ dL_dscales, float4* __restrict__ dL_drots, CompactGrads cg) {
    pdl_enter();
    __shared__ float s_view[16], s_proj[16], s_cam[3];
    __shared__ __align__(16) float s_sh[PB_THREADS / 32][32 * SH_ROW_MAX];    // SH rows in, dL/dSH rows out
    static_assert(COMPACT || !POSE, "the pose gradient is a compact-form output");
    static_assert(COMPACT || !DENS, "the densification statistics are a compact-form output");
    static_assert(!POSE_ONLY || (POSE && !DENS), "the pose-only form writes the pose partials alone");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 16) s_view[tid] = vp.view[tid];
    else if (tid < 32) s_proj[tid - 16] = vp.proj[tid - 16];
    else if (tid < 35) s_cam[tid - 32] = vp.campos[tid - 32];
    __syncthreads();
    const int idx = blockIdx.x * blockDim.x + tid;
    const int K = 3 * M;
    const bool staged = K > 0 && K <= SH_ROW_MAX && sh != nullptr;
    const int wfirst = blockIdx.x * blockDim.x + warp * 32;
    const int wcnt = min(32, P - wfirst);
    if (wcnt <= 0 && !POSE) return;                                // whole warp beyond P (warp-uniform; POSE: stays for the CTA sum)
    float* slab = s_sh[warp];
    if (staged && D > 0 && (!POSE || wcnt > 0)) warp_load_rows(sh, (size_t)wfirst, wcnt, K, slab, lane);
    float pose6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};               // POSE: this Gaussian's dL/d(rho, omega)
    // dL/dSH row of this thread: shared-memory slab (written back coalesced below) or global memory
    float* dsh = staged ? (slab + lane * K) : (dL_dsh + (size_t)(idx < P ? idx : 0) * K);
    const bool visible = idx < P && radii[idx] > 0;
    if (!visible) {
        if (idx < P) {
            if (COMPACT) {
                if (!POSE_ONLY && !cg.accumulate) {
#pragma unroll
                    for (int k = 0; k < 3; ++k) { cg.g_xyz[3 * idx + k] = 0.f; cg.g_scale[3 * idx + k] = 0.f; }
                    cg.g_rot[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
                    cg.g_opacity[idx] = 0.f;
                    if constexpr (DENS) { cg.dens_norm[idx] = 0.f; cg.dens_count[idx] = 0.f; }
                }
            } else {
#pragma unroll
                for (int k = 0; k < 3; ++k) { dL_dmeans3D[3 * idx + k] = 0.f; dL_ddc[3 * idx + k] = 0.f; dL_dscales[3 * idx + k] = 0.f; }
#pragma unroll
                for (int k = 0; k < 6; ++k) dL_dcov3D[6 * idx + k] = 0.f;
                dL_drots[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        if (!COMPACT && (idx < P || staged)) for (int k = 0; k < K; ++k) dsh[k] = 0.f;
    } else {
    const float px = means[3 * idx], py = means[3 * idx + 1], pz = means[3 * idx + 2];
    const float s0 = scales[3 * idx], s1 = scales[3 * idx + 1], s2 = scales[3 * idx + 2];
    const float4 q = rots[idx];
    Cov3 c3;
    cov3d_from_scale_rot(s0, s1, s2, mod, q, c3);
    Cov2 c2;
    cov2d_project(px, py, pz, s_view, vp.focal_x, vp.focal_y, vp.limx_neg, vp.limx_pos, vp.limy_neg, vp.limy_pos, c3.c, c2);
    const float fx = vp.focal_x, fy = vp.focal_y;
    const float* v = s_view;

    // ---- EWA backward (backward.cu:138-255) -------------------------------------------------
    const float x_grad_mul = (c2.txtz < vp.limx_neg || c2.txtz > vp.limx_pos) ? 0.f : 1.f;
    const float y_grad_mul = (c2.tytz < vp.limy_neg || c2.tytz > vp.limy_pos) ? 0.f : 1.f;
    const float tz = c2.tz, tcx = c2.lx * tz, tcy = c2.ly * tz;
    const float a = c2.a, b = c2.b, c = c2.c;
    const float gxx = dL_dconic[4 * idx], gxy = dL_dconic[4 * idx + 1], gyy = dL_dconic[4 * idx + 3];
    const float denom = a * c - b * b;
    const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
    float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
    const float T00 = c2.T00, T01 = c2.T01, T02 = c2.T02, T10 = c2.T10, T11 = c2.T11, T12 = c2.T12;
    float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (denom2inv != 0.f) {
        dL_da = denom2inv * (-c * c * gxx + 2 * b * c * gxy + (denom - a * c) * gyy);
        dL_dc = denom2inv * (-a * a * gyy + 2 * a * b * gxy + (denom - a * c) * gxx);
        dL_db = denom2inv * 2 * (b * c * gxx - (denom + 2 * b * b) * gxy + a * b * gyy);
        dcov[0] = (T00 * T00 * dL_da + T00 * T10 * dL_db + T10 * T10 * dL_dc);
        dcov[3] = (T01 * T01 * dL_da + T01 * T11 * dL_db + T11 * T11 * dL_dc);
        dcov[5] = (T02 * T02 * dL_da + T02 * T12 * dL_db + T12 * T12 * dL_dc);
        dcov[1] = 2 * T00 * T01 * dL_da + (T00 * T11 + T01 * T10) * dL_db + 2 * T10 * T11 * dL_dc;
        dcov[2] = 2 * T00 * T02 * dL_da + (T00 * T12 + T02 * T10) * dL_db + 2 * T10 * T12 * dL_dc;
        dcov[4] = 2 * T02 * T01 * dL_da + (T01 * T12 + T02 * T11) * dL_db + 2 * T11 * T12 * dL_dc;
    }
    if (!COMPACT) {
#pragma unroll
        for (int k = 0; k < 6; ++k) dL_dcov3D[6 * idx + k] = dcov[k];
    }
    const float* V = c3.c;
    // rows of T^T Vrk products: r0k = sum_m T0m * Vrk[k][m], r1k = sum_m T1m * Vrk[k][m]
    const float r00 = T00 * V[0] + T01 * V[1] + T02 * V[2], r10 = T10 * V[0] + T11 * V[1] + T12 * V[2];
    const float r01 = T00 * V[1] + T01 * V[3] + T02 * V[4], r11 = T10 * V[1] + T11 * V[3] + T12 * V[4];
    const float r02 = T00 * V[2] + T01 * V[4] + T02 * V[5], r12 = T10 * V[2] + T11 * V[4] + T12 * V[5];
    const float dT00 = 2 * r00 * dL_da + r10 * dL_db, dT01 = 2 * r01 * dL_da + r11 * dL_db, dT02 = 2 * r02 * dL_da + r12 * dL_db;
    const float dT10 = 2 * r10 * dL_dc + r00 * dL_db, dT11 = 2 * r11 * dL_dc + r01 * dL_db, dT12 = 2 * r12 * dL_dc + r02 * dL_db;
    const float dJ00 = v[0] * dT00 + v[4] * dT01 + v[8] * dT02;
    const float dJ02 = v[2] * dT00 + v[6] * dT01 + v[10] * dT02;
    const float dJ11 = v[1] * dT10 + v[5] * dT11 + v[9] * dT12;
    const float dJ12 = v[2] * dT10 + v[6] * dT11 + v[10] * dT12;
    const float itz = 1.f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
    const float dtx = x_grad_mul * -fx * itz2 * dJ02;
    const float dty = y_grad_mul * -fy * itz2 * dJ12;
    const float dtz = -fx * itz2 * dJ00 - fy * itz2 * dJ11 + (2 * fx * tcx) * itz3 * dJ02 + (2 * fy * tcy) * itz3 * dJ12;
    float dmx = v[0] * dtx + v[1] * dty + v[2] * dtz;
    float dmy = v[4] * dtx + v[5] * dty + v[6] * dtz;
    float dmz = v[8] * dtx + v[9] * dty + v[10] * dtz;

    // ---- projection term (backward.cu:339-350) ------------------------------------------------
    {
        const float* pr = s_proj;
        const float hx = xform_row(pr, 0, px, py, pz), hy = xform_row(pr, 1, px, py, pz), hw = xform_row(pr, 3, px, py, pz);
        const float m_w = 1.0f / (hw + 0.0000001f);
        const float mul1 = hx * m_w * m_w, mul2 = hy * m_w * m_w;
        const float g2x = dL_dmean2D[3 * idx], g2y = dL_dmean2D[3 * idx + 1];
        dmx += (pr[0] * m_w - pr[3] * mul1) * g2x + (pr[1] * m_w - pr[3] * mul2) * g2y;
        dmy += (pr[4] * m_w - pr[7] * mul1) * g2x + (pr[5] * m_w - pr[7] * mul2) * g2y;
        dmz += (pr[8] * m_w - pr[11] * mul1) * g2x + (pr[9] * m_w - pr[11] * mul2) * g2y;
    }

    // ---- SH backward (computeColorFromSH's adjoint, backward.cu:27-136; factored as in sh_math.cuh).  Like the
    // reference (`if (shs)`, backward.cu:352) the whole colour backward -- dL/ddc included -- is skipped when no SH-rest
    // tensor is bound (M == 0). ----------------------------------------------------------------------------------
    float dRGB[3] = {0.f, 0.f, 0.f};
    float dsx = 0.f, dsy = 0.f, dsz = 0.f;                         // POSE: the view-direction adjoint d_i
    if (sh == nullptr) {
        if (!COMPACT) { dL_ddc[3 * idx] = 0.f; dL_ddc[3 * idx + 1] = 0.f; dL_ddc[3 * idx + 2] = 0.f; }
    } else {
        const float ox = px - s_cam[0], oy = py - s_cam[1], oz = pz - s_cam[2];
        const float sum2 = ox * ox + oy * oy + oz * oz;
        const float inv = 1.0f / sqrtf(sum2);
        const float x = ox * inv, y = oy * inv, z = oz * inv;
        const unsigned cb = clamped[idx];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) dRGB[ch] = (cb >> ch) & 1u ? 0.f : dL_dcolors[3 * idx + ch];
        if (!COMPACT) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) dL_ddc[3 * idx + ch] = kSH0 * dRGB[ch];
        }
        float ddx = 0.f, ddy = 0.f, ddz = 0.f;   // dL/d(dir)
        if (D > 0) {
            float sv[SH_ROW_MAX];                                  // input row -> registers (the slab row is reused for the output)
            if (staged) {
#pragma unroll
                for (int k = 0; k < SH_ROW_MAX; ++k) sv[k] = k < K ? slab[lane * K + k] : 0.f;
            } else {
#pragma unroll
                for (int k = 0; k < SH_ROW_MAX; ++k) sv[k] = k < K ? sh[(size_t)idx * K + k] : 0.f;
            }
            const int nb = sh_rest_count(D);
            float bs[15], w[15];
            sh_basis(D, x, y, z, bs);
#pragma unroll
            for (int k = 0; k < 15; ++k) {
                if (k < nb) {
                    w[k] = sv[3 * k] * dRGB[0] + sv[3 * k + 1] * dRGB[1] + sv[3 * k + 2] * dRGB[2];
                    if (!COMPACT) {
                        dsh[3 * k + 0] = bs[k] * dRGB[0];
                        dsh[3 * k + 1] = bs[k] * dRGB[1];
                        dsh[3 * k + 2] = bs[k] * dRGB[2];
                    }
                } else {
                    w[k] = 0.f;
                }
            }
            if (!COMPACT) for (int k = nb; k < M; ++k) { dsh[3 * k] = 0.f; dsh[3 * k + 1] = 0.f; dsh[3 * k + 2] = 0.f; }
            sh_dir_gradient(D, x, y, z, w, ddx, ddy, ddz);
        } else if (!COMPACT) {
            for (int k = 0; k < 3 * M; ++k) dsh[k] = 0.f;
        }
        // adjoint of dir = o / |o| (auxiliary.h:103-114): (I |o|^2 - o o^T) / |o|^3 applied to dL/d(dir)
        const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
        dmx += ((+sum2 - ox * ox) * ddx - oy * ox * ddy - oz * ox * ddz) * invsum32;
        dmy += (-ox * oy * ddx + (sum2 - oy * oy) * ddy - oz * oy * ddz) * invsum32;
        dmz += (-ox * oz * ddx - oy * oz * ddy + (sum2 - oz * oz) * ddz) * invsum32;
        if constexpr (POSE) {
            dsx = ((+sum2 - ox * ox) * ddx - oy * ox * ddy - oz * ox * ddz) * invsum32;
            dsy = (-ox * oy * ddx + (sum2 - oy * oy) * ddy - oz * oy * ddz) * invsum32;
            dsz = (-ox * oz * ddx - oy * oz * ddy + (sum2 - oz * oz) * ddz) * invsum32;
        }
    }
    if constexpr (POSE) {
        // the projection adjoint of the block above, rotated into the view frame, plus the part through J
        const float* pr = s_proj;
        const float hx = xform_row(pr, 0, px, py, pz), hy = xform_row(pr, 1, px, py, pz), hw = xform_row(pr, 3, px, py, pz);
        const float m_w = 1.0f / (hw + 0.0000001f);
        const float mul1 = hx * m_w * m_w, mul2 = hy * m_w * m_w;
        const float g2x = dL_dmean2D[3 * idx], g2y = dL_dmean2D[3 * idx + 1];
        const float pjx = (pr[0] * m_w - pr[3] * mul1) * g2x + (pr[1] * m_w - pr[3] * mul2) * g2y;
        const float pjy = (pr[4] * m_w - pr[7] * mul1) * g2x + (pr[5] * m_w - pr[7] * mul2) * g2y;
        const float pjz = (pr[8] * m_w - pr[11] * mul1) * g2x + (pr[9] * m_w - pr[11] * mul2) * g2y;
        // W[r][c] = v[4c + r]; (W x)_r = v[r] x0 + v[4 + r] x1 + v[8 + r] x2
        const float ux = pjx + dsx, uy = pjy + dsy, uz = pjz + dsz;
        const float gvx = dtx + (v[0] * pjx + v[4] * pjy + v[8] * pjz);
        const float gvy = dty + (v[1] * pjx + v[5] * pjy + v[9] * pjz);
        const float gvz = dtz + (v[2] * pjx + v[6] * pjy + v[10] * pjz);
        pose6[0] = dtx + (v[0] * ux + v[4] * uy + v[8] * uz);
        pose6[1] = dty + (v[1] * ux + v[5] * uy + v[9] * uz);
        pose6[2] = dtz + (v[2] * ux + v[6] * uy + v[10] * uz);
        const float vx = xform_row(v, 0, px, py, pz), vy = xform_row(v, 1, px, py, pz), vz = tz;   // p_view
        // G = J^T dT with J = [[fx/tz, 0, -fx lx/tz], [0, fy/tz, -fy ly/tz]] (the clamped lx, ly of cov2d_project)
        const float J00 = fx * itz, J11 = fy * itz, J02 = -fx * c2.lx * itz, J12 = -fy * c2.ly * itz;
        const float dT[2][3] = {{dT00, dT01, dT02}, {dT10, dT11, dT12}};
        float wx = vy * gvz - vz * gvy, wy = vz * gvx - vx * gvz, wz = vx * gvy - vy * gvx;
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) {
            const float G0 = J00 * dT[0][cc], G1 = J11 * dT[1][cc], G2 = J02 * dT[0][cc] + J12 * dT[1][cc];
            const float a0 = v[4 * cc], a1 = v[4 * cc + 1], a2 = v[4 * cc + 2];
            wx += a1 * G2 - a2 * G1;
            wy += a2 * G0 - a0 * G2;
            wz += a0 * G1 - a1 * G0;
        }
        pose6[3] = wx; pose6[4] = wy; pose6[5] = wz;
    }

    // ---- cov3D backward (computeCov3D's adjoint, backward.cu:257-310): Sigma = M^T M, M = S R ------------------------
    float ds[3];
    float4 dq;
    {
        const float sv[3] = {mod * s0, mod * s1, mod * s2};
        const float dS[9] = {dcov[0], 0.5f * dcov[1], 0.5f * dcov[2], 0.5f * dcov[1], dcov[3], 0.5f * dcov[4],
                             0.5f * dcov[2], 0.5f * dcov[4], dcov[5]};
        float dMt[9];   // dMt[3j+k] = dL_dM[k][j] with dL_dM = 2*M*dL_dSigma (column-major sense)
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int j = 0; j < 3; ++j)
                dMt[3 * j + k] = 2.f * c3.M[j] * dS[3 * k] + 2.f * c3.M[3 + j] * dS[3 * k + 1] + 2.f * c3.M[6 + j] * dS[3 * k + 2];
#pragma unroll
        for (int j = 0; j < 3; ++j) ds[j] = c3.R[j] * dMt[3 * j] + c3.R[3 + j] * dMt[3 * j + 1] + c3.R[6 + j] * dMt[3 * j + 2];
        float G[9];     // G[3i+j] = dL/dR_ij of the rotation matrix R(q): row j of dL_dM scaled by s_j, transposed
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
            for (int k = 0; k < 3; ++k) G[3 * k + j] = dMt[3 * j + k] * sv[j];
        dq = quat_gradient(q, G);
        if (lambda_erank > 0.f) {   // effective-rank regulariser, backward.cu:358-375 (off in every shipped config)
            const float s1s1 = s0 * s0, s2s2 = s1 * s1, s3s3 = s2 * s2, sum = s1s1 + s2s2 + s3s3;
            const float q1 = s0 / sum, q2 = s1 / sum, q3 = s2 / sum;
            const float erank = expf(-q1 * logf(q1) - q2 * logf(q2) - q3 * logf(q3));
            if (-log((double)erank - 1 + 1e-5) > 0) {
                const float f = (float)(erank / (erank - 1 + 1e-5));
                const float e1 = f * (-logf(q1) - 1), e2 = f * (-logf(q2) - 1), e3 = f * (-logf(q3) - 1);
                const float le = lambda_erank * 2.f / (sum * sum);
                ds[0] += le * s0 * (e1 * (s2s2 + s3s3) - e2 * s2s2 - e3 * s3s3);
                ds[1] += le * s1 * (-e1 * s1s1 + e2 * (s1s1 + s3s3) - e3 * s3s3);
                ds[2] += le * s2 * (-e1 * s1s1 - e2 * s2s2 + e3 * (s1s1 + s2s2));
            }
            ds[2] += 1.f;           // backward.cu:374 adds this unconditionally; kept for parity
        }
    }
    if (!COMPACT) {
        dL_dmeans3D[3 * idx] = dmx; dL_dmeans3D[3 * idx + 1] = dmy; dL_dmeans3D[3 * idx + 2] = dmz;
        dL_dscales[3 * idx] = ds[0]; dL_dscales[3 * idx + 1] = ds[1]; dL_dscales[3 * idx + 2] = ds[2];
        dL_drots[idx] = dq;
    } else if constexpr (!POSE_ONLY) {
        // chain rule of the activations (same expressions as activations_backward_kernel, model_step.cu):
        //   sigmoid' = o (1 - o);  exp' = exp;  normalize: (g - q (q.g)) / |r|
        const float o = cg.opacity[idx];
        const float g_o = cg.dL_dopacity[idx] * (o * (1.0f - o));
        const float g_s0 = ds[0] * s0, g_s1 = ds[1] * s1, g_s2 = ds[2] * s2;
        const float4 r = cg.rot_raw[idx];
        const float nn = sqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
        float4 g_r;
        if (nn > 1e-12f) {
            const float inv = 1.0f / nn;
            const float4 qn = make_float4(r.x * inv, r.y * inv, r.z * inv, r.w * inv);
            const float qg = qn.x * dq.x + qn.y * dq.y + qn.z * dq.z + qn.w * dq.w;
            g_r = make_float4((dq.x - qn.x * qg) * inv, (dq.y - qn.y * qg) * inv, (dq.z - qn.z * qg) * inv, (dq.w - qn.w * qg) * inv);
        } else {
            const float inv = 1.0f / 1e-12f;
            g_r = make_float4(dq.x * inv, dq.y * inv, dq.z * inv, dq.w * inv);
        }
        if (cg.accumulate) {
            cg.g_xyz[3 * idx] += dmx; cg.g_xyz[3 * idx + 1] += dmy; cg.g_xyz[3 * idx + 2] += dmz;
            cg.g_scale[3 * idx] += g_s0; cg.g_scale[3 * idx + 1] += g_s1; cg.g_scale[3 * idx + 2] += g_s2;
            const float4 old = cg.g_rot[idx];
            cg.g_rot[idx] = make_float4(old.x + g_r.x, old.y + g_r.y, old.z + g_r.z, old.w + g_r.w);
            cg.g_opacity[idx] += g_o;
        } else {
            cg.g_xyz[3 * idx] = dmx; cg.g_xyz[3 * idx + 1] = dmy; cg.g_xyz[3 * idx + 2] = dmz;
            cg.g_scale[3 * idx] = g_s0; cg.g_scale[3 * idx + 1] = g_s1; cg.g_scale[3 * idx + 2] = g_s2;
            cg.g_rot[idx] = g_r;
            cg.g_opacity[idx] = g_o;
        }
        if constexpr (DENS) {
            const float g2x = dL_dmean2D[3 * idx], g2y = dL_dmean2D[3 * idx + 1];
            const float nrm = sqrtf(g2x * g2x + g2y * g2y);
            if (cg.accumulate) { cg.dens_norm[idx] += nrm; cg.dens_count[idx] += 1.0f; }
            else { cg.dens_norm[idx] = nrm; cg.dens_count[idx] = 1.0f; }
        }
    }
    }   // visible
    if (!COMPACT && staged) warp_store_rows(dL_dsh, (size_t)wfirst, wcnt, K, slab, lane);
    if constexpr (POSE) {
        __shared__ double s_pose[PB_THREADS / 32][6];
        double r6[6];
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            r6[j] = (double)pose6[j];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) r6[j] += __shfl_down_sync(0xffffffffu, r6[j], o);
        }
        if (lane == 0) {
#pragma unroll
            for (int j = 0; j < 6; ++j) s_pose[warp][j] = r6[j];
        }
        __syncthreads();
        if (tid < 6) {
            double acc = 0.0;
#pragma unroll
            for (int w = 0; w < PB_THREADS / 32; ++w) acc += s_pose[w][tid];
            cg.pose_partials[6 * (size_t)blockIdx.x + tid] = acc;
        }
    }
}

int launch_preprocess_backward(int P, int D, int M, const float* means, const float* scales, float mod,
                               const float* rots, const float* sh, const ViewParams& vp, const int* radii, GeomState g,
                               float lambda_erank, const float* dL_dmean2D, const float* dL_dconic,
                               const float* dL_dcolors, float* dL_dmeans3D, float* dL_dcov3D, float* dL_ddc,
                               float* dL_dsh, float* dL_dscales, float* dL_drots, cudaStream_t s) {
    GLIC_LAUNCH_PDL(preprocess_backward_kernel<false>, (P + PB_THREADS - 1) / PB_THREADS, PB_THREADS, 0, s,
                    P, D, M, means, scales, mod, reinterpret_cast<const float4*>(rots), sh, vp, radii, g.clamped, lambda_erank,
                    dL_dmean2D, dL_dconic, dL_dcolors, dL_dmeans3D, dL_dcov3D, dL_ddc, dL_dsh, dL_dscales,
                    reinterpret_cast<float4*>(dL_drots), CompactGrads{});
    return GLIC_OK;
}

template <bool DENS, bool POSE_ONLY = false>
static int launch_compact(int P, int D, int M, const float* means, const float* scales, float mod, const float* rots, const float* sh,
                   const ViewParams& vp, const int* radii, GeomState g, const float* dL_dmean2D, const float* dL_dconic,
                   const float* dL_dcolors, const CompactGrads& cg, cudaStream_t s) {
    const unsigned blocks = (P + PB_THREADS - 1) / PB_THREADS;
    if (cg.pose_partials) {
        GLIC_LAUNCH_PDL(preprocess_backward_kernel<true, true, DENS, POSE_ONLY>, blocks, PB_THREADS, 0, s,
                        P, D, M, means, scales, mod, reinterpret_cast<const float4*>(rots), sh, vp, radii, g.clamped, 0.0f,
                        dL_dmean2D, dL_dconic, dL_dcolors, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, cg);
        partials_finish_kernel<6><<<1, 6 * 32, 0, s>>>(blocks, cg.pose_partials, cg.pose_grad);
        GLIC_LAUNCH_CHECK();
        return GLIC_OK;
    }
    GLIC_LAUNCH_PDL(preprocess_backward_kernel<true, false, DENS>, (P + PB_THREADS - 1) / PB_THREADS, PB_THREADS, 0, s,
                    P, D, M, means, scales, mod, reinterpret_cast<const float4*>(rots), sh, vp, radii, g.clamped, 0.0f,
                    dL_dmean2D, dL_dconic, dL_dcolors, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, cg);
    return GLIC_OK;
}

int launch_preprocess_backward_compact(int P, int D, int M, const float* means, const float* scales, float mod,
                                       const float* rots, const float* sh, const ViewParams& vp, const int* radii, GeomState g,
                                       const float* dL_dmean2D, const float* dL_dconic, const float* dL_dcolors,
                                       const CompactGrads& cg, cudaStream_t s) {
    if (!cg.g_xyz) {                                               // the pose gradient alone (POSE_ONLY)
        if (!cg.pose_partials || !cg.pose_grad || cg.dens_norm) { set_error("backward_compact: the pose-only form takes the pose outputs alone"); return GLIC_ERR_INVALID_ARGUMENT; }
        return launch_compact<false, true>(P, D, M, means, scales, mod, rots, sh, vp, radii, g, dL_dmean2D, dL_dconic, dL_dcolors, cg, s);
    }
    return cg.dens_norm ? launch_compact<true>(P, D, M, means, scales, mod, rots, sh, vp, radii, g, dL_dmean2D, dL_dconic, dL_dcolors, cg, s)
                        : launch_compact<false>(P, D, M, means, scales, mod, rots, sh, vp, radii, g, dL_dmean2D, dL_dconic, dL_dcolors, cg, s);
}

size_t pose_partials_count(uint32_t Pcap) { return 6 * (size_t)((Pcap + PB_THREADS - 1) / PB_THREADS); }

}  // namespace glic

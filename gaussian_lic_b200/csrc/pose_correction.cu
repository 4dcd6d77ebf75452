// pose_correction.cu -- glic_mapper_correct_poses' record (host, float64) and its row update (include/glic_b200.h,
// "Pose corrections").
//
// The record of one keyframe is the rigid motion dT = [dR | t] from its old pose to its new one, the unit quaternion q of dR and
// the SH band rotation matrices of R(q).  The row kernel applies it to every row anchored to that keyframe: mean, stored
// quaternion and SH rest, each in float64 with one rounding per operation, so the result is a function of the row and the
// record alone (no order, no atomics on data): replicas and deterministic training stay bit-identical.
//
// Row layout: one warp per 32 consecutive rows.  The anchors decide which lanes move (a ballot); a warp with none returns after
// 128 B.  The SH rest of the moving rows ([M][3] floats per row, contiguous across the warp's rows) is staged through shared
// memory with consecutive lanes on consecutive words, so loads and stores are coalesced and rows that do not move are neither
// read nor written; each lane then rotates its own row in shared memory, band by band.
#include "common.cuh"
#include "pose_correction.cuh"

#include <cmath>
#include <cstring>

namespace glic {
namespace {

// sh_math.cuh's constants in float64 (its floats are these values rounded)
constexpr double kB1 = 0.4886025119029199;
constexpr double kB2a = 1.0925484305920792, kB2b = 0.31539156525252005, kB2c = 0.5462742152960396;
constexpr double kB3a = 0.5900435899266435, kB3b = 2.890611442640554, kB3c = 0.4570457994644658, kB3d = 0.3731763325901154,
                 kB3e = 1.445305721320277;
// where A_l (l = 1..3) starts in glic_rigid_correction::sh
__host__ __device__ constexpr int sh_offset(int l) { return l == 1 ? 0 : l == 2 ? 9 : 34; }

// the 2l + 1 SH-rest basis functions of band l (1..3) at unit (x, y, z): sh_basis's polynomials in float64
void band_basis(int l, double x, double y, double z, double* b) {
    if (l == 1) { b[0] = -kB1 * y; b[1] = kB1 * z; b[2] = -kB1 * x; return; }
    const double xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    if (l == 2) {
        b[0] = kB2a * xy; b[1] = -kB2a * yz; b[2] = kB2b * (2.0 * zz - xx - yy); b[3] = -kB2a * xz; b[4] = kB2c * (xx - yy);
        return;
    }
    b[0] = -kB3a * y * (3.0 * xx - yy);
    b[1] = kB3b * xy * z;
    b[2] = -kB3c * y * (4.0 * zz - xx - yy);
    b[3] = kB3d * z * (2.0 * zz - 3.0 * xx - 3.0 * yy);
    b[4] = -kB3c * x * (4.0 * zz - xx - yy);
    b[5] = kB3e * z * (xx - yy);
    b[6] = -kB3a * x * (xx - 3.0 * yy);
}

// R(q) of sh_math.cuh's quat_gradient, row-major, for a unit q = (r, x, y, z)
void quat_matrix(const double* q, double* R) {
    const double r = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = 1.0 - 2.0 * (y * y + z * z); R[1] = 2.0 * (x * y - r * z);       R[2] = 2.0 * (x * z + r * y);
    R[3] = 2.0 * (x * y + r * z);       R[4] = 1.0 - 2.0 * (x * x + z * z); R[5] = 2.0 * (y * z - r * x);
    R[6] = 2.0 * (x * z - r * y);       R[7] = 2.0 * (y * z + r * x);       R[8] = 1.0 - 2.0 * (x * x + y * y);
}

// the header's branch-by-largest-diagonal quaternion of R, normalised, with the sign rule
void matrix_quat(const double* R, double* q) {
    const double tr = (R[0] + R[4]) + R[8];
    int branch = 0;
    double best = tr;
    for (int b = 1; b < 4; ++b)
        if (R[4 * (b - 1)] > best) { best = R[4 * (b - 1)]; branch = b; }
    double r, x, y, z, s;
    switch (branch) {
        case 0: r = 0.5 * std::sqrt(1.0 + tr); s = 0.25 / r; x = (R[7] - R[5]) * s; y = (R[2] - R[6]) * s; z = (R[3] - R[1]) * s; break;
        case 1: x = 0.5 * std::sqrt(((1.0 + R[0]) - R[4]) - R[8]); s = 0.25 / x; r = (R[7] - R[5]) * s; y = (R[1] + R[3]) * s; z = (R[2] + R[6]) * s; break;
        case 2: y = 0.5 * std::sqrt(((1.0 - R[0]) + R[4]) - R[8]); s = 0.25 / y; r = (R[2] - R[6]) * s; x = (R[1] + R[3]) * s; z = (R[5] + R[7]) * s; break;
        default: z = 0.5 * std::sqrt(((1.0 - R[0]) - R[4]) + R[8]); s = 0.25 / z; r = (R[3] - R[1]) * s; x = (R[2] + R[6]) * s; y = (R[5] + R[7]) * s; break;
    }
    const double n = std::sqrt(((r * r + x * x) + y * y) + z * z);
    q[0] = r / n; q[1] = x / n; q[2] = y / n; q[3] = z / n;
    const double lead = q[1] != 0.0 ? q[1] : q[2] != 0.0 ? q[2] : q[3];
    if (q[0] < 0.0 || (q[0] == 0.0 && lead < 0.0))
        for (int e = 0; e < 4; ++e) q[e] = -q[e];
    q[0] = q[0] + 0.0;                         // r = -0 becomes +0
}

// ---- the row kernel -----------------------------------------------------------------------------------------------------
constexpr int CORR_THREADS = 256;

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }

// rotates the SH rest row s[k * 3 + ch] (k < M) in place by c's band matrices
template <int D>
__device__ __forceinline__ void rotate_rest(const double* __restrict__ A, float* s) {
#pragma unroll
    for (int l = 1; l <= D; ++l) {
        const int n = 2 * l + 1, k0 = l * l - 1;
        const double* Al = A + sh_offset(l);
        float in[7][3];
#pragma unroll
        for (int k = 0; k < 7; ++k)
            if (k < n)
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) in[k][ch] = s[(k0 + k) * 3 + ch];
#pragma unroll
        for (int i = 0; i < 7; ++i) {
            if (i >= n) break;
            double acc[3];
            const double a0 = Al[i * n];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) acc[ch] = dm(a0, (double)in[0][ch]);
#pragma unroll
            for (int k = 1; k < 7; ++k) {
                if (k >= n) break;
                const double a = Al[i * n + k];
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) acc[ch] = da(acc[ch], dm(a, (double)in[k][ch]));
            }
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) s[(k0 + i) * 3 + ch] = __double2float_rn(acc[ch]);
        }
    }
}

template <int D>
__global__ void __launch_bounds__(CORR_THREADS)
correct_rows_kernel(uint32_t P, float4* __restrict__ rot, float* __restrict__ xyz, float* __restrict__ rest, const int32_t* __restrict__ anchor,
                    const glic_rigid_correction* __restrict__ table, int n_table, uint32_t* __restrict__ moved) {
    constexpr int W = 3 * ((D + 1) * (D + 1) - 1);           // floats of SH rest per row
    constexpr int STRIDE = W | 1;                            // odd: the lanes' rows fall in distinct banks
    __shared__ float stage[D ? (CORR_THREADS / 32) * 32 * STRIDE : 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t row0 = blockIdx.x * CORR_THREADS + warp * 32, r = row0 + lane;
    const glic_rigid_correction* c = nullptr;
    if (r < P) {
        const int a = anchor[r];
        if (a >= 0 && a < n_table && table[a].q[0] >= 0.0) c = table + a;
    }
    const unsigned mv = __ballot_sync(~0u, c != nullptr);
    if (!mv) return;                                         // warp-uniform
    if (lane == 0) atomicAdd(moved, (uint32_t)__popc(mv));
    if constexpr (D > 0) {
        float* s = stage + warp * 32 * STRIDE;
        const uint32_t rows = min(32u, P - row0);
        float* g = rest + (size_t)row0 * W;
        for (uint32_t i = lane; i < rows * W; i += 32) {
            const uint32_t q = i / W;
            if ((mv >> q) & 1u) s[q * STRIDE + (i - q * W)] = g[i];
        }
        __syncwarp();
        if (c) rotate_rest<D>(c->sh, s + lane * STRIDE);
        __syncwarp();
        for (uint32_t i = lane; i < rows * W; i += 32) {
            const uint32_t q = i / W;
            if ((mv >> q) & 1u) g[i] = s[q * STRIDE + (i - q * W)];
        }
    }
    if (!c) return;
    const double* R = c->R;
    const double* t = c->t;
    float* p = xyz + 3 * (size_t)r;
    const double x = p[0], y = p[1], z = p[2];
    for (int i = 0; i < 3; ++i) p[i] = __double2float_rn(da(da(da(dm(R[3 * i], x), dm(R[3 * i + 1], y)), dm(R[3 * i + 2], z)), t[i]));
    const float4 o = rot[r];
    const double qr = c->q[0], qx = c->q[1], qy = c->q[2], qz = c->q[3];
    const double rr = o.x, rx = o.y, ry = o.z, rz = o.w;
    float4 n;
    n.x = __double2float_rn(da(da(da(dm(qr, rr), -dm(qx, rx)), -dm(qy, ry)), -dm(qz, rz)));
    n.y = __double2float_rn(da(da(da(dm(qr, rx), dm(qx, rr)), dm(qy, rz)), -dm(qz, ry)));
    n.z = __double2float_rn(da(da(da(dm(qr, ry), -dm(qx, rz)), dm(qy, rr)), dm(qz, rx)));
    n.w = __double2float_rn(da(da(da(dm(qr, rz), dm(qx, ry)), -dm(qy, rx)), dm(qz, rr)));
    rot[r] = n;
}

__global__ void __launch_bounds__(256) fill_anchors_kernel(int32_t* __restrict__ anchor, uint32_t first, uint32_t split, uint32_t end, int32_t value) {
    const uint32_t i = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (i < end) anchor[i] = i < split ? -1 : value;
}

}  // namespace

int launch_correct_rows(int D, uint32_t P, uint32_t Pcap, float* params, const int32_t* anchor, const glic_rigid_correction* table,
                        int n_table, uint32_t* moved, cudaStream_t s) {
    if (P == 0 || n_table == 0) return GLIC_OK;
    size_t off[6];
    const int M = (D + 1) * (D + 1) - 1;
    glic_packed_offsets(Pcap, (uint32_t)M, off);
    float4* rot = reinterpret_cast<float4*>(params + off[0]);
    float* xyz = params + off[1];
    float* rest = M ? params + off[5] : nullptr;
    const unsigned blocks = (P + CORR_THREADS - 1) / CORR_THREADS;
    switch (D) {
        case 0: correct_rows_kernel<0><<<blocks, CORR_THREADS, 0, s>>>(P, rot, xyz, rest, anchor, table, n_table, moved); break;
        case 1: correct_rows_kernel<1><<<blocks, CORR_THREADS, 0, s>>>(P, rot, xyz, rest, anchor, table, n_table, moved); break;
        case 2: correct_rows_kernel<2><<<blocks, CORR_THREADS, 0, s>>>(P, rot, xyz, rest, anchor, table, n_table, moved); break;
        default: correct_rows_kernel<3><<<blocks, CORR_THREADS, 0, s>>>(P, rot, xyz, rest, anchor, table, n_table, moved); break;
    }
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_fill_anchors(int32_t* anchor, uint32_t first, uint32_t split, uint32_t end, int32_t value, cudaStream_t s) {
    if (end <= first) return GLIC_OK;
    fill_anchors_kernel<<<(end - first + 255) / 256, 256, 0, s>>>(anchor, first, split, end, value);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

}  // namespace glic

extern "C" {

int glic_sh_rotation(const double* q, int degree, double* out) {
    if (!q || !out) { glic::set_error("sh_rotation: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (degree < 0 || degree > 3) { glic::set_error("sh_rotation: degree must be in [0, 3]"); return GLIC_ERR_INVALID_ARGUMENT; }
    for (int e = 0; e < 4; ++e)
        if (!std::isfinite(q[e])) { glic::set_error("sh_rotation: non-finite quaternion"); return GLIC_ERR_INVALID_ARGUMENT; }
    for (int e = 0; e < 83; ++e) out[e] = 0.0;
    if (degree == 0) return GLIC_OK;
    double R[9];
    glic::quat_matrix(q, R);
    // 4-point Gauss-Legendre in z times 8 azimuths: exact on the sphere for polynomials of degree <= 7 (the products here have 6)
    const double a = std::sqrt(6.0 / 5.0), pi = 3.14159265358979323846;
    const double zs[4] = {-std::sqrt(3.0 / 7.0 + 2.0 / 7.0 * a), -std::sqrt(3.0 / 7.0 - 2.0 / 7.0 * a), std::sqrt(3.0 / 7.0 - 2.0 / 7.0 * a),
                          std::sqrt(3.0 / 7.0 + 2.0 / 7.0 * a)};
    const double wo = (18.0 - std::sqrt(30.0)) / 36.0, wi = (18.0 + std::sqrt(30.0)) / 36.0;
    const double ws[4] = {wo, wi, wi, wo};
    for (int iz = 0; iz < 4; ++iz)
        for (int ip = 0; ip < 8; ++ip) {
            const double z = zs[iz], rho = std::sqrt(1.0 - z * z), phi = 2.0 * pi * ip / 8.0;
            const double d[3] = {rho * std::cos(phi), rho * std::sin(phi), z};
            const double e[3] = {R[0] * d[0] + R[3] * d[1] + R[6] * d[2], R[1] * d[0] + R[4] * d[1] + R[7] * d[2],
                                 R[2] * d[0] + R[5] * d[1] + R[8] * d[2]};                  // R(q)^T d
            const double w = ws[iz] * (pi / 4.0);
            for (int l = 1; l <= degree; ++l) {
                const int n = 2 * l + 1;
                double bd[7], be[7];
                glic::band_basis(l, d[0], d[1], d[2], bd);
                glic::band_basis(l, e[0], e[1], e[2], be);
                double* A = out + glic::sh_offset(l);
                for (int i = 0; i < n; ++i)
                    for (int k = 0; k < n; ++k) A[i * n + k] += w * bd[i] * be[k];
            }
        }
    return GLIC_OK;
}

int glic_pose_correction_record(const float* R_old, const float* t_old, const float* R_new, const float* t_new, int degree,
                                glic_rigid_correction* out) {
    if (!R_old || !t_old || !R_new || !t_new || !out) { glic::set_error("pose_correction_record: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (degree < 0 || degree > 3) { glic::set_error("pose_correction_record: degree must be in [0, 3]"); return GLIC_ERR_INVALID_ARGUMENT; }
    glic_rigid_correction c;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            c.R[3 * i + j] = ((double)R_new[3 * i] * R_old[3 * j] + (double)R_new[3 * i + 1] * R_old[3 * j + 1]) +
                             (double)R_new[3 * i + 2] * R_old[3 * j + 2];
    for (int i = 0; i < 3; ++i)
        c.t[i] = (double)t_new[i] - ((c.R[3 * i] * t_old[0] + c.R[3 * i + 1] * t_old[1]) + c.R[3 * i + 2] * t_old[2]);
    for (int e = 0; e < 9; ++e)
        if (!std::isfinite(c.R[e])) { glic::set_error("pose_correction_record: non-finite pose"); return GLIC_ERR_INVALID_ARGUMENT; }
    for (int i = 0; i < 3; ++i)
        if (!std::isfinite(c.t[i])) { glic::set_error("pose_correction_record: non-finite pose"); return GLIC_ERR_INVALID_ARGUMENT; }
    glic::matrix_quat(c.R, c.q);
    if (!std::isfinite(c.q[0])) { glic::set_error("pose_correction_record: the rotation has no quaternion (not a rotation)"); return GLIC_ERR_INVALID_ARGUMENT; }
    int rc = glic_sh_rotation(c.q, degree, c.sh);
    if (rc != GLIC_OK) return rc;
    std::memcpy(out, &c, sizeof(c));
    return GLIC_OK;
}

}  // extern "C"

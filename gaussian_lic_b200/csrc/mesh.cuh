// mesh.cuh -- what mesh.cu shares with sparse_mesh.cu and the mapper beyond the C ABI (include/glic_b200.h "Meshing" and
// "Sparse meshing"): the per-point TSDF update and the surface-nets vertex, so that the dense and the sparse grid compute every
// point and every vertex with the same operations.
#pragma once
#include "common.cuh"
#include "geom_math.cuh"

namespace glic {
// glic_mesh_count with the number of observed lattice points as well: totals3 = {vertices, faces, observed}; synchronises s
int mesh_count(const glic_tsdf_grid& g, void* scratch, size_t scratch_bytes, uint64_t totals3[3], cudaStream_t s);

// one view as glic_tsdf_integrate takes it
struct FuseView {
    const float* view;
    int W, H;
    float fx, fy, cx, cy;
    const float* depth;
    const float* rgb;
    const uint32_t* mask;
    int wpr;
    float trunc, max_depth;
};

// the checks of glic_tsdf_integrate's view arguments (everything but the grid); `what` prefixes the error
int fuse_view_check(const FuseView& f, const char* what);

// steps 1-5 of "Meshing" for the lattice point at world position (X, Y, Z): its tsdf, weight and colour (col[c * cstride]);
// a skipped point is neither read nor written
__device__ __forceinline__ void tsdf_update(const FuseView& f, float X, float Y, float Z, float* tsdf, float* weight, float* col,
                                            size_t cstride) {
    const float z = xform_row(f.view, 2, X, Y, Z);
    if (!(z > 0.0f)) return;
    const float x = xform_row(f.view, 0, X, Y, Z), y = xform_row(f.view, 1, X, Y, Z);
    const float u = fadd(fmul(f.fx, __fdiv_rn(x, z)), f.cx), v = fadd(fmul(f.fy, __fdiv_rn(y, z)), f.cy);
    if (!(u >= 0.0f && u < (float)f.W && v >= 0.0f && v < (float)f.H)) return;
    const int px = (int)floorf(u), py = (int)floorf(v);
    if (f.mask && !((f.mask[(size_t)py * f.wpr + (px >> 5)] >> (px & 31)) & 1u)) return;
    const size_t pix = (size_t)py * f.W + px;
    const float d = f.depth[pix];
    if (!(d > 0.0f) || (f.max_depth != 0.0f && !(d <= f.max_depth))) return;
    const float sdf = fsub(d, z);
    if (!(sdf >= -f.trunc)) return;
    const float t = fminf(1.0f, __fdiv_rn(sdf, f.trunc));
    const float w = *weight, w1 = fadd(w, 1.0f);
    *tsdf = __fdiv_rn(fadd(fmul(*tsdf, w), t), w1);
    if (f.rgb) {
        const size_t HW = (size_t)f.W * f.H;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float* cp = col + (size_t)c * cstride;
            *cp = __fdiv_rn(fadd(fmul(*cp, w), f.rgb[c * HW + pix]), w1);
        }
    }
    *weight = w1;
}

// corner A (a + 2 b + 4 c) of each of a cell's 12 edges in the fixed edge order: the x-edges for (b, c) = (0,0), (1,0), (0,1),
// (1,1), then the y-edges for (a, c), then the z-edges for (a, b); edge e's other end is A + (1 << (e / 4))
__host__ __device__ constexpr int edge_corner(int e) {
    return e < 4 ? 2 * (e & 1) + 4 * (e >> 1) : e < 8 ? (e & 1) + 4 * ((e >> 1) & 1) : (e & 1) + 2 * ((e >> 1) & 1);
}

// the vertex (world position) and colour (uint8) of the active cell with lower corner ijk (lattice indices from origin o),
// from its corners' tsdf t[q] and colour col[c][q], q = a + 2 b + 4 c
__device__ __forceinline__ void surface_vertex(const float t[8], const float col[3][8], const int ijk[3], const float o[3], float s,
                                               float xyz[3], uint8_t rgb[3]) {
    float sp[3] = {0.f, 0.f, 0.f}, sc[3] = {0.f, 0.f, 0.f};
    int n = 0;
#pragma unroll
    for (int e = 0; e < 12; ++e) {
        const int ax = e >> 2, A = edge_corner(e), B = A + (1 << ax);
        const float tA = t[A], tB = t[B];
        if ((tA < 0.0f) == (tB < 0.0f)) continue;
        const float f = __fdiv_rn(tA, fsub(tA, tB));
        float p[3] = {(float)(A & 1), (float)((A >> 1) & 1), (float)(A >> 2)};
        p[ax] = f;
        float cc[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) cc[ch] = fadd(col[ch][A], fmul(f, fsub(col[ch][B], col[ch][A])));
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            sp[a] = n ? fadd(sp[a], p[a]) : p[a];
            sc[a] = n ? fadd(sc[a], cc[a]) : cc[a];
        }
        ++n;
    }
    const float fn = (float)n;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        xyz[a] = fadd(o[a], fmul(s, fadd((float)ijk[a], __fdiv_rn(sp[a], fn))));
        const float c = fminf(fmaxf(__fdiv_rn(sc[a], fn), 0.0f), 1.0f);
        rgb[a] = (uint8_t)__float2int_rn(fmul(c, 255.0f));
    }
}
}  // namespace glic

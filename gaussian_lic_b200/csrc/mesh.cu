// mesh.cu -- a coloured triangle mesh from depth maps (include/glic_b200.h "Meshing"): TSDF fusion into a dense voxel grid and
// naive surface nets.  Every output is defined per lattice point, cell or lattice edge by a few correctly rounded float
// operations (no contraction: every one is an _rn intrinsic or an fma the definition names), and nothing is accumulated with
// atomics, so a NumPy float32 restatement (tests/mesh_oracle.py) matches every bit and two identical call sequences agree.
//   integration: one thread per lattice point; a point that projects outside the frame, onto a masked pixel, onto an invalid
//     depth or too far behind the surface is neither read nor written;
//   extraction, no CUB, in the style of prune.cu:
//     1. mesh_active_kernel: one CTA per tile of MESH_TILE lattice points; bit L of `act` says whether the cell with lower
//        corner L is active (one word per warp, from a ballot), and the tile's vertex and observed-point counts;
//     2. mesh_edges_kernel: per tile, the lattice edges that make a quad (their four cells' bits read from `act`);
//     3. mesh_scan_kernel, one CTA per count: exclusive scans of the per-tile counts in a fixed order, and the totals;
//     4. mesh_word_prefix_kernel: the global vertex id of the first active cell of every `act` word, so that any cell's vertex
//        id is one word read and a popcount;
//     5. mesh_emit_kernel (glic_mesh_extract): per tile, each active cell's vertex and colour at its id, and each quad's two
//        triangles at the tile's edge offset plus a block scan of the edge counts in lattice order.
// Positions depend only on ids computed from scans, never on which CTA finishes first.
#include "common.cuh"
#include "geom_math.cuh"
#include "mesh.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace glic {
namespace {

constexpr int MESH_THREADS = 256;
constexpr int MESH_ITEMS = 4;                                   // lattice points per thread, MESH_THREADS apart
constexpr uint32_t MESH_TILE = MESH_THREADS * MESH_ITEMS;      // lattice points per CTA: 32 words of cell bits
constexpr int MESH_MAX_DIM = 2048;

// the grid as the kernels see it: data = tsdf[N] | weight[N] | colour[3][N]
struct Grid {
    float o[3], s;
    int n[3];
    uint32_t N;
    float *tsdf, *weight, *col;
};

Grid device_grid(const glic_tsdf_grid& g) {
    Grid d;
    for (int a = 0; a < 3; ++a) { d.o[a] = g.origin[a]; d.n[a] = g.dims[a]; }
    d.s = g.voxel_size;
    d.N = (uint32_t)((size_t)g.dims[0] * g.dims[1] * g.dims[2]);
    d.tsdf = static_cast<float*>(g.data);
    d.weight = d.tsdf + d.N;
    d.col = d.weight + d.N;
    return d;
}

// lattice points of valid dims (each in [2, 2048], N < 2^31), 0 otherwise
size_t lattice_points(const int* dims) {
    if (!dims) return 0;
    size_t N = 1;
    for (int a = 0; a < 3; ++a) {
        if (dims[a] < 2 || dims[a] > MESH_MAX_DIM) return 0;
        N *= (size_t)dims[a];
    }
    return N < (size_t(1) << 31) ? N : 0;
}

int grid_check(const glic_tsdf_grid* g, const char* what) {
    if (!g || !g->data) { set_error(std::string(what) + ": null grid"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!lattice_points(g->dims)) {
        set_error(std::string(what) + ": every grid dimension must be in [2, 2048], with fewer than 2^31 lattice points");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!(std::isfinite(g->voxel_size) && g->voxel_size > 0.0f) || !std::isfinite(g->origin[0]) || !std::isfinite(g->origin[1]) ||
        !std::isfinite(g->origin[2])) {
        set_error(std::string(what) + ": voxel_size must be finite and > 0, the origin finite");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    return GLIC_OK;
}

// the extraction scratch of N lattice points: act[words] | wpre[words] | tile counts [3][tiles] (vertices, quad edges, observed
// points; scanned in place into tile offsets) | totals[3]
struct MeshScratch {
    uint32_t* act;
    uint32_t* wpre;
    unsigned long long* tile;
    unsigned long long* total;
    uint32_t tiles, words;
};
size_t mesh_carve(void* ws, size_t N, MeshScratch* out) {
    Carver c(ws);
    MeshScratch m;
    m.words = (uint32_t)((N + 31) / 32);
    m.tiles = (uint32_t)((N + MESH_TILE - 1) / MESH_TILE);
    m.act = c.take<uint32_t>(m.words);
    m.wpre = c.take<uint32_t>(m.words);
    m.tile = c.take<unsigned long long>(3 * (size_t)m.tiles);
    m.total = c.take<unsigned long long>(3);
    if (out) *out = m;
    return c.total();
}

__device__ __forceinline__ void lattice_ijk(const Grid& g, uint32_t L, int ijk[3]) {
    ijk[0] = (int)(L % (uint32_t)g.n[0]);
    const uint32_t q = L / (uint32_t)g.n[0];
    ijk[1] = (int)(q % (uint32_t)g.n[1]);
    ijk[2] = (int)(q / (uint32_t)g.n[1]);
}

// corner q = a + 2 b + 4 c of the cell with lower corner L (x fastest)
__device__ __forceinline__ uint32_t corner(const Grid& g, uint32_t L, int q) {
    return L + (uint32_t)(q & 1) + (uint32_t)((q >> 1) & 1) * (uint32_t)g.n[0] + (uint32_t)(q >> 2) * (uint32_t)g.n[0] * (uint32_t)g.n[1];
}

// the cell with lower corner L exists, its 8 corners are observed (weight > 0) and they are not all on one side (tsdf < 0)
__device__ __forceinline__ bool cell_active(const Grid& g, uint32_t L, const int ijk[3]) {
    if (ijk[0] >= g.n[0] - 1 || ijk[1] >= g.n[1] - 1 || ijk[2] >= g.n[2] - 1) return false;
    int inside = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const uint32_t c = corner(g, L, q);
        if (!(g.weight[c] > 0.0f)) return false;
        inside += g.tsdf[c] < 0.0f ? 1 : 0;
    }
    return inside != 0 && inside != 8;
}

__device__ __forceinline__ bool act_bit(const uint32_t* act, uint32_t C) { return (act[C >> 5] >> (C & 31)) & 1u; }

// the lattice edge of axis a from L to L + e_a makes a quad: both ends observed, exactly one inside, and the four cells with
// lower corners L - e_b - e_c, L - e_c, L, L - e_b ((b, c) the other axes in cyclic order) exist and are active; cell[] gets them
__device__ __forceinline__ bool edge_quad(const Grid& g, const uint32_t* act, uint32_t L, const int ijk[3], int a, uint32_t cell[4]) {
    const int b = a == 2 ? 0 : a + 1, c = a == 0 ? 2 : a - 1;
    if (ijk[a] >= g.n[a] - 1 || ijk[b] < 1 || ijk[c] < 1) return false;
    const uint32_t st[3] = {1u, (uint32_t)g.n[0], (uint32_t)g.n[0] * (uint32_t)g.n[1]};
    const uint32_t B = L + st[a];
    if (!(g.weight[L] > 0.0f) || !(g.weight[B] > 0.0f)) return false;
    if ((g.tsdf[L] < 0.0f) == (g.tsdf[B] < 0.0f)) return false;
    cell[0] = L - st[b] - st[c];
    cell[1] = L - st[c];
    cell[2] = L;
    cell[3] = L - st[b];
#pragma unroll
    for (int q = 0; q < 4; ++q)
        if (!act_bit(act, cell[q])) return false;
    return true;
}

// sum of v over the CTA (MESH_THREADS threads), valid in thread 0
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* warp_tot) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < MESH_THREADS / 32; ++w) t += warp_tot[w];
    __syncthreads();
    return t;
}

// exclusive scan of v over the CTA in thread order; *total gets the CTA's sum
__device__ __forceinline__ uint32_t block_exclusive(uint32_t v, uint32_t* warp_tot, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    uint32_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < MESH_THREADS / 32; ++w) {
        if (w < warp) before += warp_tot[w];
        all += warp_tot[w];
    }
    __syncthreads();
    *total = all;
    return before + incl - v;
}

__global__ void __launch_bounds__(MESH_THREADS) tsdf_integrate_kernel(Grid g, FuseView f) {
    const uint32_t p = blockIdx.x * MESH_THREADS + threadIdx.x;
    if (p >= g.N) return;
    int ijk[3];
    lattice_ijk(g, p, ijk);
    const float X = fadd(g.o[0], fmul(g.s, (float)ijk[0]));
    const float Y = fadd(g.o[1], fmul(g.s, (float)ijk[1]));
    const float Z = fadd(g.o[2], fmul(g.s, (float)ijk[2]));
    tsdf_update(f, X, Y, Z, g.tsdf + p, g.weight + p, g.col + p, g.N);
}

// act bits, and per tile: tile[0][t] = active cells, tile[2][t] = observed lattice points
__global__ void __launch_bounds__(MESH_THREADS) mesh_active_kernel(Grid g, MeshScratch m) {
    __shared__ unsigned long long warp_tot[MESH_THREADS / 32];
    unsigned long long nv = 0, no = 0;
#pragma unroll 1
    for (int e = 0; e < MESH_ITEMS; ++e) {
        const uint32_t L = blockIdx.x * MESH_TILE + e * MESH_THREADS + threadIdx.x;
        bool a = false, o = false;
        if (L < g.N) {
            int ijk[3];
            lattice_ijk(g, L, ijk);
            a = cell_active(g, L, ijk);
            o = g.weight[L] > 0.0f;
        }
        const uint32_t ba = __ballot_sync(0xffffffffu, a), bo = __ballot_sync(0xffffffffu, o);
        if ((threadIdx.x & 31) == 0) {
            if ((L >> 5) < m.words) m.act[L >> 5] = ba;
            nv += __popc(ba);
            no += __popc(bo);
        }
    }
    const unsigned long long tv = block_sum(nv, warp_tot), to = block_sum(no, warp_tot);
    if (threadIdx.x == 0) {
        m.tile[blockIdx.x] = tv;
        m.tile[2 * (size_t)m.tiles + blockIdx.x] = to;
    }
}

// per tile: tile[1][t] = lattice edges that make a quad
__global__ void __launch_bounds__(MESH_THREADS) mesh_edges_kernel(Grid g, MeshScratch m) {
    __shared__ unsigned long long warp_tot[MESH_THREADS / 32];
    unsigned long long ne = 0;
#pragma unroll 1
    for (int e = 0; e < MESH_ITEMS; ++e) {
        const uint32_t L = blockIdx.x * MESH_TILE + e * MESH_THREADS + threadIdx.x;
        if (L >= g.N) break;
        int ijk[3];
        lattice_ijk(g, L, ijk);
        uint32_t cell[4];
#pragma unroll
        for (int a = 0; a < 3; ++a) ne += edge_quad(g, m.act, L, ijk, a, cell) ? 1u : 0u;
    }
    const unsigned long long te = block_sum(ne, warp_tot);
    if (threadIdx.x == 0) m.tile[(size_t)m.tiles + blockIdx.x] = te;
}

// exclusive scan of the tile counts in place, the total into total[b]; CTA b scans the b-th array of n_tiles counts, 1024 at a time
__global__ void __launch_bounds__(1024) mesh_scan_kernel(uint32_t n_tiles, unsigned long long* __restrict__ tile, unsigned long long* __restrict__ total) {
    tile += (size_t)blockIdx.x * n_tiles;
    __shared__ unsigned long long warp_tot[32];
    __shared__ unsigned long long carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n_tiles; base += 1024) {
        const uint32_t i = base + tid;
        const unsigned long long f = i < n_tiles ? tile[i] : 0ull;
        unsigned long long incl = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const unsigned long long w = warp_tot[lane];
            unsigned long long wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            warp_tot[lane] = wi - w;
        }
        __syncthreads();
        const unsigned long long excl = carry + warp_tot[warp] + incl - f;
        if (i < n_tiles) tile[i] = excl;
        __syncthreads();
        if (tid == 1023) carry = excl + f;
        __syncthreads();
    }
    if (tid == 0) total[blockIdx.x] = carry;
}

// wpre[w] = the vertex id of the first active cell at or after word w's first lattice point: one warp per tile
__global__ void __launch_bounds__(32) mesh_word_prefix_kernel(MeshScratch m) {
    const uint32_t w = blockIdx.x * 32 + threadIdx.x;
    const uint32_t c = w < m.words ? (uint32_t)__popc(m.act[w]) : 0u;
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (threadIdx.x >= o) incl += t;
    }
    if (w < m.words) m.wpre[w] = (uint32_t)m.tile[blockIdx.x] + incl - c;
}

__device__ __forceinline__ uint32_t vertex_id(const MeshScratch& m, uint32_t C) {
    return m.wpre[C >> 5] + (uint32_t)__popc(m.act[C >> 5] & ((1u << (C & 31)) - 1u));
}

// the vertex (world position) and colour (uint8) of active cell L
__device__ __forceinline__ void cell_vertex(const Grid& g, uint32_t L, const int ijk[3], float xyz[3], uint8_t rgb[3]) {
    float t[8], col[3][8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const uint32_t c = corner(g, L, q);
        t[q] = g.tsdf[c];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) col[ch][q] = g.col[(size_t)ch * g.N + c];
    }
    surface_vertex(t, col, ijk, g.o, g.s, xyz, rgb);
}

__global__ void __launch_bounds__(MESH_THREADS)
mesh_emit_kernel(Grid g, MeshScratch m, float* __restrict__ xyz, uint8_t* __restrict__ rgb, int* __restrict__ faces) {
    __shared__ uint32_t warp_tot[MESH_THREADS / 32];
    unsigned long long base = m.tile[(size_t)m.tiles + blockIdx.x];
    for (int e = 0; e < MESH_ITEMS; ++e) {
        const uint32_t L = blockIdx.x * MESH_TILE + e * MESH_THREADS + threadIdx.x;
        int ijk[3] = {0, 0, 0};
        uint32_t cells[3][4];
        unsigned quads = 0;
        uint32_t nq = 0;
        if (L < g.N) {
            lattice_ijk(g, L, ijk);
            if (act_bit(m.act, L)) {
                float p[3];
                uint8_t c[3];
                cell_vertex(g, L, ijk, p, c);
                const size_t v = vertex_id(m, L);
#pragma unroll
                for (int a = 0; a < 3; ++a) { xyz[3 * v + a] = p[a]; rgb[3 * v + a] = c[a]; }
            }
#pragma unroll
            for (int a = 0; a < 3; ++a)
                if (edge_quad(g, m.act, L, ijk, a, cells[nq])) { quads |= 1u << a; ++nq; }
        }
        uint32_t all;
        const uint32_t before = block_exclusive(nq, warp_tot, &all);
        if (nq) {
            const bool keep = g.tsdf[L] < 0.0f;                        // L inside: the quad's normal points along +e_a, out of it
            size_t f = 2 * (size_t)(base + before);
            for (uint32_t q = 0; q < nq; ++q, f += 2) {
                int id[4];
#pragma unroll
                for (int r = 0; r < 4; ++r) id[r] = (int)vertex_id(m, cells[q][keep ? r : 3 - r]);
                int* t = faces + 3 * f;
                t[0] = id[0]; t[1] = id[1]; t[2] = id[2];
                t[3] = id[0]; t[4] = id[2]; t[5] = id[3];
            }
        }
        base += all;
    }
}

// the checks of glic_mesh_count / glic_mesh_extract; out = the carved scratch
int scratch_check(const glic_tsdf_grid* g, void* scratch, size_t bytes, const char* what, MeshScratch* out) {
    if (const int e = grid_check(g, what)) return e;
    if (!scratch) { set_error(std::string(what) + ": null scratch"); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t N = lattice_points(g->dims), need = mesh_carve(nullptr, N, nullptr);
    if (bytes < need) {
        set_error(std::string(what) + ": scratch of " + std::to_string(bytes) + " bytes, glic_mesh_scratch_bytes needs " + std::to_string(need));
        return GLIC_ERR_WORKSPACE;
    }
    mesh_carve(scratch, N, out);
    return GLIC_OK;
}

}  // namespace

int fuse_view_check(const FuseView& f, const char* what) {
    const std::string w(what);
    if (!f.view || !f.depth) { set_error(w + ": null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (f.W < 1 || f.H < 1) { set_error(w + ": width and height must be >= 1"); return GLIC_ERR_INVALID_ARGUMENT; }
    const int64_t tiles = (((int64_t)f.W + TILE - 1) / TILE) * (((int64_t)f.H + TILE - 1) / TILE);
    if (tiles > GLIC_MAX_TILES) {
        set_error(w + ": " + std::to_string(f.W) + "x" + std::to_string(f.H) + " has more than GLIC_MAX_TILES tiles of 16x16");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!(std::isfinite(f.fx) && f.fx > 0.0f) || !(std::isfinite(f.fy) && f.fy > 0.0f) || !std::isfinite(f.cx) || !std::isfinite(f.cy)) {
        set_error(w + ": fx and fy must be finite and > 0, cx and cy finite"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!(std::isfinite(f.trunc) && f.trunc > 0.0f)) { set_error(w + ": trunc must be finite and > 0"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!(std::isfinite(f.max_depth) && f.max_depth >= 0.0f)) { set_error(w + ": max_depth must be finite and >= 0"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (f.mask && f.wpr < mask_words_per_row(f.W)) {
        set_error(w + ": words_per_row must be at least glic_mask_words_per_row(W)"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    return GLIC_OK;
}

int mesh_count(const glic_tsdf_grid& gg, void* scratch, size_t scratch_bytes, uint64_t totals3[3], cudaStream_t s) {
    MeshScratch m;
    if (const int e = scratch_check(&gg, scratch, scratch_bytes, "mesh_count", &m)) return e;
    const Grid g = device_grid(gg);
    mesh_active_kernel<<<m.tiles, MESH_THREADS, 0, s>>>(g, m);
    GLIC_LAUNCH_CHECK();
    mesh_edges_kernel<<<m.tiles, MESH_THREADS, 0, s>>>(g, m);
    GLIC_LAUNCH_CHECK();
    mesh_scan_kernel<<<3, 1024, 0, s>>>(m.tiles, m.tile, m.total);
    GLIC_LAUNCH_CHECK();
    mesh_word_prefix_kernel<<<m.tiles, 32, 0, s>>>(m);
    GLIC_LAUNCH_CHECK();
    unsigned long long t[3];
    GLIC_CUDA_TRY(cudaMemcpyAsync(t, m.total, sizeof(t), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    totals3[0] = t[0];
    totals3[1] = 2 * t[1];
    totals3[2] = t[2];
    return GLIC_OK;
}

}  // namespace glic

using namespace glic;

namespace {
struct File {
    FILE* f;
    explicit File(const char* path) : f(std::fopen(path, "wb")) {}
    ~File() { if (f) std::fclose(f); }
};
}  // namespace

extern "C" {

size_t glic_tsdf_bytes(const int* dims) { return 20 * lattice_points(dims); }

size_t glic_mesh_scratch_bytes(const int* dims) {
    const size_t N = lattice_points(dims);
    return N ? mesh_carve(nullptr, N, nullptr) : 0;
}

int glic_tsdf_clear(const glic_tsdf_grid* grid, void* stream) {
    if (const int e = grid_check(grid, "tsdf_clear")) return e;
    GLIC_CUDA_TRY(cudaMemsetAsync(grid->data, 0, glic_tsdf_bytes(grid->dims), (cudaStream_t)stream));
    return GLIC_OK;
}

int glic_tsdf_integrate(const glic_tsdf_grid* grid, const float* viewmatrix_dev, int W, int H, float fx, float fy, float cx, float cy,
                        const float* depth, const float* rgb, const uint32_t* mask_words, int words_per_row, float trunc, float max_depth,
                        void* stream) {
    if (const int e = grid_check(grid, "tsdf_integrate")) return e;
    const FuseView f{viewmatrix_dev, W, H, fx, fy, cx, cy, depth, rgb, mask_words, words_per_row, trunc, max_depth};
    if (const int e = fuse_view_check(f, "tsdf_integrate")) return e;
    const Grid g = device_grid(*grid);
    tsdf_integrate_kernel<<<(g.N + MESH_THREADS - 1) / MESH_THREADS, MESH_THREADS, 0, (cudaStream_t)stream>>>(g, f);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int glic_mesh_count(const glic_tsdf_grid* grid, void* scratch, size_t scratch_bytes, uint64_t* counts_host, void* stream) {
    if (!counts_host) { set_error("mesh_count: null counts"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!grid) { set_error("mesh_count: null grid"); return GLIC_ERR_INVALID_ARGUMENT; }
    uint64_t t[3];
    if (const int e = mesh_count(*grid, scratch, scratch_bytes, t, (cudaStream_t)stream)) return e;
    counts_host[0] = t[0];
    counts_host[1] = t[1];
    return GLIC_OK;
}

int glic_mesh_extract(const glic_tsdf_grid* grid, const void* scratch, size_t scratch_bytes, float* xyz, uint8_t* rgb, int32_t* faces,
                      void* stream) {
    MeshScratch m;
    if (const int e = scratch_check(grid, const_cast<void*>(scratch), scratch_bytes, "mesh_extract", &m)) return e;
    if (!xyz || !rgb || !faces) { set_error("mesh_extract: null output"); return GLIC_ERR_INVALID_ARGUMENT; }
    mesh_emit_kernel<<<m.tiles, MESH_THREADS, 0, (cudaStream_t)stream>>>(device_grid(*grid), m, xyz, rgb, faces);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int glic_mesh_ply_write(const char* path, uint32_t V, const float* xyz, const uint8_t* rgb, uint32_t F, const int32_t* faces) {
    if (!path) { set_error("mesh_ply_write: null path"); return GLIC_ERR_INVALID_ARGUMENT; }
    if ((V > 0 && (!xyz || !rgb)) || (F > 0 && !faces)) { set_error("mesh_ply_write: null array"); return GLIC_ERR_INVALID_ARGUMENT; }
    File out(path);
    if (!out.f) { set_error(std::string("mesh_ply_write: cannot open ") + path); return GLIC_ERR_INVALID_ARGUMENT; }
    const std::string h = "ply\nformat binary_little_endian 1.0\nelement vertex " + std::to_string(V) +
                          "\nproperty float x\nproperty float y\nproperty float z\nproperty uchar red\nproperty uchar green\n"
                          "property uchar blue\nelement face " + std::to_string(F) + "\nproperty list uchar int vertex_indices\nend_header\n";
    bool ok = std::fwrite(h.data(), 1, h.size(), out.f) == h.size();
    const uint32_t CHUNK = 4096;
    std::vector<unsigned char> buf((size_t)CHUNK * 15);
    for (uint32_t i0 = 0; ok && i0 < V; i0 += CHUNK) {            // x86-64 and aarch64 hosts are little-endian: rows are copied as is
        const uint32_t n = std::min(CHUNK, V - i0);
        for (uint32_t i = 0; i < n; ++i) {
            std::memcpy(&buf[15 * (size_t)i], xyz + 3 * ((size_t)i0 + i), 12);
            std::memcpy(&buf[15 * (size_t)i + 12], rgb + 3 * ((size_t)i0 + i), 3);
        }
        ok = std::fwrite(buf.data(), 15, n, out.f) == n;
    }
    for (uint32_t i0 = 0; ok && i0 < F; i0 += CHUNK) {
        const uint32_t n = std::min(CHUNK, F - i0);
        for (uint32_t i = 0; i < n; ++i) {
            buf[13 * (size_t)i] = 3;
            std::memcpy(&buf[13 * (size_t)i + 1], faces + 3 * ((size_t)i0 + i), 12);
        }
        ok = std::fwrite(buf.data(), 13, n, out.f) == n;
    }
    const bool closed = std::fclose(out.f) == 0;
    out.f = nullptr;
    if (!ok || !closed) { set_error(std::string("mesh_ply_write: write to ") + path + " failed"); return GLIC_ERR_INVALID_ARGUMENT; }
    return GLIC_OK;
}

}  // extern "C"

// sparse_mesh.cu -- the sparse block TSDF (include/glic_b200.h "Sparse meshing"): only the 8^3-voxel blocks near some view's
// observed surface are stored, over a lattice of +-2^19 points per axis, and every stored voxel, vertex and face is what the
// dense grid of mesh.cu computes at the same lattice point (the per-point update and the vertex are mesh.cuh's, shared).
//   block set: an open-addressing hash of 64-bit block keys (2 slots per entry of capacity, linear probing, atomicCAS); one
//     thread per pixel inserts every block of its pixel's lattice range;
//   grid: the keys compacted and sorted (glic_sort_pairs_u64_u32), a block's slot = its key's rank, a 27-entry neighbour table
//     by binary search, and a planar pool of 512 points per block;
//   integration: one thread per voxel, tsdf_update;
//   extraction: per voxel, the active bit of its cell and its quad edges, read through the neighbour table; then the active
//     cells' (k, j, i) keys and the quad edges' (k, j, i, axis) keys are sorted, so vertex ids and face slots are ranks, the
//     dense grid's order on an unbounded lattice, whatever order the atomic compaction left them in.
#include "common.cuh"
#include "geom_math.cuh"
#include "mesh.cuh"

#include <algorithm>
#include <cmath>
#include <string>

#define SPARSE_TRY(expr) do { const int _e = (expr); if (_e != GLIC_OK) return _e; } while (0)

namespace glic {
namespace {

constexpr int SB = 8;                                  // block side
constexpr int SB3 = SB * SB * SB;                      // points per block
constexpr int POOL_FLOATS = 5 * SB3;                   // tsdf | weight | colour[3], planar per block
constexpr int LAT_HALF = 1 << 19;                      // lattice indices in [-2^19, 2^19)
constexpr int BLK_HALF = LAT_HALF / SB;                // block indices in [-2^16, 2^16)
constexpr uint64_t EMPTY = ~0ull;
constexpr uint32_t NONE = 0xFFFFFFFFu;
constexpr uint32_t MAX_BLOCKS = (1u << 23) - 1;        // slot * 512 + voxel < NONE (a pool of 86 GB)
constexpr int THREADS = 256;
constexpr uint32_t MAX_CAPACITY = 1u << 24;           // block set entries (256 MiB)
constexpr int SET_HEADER = 4;                          // u64: blocks, clipped pixels, overflow, unused

__host__ __device__ __forceinline__ uint64_t block_key(int bi, int bj, int bk) {
    return ((uint64_t)(bk + BLK_HALF) << 34) | ((uint64_t)(bj + BLK_HALF) << 17) | (uint64_t)(bi + BLK_HALF);
}
__device__ __forceinline__ void block_of(uint64_t key, int b[3]) {
    b[0] = (int)(key & 0x1FFFFu) - BLK_HALF;
    b[1] = (int)((key >> 17) & 0x1FFFFu) - BLK_HALF;
    b[2] = (int)(key >> 34) - BLK_HALF;
}
// the 60-bit key of lattice point (cell lower corner) i, j, k: ascending key = ascending (k, j, i)
__device__ __forceinline__ uint64_t cell_key(int i, int j, int k) {
    return ((uint64_t)(k + LAT_HALF) << 40) | ((uint64_t)(j + LAT_HALF) << 20) | (uint64_t)(i + LAT_HALF);
}

// ---- the block set ----------------------------------------------------------------------------------------------------
struct SetView {
    unsigned long long* hdr;                           // [SET_HEADER]
    unsigned long long* slots;                         // [2 capacity], EMPTY when free
    unsigned long long capacity, nslots;
};
SetView set_view(const glic_block_set& s) {
    SetView v;
    v.hdr = static_cast<unsigned long long*>(s.data);
    v.slots = v.hdr + SET_HEADER;
    v.capacity = s.capacity;
    v.nslots = 2ull * s.capacity;
    return v;
}
bool set_ok(const glic_block_set* s) { return s && s->data && s->capacity >= 1 && s->capacity <= MAX_CAPACITY; }

__device__ __forceinline__ uint64_t mix64(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return k;
}

// adds key; false when the set holds more than `capacity` keys or its slots ran out (the overflow flag is raised).  The count is
// exact (one increment per claimed slot), so a set overflows exactly when the union of what was inserted exceeds its capacity:
// up to capacity keys fill at most half the slots, and every probe then finds a free one.
__device__ bool set_insert(const SetView& s, uint64_t key) {
    unsigned long long i = mix64(key) % s.nslots;
    for (unsigned long long n = 0; n < s.nslots; ++n) {
        const unsigned long long cur = *(volatile unsigned long long*)(s.slots + i);
        if (cur == key) return true;
        if (cur == EMPTY) {
            const unsigned long long prev = atomicCAS(s.slots + i, EMPTY, key);
            if (prev == EMPTY) {
                if (atomicAdd(&s.hdr[0], 1ull) < s.capacity) return true;
                s.hdr[2] = 1;
                return false;
            }
            if (prev == key) return true;
        }
        i = i + 1 == s.nslots ? 0 : i + 1;
    }
    s.hdr[2] = 1;
    return false;
}

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// the allocation rule of one used pixel per thread (header "Sparse meshing")
__global__ void __launch_bounds__(THREADS)
block_insert_kernel(SetView set, double ox, double oy, double oz, double s, FuseView f) {
    const uint32_t pix = blockIdx.x * THREADS + threadIdx.x;
    if (pix >= (uint32_t)f.W * (uint32_t)f.H) return;
    const int px = (int)(pix % (uint32_t)f.W), py = (int)(pix / (uint32_t)f.W);
    if (f.mask && !((f.mask[(size_t)py * f.wpr + (px >> 5)] >> (px & 31)) & 1u)) return;
    const float d = f.depth[pix];
    if (!(d > 0.0f) || (f.max_depth != 0.0f && !(d <= f.max_depth))) return;
    double R[3][3], t[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        t[r] = f.view[12 + r];
#pragma unroll
        for (int a = 0; a < 3; ++a) R[r][a] = f.view[4 * a + r];
    }
    double lo[3], hi[3];
    bool finite = true;
#pragma unroll 1
    for (int q = 0; q < 8; ++q) {
        const double u = (double)(px + (q & 1)), v = (double)(py + ((q >> 1) & 1));
        const double z = (q >> 2) ? dadd((double)d, (double)f.trunc) : (double)d;
        const double c[3] = {ddiv(dmul(dsub(u, (double)f.cx), z), (double)f.fx), ddiv(dmul(dsub(v, (double)f.cy), z), (double)f.fy), z};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double X = dadd(dadd(dmul(R[0][a], dsub(c[0], t[0])), dmul(R[1][a], dsub(c[1], t[1]))), dmul(R[2][a], dsub(c[2], t[2])));
            finite = finite && isfinite(X);
            lo[a] = q ? fmin(lo[a], X) : X;
            hi[a] = q ? fmax(hi[a], X) : X;
        }
    }
    bool clipped = !finite, empty = !finite;
    int blo[3] = {0, 0, 0}, bhi[3] = {-1, -1, -1};
    const double o[3] = {ox, oy, oz};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        double l = floor(ddiv(dsub(lo[a], o[a]), s)) - 2.0, h = ceil(ddiv(dsub(hi[a], o[a]), s)) + 2.0;
        if (!(l >= -LAT_HALF)) { l = -LAT_HALF; clipped = true; }
        if (!(h <= LAT_HALF - 1)) { h = LAT_HALF - 1; clipped = true; }
        if (!(l <= h)) { empty = true; continue; }    // the whole range lies outside the lattice
        blo[a] = (int)l >> 3;                          // floor division by 8, negatives included
        bhi[a] = (int)h >> 3;
    }
    if (clipped) atomicAdd(&set.hdr[1], 1ull);
    if (empty) return;
    for (int bk = blo[2]; bk <= bhi[2]; ++bk)
        for (int bj = blo[1]; bj <= bhi[1]; ++bj)
            for (int bi = blo[0]; bi <= bhi[0]; ++bi)
                if (!set_insert(set, block_key(bi, bj, bk))) return;
}

__global__ void __launch_bounds__(THREADS) block_copy_kernel(SetView src, SetView dst) {
    const unsigned long long i = (unsigned long long)blockIdx.x * THREADS + threadIdx.x;
    if (i >= src.nslots) return;
    const unsigned long long key = src.slots[i];
    if (key != EMPTY) set_insert(dst, key);
}

// ---- the grid -----------------------------------------------------------------------------------------------------------
// data = keys[n] u64 (ascending) | nbr[27 n] u32 | pool [n][5][512] f32.  While glic_sparse_tsdf_init runs, the pool region
// holds the compaction and the sort: counter | keys[n] u64 | vals[n] u32 | sorted vals[n] u32 | sort temp
struct GridLayout {
    uint64_t* keys;
    uint32_t* nbr;
    float* pool;
    unsigned int* ctr;
    uint64_t* keys_in;
    uint32_t *vals_in, *vals_out;
    void* temp;
    size_t temp_bytes, total;
};
GridLayout grid_layout(void* data, uint32_t n) {
    GridLayout L;
    Carver c(data);
    L.keys = c.take<uint64_t>(n);
    L.nbr = c.take<uint32_t>(27 * (size_t)n);
    L.pool = c.take<float>((size_t)POOL_FLOATS * n);
    const size_t pool_end = c.total();
    Carver t(L.pool);
    L.ctr = t.take<unsigned int>(1);
    L.keys_in = t.take<uint64_t>(n);
    L.vals_in = t.take<uint32_t>(n);
    L.vals_out = t.take<uint32_t>(n);
    L.temp_bytes = sort_temp_bytes(n);
    L.temp = t.take<char>(L.temp_bytes);
    L.total = std::max(pool_end, (size_t)((char*)L.pool - (char*)data) + t.total());
    return L;
}

struct SGrid {
    float o[3], s;
    uint32_t n;
    const uint64_t* keys;
    const uint32_t* nbr;
    float* pool;
};
SGrid device_sgrid(const glic_sparse_tsdf& g) {
    const GridLayout L = grid_layout(g.data, g.n_blocks);
    SGrid d;
    for (int a = 0; a < 3; ++a) d.o[a] = g.origin[a];
    d.s = g.voxel_size;
    d.n = g.n_blocks;
    d.keys = L.keys;
    d.nbr = L.nbr;
    d.pool = L.pool;
    return d;
}
int sgrid_check(const glic_sparse_tsdf* g, const char* what) {
    if (!g || (g->n_blocks && !g->data)) { set_error(std::string(what) + ": null grid"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (g->n_blocks > MAX_BLOCKS) { set_error(std::string(what) + ": more than 2^23 blocks"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!(std::isfinite(g->voxel_size) && g->voxel_size > 0.0f) || !std::isfinite(g->origin[0]) || !std::isfinite(g->origin[1]) ||
        !std::isfinite(g->origin[2])) {
        set_error(std::string(what) + ": voxel_size must be finite and > 0, the origin finite");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    return GLIC_OK;
}

__global__ void __launch_bounds__(THREADS) compact_kernel(SetView set, uint32_t n, unsigned int* ctr, uint64_t* keys, uint32_t* vals) {
    const unsigned long long i = (unsigned long long)blockIdx.x * THREADS + threadIdx.x;
    if (i >= set.nslots) return;
    const unsigned long long key = set.slots[i];
    if (key == EMPTY) return;
    const unsigned int q = atomicAdd(ctr, 1u);
    if (q < n) { keys[q] = key; vals[q] = q; }
}

// the rank of key among keys[0, n) (ascending), NONE when absent
__device__ __forceinline__ uint32_t find_key(const uint64_t* keys, uint32_t n, uint64_t key) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (keys[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo < n && keys[lo] == key ? lo : NONE;
}

// nbr[27 b + (dx + 1) + 3 (dy + 1) + 9 (dz + 1)] = the slot of block b + (dx, dy, dz), NONE when it is not allocated
__global__ void __launch_bounds__(THREADS) neighbour_kernel(SGrid g, uint32_t* nbr) {
    const size_t e = (size_t)blockIdx.x * THREADS + threadIdx.x;
    if (e >= 27 * (size_t)g.n) return;
    const uint32_t b = (uint32_t)(e / 27), q = (uint32_t)(e % 27);
    int c[3];
    block_of(g.keys[b], c);
    const int d[3] = {(int)(q % 3) - 1, (int)((q / 3) % 3) - 1, (int)(q / 9) - 1};
    bool in = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        c[a] += d[a];
        in = in && c[a] >= -BLK_HALF && c[a] < BLK_HALF;
    }
    nbr[e] = in ? find_key(g.keys, g.n, block_key(c[0], c[1], c[2])) : NONE;
}

// lattice indices of voxel v of block b
__device__ __forceinline__ void voxel_ijk(const SGrid& g, uint32_t b, uint32_t v, int ijk[3]) {
    int c[3];
    block_of(g.keys[b], c);
    ijk[0] = SB * c[0] + (int)(v & 7);
    ijk[1] = SB * c[1] + (int)((v >> 3) & 7);
    ijk[2] = SB * c[2] + (int)(v >> 6);
}

__global__ void __launch_bounds__(THREADS) sparse_integrate_kernel(SGrid g, FuseView f) {
    const uint32_t b = blockIdx.x >> 1, v = ((blockIdx.x & 1) << 8) | threadIdx.x;
    int ijk[3];
    voxel_ijk(g, b, v, ijk);
    const float X = fadd(g.o[0], fmul(g.s, (float)ijk[0]));
    const float Y = fadd(g.o[1], fmul(g.s, (float)ijk[1]));
    const float Z = fadd(g.o[2], fmul(g.s, (float)ijk[2]));
    float* p = g.pool + (size_t)b * POOL_FLOATS + v;
    tsdf_update(f, X, Y, Z, p, p + SB3, p + 2 * SB3, SB3);
}

// ---- extraction ---------------------------------------------------------------------------------------------------------
// the point id (slot * 512 + voxel) of local point (x, y, z) of block b, each coordinate in [-1, 8]; NONE when unallocated
__device__ __forceinline__ uint32_t point_id(const SGrid& g, uint32_t b, int x, int y, int z) {
    const int dx = x < 0 ? -1 : x >= SB ? 1 : 0, dy = y < 0 ? -1 : y >= SB ? 1 : 0, dz = z < 0 ? -1 : z >= SB ? 1 : 0;
    const uint32_t nb = (dx | dy | dz) ? g.nbr[27 * (size_t)b + (dx + 1) + 3 * (dy + 1) + 9 * (dz + 1)] : b;
    return nb == NONE ? NONE : nb * SB3 + (uint32_t)((x & 7) | ((y & 7) << 3) | ((z & 7) << 6));
}
__device__ __forceinline__ const float* point_ptr(const SGrid& g, uint32_t id) { return g.pool + (size_t)(id >> 9) * POOL_FLOATS + (id & 511); }
__device__ __forceinline__ float tsdf_at(const SGrid& g, uint32_t id) { return point_ptr(g, id)[0]; }
__device__ __forceinline__ bool observed(const SGrid& g, uint32_t id) { return id != NONE && point_ptr(g, id)[SB3] > 0.0f; }

// count scratch: act[16 n] (bit v of block b's words: the cell with lower corner voxel v is active) | totals | compaction counters
struct Totals {
    unsigned long long vertices, quads, observed;
    int lo[3], hi[3];
    unsigned int ctr[2];
};
struct SScratch {
    uint32_t* act;
    Totals* tot;
};
size_t scratch_carve(void* ws, uint32_t n, SScratch* out) {
    Carver c(ws);
    SScratch m;
    m.act = c.take<uint32_t>((size_t)16 * n);
    m.tot = c.take<Totals>(1);
    if (out) *out = m;
    return c.total();
}
__device__ __forceinline__ bool act_at(const uint32_t* act, uint32_t id) { return id != NONE && ((act[id >> 5] >> (id & 31)) & 1u); }

// the lattice edge of axis a from local point (x, y, z) of block b makes a quad (edge_quad of mesh.cu through the neighbour table)
__device__ __forceinline__ bool sparse_edge_quad(const SGrid& g, const uint32_t* act, uint32_t b, const int p[3], int a) {
    const int bb = a == 2 ? 0 : a + 1, cc = a == 0 ? 2 : a - 1;
    const uint32_t L = point_id(g, b, p[0], p[1], p[2]);
    int q[3] = {p[0], p[1], p[2]};
    q[a] += 1;
    const uint32_t B = point_id(g, b, q[0], q[1], q[2]);
    if (!observed(g, L) || !observed(g, B)) return false;
    if ((tsdf_at(g, L) < 0.0f) == (tsdf_at(g, B) < 0.0f)) return false;
    int c0[3] = {p[0], p[1], p[2]}, c1[3] = {p[0], p[1], p[2]}, c3[3] = {p[0], p[1], p[2]};
    c0[bb] -= 1; c0[cc] -= 1;
    c1[cc] -= 1;
    c3[bb] -= 1;
    return act_at(act, point_id(g, b, c0[0], c0[1], c0[2])) && act_at(act, point_id(g, b, c1[0], c1[1], c1[2])) &&
           act_at(act, L) && act_at(act, point_id(g, b, c3[0], c3[1], c3[2]));
}

template <typename T>
__device__ __forceinline__ T cta_sum(T v, T* warp_tot) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < THREADS / 32; ++w) t += warp_tot[w];
    __syncthreads();
    return t;
}

// act bits, the vertex and observed-point totals and the lattice bounding box: one thread per voxel, two CTAs per block
__global__ void __launch_bounds__(THREADS) sparse_active_kernel(SGrid g, SScratch m) {
    __shared__ unsigned long long warp_tot[THREADS / 32];
    const uint32_t b = blockIdx.x >> 1, v = ((blockIdx.x & 1) << 8) | threadIdx.x;
    const int p[3] = {(int)(v & 7), (int)((v >> 3) & 7), (int)(v >> 6)};
    const uint32_t self = b * SB3 + v;
    bool act = true;
    int inside = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const uint32_t c = point_id(g, b, p[0] + (q & 1), p[1] + ((q >> 1) & 1), p[2] + (q >> 2));
        if (!observed(g, c)) { act = false; break; }
        inside += tsdf_at(g, c) < 0.0f ? 1 : 0;
    }
    act = act && inside != 0 && inside != 8;
    const bool obs = observed(g, self);
    const uint32_t ba = __ballot_sync(0xffffffffu, act), bo = __ballot_sync(0xffffffffu, obs);
    unsigned long long nv = 0, no = 0;
    if ((threadIdx.x & 31) == 0) {
        m.act[self >> 5] = ba;
        nv = __popc(ba);
        no = __popc(bo);
    }
    const unsigned long long tv = cta_sum(nv, warp_tot), to = cta_sum(no, warp_tot);
    if (threadIdx.x == 0) {
        if (tv) atomicAdd(&m.tot->vertices, tv);
        if (to) atomicAdd(&m.tot->observed, to);
        if (!(blockIdx.x & 1)) {
            int c[3];
            block_of(g.keys[b], c);
            for (int a = 0; a < 3; ++a) {
                atomicMin(&m.tot->lo[a], SB * c[a]);
                atomicMax(&m.tot->hi[a], SB * c[a] + SB - 1);
            }
        }
    }
}

__global__ void __launch_bounds__(THREADS) sparse_edges_kernel(SGrid g, SScratch m) {
    __shared__ unsigned long long warp_tot[THREADS / 32];
    const uint32_t b = blockIdx.x >> 1, v = ((blockIdx.x & 1) << 8) | threadIdx.x;
    const int p[3] = {(int)(v & 7), (int)((v >> 3) & 7), (int)(v >> 6)};
    unsigned long long ne = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) ne += sparse_edge_quad(g, m.act, b, p, a) ? 1u : 0u;
    const unsigned long long te = cta_sum(ne, warp_tot);
    if (threadIdx.x == 0 && te) atomicAdd(&m.tot->quads, te);
}

// the active cells' keys and the quad edges' keys, each with its point id, in atomic order (the sort makes it canonical)
__global__ void __launch_bounds__(THREADS)
sparse_collect_kernel(SGrid g, SScratch m, uint64_t* vkeys, uint32_t* vids, uint64_t* qkeys, uint32_t* qids) {
    const uint32_t b = blockIdx.x >> 1, v = ((blockIdx.x & 1) << 8) | threadIdx.x;
    const int p[3] = {(int)(v & 7), (int)((v >> 3) & 7), (int)(v >> 6)};
    const uint32_t self = b * SB3 + v;
    int ijk[3];
    voxel_ijk(g, b, v, ijk);
    const uint64_t key = cell_key(ijk[0], ijk[1], ijk[2]);
    if (act_at(m.act, self)) {
        const unsigned int q = atomicAdd(&m.tot->ctr[0], 1u);
        vkeys[q] = key;
        vids[q] = self;
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
        if (sparse_edge_quad(g, m.act, b, p, a)) {
            const unsigned int q = atomicAdd(&m.tot->ctr[1], 1u);
            qkeys[q] = (key << 2) | (uint64_t)a;
            qids[q] = self;
        }
}

__global__ void __launch_bounds__(THREADS)
sparse_vertex_kernel(SGrid g, uint32_t V, const uint32_t* __restrict__ vids, float* __restrict__ xyz, uint8_t* __restrict__ rgb) {
    const uint32_t r = blockIdx.x * THREADS + threadIdx.x;
    if (r >= V) return;
    const uint32_t id = vids[r], b = id >> 9, v = id & 511;
    const int p[3] = {(int)(v & 7), (int)((v >> 3) & 7), (int)(v >> 6)};
    float t[8], col[3][8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const float* c = point_ptr(g, point_id(g, b, p[0] + (q & 1), p[1] + ((q >> 1) & 1), p[2] + (q >> 2)));
        t[q] = c[0];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) col[ch][q] = c[(2 + ch) * SB3];
    }
    int ijk[3];
    voxel_ijk(g, b, v, ijk);
    float x[3];
    uint8_t c[3];
    surface_vertex(t, col, ijk, g.o, g.s, x, c);
#pragma unroll
    for (int a = 0; a < 3; ++a) { xyz[3 * (size_t)r + a] = x[a]; rgb[3 * (size_t)r + a] = c[a]; }
}

// quad r: the vertex ids of its four cells (their ranks among the sorted cell keys), wound as mesh_emit_kernel winds them
__global__ void __launch_bounds__(THREADS)
sparse_face_kernel(SGrid g, uint32_t V, uint32_t Q, const uint64_t* __restrict__ vkeys, const uint64_t* __restrict__ qkeys,
                   const uint32_t* __restrict__ qids, int* __restrict__ faces) {
    const uint32_t r = blockIdx.x * THREADS + threadIdx.x;
    if (r >= Q) return;
    const int a = (int)(qkeys[r] & 3), bb = a == 2 ? 0 : a + 1, cc = a == 0 ? 2 : a - 1;
    const uint32_t self = qids[r];
    int ijk[3];
    voxel_ijk(g, self >> 9, self & 511, ijk);
    int cell[4][3];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int e = 0; e < 3; ++e) cell[q][e] = ijk[e];
    cell[0][bb] -= 1; cell[0][cc] -= 1;
    cell[1][cc] -= 1;
    cell[3][bb] -= 1;
    const bool keep = tsdf_at(g, self) < 0.0f;
    int id[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int* c = cell[keep ? q : 3 - q];
        id[q] = (int)find_key(vkeys, V, cell_key(c[0], c[1], c[2]));
    }
    int* t = faces + 6 * (size_t)r;
    t[0] = id[0]; t[1] = id[1]; t[2] = id[2];
    t[3] = id[0]; t[4] = id[2]; t[5] = id[3];
}

// extraction workspace of V vertices and Q quads: vertex keys and ids, in and sorted | quad keys and ids, in and sorted | temp
struct SortWs {
    uint64_t *vk_in, *vk, *qk_in, *qk;
    uint32_t *vi_in, *vi, *qi_in, *qi;
    void* temp;
    size_t temp_bytes;
};
size_t sort_carve(void* ws, uint64_t V, uint64_t Q, SortWs* out) {
    Carver c(ws);
    SortWs w;
    w.vk_in = c.take<uint64_t>(V); w.vk = c.take<uint64_t>(V);
    w.vi_in = c.take<uint32_t>(V); w.vi = c.take<uint32_t>(V);
    w.qk_in = c.take<uint64_t>(Q); w.qk = c.take<uint64_t>(Q);
    w.qi_in = c.take<uint32_t>(Q); w.qi = c.take<uint32_t>(Q);
    w.temp_bytes = sort_temp_bytes((int64_t)std::max<uint64_t>(std::max(V, Q), 1));
    w.temp = c.take<char>(w.temp_bytes);
    if (out) *out = w;
    return c.total();
}

inline unsigned grid_ctas(uint32_t n) { return 2u * n; }

}  // namespace
}  // namespace glic

using namespace glic;

extern "C" {

size_t glic_block_set_bytes(uint32_t capacity) {
    return capacity >= 1 && capacity <= MAX_CAPACITY ? sizeof(unsigned long long) * (SET_HEADER + 2 * (size_t)capacity) : 0;
}

int glic_block_set_clear(const glic_block_set* set, void* stream) {
    if (!set_ok(set)) { set_error("block_set_clear: null set or capacity not in [1, 2^24]"); return GLIC_ERR_INVALID_ARGUMENT; }
    const SetView v = set_view(*set);
    GLIC_CUDA_TRY(cudaMemsetAsync(v.hdr, 0, sizeof(unsigned long long) * SET_HEADER, (cudaStream_t)stream));
    GLIC_CUDA_TRY(cudaMemsetAsync(v.slots, 0xFF, sizeof(unsigned long long) * v.nslots, (cudaStream_t)stream));
    return GLIC_OK;
}

int glic_block_set_copy(const glic_block_set* src, const glic_block_set* dst, void* stream) {
    if (!set_ok(src) || !set_ok(dst)) { set_error("block_set_copy: null set or capacity not in [1, 2^24]"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (dst->capacity / 2 < src->capacity || dst->data == src->data) {
        set_error("block_set_copy: the destination must be another set of at least twice the source's capacity"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    const SetView s = set_view(*src);
    SPARSE_TRY(glic_block_set_clear(dst, stream));
    block_copy_kernel<<<(unsigned)((s.nslots + THREADS - 1) / THREADS), THREADS, 0, (cudaStream_t)stream>>>(s, set_view(*dst));
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int glic_block_set_insert(const glic_block_set* set, const float* origin, float voxel_size, const float* viewmatrix_dev, int W, int H,
                          float fx, float fy, float cx, float cy, const float* depth, const uint32_t* mask_words, int words_per_row,
                          float trunc, float max_depth, int64_t* counters_host, void* stream) {
    if (!set_ok(set)) { set_error("block_set_insert: null set or capacity not in [1, 2^24]"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!origin || !counters_host) { set_error("block_set_insert: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!(std::isfinite(voxel_size) && voxel_size > 0.0f) || !std::isfinite(origin[0]) || !std::isfinite(origin[1]) || !std::isfinite(origin[2])) {
        set_error("block_set_insert: voxel_size must be finite and > 0, the origin finite"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    const FuseView f{viewmatrix_dev, W, H, fx, fy, cx, cy, depth, nullptr, mask_words, words_per_row, trunc, max_depth};
    if (const int e = fuse_view_check(f, "block_set_insert")) return e;
    cudaStream_t s = (cudaStream_t)stream;
    const SetView v = set_view(*set);
    GLIC_CUDA_TRY(cudaMemsetAsync(v.hdr + 1, 0, 2 * sizeof(unsigned long long), s));
    const uint32_t npix = (uint32_t)W * (uint32_t)H;
    block_insert_kernel<<<(npix + THREADS - 1) / THREADS, THREADS, 0, s>>>(v, origin[0], origin[1], origin[2], voxel_size, f);
    GLIC_LAUNCH_CHECK();
    GLIC_CUDA_TRY(cudaMemcpyAsync(counters_host, v.hdr, 3 * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    return GLIC_OK;
}

size_t glic_sparse_tsdf_bytes(uint32_t n_blocks) { return n_blocks <= MAX_BLOCKS ? grid_layout(nullptr, n_blocks).total : 0; }

int glic_sparse_tsdf_init(const glic_sparse_tsdf* grid, const glic_block_set* set, void* stream) {
    if (const int e = sgrid_check(grid, "sparse_tsdf_init")) return e;
    if (!set_ok(set)) { set_error("sparse_tsdf_init: null set or capacity not in [1, 2^24]"); return GLIC_ERR_INVALID_ARGUMENT; }
    const uint32_t n = grid->n_blocks;
    if (!n) return GLIC_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const GridLayout L = grid_layout(grid->data, n);
    const SetView v = set_view(*set);
    GLIC_CUDA_TRY(cudaMemsetAsync(L.ctr, 0, sizeof(unsigned int), s));
    compact_kernel<<<(unsigned)((v.nslots + THREADS - 1) / THREADS), THREADS, 0, s>>>(v, n, L.ctr, L.keys_in, L.vals_in);
    GLIC_LAUNCH_CHECK();
    SPARSE_TRY(glic_sort_pairs_u64_u32(n, 51, L.keys_in, L.vals_in, L.keys, L.vals_out, L.temp, L.temp_bytes, stream));
    const SGrid g = device_sgrid(*grid);
    neighbour_kernel<<<(unsigned)((27 * (size_t)n + THREADS - 1) / THREADS), THREADS, 0, s>>>(g, L.nbr);
    GLIC_LAUNCH_CHECK();
    GLIC_CUDA_TRY(cudaMemsetAsync(L.pool, 0, sizeof(float) * POOL_FLOATS * (size_t)n, s));
    return GLIC_OK;
}

int glic_sparse_tsdf_integrate(const glic_sparse_tsdf* grid, const float* viewmatrix_dev, int W, int H, float fx, float fy, float cx, float cy,
                               const float* depth, const float* rgb, const uint32_t* mask_words, int words_per_row, float trunc,
                               float max_depth, void* stream) {
    if (const int e = sgrid_check(grid, "sparse_tsdf_integrate")) return e;
    const FuseView f{viewmatrix_dev, W, H, fx, fy, cx, cy, depth, rgb, mask_words, words_per_row, trunc, max_depth};
    if (const int e = fuse_view_check(f, "sparse_tsdf_integrate")) return e;
    if (!grid->n_blocks) return GLIC_OK;
    sparse_integrate_kernel<<<grid_ctas(grid->n_blocks), THREADS, 0, (cudaStream_t)stream>>>(device_sgrid(*grid), f);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

size_t glic_sparse_mesh_scratch_bytes(uint32_t n_blocks) { return n_blocks <= MAX_BLOCKS ? scratch_carve(nullptr, n_blocks, nullptr) : 0; }

size_t glic_sparse_mesh_extract_bytes(uint32_t vertices, uint32_t faces) { return sort_carve(nullptr, vertices, faces / 2, nullptr); }

int glic_sparse_mesh_count(const glic_sparse_tsdf* grid, void* scratch, size_t scratch_bytes, glic_sparse_mesh_counts* counts_host,
                           void* stream) {
    if (const int e = sgrid_check(grid, "sparse_mesh_count")) return e;
    if (!scratch || !counts_host) { set_error("sparse_mesh_count: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t need = glic_sparse_mesh_scratch_bytes(grid->n_blocks);
    if (scratch_bytes < need) {
        set_error("sparse_mesh_count: scratch of " + std::to_string(scratch_bytes) + " bytes, glic_sparse_mesh_scratch_bytes needs " + std::to_string(need));
        return GLIC_ERR_WORKSPACE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    SScratch m;
    scratch_carve(scratch, grid->n_blocks, &m);
    Totals t{};
    for (int a = 0; a < 3; ++a) { t.lo[a] = LAT_HALF; t.hi[a] = -LAT_HALF - 1; }
    GLIC_CUDA_TRY(cudaMemcpyAsync(m.tot, &t, sizeof(t), cudaMemcpyHostToDevice, s));
    if (grid->n_blocks) {
        const SGrid g = device_sgrid(*grid);
        sparse_active_kernel<<<grid_ctas(g.n), THREADS, 0, s>>>(g, m);
        GLIC_LAUNCH_CHECK();
        sparse_edges_kernel<<<grid_ctas(g.n), THREADS, 0, s>>>(g, m);
        GLIC_LAUNCH_CHECK();
    }
    GLIC_CUDA_TRY(cudaMemcpyAsync(&t, m.tot, sizeof(t), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    if (t.vertices > 0x7FFFFFFFull || 2 * t.quads > 0xFFFFFFFFull) {
        set_error("sparse_mesh_count: more than 2^31 - 1 vertices or 2^32 - 1 faces"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    glic_sparse_mesh_counts c{};
    c.vertices = (uint32_t)t.vertices;
    c.faces = (uint32_t)(2 * t.quads);
    c.observed_voxels = t.observed;
    c.blocks = grid->n_blocks;
    for (int a = 0; a < 3; ++a) {
        c.lattice_lo[a] = grid->n_blocks ? t.lo[a] : 0;
        c.lattice_hi[a] = grid->n_blocks ? t.hi[a] : -1;
    }
    *counts_host = c;
    return GLIC_OK;
}

int glic_sparse_mesh_extract(const glic_sparse_tsdf* grid, void* scratch, size_t scratch_bytes, const glic_sparse_mesh_counts* counts,
                             void* extract_ws, size_t extract_bytes, float* xyz, uint8_t* rgb, int32_t* faces, void* stream) {
    if (const int e = sgrid_check(grid, "sparse_mesh_extract")) return e;
    if (!scratch || !counts) { set_error("sparse_mesh_extract: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const uint32_t V = counts->vertices, Q = counts->faces / 2;
    if ((V && (!xyz || !rgb)) || (Q && !faces) || ((V || Q) && !extract_ws)) { set_error("sparse_mesh_extract: null output"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (scratch_bytes < glic_sparse_mesh_scratch_bytes(grid->n_blocks) || extract_bytes < glic_sparse_mesh_extract_bytes(V, counts->faces)) {
        set_error("sparse_mesh_extract: scratch under glic_sparse_mesh_scratch_bytes or workspace under glic_sparse_mesh_extract_bytes");
        return GLIC_ERR_WORKSPACE;
    }
    if (!V && !Q) return GLIC_OK;
    cudaStream_t s = (cudaStream_t)stream;
    SScratch m;
    scratch_carve(scratch, grid->n_blocks, &m);
    SortWs w;
    sort_carve(extract_ws, V, Q, &w);
    const SGrid g = device_sgrid(*grid);
    GLIC_CUDA_TRY(cudaMemsetAsync(m.tot->ctr, 0, sizeof(m.tot->ctr), s));
    sparse_collect_kernel<<<grid_ctas(g.n), THREADS, 0, s>>>(g, m, w.vk_in, w.vi_in, w.qk_in, w.qi_in);
    GLIC_LAUNCH_CHECK();
    SPARSE_TRY(glic_sort_pairs_u64_u32(V, 60, w.vk_in, w.vi_in, w.vk, w.vi, w.temp, w.temp_bytes, stream));
    SPARSE_TRY(glic_sort_pairs_u64_u32(Q, 62, w.qk_in, w.qi_in, w.qk, w.qi, w.temp, w.temp_bytes, stream));
    if (V) {
        sparse_vertex_kernel<<<(V + THREADS - 1) / THREADS, THREADS, 0, s>>>(g, V, w.vi, xyz, rgb);
        GLIC_LAUNCH_CHECK();
    }
    if (Q) {
        sparse_face_kernel<<<(Q + THREADS - 1) / THREADS, THREADS, 0, s>>>(g, V, Q, w.vk, w.qk, w.qi, faces);
        GLIC_LAUNCH_CHECK();
    }
    return GLIC_OK;
}

int glic_debug_sparse_tsdf(const glic_sparse_tsdf* grid, uint64_t* keys, float* data, void* stream) {
    if (const int e = sgrid_check(grid, "debug_sparse_tsdf")) return e;
    if (!grid->n_blocks) return GLIC_OK;
    if (!keys || !data) { set_error("debug_sparse_tsdf: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const GridLayout L = grid_layout(grid->data, grid->n_blocks);
    cudaStream_t s = (cudaStream_t)stream;
    GLIC_CUDA_TRY(cudaMemcpyAsync(keys, L.keys, sizeof(uint64_t) * grid->n_blocks, cudaMemcpyDefault, s));
    GLIC_CUDA_TRY(cudaMemcpyAsync(data, L.pool, sizeof(float) * POOL_FLOATS * (size_t)grid->n_blocks, cudaMemcpyDefault, s));
    return GLIC_OK;
}

}  // extern "C"

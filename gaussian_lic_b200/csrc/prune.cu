// prune.cu -- stable compaction of the mapper's arenas (glic_mapper_prune): every row whose activated opacity is below a
// threshold is removed, the survivors keep their relative order, and all six parameter groups and both Adam moments move with
// them bit for bit.  No CUB:
//   1. prune_count_kernel: one CTA per tile of PRUNE_TILE rows counts the rows it keeps;
//   2. prune_scan_kernel:  one CTA scans the per-tile counts (a two-level scan: rows within a tile in step 3, tiles here; at
//      1024 rows per tile a 2 M-row map has 2048 tile counts) into tile offsets and the kept total;
//   3. prune_index_kernel: each tile places its kept rows at their new index: idx[new] = old, and the new index of row n_sky,
//      i.e. the number of kept rows before it (the surviving sky rows);
//   4. prune_gather_kernel: per arena, one launch over all six groups writes output rows [0, P_old) of each group: row r < P_new
//      takes source row idx[r], rows [P_new, P_old) become zero.  Each thread writes one float4 of a group (16-byte aligned:
//      group offsets are multiples of Pcap floats, Pcap a multiple of 256); its four source floats are consecutive whenever
//      their rows are, so loads coalesce across a run of kept rows.
// The keep decision is opacity_activation(logit) >= min_opacity, the activation kernel's own expression (common.cuh).
#include "common.cuh"

namespace glic {
namespace {

constexpr int PRUNE_THREADS = 256;
constexpr int PRUNE_ROWS = 4;                                  // consecutive rows per thread
constexpr uint32_t PRUNE_TILE = PRUNE_THREADS * PRUNE_ROWS;    // rows per CTA of the count and index passes

// the keep flags of this thread's rows [r0, r0 + 4): a float4 load when all four exist (r0 is a multiple of 4, the group
// offset a multiple of Pcap floats)
__device__ __forceinline__ void keep_flags(uint32_t P, const float* __restrict__ logit, float min_opacity, uint32_t r0, bool keep[PRUNE_ROWS]) {
    float l[PRUNE_ROWS];
    if (r0 + PRUNE_ROWS <= P) {
        const float4 v = *reinterpret_cast<const float4*>(logit + r0);
        l[0] = v.x; l[1] = v.y; l[2] = v.z; l[3] = v.w;
    } else {
#pragma unroll
        for (int e = 0; e < PRUNE_ROWS; ++e) l[e] = r0 + e < P ? logit[r0 + e] : 0.0f;
    }
#pragma unroll
    for (int e = 0; e < PRUNE_ROWS; ++e) keep[e] = r0 + e < P && !(opacity_activation(l[e]) < min_opacity);
}

__global__ void __launch_bounds__(PRUNE_THREADS)
prune_count_kernel(uint32_t P, const float* __restrict__ logit, float min_opacity, uint32_t* __restrict__ tile_count) {
    bool keep[PRUNE_ROWS];
    keep_flags(P, logit, min_opacity, blockIdx.x * PRUNE_TILE + PRUNE_ROWS * threadIdx.x, keep);
    int n = 0;
#pragma unroll
    for (int e = 0; e < PRUNE_ROWS; ++e) n += keep[e];
    __shared__ int warp_n[PRUNE_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0) warp_n[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < PRUNE_THREADS / 32; ++w) t += warp_n[w];
        tile_count[blockIdx.x] = (uint32_t)t;
    }
}

// exclusive scan of the tile counts in place, the total into *total
__global__ void __launch_bounds__(1024) prune_scan_kernel(uint32_t n_tiles, uint32_t* __restrict__ tile, uint32_t* __restrict__ total) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n_tiles; base += 1024) {
        const uint32_t i = base + tid;
        const uint32_t f = i < n_tiles ? tile[i] : 0u;
        uint32_t incl = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const uint32_t w = warp_tot[lane];
            uint32_t wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            warp_tot[lane] = wi - w;
        }
        __syncthreads();
        const uint32_t excl = carry + warp_tot[warp] + incl - f;
        if (i < n_tiles) tile[i] = excl;
        __syncthreads();
        if (tid == 1023) carry = excl + f;
        __syncthreads();
    }
    if (tid == 0) *total = carry;
}

// idx[new] = old for every kept row; *sky_new = the new index of row n_sky (written only when n_sky < P)
__global__ void __launch_bounds__(PRUNE_THREADS)
prune_index_kernel(uint32_t P, const float* __restrict__ logit, float min_opacity, const uint32_t* __restrict__ tile_offset, uint32_t n_sky,
                   uint32_t* __restrict__ idx, uint32_t* __restrict__ sky_new) {
    const uint32_t r0 = blockIdx.x * PRUNE_TILE + PRUNE_ROWS * threadIdx.x;
    bool keep[PRUNE_ROWS];
    keep_flags(P, logit, min_opacity, r0, keep);
    uint32_t n = 0;
#pragma unroll
    for (int e = 0; e < PRUNE_ROWS; ++e) n += keep[e];
    // exclusive scan of n over the CTA, in thread (= row) order
    __shared__ uint32_t warp_tot[PRUNE_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    uint32_t before = 0;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    uint32_t pos = tile_offset[blockIdx.x] + before + incl - n;
#pragma unroll
    for (int e = 0; e < PRUNE_ROWS; ++e) {
        if (r0 + e == n_sky) *sky_new = pos;
        if (keep[e]) idx[pos++] = r0 + e;
    }
}

struct GatherPlan {
    size_t off[6];          // float offset of each group in both arenas (the same capacity)
    int k[6];               // floats per row
    uint32_t first[7];      // first block of each group in the flattened grid; first[6] = the grid
};

template <int K>
__device__ __forceinline__ void gather_float4(const float* __restrict__ src, float* __restrict__ dst, const uint32_t* __restrict__ idx,
                                              uint32_t P_new, size_t t) {
    float v[4];
    if (K == 4) {
        const float4 q = t < P_new ? reinterpret_cast<const float4*>(src)[idx[t]] : make_float4(0.f, 0.f, 0.f, 0.f);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const size_t j = 4 * t + e;
            const size_t r = j / K;
            v[e] = r < P_new ? src[(size_t)idx[r] * K + (j - r * K)] : 0.0f;
        }
    }
    reinterpret_cast<float4*>(dst)[t] = make_float4(v[0], v[1], v[2], v[3]);
}

__global__ void __launch_bounds__(256)
prune_gather_kernel(const float* __restrict__ src, float* __restrict__ dst, const uint32_t* __restrict__ idx, uint32_t P_old, uint32_t P_new,
                    GatherPlan g) {
    int K = g.k[0];                                            // this block's group (static indices: the plan stays in registers)
    size_t off = g.off[0];
    uint32_t first = 0;
#pragma unroll
    for (int e = 1; e < 6; ++e)
        if (blockIdx.x >= g.first[e]) { K = g.k[e]; off = g.off[e]; first = g.first[e]; }
    const size_t t = (size_t)(blockIdx.x - first) * blockDim.x + threadIdx.x;
    if (t >= ((size_t)P_old * K + 3) / 4) return;
    const float* s = src + off;
    float* d = dst + off;
    switch (K) {
        case 1: gather_float4<1>(s, d, idx, P_new, t); break;
        case 3: gather_float4<3>(s, d, idx, P_new, t); break;
        case 4: gather_float4<4>(s, d, idx, P_new, t); break;
        case 9: gather_float4<9>(s, d, idx, P_new, t); break;
        case 24: gather_float4<24>(s, d, idx, P_new, t); break;
        case 45: gather_float4<45>(s, d, idx, P_new, t); break;
        default: break;
    }
}

}  // namespace

size_t prune_scratch_bytes(uint32_t P) {
    const uint32_t tiles = (P + PRUNE_TILE - 1) / PRUNE_TILE;
    return 256 + (((size_t)tiles * 4 + 255) & ~size_t(255)) + (size_t)P * 4;
}

// scratch: result[2] = {P_new, sky_new} (256 bytes) | tile counts | idx[P]
int launch_prune_select(uint32_t P, uint32_t n_sky, const float* opacity_logit, float min_opacity, void* scratch, uint32_t* result_host,
                        cudaStream_t s) {
    const uint32_t tiles = (P + PRUNE_TILE - 1) / PRUNE_TILE;
    uint32_t* result = static_cast<uint32_t*>(scratch);
    uint32_t* tile = reinterpret_cast<uint32_t*>(static_cast<char*>(scratch) + 256);
    uint32_t* idx = reinterpret_cast<uint32_t*>(static_cast<char*>(scratch) + 256 + (((size_t)tiles * 4 + 255) & ~size_t(255)));
    GLIC_CUDA_TRY(cudaMemsetAsync(result, 0, 2 * sizeof(uint32_t), s));
    prune_count_kernel<<<tiles, PRUNE_THREADS, 0, s>>>(P, opacity_logit, min_opacity, tile);
    GLIC_LAUNCH_CHECK();
    prune_scan_kernel<<<1, 1024, 0, s>>>(tiles, tile, result);
    GLIC_LAUNCH_CHECK();
    prune_index_kernel<<<tiles, PRUNE_THREADS, 0, s>>>(P, opacity_logit, min_opacity, tile, n_sky, idx, result + 1);
    GLIC_LAUNCH_CHECK();
    GLIC_CUDA_TRY(cudaMemcpyAsync(result_host, result, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    if (n_sky >= P) result_host[1] = result_host[0];            // every row is sky: the survivors are
    return GLIC_OK;
}

int launch_prune_gather(const float* src, float* dst, uint32_t Pcap, int M, uint32_t P_old, uint32_t P_new, const void* scratch, cudaStream_t s) {
    const uint32_t tiles = (P_old + PRUNE_TILE - 1) / PRUNE_TILE;
    const uint32_t* idx = reinterpret_cast<const uint32_t*>(static_cast<const char*>(scratch) + 256 + (((size_t)tiles * 4 + 255) & ~size_t(255)));
    GatherPlan g;
    glic_packed_offsets(Pcap, (uint32_t)M, g.off);
    const int k[6] = {4, 3, 3, 1, 3, 3 * M};
    g.first[0] = 0;
    for (int q = 0; q < 6; ++q) {
        g.k[q] = k[q];
        g.first[q + 1] = g.first[q] + (uint32_t)((((size_t)P_old * k[q] + 3) / 4 + 255) / 256);
    }
    if (g.first[6] == 0) return GLIC_OK;
    prune_gather_kernel<<<g.first[6], 256, 0, s>>>(src, dst, idx, P_old, P_new, g);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

}  // namespace glic

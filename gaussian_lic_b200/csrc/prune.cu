// prune.cu -- the one stable compaction of the mapper's arenas, behind glic_mapper_prune, glic_mapper_densify and
// glic_mapper_densify_and_prune.  Each row is kept, cloned (kept and copied once) or split (replaced by two children), and each
// of the rows it leaves in the densify result survives the prune predicate or not (row_fate).  The survivors keep their relative
// order, and all six parameter groups and both Adam moments move with them bit for bit.  glic_mapper_densify is the case without
// a prune; glic_mapper_prune is the case in which no row is selected (no statistics are given, and none are read) and both
// size tests are off, so a row's fate is its logit's alone.  No CUB:
//   1. fate_count_kernel: one CTA per tile of PRUNE_TILE rows counts its clones and splits, and the survivors of each kind;
//   2. prune_scan_kernel, one CTA per count: scans the per-tile counts (a two-level scan: rows within a tile in step 3, tiles
//      here; at 1024 rows per tile a 2 M-row map has 2048 tile counts) into tile offsets and the five totals;
//   3. fate_index_kernel: idx[new] = old for the surviving kept rows (rows that are not split, in order), then the surviving
//      clones, then the first child of every surviving split row, then the second; the children's rows start as copies of their
//      parent, and each child's key is the row it has in the densify result before the prune.  It also finds the new index of
//      row n_sky, i.e. the number of kept rows before it (the surviving sky rows);
//   4. prune_gather_kernel: per arena, one launch over all six groups writes output rows [0, rows_out) of each group: row
//      r < rows_valid takes source row idx[r], the others become zero (the rows a prune vacates; for the moments, every new
//      row).  Each thread writes one float4 of a group (16-byte aligned: group offsets are multiples of Pcap floats, Pcap a
//      multiple of 256); its four source floats are consecutive whenever their rows are, so loads coalesce across a run of
//      kept rows;
//   5. densify_children_kernel: each child row, a copy of its parent, gets its own xyz (drawn at its key) and the parent's
//      log-scale - log(1.6).
// The decisions use the activation kernel's own expressions (opacity_activation, scale_activation: common.cuh) and the child
// geometry its normalisation (rotation_activation); glic_densify_split evaluates the same child geometry on its own.
#include "common.cuh"

namespace glic {
namespace {

constexpr int PRUNE_THREADS = 256;
constexpr int PRUNE_ROWS = 4;                                  // consecutive rows per thread
constexpr uint32_t PRUNE_TILE = PRUNE_THREADS * PRUNE_ROWS;    // rows per CTA of the count and index passes

// exclusive scan of the tile counts in place, the total into *total; CTA b scans the b-th of consecutive arrays of n_tiles
// counts into total[b]
__global__ void __launch_bounds__(1024) prune_scan_kernel(uint32_t n_tiles, uint32_t* __restrict__ tile, uint32_t* __restrict__ total) {
    tile += (size_t)blockIdx.x * n_tiles;
    total += blockIdx.x;
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

int launch_gather_rows(const float* src, float* dst, uint32_t Pcap, int M, uint32_t P_old, uint32_t P_new, const uint32_t* idx,
                       cudaStream_t s) {
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

// ---- densification ---------------------------------------------------------------------------------------------------
namespace {

constexpr float SPLIT_LOG_SCALE = 0x1.e148a2p-2f;              // (float)log(1.6): log(exp(ls) / (0.8 * 2)) = ls - log(1.6)

// The fate of row r in one densify-and-prune.  Bits 0-1, the densify class: 0 keep, 1 clone, 2 split.  Sky rows are kept;
// grad = accum / denom (0 without a view); selected iff grad >= threshold; a selected row is cloned iff its largest activated
// scale is <= clone_max, split otherwise.  Bits 2-4, which of the densify result's rows that come from r survive the prune
// predicate: the row itself (kept or cloned), its clone, its two children (one logit and one log-scale: one fate).  The
// predicate: act(logit) < min_opacity, or (non-sky rows) maxr > max_screen_radius > 0, or largest scale > max_world_scale > 0.
// Clones and children have maxr 0, and the children's scale is their own (the parent's log-scale - log(1.6)).
// Without statistics (a.accum null) no row is selected; then, with both size tests off, a row's logit is all that is read.
// With the scores (a.score_max, glic_mapper_prune_unseen, where no row is selected) the row itself also goes when it is not a
// sky row, or a.score_sky is set, and its max_weight < min_weight or hits + ends < min_hits (the pixels it takes or ends).
constexpr unsigned FATE_ROW = 4u, FATE_CLONE = 8u, FATE_CHILDREN = 16u;

__device__ __forceinline__ float largest_scale(const float* ls) {
    return fmaxf(fmaxf(scale_activation(ls[0]), scale_activation(ls[1])), scale_activation(ls[2]));
}

__device__ __forceinline__ unsigned row_fate(uint32_t r, const DensitySelect& a) {
    const bool sky = r < a.n_sky;
    const float* ls = a.log_scale + 3 * (size_t)r;
    const bool world = a.max_world_scale > 0.0f;
    unsigned cls = 0;
    float smax = 0.0f;
    if (!sky) {
        bool selected = false;
        if (a.accum) {
            const float d = a.denom[r];
            selected = (d > 0.0f ? __fdiv_rn(a.accum[r], d) : 0.0f) >= a.grad_threshold;
        }
        if (selected) {
            smax = largest_scale(ls);
            cls = smax <= a.clone_max ? 1u : 2u;
        } else if (world) {
            smax = largest_scale(ls);
        }
    }
    const bool faded = opacity_activation(a.logit[r]) < a.min_opacity;
    if (cls == 2u) {
        bool gone = faded;
        if (!gone && world) {
            const float child[3] = {__fsub_rn(ls[0], SPLIT_LOG_SCALE), __fsub_rn(ls[1], SPLIT_LOG_SCALE), __fsub_rn(ls[2], SPLIT_LOG_SCALE)};
            gone = largest_scale(child) > a.max_world_scale;
        }
        return cls | (gone ? 0u : FATE_CHILDREN);
    }
    const bool copy_gone = faded || (!sky && world && smax > a.max_world_scale);
    const bool unseen = a.score_max && (!sky || a.score_sky) && (a.score_max[r] < a.min_weight || a.score_hits[r] + a.score_ends[r] < a.min_hits);
    const bool row_gone = copy_gone || unseen || (!sky && a.max_screen_radius > 0 && a.maxr[r] > a.max_screen_radius);
    return cls | (row_gone ? 0u : FATE_ROW) | (cls == 1u && !copy_gone ? FATE_CLONE : 0u);
}

// the counts of one row, two to a word (at most PRUNE_TILE = 1024 of each per CTA): A = clones | splits << 16 (of the densify
// result), B = surviving kept rows | surviving clones << 16, C = surviving split rows
__device__ __forceinline__ void fate_counts(unsigned f, uint32_t& A, uint32_t& B, uint32_t& C) {
    const unsigned cls = f & 3u;
    A += cls == 1u ? 1u : cls == 2u ? (1u << 16) : 0u;
    if (cls == 2u) C += (f & FATE_CHILDREN) ? 1u : 0u;
    else B += ((f & FATE_ROW) ? 1u : 0u) + ((f & FATE_CLONE) ? (1u << 16) : 0u);
}

// per tile: tile[q * n_tiles + tile] for q = clones, splits, surviving kept rows, surviving clones, surviving split rows
__global__ void __launch_bounds__(PRUNE_THREADS)
fate_count_kernel(DensitySelect a, uint32_t n_tiles, uint32_t* __restrict__ tile) {
    const uint32_t r0 = blockIdx.x * PRUNE_TILE + PRUNE_ROWS * threadIdx.x;
    uint32_t A = 0, B = 0, Cn = 0;
#pragma unroll
    for (int e = 0; e < PRUNE_ROWS; ++e) {
        if (r0 + e >= a.P) break;
        fate_counts(row_fate(r0 + e, a), A, B, Cn);
    }
    __shared__ uint32_t warp_n[3][PRUNE_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        A += __shfl_xor_sync(0xffffffffu, A, o);
        B += __shfl_xor_sync(0xffffffffu, B, o);
        Cn += __shfl_xor_sync(0xffffffffu, Cn, o);
    }
    if ((threadIdx.x & 31) == 0) { warp_n[0][threadIdx.x >> 5] = A; warp_n[1][threadIdx.x >> 5] = B; warp_n[2][threadIdx.x >> 5] = Cn; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t ta = 0, tb = 0, tc = 0;
        for (int w = 0; w < PRUNE_THREADS / 32; ++w) { ta += warp_n[0][w]; tb += warp_n[1][w]; tc += warp_n[2][w]; }
        const uint32_t c[5] = {ta & 0xFFFFu, ta >> 16, tb & 0xFFFFu, tb >> 16, tc};
        for (int q = 0; q < 5; ++q) tile[(size_t)q * n_tiles + blockIdx.x] = c[q];
    }
}

// totals[6] = {clones, splits, surviving kept, surviving clones, surviving split rows (the scans' totals), the new index of
// row n_sky}.  Places every surviving row's source row in idx: the surviving kept rows, the surviving clones, the first then
// the second children of the surviving split rows; key[j] = the row the first child of surviving split j has in the densify
// result before the prune (its second child's is key[j] + splits)
__global__ void __launch_bounds__(PRUNE_THREADS)
fate_index_kernel(DensitySelect a, uint32_t n_tiles, const uint32_t* __restrict__ tile_offset, uint32_t* __restrict__ totals,
                  uint32_t* __restrict__ idx, uint32_t* __restrict__ key) {
    const uint32_t r0 = blockIdx.x * PRUNE_TILE + PRUNE_ROWS * threadIdx.x;
    unsigned f[PRUNE_ROWS];
    uint32_t A = 0, B = 0, Cn = 0;
#pragma unroll
    for (int e = 0; e < PRUNE_ROWS; ++e) {
        f[e] = r0 + e < a.P ? row_fate(r0 + e, a) : 0u;
        if (r0 + e < a.P) fate_counts(f[e], A, B, Cn);
    }
    // exclusive scans of the three count words over the CTA, in thread (= row) order
    __shared__ uint32_t warp_tot[3][PRUNE_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t ia = A, ib = B, ic = Cn;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t ta = __shfl_up_sync(0xffffffffu, ia, o), tb = __shfl_up_sync(0xffffffffu, ib, o), tc = __shfl_up_sync(0xffffffffu, ic, o);
        if (lane >= o) { ia += ta; ib += tb; ic += tc; }
    }
    if (lane == 31) { warp_tot[0][warp] = ia; warp_tot[1][warp] = ib; warp_tot[2][warp] = ic; }
    __syncthreads();
    uint32_t ba = 0, bb = 0, bc = 0;
    for (int w = 0; w < warp; ++w) { ba += warp_tot[0][w]; bb += warp_tot[1][w]; bc += warp_tot[2][w]; }
    const uint32_t ea = ba + ia - A, eb = bb + ib - B, ec = bc + ic - Cn;
    const uint32_t n_clone = totals[0], n_split = totals[1], n_kept = totals[2], n_cloned = totals[3], n_split_s = totals[4];
    uint32_t split = tile_offset[1 * (size_t)n_tiles + blockIdx.x] + (ea >> 16);
    uint32_t kept = tile_offset[2 * (size_t)n_tiles + blockIdx.x] + (eb & 0xFFFFu);
    uint32_t clone = tile_offset[3 * (size_t)n_tiles + blockIdx.x] + (eb >> 16);
    uint32_t child = tile_offset[4 * (size_t)n_tiles + blockIdx.x] + ec;
    const uint32_t first_child = a.P - n_split + n_clone;                  // before the prune
    const uint32_t first_child_s = n_kept + n_cloned;                      // after it
#pragma unroll
    for (int e = 0; e < PRUNE_ROWS; ++e) {
        const uint32_t r = r0 + e;
        if (r >= a.P) break;
        if (r == a.n_sky) totals[5] = kept;
        if ((f[e] & 3u) == 2u) {
            if (f[e] & FATE_CHILDREN) {
                idx[first_child_s + child] = r;
                idx[first_child_s + n_split_s + child] = r;
                key[child++] = first_child + split;
            }
            ++split;
        } else {
            if (f[e] & FATE_ROW) idx[kept++] = r;
            if (f[e] & FATE_CLONE) idx[n_kept + clone++] = r;
        }
    }
}

// child `row` of densify call `call`, axis a: the uniforms of the skybox's generator at counter
// k = ((call + 1) * 2^32 + row) * 3 + a, then Box-Muller
__device__ __forceinline__ float split_normal(uint64_t seed, uint64_t call, uint32_t row, int a) {
    const uint64_t k = (((call + 1) << 32) + row) * 3 + (uint64_t)a;
    const uint64_t r = splitmix64_mix(seed + (k + 1) * 0x9E3779B97F4A7C15ull);
    const float u1 = __fmul_rn((float)(uint32_t)(r >> 40), 5.9604644775390625e-08f);               // * 2^-24: exact
    const float u2 = __fmul_rn((float)(uint32_t)((r >> 16) & 0xFFFFFFu), 5.9604644775390625e-08f);
    const float rad = sqrtf(__fmul_rn(-2.0f, logf(__fsub_rn(1.0f, u1))));
    return __fmul_rn(rad, cospif(__fmul_rn(2.0f, u2)));
}

// xyz of a split child: p + R(q) (s * z), R = build_rotation of the normalised q = (r, x, y, z), every operation rounded once
__device__ __forceinline__ void split_child(const float p[3], const float s[3], float4 q, const float z[3], float out[3]) {
    const float r = q.x, x = q.y, y = q.z, w = q.w;
    const float R[9] = {
        __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, y), __fmul_rn(w, w)))),
        __fmul_rn(2.0f, __fsub_rn(__fmul_rn(x, y), __fmul_rn(r, w))),
        __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, w), __fmul_rn(r, y))),
        __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, y), __fmul_rn(r, w))),
        __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(w, w)))),
        __fmul_rn(2.0f, __fsub_rn(__fmul_rn(y, w), __fmul_rn(r, x))),
        __fmul_rn(2.0f, __fsub_rn(__fmul_rn(x, w), __fmul_rn(r, y))),
        __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, w), __fmul_rn(r, x))),
        __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))))};
    const float v[3] = {__fmul_rn(s[0], z[0]), __fmul_rn(s[1], z[1]), __fmul_rn(s[2], z[2])};
#pragma unroll
    for (int i = 0; i < 3; ++i)
        out[i] = __fadd_rn(p[i], __fadd_rn(__fadd_rn(__fmul_rn(R[3 * i], v[0]), __fmul_rn(R[3 * i + 1], v[1])), __fmul_rn(R[3 * i + 2], v[2])));
}

// rows [first, first + 2 n) of the arena (copies of their parents) become the split children: xyz and log-scale.  Child t
// draws its normals at the row it has in the densify result before the prune: key[t] (first children, t < n), key[t - n] +
// n_split (second children)
__global__ void __launch_bounds__(256)
densify_children_kernel(float* __restrict__ params, size_t off_rot, size_t off_xyz, size_t off_ls, uint32_t first, uint32_t n,
                        const uint32_t* __restrict__ key, uint32_t n_split, uint64_t seed, uint64_t call) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * n) return;
    const uint32_t row = first + t, k = t < n ? key[t] : key[t - n] + n_split;
    float* xyz = params + off_xyz + 3 * (size_t)row;
    float* ls = params + off_ls + 3 * (size_t)row;
    const float4 q = rotation_activation(reinterpret_cast<const float4*>(params + off_rot)[row]);
    float p[3], s[3], z[3], out[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        p[a] = xyz[a];
        s[a] = scale_activation(ls[a]);
        z[a] = split_normal(seed, call, k, a);
    }
    split_child(p, s, q, z, out);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        xyz[a] = out[a];
        ls[a] = __fsub_rn(ls[a], SPLIT_LOG_SCALE);
    }
}

__global__ void __launch_bounds__(256)
densify_split_kernel(int n, const float* __restrict__ xyz, const float* __restrict__ scale, const float4* __restrict__ rot, uint64_t seed,
                     uint64_t call, uint32_t first_row, float* __restrict__ xyz_out, float* __restrict__ z_out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    float p[3], s[3], z[3], out[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        p[a] = xyz[3 * (size_t)t + a];
        s[a] = scale[3 * (size_t)t + a];
        z[a] = split_normal(seed, call, first_row + (uint32_t)t, a);
    }
    split_child(p, s, rot[t], z, out);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        xyz_out[3 * (size_t)t + a] = out[a];
        if (z_out) z_out[3 * (size_t)t + a] = z[a];
    }
}

__global__ void __launch_bounds__(256)
gather_words_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, uint32_t rows_out, uint32_t rows_valid,
                    const uint32_t* __restrict__ idx) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows_out) dst[r] = r < rows_valid ? src[idx[r]] : 0u;
}

// rows [first, P) (glic_mapper_reset_opacity): a logit whose activation is above max_opacity becomes `logit`; both moments of
// the opacity group become zero
__global__ void __launch_bounds__(256)
reset_opacity_kernel(uint32_t first, uint32_t P, float* __restrict__ logit, float* __restrict__ m1, float* __restrict__ m2, float max_opacity,
                     float reset_logit) {
    const uint32_t r = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= P) return;
    if (opacity_activation(logit[r]) > max_opacity) logit[r] = reset_logit;
    m1[r] = 0.0f;
    m2[r] = 0.0f;
}

// The selection's scratch for P rows, as byte offsets: totals[6] (256 bytes) | 5 arrays of `tiles` counts | idx[2P] | key[P]
struct ScratchLayout {
    uint32_t tiles;
    size_t tile, idx, key, bytes;
    explicit ScratchLayout(uint32_t P) : tiles((P + PRUNE_TILE - 1) / PRUNE_TILE) {
        tile = 256;
        idx = tile + 5 * (((size_t)tiles * 4 + 255) & ~size_t(255));
        key = idx + (size_t)P * 8;
        bytes = key + (size_t)P * 4;
    }
};

}  // namespace

size_t density_scratch_bytes(uint32_t P) { return ScratchLayout(P).bytes; }

const uint32_t* density_index(const void* scratch, uint32_t P) {
    return reinterpret_cast<const uint32_t*>(static_cast<const char*>(scratch) + ScratchLayout(P).idx);
}

int launch_density_select(const DensitySelect& a, void* scratch, uint32_t* result_host, cudaStream_t s) {
    const ScratchLayout l(a.P);
    const uint32_t tiles = l.tiles;
    char* base = static_cast<char*>(scratch);
    uint32_t* totals = reinterpret_cast<uint32_t*>(base);
    uint32_t* tile = reinterpret_cast<uint32_t*>(base + l.tile);
    uint32_t* idx = reinterpret_cast<uint32_t*>(base + l.idx);
    uint32_t* key = reinterpret_cast<uint32_t*>(base + l.key);
    GLIC_CUDA_TRY(cudaMemsetAsync(totals + 5, 0, sizeof(uint32_t), s));
    fate_count_kernel<<<tiles, PRUNE_THREADS, 0, s>>>(a, tiles, tile);
    GLIC_LAUNCH_CHECK();
    prune_scan_kernel<<<5, 1024, 0, s>>>(tiles, tile, totals);
    GLIC_LAUNCH_CHECK();
    fate_index_kernel<<<tiles, PRUNE_THREADS, 0, s>>>(a, tiles, tile, totals, idx, key);
    GLIC_LAUNCH_CHECK();
    GLIC_CUDA_TRY(cudaMemcpyAsync(result_host, totals, 6 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    if (a.n_sky >= a.P) result_host[5] = result_host[2];         // every row is sky: the surviving kept rows are
    return GLIC_OK;
}

int launch_densify_children(float* params, uint32_t Pcap, int M, uint32_t first, uint32_t n, const void* scratch, uint32_t P_select,
                            uint32_t n_split, uint64_t seed, uint64_t call, cudaStream_t s) {
    if (n == 0) return GLIC_OK;
    size_t off[6];
    glic_packed_offsets(Pcap, (uint32_t)M, off);
    const uint32_t* key = reinterpret_cast<const uint32_t*>(static_cast<const char*>(scratch) + ScratchLayout(P_select).key);
    densify_children_kernel<<<(2 * n + 255) / 256, 256, 0, s>>>(params, off[0], off[1], off[2], first, n, key, n_split, seed, call);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_gather_words(const void* src, void* dst, uint32_t rows_out, uint32_t rows_valid, const uint32_t* idx, cudaStream_t s) {
    if (rows_out == 0) return GLIC_OK;
    gather_words_kernel<<<(rows_out + 255) / 256, 256, 0, s>>>(static_cast<const uint32_t*>(src), static_cast<uint32_t*>(dst), rows_out,
                                                               rows_valid, idx);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_reset_opacity(uint32_t first, uint32_t P, uint32_t Pcap, int M, float* params, float* m1, float* m2, float max_opacity,
                         float reset_logit, cudaStream_t s) {
    if (first >= P) return GLIC_OK;
    size_t off[6];
    glic_packed_offsets(Pcap, (uint32_t)M, off);
    reset_opacity_kernel<<<(P - first + 255) / 256, 256, 0, s>>>(first, P, params + off[3], m1 + off[3], m2 + off[3], max_opacity, reset_logit);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

}  // namespace glic

extern "C" int glic_densify_split(int n, const float* xyz, const float* scale, const float* rot, uint64_t seed, uint64_t call,
                                  uint32_t first_row, float* xyz_out, float* z_out, void* stream) {
    if (n < 0) { glic::set_error("densify_split: n must be >= 0"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (n == 0) return GLIC_OK;
    if (!xyz || !scale || !rot || !xyz_out) { glic::set_error("densify_split: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if ((reinterpret_cast<uintptr_t>(rot) & 15u) != 0) { glic::set_error("densify_split: rot must be 16-byte aligned"); return GLIC_ERR_INVALID_ARGUMENT; }
    glic::densify_split_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, xyz, scale, reinterpret_cast<const float4*>(rot), seed,
                                                                                  call, first_row, xyz_out, z_out);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

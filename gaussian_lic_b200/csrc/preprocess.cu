// preprocess.cu -- forward per-Gaussian stage, fused with the tile-count prefix sum, and the
// (tile|depth) key emission.
//
// Replaces, behind the C ABI: FORWARD::preprocess (reference forward.cu:232-319, 518-580),
// cub::DeviceScan::InclusiveSum (rasterizer_impl.cu:395) and duplicateWithKeys
// (rasterizer_impl.cu:59-193).  Design (not a translation):
//   * DEPTH-FIRST BINNING.  The reference sorts R (tile|depth) 64-bit keys on 45 bits (6 radix passes over
//     R pairs).  All duplicates of a Gaussian share its depth, so we sort the P Gaussians by depth ONCE
//     (32-bit keys, P << R), emit the (tile, index) pairs in that order, and are left with a stable sort of R
//     pairs on the 13 tile bits only (2 passes, 32-bit keys).  A stable sort by tile of a sequence ordered
//     by (depth, index) is ordered by (tile, depth, index): the final list is bit-identical to the
//     reference's, at ~1/4 of the sort traffic;
//   * the prefix sum of tiles_touched over the depth order is a single-pass decoupled look-back scan;
//   * the exact tile test runs ONCE per candidate tile: the counting walk stores each Gaussian's accept set (32-bit mask
//     or per-row spans), the emitting walk only expands it; both walks are balanced across the CTA;
//   * the digit histograms of both radix sorts are accumulated by the kernels that produce the keys;
//   * one 48-byte AoS splat record per Gaussian feeds emit, render-forward and render-backward;
//   * every key-defining operation uses the fixed-order intrinsics of geom_math.cuh.
#include "geom_math.cuh"
#include "warp_rows.cuh"
#include "async_copy.cuh"
#include <algorithm>

namespace glic {

// ---- SH basis (auxiliary.h:22-39, forward.cu:29-77) ---------------------------------------
__device__ __constant__ float kSH_C1 = 0.4886025119029199f;
__device__ __constant__ float kSH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                           -1.0925484305920792f, 0.5462742152960396f};
__device__ __constant__ float kSH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                           0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                           -0.5900435899266435f};
constexpr float kSH_C0 = 0.28209479177387814f;

// ---- decoupled look-back status words ------------------------------------------------------
constexpr unsigned long long ST_AGG = 1ull << 32;
constexpr unsigned long long ST_PREFIX = 2ull << 32;

GLIC_DI void st_release(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
GLIC_DI unsigned long long ld_acquire(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// Exclusive prefix of `aggregate` over all CTAs with a smaller ticket.  Called by warp 0 only.
GLIC_DI uint32_t lookback_exclusive(unsigned long long* status, int block, uint32_t aggregate, int lane) {
    if (block == 0) {
        if (lane == 0) st_release(&status[0], ST_PREFIX | aggregate);
        return 0;
    }
    if (lane == 0) st_release(&status[block], ST_AGG | aggregate);
    uint32_t exclusive = 0;
    int look = block - 1;
    unsigned spins = 0;
    while (true) {
        const int j = look - lane;
        unsigned long long st = ST_PREFIX;      // virtual predecessors before CTA 0 contribute 0
        if (j >= 0) st = ld_acquire(&status[j]);
        while (__any_sync(0xffffffffu, (st >> 32) == 0)) {
            if (j >= 0 && (st >> 32) == 0) st = ld_acquire(&status[j]);
            if (++spins > (1u << 24)) __trap();  // never hang the GPU: fail loudly instead
        }
        const unsigned pref = __ballot_sync(0xffffffffu, (st >> 32) == 2);
        const int first = pref ? (__ffs(pref) - 1) : 31;
        uint32_t v = (lane <= first) ? (uint32_t)st : 0u;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        exclusive += v;
        if (pref) break;
        look -= 32;
    }
    if (lane == 0) st_release(&status[block], ST_PREFIX | (unsigned long long)(exclusive + aggregate));
    return exclusive;
}


// ---- load-balanced walk over the candidate tiles of a CTA's 256 Gaussians -------------------------------
// Rect sizes span 1 .. 8160 tiles (median 4, 99th percentile ~900 at cfg2) and the big rects carry most of
// the pairs.  Small rects (<= WALK_SMALL tiles) are walked tile by tile by their own lane.  Big rects are
// compacted into a shared-memory table and processed ROW by ROW, 32 rows per warp step: the accepted tiles
// of one rect row form an interval (the tile test is the distance of a translating convex box to a convex
// ellipse, quasi-convex along the row), so a lane predicts the interval analytically from the conic and
// only runs the exact test at its two ends (~4 tests per row instead of one per tile).  The interval ends
// are always decided by the exact fixed-order test, so the accept set is the reference's bit for bit.
// EMIT writes key = tile id, value = Gaussian index into the Gaussian's slot range; the order inside a slot
// range is arbitrary for big rects -- the tile ids of one Gaussian are distinct, so the sorted list does
// not depend on it.
constexpr int WALK_SMALL = 32;
constexpr uint32_t NO_SPANS = 0xFFFFFFFFu;

// What the counting walk (preprocess) leaves behind for the emitting walk, so that no exact tile test runs twice:
//   rects of <= 32 tiles: the accept set as a 32-bit mask (bit t <-> t-th tile of the rect, row-major) in tmask[i];
//   bigger rects: one (xa | xb << 16) word per rect row in a bump-allocated arena, first entry in tmask[i]
//   (NO_SPANS when the arena is full: the emitting walk then recomputes that rect's rows with the exact test).
struct SpanStore {
    uint32_t* spans;
    uint32_t cap;
    unsigned int* counter;
};

struct WalkSmem {
    uint32_t row_prefix[PRE_THREADS + 1];     // exclusive prefix of row counts over the compacted big list
    uint32_t cursor[PRE_THREADS];             // accepted tiles so far, per big slot
    float mx[PRE_THREADS], my[PRE_THREADS], cox[PRE_THREADS], coy[PRE_THREADS], coz[PRE_THREADS], thr[PRE_THREADS];
    int x0[PRE_THREADS], y0[PRE_THREADS], rw[PRE_THREADS], n[PRE_THREADS];
    uint32_t off[PRE_THREADS], idx[PRE_THREADS];
    uint32_t base[PRE_THREADS];               // first entry of the rect's row spans in the span arena (NO_SPANS: none)
    uint32_t small_mask[PRE_THREADS];         // accept bits of the small rects, gathered from the flat candidate test
    uint32_t warp_big[PRE_THREADS / 32];
    uint32_t n_big, n_rows;
};

// Accepted tile interval [xa, xb] (inclusive; xa > xb = empty) of rect row `ty`, columns [x0, x1).
GLIC_DI void row_span(float cox, float coy, float coz, float mx, float my, float thr, int ty, int x0, int x1, int& xa, int& xb) {
    auto accept = [&](int x) { return tile_max_power(cox, coy, coz, mx, my, x, ty) <= thr; };
    const float d0 = (float)(ty * TILE) - my, d1 = d0 + (float)(TILE - 1);      // dy range of the row's pixel centres
    const float det = cox * coz - coy * coy;
    const float t2 = 2.0f * thr;
    int pa = x0, pb = x1 - 1;
    bool predicted = false;
    if (det > 0.0f && cox > 0.0f && coz > 0.0f && t2 >= 0.0f) {
        // the slab misses the ellipse {power <= thr} by a clear margin: no tile of this row can pass the exact test
        const float e0 = fminf(fmaxf(0.0f, d0), d1);
        if (det * e0 * e0 > t2 * cox * 1.002f + 1e-6f) { xa = 1; xb = 0; return; }
        // x-projection [xl, xr] of ellipse /\ slab (extreme points of the ellipse clamped into the slab)
        const float hx = sqrtf(t2 * coz / det);
        const float dyR = -coy * hx / coz;
        float e = fminf(fmaxf(dyR, d0), d1);
        const float xr = mx + (-coy * e + sqrtf(fmaxf(t2 * cox - det * e * e, 0.0f))) / cox;
        e = fminf(fmaxf(-dyR, d0), d1);
        const float xl = mx + (-coy * e - sqrtf(fmaxf(t2 * cox - det * e * e, 0.0f))) / cox;
        if (xl == xl && xr == xr && fabsf(xl) < 1e7f && fabsf(xr) < 1e7f) {
            pa = max(x0, min(x1 - 1, (int)ceilf((xl - (float)(TILE - 1)) * (1.0f / TILE))));
            pb = max(x0, min(x1 - 1, (int)floorf(xr * (1.0f / TILE))));
            predicted = pa <= pb;
        }
    }
    int seed = -1;
    if (predicted) { const int mid = (pa + pb) >> 1; if (accept(mid)) seed = mid; }
    if (seed < 0) {                                   // rare: borderline / degenerate rows -> exact scan of the row
        int l = x0;
        while (l < x1 && !accept(l)) ++l;
        if (l == x1) { xa = 1; xb = 0; return; }
        int r = l;
        while (r + 1 < x1 && accept(r + 1)) ++r;
        xa = l; xb = r;
        return;
    }
    int l = min(pa, seed);
    if (accept(l)) { while (l > x0 && accept(l - 1)) --l; }
    else { do { ++l; } while (l < seed && !accept(l)); }
    int r = max(pb, seed);
    if (accept(r)) { while (r + 1 < x1 && accept(r + 1)) ++r; }
    else { do { --r; } while (r > seed && !accept(r)); }
    xa = l; xb = r;
}

// Returns the number of accepted tiles of THIS thread's Gaussian.  Must be called by all PRE_THREADS threads.
template <bool EMIT>
GLIC_DI uint32_t block_tile_walk(WalkSmem& w, int n, float mx, float my, float cox, float coy, float coz, float thr, int x0,
                                 int y0, int rw, int grid_x, uint32_t idx, uint32_t off, uint32_t* __restrict__ keys,
                                 uint32_t* __restrict__ vals, SpanStore ss, uint32_t& mask_or_base, uint32_t* s_hist = nullptr,
                                 int lo_bits = 8, uint32_t hi_mask = 0) {
    // EMIT: every key written also counts into the CTA's two digit histograms of the tile sort (bits [0,lo_bits) and
    // [lo_bits,..))
    auto count_key = [&](uint32_t key) {
        atomicAdd(&s_hist[key & ((1u << lo_bits) - 1u)], 1u);
        if (hi_mask) atomicAdd(&s_hist[256 + ((key >> lo_bits) & hi_mask)], 1u);
    };
    constexpr unsigned FULL = 0xffffffffu;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool big = n > WALK_SMALL;
    // -- compact the big rects of the CTA
    const uint32_t bal = __ballot_sync(FULL, big);
    if (lane == 0) w.warp_big[warp] = __popc(bal);
    __syncthreads();
    uint32_t base = 0, total_big = 0;
#pragma unroll
    for (int i = 0; i < PRE_THREADS / 32; ++i) {
        const uint32_t c = w.warp_big[i];
        if (i < warp) base += c;
        total_big += c;
    }
    int slot = -1;
    if (big) {
        slot = (int)(base + __popc(bal & ((1u << lane) - 1u)));
        w.mx[slot] = mx; w.my[slot] = my; w.cox[slot] = cox; w.coy[slot] = coy; w.coz[slot] = coz; w.thr[slot] = thr;
        w.x0[slot] = x0; w.y0[slot] = y0; w.rw[slot] = rw; w.n[slot] = n;
        w.off[slot] = off; w.idx[slot] = idx;
        w.cursor[slot] = 0;
        if (!EMIT) {                                     // room for this rect's row spans
            const uint32_t rows = (uint32_t)(n / rw);
            const uint32_t b = atomicAdd(ss.counter, rows);
            mask_or_base = (b + rows <= ss.cap) ? b : NO_SPANS;
        }
        w.base[slot] = mask_or_base;
    }
    // -- small rects (<= 32 tiles).  EMIT: own lane expands its stored mask.  COUNT: the warp's (Gaussian, tile) candidates are
    // tested FLAT -- lane l takes candidates l, l + 32, ... of the warp's concatenated rects and finds its Gaussian with a 5-step
    // search over the inclusive counts (parameters fetched by shuffle) -- so a warp needs ceil(sum n / 32) rounds instead of
    // max n rounds with most lanes idle (median rect 4 tiles, maximum 32).  The accept bits return to the owning lane through a
    // 32-word per-warp mask array.
    uint32_t count = 0;
    if (EMIT) {
        // accepted tiles of the warp's small rects, written flat: lane l takes pairs l, l + 32, ... and finds its Gaussian by the
        // same 5-step search; the k-th accepted tile of a rect is the k-th set bit of its mask
        const uint32_t mask = (n > 0 && !big) ? mask_or_base : 0u;
        const uint32_t cnt_s = (uint32_t)__popc(mask);
        uint32_t fin = cnt_s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, fin, o);
            if (lane >= o) fin += t;
        }
        const uint32_t tot = __shfl_sync(FULL, fin, 31);
        const uint32_t recip = (65536u + (uint32_t)rw - 1u) / (uint32_t)rw;
        for (uint32_t e = lane; e < ((tot + 31u) & ~31u); e += 32) {
            int r = 0;
#pragma unroll
            for (int st = 16; st > 0; st >>= 1) {
                const uint32_t probe = __shfl_sync(FULL, fin, r + st - 1);
                if (probe <= e) r += st;
            }
            const uint32_t r_fin = __shfl_sync(FULL, fin, r), r_cnt = __shfl_sync(FULL, cnt_s, r), r_mask = __shfl_sync(FULL, mask, r);
            const uint32_t r_off = __shfl_sync(FULL, off, r), r_idx = __shfl_sync(FULL, idx, r), r_rc = __shfl_sync(FULL, recip, r);
            const int r_x0 = __shfl_sync(FULL, x0, r), r_y0 = __shfl_sync(FULL, y0, r), r_rw = __shfl_sync(FULL, rw, r);
            if (e < tot) {
                const uint32_t kth = e - (r_fin - r_cnt);                           // which accepted tile of the rect
                const uint32_t j = __fns(r_mask, 0, (int)kth + 1);                  // its candidate index (row-major)
                const uint32_t q = (j * r_rc) >> 16;
                const uint32_t key = (uint32_t)((r_y0 + (int)q) * grid_x + r_x0 + (int)(j - q * (uint32_t)r_rw));
                keys[r_off + kth] = key; vals[r_off + kth] = r_idx; count_key(key);
            }
        }
        count = cnt_s;
    } else {
        const uint32_t ns = (n > 0 && !big) ? (uint32_t)n : 0u;
        uint32_t fin = ns;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, fin, o);
            if (lane >= o) fin += t;
        }
        const uint32_t tot = __shfl_sync(FULL, fin, 31);
        w.small_mask[tid] = 0u;
        __syncwarp();
        const uint32_t recip = (65536u + (uint32_t)rw - 1u) / (uint32_t)rw;      // j / rw == (j * recip) >> 16 for j < 32, rw <= 32
        for (uint32_t e = lane; e < ((tot + 31u) & ~31u); e += 32) {
            int r = 0;
#pragma unroll
            for (int st = 16; st > 0; st >>= 1) {
                const uint32_t probe = __shfl_sync(FULL, fin, r + st - 1);
                if (probe <= e) r += st;
            }
            const uint32_t r_fin = __shfl_sync(FULL, fin, r), r_n = __shfl_sync(FULL, ns, r);
            const float r_mx = __shfl_sync(FULL, mx, r), r_my = __shfl_sync(FULL, my, r), r_thr = __shfl_sync(FULL, thr, r);
            const float r_cox = __shfl_sync(FULL, cox, r), r_coy = __shfl_sync(FULL, coy, r), r_coz = __shfl_sync(FULL, coz, r);
            const int r_x0 = __shfl_sync(FULL, x0, r), r_y0 = __shfl_sync(FULL, y0, r), r_rw = __shfl_sync(FULL, rw, r);
            const uint32_t r_rc = __shfl_sync(FULL, recip, r);
            if (e < tot) {
                const uint32_t j = e - (r_fin - r_n);                               // candidate index inside the rect, row-major
                const uint32_t q = (j * r_rc) >> 16;
                const int tx = r_x0 + (int)(j - q * (uint32_t)r_rw), ty = r_y0 + (int)q;
                if (tile_max_power(r_cox, r_coy, r_coz, r_mx, r_my, tx, ty) <= r_thr) atomicOr(&w.small_mask[(tid & ~31) + r], 1u << j);
            }
        }
        __syncwarp();
        if (ns) { mask_or_base = w.small_mask[tid]; count = (uint32_t)__popc(mask_or_base); }
    }
    __syncthreads();
    if (total_big == 0) return count;
    // -- exclusive prefix of row counts over the compacted list (one warp; <= 256 entries)
    if (warp == 0) {
        uint32_t run = 0;
        for (uint32_t b0 = 0; b0 < total_big; b0 += 32) {
            const uint32_t s = b0 + lane;
            const uint32_t c = s < total_big ? (uint32_t)(w.n[s] / w.rw[s]) : 0u;      // rect height
            uint32_t incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(FULL, incl, o);
                if (lane >= o) incl += t;
            }
            if (s < total_big) w.row_prefix[s] = run + incl - c;
            run += __shfl_sync(FULL, incl, 31);
        }
        if (lane == 0) { w.row_prefix[total_big] = run; w.n_rows = run; w.n_big = total_big; }
    }
    __syncthreads();
    const uint32_t n_rows = w.n_rows;
    // -- 32 rect rows per warp step, round-robin over the warps
    for (uint32_t rb = warp * 32; rb < n_rows; rb += PRE_THREADS) {
        const uint32_t item = rb + lane;
        const bool valid = item < n_rows;
        int s = 0;
        if (valid) {                               // last slot with row_prefix[s] <= item (<= 8 probes)
            int lo = 0, hi = (int)total_big - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (w.row_prefix[mid] <= item) lo = mid; else hi = mid - 1;
            }
            s = lo;
        }
        int xa = 1, xb = 0, ty = 0;
        if (valid) {
            const uint32_t row = item - w.row_prefix[s];
            ty = w.y0[s] + (int)row;
            const uint32_t sb = w.base[s];
            if (EMIT && sb != NO_SPANS) {
                const uint32_t sp = ss.spans[sb + row];
                xa = (int)(sp & 0xFFFFu); xb = (int)(sp >> 16);
            } else {
                row_span(w.cox[s], w.coy[s], w.coz[s], w.mx[s], w.my[s], w.thr[s], ty, w.x0[s], w.x0[s] + w.rw[s], xa, xb);
                if (!EMIT && sb != NO_SPANS) ss.spans[sb + row] = xb >= xa ? ((uint32_t)xa | ((uint32_t)xb << 16)) : 1u;   // (1, 0) = empty
            }
        }
        const uint32_t cnt = xb >= xa ? (uint32_t)(xb - xa + 1) : 0u;
        // rows of one Gaussian sit in consecutive lanes: segmented (by slot) inclusive scan, one atomic per segment
        const int key = valid ? s : -1;
        uint32_t incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, incl, o);
            const int k = __shfl_up_sync(FULL, key, o);
            if (lane >= o && k == key) incl += t;
        }
        const int next_key = __shfl_down_sync(FULL, key, 1);
        const bool seg_last = valid && (lane == 31 || next_key != key);
        uint32_t seg_base = 0;
        if (seg_last && incl) seg_base = atomicAdd(&w.cursor[s], incl);
        if (EMIT) {
            // broadcast the segment's base from its last lane to the whole segment
            const uint32_t lastmask = __ballot_sync(FULL, seg_last);
            const uint32_t ahead = lastmask & ~((1u << lane) - 1u);          // segment ends at or after this lane
            const int src = ahead ? (__ffs(ahead) - 1) : lane;
            const uint32_t basev = __shfl_sync(FULL, seg_base, src);
            // The 32 rows of this step hold `tot` pairs.  They are written FLAT: lane l takes pairs l, l + 32, ... of the step and
            // finds its row with a 5-step search over the rows' inclusive counts, so that one store instruction covers up to
            // 32 consecutive slots of a row (rows of one Gaussian are adjacent in memory too) instead of 32 different rows.
            const uint32_t row_pos = cnt ? w.off[s] + basev + (incl - cnt) : 0u;     // first slot of this lane's row
            const uint32_t row_key = (uint32_t)(ty * grid_x + xa);
            const uint32_t row_gid = valid ? w.idx[s] : 0u;
            uint32_t fin = cnt;                                                       // inclusive count over the step's rows
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(FULL, fin, o);
                if (lane >= o) fin += t;
            }
            const uint32_t tot = __shfl_sync(FULL, fin, 31);
            for (uint32_t e = lane; e < ((tot + 31u) & ~31u); e += 32) {
                // row r = first lane whose inclusive count exceeds e
                int r = 0;
#pragma unroll
                for (int st = 16; st > 0; st >>= 1) {
                    const uint32_t probe = __shfl_sync(FULL, fin, r + st - 1);
                    if (probe <= e) r += st;
                }
                const uint32_t r_fin = __shfl_sync(FULL, fin, r), r_cnt = __shfl_sync(FULL, cnt, r);
                const uint32_t r_pos = __shfl_sync(FULL, row_pos, r), r_key = __shfl_sync(FULL, row_key, r), r_gid = __shfl_sync(FULL, row_gid, r);
                if (e < tot) {
                    const uint32_t j = e - (r_fin - r_cnt);                           // position inside the row
                    keys[r_pos + j] = r_key + j; vals[r_pos + j] = r_gid; count_key(r_key + j);
                }
            }
        }
    }
    __syncthreads();
    if (big) count = w.cursor[slot];
    return count;
}

__global__ void __launch_bounds__(PRE_THREADS)
preprocess_forward_kernel(int P, int D, int M, const float* __restrict__ means, const float* __restrict__ scales,
                          float mod, const float4* __restrict__ rots, const float* __restrict__ opac,
                          const float* __restrict__ dc, const float* __restrict__ sh, ViewParams vp, bool no_color,
                          int* __restrict__ radii, GeomState g, uint32_t* __restrict__ depth_hist) {
    pdl_enter();
    __shared__ float s_view[16], s_proj[16], s_cam[3];
    __shared__ uint32_t s_warp_sum[PRE_THREADS / 32];
    __shared__ uint32_t s_dhist[4 * 256];                   // digit histograms of the depth keys (the P-sized sort's four passes)
    for (int i = threadIdx.x; i < 4 * 256; i += PRE_THREADS) s_dhist[i] = 0;
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    float (*s_sh)[32 * SH_ROW_MAX] = reinterpret_cast<float (*)[32 * SH_ROW_MAX]>(dyn_smem);   // one 32-row SH slab per warp
    WalkSmem& walk = *reinterpret_cast<WalkSmem*>(dyn_smem + sizeof(float) * (PRE_THREADS / 32) * 32 * SH_ROW_MAX);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 16) s_view[tid] = vp.view[tid];
    else if (tid < 32) s_proj[tid - 16] = vp.proj[tid - 16];
    else if (tid < 35) s_cam[tid - 32] = vp.campos[tid - 32];
    __syncthreads();
    const int block = (int)blockIdx.x;
    const int idx = block * PRE_THREADS + tid;
    // The CTA's 256 SH rows are ONE contiguous run of HBM (up to 46 080 B): a single TMA bulk copy brings it into
    // shared memory while the geometry and the tile walk run; threads wait on the mbarrier only when they need colour.
    const int K = 3 * M;
    __shared__ __align__(8) uint64_t s_bar;
    bool sh_tma = false, sh_staged = false;
    if (!no_color && D > 0 && K <= SH_ROW_MAX) {
        const int bfirst = block * PRE_THREADS;
        const int bcnt = min(PRE_THREADS, P - bfirst);
        const size_t bytes = (size_t)bcnt * K * sizeof(float);
        const float* src = sh + (size_t)bfirst * K;
        sh_staged = bcnt > 0;
        sh_tma = sh_staged && (bytes % 16 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0);   // CTA-uniform
        if (sh_tma) {
            if (tid == 0) {
                mbar_init(&s_bar, 1);
                mbar_fence_init();
                mbar_arrive_expect_tx(&s_bar, (uint32_t)bytes);
                bulk_copy_g2s(&s_sh[0][0], src, (uint32_t)bytes, &s_bar);
            }
        } else if (sh_staged) {                   // ragged tail / unaligned tensor: coalesced 128-bit loads per warp
            const int wfirst = bfirst + warp * 32;
            const int wcnt = min(32, P - wfirst);
            if (wcnt > 0) warp_load_rows(sh, (size_t)wfirst, wcnt, K, s_sh[warp], lane);
        }
    }

    uint32_t tiles = 0;
    int radius = 0;
    float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0;
    float blue = 0.f, depth = 0.f, hy = 0.f;
    unsigned clampbits = 0;
    // ---- phase 1: geometry of my Gaussian (fixed-order arithmetic) ----------------------------------
    float px = 0.f, py = 0.f, pz = 0.f, mx = 0.f, my = 0.f, cox = 0.f, coy = 0.f, coz = 0.f, o = 0.f, thr = 0.f, tz = 0.f;
    int irad = 0, n = 0, rx0 = 0, ry0 = 0, rw = 1;
    if (idx < P) {
        px = means[3 * idx]; py = means[3 * idx + 1]; pz = means[3 * idx + 2];
        Cov3 c3;
        cov3d_from_scale_rot(scales[3 * idx], scales[3 * idx + 1], scales[3 * idx + 2], mod, rots[idx], c3);
        Cov2 c2;
        cov2d_project(px, py, pz, s_view, vp.focal_x, vp.focal_y, vp.limx_neg, vp.limx_pos, vp.limy_neg, vp.limy_pos,
                      c3.c, c2);
        tz = c2.tz;
        bool active = !(c2.tz <= 0.2f);                              // near cull, auxiliary.h:160
        const float hx = xform_row(s_proj, 0, px, py, pz);
        const float hy = xform_row(s_proj, 1, px, py, pz);
        const float hw = xform_row(s_proj, 3, px, py, pz);
        const float pw = __frcp_rn(fadd(hw, 0.0000001f));
        const float ndcx = fmul(hx, pw), ndcy = fmul(hy, pw);
        const float det = ffma(c2.a, c2.c, -fmul(c2.b, c2.b));        // a*c - b*b as fma(a, c, -(b*b))
        if (det == 0.0f) active = false;
        const float det_inv = __frcp_rn(det);
        cox = fmul(c2.c, det_inv); coy = fmul(det_inv, -c2.b); coz = fmul(c2.a, det_inv);
        o = opac[idx];
        if (o < (1.0f / 255.0f)) active = false;                     // forward.h:30, forward.cu:293
        if (active) {
            const float mid = fmul(fadd(c2.a, c2.c), 0.5f);
            const float lambda1 = fadd(mid, __fsqrt_rn(fmaxf(ffma(mid, mid, -det), 0.1f)));
            const float frad = ceilf(fmul(__fsqrt_rn(lambda1), 3.0f));
            mx = ndc_to_pix(ndcx, vp.W); my = ndc_to_pix(ndcy, vp.H);
            irad = (int)frad;
            const TileRect rc = tile_rect(mx, my, irad, vp.grid_x, vp.grid_y);
            thr = logf(__fdiv_rn(o, 1.0f / 255.0f));                 // forward.cu:302
            rw = rc.x1 - rc.x0; rx0 = rc.x0; ry0 = rc.y0;
            n = (rc.y1 - rc.y0) * rw;
        }
    }
    // ---- phase 2: exact tile counting, balanced across the CTA --------------------------------------------
    uint32_t mask_or_base = 0;
    const SpanStore ss{g.spans, g.span_cap, &g.hdr->span_count};
    const uint32_t cnt = block_tile_walk<false>(walk, n, mx, my, cox, coy, coz, thr, rx0, ry0, rw, vp.grid_x, 0u, 0u, nullptr, nullptr, ss, mask_or_base);
    // ---- phase 3: colour of the survivors -----------------------------------------------------------------
    if (sh_tma) mbar_wait(&s_bar, 0);      // (the walk's __syncthreads order thread 0's barrier init before every wait)
    if (cnt > 0) {
        tiles = cnt;
        radius = irad;
        depth = tz;
        float red = 0.f, green = 0.f;
        if (!no_color) {
            // SH -> RGB (forward.cu:29-77); tolerance-pinned, natural arithmetic.
            float dx = px - s_cam[0], dy = py - s_cam[1], dz = pz - s_cam[2];
            const float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
            dx *= inv; dy *= inv; dz *= inv;
            float res[3];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) res[ch] = kSH_C0 * dc[3 * idx + ch];
            if (D > 0) {
                const float* s = sh_tma ? (&s_sh[0][0] + (size_t)tid * K)
                                        : (sh_staged ? (s_sh[warp] + lane * K) : (sh + (size_t)idx * K));
                const float x = dx, y = dy, z = dz;
                float b[15];
                b[0] = -kSH_C1 * y; b[1] = kSH_C1 * z; b[2] = -kSH_C1 * x;
                int nb = 3;
                if (D > 1) {
                    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    b[3] = kSH_C2[0] * xy; b[4] = kSH_C2[1] * yz; b[5] = kSH_C2[2] * (2.0f * zz - xx - yy);
                    b[6] = kSH_C2[3] * xz; b[7] = kSH_C2[4] * (xx - yy);
                    nb = 8;
                    if (D > 2) {
                        b[8] = kSH_C3[0] * y * (3.0f * xx - yy);
                        b[9] = kSH_C3[1] * xy * z;
                        b[10] = kSH_C3[2] * y * (4.0f * zz - xx - yy);
                        b[11] = kSH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
                        b[12] = kSH_C3[4] * x * (4.0f * zz - xx - yy);
                        b[13] = kSH_C3[5] * z * (xx - yy);
                        b[14] = kSH_C3[6] * x * (xx - 3.0f * yy);
                        nb = 15;
                    }
                }
#pragma unroll
                for (int k = 0; k < 15; ++k) {
                    if (k < nb) {
                        res[0] += b[k] * s[3 * k + 0];
                        res[1] += b[k] * s[3 * k + 1];
                        res[2] += b[k] * s[3 * k + 2];
                    }
                }
            }
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                res[ch] += 0.5f;
                if (res[ch] < 0.0f) clampbits |= 1u << ch;
                res[ch] = fmaxf(res[ch], 0.0f);
            }
            red = res[0]; green = res[1]; blue = res[2];
        }
        r0 = make_float4(mx, my, cox, coy);
        r1 = make_float4(coz, o, red, green);
        // conservative vertical half-extent of {alpha >= 1/255} (dy^2 <= 2*thr*cox/det(conic)); falls back to the
        // looser 3.33-sigma bound from the radius when det cancels badly.  Used by the render kernel's row cull.
        {
            const float thr2 = __logf(255.0f * o) + 1e-3f;
            const float prod = cox * coz, dcon = prod - coy * coy;
            hy = 1.11f * (float)irad + 1.0f;
            if (dcon > 1e-3f * prod) hy = fminf(hy, sqrtf(2.0f * thr2 * cox / dcon) * 1.001f + 0.01f);
        }
    }

    // ---- R = sum of tiles_touched: CTA reduce + one atomic; record + depth key out -------------------
    uint32_t wsum = tiles;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
    if (lane == 0) s_warp_sum[warp] = wsum;
    __syncthreads();
    if (tid == 0) {
        uint32_t tot = 0;
#pragma unroll
        for (int w = 0; w < PRE_THREADS / 32; ++w) tot += s_warp_sum[w];
        if (tot) atomicAdd(&g.hdr->total, tot);
    }
    if (idx < P) {
        radii[idx] = radius;
        g.rec[3 * idx + 0] = r0;
        g.rec[3 * idx + 1] = r1;
        g.rec[3 * idx + 2] = make_float4(blue, depth, __int_as_float(radius), hy);
        g.clamped[idx] = (uint8_t)clampbits;
        g.tiles[idx] = tiles;
        g.tmask[idx] = mask_or_base;
        const uint32_t dkey = tiles ? __float_as_uint(depth) : 0xFFFFFFFFu;   // culled Gaussians sort to the end
        g.depth_keys[0][idx] = dkey;
        g.order[0][idx] = (uint32_t)idx;
#pragma unroll
        for (int p = 0; p < 4; ++p) atomicAdd(&s_dhist[p * 256 + ((dkey >> (8 * p)) & 255u)], 1u);
    }
    __syncthreads();
    for (int i = tid; i < 4 * 256; i += PRE_THREADS) {
        const uint32_t v = s_dhist[i];
        if (v) atomicAdd(&depth_hist[i], v);
    }
}

// ---- key emission ----------------------------------------------------------------------------
// Prefix sum of tiles_touched over the DEPTH order (single-pass decoupled look-back; the per-CTA work is a
// few loads, so no CTA ever delays its successors): Gaussian order[pos] owns slots [end - tiles, end) and
// `end` is scattered to offsets[gaussian] so that the emit kernel can run in (well mixed) index order.
constexpr int SCAN_ITEMS = 4;

__global__ void __launch_bounds__(PRE_THREADS)
depth_scan_kernel(int P, GeomState g, const uint32_t* __restrict__ order, unsigned int capacity) {
    pdl_enter();
    __shared__ unsigned s_block;
    __shared__ uint32_t s_warp_sum[PRE_THREADS / 32];
    __shared__ uint32_t s_block_excl;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_block = atomicAdd(&g.hdr->ticket, 1u);
    __syncthreads();
    const int block = (int)s_block;
    const int pos0 = (block * PRE_THREADS + tid) * SCAN_ITEMS;
    uint32_t gid[SCAN_ITEMS], run[SCAN_ITEMS];
    uint32_t mine = 0;
#pragma unroll
    for (int e = 0; e < SCAN_ITEMS; ++e) {
        gid[e] = 0;
        uint32_t tiles = 0;
        if (pos0 + e < P) { gid[e] = order[pos0 + e]; tiles = g.tiles[gid[e]]; }
        mine += tiles;
        run[e] = mine;                                       // inclusive within the thread
    }
    uint32_t incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp_sum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t ws = lane < PRE_THREADS / 32 ? s_warp_sum[lane] : 0u;
        uint32_t wi = ws;
#pragma unroll
        for (int o = 1; o < PRE_THREADS / 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        const uint32_t aggregate = __shfl_sync(0xffffffffu, wi, PRE_THREADS / 32 - 1);
        if (lane < PRE_THREADS / 32) s_warp_sum[lane] = wi - ws;      // exclusive per-warp base
        const uint32_t excl = lookback_exclusive(g.scan_status, block, aggregate, lane);
        if (lane == 0) {
            s_block_excl = excl;
            if (block == (int)gridDim.x - 1) {              // the last ticket sees the grand total
                const unsigned int total = excl + aggregate;
                // on overflow nothing downstream may touch the (partly unwritten) pair list: render an empty frame
                g.hdr->r_eff = total > capacity ? 0u : total;
                g.hdr->overflow = total > capacity ? 1u : 0u;
            }
        }
    }
    __syncthreads();
    const uint32_t base = s_block_excl + s_warp_sum[warp] + incl - mine;
#pragma unroll
    for (int e = 0; e < SCAN_ITEMS; ++e)
        if (pos0 + e < P) g.offsets[gid[e]] = base + run[e];
}

// Key emission in index order: Gaussian idx expands the accept set the counting walk stored (tile mask / row spans; the
// exact test is only re-run for rects whose spans did not fit the arena) and writes key = tile id, value = idx into its
// slot range [offsets[idx] - tiles, offsets[idx]); the tile sort's digit histograms are counted on the way.
__global__ void __launch_bounds__(PRE_THREADS)
emit_keys_kernel(int P, ViewParams vp, GeomState g, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, unsigned int capacity,
                 uint32_t* __restrict__ sort_hist, int lo_bits, uint32_t hi_mask) {
    pdl_enter();
    __shared__ WalkSmem walk;
    __shared__ uint32_t s_hist[2 * 256];
    for (int i = threadIdx.x; i < 2 * 256; i += PRE_THREADS) s_hist[i] = 0;
    __syncthreads();
    const int idx = blockIdx.x * PRE_THREADS + threadIdx.x;
    int n = 0, x0 = 0, y0 = 0, rw = 1;
    float mx = 0.f, my = 0.f, cox = 0.f, coy = 0.f, coz = 0.f, thr = 0.f;
    uint32_t off = 0, mask_or_base = 0;
    bool skip = false;
    if (idx < P) {
        const uint32_t tiles = g.tiles[idx];
        if (tiles != 0) {
            mask_or_base = g.tmask[idx];
            const float4 r0 = g.rec[3 * (size_t)idx + 0];
            const float4 r1 = g.rec[3 * (size_t)idx + 1];
            const float4 r2 = g.rec[3 * (size_t)idx + 2];
            const uint32_t end = g.offsets[idx];
            off = end - tiles;
            if (end > capacity) { skip = true; }           // would overrun the workspace: overflow is flagged by the scan
            mx = r0.x; my = r0.y; cox = r0.z; coy = r0.w; coz = r1.x;
            const TileRect rc = tile_rect(mx, my, __float_as_int(r2.z), vp.grid_x, vp.grid_y);
            thr = logf(__fdiv_rn(r1.y, 1.0f / 255.0f));
            rw = rc.x1 - rc.x0; x0 = rc.x0; y0 = rc.y0;
            n = (rc.y1 - rc.y0) * rw;
        }
    }
    const SpanStore ss{g.spans, g.span_cap, &g.hdr->span_count};
    block_tile_walk<true>(walk, skip ? 0 : n, mx, my, cox, coy, coz, thr, x0, y0, rw, vp.grid_x, (uint32_t)idx, off, keys, vals, ss, mask_or_base,
                          s_hist, lo_bits, hi_mask);
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * 256; i += PRE_THREADS) {
        const uint32_t v = s_hist[i];
        if (v) atomicAdd(&sort_hist[i], v);
    }
}

int launch_preprocess_forward(int P, int D, int M, const float* means, const float* scales, float mod,
                              const float* rots, const float* opac, const float* dc, const float* sh,
                              const ViewParams& vp, bool no_color, int* radii, GeomState g, cudaStream_t s) {
    const int blocks = (P + PRE_THREADS - 1) / PRE_THREADS;
    const size_t dyn = sizeof(float) * (PRE_THREADS / 32) * 32 * SH_ROW_MAX + sizeof(WalkSmem);
    static bool attr_set[64] = {};
    if (first_use_on_device(attr_set)) {
        GLIC_CUDA_TRY(cudaFuncSetAttribute(preprocess_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
    }
    GLIC_LAUNCH_PDL(preprocess_forward_kernel, blocks, PRE_THREADS, dyn, s, P, D, M, means, scales, mod,
                    reinterpret_cast<const float4*>(rots), opac, dc, sh, vp, no_color, radii, g, sort_hist(g.sort_temp));
    return GLIC_OK;
}

int launch_depth_scan(int P, GeomState g, const uint32_t* order, int64_t capacity, cudaStream_t s) {
    const unsigned int cap = (unsigned int)std::min<int64_t>(capacity, 0xFFFFFFFFll);
    const int per_cta = PRE_THREADS * SCAN_ITEMS;
    GLIC_LAUNCH_PDL(depth_scan_kernel, (P + per_cta - 1) / per_cta, PRE_THREADS, 0, s, P, g, order, cap);
    return GLIC_OK;
}

// sort_hist_out: the [passes][256] digit histograms of the following tile sort (zeroed by sort_prepare); end_bit = its key bits
int launch_emit_keys(int P, const ViewParams& vp, GeomState g, uint32_t* tile_keys, uint32_t* vals, int64_t capacity, uint32_t* sort_hist_out,
                     int end_bit, cudaStream_t s) {
    const unsigned int cap = (unsigned int)std::min<int64_t>(capacity, 0xFFFFFFFFll);
    if (end_bit > 16) { set_error("emit_keys: more than 16 tile bits"); return GLIC_ERR_INVALID_ARGUMENT; }
    // the sort's digit split: one pass of end_bit bits, or two of sort_pass_bits(end_bit, 0) + sort_pass_bits(end_bit, 1)
    const int lo_bits = sort_pass_bits(end_bit, 0);
    const uint32_t hi_mask = sort_passes(end_bit) > 1 ? (1u << sort_pass_bits(end_bit, 1)) - 1u : 0u;
    GLIC_LAUNCH_PDL(emit_keys_kernel, (P + PRE_THREADS - 1) / PRE_THREADS, PRE_THREADS, 0, s, P, vp, g, tile_keys, vals, cap,
                    sort_hist_out, lo_bits, hi_mask);
    return GLIC_OK;
}

}  // namespace glic

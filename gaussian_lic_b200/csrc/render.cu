// render.cu -- tile ranges, bucket offsets, per-tile front-to-back blend (forward) and the
// per-splat ("bucketed") backward.
//
// Replaces identifyTileRanges + perTileBucketCount + InclusiveSum (reference
// rasterizer_impl.cu:195-231,426-442), renderCUDA (forward.cu:321-481) incl. the D2D colour
// copy (rasterizer_impl.cu:471), and PerGaussianRenderCUDA (backward.cu:379-597).
//
// Design notes (ours):
//   * splat data of a batch is gathered ONCE per tile from the 48-byte records into shared
//     memory (xy, conic, opacity AND rgb -- the reference re-gathers rgb from global memory for
//     every contributing pixel-splat pair);
//   * each splat record carries a conservative vertical half-extent of its alpha >= 1/255 ellipse: warp w (rows
//     4w .. 4w+3 of the tile) skips, warp-uniformly, splats that cannot reach its rows.  The bound
//     is conservative, so results are bit-identical to evaluating every pair;
//   * checkpoints are one float4 (T, C.r, C.g, C.b) per pixel per 32-splat bucket -> 16-byte
//     coalesced stores / loads;
//   * the final colour is written to the caller's image and to the saved-state copy by the same
//     kernel (no separate D2D copy);
//   * backward: one warp per LIVE bucket (a bucket some pixel reached), handed out by a device ticket to a persistent
//     grid; pixel-major inside the bucket (every pixel restarts from the checkpoint), no lane-to-lane pipeline.
// The per-pixel arithmetic (power, alpha, T, C) keeps the reference's operation order through the
// fixed-order intrinsics of geom_math.cuh, so colours/transmittance agree bit-for-bit with the
// reference build on the same sorted list.
#include "geom_math.cuh"
#include "async_copy.cuh"
#include "f32x2.cuh"
#include <algorithm>

namespace glic {

// ---- tile ranges -------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
tile_ranges_kernel(int64_t R, const unsigned int* __restrict__ r_dev, const uint32_t* __restrict__ keys, uint32_t T,
                   uint2* __restrict__ ranges) {
    pdl_enter();
    if (r_dev) R = min(R, (int64_t)*r_dev);
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;     // four consecutive sorted keys per thread
    if (i0 >= R) return;
    uint32_t k[4];
    if (i0 + 3 < R) {
        const uint4 v = *reinterpret_cast<const uint4*>(keys + i0);
        k[0] = v.x; k[1] = v.y; k[2] = v.z; k[3] = v.w;
    } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) k[e] = i0 + e < R ? keys[i0 + e] : 0xFFFFFFFFu;
    }
    uint32_t prev = i0 > 0 ? keys[i0 - 1] : 0xFFFFFFFFu;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int64_t i = i0 + e;
        if (i >= R) break;
        const uint32_t cur = k[e];
        if (cur < T) {
            if (i == 0) ranges[cur].x = 0;
            else if (cur != prev) {
                if (prev < T) ranges[prev].y = (uint32_t)i;
                ranges[cur].x = (uint32_t)i;
            }
            if (i == R - 1) ranges[cur].y = (uint32_t)R;
        }
        prev = cur;
    }
}

// Inclusive scan over the T tiles by ONE CTA of 1024 threads, 8 consecutive tiles per thread (8192 tiles per sweep: one sweep
// covers a 1080p frame): thread-serial scan of its 8 values, warp scan, scan of the 32 warp totals -- two barriers per sweep.
template <typename Load, typename Store>
__device__ __forceinline__ uint32_t cta_scan_tiles(int T, Load load, Store store) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry;
    constexpr int PER = 8;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < T; base += 1024 * PER) {
        const int t0 = base + tid * PER;
        uint32_t v[PER];
        uint32_t mine = 0;
#pragma unroll
        for (int e = 0; e < PER; ++e) { v[e] = t0 + e < T ? load(t0 + e) : 0u; mine += v[e]; v[e] = mine; }
        uint32_t incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += n;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        uint32_t wbase = 0;
        {
            const uint32_t w = warp_tot[lane];
            uint32_t wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t n = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += n;
            }
            wbase = __shfl_sync(0xffffffffu, wi - w, warp);            // exclusive total of the warps before mine
        }
        const uint32_t before = carry + wbase + incl - mine;
#pragma unroll
        for (int e = 0; e < PER; ++e) if (t0 + e < T) store(t0 + e, before + v[e]);
        __syncthreads();
        if (tid == 1023) carry = before + mine;
        __syncthreads();
    }
    return carry;
}

// bucket_offsets = inclusive scan of ceil(n_t / 32)
__global__ void __launch_bounds__(1024)
bucket_scan_kernel(int T, const uint2* __restrict__ ranges, uint32_t* __restrict__ bucket_offsets, ImageHeader* hdr,
                   long long R, const GeomHeader* __restrict__ ghdr, int buckets, unsigned int* __restrict__ sorted_in_b, int cur) {
    pdl_enter();
    const uint32_t total = cta_scan_tiles(
        T, [&](int t) { if (!buckets) return 0u; const uint2 r = ranges[t]; return (r.y - r.x + BUCKET - 1) / BUCKET; },
        [&](int t, uint32_t v) { bucket_offsets[t] = v; });
    if (threadIdx.x == 0) {
        long long true_R = R, ovf = 0;
        if (ghdr) { R = ghdr->r_eff; true_R = ghdr->total; ovf = ghdr->overflow; }
        hdr->num_buckets = total; hdr->num_rendered = R;
        hdr->counters[0] = true_R; hdr->counters[1] = total; hdr->counters[2] = ovf; hdr->counters[3] = 0;
        *sorted_in_b = (unsigned int)cur;
    }
}

// ---- forward blend -------------------------------------------------------------------------
// Splat batches are staged by the TMA engine: every thread issues one 48-byte cp.async.bulk (its splat's
// record, gathered by sorted index) into a double-buffered shared-memory tile buffer; an mbarrier per
// buffer counts the bytes.  Batch i+1 is in flight while batch i is blended, no register staging.
struct __align__(16) SplatRec { float4 a, b, c; };     // (x, y, conic.x, conic.y) (conic.z, opacity, r, g) (b, depth, radius, hy)

// Four warps per 16x16 tile; lane l owns the two vertically adjacent pixels (column l & 15, rows 4w + 2(l >> 4) + {0, 1}).
// The pair shares the column, hence dx, dx*conic.x and dx*conic.y, the three broadcast loads of the splat record and the
// row cull; everything that differs between the two pixels is evaluated as a pair (f32x2.cuh), in exactly the per-pixel
// operation order of the scalar formulation (forward.cu:430-453 as pinned in
// DESIGN.md 3.1), so colour, transmittance and contributor counts keep their bits.
//
// INFER (glic_render) is the inference form: the same blend over the same lists in the same operation order, so colour and
// final T keep their bits, plus the expected depth sum_i T_i alpha_i z_i (unnormalised, like the colour: one more FMA per taken
// pair, z from the record) and the median depth (z of the first taken splat after which T < 0.5, else 0).  It writes none of
// the backward's state (checkpoints, bucket_to_tile, n_contrib, max_contrib, pixel_colors); out_depth / out_median may be
// null.
//
// SCORE (glic_contribution) is the alpha-only scoring form: the no_color training blend over the same lists in the same operation
// order, so T and the set of taken (pixel, splat) pairs are the training blend's, bit for bit.  For each taken pair it forms the
// weight w = fl(T alpha) (T before the splat) and adds it to the splat's two scores: score_max[gid] = max(score_max[gid], w), as
// atomicMax on the bits of a non-negative float, and score_hits[gid] += 1.  A splat that ends a pixel (T (1 - alpha) < 1e-4) is
// not taken there, but removing it would let the pixel blend on, so it counts in score_ends[gid] (may be null: not counted).
// The pairs land first in a shared-memory slot per splat of the 256-splat batch (shared atomics; taken pixels in the low 16
// bits of the count, ended pixels in the high 16, at most 256 of each), double-buffered by batch parity; after the barrier that
// ends a batch, each non-empty slot sends one global atomic of each kind it holds and is zeroed.  out_T (may be null) gets the final T; nothing else is
// written.  The training form compiles every INFER and SCORE line out, INFER every SCORE line.
constexpr int FWD_THREADS = 128;
enum FwdForm { FWD_TRAIN, FWD_INFER, FWD_SCORE };

template <int FORM>
__global__ void __launch_bounds__(FWD_THREADS)
render_forward_kernel(ViewParams vp, bool no_color, const uint2* __restrict__ ranges,
                      const uint32_t* __restrict__ point_list, const float4* __restrict__ rec,
                      const uint32_t* __restrict__ bucket_offsets, uint32_t* __restrict__ bucket_to_tile,
                      float4* __restrict__ ckpt, uint32_t* __restrict__ n_contrib, uint32_t* __restrict__ max_contrib,
                      float* __restrict__ pixel_colors, float* __restrict__ out_color, float* __restrict__ out_T,
                      float* __restrict__ out_depth, float* __restrict__ out_median, unsigned int* __restrict__ score_max,
                      unsigned long long* __restrict__ score_hits, unsigned long long* __restrict__ score_ends) {
    constexpr bool INFER = FORM == FWD_INFER, SCORE = FORM == FWD_SCORE;
    if (INFER) no_color = false;                                 // the inference form always blends colour
    if (SCORE) no_color = true;                                  // the scoring form blends alpha only
    __shared__ SplatRec s_rec[2][TILE_PIX];
    __shared__ __align__(8) uint64_t s_bar[2];
    __shared__ uint32_t s_red[FWD_THREADS / 32];
    __shared__ uint32_t s_wmax[2][TILE_PIX], s_hits[2][TILE_PIX];    // SCORE: the batch's slots (max weight bits, pixel counts)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile = blockIdx.y * vp.grid_x + blockIdx.x;
    const int pix_min_x = blockIdx.x * TILE, pix_min_y = blockIdx.y * TILE;
    const int col = lane & (TILE - 1);
    const int row0 = 4 * warp + 2 * (lane >> 4);                 // tile row of the lane's upper pixel
    const int px = pix_min_x + col, py0 = pix_min_y + row0;
    const bool inside0 = px < vp.W && py0 < vp.H, inside1 = px < vp.W && py0 + 1 < vp.H;
    const float pfx = (float)px;
    const f2 pfy = f2_pack((float)py0, (float)(py0 + 1));
    const size_t pid0 = (size_t)py0 * vp.W + px, pid1 = pid0 + vp.W;
    const int pin0 = row0 * TILE + col, pin1 = pin0 + TILE;       // row-major pixel index inside the tile (checkpoint layout)
    const uint2 range = ranges[tile];
    const int n_splats = (int)(range.y - range.x);
    const int rounds = (n_splats + TILE_PIX - 1) / TILE_PIX;

    if (tid == 0) { mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); mbar_fence_init(); }
    if (SCORE)
        for (int u = tid; u < 2 * TILE_PIX; u += FWD_THREADS) { (&s_wmax[0][0])[u] = 0u; (&s_hits[0][0])[u] = 0u; }
    uint32_t bbm = 0;
    if (!INFER && !no_color) {
        bbm = tile == 0 ? 0u : bucket_offsets[tile - 1];
        const int nb = (n_splats + BUCKET - 1) / BUCKET;
        for (int b = tid; b < nb; b += FWD_THREADS) bucket_to_tile[bbm + b] = tile;
    }
    __syncthreads();
    // issue the gather of batch `r` into buffer r & 1 (two 48-byte bulk copies per thread)
    auto prefetch = [&](int r) {
        const int cnt = min(TILE_PIX, n_splats - r * TILE_PIX);
        if (tid == 0) mbar_arrive_expect_tx(&s_bar[r & 1], (uint32_t)(cnt * sizeof(SplatRec)));
#pragma unroll
        for (int u = tid; u < TILE_PIX; u += FWD_THREADS) {
            if (u < cnt) {
                const uint32_t id = point_list[range.x + r * TILE_PIX + u];
                bulk_copy_g2s(&s_rec[r & 1][u], rec + 3 * (size_t)id, (uint32_t)sizeof(SplatRec), &s_bar[r & 1]);
            }
        }
    };
    if (rounds > 0) prefetch(0);
    // SCORE: batch r's non-empty slots to the global scores, then zeroed for batch r + 2 (after the barrier that ends batch r)
    auto score_flush = [&](int r) {
        const int cnt = min(TILE_PIX, n_splats - r * TILE_PIX);
        for (int u = tid; u < cnt; u += FWD_THREADS) {
            const uint32_t h = s_hits[r & 1][u];
            if (h) {
                const uint32_t id = point_list[range.x + r * TILE_PIX + u];
                if (h & 0xFFFFu) {
                    atomicMax(score_max + id, s_wmax[r & 1][u]);
                    atomicAdd(score_hits + id, (unsigned long long)(h & 0xFFFFu));
                }
                if ((h >> 16) && score_ends) atomicAdd(score_ends + id, (unsigned long long)(h >> 16));
                s_wmax[r & 1][u] = 0u; s_hits[r & 1][u] = 0u;
            }
        }
    };

    // this warp covers tile rows 4w .. 4w+3: splats whose alpha >= 1/255 ellipse cannot reach them are skipped
    // warp-uniformly (conservative half-extent `hy` precomputed per splat => bit-identical results)
    const float band_mid = (float)(pix_min_y + 4 * warp) + 1.5f;

    bool done0 = !inside0, done1 = !inside1;
    f2 Tp = f2_bcast(1.0f), Cr = f2_bcast(0.f), Cg = Cr, Cb = Cr;
    // INFER: a pixel outside the frame is never written and never takes a splat, so it starts at T = 0; the median test below
    // then stops for its lane as soon as the other pixel is past T = 0.5 (bottom-edge tiles)
    if (INFER) Tp = f2_pack(inside0 ? 1.0f : 0.0f, inside1 ? 1.0f : 0.0f);
    f2 Dp = Cr;                             // INFER: expected depth (unnormalised)
    float med0 = 0.f, med1 = 0.f;           // INFER: median depth (0 until T falls below 0.5)
    uint32_t last0 = 0, last1 = 0;
    int waited = 0;                         // batches whose barrier this thread has consumed

    for (int i = 0; i < rounds; ++i) {
        // everyone is past batch i-1 (its buffer may be refilled) -- and we may stop if all pixels are done
        if (__syncthreads_count(done0 && done1) == FWD_THREADS) break;
        if (SCORE && i > 0) score_flush(i - 1);
        if (i + 1 < rounds) prefetch(i + 1);
        mbar_wait(&s_bar[i & 1], (uint32_t)((i >> 1) & 1));
        waited = i + 1;
        const SplatRec* batch = s_rec[i & 1];
        const int nb = min(TILE_PIX, n_splats - i * TILE_PIX);
        // one checkpoint per 32-splat bucket, then the bucket's splats
        for (int jb = 0; jb < nb && !(done0 && done1); jb += BUCKET) {
            if (!INFER && !no_color) {
                float t0, t1, r0, r1, g0, g1, b0, b1;
                f2_unpack(Tp, t0, t1); f2_unpack(Cr, r0, r1); f2_unpack(Cg, g0, g1); f2_unpack(Cb, b0, b1);
                float4* k = ckpt + (size_t)bbm * TILE_PIX;
                k[pin0] = make_float4(t0, r0, g0, b0);
                k[pin1] = make_float4(t1, r1, g1, b1);
                ++bbm;
            }
            const int je = min(jb + BUCKET, nb);
            const SplatRec* sr = batch + jb;
            for (int j = jb; j < je; ++j, ++sr) {
                const float4 c = sr->c;
                const float4 a = sr->a;
                if (fabsf(band_mid - a.y) > c.w + 1.5f) continue;      // warp-uniform band cull
                const float4 b = sr->b;
                const float dx = fsub(a.x, pfx);
                const f2 dy = f2_sub(f2_bcast(a.y), pfy);
                // power = fsub(fmul(ffma(dx, dx*cx, dy*(dy*cz)), -0.5), dy*(dx*cy)) for both pixels at once
                const f2 q = f2_fma(dx, fmul(dx, a.z), f2_mul(dy, f2_mul(dy, b.x)));
                const f2 power = f2_sub(f2_mul(q, -0.5f), f2_mul(dy, fmul(dx, a.w)));
                float p0, p1;
                f2_unpack(power, p0, p1);
                bool skip0 = done0 || p0 > 0.0f, skip1 = done1 || p1 > 0.0f;
                if (skip0 && skip1) continue;
                const f2 al = f2_mul(f2_pack(expf(p0), expf(p1)), b.y);
                float a0, a1;
                f2_unpack(al, a0, a1);
                a0 = fminf(0.99f, a0); a1 = fminf(0.99f, a1);
                skip0 |= a0 < (1.0f / 255.0f); skip1 |= a1 < (1.0f / 255.0f);
                if (skip0 && skip1) continue;
                const f2 alpha = f2_pack(a0, a1);
                const f2 test_T = f2_mul(Tp, f2_sub(f2_bcast(1.0f), alpha));
                float tt0, tt1, t0, t1;
                f2_unpack(test_T, tt0, tt1);
                f2_unpack(Tp, t0, t1);
                const bool end0 = SCORE && !skip0 && tt0 < 0.0001f, end1 = SCORE && !skip1 && tt1 < 0.0001f;
                if (!skip0 && tt0 < 0.0001f) { done0 = true; skip0 = true; }
                if (!skip1 && tt1 < 0.0001f) { done1 = true; skip1 = true; }
                if (SCORE && (!(skip0 && skip1) || end0 || end1)) {
                    // a positive float's bits order as the float does, so the slot keeps max w as an integer max
                    const float w0 = skip0 ? 0.0f : __fmul_rn(t0, a0), w1 = skip1 ? 0.0f : __fmul_rn(t1, a1);
                    if (!(skip0 && skip1)) atomicMax(&s_wmax[i & 1][j], __float_as_uint(fmaxf(w0, w1)));
                    atomicAdd(&s_hits[i & 1][j], (skip0 ? 0u : 1u) + (skip1 ? 0u : 1u) + (((end0 ? 1u : 0u) + (end1 ? 1u : 0u)) << 16));
                }
                if (done0 && done1) break;
                if (!no_color) {
                    // a pixel that does not take the splat blends with alpha = 0: C = fma(T, 0, C) = C exactly
                    const f2 ae = f2_pack(skip0 ? 0.0f : a0, skip1 ? 0.0f : a1);
                    Cr = f2_fma(Tp, f2_mul(ae, b.z), Cr);
                    Cg = f2_fma(Tp, f2_mul(ae, b.w), Cg);
                    Cb = f2_fma(Tp, f2_mul(ae, c.x), Cb);
                    if (INFER) {
                        Dp = f2_fma(Tp, f2_mul(ae, c.y), Dp);
                        // T only falls: T >= 0.5 before a taken splat and < 0.5 after it marks the first crossing.  Past it
                        // (most of the pairs of a deep tile) the lane skips the median test altogether
                        if (fmaxf(t0, t1) >= 0.5f) {
                            if (!skip0 && t0 >= 0.5f && tt0 < 0.5f) med0 = c.y;
                            if (!skip1 && t1 >= 0.5f && tt1 < 0.5f) med1 = c.y;
                        }
                    }
                }
                Tp = f2_pack(skip0 ? t0 : tt0, skip1 ? t1 : tt1);
                const uint32_t me = (uint32_t)(i * TILE_PIX + j + 1);
                if (!skip0) last0 = me;
                if (!skip1) last1 = me;
            }
        }
    }
    // never leave the CTA with a bulk copy still in flight towards its shared memory
    {
        const int issued = min(rounds, waited + 1);
        if (issued > waited) mbar_wait(&s_bar[waited & 1], (uint32_t)((waited >> 1) & 1));
    }

    float t0, t1, r0, r1, g0, g1, b0, b1;
    f2_unpack(Tp, t0, t1); f2_unpack(Cr, r0, r1); f2_unpack(Cg, g0, g1); f2_unpack(Cb, b0, b1);
    const size_t HW = (size_t)vp.W * vp.H;
    if (SCORE) {
        __syncthreads();                                          // the last batch's slots are complete
        if (waited > 0) score_flush(waited - 1);
        if (out_T) {
            if (inside0) out_T[pid0] = t0;
            if (inside1) out_T[pid1] = t1;
        }
        return;
    }
    if (INFER) {
        float d0, d1;
        f2_unpack(Dp, d0, d1);
        if (inside0) {
            out_T[pid0] = t0;
            out_color[pid0] = r0; out_color[HW + pid0] = g0; out_color[2 * HW + pid0] = b0;
            if (out_depth) out_depth[pid0] = d0;
            if (out_median) out_median[pid0] = med0;
        }
        if (inside1) {
            out_T[pid1] = t1;
            out_color[pid1] = r1; out_color[HW + pid1] = g1; out_color[2 * HW + pid1] = b1;
            if (out_depth) out_depth[pid1] = d1;
            if (out_median) out_median[pid1] = med1;
        }
        return;
    }
    if (inside0) {
        out_T[pid0] = t0;
        if (!no_color) {
            n_contrib[pid0] = last0;
            out_color[pid0] = r0; out_color[HW + pid0] = g0; out_color[2 * HW + pid0] = b0;
            pixel_colors[pid0] = r0; pixel_colors[HW + pid0] = g0; pixel_colors[2 * HW + pid0] = b0;
        }
    }
    if (inside1) {
        out_T[pid1] = t1;
        if (!no_color) {
            n_contrib[pid1] = last1;
            out_color[pid1] = r1; out_color[HW + pid1] = g1; out_color[2 * HW + pid1] = b1;
            pixel_colors[pid1] = r1; pixel_colors[HW + pid1] = g1; pixel_colors[2 * HW + pid1] = b1;
        }
    }
    if (no_color) return;
    uint32_t m = max(last0, last1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) s_red[warp] = m;
    __syncthreads();
    if (tid == 0) {
        uint32_t mm = 0;
#pragma unroll
        for (int w = 0; w < FWD_THREADS / 32; ++w) mm = max(mm, s_red[w]);
        max_contrib[tile] = mm;
    }
}

// ---- per-splat backward --------------------------------------------------------------------
// Only buckets that some pixel actually reached are worth a warp: tile t has ceil(max_contrib[t]/32) LIVE
// buckets (at cfg2: 19 k of 245 k).  live_scan_kernel prefix-sums them; the backward kernel is persistent
// (a fixed number of CTAs, warps stride over the live list), so every resident warp does useful work and no
// launch geometry depends on a device-side count.
__global__ void __launch_bounds__(1024)
live_scan_kernel(int T, const uint32_t* __restrict__ max_contrib, uint32_t* __restrict__ live_offsets, ImageHeader* hdr) {
    pdl_enter();
    const uint32_t total = cta_scan_tiles(T, [&](int t) { return (max_contrib[t] + BUCKET - 1) / BUCKET; },
                                          [&](int t, uint32_t v) { live_offsets[t] = v; });
    if (threadIdx.x == 0) { hdr->num_live_buckets = total; hdr->bwd_ticket = 0; }
}

constexpr int BWD_WARPS = 4;              // warps per CTA; every warp owns one live bucket at a time
constexpr int BWD_ROWPAIRS = TILE / 2;    // row pairs of a tile: a lane owns one pixel of each

// Backward of the blend, pixel-major inside a 32-splat bucket (replaces PerGaussianRenderCUDA, backward.cu:400-597).
//
// One warp per LIVE bucket in a persistent grid-stride loop, covering the bucket's whole 16x16 tile: lane l owns the 8
// pixels (column l & 15, rows 2j + (l >> 4), j = 0..7), one per row pair.  Every pixel restarts from the bucket's
// checkpoint (T, C) and walks the bucket's splats in list order exactly like the forward, so T and the colour prefix
// need no hand-over between lanes and the eight pixels of a lane
// are eight independent dependency chains.  A (splat, row pair) is visited only if the splat's alpha >= 1/255 ellipse can
// reach those rows (the forward's conservative half-extent test => skipped pairs contribute exactly zero) and some pixel
// of the pair got this far.  The nine per-splat sums are accumulated over the lane's pixels in registers, combined across
// the warp by one reduce-scatter (8 values in 3 halving exchanges + 2 butterflies; the 9th by butterfly) and leave as
// 9 RED per splat and bucket -- the same global-atomic count as the reference's per-splat formulation, without its
// 287-step shuffle pipeline (4 shuffles + bookkeeping per pixel-splat pair).
//
// FAST (the production form) takes G = 2^(power * log2 e) from one MUFU.EX2 instead of the bit-exact expf (8 instructions),
// and falls back to expf for a pixel whose fast alpha lies within a guard band of 1/255, so every take/skip decision stays
// the forward's.  It also carries one colour suffix per pixel (sum_c a_c dL/dpix_c) instead of three, which halves the
// dL/dalpha arithmetic and frees the 16 registers that let 6 CTAs (24 warps) per SM fit in 80 registers without spilling
// (the former body needs 96 and runs at 5).  !FAST is the former body (expf for every pixel, three suffixes); tests compare the two.  COUNT adds work counters
// (BwdCount) and is used by tests and scripts/render_bwd_bench.py only.  No visit is skipped for want of a taking pixel:
// at cfg2, 98 % of the (splat, two row pairs) visits have one, and a per-visit ballot cost more than it saved.
//
// DET (the deterministic form, FAST only; the exact and counting forms stay atomic-only) runs the same body
// but sends no RED: the nine values of (live bucket `live`, splat k) -- bit for bit what the atomic form would add -- are stored
// to entry e = 32 live + k of `det` (DetOut), with the splat's gid as the entry's key.  A slot that adds nothing (past n_valid,
// no visit, or all nine sums exactly zero: the cases the atomic form skips) gets the key `sentinel` = P.  Live buckets are
// numbered in tile order, so the entry index orders a Gaussian's contributions by ascending tile.  launch_render_backward_det
// then sorts the keys stably and folds each Gaussian's run (det_reduce_kernel).
enum BwdCount { BC_LIVE, BC_SPLATS, BC_SPLATS_TAKEN, BC_VISITS, BC_VISITS_TAKEN, BC_CAND, BC_TAKEN, BC_FALLBACK, BC_N };
struct DetOut {
    uint32_t* keys;           // [cap_live * 32] gid or sentinel
    uint32_t* idx;            // [cap_live * 32] entry index (the sort's values)
    float* vals;              // [cap_live * 32][9]
    unsigned int* count;      // min(32 * live buckets, 32 * cap_live): the entries the sort and the reduction see
    uint32_t cap_live;        // live buckets the arrays hold; a bucket past it (garbage counts of an overflowed forward) is dropped
    uint32_t sentinel;
};
template <int MIN_CTAS, bool FAST, bool COUNT, bool DET = false>
__global__ void __launch_bounds__(BWD_WARPS * 32, MIN_CTAS)
render_backward_kernel(ViewParams vp, int T_tiles, ImageHeader* __restrict__ hdr, const uint2* __restrict__ ranges,
                       const uint32_t* __restrict__ point_list, const float4* __restrict__ rec,
                       const uint32_t* __restrict__ bucket_offsets, const uint32_t* __restrict__ live_offsets,
                       const float4* __restrict__ ckpt, const uint32_t* __restrict__ n_contrib,
                       const float* __restrict__ pixel_colors, const float* __restrict__ dL_dpix,
                       float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic, float* __restrict__ dL_dopacity,
                       float* __restrict__ dL_dcolors, unsigned long long* __restrict__ counters, DetOut det) {
    pdl_enter();
    static_assert(!DET || (FAST && !COUNT), "the deterministic form is the production body only");
    __shared__ float4 s_sp[BWD_WARPS][BUCKET][3];            // the bucket's splat records, per warp
    __shared__ uint32_t s_gid[BWD_WARPS][BUCKET];
    __shared__ uint32_t s_rows[BWD_WARPS][BUCKET];           // row pairs each splat can reach (8-bit mask)
    // dL/dpixel of the lane's pixel pairs, [pair][channel][lane] as packed (row pair 2p, row pair 2p+1) values: read-only inside a
    // bucket, so it lives in shared memory instead of 24 registers (128 -> fewer registers = one more CTA per SM)
    __shared__ float2 s_g[BWD_WARPS][BWD_ROWPAIRS / 2][3][32];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t n_live = hdr->num_live_buckets;
    if (DET && blockIdx.x == 0 && threadIdx.x == 0) *det.count = 32u * min(n_live, det.cap_live);
    const size_t HW = (size_t)vp.W * vp.H;
    const float ddelx_dx = 0.5f * vp.W, ddely_dy = 0.5f * vp.H;
    float4 (*sp)[3] = s_sp[warp];

    // destination of this lane's reduce-scatter result: value slot v = lane >> 2 (held by lanes with (lane & 3) == 0)
    //   slot: 0 mean.x, 1 mean.y, 2 conic.x, 3 conic.y, 4 conic.w, 5..7 colour; lane 1 additionally carries opacity
    const int slot = lane >> 2;
    float* dst_base; int dst_stride, dst_off; float f_op, f_one;
    if (lane == 1) { dst_base = dL_dopacity; dst_stride = 1; dst_off = 0; f_op = 0.f; f_one = 1.f; }
    else if (slot < 2) { dst_base = dL_dmean2D; dst_stride = 3; dst_off = slot; f_op = slot == 0 ? -ddelx_dx : -ddely_dy; f_one = 0.f; }
    else if (slot < 5) { dst_base = dL_dconic; dst_stride = 4; dst_off = slot == 4 ? 3 : slot - 2; f_op = -0.5f; f_one = 0.f; }
    else { dst_base = dL_dcolors; dst_stride = 3; dst_off = slot - 5; f_op = 0.f; f_one = 1.f; }
    const bool i_write = (lane & 3) == 0 || lane == 1;
    unsigned ctr[BC_N] = {};                                     // COUNT only: this lane's share of the counters

    // live buckets are handed out dynamically (one ticket per warp and bucket): buckets differ by more than 10x in cost
    for (;;) {
        uint32_t live = 0;
        if (lane == 0) live = atomicAdd(&hdr->bwd_ticket, 1u);
        live = __shfl_sync(0xffffffffu, live, 0);
        if (live >= n_live) break;
        // tile of this live bucket: first t with live_offsets[t] > live -- 32-ary search, one probe per lane
        int lo = 0, cnt = T_tiles;
        while (cnt > 1) {
            const int step = (cnt + 31) >> 5;
            const int probe = lo + min((lane + 1) * step, cnt) - 1;              // last tile of this lane's sub-range
            const unsigned hit = __ballot_sync(0xffffffffu, live_offsets[probe] > live);
            const int first = __ffs(hit) - 1;                                      // hit != 0: live < live_offsets[T-1]
            lo += first * step;
            cnt = min(step, cnt - first * step);
        }
        const uint32_t tile = (uint32_t)lo;
        const int bucket_in_tile = (int)(live - (tile == 0 ? 0u : live_offsets[tile - 1]));
        const uint32_t bucket = (tile == 0 ? 0u : bucket_offsets[tile - 1]) + (uint32_t)bucket_in_tile;
        const uint2 range = ranges[tile];
        const int n_splats = (int)(range.y - range.x);
        const int bucket_start = bucket_in_tile * BUCKET;
        const int n_valid = min(BUCKET, n_splats - bucket_start);
        const int tile_x = tile % vp.grid_x, tile_y = tile / vp.grid_x;
        const int row0 = tile_y * TILE;
        const int qx = tile_x * TILE + (lane & (TILE - 1)), qy0 = row0 + (lane >> 4);
        const float pfx = (float)qx;

        // this lane's 8 pixels, as 4 PAIRS of row pairs (p <-> rows 2(2p) + h and 2(2p+1) + h, h = lane >> 4): contributors left
        // inside this bucket (0 = never got here) and the restart state, kept as fp32 pairs (f32x2.cuh)
        constexpr int NP = BWD_ROWPAIRS / 2;
        int rel[BWD_ROWPAIRS];
        // FAST keeps one suffix per pixel, Ag = sum_c a_c dL/dpix_c, instead of the three a_c: dL/dalpha only needs that sum
        f2 Tr[NP], a0[NP], a1[NP], a2[NP], Ag[NP];
        const float qy0f = (float)qy0;
        int rel_max[BWD_ROWPAIRS];                            // warp-uniform: deepest pixel of each row pair
        int n_max = 0;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            float st[2][7];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = 2 * p + h;
                const int qy = qy0 + 2 * j;
                int n = 0;
                size_t qi = 0;
                if (qx < vp.W && qy < vp.H) { qi = (size_t)qy * vp.W + qx; n = (int)n_contrib[qi]; }
                rel[j] = min(max(n - bucket_start, 0), BUCKET);
#pragma unroll
                for (int e = 0; e < 7; ++e) st[h][e] = 0.f;
                if (rel[j] > 0) {
                    const float4 k4 = ckpt[(size_t)bucket * TILE_PIX + j * 32 + lane];
                    st[h][0] = k4.x;
                    st[h][1] = k4.y - pixel_colors[qi]; st[h][2] = k4.z - pixel_colors[HW + qi]; st[h][3] = k4.w - pixel_colors[2 * HW + qi];
                    st[h][4] = dL_dpix[qi]; st[h][5] = dL_dpix[HW + qi]; st[h][6] = dL_dpix[2 * HW + qi];
                }
                rel_max[j] = (int)__reduce_max_sync(0xffffffffu, (unsigned)rel[j]);
                n_max = max(n_max, rel_max[j]);
            }
            Tr[p] = f2_pack(st[0][0], st[1][0]);
            a0[p] = f2_pack(st[0][1], st[1][1]); a1[p] = f2_pack(st[0][2], st[1][2]); a2[p] = f2_pack(st[0][3], st[1][3]);
            Ag[p] = f2_fma(a2[p], f2_pack(st[0][6], st[1][6]), f2_fma(a1[p], f2_pack(st[0][5], st[1][5]), f2_mul(a0[p], f2_pack(st[0][4], st[1][4]))));
            s_g[warp][p][0][lane] = make_float2(st[0][4], st[1][4]);
            s_g[warp][p][1][lane] = make_float2(st[0][5], st[1][5]);
            s_g[warp][p][2][lane] = make_float2(st[0][6], st[1][6]);
        }

        // stage the bucket's splats (lane l <-> splat l) and the row pairs each one can reach
        {
            uint32_t gid = 0;
            float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0, r2 = r0;
            uint32_t rows = 0;
            if (lane < n_valid && lane < n_max) {
                gid = point_list[range.x + bucket_start + lane];
                r0 = rec[3 * (size_t)gid + 0]; r1 = rec[3 * (size_t)gid + 1]; r2 = rec[3 * (size_t)gid + 2];
#pragma unroll
                for (int j = 0; j < BWD_ROWPAIRS; ++j) {
                    const float row_mid = (float)(row0 + 2 * j) + 0.5f;
                    if (lane < rel_max[j] && !(fabsf(row_mid - r0.y) > r2.w + 0.5f)) rows |= 1u << j;
                }
            }
            __syncwarp();                                    // previous bucket's readers are done
            sp[lane][0] = r0; sp[lane][1] = r1; sp[lane][2] = r2;
            s_gid[warp][lane] = gid;
            s_rows[warp][lane] = rows;
            __syncwarp();
        }

        uint32_t todo = __ballot_sync(0xffffffffu, s_rows[warp][lane] != 0);
        if (COUNT && lane == 0) ctr[BC_SPLATS] += __popc(todo);
        uint32_t emitted = 0;                                    // DET: slots whose nine values were stored (warp-uniform)
        while (todo) {
            const int k = __ffs(todo) - 1;
            todo &= todo - 1;
            const float4 a = sp[k][0], b = sp[k][1];
            const float c2 = sp[k][2].x;
            const uint32_t rows = s_rows[warp][k];
            const float dx = fsub(a.x, pfx);
            const float cxdx = fmul(dx, a.z), cydx = fmul(dx, a.w);      // shared by the lane's pixels: same column
            // Per-splat sums of this lane.  dx is the same for all of the lane's pixels, so only three moments of
            // w = G * dL/dalpha over the pixels are needed: S0 = sum w, S1 = sum w dy, S2 = sum w dy^2 (the five geometric
            // gradients are linear combinations of them, formed once per splat below), plus the three colour sums.
            f2 S0 = f2_bcast(0.f), S1 = S0, S2 = S0, c0s = S0, c1s = S0, c2s = S0;
            // Row pairs are taken two at a time: one warp-uniform branch per PAIR of row pairs, the two pixels evaluated by
            // the same pair operations WITHOUT branches (a pixel that does not take the splat gets
            // alpha = G = 0, which makes every term an exact zero and leaves T untouched).
#pragma unroll
            for (int p = 0; p < NP; ++p) {
                const unsigned two = (rows >> (2 * p)) & 3u;
                if (!two) continue;                                       // warp-uniform
                const f2 dy = f2_sub(f2_bcast(a.y), f2_pack(qy0f + (float)(4 * p), qy0f + (float)(4 * p + 2)));   // integers < 2^24: exact
                // splat_power(dx, dy, cx, cy, cz) in the forward's operation order, both pixels at once
                const f2 power = f2_sub(f2_mul(f2_fma(dx, cxdx, f2_mul(dy, f2_mul(dy, b.x))), -0.5f), f2_mul(dy, cydx));
                float p0, p1;
                f2_unpack(power, p0, p1);
                const bool cand0 = ((two & 1u) != 0) & (k < rel[2 * p]) & (p0 <= 0.0f);
                const bool cand1 = ((two & 2u) != 0) & (k < rel[2 * p + 1]) & (p1 <= 0.0f);
                float G0, G1, x0, x1;
                bool take0, take1;
                if (FAST) {
                    // G = 2^(power log2 e) by MUFU.EX2.  The decision x = o G >= 1/255 must be the forward's, which computes
                    // x from the libdevice expf.  Only a pixel with x near 1/255 can be decided differently, and there
                    // G ~ 1/(255 o), so |power| ~ ln(255 o) <= ln 255 (o <= 1 is a sigmoid) and |y| = |power log2 e| <= 8.
                    // Relative distance between the fast x and the forward's x:
                    //   y = fl(power * fl(log2 e)): |dy| <= 8 * (2^-24 + 2^-24.5)   -> 2^y off by <= ln 2 * 2^-20.4 = 2^-20.9
                    //   ex2.approx.ftz.f32 <= 2 ulp = 2^-22, libdevice expf <= 2 ulp = 2^-22, the two products with o 2^-24 each
                    // in all < 2^-19.7.  A pixel whose fast x lies within 2^-16 (relative) of 1/255 is decided from the
                    // exact expf instead, so every decision is the forward's with a margin of 8x.  (o > 1 only widens
                    // |y| to log2(255 o): the band still covers that up to o ~ 2^56.)  Subnormal G flushes to 0, far
                    // below the band.  The fast G feeds the gradient terms: 2^-19.7 relative, far inside fp32 atomics noise.
                    float e0, e1;
                    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(fmul(fminf(p0, 0.0f), 1.44269504088896341f)));
                    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(fmul(fminf(p1, 0.0f), 1.44269504088896341f)));
                    G0 = e0; G1 = e1;
                    f2_unpack(f2_mul(f2_pack(G0, G1), b.y), x0, x1);
                    constexpr float thr = 1.0f / 255.0f, band = (1.0f / 255.0f) * (1.0f / 65536.0f);
                    const bool near0 = cand0 & (fabsf(x0 - thr) <= band), near1 = cand1 & (fabsf(x1 - thr) <= band);
                    if (near0 | near1) {                                  // rare: the forward's expf for these pixels
                        if (near0) { G0 = expf(p0); x0 = fmul(G0, b.y); }
                        if (near1) { G1 = expf(p1); x1 = fmul(G1, b.y); }
                    }
                    if (COUNT) ctr[BC_FALLBACK] += (unsigned)near0 + (unsigned)near1;
                    x0 = fminf(0.99f, x0); x1 = fminf(0.99f, x1);
                    take0 = cand0 & (x0 >= thr);
                    take1 = cand1 & (x1 >= thr);
                    if (COUNT) {
                        const bool any = __any_sync(0xffffffffu, take0 | take1);
                        if (lane == 0) { ++ctr[BC_VISITS]; ctr[BC_VISITS_TAKEN] += any; }
                        ctr[BC_CAND] += (unsigned)cand0 + (unsigned)cand1; ctr[BC_TAKEN] += (unsigned)take0 + (unsigned)take1;
                    }
                } else {
                    G0 = expf(fminf(p0, 0.0f)); G1 = expf(fminf(p1, 0.0f));
                    f2_unpack(f2_mul(f2_pack(G0, G1), b.y), x0, x1);
                    x0 = fminf(0.99f, x0); x1 = fminf(0.99f, x1);
                    take0 = cand0 & (x0 >= (1.0f / 255.0f));
                    take1 = cand1 & (x1 >= (1.0f / 255.0f));
                    if (COUNT) {
                        const bool any = __any_sync(0xffffffffu, take0 | take1);
                        if (lane == 0) { ++ctr[BC_VISITS]; ctr[BC_VISITS_TAKEN] += any; }
                        ctr[BC_CAND] += (unsigned)cand0 + (unsigned)cand1; ctr[BC_TAKEN] += (unsigned)take0 + (unsigned)take1;
                    }
                }
                const f2 G = f2_pack(take0 ? G0 : 0.0f, take1 ? G1 : 0.0f);
                const f2 alpha = f2_pack(take0 ? x0 : 0.0f, take1 ? x1 : 0.0f);
                const f2 one_m = f2_sub(f2_bcast(1.0f), alpha);
                const f2 T = Tr[p];
                const f2 dch = f2_mul(alpha, T);                          // d(channel) / d(colour)
                float m0, m1, i0, i1;                                     // 1/(1-alpha), 1-alpha in [0.01, 1]: MUFU.RCP
                f2_unpack(one_m, m0, m1);
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(i0) : "f"(m0));
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(i1) : "f"(m1));
                const f2 ainv = f2_pack(i0, i1);
                const float2 gr = s_g[warp][p][0][lane], gg = s_g[warp][p][1][lane], gb = s_g[warp][p][2][lane];
                const f2 g0 = f2_pack(gr.x, gr.y), g1 = f2_pack(gg.x, gg.y), g2 = f2_pack(gb.x, gb.y);
                c0s = f2_fma(dch, g0, c0s); c1s = f2_fma(dch, g1, c1s); c2s = f2_fma(dch, g2, c2s);
                f2 dLa;
                if (FAST) {
                    // dL/dalpha = sum_c (a_c' / (1 - alpha) + T c_c) g_c with a_c' = a_c + dch c_c, so with cg = sum_c c_c g_c:
                    // Ag' = Ag + dch cg and dL/dalpha = Ag' / (1 - alpha) + T cg (6 operations per pixel instead of 12)
                    const f2 cg = f2_fma(g2, c2, f2_fma(g1, b.w, f2_mul(g0, b.z)));
                    Ag[p] = f2_fma(dch, cg, Ag[p]);
                    dLa = f2_fma(ainv, Ag[p], f2_mul(T, cg));
                } else {
                    a0[p] = f2_fma(dch, f2_bcast(b.z), a0[p]);
                    dLa = f2_mul(f2_fma(ainv, a0[p], f2_mul(T, b.z)), g0);
                    a1[p] = f2_fma(dch, f2_bcast(b.w), a1[p]);
                    dLa = f2_fma(f2_fma(ainv, a1[p], f2_mul(T, b.w)), g1, dLa);
                    a2[p] = f2_fma(dch, f2_bcast(c2), a2[p]);
                    dLa = f2_fma(f2_fma(ainv, a2[p], f2_mul(T, c2)), g2, dLa);
                }
                Tr[p] = f2_mul(T, one_m);
                // constant factors (opacity, 0.5*W, 0.5*H, -0.5) are applied once per splat below
                const f2 w = f2_mul(G, dLa);                              // = dL_dG / opacity
                const f2 wy = f2_mul(w, dy);
                S0 = f2_add(S0, w);
                S1 = f2_add(S1, wy);
                S2 = f2_fma(wy, dy, S2);
            }
            float v_o = f2_lo(S0) + f2_hi(S0);
            float v_c0 = f2_lo(c0s) + f2_hi(c0s), v_c1 = f2_lo(c1s) + f2_hi(c1s), v_c2 = f2_lo(c2s) + f2_hi(c2s);
            // every sum of the lane is an exact 0 when no pixel contributed (w = 0 and dch = 0 term by term): skipping is exact
            if (!__any_sync(0xffffffffu, v_o != 0.f || v_c0 != 0.f || v_c1 != 0.f || v_c2 != 0.f)) continue;
            if (COUNT && lane == 0) ++ctr[BC_SPLATS_TAKEN];
            const float s1 = f2_lo(S1) + f2_hi(S1), s2 = f2_lo(S2) + f2_hi(S2);
            const float sx = dx * v_o;                                   // sum w dx
            const float v_mx = sx * a.z + s1 * a.w;                      // -> * (-opacity * 0.5 * W)
            const float v_my = s1 * b.x + sx * a.w;                      // -> * (-opacity * 0.5 * H)
            const float v_cx = sx * dx;                                  // -> * (-0.5 * opacity)
            const float v_cy = s1 * dx;
            const float v_cw = s2;
            // reduce-scatter of 8 values over the 32 lanes: halve the value set at xor 16, 8, 4, then plain butterflies
            const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
            const float r0 = (h16 ? v_cw : v_mx) + __shfl_xor_sync(0xffffffffu, h16 ? v_mx : v_cw, 16);
            const float r1 = (h16 ? v_c0 : v_my) + __shfl_xor_sync(0xffffffffu, h16 ? v_my : v_c0, 16);
            const float r2 = (h16 ? v_c1 : v_cx) + __shfl_xor_sync(0xffffffffu, h16 ? v_cx : v_c1, 16);
            const float r3 = (h16 ? v_c2 : v_cy) + __shfl_xor_sync(0xffffffffu, h16 ? v_cy : v_c2, 16);
            const float q0 = (h8 ? r2 : r0) + __shfl_xor_sync(0xffffffffu, h8 ? r0 : r2, 8);
            const float q1 = (h8 ? r3 : r1) + __shfl_xor_sync(0xffffffffu, h8 ? r1 : r3, 8);
            float w0 = (h4 ? q1 : q0) + __shfl_xor_sync(0xffffffffu, h4 ? q0 : q1, 4);
            w0 += __shfl_xor_sync(0xffffffffu, w0, 2);
            w0 += __shfl_xor_sync(0xffffffffu, w0, 1);
            v_o += __shfl_xor_sync(0xffffffffu, v_o, 16);
            v_o += __shfl_xor_sync(0xffffffffu, v_o, 8);
            v_o += __shfl_xor_sync(0xffffffffu, v_o, 4);
            v_o += __shfl_xor_sync(0xffffffffu, v_o, 2);
            v_o += __shfl_xor_sync(0xffffffffu, v_o, 1);
            if constexpr (DET) {
                // value order of an entry: mean.x, mean.y, conic.x, conic.y, conic.w, colour r, g, b, opacity
                emitted |= 1u << k;
                if (i_write && live < det.cap_live) {
                    const float val = lane == 1 ? v_o : w0;
                    det.vals[(size_t)9 * (32u * live + (uint32_t)k) + (lane == 1 ? 8 : slot)] = val * (f_op * b.y + f_one);
                }
            } else if (i_write) {
                const size_t gid = s_gid[warp][k];
                const float val = lane == 1 ? v_o : w0;
                atomicAdd(dst_base + dst_stride * gid + dst_off, val * (f_op * b.y + f_one));
            }
        }
        if constexpr (DET) {
            if (live < det.cap_live) {
                const uint32_t e = 32u * live + (uint32_t)lane;
                det.keys[e] = (emitted >> lane) & 1u ? s_gid[warp][lane] : det.sentinel;
                det.idx[e] = e;
            }
        }
    }
    if (COUNT) {
        if (blockIdx.x == 0 && threadIdx.x == 0) counters[BC_LIVE] = n_live;
#pragma unroll
        for (int c = BC_SPLATS; c < BC_N; ++c) {
            const unsigned s = __reduce_add_sync(0xffffffffu, ctr[c]);
            if (lane == 0 && s) atomicAdd(counters + c, (unsigned long long)s);
        }
    }
}

// ---- launchers ------------------------------------------------------------------------------
int launch_tile_ranges(int64_t R, const GeomHeader* ghdr, const uint32_t* keys_sorted, int T, ImageState img, bool buckets,
                       unsigned int* sorted_in_b, int cur, cudaStream_t s) {
    const unsigned int* r_dev = ghdr ? &ghdr->r_eff : nullptr;
    if (R > 0) {
        GLIC_LAUNCH_PDL(tile_ranges_kernel, (unsigned)((R + 1023) / 1024), 256, 0, s, R, r_dev, keys_sorted, (uint32_t)T, img.ranges);
    }
    GLIC_LAUNCH_PDL(bucket_scan_kernel, 1, 1024, 0, s, T, img.ranges, img.bucket_offsets, img.hdr, (long long)R, ghdr, buckets ? 1 : 0,
                    sorted_in_b, cur);
    return GLIC_OK;
}

int launch_render_forward(const ViewParams& vp, bool no_color, const uint32_t* point_list, GeomState g, ImageState img,
                          SampleState smp, float* out_color, float* out_final_T, cudaStream_t s) {
    dim3 grid(vp.grid_x, vp.grid_y), block(FWD_THREADS);
    render_forward_kernel<FWD_TRAIN><<<grid, block, 0, s>>>(vp, no_color, img.ranges, point_list, g.rec, img.bucket_offsets,
                                                            smp.bucket_to_tile, smp.ckpt,
                                                            img.n_contrib, img.max_contrib, img.pixel_colors, out_color,
                                                            out_final_T, nullptr, nullptr, nullptr, nullptr, nullptr);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_render_infer(const ViewParams& vp, const uint32_t* point_list, GeomState g, ImageState img, float* out_color,
                        float* out_final_T, float* out_depth, float* out_median, cudaStream_t s) {
    dim3 grid(vp.grid_x, vp.grid_y), block(FWD_THREADS);
    render_forward_kernel<FWD_INFER><<<grid, block, 0, s>>>(vp, false, img.ranges, point_list, g.rec, nullptr, nullptr, nullptr,
                                                            nullptr, nullptr, nullptr, out_color, out_final_T, out_depth, out_median,
                                                            nullptr, nullptr, nullptr);
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_render_score(const ViewParams& vp, const uint32_t* point_list, GeomState g, ImageState img, float* max_weight,
                        uint64_t* hits, uint64_t* ends, float* out_final_T, cudaStream_t s) {
    dim3 grid(vp.grid_x, vp.grid_y), block(FWD_THREADS);
    render_forward_kernel<FWD_SCORE><<<grid, block, 0, s>>>(vp, true, img.ranges, point_list, g.rec, nullptr, nullptr, nullptr,
                                                            nullptr, nullptr, nullptr, nullptr, out_final_T, nullptr, nullptr,
                                                            reinterpret_cast<unsigned int*>(max_weight),
                                                            reinterpret_cast<unsigned long long*>(hits),
                                                            reinterpret_cast<unsigned long long*>(ends));
    GLIC_LAUNCH_CHECK();
    return GLIC_OK;
}

int launch_render_backward(int P, const ViewParams& vp, int64_t max_buckets, const uint32_t* point_list, GeomState g,
                           ImageState img, SampleState smp, const float* dL_dpix, float* dL_dmean2D, float* dL_dconic,
                           float* dL_dopacity, float* dL_dcolors, cudaStream_t s, bool exact, unsigned long long* counters) {
    (void)P; (void)smp.bucket_to_tile;
    if (max_buckets <= 0) return GLIC_OK;
    const int T = vp.grid_x * vp.grid_y;
    GLIC_LAUNCH_PDL(live_scan_kernel, 1, 1024, 0, s, T, img.max_contrib, img.live_offsets, img.hdr);
    // The occupancy-derived grid size is a property of the DEVICE and the kernel: cached per device.
    using Kern = void (*)(ViewParams, int, ImageHeader*, const uint2*, const uint32_t*, const float4*, const uint32_t*,
                          const uint32_t*, const float4*, const uint32_t*, const float*, const float*, float*, float*, float*, float*,
                          unsigned long long*, DetOut);
    const int form = 2 * (int)exact + (counters != nullptr);
    const Kern kerns[4] = {render_backward_kernel<6, true, false>, render_backward_kernel<6, true, true>,
                           render_backward_kernel<5, false, false>, render_backward_kernel<5, false, true>};
    const Kern kern = kerns[form];
    static int blocks_per_device[4][64] = {};
    int dev = 0;
    GLIC_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) { set_error("render_backward: device index out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!blocks_per_device[form][dev]) {
        int sms = NUM_SMS, per_sm = 4;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, BWD_WARPS * 32, 0);
        blocks_per_device[form][dev] = sms * (per_sm > 0 ? per_sm : 1);
    }
    const int blocks = blocks_per_device[form][dev];
    const int64_t need = (max_buckets + BWD_WARPS - 1) / BWD_WARPS;
    GLIC_LAUNCH_PDL(kern, (unsigned)std::min<int64_t>(blocks, need), BWD_WARPS * 32, 0, s, vp, T, img.hdr, img.ranges, point_list, g.rec,
                    img.bucket_offsets, img.live_offsets, smp.ckpt, img.n_contrib, img.pixel_colors, dL_dpix, dL_dmean2D, dL_dconic,
                    dL_dopacity, dL_dcolors, counters, DetOut{});
    return GLIC_OK;
}

// ---- deterministic render backward: stable sort of the entries by gid, then one fold per Gaussian ---------------------------
// Association of a Gaussian's contributions v_0 .. v_{n-1} (ascending tile), per value:
//   chunk c = v_{32c} .. v_{32c+31} (the last one shorter) is left-folded from its first element: s_c = ((v_{32c} + v_{32c+1}) + ...);
//   the result is the left fold of the chunk sums in chunk order: ((s_0 + s_1) + s_2) + ...
// For n <= 32 that is the strict left fold.  One warp per window of 32 sorted positions: each lane that heads a run of at most 32
// entries folds it alone; a longer run is folded by the whole warp, one chunk per lane and 32 chunks per round, and lane order
// folds the chunk sums.
__device__ __forceinline__ void det_load9(const float* __restrict__ vals, uint32_t e, float (&v)[9]) {
#pragma unroll
    for (int j = 0; j < 9; ++j) v[j] = vals[(size_t)9 * e + j];
}
__device__ __forceinline__ void det_store9(uint32_t gid, const float (&s)[9], float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic,
                                           float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolors) {
    dL_dmean2D[3 * (size_t)gid + 0] = s[0]; dL_dmean2D[3 * (size_t)gid + 1] = s[1];
    dL_dconic[4 * (size_t)gid + 0] = s[2]; dL_dconic[4 * (size_t)gid + 1] = s[3]; dL_dconic[4 * (size_t)gid + 3] = s[4];
    dL_dcolors[3 * (size_t)gid + 0] = s[5]; dL_dcolors[3 * (size_t)gid + 1] = s[6]; dL_dcolors[3 * (size_t)gid + 2] = s[7];
    dL_dopacity[gid] = s[8];
}

__global__ void __launch_bounds__(256)
det_reduce_kernel(const unsigned int* __restrict__ count, uint32_t P, const uint32_t* __restrict__ keys, const uint32_t* __restrict__ idx,
                  const float* __restrict__ vals, float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic,
                  float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolors) {
    pdl_enter();
    const uint32_t n = *count;
    const int lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t base = 32u * (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)); base < n; base += 32u * warps) {
        const uint32_t i = base + lane;
        const uint32_t key = i < n ? keys[i] : P;
        const bool head = key < P && (i == 0 || keys[i - 1] != key);
        const bool is_long = head && i + 32 < n && keys[i + 32] == key;
        if (head && !is_long) {
            float s[9], v[9];
            det_load9(vals, idx[i], s);
            for (uint32_t j = i + 1; j < n && keys[j] == key; ++j) {
                det_load9(vals, idx[j], v);
#pragma unroll
                for (int q = 0; q < 9; ++q) s[q] = __fadd_rn(s[q], v[q]);
            }
            det_store9(key, s, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolors);
        }
        uint32_t longs = __ballot_sync(0xffffffffu, is_long);
        while (longs) {
            const int h = __ffs(longs) - 1;
            longs &= longs - 1;
            const uint32_t start = base + (uint32_t)h, gid = __shfl_sync(0xffffffffu, key, h);
            float tot[9] = {};
            bool first = true, more = true;
            for (uint32_t round = 0; more; ++round) {
                const uint32_t cs = start + 32u * (32u * round + (uint32_t)lane);     // this lane's chunk
                const bool mine = cs < n && keys[cs] == gid;
                float s[9] = {}, v[9];
                if (mine) {
                    det_load9(vals, idx[cs], s);
                    for (uint32_t j = cs + 1; j < cs + 32 && j < n && keys[j] == gid; ++j) {
                        det_load9(vals, idx[j], v);
#pragma unroll
                        for (int q = 0; q < 9; ++q) s[q] = __fadd_rn(s[q], v[q]);
                    }
                }
                const uint32_t have = __ballot_sync(0xffffffffu, mine);      // a prefix of the lanes: the run is contiguous
                for (int l = 0; l < 32 && ((have >> l) & 1u); ++l) {
#pragma unroll
                    for (int q = 0; q < 9; ++q) {
                        const float c = __shfl_sync(0xffffffffu, s[q], l);
                        tot[q] = first ? c : __fadd_rn(tot[q], c);
                    }
                    first = false;
                }
                more = have == 0xffffffffu;
            }
            if (lane == 0) det_store9(gid, tot, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolors);
        }
    }
}

int launch_render_backward_det(int P, const ViewParams& vp, int64_t max_buckets, const uint32_t* point_list, GeomState g,
                               ImageState img, SampleState smp, DetState det, const float* dL_dpix, float* dL_dmean2D,
                               float* dL_dconic, float* dL_dopacity, float* dL_dcolors, cudaStream_t s) {
    if (max_buckets <= 0 || P <= 0) return GLIC_OK;
    const int T = vp.grid_x * vp.grid_y;
    GLIC_LAUNCH_PDL(live_scan_kernel, 1, 1024, 0, s, T, img.max_contrib, img.live_offsets, img.hdr);
    const auto kern = render_backward_kernel<6, true, false, true>;
    static int blocks_per_device[64] = {};
    int dev = 0;
    GLIC_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) { set_error("render_backward: device index out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!blocks_per_device[dev]) {
        int sms = NUM_SMS, per_sm = 4;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, BWD_WARPS * 32, 0);
        blocks_per_device[dev] = sms * (per_sm > 0 ? per_sm : 1);
    }
    const int64_t need = (max_buckets + BWD_WARPS - 1) / BWD_WARPS;
    const DetOut out{det.keys[0], det.idx[0], det.vals, det.count, (uint32_t)(det.cap / 32), (uint32_t)P};
    GLIC_LAUNCH_PDL(kern, (unsigned)std::min<int64_t>(blocks_per_device[dev], need), BWD_WARPS * 32, 0, s, vp, T, img.hdr, img.ranges,
                    point_list, g.rec, img.bucket_offsets, img.live_offsets, smp.ckpt, img.n_contrib, img.pixel_colors, dL_dpix, nullptr,
                    nullptr, nullptr, nullptr, nullptr, out);
    const int cur = launch_sort_pairs32(det.cap, det_key_bits(P), det.keys, det.idx, det.sort_temp, det.sort_temp_size, s, det.count, false);
    if (cur < 0) return cur;
    const int64_t windows = (det.cap + 31) / 32;
    const unsigned blocks = (unsigned)std::min<int64_t>((windows + 7) / 8, (int64_t)NUM_SMS * 16);
    GLIC_LAUNCH_PDL(det_reduce_kernel, blocks, 256, 0, s, det.count, (uint32_t)P, det.keys[cur], det.idx[cur], det.vals, dL_dmean2D,
                    dL_dconic, dL_dopacity, dL_dcolors);
    return GLIC_OK;
}

}  // namespace glic

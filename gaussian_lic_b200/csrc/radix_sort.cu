// radix_sort.cu -- CUB-free "onesweep" least-significant-digit radix sort of (u64 key, u32 value)
// pairs on key bits [0, end_bit).  Stable.
//
// Replaces cub::DeviceRadixSort::SortPairs(begin_bit = 0, end_bit = 32 + bit) as called at
// reference rasterizer_impl.cu:417-424 (and the Morton sort of simple_knn.cu:210-213).
//
// Structure (ceil(end_bit/8) passes, the key bits split evenly over them -- sort_pass_bits(): 13 -> 7 + 6, 45 -> 8,8,8,7,7,7 --
// so that no pass carries digits that cannot occur):
//   1. one histogram kernel builds the global digit histogram of EVERY pass in a single read of
//      the keys (8 B/pair);
//   2. a tiny kernel turns each histogram into exclusive digit offsets;
//   3. one kernel per pass: each CTA loads a 4096-pair tile (keys into registers, values straight into shared memory with
//      cp.async), counts its digits in shared memory and publishes those counts at once, ranks the tile (warp-synchronous,
//      stable: a branch-free cascade of one ballot per digit bit, then a leaderless update of the warp's digit counters --
//      MATCH.ANY measured slower), resolves its global digit
//      offsets with a per-digit decoupled look-back over dynamically ordered CTAs (no second read of the data), stages the
//      tile in shared memory in sorted order and writes digit runs out coalesced (24 B/pair/pass).
// Algorithmic HBM traffic: (8 + 24*passes) B per pair (152 B @ 45 bits).
#include "common.cuh"
#include <algorithm>

namespace glic {

size_t sort_temp_bytes(int64_t n);

namespace {

// Widest digit of a pass.  A pass is bound by the warp-synchronous ranking (one ballot per digit bit and item), not by its
// 24 B/pair of HBM traffic, so 9-bit digits cost more than the pass they save on 64-bit keys (measured, NOTES.md).
constexpr int RADIX_BITS = 8;
constexpr int RADIX = 1 << RADIX_BITS;
// Words the temp block reserves per pass for the histograms and, per CTA, for the status words: 512, twice the bins of
// the widest digit.  The reservation sets sort_temp_bytes and, through it, the workspace sizes and the binning capacity
// a workspace yields.
constexpr int RADIX_RESERVED = 512;
constexpr int SORT_THREADS = 256;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int SORT_ITEMS_BIG = 16;                     // 4096 pairs per CTA: the R-sized tile sort
constexpr int SORT_ITEMS_SMALL = 4;                    // 1024 pairs per CTA: inputs that would not fill the GPU with 4096-pair tiles
constexpr int64_t SORT_SMALL_LIMIT = (int64_t)NUM_SMS * 4 * SORT_THREADS * SORT_ITEMS_BIG;     // below ~2.2 M pairs use the small tile
constexpr int MAX_PASSES = 8;

constexpr uint32_t FLAG_AGG = 1u << 30;
constexpr uint32_t FLAG_PREFIX = 2u << 30;
constexpr uint32_t VALUE_MASK = (1u << 30) - 1;

struct SortTemp {
    uint32_t* hist;     // [MAX_PASSES][RADIX]  digit histograms -> exclusive offsets (MAX_PASSES * RADIX_RESERVED words reserved)
    uint32_t* tickets;  // [MAX_PASSES]
    uint32_t* status;   // per pass p: [blocks][1 << sort_pass_bits(p)], passes packed back to back
};

__host__ inline int sort_items(int64_t n) { return n < SORT_SMALL_LIMIT ? SORT_ITEMS_SMALL : SORT_ITEMS_BIG; }
__host__ inline int64_t sort_blocks(int64_t n) { const int64_t tile = (int64_t)SORT_THREADS * sort_items(n); return (n + tile - 1) / tile; }

// live digits of all passes together: the status words one CTA needs over the whole sort
__host__ inline int64_t sort_live_digits(int end_bit) {
    int64_t d = 0;
    for (int p = 0; p < sort_passes(end_bit); ++p) d += (int64_t)1 << sort_pass_bits(end_bit, p);
    return d;
}

__host__ inline SortTemp carve_sort_temp(void* temp) {
    char* p = static_cast<char*>(temp);
    SortTemp t;
    t.hist = reinterpret_cast<uint32_t*>(p);
    t.tickets = t.hist + MAX_PASSES * RADIX_RESERVED;
    t.status = t.tickets + 32;
    return t;
}

__device__ __forceinline__ uint32_t ld_volatile(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile(uint32_t* p, uint32_t v) {
    asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// 4-byte global -> shared copy that holds no register while in flight (LDGSTS); completed by cp_async_wait_all()
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src)
                 : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// ---- 1. all-pass histogram --------------------------------------------------------------
template <typename KeyT>
__global__ void __launch_bounds__(256)
sort_histogram_kernel(const KeyT* __restrict__ keys, int64_t n, const unsigned int* __restrict__ n_dev, int passes, int end_bit,
                      uint32_t* __restrict__ hist) {
    pdl_enter();
    if (n_dev) n = min(n, (int64_t)*n_dev);
    __shared__ uint32_t sh[MAX_PASSES * RADIX];
    for (int i = threadIdx.x; i < passes * RADIX; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const KeyT k = keys[i];
        for (int p = 0; p < passes; ++p) {
            const int bits = sort_pass_bits(end_bit, p);
            const uint32_t d = (uint32_t)(k >> sort_pass_shift(end_bit, p)) & ((1u << bits) - 1u);
            atomicAdd(&sh[p * RADIX + d], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < passes * RADIX; i += blockDim.x) {
        const uint32_t v = sh[i];
        if (v) atomicAdd(&hist[i], v);
    }
}

// ---- 2. exclusive scan of each pass's bins --------------------------------------------
__global__ void __launch_bounds__(RADIX_RESERVED) sort_scan_hist_kernel(uint32_t* __restrict__ hist) {
    pdl_enter();
    __shared__ uint32_t warp_tot[RADIX_RESERVED / 32];
    uint32_t* h = hist + blockIdx.x * blockDim.x;          // blockDim.x = RADIX: one pass's bins
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t v = h[tid];
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    uint32_t base = 0;
    for (int w = 0; w < warp; ++w) base += warp_tot[w];
    h[tid] = base + incl - v;
}

// ---- 3. one onesweep pass -------------------------------------------------------------------
template <typename KeyT, int SORT_ITEMS>
struct __align__(16) PassSmem {
    static constexpr int SORT_TILE = SORT_THREADS * SORT_ITEMS;
    KeyT keys[SORT_TILE];
    uint32_t vals[SORT_TILE];
    uint32_t warp_cnt[SORT_WARPS][RADIX];
    uint32_t tile_cnt[RADIX];
    uint32_t digit_excl[RADIX];
    uint32_t global_base[RADIX];
    uint32_t warp_tot[SORT_WARPS];
    uint32_t block_id;
};

// `bits` <= RADIX_BITS: this pass's digit width.  Only the 1 << bits live digits are counted, published and looked back on;
// `status` holds [blocks][1 << bits] words.
template <typename KeyT, int SORT_ITEMS>
__global__ void __launch_bounds__(SORT_THREADS, SORT_ITEMS <= 4 ? 6 : (sizeof(KeyT) == 4 ? 4 : 3))
onesweep_pass_kernel(const KeyT* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                     KeyT* __restrict__ keys_out, uint32_t* __restrict__ vals_out, int64_t n, const unsigned int* __restrict__ n_dev,
                     int shift, int bits, const uint32_t* __restrict__ digit_base, uint32_t* __restrict__ status,
                     uint32_t* __restrict__ ticket) {
    pdl_enter();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int SORT_TILE = SORT_THREADS * SORT_ITEMS;
    static_assert(RADIX == SORT_THREADS, "the per-digit phase gives each thread one digit");
    PassSmem<KeyT, SORT_ITEMS>& sm = *reinterpret_cast<PassSmem<KeyT, SORT_ITEMS>*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nd = 1 << bits;                               // live digits of this pass
    const uint32_t dmask = (uint32_t)nd - 1u;

    if (tid == 0) sm.block_id = atomicAdd(ticket, 1u);
    for (int i = tid; i < SORT_WARPS * RADIX; i += SORT_THREADS) (&sm.warp_cnt[0][0])[i] = 0;
    for (int i = tid; i < RADIX; i += SORT_THREADS) sm.tile_cnt[i] = 0;
    __syncthreads();
    if (n_dev) n = min(n, (int64_t)*n_dev);   // capacity-sized launch: the true count lives on the device
    const int64_t block = sm.block_id;
    const int64_t tile_base = block * SORT_TILE;
    if (tile_base >= n) return;                 // (CTA-uniform) nothing for this ticket
    const int count = (int)min((int64_t)SORT_TILE, n - tile_base);

    // -- load keys (warp-striped: lane l, item j <-> element warp*512 + j*32 + l; order-preserving) and count the tile's
    //    digits; the values travel to shared memory (tile order) asynchronously meanwhile, in no register
    KeyT k[SORT_ITEMS];
    uint32_t rank[SORT_ITEMS];
    const int wbase = warp * (32 * SORT_ITEMS);
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) {
        const int li = wbase + j * 32 + lane;
        if (li < count) cp_async4(&sm.vals[li], vals_in + tile_base + li);
        k[j] = li < count ? keys_in[tile_base + li] : (KeyT)~(KeyT)0;
    }
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j)
        if (wbase + j * 32 + lane < count) atomicAdd(&sm.tile_cnt[(uint32_t)(k[j] >> shift) & dmask], 1u);
    __syncthreads();
    // -- publish the tile's digit counts before ranking it: successors' look-backs need not wait for this CTA's ranking
    //    (thread t owns digit t here and in the per-digit phase)
    const uint32_t tot = tid < nd ? sm.tile_cnt[tid] : 0u;
    if (tid < nd) st_volatile(status + (size_t)block * nd + tid, (block == 0 ? FLAG_PREFIX : FLAG_AGG) | tot);

    // -- stable rank inside the warp's digit streams
    const uint32_t lt_mask = (1u << lane) - 1u;
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) {
        const int li = wbase + j * 32 + lane;
        const bool valid = li < count;
        const uint32_t d = (uint32_t)(k[j] >> shift) & dmask;
        const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
        uint32_t r = 0;
        // peers from RADIX_BITS ballots, with no branch on `bits` (the bits past it are clear in every d and change nothing): the
        // branch-free cascade measured faster than skipping the dead ballots.  Cost is independent of the digit
        // distribution; MATCH.ANY measured ~1.35x slower per pass on H100
        uint32_t bpeers = vmask;
#pragma unroll
        for (int b = 0; b < RADIX_BITS; ++b) {
            const bool bit = (d >> b) & 1u;
            const uint32_t bal = __ballot_sync(0xffffffffu, bit && valid);
            bpeers &= bit ? bal : ~bal;
        }
        // every peer reads its digit's running count and writes back the same new value: no leader election, no shuffle,
        // no divergent branch in the per-item chain
        const uint32_t c = sm.warp_cnt[warp][d];
        __syncwarp();
        if (valid) {
            sm.warp_cnt[warp][d] = c + __popc(bpeers);
            r = c + __popc(bpeers & lt_mask);
        }
        rank[j] = r;
        __syncwarp();
    }
    __syncthreads();

    // -- per digit (thread t owns digit t): warp bases, CTA-local placement, look-back
    {
        if (tid < nd) {
            uint32_t t = 0;
#pragma unroll
            for (int w = 0; w < SORT_WARPS; ++w) {
                const uint32_t c = sm.warp_cnt[w][tid];
                sm.warp_cnt[w][tid] = t;
                t += c;
            }
        }
        // CTA-local exclusive scan over digits (placement inside the staged tile)
        uint32_t incl = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) sm.warp_tot[warp] = incl;
        __syncthreads();
        uint32_t dbase = 0;
        for (int w = 0; w < warp; ++w) dbase += sm.warp_tot[w];
        const uint32_t excl = dbase + incl - tot;
        if (tid < nd) {
            sm.digit_excl[tid] = excl;
            // decoupled look-back for this digit (its aggregate went out before the ranking)
            uint32_t prev = 0;
            if (block > 0) {
                int64_t b = block - 1;
                unsigned spins = 0;
                while (true) {
                    const uint32_t s = ld_volatile(status + (size_t)b * nd + tid);
                    const uint32_t f = s & ~VALUE_MASK;
                    if (f == 0) {
                        if (++spins > (1u << 26)) __trap();   // fail loudly rather than hang the GPU
                        continue;
                    }
                    prev += s & VALUE_MASK;
                    if (f == FLAG_PREFIX) break;
                    --b;
                }
                st_volatile(status + (size_t)block * nd + tid, FLAG_PREFIX | (prev + tot));
            }
            sm.global_base[tid] = digit_base[tid] + prev - excl;
        }
    }
    __syncthreads();

    // -- stage the tile in sorted order: keys straight from registers (their ranks become positions), then the values,
    //    which sit in the same buffer in tile order, through registers
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) {
        const int li = wbase + j * 32 + lane;
        if (li < count) {
            const uint32_t d = (uint32_t)(k[j] >> shift) & dmask;
            rank[j] += sm.digit_excl[d] + sm.warp_cnt[warp][d];
            sm.keys[rank[j]] = k[j];
        }
    }
    cp_async_wait_all();
    __syncthreads();
    uint32_t v[SORT_ITEMS];
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) {
        const int li = wbase + j * 32 + lane;
        v[j] = li < count ? sm.vals[li] : 0u;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j)
        if (wbase + j * 32 + lane < count) sm.vals[rank[j]] = v[j];
    __syncthreads();

    // -- coalesced write-out of digit runs
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) {
        const int i = j * SORT_THREADS + tid;
        if (i < count) {
            const KeyT key = sm.keys[i];
            const uint32_t d = (uint32_t)(key >> shift) & dmask;
            const size_t dst = (size_t)sm.global_base[d] + i;
            keys_out[dst] = key;
            vals_out[dst] = sm.vals[i];
        }
    }
}

}  // namespace

// zeroes the histograms, tickets and look-back status words of a sort of n pairs on bits [0, end_bit)
size_t sort_prepare_bytes(int64_t n, int end_bit) {
    return n <= 0 ? 0 : sizeof(uint32_t) * (MAX_PASSES * RADIX_RESERVED + 32 + (size_t)sort_blocks(n) * sort_live_digits(end_bit));
}

int sort_prepare(int64_t n, int end_bit, void* temp, cudaStream_t s) {
    if (n <= 0) return GLIC_OK;
    GLIC_CUDA_TRY(cudaMemsetAsync(temp, 0, sort_prepare_bytes(n, end_bit), s));
    return GLIC_OK;
}

uint32_t* sort_hist(void* temp) { return static_cast<uint32_t*>(temp); }      // [MAX_PASSES][256], pass-major

size_t sort_temp_bytes(int64_t n) {
    const size_t blocks = (size_t)sort_blocks(n > 0 ? n : 1);
    return sizeof(uint32_t) * (MAX_PASSES * RADIX_RESERVED + 32 + (size_t)MAX_PASSES * blocks * RADIX_RESERVED) + 256;
}

template <typename KeyT, int ITEMS>
static int run_passes(int64_t n, int passes, int end_bit, int64_t blocks, KeyT* keys[2], uint32_t* vals[2], const SortTemp& t, cudaStream_t s,
                      const unsigned int* n_dev) {
    static bool attr_set[64] = {};
    if (first_use_on_device(attr_set)) {
        GLIC_CUDA_TRY(cudaFuncSetAttribute(onesweep_pass_kernel<KeyT, ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)sizeof(PassSmem<KeyT, ITEMS>)));
    }
    int cur = 0;
    uint32_t* status = t.status;
    for (int p = 0; p < passes; ++p) {
        const int bits = sort_pass_bits(end_bit, p);
        GLIC_LAUNCH_PDL(onesweep_pass_kernel<KeyT, ITEMS>, (unsigned)blocks, SORT_THREADS, sizeof(PassSmem<KeyT, ITEMS>), s,
                        keys[cur], vals[cur], keys[cur ^ 1], vals[cur ^ 1], n, n_dev, sort_pass_shift(end_bit, p), bits,
                        t.hist + p * RADIX, status, t.tickets + p);
        status += (size_t)blocks << bits;     // each pass's status words cover its live digits only
        cur ^= 1;
    }
    return cur;
}

// hist_ready: the caller zeroed the temp block with sort_prepare() and a producer kernel already accumulated the digit
// histograms of every pass into sort_hist(temp) (digits of sort_pass_bits(end_bit, p)): the histogram kernel -- one more
// read of all keys -- is skipped.
template <typename KeyT>
static int launch_sort_pairs_t(int64_t n, int end_bit, KeyT* keys[2], uint32_t* vals[2], void* temp, size_t temp_bytes,
                               cudaStream_t s, const unsigned int* n_dev = nullptr, bool hist_ready = false) {
    if (end_bit < 1 || end_bit > (int)(8 * sizeof(KeyT))) { set_error("sort: end_bit out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (n >= (int64_t)VALUE_MASK) { set_error("sort: n too large"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (n <= 0) return 0;
    const int passes = sort_passes(end_bit);
    if (passes > MAX_PASSES) { set_error("sort: too many passes"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (temp_bytes < sort_temp_bytes(n)) { set_error("sort: temp too small"); return GLIC_ERR_WORKSPACE; }
    const int64_t blocks = sort_blocks(n);
    SortTemp t = carve_sort_temp(temp);
    if (!hist_ready) {
        if (int e = sort_prepare(n, end_bit, temp, s)) return e;
        int hist_blocks = (int)std::min<int64_t>((n + 256 * 16 - 1) / (256 * 16), (int64_t)NUM_SMS * 8);
        GLIC_LAUNCH_PDL(sort_histogram_kernel<KeyT>, hist_blocks, 256, 0, s, keys[0], n, n_dev, passes, end_bit, t.hist);
    }
    GLIC_LAUNCH_PDL(sort_scan_hist_kernel, passes, RADIX, 0, s, t.hist);
    return sort_items(n) == SORT_ITEMS_SMALL ? run_passes<KeyT, SORT_ITEMS_SMALL>(n, passes, end_bit, blocks, keys, vals, t, s, n_dev)
                                             : run_passes<KeyT, SORT_ITEMS_BIG>(n, passes, end_bit, blocks, keys, vals, t, s, n_dev);
}

int launch_sort_pairs(int64_t n, int end_bit, uint64_t* keys[2], uint32_t* vals[2], void* temp, size_t temp_bytes,
                      cudaStream_t s) {
    return launch_sort_pairs_t<uint64_t>(n, end_bit, keys, vals, temp, temp_bytes, s);
}

int launch_sort_pairs32(int64_t n, int end_bit, uint32_t* keys[2], uint32_t* vals[2], void* temp, size_t temp_bytes,
                        cudaStream_t s, const unsigned int* n_dev, bool hist_ready) {
    return launch_sort_pairs_t<uint32_t>(n, end_bit, keys, vals, temp, temp_bytes, s, n_dev, hist_ready);
}

}  // namespace glic

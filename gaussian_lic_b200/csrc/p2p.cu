// p2p.cu -- in-place mean all-reduce of the packed gradient buffer over NVLink peer memory (our own collective).
//
// The view-sharded mapping iteration (SURVEY.md 8e) has exactly one exchange step: every rank holds the
// per-Gaussian gradients of its own view and needs their mean, plus the union of the visibility bytes.
// Instead of handing that to a library, each rank maps every peer's gradient buffer (CUDA IPC) and runs a
// two-shot all-reduce itself: rank r owns slice r of the buffer, loads that slice from all peers straight
// over NVLink (128-bit loads), reduces in registers and stores the result back into every peer's buffer
// (128-bit stores).  Slice r of any buffer is read and written by rank r only, so the exchange is in place.
// Two tiny signalling kernels (system-scope release/acquire flags in the mapped buffers) order it against
// the peers' backward kernels and against their readers.  Bytes over NVLink per rank: 2*(N-1)/N of the
// payload, the minimum for an all-reduce.
#include "common.cuh"
#include "adam_math.cuh"
#include <algorithm>
#include <cstring>
#include <cstdlib>

namespace glic {

namespace {

constexpr int P2P_MAX_RANKS = 8;

struct PeerBufs { char* p[P2P_MAX_RANKS]; };

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// Flag block (256 B at flag_off of every rank's buffer): words [0, 8) = "peer q reached epoch e" (written by peer q),
// word 8 = this rank's epoch counter, word 9 = sticky error word (1 = a barrier timed out).
constexpr int P2P_EPOCH_WORD = P2P_MAX_RANKS;
constexpr int P2P_ERROR_WORD = P2P_MAX_RANKS + 1;

// Thread q tells peer q "rank `rank` reached epoch e", then waits until peer q has told us the same.
// The epoch lives in the rank's own flag block and advances by one per barrier, so the launch carries no per-call
// argument and the whole exchange can sit inside a replayed CUDA graph.  The wait is bounded in TIME (%globaltimer,
// GLIC_P2P_TIMEOUT_MS, default 20 s): a slow peer (first-iteration module load, graph instantiation, two ranks
// time-sliced on one GPU) never trips it, a lost peer sets the sticky error word and lets the kernel end -- the context
// stays healthy and the host reads the error with glic_p2p_check().
__global__ void p2p_barrier_kernel(PeerBufs bufs, int rank, int world, size_t flag_off, unsigned long long timeout_ns) {
    const int q = threadIdx.x;
    uint32_t epoch = 0;
    uint32_t* own = reinterpret_cast<uint32_t*>(bufs.p[rank] + flag_off);
    if (q == 0) {
        epoch = own[P2P_EPOCH_WORD] + 1;
        own[P2P_EPOCH_WORD] = epoch;
    }
    epoch = __shfl_sync(0xffffffffu, epoch, 0);
    if (q >= world) return;
    __threadfence_system();
    uint32_t* remote = reinterpret_cast<uint32_t*>(bufs.p[q] + flag_off) + rank;
    st_release_sys(remote, epoch);
    const uint32_t* local = own + q;
    const unsigned long long t0 = globaltimer_ns();
    unsigned int polls = 0;
    while ((int)(ld_acquire_sys(local) - epoch) < 0) {
        if ((++polls & 1023u) == 0 && globaltimer_ns() - t0 > timeout_ns) {
            own[P2P_ERROR_WORD] = 1u;
            break;
        }
    }
}

// slice [lo4, hi4) in float4 units: mean over ranks; [vlo4, vhi4) in uint4 units: bitwise OR (visibility bytes are 0/1).
// UNROLL independent 16-byte loads per peer are issued before the first use so that a thread keeps
// world*UNROLL NVLink requests in flight (remote-load latency is a few microseconds).
template <int WORLD, int UNROLL>
__global__ void __launch_bounds__(512)
p2p_reduce_kernel(PeerBufs bufs, size_t lo4, size_t hi4, size_t vis_off, size_t vlo4, size_t vhi4, float inv) {
    const size_t tile = (size_t)blockDim.x * UNROLL;
    const size_t stride = (size_t)gridDim.x * tile;
    for (size_t base = lo4 + (size_t)blockIdx.x * tile + threadIdx.x; base < hi4; base += stride) {
        float4 v[WORLD][UNROLL];
#pragma unroll
        for (int q = 0; q < WORLD; ++q)
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const size_t i = base + (size_t)u * blockDim.x;
                v[q][u] = i < hi4 ? __ldcv(reinterpret_cast<const float4*>(bufs.p[q]) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const size_t i = base + (size_t)u * blockDim.x;
            float4 acc = v[0][u];
#pragma unroll
            for (int q = 1; q < WORLD; ++q) { acc.x += v[q][u].x; acc.y += v[q][u].y; acc.z += v[q][u].z; acc.w += v[q][u].w; }
            acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
            if (i < hi4) {
#pragma unroll
                for (int q = 0; q < WORLD; ++q) reinterpret_cast<float4*>(bufs.p[q])[i] = acc;
            }
        }
    }
    const size_t vstride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = vlo4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < vhi4; i += vstride) {
        uint4 acc = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int q = 0; q < WORLD; ++q) {
            const uint4 w = __ldcv(reinterpret_cast<const uint4*>(bufs.p[q] + vis_off) + i);
            acc.x |= w.x; acc.y |= w.y; acc.z |= w.z; acc.w |= w.w;
        }
#pragma unroll
        for (int q = 0; q < WORLD; ++q) reinterpret_cast<uint4*>(bufs.p[q] + vis_off)[i] = acc;
    }
}

unsigned long long p2p_timeout_ns() {
    static const unsigned long long ns = [] {
        const char* e = getenv("GLIC_P2P_TIMEOUT_MS");
        const long long ms = e ? atoll(e) : 20000;
        return (unsigned long long)(ms > 0 ? ms : 20000) * 1000000ull;
    }();
    return ns;
}

constexpr int P2P_CTAS_PER_SM = 2;        // CTAs of p2p_reduce_kernel per SM, at most

template <int WORLD, int UNROLL>
void launch_reduce(const PeerBufs& pb, size_t lo4, size_t hi4, size_t vis_off, size_t vlo4, size_t vhi4, cudaStream_t s) {
    const size_t work = std::max((hi4 - lo4 + UNROLL - 1) / UNROLL, vhi4 - vlo4);
    const unsigned blocks = (unsigned)std::max<size_t>(1, std::min<size_t>((work + 511) / 512, (size_t)NUM_SMS * P2P_CTAS_PER_SM));
    p2p_reduce_kernel<WORLD, UNROLL><<<blocks, 512, 0, s>>>(pb, lo4, hi4, vis_off, vlo4, vhi4, 1.0f / (float)WORLD);
}

// ---- reduce-scatter -> Adam on the local slice -> all-gather of PARAMETERS (DESIGN.md 7) ---------------------------------
// Same NVLink bytes as the all-reduce (gradients in, parameters out), Adam's HBM traffic and its moment buffers divided by
// `world`; bit-identical to all-reduce + packed Adam (tests/test_gpu_p2p_adam.py).
struct P2PLayout {
    size_t begin[6], end[6];
    uint32_t k[6];
    float lr[6];
};

template <int WORLD>
__global__ void __launch_bounds__(256)
p2p_reduce_adam_kernel(PeerBufs bufs, int rank, size_t lo4, size_t hi4, size_t vis_off, size_t params_off,
                       float4* __restrict__ exp_avg, float4* __restrict__ exp_avg_sq, P2PLayout L, size_t total, float b1, float b2,
                       float eps) {
    const float inv = 1.0f / (float)WORLD;
    const uint8_t* __restrict__ visible = reinterpret_cast<const uint8_t*>(bufs.p[rank] + vis_off);   // union, reduced just before
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = lo4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi4; i += stride) {
        float4 g4[WORLD];
#pragma unroll
        for (int q = 0; q < WORLD; ++q) g4[q] = __ldcv(reinterpret_cast<const float4*>(bufs.p[q]) + i);
        float4 acc = g4[0];
#pragma unroll
        for (int q = 1; q < WORLD; ++q) { acc.x += g4[q].x; acc.y += g4[q].y; acc.z += g4[q].z; acc.w += g4[q].w; }
        float g[4] = {acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv};
        float4 p4 = reinterpret_cast<const float4*>(bufs.p[rank] + params_off)[i];
        float4 m4 = exp_avg[i], v4 = exp_avg_sq[i];
        float p[4] = {p4.x, p4.y, p4.z, p4.w}, m[4] = {m4.x, m4.y, m4.z, m4.w}, v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const size_t j = 4 * i + c;
            if (j >= total) continue;
            int grp = 0;
#pragma unroll
            for (int q = 0; q < 5; ++q) grp += j >= L.end[q];
            if (!visible[(j - L.begin[grp]) / L.k[grp]]) continue;
            adam_element(p[c], m[c], v[c], g[c], L.lr[grp], b1, b2, eps);     // adam_math.cuh: shared with adam_kernel / adam_packed_kernel
        }
        exp_avg[i] = make_float4(m[0], m[1], m[2], m[3]);
        exp_avg_sq[i] = make_float4(v[0], v[1], v[2], v[3]);
        const float4 out = make_float4(p[0], p[1], p[2], p[3]);
#pragma unroll
        for (int q = 0; q < WORLD; ++q) reinterpret_cast<float4*>(bufs.p[q] + params_off)[i] = out;
    }
}

}  // namespace
}  // namespace glic

using namespace glic;

extern "C" {

size_t glic_p2p_buffer_bytes(size_t n_floats, size_t n_vis_bytes) {
    const size_t f = (n_floats * 4 + 255) & ~size_t(255);
    const size_t v = (n_vis_bytes + 255) & ~size_t(255);
    return f + v + 256;                     // + flag words (one per rank)
}

int glic_p2p_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64) {
    if (!dev_ptr || !handle64) { set_error("p2p_alloc: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    GLIC_CUDA_TRY(cudaMalloc(dev_ptr, bytes));
    GLIC_CUDA_TRY(cudaMemset(*dev_ptr, 0, bytes));
    cudaIpcMemHandle_t h;
    GLIC_CUDA_TRY(cudaIpcGetMemHandle(&h, *dev_ptr));
    static_assert(sizeof(h) == 64, "ipc handle size");
    memcpy(handle64, &h, 64);
    return GLIC_OK;
}

int glic_p2p_open(const unsigned char* handle64, void** peer_ptr) {
    if (!handle64 || !peer_ptr) { set_error("p2p_open: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    GLIC_CUDA_TRY(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return GLIC_OK;
}

int glic_p2p_close(void* peer_ptr) { GLIC_CUDA_TRY(cudaIpcCloseMemHandle(peer_ptr)); return GLIC_OK; }
int glic_p2p_free(void* dev_ptr) { GLIC_CUDA_TRY(cudaFree(dev_ptr)); return GLIC_OK; }

// Rank r's share of the two-shot exchange, in 16-byte units: floats [lo4, hi4), visibility [vlo4, vhi4) (relative to the
// visibility block at byte f_bytes); also the byte offsets of the visibility block and of the flag words.  The slices of the
// `world` ranks partition both blocks exactly (tests/test_cabi.py), so every 16-byte unit is reduced by exactly one rank.
int glic_p2p_slice(int rank, int world, size_t n_floats, size_t n_vis_bytes, size_t* out6) {
    if (world < 1 || world > P2P_MAX_RANKS || rank < 0 || rank >= world || !out6) { set_error("p2p_slice: bad rank / world"); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t f_bytes = (n_floats * 4 + 255) & ~size_t(255);
    const size_t v_bytes = (n_vis_bytes + 255) & ~size_t(255);
    const size_t f4 = f_bytes / 16, v4 = v_bytes / 16;
    const size_t fper = (f4 + world - 1) / world, vper = (v4 + world - 1) / world;
    out6[0] = std::min(f4, fper * rank); out6[1] = std::min(f4, fper * (rank + 1));
    out6[2] = std::min(v4, vper * rank); out6[3] = std::min(v4, vper * (rank + 1));
    out6[4] = f_bytes; out6[5] = f_bytes + v_bytes;
    return GLIC_OK;
}

int glic_p2p_allreduce_mean(int rank, int world, void* const* bufs_host, size_t n_floats, size_t n_vis_bytes, void* stream) {
    if (world < 1 || world > P2P_MAX_RANKS || rank < 0 || rank >= world || !bufs_host) { set_error("p2p_allreduce: bad rank / world"); return GLIC_ERR_INVALID_ARGUMENT; }
    cudaStream_t s = (cudaStream_t)stream;
    PeerBufs pb;
    for (int q = 0; q < P2P_MAX_RANKS; ++q) pb.p[q] = q < world ? static_cast<char*>(bufs_host[q]) : nullptr;
    size_t sl[6];
    glic_p2p_slice(rank, world, n_floats, n_vis_bytes, sl);
    const size_t lo4 = sl[0], hi4 = sl[1], vlo4 = sl[2], vhi4 = sl[3], f_bytes = sl[4], flag_off = sl[5];
    { StageTimer _t(GLIC_STAGE_ALLREDUCE, s);
      p2p_barrier_kernel<<<1, 32, 0, s>>>(pb, rank, world, flag_off, p2p_timeout_ns());         // every peer's gradients are complete
      GLIC_LAUNCH_CHECK();
      // UNROLL 16-byte loads in flight per peer: 4 up to 4 ranks, 2 above (at most 16 per thread)
#define GLIC_P2P_MEAN(WD) case WD: launch_reduce<WD, WD <= 4 ? 4 : 2>(pb, lo4, hi4, f_bytes, vlo4, vhi4, s); break;
      switch (world) { GLIC_P2P_MEAN(1) GLIC_P2P_MEAN(2) GLIC_P2P_MEAN(3) GLIC_P2P_MEAN(4) GLIC_P2P_MEAN(5) GLIC_P2P_MEAN(6) GLIC_P2P_MEAN(7) GLIC_P2P_MEAN(8) }
#undef GLIC_P2P_MEAN
      GLIC_LAUNCH_CHECK();
      p2p_barrier_kernel<<<1, 32, 0, s>>>(pb, rank, world, flag_off, p2p_timeout_ns());      // every slice has been written everywhere
      GLIC_LAUNCH_CHECK(); }
    return GLIC_OK;
}

// Synchronises `stream` and reports a barrier timeout recorded by any earlier exchange on this rank's buffer
// (GLIC_ERR_TIMEOUT; the error word is cleared).  buf = this rank's own block.
int glic_p2p_check(void* buf, size_t n_floats, size_t n_vis_bytes, void* stream) {
    if (!buf) { set_error("p2p_check: null buffer"); return GLIC_ERR_INVALID_ARGUMENT; }
    size_t sl[6];
    glic_p2p_slice(0, 1, n_floats, n_vis_bytes, sl);
    uint32_t* word = reinterpret_cast<uint32_t*>(static_cast<char*>(buf) + sl[5]) + P2P_ERROR_WORD;
    uint32_t err = 0;
    cudaStream_t s = (cudaStream_t)stream;
    GLIC_CUDA_TRY(cudaMemcpyAsync(&err, word, sizeof(err), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    if (err) {
        GLIC_CUDA_TRY(cudaMemsetAsync(word, 0, sizeof(err), s));
        set_error("p2p exchange: a peer did not reach the barrier within GLIC_P2P_TIMEOUT_MS");
        return GLIC_ERR_TIMEOUT;
    }
    return GLIC_OK;
}

// Buffer of the fused variant: gradients | visibility | flags (as glic_p2p_buffer_bytes) | parameters.
size_t glic_p2p_model_bytes(size_t n_floats, size_t n_vis_bytes) {
    return glic_p2p_buffer_bytes(n_floats, n_vis_bytes) + ((n_floats * 4 + 255) & ~size_t(255));
}

// bufs_host[q]: rank q's glic_p2p_model_bytes block.  exp_avg / exp_avg_sq: LOCAL, 16-byte aligned,
// n_floats rounded up to a multiple of 4 floats each (only this rank's slice is ever touched).  After the call every rank's parameter block holds the updated model.
int glic_p2p_reduce_adam(int rank, int world, void* const* bufs_host, uint32_t P, uint32_t M, float* exp_avg, float* exp_avg_sq,
                         const float* lr6_host, float b1, float b2, float eps, void* stream) {
    if (world < 1 || world > P2P_MAX_RANKS || rank < 0 || rank >= world || !bufs_host || !exp_avg || !exp_avg_sq || !lr6_host) {
        set_error("p2p_reduce_adam: bad arguments"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t s = (cudaStream_t)stream;
    PeerBufs pb;
    for (int q = 0; q < P2P_MAX_RANKS; ++q) pb.p[q] = q < world ? static_cast<char*>(bufs_host[q]) : nullptr;
    P2PLayout L;
    const uint32_t k[6] = {4, 3, 3, 1, 3, 3 * M};
    size_t off = 0;
    for (int q = 0; q < 6; ++q) { L.begin[q] = off; L.k[q] = k[q] ? k[q] : 1; L.lr[q] = lr6_host[q]; off += (size_t)P * k[q]; L.end[q] = off; }
    const size_t n_floats = off;
    size_t sl[6];
    glic_p2p_slice(rank, world, n_floats, (size_t)P, sl);
    // float4 units past the last real float belong to the padding: never touched (the moment buffers are not padded to 256 B)
    const size_t used4 = (n_floats + 3) / 4;
    const size_t lo4 = std::min(sl[0], used4), hi4 = std::min(sl[1], used4), vlo4 = sl[2], vhi4 = sl[3], f_bytes = sl[4], flag_off = sl[5];
    const size_t params_off = flag_off + 256;
    { StageTimer _t(GLIC_STAGE_ALLREDUCE, s);
      p2p_barrier_kernel<<<1, 32, 0, s>>>(pb, rank, world, flag_off, p2p_timeout_ns());          // every peer's gradients and visibility are complete
      GLIC_LAUNCH_CHECK();
#define GLIC_P2P_VIS(WD) case WD: launch_reduce<WD, 1>(pb, 0, 0, f_bytes, vlo4, vhi4, s); break;
      switch (world) { GLIC_P2P_VIS(1) GLIC_P2P_VIS(2) GLIC_P2P_VIS(3) GLIC_P2P_VIS(4) GLIC_P2P_VIS(5) GLIC_P2P_VIS(6) GLIC_P2P_VIS(7) GLIC_P2P_VIS(8) }
#undef GLIC_P2P_VIS
      GLIC_LAUNCH_CHECK();
      p2p_barrier_kernel<<<1, 32, 0, s>>>(pb, rank, world, flag_off, p2p_timeout_ns());          // the visibility union is everywhere
      GLIC_LAUNCH_CHECK();
      const unsigned blocks = (unsigned)std::max<size_t>(1, std::min<size_t>((hi4 - lo4 + 255) / 256, (size_t)NUM_SMS * 4));
#define GLIC_P2P_ADAM(WD) case WD: p2p_reduce_adam_kernel<WD><<<blocks, 256, 0, s>>>(pb, rank, lo4, hi4, f_bytes, params_off, \
          reinterpret_cast<float4*>(exp_avg), reinterpret_cast<float4*>(exp_avg_sq), L, n_floats, b1, b2, eps); break;
      switch (world) { GLIC_P2P_ADAM(1) GLIC_P2P_ADAM(2) GLIC_P2P_ADAM(3) GLIC_P2P_ADAM(4) GLIC_P2P_ADAM(5) GLIC_P2P_ADAM(6) GLIC_P2P_ADAM(7) GLIC_P2P_ADAM(8) }
#undef GLIC_P2P_ADAM
      GLIC_LAUNCH_CHECK();
      p2p_barrier_kernel<<<1, 32, 0, s>>>(pb, rank, world, flag_off, p2p_timeout_ns());          // every parameter slice has been written everywhere
      GLIC_LAUNCH_CHECK(); }
    return GLIC_OK;
}

}  // extern "C"

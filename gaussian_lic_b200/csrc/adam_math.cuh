// adam_math.cuh -- ONE definition of the visibility-masked Adam element update (adamUpdateCUDA, reference
// rasterizer/cuda_rasterizer/adam.cu:27-36: no bias correction, no weight decay), shared by the per-tensor kernel
// (adam_knn.cu), the packed-model kernel (model_step.cu) and the fused exchange + optimiser kernel (p2p.cu), so that the
// three are bit-identical by construction.  The operation order is pinned with round-to-nearest intrinsics (the compiler
// may neither fuse nor reassociate them): it is the order nvcc 12.9 picks for the reference's expression on sm_90a,
//     m' = fma(1-b1, g, b1*m)      v' = fma(g, (1-b2)*g, b2*v)      p' = p + (-lr*m') / (sqrt(v') + eps)
// with IEEE division and square root (the reference builds without fast-math).
#pragma once
#include <cuda_runtime.h>

namespace glic {

__device__ __forceinline__ void adam_element(float& p, float& m, float& v, float g, float lr, float b1, float b2, float eps) {
    const float mm = __fmaf_rn(__fsub_rn(1.0f, b1), g, __fmul_rn(b1, m));
    const float vv = __fmaf_rn(g, __fmul_rn(__fsub_rn(1.0f, b2), g), __fmul_rn(b2, v));
    p = __fadd_rn(p, __fdiv_rn(__fmul_rn(-lr, mm), __fadd_rn(__fsqrt_rn(vv), eps)));
    m = mm;
    v = vv;
}

// ---- the per-keyframe parameters of the mapper (exposure, pose): torch::optim::Adam, one step per batch ----------------

// torch::optim::Adam's update of one element at step `step` (1-based): betas (0.9, 0.999), eps 1e-8, no weight decay, float64
// bias corrections.  Moves m and v, returns the delta to add to the parameter.  Every operation is rounded on its own (no
// contraction), so that the CPU restatements (tests/exposure_oracle.py, tests/pose_oracle.py) can follow it.
__device__ __forceinline__ float torch_adam_delta(float g, float& m, float& v, float lr, int step) {
    const float b1 = 0.9f, b2 = 0.999f, eps = 1e-8f;
    const double bc1 = 1.0 - pow(0.9, (double)step), bc2 = 1.0 - pow(0.999, (double)step);
    const float m1 = fmaf(1.0f - b1, g, __fmul_rn(b1, m));
    const float v1 = fmaf(1.0f - b2, __fmul_rn(g, g), __fmul_rn(b2, v));
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v1), (float)sqrt(bc2)), eps);
    const float step_size = (float)((double)lr / bc1);
    m = m1;
    v = v1;
    return __fmul_rn(-step_size, __fdiv_rn(m1, denom));
}

// A batch of S slots may hold a keyframe more than once: the first slot holding it steps it ...
__device__ __forceinline__ bool first_slot_of_keyframe(const int* kf_of_slot, int s) {
    for (int q = 0; q < s; ++q)
        if (kf_of_slot[q] == kf_of_slot[s]) return false;
    return true;
}

// ... with g[j] = (1/S) * sum over the slots q >= s holding it (slot order, float64) of slot_grads[stride * q + j]
__device__ __forceinline__ float keyframe_batch_grad(const int* kf_of_slot, int S, int s, const float* slot_grads, int stride, int j) {
    double acc = 0.0;
    for (int q = s; q < S; ++q)
        if (kf_of_slot[q] == kf_of_slot[s]) acc += (double)slot_grads[stride * q + j];
    return (float)(acc / (double)S);
}

}  // namespace glic

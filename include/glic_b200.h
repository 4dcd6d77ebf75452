/*
 * glic_b200.h -- C ABI of the H100-native (sm_90a) Gaussian rasterizer hot path.
 *
 * Drop-in boundary for Gaussian-LIC (APRIL-ZJU/Gaussian-LIC @ 4566e6e).  Every entry point
 * replaces one raw-pointer interface of the reference; the LibTorch symbols the SLAM code
 * actually links against (RasterizeGaussiansCUDA, RasterizeGaussiansBackwardCUDA, adamUpdate,
 * fusedssim, fusedssim_backward, distCUDA2) are thin shims over this ABI
 * (gaussian_lic_b200/csrc/torch_shim.cpp, see INTEGRATION.md).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types, no exceptions across the ABI.
 *   - every pointer is a DEVICE pointer unless the parameter name ends in `_host`.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream, which is what
 *     the reference uses for every launch).
 *   - the library never allocates device memory: the caller provides workspaces whose sizes
 *     come from the glic_*_bytes() queries (replaces the reference's four
 *     std::function<char*(size_t)> resize callbacks, rasterizer.h:29-34).
 *   - return value: GLIC_OK (0) or a negative glic_status; glic_last_error() gives text.
 *   - all floating point is IEEE fp32; indices are 32-bit, keys 64-bit.
 *
 * Reference citations are relative to /root/reference/src/.
 */
#ifndef GLIC_B200_H_INCLUDED
#define GLIC_B200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GLIC_ABI_VERSION 1

#if defined(__GNUC__)
#define GLIC_API __attribute__((visibility("default")))
#else
#define GLIC_API
#endif

typedef enum glic_status {
    GLIC_OK = 0,
    GLIC_ERR_INVALID_ARGUMENT = -1, /* bad shape / null pointer / unsupported degree        */
    GLIC_ERR_WORKSPACE = -2,        /* a workspace is smaller than glic_*_bytes() requires   */
    GLIC_ERR_CUDA = -3,             /* a CUDA runtime call failed (text in glic_last_error)  */
    GLIC_ERR_NO_DEVICE = -4,        /* no CUDA device / wrong architecture                   */
    GLIC_ERR_TIMEOUT = -5           /* a multi-GPU peer did not reach the exchange barrier   */
} glic_status;

/* Tile geometry is part of the parity contract (rasterizer/cuda_rasterizer/config.h:16-17). */
#define GLIC_TILE 16
#define GLIC_BUCKET 32 /* checkpoint period of the per-splat backward (forward.cu:412) */
/* Largest frame: ceil(width/16) * ceil(height/16) <= GLIC_MAX_TILES (4096x4096 is the largest square frame).  Tile ids are
 * sorted on at most 16 bits.  Every call that takes a glic_view refuses a larger frame with GLIC_ERR_INVALID_ARGUMENT
 * before it enqueues any work. */
#define GLIC_MAX_TILES 65536

GLIC_API const char* glic_last_error(void);
GLIC_API int glic_abi_version(void);

/* Per-view camera block, all DEVICE pointers except the scalars.
 * view/proj: 16 floats each, column-major Rt and P*Rt exactly as the reference's kernels get
 * them (rasterize_points.cu:129-130, camera.h:60,86,109).  campos: 3 floats. */
typedef struct glic_view {
    const float* viewmatrix;
    const float* projmatrix;
    const float* campos;
    float tan_fovx, tan_fovy;
    float limx_neg, limx_pos, limy_neg, limy_pos; /* camera.h:63-66 */
    int width, height;
} glic_view;

/* ---------------------------------------------------------------------------------------
 * Workspace sizes.  Replaces required<GeometryState/ImageState/BinningState/SampleState>()
 * (rasterizer/cuda_rasterizer/rasterizer_impl.h:92-108, rasterizer_impl.cu:233-291).
 * The four buffers are opaque and may be round-tripped by the caller between forward and
 * backward (rasterizer.cpp:83-98 saves them in the autograd context).
 * ------------------------------------------------------------------------------------- */
GLIC_API size_t glic_geom_bytes(int P);
GLIC_API size_t glic_image_bytes(int width, int height);
GLIC_API size_t glic_binning_bytes(int64_t num_rendered);
GLIC_API size_t glic_sample_bytes(int64_t num_rendered, int width, int height); /* upper bound on buckets */
GLIC_API int64_t glic_max_buckets(int64_t num_rendered, int width, int height);

/* ---------------------------------------------------------------------------------------
 * Forward, stage 1: per-Gaussian preprocess + tile counting + prefix sum.
 * Replaces FORWARD::preprocess + cub::DeviceScan::InclusiveSum + the D2H read of
 * num_rendered (rasterizer_impl.cu:362-398; forward.cu:232-319).
 *   means3D[P,3] scales[P,3] rotations[P,4] opacities[P] dc[P,3] sh[P,M,3]: activated inputs
 *   (rasterize_points.h:25-50).  sh may be NULL when M == 0.
 *   radii[P] (int32) is written for every Gaussian (0 = culled).
 *   *num_rendered_host receives R (the call synchronises `stream` once, exactly where the
 *   reference does its blocking cudaMemcpy at rasterizer_impl.cu:398).
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_forward_preprocess(int P, int sh_degree, int M, const float* means3D, const float* scales,
                            float scale_modifier, const float* rotations, const float* opacities,
                            const float* dc, const float* sh, const glic_view* view, int no_color,
                            int* radii, void* geom_ws, size_t geom_bytes, void* image_ws,
                            size_t image_bytes, int64_t* num_rendered_host, void* stream);

/* Forward, stage 2: key emission, stable radix sort of (tile|depth) keys, tile ranges, bucket
 * offsets, per-tile front-to-back blend.  Replaces duplicateWithKeys, cub::DeviceRadixSort,
 * identifyTileRanges, perTileBucketCount, the second InclusiveSum + D2H read, FORWARD::render
 * and the D2D copy of the colour image (rasterizer_impl.cu:400-473; forward.cu:321-481).
 *   out_color[3,H,W], out_final_T[H,W]; no background term (forward.cu:466-467).
 *   *num_buckets_host receives B when non-NULL (costs one stream sync; pass NULL to stay
 *   asynchronous -- backward only needs the value stored inside image_ws).
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_forward_render(int P, const glic_view* view, int no_color, int64_t num_rendered,
                        void* geom_ws, void* image_ws, void* binning_ws, size_t binning_bytes,
                        void* sample_ws, size_t sample_bytes, float* out_color, float* out_final_T,
                        int64_t* num_buckets_host, void* stream);

/* ---------------------------------------------------------------------------------------
 * Forward in ONE asynchronous call (no host synchronisation inside): the same stages as
 * glic_forward_preprocess + glic_forward_render, but the binning / sample workspaces are sized by
 * the CALLER'S CAPACITY instead of the exact num_rendered, which therefore never has to travel
 * to the host mid-frame (the reference blocks twice per forward, rasterizer_impl.cu:398,442).
 *   capacity = glic_binning_capacity(binning_bytes, sample_bytes, W, H, no_color) pairs.
 *   counters_host[3] = {R, B, overflow} is written ASYNCHRONOUSLY (use pinned memory); it is valid
 *   once `stream` has been synchronised.  overflow != 0 means R exceeded the capacity: the
 *   images are invalid and the call must be repeated with workspaces for at least R pairs.
 *   For glic_backward pass num_rendered = that same capacity (the value the workspaces were
 *   carved with), not R.
 * ------------------------------------------------------------------------------------- */
GLIC_API int64_t glic_binning_capacity(size_t binning_bytes, size_t sample_bytes, int width, int height, int no_color);
GLIC_API int glic_forward(int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier,
                          const float* rotations, const float* opacities, const float* dc, const float* sh,
                          const glic_view* view, int no_color, int* radii, void* geom_ws, size_t geom_bytes,
                          void* image_ws, size_t image_bytes, void* binning_ws, size_t binning_bytes, void* sample_ws,
                          size_t sample_bytes, float* out_color, float* out_final_T, int64_t* counters_host,
                          void* stream);

/* ---------------------------------------------------------------------------------------
 * Render only (inference): the stages of glic_forward up to the blend, unchanged (same preprocess, depth sort, key emission,
 * tile sort and ranges, hence the same tile lists), then the inference form of the blend.  Per pixel it does the training
 * blend's work in the training blend's operation order, so out_color and out_final_T equal glic_forward's bit for bit; it
 * adds two planes and writes none of the state the backward needs (checkpoints, bucket ids, contributor counts, the saved
 * colour), so there is no sample workspace and no glic_backward after it.
 *   out_depth[H,W] (may be NULL): expected depth sum_i T_i alpha_i z_i over the splats a pixel takes, z the view-space depth;
 *     unnormalised like the colour (divide by 1 - out_final_T for the mean depth of what the pixel sees).
 *   out_median_depth[H,W] (may be NULL): z of the first taken splat after which T < 0.5; 0 where T never falls below 0.5.
 *   capacity = glic_binning_capacity(binning_bytes, 0, W, H, 1) pairs.  counters_host[3] = {R, 0, overflow} as glic_forward
 *   with no_color = 1 writes it (asynchronously; overflow != 0: the images are invalid, repeat with room for R pairs).
 *   No host synchronisation.  P = 0: out_final_T is 1 and every other output 0 (glic_forward writes T = 0 there).  Arguments are checked as glic_forward checks
 *   them (frame size, GLIC_MAX_TILES, workspaces, null pointers, the 16-byte alignment of rotations).  Profiled under
 *   GLIC_STAGE_PREPROCESS, _SORT, _EMIT, _RANGES and _RENDER_FWD.
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_render(int P, int sh_degree, int M, const float* means3D, const float* scales, float scale_modifier,
                         const float* rotations, const float* opacities, const float* dc, const float* sh, const glic_view* view,
                         int* radii, void* geom_ws, size_t geom_bytes, void* image_ws, size_t image_bytes,
                         void* binning_ws, size_t binning_bytes, float* out_color, float* out_final_T,
                         float* out_depth /* may be NULL */, float* out_median_depth /* may be NULL */,
                         int64_t* counters_host, void* stream);

/* ---------------------------------------------------------------------------------------
 * Contribution scores: how much each Gaussian adds to a view.  Definitions: for a view and a pixel, walk the pixel's tile list
 * front to back as the training blend does.  A splat is TAKEN when all of
 *   power <= 0;   alpha = min(0.99, o expf(power)) >= 1/255;   T (1 - alpha) >= 1e-4
 * hold (a splat that would push T below 1e-4 ends the pixel and is not taken).  These are the pairs the colour, the contributor
 * counts and the render backward see.  A taken pair's WEIGHT is w = __fmul_rn(T, alpha), T the pixel's transmittance just
 * before the splat.  Over a set of views, row i's scores are
 *   max_weight[i]: the largest w of any taken pair of row i, 0 if none;
 *   hits[i]:       the number of taken (view, pixel) pairs of row i;
 *   ends[i]:       the number of (view, pixel) pairs row i ENDS: the splat passes the first two tests but T (1 - alpha) < 1e-4.
 *                  It is not taken, yet it stops the pixel's blend, so without it the splats behind would be blended there.
 * All three are order-free (a float max and integer sums): bit-reproducible under any scheduling and independent of view order.
 * A row with hits = ends = 0 over a set of views changes none of their pixels: at every pixel it is skipped by tests that do not
 * depend on T, or reached only after the pixel has ended, so removing it leaves every pixel's sequence of blended splats as it was.
 * glic_contribution scores one view: the stages of glic_forward with no_color = 1 up to the blend, unchanged (the same tile
 * lists), then an alpha-only form of the blend that ACCUMULATES into the caller's max_weight[P] (max), hits[P] and ends[P] (sums) --
 * zero them once, then call once per view.  out_final_T (may be NULL) equals glic_forward's final_T bit for bit.  Nothing
 * else is written; there is no sample workspace and no host synchronisation.
 *   capacity = glic_binning_capacity(binning_bytes, 0, W, H, 1) pairs; counters_host[3] = {R, 0, overflow} as glic_render
 *   writes it.  A call that overflows adds nothing to any array, so repeating it with room for R pairs is exact.
 *   P = 0: nothing is scored, out_final_T is 0 (as glic_forward).  Arguments are checked as glic_render checks them; max_weight
 *   and hits must be non-NULL when P > 0; ends may be NULL (not counted).  Profiled under GLIC_STAGE_PREPROCESS, _SORT, _EMIT, _RANGES and _RENDER_FWD.
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_contribution(int P, const float* means3D, const float* scales, float scale_modifier, const float* rotations,
                               const float* opacities, const glic_view* view, int* radii, void* geom_ws, size_t geom_bytes,
                               void* image_ws, size_t image_bytes, void* binning_ws, size_t binning_bytes,
                               float* max_weight /*[P], accumulated*/, uint64_t* hits /*[P], accumulated*/,
                               uint64_t* ends /*[P], accumulated, may be NULL*/, float* out_final_T /* may be NULL */, int64_t* counters_host, void* stream);

/* Backward.  Replaces CudaRasterizer::Rasterizer::backward (rasterizer_impl.cu:476-580;
 * backward.cu:138-597) AND the ten torch::zeros of rasterize_points.cu:192-201: every output
 * element is written (exact zeros for culled Gaussians), nothing needs pre-zeroing.
 *   dL_dpix[3,H,W]; outputs shaped as RasterizeGaussiansBackwardCUDA's tensors
 *   (rasterize_points.h:52-82): dL_dmeans2D[P,3] (NDC-scaled, .z = 0), dL_dcolors[P,3],
 *   dL_dopacity[P], dL_dmeans3D[P,3], dL_dcov3D[P,6], dL_ddc[P,3], dL_dsh[P,M,3],
 *   dL_dscales[P,3], dL_drotations[P,4].  dL_dconic[P,4] (x,y,0,w) is scratch and may alias
 *   nothing else.  Gradients are w.r.t. the ACTIVATED inputs.
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_backward(int P, int sh_degree, int M, const float* means3D, const float* scales,
                  float scale_modifier, const float* rotations, const float* dc, const float* sh,
                  const glic_view* view, const int* radii, int64_t num_rendered, const void* geom_ws,
                  const void* binning_ws, const void* image_ws, const void* sample_ws,
                  const float* dL_dpix, float lambda_erank, float* dL_dmeans2D, float* dL_dconic,
                  float* dL_dopacity, float* dL_dcolors, float* dL_dmeans3D, float* dL_dcov3D,
                  float* dL_ddc, float* dL_dsh, float* dL_dscales, float* dL_drotations, void* stream);

/* Deterministic backward: glic_backward's arguments and outputs, plus a workspace of glic_deterministic_bytes(num_rendered,
 * width, height) bytes (num_rendered as glic_backward takes it).  Every output is a function of the saved forward state and
 * dL_dpix alone: calls on the same state give the same bits, whatever the grid size, scheduling or order of the GPU's work.
 * The render backward (the production body only) stores each (tile, Gaussian) pair's nine contributions -- bit for bit
 * the values glic_backward adds atomically -- and adds a Gaussian's contributions in ascending tile index:
 *   chunks of 32 consecutive contributions are each left-folded from their first element, then the chunk sums are
 *   left-folded in chunk order; for 32 or fewer contributions that is the strict left fold.
 * Rows with no contribution are zero.  Agreement with glic_backward: within the reassociation bound of the n contributions.
 * A short det_ws returns GLIC_ERR_WORKSPACE with nothing enqueued.  The workspace is 32 entries per checkpoint bucket (36 B of
 * values + 16 B of sort keys and indices each) plus the sort's temp; the exact and counting forms of the debug hook have no
 * deterministic form. */
GLIC_API size_t glic_deterministic_bytes(int64_t num_rendered, int width, int height);
GLIC_API int glic_backward_deterministic(int P, int sh_degree, int M, const float* means3D, const float* scales,
                  float scale_modifier, const float* rotations, const float* dc, const float* sh,
                  const glic_view* view, const int* radii, int64_t num_rendered, const void* geom_ws,
                  const void* binning_ws, const void* image_ws, const void* sample_ws,
                  const float* dL_dpix, float lambda_erank, float* dL_dmeans2D, float* dL_dconic,
                  float* dL_dopacity, float* dL_dcolors, float* dL_dmeans3D, float* dL_dcov3D,
                  float* dL_ddc, float* dL_dsh, float* dL_dscales, float* dL_drotations, void* det_ws, size_t det_bytes,
                  void* stream);

/* ---------------------------------------------------------------------------------------
 * Stable LSD radix sort of (uint64 key, uint32 value) pairs on key bits [0, end_bit).
 * Replaces cub::DeviceRadixSort::SortPairs<uint64,uint32>(begin_bit=0, end_bit)
 * (rasterizer_impl.cu:419-424).  Own onesweep implementation, no CUB.
 * Result lands in keys_out/vals_out; keys_in/vals_in are clobbered (used as ping-pong).
 * ------------------------------------------------------------------------------------- */
GLIC_API size_t glic_sort_temp_bytes(int64_t n);
GLIC_API int glic_sort_pairs_u64_u32(int64_t n, int end_bit, uint64_t* keys_in, uint32_t* vals_in,
                            uint64_t* keys_out, uint32_t* vals_out, void* temp, size_t temp_bytes,
                            void* stream);
/* Test hook: the 32-bit-key sort of the binning (depth keys, tile ids) on key bits [0, end_bit), ping-ponging between
 * (keys, vals) and (keys_alt, vals_alt).  n_dev (optional, device memory): the true count <= n; the kernels are launched
 * for n, as the forward launches its capacity-sized tile sort.  Returns 0/1 = which pair holds the result (1: the _alt
 * pair), < 0 on error. */
GLIC_API int glic_debug_sort_pairs_u32(int64_t n, int end_bit, uint32_t* keys, uint32_t* vals, uint32_t* keys_alt,
                                       uint32_t* vals_alt, const unsigned int* n_dev, void* temp, size_t temp_bytes,
                                       void* stream);

/* ---------------------------------------------------------------------------------------
 * Visibility-masked Adam.  Replaces ADAM::adamUpdate (rasterizer/cuda_rasterizer/adam.cu:9-67,
 * adam.h:12-23).  In place on param / exp_avg / exp_avg_sq; element j belongs to Gaussian j/M;
 * no bias correction.  `visible` is N bytes (bool).
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_adam_update(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                     const uint8_t* visible, float lr, float b1, float b2, float eps, uint32_t N,
                     uint32_t M, void* stream);

/* ---------------------------------------------------------------------------------------
 * Packed model step (SURVEY 8f rank 1; extension, no single reference symbol).  The model lives in one planar buffer
 *     rotation[4P] | xyz[3P] | log-scale[3P] | opacity logit[P] | dc[3P] | sh-rest[3MP]      (glic_packed_offsets)
 * which is also the layout of the packed gradient buffer (glic_p2p_allreduce_mean's payload).
 *  - glic_activations_forward replaces GaussianModel::getOpacity / getScaling / getRotation (gaussian.cpp:147-175:
 *    torch::sigmoid, torch::exp, normalize) with one kernel;
 *  - glic_activations_backward applies their chain rule IN PLACE to the gradients glic_backward wrote (what autograd's
 *    SigmoidBackward / ExpBackward / normalize backward do for the reference);
 *  - glic_adam_update_packed is SparseGaussianAdam::custom_step (optim_utils.h:102-137) for all six groups in ONE
 *    launch, element-wise identical to six glic_adam_update calls; lr6_host in buffer order
 *    {rotation, xyz, scaling, opacity, f_dc, f_rest}.
 * ------------------------------------------------------------------------------------- */
GLIC_API size_t glic_packed_floats(uint32_t P, uint32_t M);
GLIC_API int glic_packed_offsets(uint32_t P, uint32_t M, size_t* offsets6_host);
GLIC_API int glic_activations_forward(int P, const float* opacity_logit, const float* log_scale, const float* rot_raw,
                                      float* opacity, float* scale, float* rot, void* stream);
GLIC_API int glic_activations_backward(int P, const float* opacity, const float* scale, const float* rot_raw,
                                       float* dL_dopacity, float* dL_dscale, float* dL_drot, void* stream);
GLIC_API int glic_adam_update_packed(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                                     const uint8_t* visible, const float* lr6_host, float b1, float b2, float eps,
                                     uint32_t P, uint32_t M, void* stream);

/* ---------------------------------------------------------------------------------------
 * extend() on the GPU (SURVEY 8f rank 2; gaussian.cpp:499-638): which LiDAR points of the newest frame become Gaussians
 * and with which initial parameters.  One 64-bit atomicMin per in-image point on a (orderable depth | index) word per
 * pixel replaces the reference's host-side unordered_map<std::string, ...>; survivors (nearest point of their pixel,
 * depth_rsp > 0, rendered alpha < 0.99) are compacted in ascending index order and initialised.  Pinned against the CPU
 * oracle's restatement (tests/test_gpu_extend.py).  Device pointers except R_cw_host[9] (row-major), t_cw_host[3] and
 * count_host.  final_T comes from a no_color forward of the newest view.  glic_mapper_extend wires it to the model.
 * ------------------------------------------------------------------------------------- */
GLIC_API size_t glic_extend_bytes(int n, int width, int height);
GLIC_API int glic_extend(int n, const float* points, const float* colors, const float* depth_rsp, const float* R_cw_host,
                         const float* t_cw_host, float fx, float fy, float cx, float cy, int width, int height,
                         const float* final_T, float scaling_scale, void* ws, size_t ws_bytes, int* keep_idx, float* xyz,
                         float* f_dc, float* log_scale, float* rot, float* opacity_logit, int* count_host, void* stream);

/* ---------------------------------------------------------------------------------------
 * initialize() on the GPU (gaussian.cpp:212-304): the first map's rows, written where the caller points (device pointers;
 * rot 16-byte aligned).  Neither call touches f_rest or Adam moments (the reference's are zero).  Both are asynchronous on
 * `stream`.  glic_mapper_initialize_lidar wires them to the model: sky rows [0, S), then the LiDAR rows in input order.
 *   glic_lidar_init: xyz = points; f_dc = (float)((colors - 0.5) / C0) in double (colors: the Dataset's rgb / 255.0
 *   doubles); log_scale = (float)log(scaling_scale * depth_rsp / focal) in double on all three axes, focal = (fx + fy) / 2
 *   from the configuration's doubles; rot = (1, 0, 0, 0); opacity_logit = log(0.1 / 0.9) in float.
 *   glic_skybox_init: n points on the cap z > -0.4 of the sphere of radius 10 * radius, positions in torch's float order
 *   from two uniforms per row drawn by a counter-based generator keyed by (seed, row) -- the SplitMix64 output seed +
 *   (row + 1) * 0x9E3779B97F4A7C15 through the SplitMix64 finaliser; u1 = its top 24 bits * 2^-24, u2 = bits 16..39 *
 *   2^-24 --; f_dc = (0.7, 0.8, 0.95) raw; log_scale = logf(sqrtf(fmaxf(d2, 1e-7f))) with d2 = glic_knn_mean_dist2 over
 *   the n sky points alone; rot = (1, 0, 0, 0); opacity_logit = log(0.7 / 0.3) in float.  uv (optional, device, [n][2])
 *   receives the uniforms.  ws: glic_skybox_init_bytes(n) bytes of device memory.
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_lidar_init(int n, const float* points, const double* colors, const float* depth_rsp, double scaling_scale,
                             double focal, float* xyz, float* f_dc, float* log_scale, float* rot, float* opacity_logit,
                             void* stream);
GLIC_API size_t glic_skybox_init_bytes(int n);
GLIC_API int glic_skybox_init(int n, int radius, uint64_t seed, void* ws, size_t ws_bytes, float* xyz, float* f_dc,
                              float* log_scale, float* rot, float* opacity_logit, float* uv, void* stream);

/* 8-bit camera frame -> the float image the loss sees (Dataset::addFrame, gaussian.cpp:44-49: cv_bridge BGR8,
 * cvtColor(BGR2RGB), convertTo(CV_32FC3, 1.0f / 255.0f)).  bgr: packed [H][W][3] bytes (B, G, R); rgb: [3][H][W] floats,
 *     rgb[c][y][x] = __fmul_rn((float)bgr[y][x][2 - c], 1.0f / 255.0f)
 * one rounding of x * fl32(1/255), which is what OpenCV's 8U -> 32F convertTo computes; it is not (float)(x / 255.0), which
 * differs for 126 of the 256 byte values.  No host synchronisation. */
GLIC_API int glic_decode_bgr8(int H, int W, const uint8_t* bgr, float* rgb, void* stream);

/* ---------------------------------------------------------------------------------------
 * On-disk map (SURVEY 8f rank 4).  Replaces GaussianModel::saveMap (gaussian.cpp:305-397, through tinyply.h:588-703):
 * binary little-endian PLY, element vertex, float properties x y z | f_dc_0..2 | f_rest_0..3M-1 | opacity | scale_0..2 |
 * rot_0..3; RAW parameters; f_rest channel-major.  The file is byte-identical to the reference's for the same tensors
 * (pinned against the reference's own tinyply in tests/test_map_io.py).  All pointers are HOST pointers; f_dc is
 * [P,1,3], f_rest [P,M,3] in the in-memory (coefficient-major) layout.  glic_ply_read* accept exactly this layout
 * (comments allowed) and fail loudly on anything else.
 * ------------------------------------------------------------------------------------- */
GLIC_API size_t glic_ply_bytes(uint32_t P, uint32_t M);
GLIC_API int glic_ply_write(const char* path, uint32_t P, uint32_t M, const float* xyz, const float* f_dc, const float* f_rest,
                            const float* opacity, const float* scale, const float* rotation);
GLIC_API int glic_ply_write_packed(const char* path, uint32_t P, uint32_t M, const float* params_host);
GLIC_API int glic_ply_read_header(const char* path, uint32_t* P, uint32_t* M, size_t* data_offset);
GLIC_API int glic_ply_read(const char* path, uint32_t P, uint32_t M, float* xyz, float* f_dc, float* f_rest, float* opacity,
                           float* scale, float* rotation);

/* ---------------------------------------------------------------------------------------
 * Fused SSIM.  Replaces fusedssimCUDA / fusedssim_backwardCUDA (fused-ssim/ssim.cu:186-365).
 * img*: [B,CH,H,W] contiguous.  Partial-derivative maps may be NULL in forward (train = false).
 * At most 65535 planes (B*CH) per call; more is GLIC_ERR_INVALID_ARGUMENT with nothing enqueued.
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_fused_ssim(int B, int CH, int H, int W, float C1, float C2, const float* img1, const float* img2,
                    float* ssim_map, float* dm_dmu1, float* dm_dsigma1_sq, float* dm_dsigma12, void* stream);
GLIC_API int glic_fused_ssim_backward(int B, int CH, int H, int W, float C1, float C2, const float* img1,
                             const float* img2, const float* dL_dmap, const float* dm_dmu1,
                             const float* dm_dsigma1_sq, const float* dm_dsigma12, float* dL_dimg1,
                             void* stream);

/* Whole photometric loss of one mapping iteration in two launches (gaussian.cpp:685-691,
 * loss_utils.h:30-33,189-193): L = (1-lambda)*mean|img-gt| + lambda*(1-mean(SSIM)), and
 * dL/dimg.  loss_out: 1 device float (accumulated; zeroed by the call).  scratch: 3*CH*H*W floats.  CH <= 65535.
 * dL/dimg is bit-reproducible; the loss is not (one float atomicAdd per 32x32 tile, in the order the tiles finish). */
GLIC_API size_t glic_loss_scratch_bytes(int CH, int H, int W);
GLIC_API int glic_l1_ssim_loss(int CH, int H, int W, float lambda_dssim, const float* img, const float* gt,
                      float* loss_out, float* dL_dimg, void* scratch, size_t scratch_bytes, void* stream);

/* The same loss on an exposed image (Inria 3DGS's trained exposure; no counterpart in the reference, whose render()
 * ignores use_trained_exposure).  E_dev: 12 device floats, a 3x4 row-major matrix; the loss and its gradients are those
 * of out[3,H,W],
 *     out_c = E[0][c]*r + E[1][c]*g + E[2][c]*b + E[c][3]          (matmul(img_hwc, E[:3,:3]) + E[:3,3])
 * evaluated as acc = E[c][3], then fmaf with r, g, b in that order: E = [I | 0] gives out == img exactly for the
 * non-negative finite images the renderer produces.  out is formed inside the loss kernels and never written.
 *   dL_dimg[3,H,W] = sum_c E[k][c] * dL/dout_c;  dL_dE_dev[12]: dL/dE[k][c] = sum_px img_k * dL/dout_c (k < 3) and
 *   dL/dE[c][3] = sum_px dL/dout_c, summed in float64 in a fixed order (per-CTA partials, then one fixed-order total, no
 *   atomics): two identical calls give identical bits.  dL_dimg and dL_dE_dev are both NULL (loss only) or both set.
 *   img: 3 channels; scratch: glic_loss_exposure_scratch_bytes(H, W).  Profiled as GLIC_STAGE_LOSS_FWD / GLIC_STAGE_LOSS_BWD
 *   (the dL/dE kernels are part of the latter); the mapper's exposure step is timed under GLIC_STAGE_ADAM. */
GLIC_API size_t glic_loss_exposure_scratch_bytes(int H, int W);
GLIC_API int glic_l1_ssim_loss_exposure(int H, int W, float lambda_dssim, const float* img, const float* gt, const float* E_dev,
                                        float* loss_out, float* dL_dimg, float* dL_dE_dev, void* scratch, size_t scratch_bytes,
                                        void* stream);

/* Valid-pixel masks.  A mask marks the pixels of a frame that the loss and the evaluation use (1) and leave out (0): moving
 * objects, the rig's own platform.  On the device it is bit-packed: row y is glic_mask_words_per_row(W) uint32 words, pixel
 * (y, x) is bit x & 31 of word y * words_per_row + (x >> 5); the pad bits of a row's last word are 0.  A view of a mask is
 * (words, words_per_row, x0): the viewed H x W region's pixel (y, x) is the mask's pixel (y, x0 + x), so a column crop reads
 * its frame's mask in place.
 *   glic_pack_mask: valid_dev [H][W] bytes (nonzero = used) into words_dev (H * words_per_row words) and count_dev (1 device
 *   uint32, the number of used pixels, an exact integer sum), on `stream`.
 *
 * The masked loss, with a the image (exposed by E_dev when given), b = gt and w the mask:
 *     a' = w ? a : 0,  b' = w ? b : 0   (a select: NaN or Inf under the mask never enters; the masked pixels act exactly
 *                                         like the SSIM's zero padding at the frame border)
 *     L  = (1-lambda) * sum_used |a'-b'| / Nw + lambda * (1 - sum_used SSIM(a', b') / Nw),   Nw = 3 * valid_count
 *     dL/da = w ? dL/da' : +0
 * An all-ones mask gives glic_l1_ssim_loss / glic_l1_ssim_loss_exposure bit for bit (loss value, dL/dimg and dL/dE).
 *   glic_l1_ssim_loss_masked: 3 channels; E_dev NULL or the 12 floats of glic_l1_ssim_loss_exposure (then dL_dimg and dL_dE_dev
 *   are both NULL or both set, as there); valid_count = the view's used pixels (> 0, or GLIC_ERR_INVALID_ARGUMENT before any
 *   launch); fixed_order = 1: the loss value summed in a fixed order (bit-reproducible, as the mapper's deterministic option);
 *   mask_words = NULL: the unmasked loss (the same kernels as glic_l1_ssim_loss / _exposure).  scratch:
 *   glic_loss_masked_scratch_bytes(H, W).
 *   glic_eval_psnr_ssim_masked: glic_eval_psnr_ssim's scores (with E_dev, of the exposed image, CH = 3) where both clamped
 *   images are 0 under the mask and MSE and the SSIM mean are taken over the CH * valid_count used elements (the SSIM map
 *   itself is that of the masked pair).  fixed_order = 1: both sums in a fixed order.  scratch:
 *   glic_eval_masked_scratch_bytes(CH, H, W). */
GLIC_API int glic_mask_words_per_row(int W);
GLIC_API int glic_pack_mask(int H, int W, const uint8_t* valid_dev, uint32_t* words_dev, uint32_t* count_dev, void* stream);
GLIC_API size_t glic_loss_masked_scratch_bytes(int H, int W);
GLIC_API int glic_l1_ssim_loss_masked(int H, int W, float lambda_dssim, const float* img, const float* gt, const float* E_dev,
                                      const uint32_t* mask_words, int words_per_row, int mask_x0, uint32_t valid_count,
                                      int fixed_order, float* loss_out, float* dL_dimg, float* dL_dE_dev, void* scratch,
                                      size_t scratch_bytes, void* stream);
GLIC_API size_t glic_eval_masked_scratch_bytes(int CH, int H, int W);
GLIC_API int glic_eval_psnr_ssim_masked(int CH, int H, int W, const float* img, const float* gt, const float* E_dev,
                                        const uint32_t* mask_words, int words_per_row, int mask_x0, uint32_t valid_count,
                                        int fixed_order, float* out2, void* scratch, size_t scratch_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * simple-knn.  Replaces SimpleKNN::knn (simple-knn/simple_knn.cu:185-221): mean of the three
 * smallest squared distances to other points.  points[P,3] -> mean_dists[P].
 * ------------------------------------------------------------------------------------- */
GLIC_API size_t glic_knn_temp_bytes(int P);
GLIC_API int glic_knn_mean_dist2(int P, const float* points, float* mean_dists, void* temp, size_t temp_bytes,
                        void* stream);

/* ---------------------------------------------------------------------------------------
 * Introspection for parity tests (copies internal state to caller DEVICE buffers; any pointer
 * may be NULL).  Shapes: depth[P] xy[P,2] conic_opacity[P,4] rgb[P,3] tiles_touched[P]
 * offsets[P] (end of each Gaussian's slot range in the depth-ordered key list) clamped[P,3] (u8) |
 * point_list[R] keys_sorted[R] ((tile<<32)|depth bits, rebuilt) | ranges[T,2] bucket_offsets[T]
 * n_contrib[H*W] max_contrib[T].
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_debug_geom(int P, const void* geom_ws, float* depth, float* xy, float* conic_opacity, float* rgb,
                    uint32_t* tiles_touched, uint32_t* offsets, uint8_t* clamped, void* stream);
/* num_rendered = the value the binning workspace was carved with (exact R, or the capacity after glic_forward);
 * count = how many sorted entries to copy out (the true R). */
GLIC_API int glic_debug_binning(int P, const void* geom_ws, int64_t num_rendered, int64_t count, const void* binning_ws,
                                uint32_t* point_list, uint64_t* keys_sorted, void* stream);
GLIC_API int glic_debug_image(int width, int height, const void* image_ws, uint32_t* ranges, uint32_t* bucket_offsets,
                     uint32_t* n_contrib, uint32_t* max_contrib, int64_t* counters2_host /* {R,B}, HOST pointer */, void* stream);
/* Fill level of the row-span arena of the last forward: count_cap_host[2] = {rows requested, capacity} (HOST pointer;
 * synchronises `stream`).  Rects of more than 32 tiles store one span per row while the arena has room; when requested >
 * capacity, the later rects had their rows recomputed by the key emission instead. */
GLIC_API int glic_debug_spans(int P, const void* geom_ws, uint32_t* count_cap_host, void* stream);
/* The render backward alone on the saved state of the last glic_forward (R = its binning capacity), ACCUMULATING into the
 * four 2-D gradient buffers (the caller zeroes them).  exact != 0: the former kernel body (expf for every pixel) instead
 * of the production one.  counters (optional, DEVICE, 8 x uint64, zeroed by the caller): the
 * counting form of the same kernel adds {live buckets, splats walked, splats with a taker, (splat, two row pairs) visits,
 * visits with a taker, candidate pixels, pixel-splat pairs taken, pixels decided by the exact expf fallback}. */
GLIC_API int glic_debug_render_backward(int P, const glic_view* view, int64_t R, const void* geom_ws, const void* binning_ws,
                                        const void* image_ws, const void* sample_ws, const float* dL_dpix, float* dL_dmeans2D,
                                        float* dL_dconic, float* dL_dopacity, float* dL_dcolors, int exact,
                                        unsigned long long* counters, void* stream);
/* The deterministic render backward alone on the saved state of the last glic_forward (R = its binning capacity): WRITES the
 * four 2-D gradient buffers as glic_backward_deterministic does (zeroing them first), then copies out the ordered entry list:
 * *count_host (HOST) = n entries, and for entry i < n gid[i], tile[i] (u32) and values[9 i .. 9 i + 8] (mean.x, mean.y,
 * conic.x, conic.y, conic.w, colour r, g, b, opacity) in the order the reduction adds them: by gid, then ascending tile.
 * gid, tile and values (DEVICE) hold 32 * glic_max_buckets(R, W, H) entries.  Synchronises `stream`. */
GLIC_API int glic_debug_deterministic_entries(int P, const glic_view* view, int64_t R, const void* geom_ws, const void* binning_ws,
                                              const void* image_ws, const void* sample_ws, const float* dL_dpix, void* det_ws,
                                              size_t det_bytes, float* dL_dmeans2D, float* dL_dconic, float* dL_dopacity,
                                              float* dL_dcolors, int64_t* count_host, uint32_t* gid, uint32_t* tile, float* values,
                                              void* stream);
/* The mapper's per-Gaussian backward alone, on the saved state of the last glic_forward and given render-backward outputs
 * (device arrays; rotations activated, rot_raw the raw ones, opacity activated).  pose_only = 0: the COMPACT + POSE form of an
 * iteration under pose refinement, writing the 11 geometric floats of every row to g_geo [11 P] (rotation [P,4] | xyz [P,3] |
 * log-scale [P,3] | opacity logit [P]); pose_only = 1: the POSE_ONLY form of glic_mapper_align, which writes no row (g_geo,
 * rot_raw, opacity and dL_dopacity may be NULL).  Both write dL/d(rho, omega) of the view to pose6 (device, 6 floats) through
 * partials (device, 48 * ceil(P / 128) bytes).  Asynchronous on `stream`. */
GLIC_API int glic_debug_pose_backward(int P, int sh_degree, int M, const float* means3D, const float* scales, const float* rotations,
                                      const float* rot_raw, const float* opacity, const float* sh, const glic_view* view,
                                      const int* radii, const void* geom_ws, const float* dL_dmeans2D, const float* dL_dconic,
                                      const float* dL_dopacity, const float* dL_dcolors, int pose_only, float* g_geo,
                                      void* partials, float* pose6, void* stream);
/* Allocation failures of the native mapper, simulated on the host (no CUDA call is made for the failing one): the n-th device
 * or pinned allocation a mapper makes from now on returns cudaErrorMemoryAllocation; n = 0 disarms it, n < 0 is refused.
 * glic_debug_mapper_allocations is the number of allocations the mappers of this process hold right now. */
GLIC_API int glic_debug_fail_allocation(int n);
GLIC_API int64_t glic_debug_mapper_allocations(void);

/* ---------------------------------------------------------------------------------------
 * Multi-GPU exchange step (no counterpart in the reference, which is single-GPU): in-place MEAN all-reduce of the
 * packed per-Gaussian gradients + OR of the visibility bytes, done by our own kernels over NVLink peer memory
 * (CUDA IPC mappings of every rank's buffer; two-shot: rank r reduces slice r from all peers and writes it back
 * to all peers).  Buffer layout: n_floats fp32 | n_vis_bytes bytes | flag words, each part padded to 256 B
 * (glic_p2p_buffer_bytes).  Every rank must make the same sequence of calls (the barrier epoch is kept on the device,
 * so the call is CUDA-graph capturable).
 * glic_p2p_alloc is the one place this library allocates device memory: IPC needs a dedicated cudaMalloc block.
 * ------------------------------------------------------------------------------------- */
GLIC_API size_t glic_p2p_buffer_bytes(size_t n_floats, size_t n_vis_bytes);
GLIC_API int glic_p2p_slice(int rank, int world, size_t n_floats, size_t n_vis_bytes, size_t* out6_host);
GLIC_API int glic_p2p_alloc(size_t bytes, void** dev_ptr_host, unsigned char* handle64_host);
GLIC_API int glic_p2p_open(const unsigned char* handle64_host, void** peer_ptr_host);
GLIC_API int glic_p2p_close(void* peer_ptr);
GLIC_API int glic_p2p_free(void* dev_ptr);
GLIC_API int glic_p2p_allreduce_mean(int rank, int world, void* const* bufs_host, size_t n_floats, size_t n_vis_bytes,
                                     void* stream);
/* The device-side barriers wait at most GLIC_P2P_TIMEOUT_MS (environment, default 20000) for a peer; a timeout sets a
 * sticky error word in the rank's own block instead of hanging or trapping.  glic_p2p_check synchronises `stream` and
 * returns GLIC_ERR_TIMEOUT if one was recorded since the last check (and clears it). */
GLIC_API int glic_p2p_check(void* own_buf, size_t n_floats, size_t n_vis_bytes, void* stream);

/* Fused exchange + optimiser on the FULL packed gradient form: reduce-scatter of the gradients, visibility-masked Adam on
 * the local slice, all-gather of the updated PARAMETERS, in one kernel over peer memory (same NVLink bytes as the all-reduce,
 * Adam traffic and moment buffers / world).  Buffer = glic_p2p_model_bytes: gradients | visibility | flags | parameters
 * (packed layout).  Bit-identical to all-reduce + glic_adam_update_packed (tests/test_gpu_p2p_adam.py).  The mapper uses the
 * compact exchange instead (colour-gradient push + 11-float reduce, see "Native mapping host"). */
GLIC_API size_t glic_p2p_model_bytes(size_t n_floats, size_t n_vis_bytes);
GLIC_API int glic_p2p_reduce_adam(int rank, int world, void* const* bufs_host, uint32_t P, uint32_t M, float* exp_avg,
                                  float* exp_avg_sq, const float* lr6_host, float b1, float b2, float eps, void* stream);

/* ---------------------------------------------------------------------------------------
 * Evaluation metrics (SURVEY 8f rank 4; evaluateVisualQuality, gaussian.cpp:721-830 with loss_utils.h:35-39,
 * 84-127): both images are clamped to [0,1]; PSNR = 10 log10(1 / mean((a-b)^2)); SSIM = mean of the 11x11 /
 * sigma 1.5 zero-padded SSIM map (the conv2d formulation, same window as the fused kernel).  out2[0] = PSNR,
 * out2[1] = SSIM (device floats).  scratch: glic_eval_scratch_bytes.  LPIPS: glic_lpips below.
 * ------------------------------------------------------------------------------------- */
GLIC_API size_t glic_eval_scratch_bytes(int CH, int H, int W);
GLIC_API int glic_eval_psnr_ssim(int CH, int H, int W, const float* img, const float* gt, float* out2, void* scratch,
                                 size_t scratch_bytes, void* stream);

/* LPIPS with the AlexNet trunk, exactly the TorchScript module evaluateVisualQuality loads (src/lpips/lpips_alex.pt,
 * gaussian.cpp:741-800; lpipsPyTorch/modules/{lpips,networks,utils}.py): both [3,H,W] images are clamped to [0,1] (not
 * rescaled to [-1,1]), normalised with the file's mean / std, run through conv0/3/6/8/10 (+ReLU; 3/2 max pool after the first
 * two), and each of the five taps contributes mean_px sum_c lin_c (x_c/(|x|+1e-10) - y_c/(|y|+1e-10))^2.
 *   Weights: a flat little-endian file, 16-byte header (uint32 magic "LPIP", version 1, float count, 0) followed by
 *   glic_lpips_weight_floats() floats: mean[3] std[3] | conv0 OIHW weight, bias | conv3 .. | conv6 .. | conv8 .. | conv10 .. |
 *   lin0[64] lin1[192] lin2[384] lin3[256] lin4[256].  gaussian_lic_b200.lpips_weights converts the .pt file.
 *   glic_lpips_read_weights (host) fills `host` with the payload and fails on a wrong magic, version, count or file size.
 *   glic_lpips: device pointers; `weights` holds the payload; out1: 1 device float.  Frames from 31x31 (the smallest the network
 *   accepts) to 8192x8192; anything else is refused with GLIC_ERR_INVALID_ARGUMENT before any launch, and
 *   glic_lpips_scratch_bytes returns 0 for it.  No host synchronisation; per-CTA float64 partials added in a fixed order, so two
 *   identical calls give identical bits and identical images give exactly 0. */
GLIC_API size_t glic_lpips_weight_floats(void);
GLIC_API int glic_lpips_read_weights(const char* path, float* host);
GLIC_API size_t glic_lpips_scratch_bytes(int H, int W);
GLIC_API int glic_lpips(int H, int W, const float* img, const float* gt, const float* weights, float* out1, void* scratch,
                        size_t scratch_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Capacity-laid-out model arena (SURVEY 8f rank 1; replaces the torch::cat re-allocation of all parameters and Adam
 * state in GaussianModel::densificationPostfix, gaussian.cpp:426-497).  Same planar group order as the packed model,
 * but the group offsets come from the CAPACITY:  rotation[4*Pcap] | xyz[3*Pcap] | log-scale[3*Pcap] | opacity[Pcap] |
 * dc[3*Pcap] | sh-rest[3M*Pcap]  (glic_packed_offsets(Pcap, M)); rows [0, P) of every group are live.  Appending n rows
 * writes rows [P, P+n) in place (Adam moments of the new rows = 0, sh-rest = 0, like the zeros_like extension tensors);
 * growing copies the six live prefixes into an arena of a larger capacity.  Pcap must be a multiple of 4.
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_arena_append(float* params, float* exp_avg, float* exp_avg_sq, uint32_t P, uint32_t Pcap, uint32_t M,
                               uint32_t n_new, const float* xyz, const float* f_dc, const float* log_scale, const float* rot,
                               const float* opacity_logit, void* stream);
GLIC_API int glic_arena_regrow(const float* src, uint32_t Pcap_src, float* dst, uint32_t Pcap_dst, uint32_t M, uint32_t P,
                               void* stream);

/* ---------------------------------------------------------------------------------------
 * Native mapping host (SURVEY 8f ranks 1-4): the C++ counterpart of GaussianModel + extend() + optimize() +
 * evaluateVisualQuality() + saveMap() (gaussian.cpp:113-830) on top of the kernels above -- one object per GPU, no
 * torch, no Python.  The mapper OWNS its device memory (arena, Adam state, workspaces; float keyframe images stay pinned on
 * the host like Camera::original_image_, gaussian.cpp:80, frames of glic_mapper_add_frame are kept as 8 bits on the device):
 * it is the host of the loop, not an operator.
 *
 *   create -> initialize(raw parameters) | initialize_lidar(first scan) -> { add_keyframe -> [extend] -> optimize }*
 *          -> evaluate / save_map
 *
 * One iteration (gaussian.cpp:674-716) = for each of this rank's views: H2D of the pinned image (copy stream,
 * double-buffered), fused activations, forward (capacity-sized binning, no host sync), fused L1/D-SSIM loss, backward
 * with the activation chain rule fused in; then ONE masked Adam launch.  Gradients never exist as [P,59]: the
 * backward leaves 11 geometric floats (rotation, xyz, log-scale, opacity logit; summed over the rank's views) plus the
 * clamp-masked dL/dcolour (3 floats) of every view, and the Adam kernel rebuilds dL/d(dc, sh-rest) -- linear in
 * dL/dcolour with a per-view SH basis -- on the fly.  With world > 1 (view-sharded data parallelism, SURVEY 8e) the
 * exchange step moves exactly that compact form over NVLink peer memory: colour gradients are pushed to every peer while
 * the per-Gaussian backward still runs, the 11 geometric floats are mean-reduced by the two-shot kernel; every replica
 * then applies the identical Adam step (replicas stay bit-identical).  Semantics: mean of the per-view losses over all
 * world * views_per_rank views, one optimiser step per batch.
 * All host pointers unless stated.  Status codes as everywhere; the mapper never throws.
 * Failure contract: a mapper call that cannot allocate returns GLIC_ERR_CUDA and leaves everything the getters return unchanged,
 * except that capacities (stats.capacity, the workspaces) may have grown; the host may free memory (glic_mapper_prune) and call
 * again.  glic_mapper_optimize is the one exception: a binning regrow that fails between its batches returns the error with the
 * old workspace intact, and the batches already enqueued stand, as they do for any error in the middle of the list.
 * ------------------------------------------------------------------------------------- */
typedef struct glic_mapper glic_mapper;

typedef struct glic_mapper_config {
    int width, height;
    float fx, fy, cx, cy;          /* pinhole intrinsics of every keyframe (mapping.h:53-118 Params) */
    int sh_degree;                 /* 0..3; M = (sh_degree+1)^2 - 1 */
    float position_lr, feature_lr, opacity_lr, scaling_lr, rotation_lr;  /* config/fastlivo.yaml:18-22; sh-rest: feature_lr/20 */
    float lambda_dssim;            /* 0.2 */
    float scaling_scale;           /* extend(): log(scaling_scale * depth / focal), gaussian.cpp:623 */
    uint32_t capacity;             /* initial arena capacity in Gaussians (doubles when an append does not fit; fixed when world > 1) */
    int max_iters;                 /* optimize(): 100 (gaussian.cpp:645) */
    uint64_t seed;                 /* view sampler (the reference seeds from std::random_device) */
    int rank, world;               /* world > 1: call glic_mapper_export / glic_mapper_connect before the first iteration */
    int views_per_rank;            /* views each rank renders per iteration (gradient accumulation); >= 1 */
} glic_mapper_config;

typedef struct glic_keyframe {     /* Camera (camera.h:38-110): pose of the camera in the world + its image */
    float R_wc[9];                 /* row-major */
    float t_wc[3];
    const float* image;            /* [3,H,W] in [0,1], host memory that stays valid (pinned => asynchronous H2D) */
} glic_keyframe;

typedef struct glic_mapper_stats {
    uint32_t num_gaussians, capacity;
    uint64_t iterations;           /* optimiser steps so far */
    uint32_t last_inserted;        /* Gaussians appended by the last extend() */
    float last_loss;               /* loss of the last finished iteration's last local view */
    double mean_visible;           /* optimize()'s return value: mean #visible Gaussians per iteration (gaussian.cpp:719) */
    uint32_t overflow_regrows;     /* times the binning capacity had to grow (the frame is redone) */
    float ms_extend, ms_optimize;  /* device time of the last extend() / optimize() */
} glic_mapper_stats;

GLIC_API int glic_mapper_create(const glic_mapper_config* cfg, glic_mapper** out);
GLIC_API int glic_mapper_destroy(glic_mapper* m);
/* raw parameters (host): xyz[P,3] f_dc[P,3] f_rest[P,M,3] (may be NULL: zeros) opacity_logit[P] log_scale[P,3] rot[P,4] */
GLIC_API int glic_mapper_initialize(glic_mapper* m, uint32_t P, const float* xyz, const float* f_dc, const float* f_rest,
                                    const float* opacity_logit, const float* log_scale, const float* rot);
/* initialize() (gaussian.cpp:212-304) from the first scan, on the GPU (glic_skybox_init, glic_lidar_init): replaces the model
 * like glic_mapper_initialize, with sky_points sky rows [0, S) followed by the n LiDAR rows in input order; P = S + n, all
 * Adam moments zero.  points[n,3] colors[n,3] (doubles, rgb / 255.0) depth_rsp[n] are host arrays; focal = (fx + fy) / 2 of
 * the configuration in double; the sky is keyed by cfg.seed (the view sampler's state is left alone).  n < 1,
 * sky_points < 0, sky_radius <= 0 with sky_points > 0 or a NULL pointer return GLIC_ERR_INVALID_ARGUMENT and change
 * nothing.  Synchronises.  save_map writes rows [S, P) only (saveMap, gaussian.cpp:310-316); every other call sees every
 * row.  glic_mapper_sky_rows returns S (0 after glic_mapper_initialize). */
GLIC_API int glic_mapper_initialize_lidar(glic_mapper* m, int n, const float* points, const double* colors, const float* depth_rsp,
                                          double focal, int sky_points, int sky_radius);
GLIC_API int glic_mapper_sky_rows(glic_mapper* m, uint32_t* out);
GLIC_API int glic_mapper_add_keyframe(glic_mapper* m, const glic_keyframe* kf, int is_train);
/* extend() (gaussian.cpp:499-638) on the newest training keyframe: alpha-only render, z-buffer de-duplication of the n
 * LiDAR points, filter, initialisation, in-place append.  points[n,3] colors[n,3] depth_rsp[n] are host arrays. */
GLIC_API int glic_mapper_extend(glic_mapper* m, int n, const float* points, const float* colors, const float* depth_rsp);
/* optimize() (gaussian.cpp:640-719): view sampler (all keyframes when <= max_iters, else a random subset; shuffled),
 * then one iteration per sampled view batch.  views_host (optional, n_views entries) overrides the sampler. */
GLIC_API int glic_mapper_optimize(glic_mapper* m, const int* views_host, int n_views);
/* the sampler alone (tests): writes up to max_iters keyframe indices, returns their number in *count */
GLIC_API int glic_mapper_sample_views(glic_mapper* m, int* views_host, int* count);
/* PSNR / SSIM of one keyframe (train = 1: training list, 0: held-out list); synchronises */
GLIC_API int glic_mapper_evaluate(glic_mapper* m, int is_train, int index, float* psnr, float* ssim);
/* evaluateVisualQuality's three metrics.  load_lpips reads a glic_lpips weight file and uploads it (the mapper owns the copy;
 * a second call replaces it).  evaluate_lpips renders the keyframe once and returns the PSNR and SSIM glic_mapper_evaluate
 * returns, bit for bit, plus the LPIPS of the same clamped image against the keyframe's image; without weights loaded, or on
 * a frame under 31x31, it returns GLIC_ERR_INVALID_ARGUMENT.  render writes that scored image to rgb_host[3,H,W] (host): the
 * keyframe drawn at its current pose, a training keyframe's exposure E applied, clamped to [0,1].  All three synchronise. */
GLIC_API int glic_mapper_load_lpips(glic_mapper* m, const char* path);
GLIC_API int glic_mapper_evaluate_lpips(glic_mapper* m, int is_train, int index, float* psnr, float* ssim, float* lpips);
GLIC_API int glic_mapper_render(glic_mapper* m, int is_train, int index, float* rgb_host);
GLIC_API int glic_mapper_save_map(glic_mapper* m, const char* path);
GLIC_API int glic_mapper_stats_get(glic_mapper* m, glic_mapper_stats* out);
/* live rows of the arena copied to host arrays shaped like glic_mapper_initialize's (any pointer may be NULL); synchronises */
GLIC_API int glic_mapper_download(glic_mapper* m, float* xyz, float* f_dc, float* f_rest, float* opacity_logit,
                                  float* log_scale, float* rot, float* exp_avg_packed, float* exp_avg_sq_packed);
/* Removes every row whose activated opacity is below min_opacity; *removed (may be NULL) gets the count.
 *   A row goes iff act(logit) < min_opacity, act the activation kernel's own float expression 1 / (1 + expf(-logit)) (a NaN
 *   logit stays).  At GLIC_MAPPER_DEAD_OPACITY that is the preprocess's o < 1/255 cull bit for bit: such a row is culled in
 *   every view, so it is never visible, the masked Adam never steps it and it can never render or train again.
 *   The compaction is stable: survivors keep their relative order, and their six parameter groups and both Adam moments move
 *   with them bit for bit.  Sky rows stay in front; glic_mapper_sky_rows becomes the number of surviving sky rows, so save_map
 *   still writes exactly the non-sky survivors.  P and stats.num_gaussians drop, the capacity is unchanged, and the vacated rows
 *   [P_new, P_old) of the parameter and moment arenas are zeroed.  Keyframes, exposure and pose state are untouched.
 *   dry_run != 0 only counts.  A NULL mapper, a non-finite min_opacity or one outside [0, 1], and a prune that would remove
 *   every row (dry run or not) return GLIC_ERR_INVALID_ARGUMENT and change nothing; a mapper with no rows returns GLIC_OK with
 *   0 removed.  The call drains the iteration pipeline first (as download / save_map, including the lagged overflow ring) and
 *   synchronises.  It needs one spare arena of the capacity (glic_packed_floats(capacity, M) floats) while it runs.
 *   world > 1: every rank must make the same call between the same optimize() calls; replicas are bit-identical, so they remove
 *   the same rows and stay identical without any exchange. */
#define GLIC_MAPPER_DEAD_OPACITY (1.0f / 255.0f)
GLIC_API int glic_mapper_prune(glic_mapper* m, float min_opacity, int dry_run, uint32_t* removed);
/* Densification: Inria 3DGS's densify_and_clone + densify_and_split (N = 2) driven by view-space gradients (no counterpart in
 * the reference, whose densificationPostfix is only the concatenation extend() uses).  Off by default; with it never enabled an
 * iteration enqueues the same work as before.
 *   glic_mapper_enable_densification(m): from now on every row i keeps two floats, accum_i and denom_i, starting at 0.  In every
 *   iteration that steps the Gaussians, for every view v of the batch (all world * views_per_rank of them) with radii_v,i > 0:
 *       accum_i += |(g.x, g.y)|,   denom_i += 1,
 *   g = that view's own dL_v/dmean2D (NDC-scaled, what glic_backward returns as dL_dmeans2D; not divided by the batch size, so
 *   the threshold does not depend on world * views_per_rank).  The per-view values are summed over a rank's views inside the
 *   per-Gaussian backward and committed by the Adam launch; an iteration skipped for a binning overflow leaves them unchanged,
 *   and so does GLIC_MAPPER_OPT_OPTIMIZER = 0.  extend() appends rows with zero statistics, a capacity growth keeps them,
 *   glic_mapper_prune moves them with their rows bit for bit, initialize / initialize_lidar zero them.  A second call does
 *   nothing.  With world > 1 it must come before glic_mapper_export (GLIC_ERR_INVALID_ARGUMENT otherwise; the exchange block
 *   gains two rows of Pcap floats, which the reduce carries: the committed statistics are world times the mean over the ranks,
 *   exactly the sums over all views when world is a power of two).
 *   Every row also keeps maxr_i, an int32 screen radius starting at 0 (Inria's max_radii2D): in every iteration that steps the
 *   Gaussians, maxr_i = max(maxr_i, radii_v,i) over every view v of the batch with radii_v,i > 0, radii_v the forward's radii of
 *   that view.  Each view's radii travel in a slot of the exchange block next to its flag byte (pushed to the peers with it
 *   when world > 1); the max is order-free, so replicas agree exactly.  maxr follows the rules of accum / denom above (overflow
 *   and OPT_OPTIMIZER = 0 leave it, extend() appends 0, growth keeps it, prune moves it, initialize zeroes it) and every real
 *   densify zeroes it.  Memory: 4 B per row of capacity, plus 2 * S * 4 B per row of capacity in the exchange block.
 *   glic_mapper_densify_stats(m, accum, denom): the P statistics of each kind to host arrays; synchronises.
 *   glic_mapper_screen_radii(m, out): the P values of maxr to a host array; densification must be enabled; synchronises.
 *   glic_mapper_densify(m, grad_threshold, percent_dense, scene_extent, dry_run, &cloned, &split) (the counts may be NULL):
 *   - candidates are the non-sky rows [S, P) (sky rows are never densified, so the sky prefix and save_map stay valid);
 *     grad_i = denom_i > 0 ? accum_i / denom_i : 0 (one IEEE division), selected iff grad_i >= grad_threshold;
 *     smax_i = the largest of the row's three activated scales (expf, the activation kernel's), cloned iff
 *     smax_i <= percent_dense * scene_extent (the product in float), split otherwise;
 *   - the result rows, in Inria's order: every row that is not split, in its order; the clones, in index order; the first child
 *     of every split row in index order; then the second child of every split row.  Kept rows keep their parameters and both Adam
 *     moments bit for bit; clones are bit-identical copies of their parent's six groups; children copy rotation, f_dc, f_rest
 *     and opacity, take log_scale = __fsub_rn(ls, (float)log(1.6)) (Inria's log(exp(ls) / (0.8 * 2)) up to rounding), and
 *     xyz = glic_densify_split of the parent's xyz, activated scale s and normalised rotation q (the activation kernel's) at
 *     key (cfg.seed, call, row), row = the child's result row, call = the number of earlier real densify calls of this mapper;
 *     every new row has zero moments; sky rows, n_sky, keyframes, exposure and pose state are untouched;
 *   - a real call (dry_run == 0) then zeroes every row's statistics (densification_postfix) and advances `call`; a dry run only
 *     counts, changes nothing and does not advance `call`;
 *   - capacity: a result that does not fit grows the arenas like extend() (to max(rows, 2 * capacity)); with world > 1 and the
 *     mapper connected it returns GLIC_ERR_WORKSPACE and changes nothing (the dry-run counts let the host prune first);
 *   - densification not enabled, a NULL mapper, a non-finite or negative grad_threshold or percent_dense, or a scene_extent
 *     that is not finite and > 0 return GLIC_ERR_INVALID_ARGUMENT and change nothing.  Allocation failures follow the failure
 *     contract above.  The call drains the iteration pipeline (as prune does) and synchronises.  It needs one spare arena of the
 *     capacity while it runs, and its selection scratch (12 B per row) lives in the extend() staging buffer.  It is
 *     glic_mapper_densify_and_prune with min_opacity = 0 and both size tests off, which removes nothing (act(l) < 0 never holds),
 *     except that a mapper without rows returns GLIC_OK with zero counts.
 *   - world > 1: every rank makes the same calls between the same optimize() calls; replicas stay bit-identical in parameters,
 *     moments and statistics with no exchange.
 * glic_densify_split(n, xyz, scale, rot, seed, call, first_row, xyz_out, z_out, stream): the children's geometry on its own, for
 *   n children (device arrays; child t has parent xyz[t], activated scale[t], normalised rot[t] = (r, x, y, z), 16-byte aligned,
 *   and result row first_row + t).  Per axis a the standard normal z_a comes from the skybox's counter-based generator
 *   (glic_skybox_init) at counter k = ((call + 1) * 2^32 + row) * 3 + a (mod 2^64): r = mix64(seed + (k + 1) * 0x9E3779B97F4A7C15),
 *   u1 = (r >> 40) * 2^-24, u2 = ((r >> 16) & 0xFFFFFF) * 2^-24, then Box-Muller
 *       z_a = __fmul_rn(sqrtf(__fmul_rn(-2, logf(__fsub_rn(1, u1)))), cospif(__fmul_rn(2, u2))).
 *   With v_a = __fmul_rn(s_a, z_a) and R = Inria's build_rotation(q), each entry one of
 *       1 - 2 (y y + z z), 2 (x y - r z), 2 (x z + r y) / 2 (x y + r z), 1 - 2 (x x + z z), 2 (y z - r x) /
 *       2 (x z - r y), 2 (y z + r x), 1 - 2 (x x + y y)
 *   with every product, sum and difference rounded once (_rn), xyz_out_i = p_i + ((R_i0 v_0 + R_i1 v_1) + R_i2 v_2), rounded
 *   in that order.  z_out (optional, [n][3]) receives the normals.  No host synchronisation. */
#define GLIC_MAPPER_DENSIFY_GRAD_THRESHOLD 0.0002f   /* Inria's densify_grad_threshold */
#define GLIC_MAPPER_PERCENT_DENSE 0.01f
GLIC_API int glic_mapper_enable_densification(glic_mapper* m);
GLIC_API int glic_mapper_densify(glic_mapper* m, float grad_threshold, float percent_dense, float scene_extent, int dry_run,
                                 uint32_t* cloned, uint32_t* split);
GLIC_API int glic_mapper_densify_stats(glic_mapper* m, float* grad_accum, float* denom);
GLIC_API int glic_densify_split(int n, const float* xyz, const float* scale, const float* rot, uint64_t seed, uint64_t call,
                                uint32_t first_row, float* xyz_out, float* z_out, void* stream);
GLIC_API int glic_mapper_screen_radii(glic_mapper* m, int32_t* out);
/* Opacity reset (Inria's reset_opacity).  glic_mapper_reset_opacity(m, max_opacity): every non-sky row [S, P) whose
 * act(logit) > max_opacity (act as in glic_mapper_prune) gets logit = (float)log(r / (1 - r)), computed in double with
 * r = (double)max_opacity; every other logit stays bit for bit.  (Inria's inverse_sigmoid(min(sigmoid(l), 0.01)) also moves
 * the rows already below the cut, by rounding; this does not.)  Both Adam moments of the opacity group become zero for every
 * non-sky row, as Inria's replace_tensor_to_optimizer does.  Sky rows, every other group and every other moment stay bit for
 * bit.  A NULL mapper, or a max_opacity that is not finite or not in (0, 1), returns GLIC_ERR_INVALID_ARGUMENT and changes
 * nothing.  Drains the iteration pipeline (as prune does) and synchronises.  world > 1: every rank makes the same call between
 * the same optimize() calls; no exchange is needed. */
#define GLIC_MAPPER_RESET_OPACITY 0.01f
GLIC_API int glic_mapper_reset_opacity(glic_mapper* m, float max_opacity);
/* Densify and prune in one compaction (Inria's densify_and_prune).  The result is defined in two steps:
 *   1. exactly what glic_mapper_densify(grad_threshold, percent_dense, scene_extent) would produce: the same selection, row
 *      order and bits;
 *   2. every row of that result that meets the prune predicate is removed:
 *        act(logit) < min_opacity (prune's own test; sky rows can go by it), or, for non-sky rows,
 *        max_screen_radius > 0 and maxr > max_screen_radius, or
 *        max_world_scale > 0 and the largest activated scale (expf of the row's own log-scale) > max_world_scale,
 *      where maxr is the statistic gathered before the call for the rows that existed and 0 for clones and children, and a
 *      split child is judged at its own, reduced scale.  (Inria's code compares max_radii2D after densification_postfix has
 *      zeroed it, so its screen-size test never fires; here it does.)
 * Survivors keep the result order.  A split child draws its xyz at the row it has in the unpruned densify result, so the call
 * equals glic_mapper_densify followed by the predicate, bit for bit, children's xyz included.  Computed in one pass: one
 * selection, one gather per arena into one spare arena (moments for the surviving kept rows only; new rows get zero moments).
 * After a real call accum, denom and maxr are zero for every row, `call` advances (as in densify) and glic_mapper_sky_rows is
 * the number of surviving sky rows.  *out (may be NULL): cloned and split as glic_mapper_densify counts them, pruned = the rows
 * of the densify result the predicate removed, rows = the rows after the call.
 * Capacity: only the final row count must fit; a result that does not grows the arenas like extend() when the mapper is not
 * connected, and returns GLIC_ERR_WORKSPACE and changes nothing when it is (world > 1), so a connected mapper can densify
 * whenever pruning makes room.  Rejected with GLIC_ERR_INVALID_ARGUMENT, changing nothing: what glic_mapper_densify rejects, a
 * NULL p, min_opacity not finite or not in [0, 1], a negative max_screen_radius, max_world_scale not finite or negative, and a
 * result with no rows (dry run or not).  dry_run != 0 only counts.  Allocation failures follow the failure contract.  Drains
 * the iteration pipeline and synchronises.  world > 1: every rank makes the same calls between the same optimize() calls. */
typedef struct glic_density_params {
    float grad_threshold, percent_dense, scene_extent;   /* as glic_mapper_densify */
    float min_opacity;                                    /* remove iff act(logit) < min_opacity (prune's own test) */
    int32_t max_screen_radius;                            /* > 0: remove non-sky rows with maxr > it; 0: off */
    float max_world_scale;                                /* > 0: remove non-sky rows whose largest activated scale > it; 0: off */
} glic_density_params;
typedef struct glic_density_counts { uint32_t cloned, split, pruned, rows; } glic_density_counts;
GLIC_API int glic_mapper_densify_and_prune(glic_mapper* m, const glic_density_params* p, int dry_run, glic_density_counts* out);
/* Density control inside optimize() (Inria's schedule).  glic_mapper_set_density_schedule(m, s) sets the schedule (NULL: off,
 * the default) and restarts the totals; densification must be enabled to set one.  Rejected with GLIC_ERR_INVALID_ARGUMENT:
 * densify_interval 0, grad_threshold, percent_dense, world_scale_factor or scene_extent not finite or negative, min_opacity not
 * finite or not in [0, 1], reset_opacity not finite or not in (0, 1), a negative screen_radius.
 * After each iteration optimize() enqueues, with n = stats.iterations after it (counted across calls, overflow-skipped
 * iterations included):
 *   - if densify_from < n < densify_until and n % densify_interval == 0: glic_mapper_densify_and_prune with the schedule's
 *     grad_threshold, percent_dense and min_opacity, scene_extent = the schedule's when > 0, glic_mapper_scene_extent
 *     otherwise, and, only when opacity_reset_interval > 0 and n > opacity_reset_interval (Inria enables them together),
 *     max_screen_radius = screen_radius and max_world_scale = world_scale_factor * extent (in float); both off before.  A
 *     derived extent that is not > 0 (one keyframe, or all at one place) skips this step and leaves the statistics;
 *   - then, if opacity_reset_interval > 0, n < densify_until and n % opacity_reset_interval == 0: glic_mapper_reset_opacity
 *     (reset_opacity).
 * With GLIC_MAPPER_OPT_OPTIMIZER = 0 the schedule does nothing.  A scheduled step drains the pipeline (the only new
 * synchronisation); one that fails (GLIC_ERR_WORKSPACE on a connected mapper, say) ends optimize() with its error, and the
 * iterations before it stand.  stats.ms_optimize covers the whole call.
 * glic_mapper_scene_extent(m, out): Inria's getNerfppNorm radius over the training keyframes' current camera centres c_k (the
 * device poses under pose refinement, as glic_mapper_pose_get returns them): 1.1 * max_k |c_k - mean(c)| in double, rounded to
 * float; 0 without keyframes.
 * glic_mapper_density_totals(m, out, steps, resets) (each may be NULL): since the schedule was set, the summed cloned, split and
 * pruned counts of its densify steps, rows = the rows after the latest one (0 before any), the number of densify steps and the
 * number of opacity resets. */
typedef struct glic_density_schedule {
    uint32_t densify_from, densify_until, densify_interval;  /* Inria: 500, 15000, 100 */
    uint32_t opacity_reset_interval;                         /* 3000; 0 = never */
    float grad_threshold, percent_dense, min_opacity;        /* 0.0002, 0.01, 0.005 */
    float reset_opacity;                                     /* 0.01 */
    int32_t screen_radius;                                   /* 20 */
    float world_scale_factor;                                /* 0.1 */
    float scene_extent;                                      /* > 0: fixed; 0: derived at each step */
} glic_density_schedule;
#define GLIC_MAPPER_DENSIFY_FROM 500u
#define GLIC_MAPPER_DENSIFY_UNTIL 15000u
#define GLIC_MAPPER_DENSIFY_INTERVAL 100u
#define GLIC_MAPPER_OPACITY_RESET_INTERVAL 3000u
#define GLIC_MAPPER_MIN_OPACITY 0.005f
#define GLIC_MAPPER_SCREEN_RADIUS 20
#define GLIC_MAPPER_WORLD_SCALE_FACTOR 0.1f
GLIC_API int glic_mapper_set_density_schedule(glic_mapper* m, const glic_density_schedule* s);
GLIC_API int glic_mapper_scene_extent(glic_mapper* m, float* out);
GLIC_API int glic_mapper_density_totals(glic_mapper* m, glic_density_counts* out, uint32_t* steps, uint32_t* resets);
/* multi-GPU wiring: every rank exports the 64-byte IPC handle of its exchange block, the caller all-gathers them
 * (torch.distributed / MPI / a file: plumbing) and hands all `world` handles back. */
GLIC_API int glic_mapper_export(glic_mapper* m, unsigned char* handle64);
GLIC_API int glic_mapper_connect(glic_mapper* m, const unsigned char* handles /* [world][64] */);
GLIC_API int glic_mapper_synchronize(glic_mapper* m);
/* options: GLIC_MAPPER_OPT_OPTIMIZER (default 1): 0 leaves the Adam launch out of the iteration, so that a benchmark can time
 * the rasterization step (activations, forward, loss, backward, exchange) on its own.  Keyframe images may be device pointers
 * (the copy uses cudaMemcpyDefault): that is how "inputs resident in HBM" is measured. */
/* GLIC_MAPPER_OPT_DETERMINISTIC (default 0): 1 makes every later optimize, align, evaluate, evaluate_lpips and render use the
 * deterministic render backward of glic_backward_deterministic and fixed-order sums for the loss value and the PSNR / SSIM sums;
 * 0 switches them off again.  Either call drains the pipeline.  With the option on, given the same calls, seeds and inputs, on
 * the same GPU model and library build, every getter returns the same bits: the parameters, both Adam moments, the poses, E and
 * their Adam state, the densification statistics, the screen radii, the sky rows, stats (last_loss included) and the density
 * totals, and the metrics and images of evaluate, render, align and render_camera.  The option costs a workspace that follows the
 * binning capacity (glic_deterministic_bytes of it), allocated by the call and grown with the capacity under the failure contract
 * above (a failed allocation returns GLIC_ERR_CUDA and leaves the mapper, the option included, as it was).  With world > 1 every
 * rank must set it identically; the reduce adds in rank order, so runs then repeat across runs and replicas. */
enum { GLIC_MAPPER_OPT_OPTIMIZER = 1, GLIC_MAPPER_OPT_BINNING_PAIRS = 2 /* (tile, Gaussian) pairs the binning workspace holds; grows by itself on overflow */,
       GLIC_MAPPER_OPT_DETERMINISTIC = 3 };
GLIC_API int glic_mapper_set_option(glic_mapper* m, int option, int value);
/* Per-keyframe exposure (the reference's apply_exposure / exposure_lr, config/fastlivo.yaml:25-26, which its render()
 * never applies).  Off by default.  glic_mapper_enable_exposure(m, lr) may be called before or between optimize() calls:
 * from then on every training keyframe k has a 3x4 affine colour transform E_k (row-major, see glic_l1_ssim_loss_exposure),
 * starting at [I | 0] (keyframes added later start there too).  Each iteration's loss is taken on E_k applied to the
 * rendered image of every view of keyframe k; after the Gaussian step one launch steps the batch's keyframes with
 * torch::optim::Adam's rule (betas 0.9 / 0.999, eps 1e-8, no weight decay, lr = exposure_lr, bias correction from the
 * keyframe's own step count t, which rises by one per batch that holds the keyframe):
 *     g = (1/S) * sum over the batch slots holding k of dL/dE,  m = b1 m + (1-b1) g,  v = b2 v + (1-b2) g^2,
 *     E -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps).
 * An iteration skipped for a binning overflow leaves E, m, v and t unchanged; GLIC_MAPPER_OPT_OPTIMIZER = 0 leaves the
 * exposure step out too.  With world > 1 every rank pushes its slots' 12-float dL/dE to its peers and every replica
 * applies the same step: E, m, v and t stay bit-identical across ranks (call enable / set identically on every rank).
 * glic_mapper_evaluate(is_train = 1) applies the keyframe's E before the [0,1] clamp; held-out keyframes (is_train = 0)
 * are evaluated with the identity, since no exposure was ever fitted for them; extend() renders alpha only and is not
 * affected.  exposure_get / exposure_set read and write E of training keyframe `index` (host arrays of 12 floats; they
 * synchronise and need exposure enabled); set leaves that keyframe's Adam state (m, v, t) alone. */
GLIC_API int glic_mapper_enable_exposure(glic_mapper* m, float exposure_lr);
GLIC_API int glic_mapper_exposure_get(glic_mapper* m, int index, float* out12);
GLIC_API int glic_mapper_exposure_set(glic_mapper* m, int index, const float* in12);
/* the exposure's Adam state of training keyframe `index`: both moments (12 floats each) and the step count; synchronises */
GLIC_API int glic_mapper_exposure_adam_state(glic_mapper* m, int index, float* exp_avg12, float* exp_avg_sq12, int* step);
/* Per-keyframe pose refinement (no counterpart in the reference, which takes every odometry pose as exact).  Off by default.
 * glic_mapper_enable_pose_refinement(m, lr_translation, lr_rotation) may be called before or between optimize() calls; a
 * repeated call changes the rates only.  Training keyframe k's pose (R_wc, t_wc) defines T_cw = [R_wc^T | -R_wc^T t_wc]
 * (kept in float64, initialised exactly from the floats), perturbed as T_cw(delta) = Exp(delta) T_cw with
 * delta = (rho, omega) in the camera frame, translation first, Exp the SE(3) exponential.  Its gradient at delta = 0 is
 *     g_k = (1/S) * sum over the batch slots holding k of dL_view/ddelta,
 * computed inside the per-Gaussian backward.  After the Gaussian step one launch steps the batch's keyframes with
 * torch::optim::Adam's rule (betas 0.9 / 0.999, eps 1e-8, bias correction from the keyframe's own step count t, lr =
 * lr_translation for rho and lr_rotation for omega), then T_cw <- Exp(u) T_cw for the update u, re-derives the float
 * (R_wc, t_wc) and rebuilds the keyframe's camera block from them: that block always equals glic_camera_block(R_wc, t_wc)
 * of the current float pose, bit for bit, and an update of exactly zero leaves it unchanged.  The moments persist when the
 * pose moves.  An iteration skipped for a binning overflow leaves pose, m, v and t unchanged; GLIC_MAPPER_OPT_OPTIMIZER = 0
 * leaves the pose step out too.  With world > 1 each rank pushes its slots' 6-float gradients to its peers and every replica
 * applies the same step.  Training keyframes are rendered, evaluated and (extend(), on the newest) projected with their
 * current pose; held-out keyframes keep theirs; keyframes added later start at their given pose with zero state.
 * pose_get returns the current float pose of training keyframe `index` and, if cam41 is not NULL, its camera block in
 * glic_camera_block's layout, read back from the device.  pose_set rejects non-finite input and an R_wc that is not a
 * rotation; it leaves the Adam state alone.  These calls synchronise and need pose refinement enabled. */
GLIC_API int glic_mapper_enable_pose_refinement(glic_mapper* m, float lr_translation, float lr_rotation);
GLIC_API int glic_mapper_pose_get(glic_mapper* m, int index, float* R_wc9, float* t_wc3, float* cam41_or_null);
GLIC_API int glic_mapper_pose_set(glic_mapper* m, int index, const float* R_wc9, const float* t_wc3);
/* the pose's Adam state of training keyframe `index`: both moments (6 floats each, rho then omega) and the step count */
GLIC_API int glic_mapper_pose_adam_state(glic_mapper* m, int index, float* exp_avg6, float* exp_avg_sq6, int* step);
/* Test-time alignment (BARF-style evaluation; Inria 3DGS's train_test_exp): fit one keyframe's camera pose and exposure to its
 * image against the frozen map, then score it there.  glic_mapper_evaluate scores a held-out keyframe at its odometry pose
 * with the identity exposure; once pose refinement and exposure have moved the training keyframes (and with them the map),
 * that measures the drift and the brightness of the frame as well as the map.  glic_mapper_align(m, is_train, index, p, out,
 * rgb_host) works on either list:
 *   - start: the keyframe's current float pose (the refined pose of a training keyframe under pose refinement, the stored pose
 *     otherwise; the float64 T_cw is the refined master, or derived from the floats as glic_camera_block does) and
 *     E = the training keyframe's E when exposure is enabled, [I | 0] otherwise; zero Adam moments and step counts;
 *   - each of p->iterations iterations: render at the current pose; the L1 + D-SSIM loss (cfg.lambda_dssim) on the fit region,
 *     with E applied when exposure_lr > 0 or the start E is a trained one; the render backward and the pose-only per-Gaussian
 *     backward on that region's dL/dpixel (zero elsewhere); one Adam step of the pose and, when exposure_lr > 0, one of E, with
 *     the rules, betas, eps and bias correction of pose refinement and exposure above for a batch of one slot (T_cw <- Exp(u)
 *     T_cw in float64, the float pose and camera block re-derived from it).  A zero rate leaves that part of the pose at its
 *     start (its moments still advance, as in training); exposure_lr = 0 leaves E at its start and its moments at zero;
 *   - fit region: split = 0 the whole frame; split = 1 columns [0, W/2), the loss taken on the cropped planes [3, H, W/2]
 *     (SSIM pads at the crop edge as at a frame border).  Score region: the whole frame, or columns [W/2, W);
 *   - an iteration whose forward overflows the binning workspace changes nothing and counts in `skipped`; after the loop the
 *     workspace grows as it does after an overflowed training iteration (stats.overflow_regrows counts it);
 *   - scoring, once at the end: the keyframe drawn at the fitted pose (as glic_mapper_evaluate draws, overflow redone), the
 *     fitted E applied when it was in the loss, clamped to [0,1]; PSNR / SSIM as glic_mapper_evaluate computes them and LPIPS as
 *     glic_mapper_evaluate_lpips does (NaN without glic_mapper_load_lpips), on the score region (with split = 1 the right-half
 *     crops of the clamped frame and image, exactly glic_eval_psnr_ssim of those crops).  rgb_host (may be NULL) receives the
 *     whole clamped, exposed frame [3,H,W] as glic_mapper_render writes it.  With no fit (iterations = 0, or all three rates 0)
 *     and split = 0 the scores are glic_mapper_evaluate_lpips's and the image glic_mapper_render's, bit for bit;
 *   - out: the fitted float pose, E, the scores, the fit loss of the first and of the last stepped iteration (NaN without one),
 *     both Adam moments of the pose and of E (the first step from zero moments stores m = fl((1 - b1) g)), and the counts.
 * The map is frozen: the call changes no parameter, moment, densification statistic, maxr, sky row count, keyframe, pose,
 * camera block, E, Adam state, sampler state or density-control counter, and no stats field but overflow_regrows.  It drains
 * the iteration pipeline (as glic_mapper_evaluate does), enqueues the iterations without a host synchronisation (the overflow
 * skip stays on the device) and synchronises at the end.  With world > 1 it is rank-local: it reads and writes none of the
 * exchange block the peers push into, so one rank may align between optimize() calls while the others do not.
 * Memory: its workspace (kept for the next call) is 12 B per row of capacity (the colour gradients) + 6 doubles per 128 rows
 * (the pose partials) + with split three planes of 12 * H * (W - W/2) B + a state row under 1 KB; the exposure loss's scratch and
 * LPIPS's grow as for training and evaluation.  Everything is reserved before anything runs (failure contract above).
 * Rejected with GLIC_ERR_INVALID_ARGUMENT, changing nothing: a NULL m, p or out; an index out of range; iterations < 0; a
 * rate that is negative or not finite; split not 0 or 1; split = 1 on a frame under 2 columns; a score region under 31x31
 * with LPIPS weights loaded; a mapper with no rows. */
typedef struct glic_align_params {
    int iterations;                    /* >= 0 */
    float lr_translation, lr_rotation; /* pose Adam rates, >= 0; 0 leaves that part of the pose fixed */
    float exposure_lr;                 /* >= 0; 0 leaves E fixed */
    int split;                         /* 0: fit and score on the whole frame; 1: fit on columns [0, W/2), score on [W/2, W) */
} glic_align_params;
typedef struct glic_align_result {
    float R_wc[9], t_wc[3];            /* the fitted float pose */
    float E[12];                       /* the fitted exposure (row-major 3x4, as glic_mapper_exposure_get) */
    float psnr, ssim, lpips;           /* at the fitted pose and E, on the score region; lpips is NaN without glic_mapper_load_lpips */
    float first_loss, last_loss;       /* fit-region loss of the first and of the last stepped iteration */
    float pose_exp_avg[6], pose_exp_avg_sq[6], expo_exp_avg[12], expo_exp_avg_sq[12];
    int steps, skipped;                /* stepped iterations, and iterations skipped for a binning overflow */
} glic_align_result;
GLIC_API int glic_mapper_align(glic_mapper* m, int is_train, int index, const glic_align_params* p, glic_align_result* out,
                               float* rgb_host /* [3,H,W] or NULL */);
/* Camera (camera.h:38-110) in closed form, as the mapper derives it from a keyframe pose: out41 = view[16] (column-major
 * Rt) | proj[16] (column-major P*Rt) | campos[3] | tan_fovx, tan_fovy | limx_neg, limx_pos, limy_neg, limy_pos. */
GLIC_API int glic_camera_block(int width, int height, float fx, float fy, float cx, float cy, const float* R_wc /*[9] row-major*/,
                               const float* t_wc /*[3]*/, float* out41);
/* Rendering the map from any camera: glic_mapper_render_camera(m, cam, exposure_index, with_sky, rgb, final_T, depth,
 * median_depth) draws the current map (parameters, sky rows, fitted exposures, refined poses as they stand) with glic_render
 * from a camera the caller chooses: a fly-through, a frame at display resolution, a depth map for meshing or a LiDAR check.
 *   - camera: glic_camera_block(cam->width, cam->height, fx, fy, cx, cy, R_wc, t_wc), the closed form every keyframe uses;
 *   - rgb [3,H,W]: the colour with training keyframe exposure_index's E applied (-1: the identity), clamped to [0,1], by the
 *     device code glic_mapper_render's image goes through; final_T [H,W], depth [H,W] and median_depth [H,W] are glic_render's
 *     raw planes.  Each output is host or device memory (copied with cudaMemcpyDefault) or NULL; at least one is non-NULL;
 *   - with_sky = 1 draws every row; 0 only rows [S, P) (glic_mapper_sky_rows), the map without the skybox;
 *   - at training keyframe k's current float pose (glic_mapper_pose_get, or the stored pose), the configured intrinsics and
 *     size, exposure_index = k with exposure enabled (-1 otherwise) and with_sky = 1, rgb equals glic_mapper_render(m, 1, k)
 *     bit for bit; at a held-out keyframe's pose with exposure_index = -1 it equals glic_mapper_render(m, 0, k);
 *   - with_sky = 0 on a map of sky rows only draws nothing: final_T 1, every other plane 0;
 *   - binning: the mapper's binning workspace; a frame that overflows it grows it and is drawn again, as evaluation does
 *     (stats.overflow_regrows counts it).  Only the binning workspace grows, to about 20-32 B per (tile, Gaussian) pair of the
 *     largest frame drawn, and it is kept; the training's checkpoint (sample) workspace is neither used nor grown;
 *   - memory: a render workspace kept for the next call, for the largest frame asked for so far: the camera block, an image
 *     workspace and six planes, about 52 B per pixel.  Everything is reserved before anything runs (failure contract above).
 * The map is frozen, exactly as under glic_mapper_align: no parameter, moment, statistic, keyframe, pose, camera block, E, Adam
 * state, sampler state or density-control counter changes, and no stats field but overflow_regrows.  The call drains the
 * iteration pipeline first and synchronises at the end.  With world > 1 it is rank-local and touches no exchange slot.
 * Rejected with GLIC_ERR_INVALID_ARGUMENT, changing nothing: a NULL m or cam, or all four outputs NULL; width or height < 1,
 * or more than GLIC_MAX_TILES tiles; fx or fy not finite and > 0, cx or cy not finite; a non-finite pose, or an R_wc that is
 * not a rotation (glic_mapper_pose_set's test); exposure_index not -1 and not a training index with exposure enabled;
 * with_sky not 0 or 1; a mapper with no rows. */
typedef struct glic_render_camera {
    float R_wc[9], t_wc[3];            /* row-major, as glic_keyframe */
    float fx, fy, cx, cy;
    int width, height;
} glic_render_camera;
GLIC_API int glic_mapper_render_camera(glic_mapper* m, const glic_render_camera* cam, int exposure_index, int with_sky,
                                       float* rgb, float* final_T, float* depth, float* median_depth);
/* Pruning the rows no view blends.  glic_mapper_contribution(m, views_host, n_views, max_weight, hits, ends) computes the
 * contribution scores (glic_contribution) of every row, sky rows included, over training keyframes views_host[0 .. n_views)
 * (NULL: every training keyframe; held-out keyframes are never scored, which would leak the test set into the map).  Each view
 * is drawn at its current camera block (the refined pose under pose refinement), every row drawn, as training draws it; a
 * view that overflows the binning workspace grows it and is drawn again (stats.overflow_regrows counts it), and only the
 * binning workspace grows; a view that still overflows after four draws fails the call with GLIC_ERR_WORKSPACE rather than go
 * unscored.  max_weight [P] floats, hits [P] and ends [P] uint64 are host or device memory (cudaMemcpyDefault); any of them may
 * be NULL, not all three.  The map is frozen as under glic_mapper_render_camera.  The call drains the iteration pipeline first
 * and synchronises at the end; with world > 1 it is rank-local and touches no exchange slot.
 * glic_mapper_prune_unseen(m, p, dry_run, removed) computes the scores over p->views as above and removes every row for which
 *   (the row is not a sky row, or p->sky = 1) and (max_weight < p->min_weight or hits + ends < p->min_hits);
 * with min_hits = GLIC_MAPPER_UNSEEN_MIN_HITS and min_weight = 0 that is exactly the rows that neither take nor end a pixel of
 * any scored view, so no pixel of those views changes: their render, evaluation and render_camera planes at their poses keep
 * every bit.
 * The compaction is glic_mapper_prune's (stable order, parameters and both moments bit for
 * bit, the densification statistics moving with their rows, the sky-row count updated so save_map still writes the non-sky
 * survivors, the densify call counter untouched, vacated rows zeroed, capacity unchanged).  *removed (may be NULL) gets the
 * count; dry_run != 0 only counts.  Memory: the score buffers (20 B per row of capacity, kept for the next call) and the
 * selection scratch are reserved before the scores are computed; the spare arena is allocated, as glic_mapper_prune allocates
 * it, before the map changes (failure contract above).  Rejected with GLIC_ERR_INVALID_ARGUMENT, changing nothing:
 * a NULL m or p, n_views < 0, a view index out of range, min_weight not finite or not in [0, 1], sky not 0 or 1, a result with
 * no rows (dry run or not).  A mapper with no rows returns GLIC_OK with 0 removed.  world > 1: every rank makes the same call
 * between the same optimize() calls; every rank holds every training keyframe and the scores are order-free, so replicas
 * remove the same rows with no exchange. */
#define GLIC_MAPPER_UNSEEN_MIN_HITS 1
typedef struct glic_unseen_params {
    const int* views;              /* host, training keyframe indices; NULL: every training keyframe */
    int n_views;                   /* >= 0; ignored when views is NULL */
    float min_weight;              /* in [0, 1]: remove rows whose max_weight < min_weight */
    uint64_t min_hits;             /* remove rows whose hits + ends < min_hits */
    int sky;                       /* 1: sky rows can be removed too; 0: they stay */
} glic_unseen_params;
GLIC_API int glic_mapper_contribution(glic_mapper* m, const int* views_host, int n_views, float* max_weight, uint64_t* hits,
                                      uint64_t* ends);
GLIC_API int glic_mapper_prune_unseen(glic_mapper* m, const glic_unseen_params* p, int dry_run, uint32_t* removed);
/* Raw frames (Dataset::addFrame, gaussian.cpp:41-111, and the keyframe hand-off of mapping.cpp:158-174): the host feeds every
 * aligned camera frame with its odometry pose and LiDAR scan; the mapper selects the keyframes, keeps each image as 8 bits
 * in HBM and builds or extends the map on the GPU.  optimize() stays the caller's call (mapping.cpp:178).
 *   glic_mapper_enable_frames(m, k, sky_points, sky_radius): select_every_k_frame (>= 1) and the skybox settings of the
 *   initial map (skybox_points_num, skybox_radius; sky_radius > 0 when sky_points > 0).  Once per mapper, before the first
 *   add_frame; a second call returns GLIC_ERR_INVALID_ARGUMENT.
 *   glic_mapper_add_frame(m, f, is_keyframe):
 *   - R = Eigen::Quaterniond(w, x, y, z).toRotationMatrix() in double, Eigen's formula and operation order, no normalisation;
 *     the keyframe's float pose is R_wc = (float)R, t_wc = (float)t, and its camera block is glic_camera_block of those
 *     floats (the reference's Camera rounds t_cw from the doubles instead: t_cw may differ by 1 ulp);
 *   - the image is copied once into a mapper-owned device store (packed HWC BGR8, row padding dropped, allocated in chunks
 *     that never move); the mapper keeps no host pointer;
 *   - the points are appended to a device scan buffer with depth_rsp = (float)(((Rcw20 p0 + Rcw21 p1) + Rcw22 p2) + tcw2) in
 *     double without FMA, p = (double)xyz, R_cw = R^T, t_cw = -R_cw t_wc in the same order (gaussian.cpp:64-70);
 *   - the frame is a training keyframe iff (frames added before it + 1) % k == 0, a held-out keyframe otherwise;
 *   - at a training keyframe the accumulated scan initializes the map (glic_mapper_initialize_lidar with the enable_frames
 *     sky, colours (double)c / 255.0, focal = ((double)fx + (double)fy) / 2 of the configuration) if neither initialize
 *     nor initialize_lidar has run, and extends it otherwise (glic_mapper_extend with colours (float)((double)c / 255.0));
 *     either way the scan buffer is emptied.
 *   A NULL mapper, frame or pointer (xyz / rgb may be NULL when n_points is 0), row_bytes < 3 W, n_points < 0, frames not
 *   enabled, or a first training keyframe with an empty accumulated scan return GLIC_ERR_INVALID_ARGUMENT and change
 *   nothing.  Synchronises.  *is_keyframe (optional) is 1 for a training keyframe, 0 for a held-out one.
 *   Frame keyframes train, evaluate and render like glic_keyframe ones: the 8-bit image is decoded on the device
 *   (glic_decode_bgr8) where the float image would be copied, so an iteration moves no image bytes over PCIe.
 *   glic_mapper_keyframe_image writes the float [3,H,W] image the loss sees of any keyframe to rgb_host (synchronises).
 *   glic_mapper_frames_get returns the counters below. */
typedef struct glic_frame {
    double q_wc[4];                /* odometry orientation, geometry_msgs order (x, y, z, w) */
    double t_wc[3];
    const uint8_t* bgr;            /* host [H][row_bytes]: BGR8 rows of 3 W bytes (sensor_msgs/Image "bgr8", cv_bridge BGR8) */
    size_t row_bytes;              /* >= 3 W */
    int n_points;                  /* >= 0 */
    const float* xyz;              /* host [n,3], world frame (PCL PointXYZRGB x, y, z) */
    const uint8_t* rgb;            /* host [n,3] (PCL r, g, b) */
} glic_frame;
typedef struct glic_frame_stats {
    uint32_t frames, train, test;  /* frames added so far, and how many became training / held-out keyframes */
    uint32_t pending_points;       /* scan points waiting for the next training keyframe */
    uint64_t image_bytes;          /* device bytes held by the 8-bit frame store */
} glic_frame_stats;
GLIC_API int glic_mapper_enable_frames(glic_mapper* m, int select_every_k_frame, int sky_points, int sky_radius);
GLIC_API int glic_mapper_add_frame(glic_mapper* m, const glic_frame* f, int* is_keyframe /* may be NULL */);
GLIC_API int glic_mapper_keyframe_image(glic_mapper* m, int is_train, int index, float* rgb_host /* [3,H,W] */);
GLIC_API int glic_mapper_frames_get(glic_mapper* m, glic_frame_stats* out);

/* Per-keyframe valid-pixel masks: leave moving objects and the rig's own platform out of the map.  A mask is a host [H][W]
 * byte map of one keyframe, nonzero = the pixel is used; it is kept bit-packed on the device (glic_pack_mask: H *
 * ceil(W / 32) words, 259 200 bytes at 1920x1080).  Where it is used, with the semantics of glic_l1_ssim_loss_masked:
 *   - every training iteration's loss of the keyframe: the ground truth under the mask has no influence on any bit of
 *     training, and dL/dimg is +0 there, so exposure, pose refinement, the densification statistics and the multi-GPU
 *     exchange follow from the masked dL/dimg unchanged;
 *   - glic_mapper_evaluate / evaluate_lpips: PSNR and SSIM of glic_eval_psnr_ssim_masked; LPIPS is taken on the same clamped
 *     pair, which is 0 in both images under the mask, with its usual mean over every pixel;
 *   - glic_mapper_align: the fit loss and the scores, each over its own columns of the mask; a mask that leaves the fit or the
 *     score columns without a used pixel is refused (GLIC_ERR_INVALID_ARGUMENT); rgb_host is the scored image, 0 under the mask;
 *   - extend() on the newest training keyframe (glic_mapper_extend, and add_frame's hand-off): no point is inserted at a masked
 *     pixel.  Exactly: the selection is that of glic_extend with final_T set to 0 at the masked pixels.
 * Not affected: glic_mapper_render, glic_mapper_render_camera, contribution scoring and prune_unseen, save_map.  A mapper
 * with no mask on any keyframe enqueues exactly the launches it did before masks existed.  With world > 1 every rank sets
 * the same masks, as it adds the same keyframes.  Under GLIC_MAPPER_OPT_DETERMINISTIC the masked loss and evaluation use
 * their fixed-order sums: the same calls give the same bits.
 *   glic_mapper_set_keyframe_mask(m, is_train, index, valid): sets (valid != NULL) or clears (valid = NULL) the mask of a
 *   keyframe.  Packs and counts on the device and synchronises.  A NULL mapper, an index out of range or a mask with no used
 *   pixel return GLIC_ERR_INVALID_ARGUMENT; a failed allocation returns GLIC_ERR_CUDA; either way nothing changes.
 *   glic_mapper_keyframe_mask(m, is_train, index, out, valid_count): *valid_count = the used pixels (0: no mask); out
 *   (optional, [H][W] bytes) receives the stored mask as 0 / 1 when there is one and is left as it is otherwise.  Synchronises.
 *   glic_mapper_add_frame_masked(m, f, valid, is_keyframe): glic_mapper_add_frame with the frame's mask (valid NULL: none), set
 *   before the keyframe hand-off so that its extend() leaves the masked pixels out; a held-out frame keeps its mask for the
 *   evaluation and the alignment.  A mask with no used pixel is refused like the other bad arguments, changing nothing. */
GLIC_API int glic_mapper_set_keyframe_mask(glic_mapper* m, int is_train, int index, const uint8_t* valid /* host [H][W] or NULL */);
GLIC_API int glic_mapper_keyframe_mask(glic_mapper* m, int is_train, int index, uint8_t* out /* may be NULL */, uint32_t* valid_count);
GLIC_API int glic_mapper_add_frame_masked(glic_mapper* m, const glic_frame* f, const uint8_t* valid /* host [H][W] or NULL */,
                                          int* is_keyframe /* may be NULL */);

/* ---------------------------------------------------------------------------------------
 * Meshing (no counterpart in the reference): a coloured triangle mesh from depth maps, by TSDF fusion into a dense voxel grid and
 * naive surface nets, for collision checking, inspection, measurement or a viewer that does not draw splats.  Every step below
 * is one correctly rounded float operation, in the order written, with no contraction (the fmas are xform_row's own); nothing is
 * accumulated with atomics, so each output depends only on the inputs and the call order, and two identical call sequences give
 * identical bits.
 *   Grid: glic_tsdf_grid, data = DEVICE memory of glic_tsdf_bytes(dims) = 20 N bytes, planar tsdf[N] | weight[N] | colour[3][N]
 *   (f32), N = nx ny nz.  Lattice point (i, j, k) has index i + nx (j + ny k) and world position o + s (i, j, k), each coordinate
 *   __fadd_rn(o.x, __fmul_rn(s, (float)i)).  Every dimension in [2, 2048] with N < 2^31; voxel_size finite and > 0, origin
 *   finite.  glic_tsdf_bytes and glic_mesh_scratch_bytes return 0 for other dims.  glic_tsdf_clear zeroes it: unobserved
 *   everywhere.
 *   glic_tsdf_integrate fuses one W x H view.  viewmatrix_dev: the 16 column-major floats of a camera block (device memory, so
 *   a mapper keyframe's refined block needs no host round trip); depth [H,W]; rgb [3,H,W] or NULL (colour left untouched);
 *   mask_words a bit-packed mask of glic_pack_mask's layout (words_per_row >= glic_mask_words_per_row(W)) or NULL.  Per lattice
 *   point p at world position (X, Y, Z):
 *     1. (x, y, z) = rows 0..2 of the view matrix applied to (X, Y, Z, 1) as the renderer does it (xform_row, geom_math.cuh:
 *        m[12+r] + fma(Z, m[8+r], fma(X, m[r], Y m[4+r]))), so z is the view-space depth the renderer reports; skip unless z > 0;
 *     2. u = fx (x / z) + cx, v = fy (y / z) + cy; skip unless 0 <= u < W and 0 <= v < H (float comparisons: NaN skips);
 *        px = (int)floorf(u), py = (int)floorf(v) (pixel px covers u in [px, px + 1), the renderer's convention);
 *     3. skip a masked-out pixel; d = depth[py][px]; skip unless d > 0 and (max_depth == 0 or d <= max_depth): NaN skips, and so
 *        does 0, the median depth of a pixel whose T never falls below 0.5;
 *     4. sdf = d - z; skip unless sdf >= -trunc;
 *     5. t = fminf(1, sdf / trunc); with w the stored weight: tsdf = (tsdf w + t) / (w + 1), each colour channel
 *        col = (col w + rgb[c][py][px]) / (w + 1), weight = w + 1.
 *   A skipped point is neither read nor written.
 *   Extraction (naive surface nets): a lattice point is INSIDE iff tsdf < 0 and OBSERVED iff weight > 0.  Cell (i, j, k) has
 *   corners (i + a, j + b, k + c), a, b, c in {0, 1}; it is ACTIVE iff all 8 corners are observed and they are not all on one
 *   side.  Its 12 edges go in this order: the x-edges for (b, c) = (0,0), (1,0), (0,1), (1,1), the y-edges for (a, c) in the
 *   same order, then the z-edges for (a, b).  An edge from A to B (B the upper end) CROSSES when exactly one end is inside, at
 *   f = tA / (tA - tB).  The cell's vertex offset is the left fold, in edge order, of the crossing points in voxel units from the
 *   cell's lower corner, divided by the number of crossings; the vertex is o + s ((float)i + off) per axis, and its colour the
 *   same mean of cA + f (cB - cA), stored as __float2int_rn(fminf(fmaxf(c, 0), 1) 255).  Vertex ids are the ranks of the active
 *   cells in ascending linear index (of the lower corner).  Every lattice edge from L to L + e_a with both ends observed and
 *   exactly one inside, whose four cells with lower corners L - e_b - e_c, L - e_c, L, L - e_b ((a, b, c) cyclic) exist and are
 *   active, makes the quad of their vertices in that order, reversed unless L is inside (normals point out, into free space),
 *   split into the triangles (q0, q1, q2) and (q0, q2, q3).  Faces are ordered by 3 index(L) + a.
 *   glic_mesh_count(grid, scratch, bytes, counts_host, stream): counts_host[2] (HOST) = {vertices V, faces F}; the scans stay in
 *   the scratch (glic_mesh_scratch_bytes(dims): about N / 4 bytes); synchronises once.  glic_mesh_extract then fills xyz [V,3]
 *   f32, rgb [V,3] u8 and faces [F,3] i32 (device, all non-NULL) from them, asynchronously; the grid must be as it was counted.
 *   glic_mesh_ply_write(path, V, xyz, rgb, F, faces): HOST arrays to a binary little-endian PLY, element vertex V (float x y z,
 *   uchar red green blue), element face F (property list uchar int vertex_indices); an I/O failure returns
 *   GLIC_ERR_INVALID_ARGUMENT with the path in glic_last_error, as glic_ply_write does.
 *   Every call checks its arguments before it enqueues anything: a NULL pointer, bad dims, a bad voxel size or origin, a frame
 *   under 1x1 or above GLIC_MAX_TILES tiles, fx or fy not finite and > 0, cx or cy not finite, trunc not finite and > 0, max_depth
 *   not finite and >= 0 or a short words_per_row return GLIC_ERR_INVALID_ARGUMENT; a scratch under glic_mesh_scratch_bytes
 *   returns GLIC_ERR_WORKSPACE.
 * ------------------------------------------------------------------------------------- */
typedef struct glic_tsdf_grid {
    float origin[3];               /* world position of lattice point (0, 0, 0) */
    float voxel_size;              /* lattice spacing */
    int dims[3];                   /* nx, ny, nz */
    void* data;                    /* device, glic_tsdf_bytes(dims) bytes */
} glic_tsdf_grid;
GLIC_API size_t glic_tsdf_bytes(const int* dims /*[3]*/);
GLIC_API int glic_tsdf_clear(const glic_tsdf_grid* grid, void* stream);
GLIC_API int glic_tsdf_integrate(const glic_tsdf_grid* grid, const float* viewmatrix_dev, int W, int H, float fx, float fy, float cx,
                                 float cy, const float* depth, const float* rgb /* may be NULL */, const uint32_t* mask_words /* may be NULL */,
                                 int words_per_row, float trunc, float max_depth, void* stream);
GLIC_API size_t glic_mesh_scratch_bytes(const int* dims /*[3]*/);
GLIC_API int glic_mesh_count(const glic_tsdf_grid* grid, void* scratch, size_t scratch_bytes, uint64_t* counts_host /*[2]*/, void* stream);
GLIC_API int glic_mesh_extract(const glic_tsdf_grid* grid, const void* scratch, size_t scratch_bytes, float* xyz, uint8_t* rgb,
                               int32_t* faces, void* stream);
GLIC_API int glic_mesh_ply_write(const char* path, uint32_t V, const float* xyz, const uint8_t* rgb, uint32_t F, const int32_t* faces);

/* Meshing the map.  glic_mapper_extract_mesh(m, p, out) is exactly this composition:
 *   1. clear a grid of p's origin, voxel_size and dims;
 *   2. for each listed training keyframe k (p->views[0 .. n_views), NULL: every training keyframe; held-out keyframes are not
 *      used), in list order: draw the map WITHOUT the sky rows at k's current camera block (the refined pose under pose
 *      refinement), the configured intrinsics and size, by glic_mapper_render_camera's path with exposure_index -1 (the map's
 *      colour, not the frame's brightness); take its median depth and its clamped rgb; glic_tsdf_integrate them with k's view
 *      matrix, the configured fx, fy, cx, cy, p's trunc and max_depth and k's mask when it has one (masked pixels, moving objects
 *      say, are not baked into the mesh);
 *   3. glic_mesh_count and glic_mesh_extract.
 * A view whose draw overflows the binning workspace grows it and is drawn again, as evaluation does (stats.overflow_regrows
 * counts it); a view that still overflows after four draws fails the call with GLIC_ERR_WORKSPACE.  *out (may be NULL): the
 * vertex and face counts and the number of observed lattice points (weight > 0).  The mesh (xyz, rgb8, faces) stays in the
 * mapper's device memory until the next successful extract_mesh or destroy: glic_mapper_mesh_get copies it out (cudaMemcpyDefault,
 * so host or device memory; any pointer may be NULL; counts = the last call's *out, zeros before any) and glic_mapper_save_mesh
 * writes it with glic_mesh_ply_write (GLIC_ERR_INVALID_ARGUMENT before any extract_mesh).  Memory while the call runs: the grid
 * (20 B per lattice point: 2.7 GB for 512^3) and the extraction scratch, both released when it returns, the render workspace of
 * glic_mapper_render_camera (kept), then the new mesh (15 B per vertex + 12 B per face, kept); the grid, the scratch and the render
 * workspace are reserved before anything runs, and a failed allocation returns GLIC_ERR_CUDA with the previous mesh and the mapper
 * as they were (failure contract above).
 * The map is frozen exactly as under glic_mapper_render_camera; no stats field but overflow_regrows changes.  The call drains the
 * iteration pipeline first and synchronises at the end.  With world > 1 it is rank-local and touches no exchange slot.  A mapper
 * that never calls it allocates and enqueues nothing for it.  Rejected with GLIC_ERR_INVALID_ARGUMENT, changing nothing: a NULL m
 * or p, what glic_tsdf_integrate rejects in the grid, trunc and max_depth, n_views < 0, a view index out of range, a mapper with
 * no non-sky rows. */
typedef struct glic_mesh_params {
    const int* views;              /* host, training keyframe indices; NULL: every training keyframe */
    int n_views;                   /* >= 0; ignored when views is NULL */
    float origin[3];
    float voxel_size;
    int dims[3];
    float trunc;                   /* > 0: the truncation distance, world units */
    float max_depth;               /* > 0: depths beyond it are not fused; 0: no limit */
} glic_mesh_params;
typedef struct glic_mesh_counts {
    uint32_t vertices, faces;
    uint64_t observed_voxels;
} glic_mesh_counts;
GLIC_API int glic_mapper_extract_mesh(glic_mapper* m, const glic_mesh_params* p, glic_mesh_counts* out /* may be NULL */);
GLIC_API int glic_mapper_mesh_get(glic_mapper* m, glic_mesh_counts* counts, float* xyz /*[V,3]*/, uint8_t* rgb /*[V,3]*/,
                                  int32_t* faces /*[F,3]*/);
GLIC_API int glic_mapper_save_mesh(glic_mapper* m, const char* path);

/* ---------------------------------------------------------------------------------------
 * Sparse meshing (no counterpart in the reference): the TSDF of "Meshing" stored only in the 8^3-voxel blocks near some view's
 * observed surface, so a map hundreds of metres long meshes at a few centimetres.  Its mesh equals the dense grid's bit for bit
 * whenever a dense grid of the same origin and voxel size can hold the same blocks (the equivalence below).
 *   Lattice: point (i, j, k), integers in [-2^19, 2^19), at world position __fadd_rn(o.x, __fmul_rn(s, (float)i)) per axis (the
 *   dense grid's formula, with no box).  Block (bi, bj, bk) holds the points with floor(i / 8) = bi (floor division on negatives),
 *   and so on; its key is ((bk + 2^16) << 34) | ((bj + 2^16) << 17) | (bi + 2^16).  A block is allocated or not; every point of an
 *   allocated block takes exactly the per-point update of "Meshing" (steps 1-5); a point of no allocated block is unobserved
 *   (weight 0) and is never read or written.
 *   Allocation rule (the block set of one view): a pixel (px, py) is USED when step 3's tests pass (not masked, d = depth[py][px]
 *   > 0, max_depth == 0 or d <= max_depth).  For a used pixel, in float64, each operation rounded once in the order written: the
 *   8 corners (u, v, z), u in {px, px + 1}, v in {py, py + 1}, z in {d, d + trunc}; camera point c = ((u - cx) z / fx,
 *   (v - cy) z / fy, z); world point X_a = (R_0a (c_0 - t_0) + R_1a (c_1 - t_1)) + R_2a (c_2 - t_2) with R_ra = view[4a + r],
 *   t_r = view[12 + r]; per axis the range [lo, hi] of the 8 X_a; lattice range floor((lo - o) / s) - 2 .. ceil((hi - o) / s) + 2;
 *   every block meeting that range is in the view's set.  Where the range leaves the lattice (or a corner is not finite) the
 *   part outside is dropped and the pixel counts as CLIPPED.  A grid's block set is the union over the views inserted, in any
 *   order.  (The margin of 2: a point gets t < 0 only from a used pixel whose frustum piece z in (d, d + trunc] it lies in;
 *   surface nets reads the +-1 neighbourhood of such points; one voxel covers that, the other rounding.  DESIGN.md.)
 *   Equivalence: insert views V_1..V_n, build the grid, then integrate them in some order; integrate the same views in the same
 *   order into a dense grid of origin o and voxel size s whose box holds every allocated block.  If no pixel was clipped, every
 *   point of every allocated block holds the dense grid's tsdf, weight and colour bit for bit; the meshes (vertices xyz and rgb,
 *   faces) are equal element for element, vertices by ascending (k, j, i) of their cell's lower corner and faces by ascending
 *   (k, j, i, axis) of their lattice edge (the dense orders on any box); and the sparse count of observed points is <= the
 *   dense one (the dense grid also holds free space far from every surface).  Every insertion must come before the grid is
 *   built: a block made after a view was integrated would miss that view's free-space updates.
 *   Block set: glic_block_set, data = DEVICE memory of glic_block_set_bytes(capacity) = 32 + 16 capacity bytes (a hash of 2
 *   capacity key slots), capacity in [1, 2^24] (0 bytes otherwise).  glic_block_set_clear empties it.  glic_block_set_insert
 *   adds one view's blocks (W, H, intrinsics, depth, mask_words, words_per_row, trunc and max_depth as glic_tsdf_integrate takes
 *   them; origin[3] (HOST) and voxel_size as the grid's) and writes counters_host[3] = {blocks in the set, clipped pixels of this
 *   call, overflow} ASYNCHRONOUSLY, as glic_forward writes its counters (valid after a stream synchronise).  The count is exact, and
 *   overflow != 0 exactly when the set's blocks would exceed its capacity; the set then holds part of this view's blocks (and up
 *   to twice its capacity).  glic_block_set_copy(src, dst) rehashes src into dst (another set of at least twice src's capacity,
 *   cleared first), and repeating the insertion into dst gives the set a call that never overflowed gives.
 *   Grid: glic_sparse_tsdf, data = DEVICE memory of glic_sparse_tsdf_bytes(n_blocks) (0 above 2^23 - 1 blocks):
 *   keys[n] u64 ascending | neighbours[27 n] u32 | pool, block b's points at pool + 2560 b, planar tsdf[512] | weight[512] |
 *   colour[3][512], point (x, y, z) of the block at x + 8 y + 64 z: 10 KiB + 116 B per block (the pool region is at least the
 *   sort workspace of n keys, which only matters below a few blocks).  glic_sparse_tsdf_init(grid, set) builds it from the set:
 *   n_blocks must be the set's block count (counters_host[0] of its last insertion); the keys are compacted and sorted with
 *   glic_sort_pairs_u64_u32, block slot = rank of its key (so the layout depends on the set alone), every point is cleared.
 *   glic_sparse_tsdf_integrate takes glic_tsdf_integrate's view arguments, one thread per point of every allocated block.
 *   glic_sparse_mesh_count(grid, scratch, bytes, counts_host, stream): scratch of glic_sparse_mesh_scratch_bytes(n_blocks) (64 B
 *   per block: the active-cell bits), *counts_host (HOST) = vertices, faces, observed points, blocks and the lattice bounding box
 *   of the allocated blocks (inclusive; lo 0 and hi -1 for none); clipped_pixels is 0 there (the mapper fills it).  Synchronises
 *   once.  glic_sparse_mesh_extract(grid, scratch, bytes, counts, ws, ws_bytes, xyz, rgb, faces): counts as counted, ws of
 *   glic_sparse_mesh_extract_bytes(vertices, faces) (32 B per vertex and per quad, plus the sort's temp), fills xyz [V,3] f32,
 *   rgb [V,3] u8 and faces [F,3] i32 asynchronously; the grid must be as it was counted.  Nothing depends on which CTA finishes
 *   first.  glic_debug_sparse_tsdf copies the sorted keys [n] and the pool [n * 2560] (any memory) for tests.
 *   Every call checks its arguments before it enqueues anything: what glic_tsdf_integrate rejects, a NULL set, a capacity out of
 *   range, a copy into a smaller or the same set, a NULL counts pointer or output return GLIC_ERR_INVALID_ARGUMENT; a short
 *   scratch or workspace GLIC_ERR_WORKSPACE.
 * ------------------------------------------------------------------------------------- */
typedef struct glic_block_set {
    uint32_t capacity;             /* blocks it can hold */
    void* data;                    /* device, glic_block_set_bytes(capacity) bytes */
} glic_block_set;
typedef struct glic_sparse_tsdf {
    float origin[3];               /* world position of lattice point (0, 0, 0) */
    float voxel_size;
    uint32_t n_blocks;
    void* data;                    /* device, glic_sparse_tsdf_bytes(n_blocks) bytes */
} glic_sparse_tsdf;
typedef struct glic_sparse_mesh_counts {
    uint32_t vertices, faces;
    uint64_t observed_voxels;
    uint32_t blocks;
    uint32_t clipped_pixels;       /* pixels whose lattice range was clipped (glic_mapper_extract_mesh_sparse; 0 from glic_sparse_mesh_count) */
    int32_t lattice_lo[3], lattice_hi[3];  /* inclusive lattice bounding box of the allocated blocks */
} glic_sparse_mesh_counts;
GLIC_API size_t glic_block_set_bytes(uint32_t capacity);
GLIC_API int glic_block_set_clear(const glic_block_set* set, void* stream);
GLIC_API int glic_block_set_copy(const glic_block_set* src, const glic_block_set* dst, void* stream);
GLIC_API int glic_block_set_insert(const glic_block_set* set, const float* origin /*[3], host*/, float voxel_size, const float* viewmatrix_dev,
                                   int W, int H, float fx, float fy, float cx, float cy, const float* depth,
                                   const uint32_t* mask_words /* may be NULL */, int words_per_row, float trunc, float max_depth,
                                   int64_t* counters_host /*[3]*/, void* stream);
GLIC_API size_t glic_sparse_tsdf_bytes(uint32_t n_blocks);
GLIC_API int glic_sparse_tsdf_init(const glic_sparse_tsdf* grid, const glic_block_set* set, void* stream);
GLIC_API int glic_sparse_tsdf_integrate(const glic_sparse_tsdf* grid, const float* viewmatrix_dev, int W, int H, float fx, float fy, float cx,
                                        float cy, const float* depth, const float* rgb /* may be NULL */,
                                        const uint32_t* mask_words /* may be NULL */, int words_per_row, float trunc, float max_depth,
                                        void* stream);
GLIC_API size_t glic_sparse_mesh_scratch_bytes(uint32_t n_blocks);
GLIC_API size_t glic_sparse_mesh_extract_bytes(uint32_t vertices, uint32_t faces);
GLIC_API int glic_sparse_mesh_count(const glic_sparse_tsdf* grid, void* scratch, size_t scratch_bytes, glic_sparse_mesh_counts* counts_host,
                                    void* stream);
GLIC_API int glic_sparse_mesh_extract(const glic_sparse_tsdf* grid, void* scratch, size_t scratch_bytes, const glic_sparse_mesh_counts* counts,
                                      void* extract_ws, size_t extract_bytes, float* xyz, uint8_t* rgb, int32_t* faces, void* stream);
GLIC_API int glic_debug_sparse_tsdf(const glic_sparse_tsdf* grid, uint64_t* keys, float* data, void* stream);

/* Sparse meshing of the map.  glic_mapper_extract_mesh_sparse(m, p, out) is exactly this composition:
 *   1. pass 1: for each listed training keyframe (p->views as glic_mapper_extract_mesh takes them), draw the map without the sky
 *      exactly as glic_mapper_extract_mesh draws it and glic_block_set_insert its median depth under its mask, with p's origin,
 *      voxel_size, trunc and max_depth; an insertion that overflows grows the set (glic_block_set_copy into twice the capacity)
 *      and is repeated;
 *   2. glic_sparse_tsdf_init a grid of the set's blocks;
 *   3. pass 2: draw every listed view again and glic_sparse_tsdf_integrate its median depth and clamped rgb (the inference draw
 *      is deterministic, so both passes see the same planes);
 *   4. glic_sparse_mesh_count and glic_sparse_mesh_extract.
 * max_blocks > 0 caps the set: a set of more blocks returns GLIC_ERR_WORKSPACE before the grid is allocated, changing nothing;
 * so does a set of more than 2^23 - 1 blocks.
 * *out (may be NULL): vertices, faces, observed points, blocks, the pixels clipped in pass 1 and the lattice bounding box.  On the
 * same map, glic_mapper_extract_mesh with the same views, origin, voxel_size, trunc and max_depth and dims covering that box
 * (lo >= 0) gives the same mesh arrays when nothing was clipped.  Everything else is glic_mapper_extract_mesh's contract: the
 * frozen map, the drain, rank-local, the binning redraw (GLIC_ERR_WORKSPACE after four draws), the failure contract (the grid,
 * scratch and set are this call's own and released when it returns; the pool is allocated after pass 1, once its size is known,
 * and before the map or the previous mesh changes), and the new mesh replaces the last one only once it is complete, so
 * glic_mapper_mesh_get and glic_mapper_save_mesh serve both calls.  A mapper that never calls it allocates and enqueues nothing
 * for it.  Rejected with GLIC_ERR_INVALID_ARGUMENT, changing nothing: what glic_mapper_extract_mesh rejects but dims. */
typedef struct glic_sparse_mesh_params {
    const int* views;              /* host, training keyframe indices; NULL: every training keyframe */
    int n_views;
    float origin[3];               /* the lattice's alignment; there is no box */
    float voxel_size;
    float trunc;
    float max_depth;
    uint32_t max_blocks;           /* 0: no limit */
} glic_sparse_mesh_params;
GLIC_API int glic_mapper_extract_mesh_sparse(glic_mapper* m, const glic_sparse_mesh_params* p, glic_sparse_mesh_counts* out /* may be NULL */);

/* ---------------------------------------------------------------------------------------
 * Pose corrections: moving the map with corrected keyframe poses (loop closure, a smoother's
 * revision, a re-anchored trajectory).
 *
 * Anchors.  Every row of the map carries anchor[i]: the index of a training keyframe, or -1 (the row never moves).  Rows made by
 * the glic_mapper_add_frame hand-off (initialize or extend) take the index of the training keyframe handed off (under
 * glic_mapper_add_frame_masked too: it is the keyframe pushed right after the hand-off); rows of glic_mapper_extend and the LiDAR
 * rows of glic_mapper_initialize_lidar take the newest training keyframe, or -1 when there is none; skybox rows and the rows of
 * glic_mapper_initialize take -1.  Growth keeps the column; every compaction (prune, prune_unseen, densify, densify_and_prune,
 * the density schedule) gathers it with the arenas, so clones and split children take their parent's anchor.  Anchors are not in
 * glic_mapper_save_map's file.  glic_mapper_anchors copies anchor[0 .. P) to host memory; glic_mapper_set_anchors overwrites it
 * from host memory (for maps not built through extend, say a PLY loaded by the caller): every value must be -1 or a training
 * keyframe index in range, otherwise GLIC_ERR_INVALID_ARGUMENT and nothing changes.
 *
 * The correction record of one keyframe, float64, computed on the host from its old and its new pose (R_wc row-major, t_wc, the
 * floats glic_keyframe takes); every operation below rounds once (host code is built without FMA):
 *   R = dR = R_new R_old^T:   R[3i+j] = (R_new[3i] R_old[3j] + R_new[3i+1] R_old[3j+1]) + R_new[3i+2] R_old[3j+2]
 *   t = t_new - dR t_old:     t[i] = t_new[i] - ((R[3i] t_old[0] + R[3i+1] t_old[1]) + R[3i+2] t_old[2])
 *   q = (r, x, y, z), the unit quaternion of dR in the convention of R(q) = [1-2(yy+zz) 2(xy-rz) 2(xz+ry); 2(xy+rz) 1-2(xx+zz)
 *       2(yz-rx); 2(xz-ry) 2(yz+rx) 1-2(xx+yy)] (Hamilton product: R(a (x) b) = R(a) R(b)).  With tr = (R0 + R4) + R8, the first
 *       strictly largest of (tr, R0, R4, R8) picks the branch (a tie goes to the earlier one):
 *         tr: r = sqrt(1 + tr) / 2,           s = 0.25 / r, x = (R7 - R5) s, y = (R2 - R6) s, z = (R3 - R1) s
 *         R0: x = sqrt(((1 + R0) - R4) - R8) / 2, s = 0.25 / x, r = (R7 - R5) s, y = (R1 + R3) s, z = (R2 + R6) s
 *         R4: y = sqrt(((1 - R0) + R4) - R8) / 2, s = 0.25 / y, r = (R2 - R6) s, x = (R1 + R3) s, z = (R5 + R7) s
 *         R8: z = sqrt(((1 - R0) - R4) + R8) / 2, s = 0.25 / z, r = (R3 - R1) s, x = (R2 + R6) s, y = (R5 + R7) s
 *       then q is divided by n = sqrt(((r r + x x) + y y) + z z), and negated when r < 0, or when r == 0 and the first non-zero of
 *       (x, y, z) is negative (r = +0 after the sign rule).
 *   sh = the band rotation matrices of R(q) (glic_sh_rotation(q)): A_1 (3x3) at sh[0], A_2 (5x5) at sh[9], A_3 (7x7) at sh[34],
 *       row-major, in this library's SH-rest order and signs; entries of bands above `degree` are 0.
 * glic_sh_rotation(q, degree, out), the band-matrix builder of the record, is also exported on its own: it gives the matrices of any
 * unit quaternion, so a caller (or a test) can check them, or rotate SH coefficients it holds, without going through two poses.  For a
 * unit q, A_l[m][n] = integral over the unit sphere of b_m(d) b_n(R(q)^T d), so that
 * sum_m (A_l c)_m b_m(d) = sum_n c_n b_n(R(q)^T d) for every unit d and coefficient vector c of band l: the colour a moved splat
 * shows towards R(q) d is the colour it showed towards d.  b_k are the SH-rest basis polynomials of the renderer (degree 1: -c1 y,
 * c1 z, -c1 x, then degree 2 and 3 in the same order) with their constants in float64.  The integral is a product quadrature
 * exact for polynomials of degree <= 7 (4-point Gauss-Legendre in z times 8 equally spaced azimuths), so A_l is exact up to
 * rounding.  It is built from R(q) rather than dR because dR, the product of two float rotations, is orthonormal only to float
 * precision; R(q) is the rotation the row's quaternion gets.
 *
 * glic_mapper_correct_poses(m, n, c, moved): c[0 .. n) each give the corrected pose of one keyframe, training (is_train != 0) or
 * held-out.  Checked before anything changes (GLIC_ERR_INVALID_ARGUMENT, nothing changed): n >= 0, c non-NULL when n > 0, every
 * index in range, every pose a rotation with finite entries (the test of glic_mapper_pose_set), no keyframe listed twice.  n = 0
 * is a no-op.  The call drains the iteration pipeline, then:
 *   1. for every listed training keyframe k, the record from its current given pose (the one last passed to add or to
 *      glic_mapper_pose_set; not a refined pose) to the new one;
 *   2. one pass over rows [0, P): a row whose anchor is a corrected keyframe gets, in float64 with one rounding per operation and
 *      one final rounding to float,
 *        xyz'_i = fl32(((R[3i] x + R[3i+1] y) + R[3i+2] z) + t[i]),
 *        rot' = fl32(q (x) rot) on the stored (unnormalised) quaternion: r' = ((qr rr - qx rx) - qy ry) - qz rz,
 *          x' = ((qr rx + qx rr) + qy rz) - qz ry, y' = ((qr ry - qx rz) + qy rr) + qz rx, z' = ((qr rz + qx ry) - qy rx) + qz rr,
 *        every band l and channel ch of the SH rest (stored [M][3]): c'_m = fl32(sum_n A_l[m][n] c_n), summed from n = 0 up,
 *      and dc, log-scale and opacity unchanged.  Every other row and rows [P, capacity) are not written.  The Adam moments of
 *      every row stay as they are (as under glic_mapper_pose_set);
 *   3. every listed keyframe's given pose becomes the new one.  Without pose refinement (and for held-out keyframes) its camera
 *      block is rebuilt from it, exactly as at glic_mapper_add_keyframe.  With pose refinement a training keyframe's float64 master
 *      becomes T_cw' = T_cw dT^-1 (R_cw' = R_cw dR^T, t_cw' = t_cw - R_cw' t), which keeps the refinement's offset in the
 *      keyframe's own frame, and its float pose and device camera block are re-derived from it by the pose step's code; its Adam
 *      state is kept.
 * *moved (may be NULL): the number of rows written.  Exposure, masks, the densification statistics, contribution scores and the
 * last mesh are left as they are (extract the mesh again).  The update is elementwise, so replicas that make the same call stay
 * bit-identical without an exchange, and deterministic training stays bit-reproducible.  Memory: one table of
 * sizeof(glic_rigid_correction) per training keyframe, released when the call returns; a failed allocation returns GLIC_ERR_CUDA
 * with the mapper as it was.
 * Not covered: computing the corrections, blending several keyframes' corrections per row, moving the skybox, transforming
 * Adam moments, re-seeding scan points still pending from frames not yet handed off, anchors in the PLY.
 * ------------------------------------------------------------------------------------- */
typedef struct glic_rigid_correction {
    double R[9];                   /* dR, row-major */
    double t[3];
    double q[4];                   /* (r, x, y, z), unit, r >= 0 */
    double sh[9 + 25 + 49];        /* A_1 | A_2 | A_3, row-major */
} glic_rigid_correction;
typedef struct glic_pose_correction {
    int is_train;                  /* non-zero: a training keyframe; 0: held-out */
    int index;
    float R_wc[9];                 /* the corrected pose, as glic_keyframe takes it */
    float t_wc[3];
} glic_pose_correction;
GLIC_API int glic_pose_correction_record(const float* R_old /*[9]*/, const float* t_old /*[3]*/, const float* R_new /*[9]*/,
                                         const float* t_new /*[3]*/, int degree, glic_rigid_correction* out);
GLIC_API int glic_sh_rotation(const double* q /*[4], unit*/, int degree, double* out /*[83]*/);
GLIC_API int glic_mapper_anchors(glic_mapper* m, int32_t* out /*[P]*/);
GLIC_API int glic_mapper_set_anchors(glic_mapper* m, const int32_t* in /*[P]*/);
GLIC_API int glic_mapper_correct_poses(glic_mapper* m, int n, const glic_pose_correction* c, uint32_t* moved /* may be NULL */);

/* ---------------------------------------------------------------------------------------
 * Checkpoints: the mapper's whole state in one file, and a new mapper (in a new process, on another machine) that continues
 * from it.
 *
 * Resume: glic_mapper_checkpoint_config(path, &cfg) -> glic_mapper_create(&cfg) -> [glic_mapper_load_lpips, glic_mapper_set_option]
 * -> glic_mapper_load_checkpoint -> (world > 1: glic_mapper_export / glic_mapper_connect) -> carry on.  A restored mapper returns
 * what the saved one returned from every getter, bit for bit, and under GLIC_MAPPER_OPT_DETERMINISTIC it trains on exactly as the
 * saved one would have (same GPU model and library build).  Without the option the restored state is still exact; continued
 * training differs as any two runs do (float atomics).
 *
 * glic_mapper_save_checkpoint(m, path): drains the iteration pipeline (the lagged overflow ring included) and synchronises, then
 * writes the file; it changes nothing in the mapper.  The arrays stream through a pinned staging buffer of two 8 MiB chunks (the
 * device-to-host copy of one, on the copy stream, overlaps the write of the other), so host memory does not grow with the map or
 * the keyframes; float keyframe images in host memory are written from where the caller keeps them.  The file is written as
 * <path>.tmp in the same directory, flushed (fflush, fsync) and renamed over path: on any failure the temporary file is removed and
 * an existing file at path is left as it was.  A connected mapper (world > 1) may save; each rank writes its own file.
 * glic_mapper_checkpoint_config(path, out): host only, no device: the configuration of the fixed header, capacity = the saved arena
 * capacity.  A missing or unreadable file, a short header, a bad magic or version, or a configuration glic_mapper_create would
 * refuse (or a capacity that is not a positive multiple of 256) return GLIC_ERR_INVALID_ARGUMENT.
 * glic_mapper_load_checkpoint(m, path): m must be fresh: created, with no rows (no initialize), no keyframe, no feature enabled
 * (exposure, pose refinement, densification, frames) and not exported; load_lpips and set_option before it are allowed, and the
 * file's options replace them.  The configuration must equal the file's in every field but capacity (floats by their bits); the
 * mapper takes the saved capacity.  The whole file is validated before anything is allocated; GLIC_ERR_INVALID_ARGUMENT, with the
 * mapper still fresh, for: a bad magic or version, a section frame with a non-zero reserved word, a missing, duplicated or unknown
 * section (or one of a feature the counters say is off), a section length that disagrees with its counts, P > capacity, sky rows >
 * P, counts that disagree between sections (rows, keyframes, frames), a truncated file or bytes after the end marker, an
 * out-of-range field, a configuration mismatch, or a mapper that is not fresh.  Every allocation (keyframes, frame store, then the
 * arenas and workspaces at the saved capacity, the binning workspaces at their saved sizes, the deterministic workspace as
 * set_option sizes it) is made before any state is swapped in: a failed one returns GLIC_ERR_CUDA and leaves the mapper fresh, so a
 * second load can succeed.  Float keyframe images keep their memory class in mapper-owned memory (device memory read in place by
 * the loss, or pinned host memory), released by glic_mapper_destroy; 8-bit frames go back into the frame store and the pending scan
 * into the scan buffers.  Synchronises.  With world > 1, rank and world must match the file (they are configuration fields) and
 * the load comes before glic_mapper_export.
 * Not saved: the LPIPS weights (a file the caller has: call glic_mapper_load_lpips again), the last mesh (derived: extract it
 * again), and every workspace's contents (scratch that each call rewrites before reading).
 *
 * The file (version 1, little-endian, no padding; u32 / i32 / u64 / i64 / f32 / f64 are the usual fixed-width types):
 *   header, 96 bytes: u8 magic[8] = "GLICCKPT" | u32 version = 1 | the glic_mapper_config fields in declaration order, one by one:
 *     i32 width, height | f32 fx, fy, cx, cy | i32 sh_degree | f32 position_lr, feature_lr, opacity_lr, scaling_lr, rotation_lr,
 *     lambda_dssim, scaling_scale | u32 capacity (the arena capacity Pcap) | i32 max_iters | u64 seed | i32 rank, world,
 *     views_per_rank
 *   then sections, each: u32 tag (four ASCII bytes) | u32 0 | u64 length (bytes of payload that follow), in any order, each at
 *   most once; then the end marker "END " | 0 | 0, which ends the file.  M = (sh_degree + 1)^2 - 1; P = rows; n = training
 *   keyframes.
 *   "MAP " (always), 12 + P (12 (14 + 3M) + 4) bytes: u32 P, Pcap, n_sky | for each of params, exp_avg, exp_avg_sq: f32 rows
 *     [0, P) of rot [P][4], xyz [P][3], log_scale [P][3], opacity [P], f_dc [P][3], f_rest [P][M][3] | i32 anchor [P]
 *   "CNTR" (always), 92 + L bytes: glic_mapper_stats field by field (u32 num_gaussians, capacity | u64 iterations | u32
 *     last_inserted | f32 last_loss | f64 mean_visible | u32 overflow_regrows | f32 ms_extend, ms_optimize) | u64 view_counter
 *     (images sent through the double buffer) | i64 bin_cap (the binning capacity in pairs: a frame needing more is skipped, so it
 *     changes training) | u64 binning and sample workspace bytes (bin_cap is the largest capacity both hold) | u32 optimizer,
 *     deterministic (GLIC_MAPPER_OPT_* values, 0 or 1) | u32 flags (1 initialized, 2 exposure, 4 pose refinement, 8 densification,
 *     16 frames) | u32 L | u8 [L] the view sampler's std::mt19937_64 as its operator<< writes it (decimal words)
 *   "KEYF" (always): u32 n, n_test | n + n_test records, training then held-out, each: f32 R_wc[9], t_wc[3] | f32 cam[42], the host
 *     camera block (view16 proj16 campos4 tanfovx tanfovy lim4) | f32 cam_dev[36], the device camera block copied back verbatim
 *     (view16 proj16 campos4) | u32 image kind (0: 8-bit add_frame image, 1: float image in host memory, 2: float image in
 *     device memory) | u32 frame (kind 0: its slot in the frame store, in add_frame order; else 0xFFFFFFFF) | u32 mask_valid,
 *     mask_valid_left | the image: kind 0 u8 [H][W][3] BGR, else f32 [3][H][W] | u32 mask words [H][(W + 31) / 32] when mask_valid
 *     > 0 (bit x & 31 of word x >> 5 of a row: pixel x used)
 *   "EXPO" (exposure on), 8 + 148 n bytes: f32 exposure_lr | u32 n | f32 E [n][12], exp_avg [n][12], exp_avg_sq [n][12] | i32
 *     step [n]
 *   "POSE" (pose refinement on), 12 + 196 n bytes: f32 lr_translation, lr_rotation | u32 n | f64 T_cw [n][12] (R_cw row-major |
 *     t_cw) | f32 pose [n][12] (R_wc | t_wc) | f32 exp_avg [n][6], exp_avg_sq [n][6] | i32 step [n]
 *   "DENS" (densification on), 12 + 12 P bytes: u64 densify calls so far | u32 P | f32 grad_accum [P], denom [P] | i32 max screen
 *     radius [P]
 *   "SCHD" (always), 72 bytes: u32 schedule set | glic_density_schedule field by field | glic_density_counts totals field by field
 *     | u32 steps, resets
 *   "FRMS" (frames on), 36 + 19 p bytes: i32 select_every_k_frame, sky_points, sky_radius | glic_frame_stats field by field (u32
 *     frames, train, test, pending_points p | u64 image_bytes) | the pending scan: f32 xyz [p][3] | u8 rgb [p][3] | f32 depth [p]
 * Bytes per row at degree 3: 712 (+ 12 with densification); per keyframe at 1920x1080: 6.22 MB (8-bit) or 24.9 MB (float), plus
 * 259 200 per mask.
 * ------------------------------------------------------------------------------------- */
GLIC_API int glic_mapper_save_checkpoint(glic_mapper* m, const char* path);
GLIC_API int glic_mapper_checkpoint_config(const char* path, glic_mapper_config* out);   /* host only, no device */
GLIC_API int glic_mapper_load_checkpoint(glic_mapper* m, const char* path);

/* ---------------------------------------------------------------------------------------
 * Stage timing (cudaEvent pairs recorded on the launching stream around each stage; off by
 * default).  glic_profile_enable(1) starts recording and resets the accumulators;
 * glic_profile_read() synchronises the recorded events and returns, per stage, the summed
 * milliseconds and the number of recordings since the last enable.  Stage ids: GLIC_STAGE_*.
 * ------------------------------------------------------------------------------------- */
enum {
    GLIC_STAGE_PREPROCESS = 0, GLIC_STAGE_EMIT = 1, GLIC_STAGE_SORT = 2, GLIC_STAGE_RANGES = 3,
    GLIC_STAGE_RENDER_FWD = 4, GLIC_STAGE_LOSS_FWD = 5, GLIC_STAGE_LOSS_BWD = 6, GLIC_STAGE_RENDER_BWD = 7,
    GLIC_STAGE_PREPROCESS_BWD = 8, GLIC_STAGE_ADAM = 9, GLIC_STAGE_ZERO = 10, GLIC_STAGE_ALLREDUCE = 11, GLIC_STAGE_COUNT = 12
};
GLIC_API int glic_profile_enable(int on);
GLIC_API int glic_profile_read(float* ms_host /*[GLIC_STAGE_COUNT]*/, int* count_host /*[GLIC_STAGE_COUNT]*/);

/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
GLIC_API uint64_t glic_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* GLIC_B200_H_INCLUDED */

// mapper_views.cu -- the native mapper's views outside training: test-time alignment of a keyframe (glic_mapper_align) and
// rendering from a caller's camera (glic_mapper_render_camera).
#include "mapper_state.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>

namespace mapper_impl {

bool finite_at_least_zero(float x) { return std::isfinite(x) && x >= 0.0f; }

__global__ void overflow_word_kernel(const GeomHeader* ghdr, float* word) { if (ghdr->overflow) *word = 1.0f; }

// ---- test-time alignment (glic_mapper_align) ------------------------------------------------------------------------------
// The call's one-row state on the device: the pose and exposure being fitted with their Adam states, laid out as
// pose_step_kernel and exposure_adam_kernel index them (keyframe 0 of one-row arrays); the last iteration's gradients, loss and
// overflow word; and the tally of the iterations.
struct AlignState {
    double T[12];                     // float64 T_cw = R_cw (row-major) | t_cw
    float pose_f[12];                 // R_wc | t_wc
    float cam[36];                    // view16 | proj16 | campos4 of pose_f
    float pose_m[6], pose_v[6];
    float E[12], expo_m[12], expo_v[12];
    float pose_grad[8];               // dL/d(rho, omega) (6 used)
    float dE[12];                     // dL/dE
    float loss;                       // fit-region loss
    float overflow;                   // overflow_word_kernel's word: non-zero skips both steps
    int pose_t, expo_t;
    int steps, skipped;
    float first_loss, last_loss;
    unsigned int max_pairs;           // the largest (tile, Gaussian) pair count of a skipped iteration
};

// closes an alignment iteration: counted as stepped (with its loss) or skipped (with its pair count); the word is cleared
__global__ void align_tally_kernel(const GeomHeader* __restrict__ ghdr, AlignState* __restrict__ st) {
    if (st->overflow != 0.0f) {
        ++st->skipped;
        st->max_pairs = max(st->max_pairs, ghdr->total);
    } else {
        if (st->steps == 0) st->first_loss = st->loss;
        st->last_loss = st->loss;
        ++st->steps;
    }
    st->overflow = 0.0f;
}

// dst[3][H][w] = columns [x0, x0 + w) of src[3][H][W]
__global__ void __launch_bounds__(256)
crop_columns_kernel(int H, int W, int x0, int w, const float* __restrict__ src, float* __restrict__ dst) {
    const size_t n = (size_t)3 * H * w;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i / w;
        dst[i] = src[row * W + x0 + (i - row * w)];
    }
}

// dst[3][H][W] = src[3][H][w] in columns [0, w), zero in the others
__global__ void __launch_bounds__(256)
pad_columns_kernel(int H, int W, int w, const float* __restrict__ src, float* __restrict__ dst) {
    const size_t n = (size_t)3 * H * W;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i / W, x = i - row * W;
        dst[i] = x < (size_t)w ? src[row * w + x] : 0.0f;
    }
}

unsigned plane_blocks(size_t n) { return (unsigned)std::min<size_t>((n + 255) / 256, (size_t)NUM_SMS * 8); }

// The workspace of glic_mapper_align: colour gradients [3 Pcap] | pose partials | with split, three planes [3][H][W - W/2]
// (rendered and ground-truth crops, the fit crop's dL/dpixel) | the one-row state
size_t align_carve(void* ws, uint32_t Pcap, int W, int H, bool split, float** col, double** part, float** crops, AlignState** st) {
    Carver c(ws);
    float* a = c.take<float>((size_t)3 * Pcap);
    double* b = c.take<double>(pose_partials_count(Pcap));
    for (int q = 0; q < 3; ++q) {
        float* x = c.take<float>(split ? (size_t)3 * H * (W - W / 2) : 0);
        if (crops) crops[q] = x;
    }
    AlignState* t = c.take<AlignState>(1);
    if (col) *col = a;
    if (part) *part = b;
    if (st) *st = t;
    return c.total();
}

// glic_mapper_align after its checks: reserve, start state, the fit loop (enqueued without a host synchronisation), the
// overflow regrow, the scoring
int align(glic_mapper* m, const Keyframe& kf, bool train, int index, const glic_align_params& p, glic_align_result* out, float* rgb_host) {
    const int W = m->cfg.width, H = m->cfg.height;
    const bool split = p.split != 0;
    const int Wf = split ? W / 2 : W, x_score = split ? W / 2 : 0, Ws = W - x_score;     // fit and score columns
    const bool use_expo = p.exposure_lr > 0.0f || (train && m->expo_on);                  // the loss applies E
    // under the keyframe's mask: the fit loss and both scores are masked, each region read from the mask in place
    MaskView fit_mv, full_mv, score_mv;
    const MaskView* fit_mask = keyframe_mask(kf, W, fit_mv);
    const MaskView* full_mask = keyframe_mask(kf, W, full_mv);
    const MaskView* score_mask = keyframe_mask(kf, W, score_mv, x_score);
    const uint32_t fit_valid = split ? kf.mask_valid_left : kf.mask_valid, score_valid = kf.mask_valid - (split ? kf.mask_valid_left : 0);
    if (kf.mask_valid && (fit_valid == 0 || score_valid == 0)) {
        set_error("mapper_align: the keyframe's mask leaves no valid pixel in the fit or the score columns"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t s = m->stream;
    MAP_TRY(poll_ring(m, true));
    MAP_TRY(reserve(m, m->align_ws, align_carve(nullptr, m->Pcap, W, H, split, nullptr, nullptr, nullptr, nullptr)));
    if (use_expo) MAP_TRY(reserve(m, m->loss_scratch, glic_loss_exposure_scratch_bytes(H, Wf)));
    if (m->lpips_w) MAP_TRY(reserve(m, m->lpips_scratch, glic_lpips_scratch_bytes(H, Ws)));
    float *col = nullptr, *crops[3] = {nullptr, nullptr, nullptr};
    double* part = nullptr;
    AlignState* st = nullptr;
    align_carve(m->align_ws, m->Pcap, W, H, split, &col, &part, crops, &st);
    // start: the stored pose (its camera block is the keyframe's), or a training keyframe's refined one; E = [I | 0], or a
    // training keyframe's trained E; zero moments and step counts
    AlignState h{};
    CamBlock cb;
    config_camera_block(m, kf.R_wc, kf.t_wc, cb, h.T);
    std::memcpy(h.pose_f, kf.R_wc, sizeof(kf.R_wc)); std::memcpy(h.pose_f + 9, kf.t_wc, sizeof(kf.t_wc));
    std::memcpy(h.cam, cb.view, sizeof(h.cam));
    h.E[0] = h.E[5] = h.E[10] = 1.0f;
    h.first_loss = h.last_loss = std::numeric_limits<float>::quiet_NaN();
    GLIC_CUDA_TRY(cudaMemcpyAsync(st, &h, sizeof(h), cudaMemcpyHostToDevice, s));
    if (train && m->pose_on) {
        GLIC_CUDA_TRY(cudaMemcpyAsync(st->T, m->pose_T + 12 * (size_t)index, sizeof(h.T), cudaMemcpyDeviceToDevice, s));
        GLIC_CUDA_TRY(cudaMemcpyAsync(st->pose_f, m->pose_f + 12 * (size_t)index, sizeof(h.pose_f), cudaMemcpyDeviceToDevice, s));
        GLIC_CUDA_TRY(cudaMemcpyAsync(st->cam, kf.cam_dev, sizeof(h.cam), cudaMemcpyDeviceToDevice, s));
    }
    if (train && m->expo_on) GLIC_CUDA_TRY(cudaMemcpyAsync(st->E, m->expo_E + 12 * (size_t)index, sizeof(h.E), cudaMemcpyDeviceToDevice, s));
    const glic_view v = make_view(cb, st->cam, W, H);   // the keyframe's view, drawn from the call's own camera block
    MAP_TRY(load_gt(m, kf, m->gt_dev[0], cudaMemcpyHostToDevice, s));
    const float* gt_fit = m->gt_dev[0];
    if (split) {
        crop_columns_kernel<<<plane_blocks((size_t)3 * H * Wf), 256, 0, s>>>(H, W, 0, Wf, m->gt_dev[0], crops[1]);
        GLIC_LAUNCH_CHECK();
        gt_fit = crops[1];
    }
    MAP_TRY(activate(m));
    PoseBatch b{};
    b.cam[0] = st->cam;
    const int slot_kf[1] = {0};
    const unsigned int* skip = reinterpret_cast<const unsigned int*>(&st->overflow);
    CompactGrads cg{};                              // null row pointers: the pose-only backward
    cg.pose_partials = part;
    cg.pose_grad = st->pose_grad;
    const GeomHeader* ghdr = GeomState::carve(m->geom_ws, (int)m->P).hdr;
    for (int it = 0; it < p.iterations; ++it) {
        MAP_TRY(forward_view(m, v, 0, nullptr));
        overflow_word_kernel<<<1, 1, 0, s>>>(ghdr, &st->overflow);
        GLIC_LAUNCH_CHECK();
        const float* img_fit = m->color;
        float* dL_fit = m->dL_dpix;
        if (split) {
            crop_columns_kernel<<<plane_blocks((size_t)3 * H * Wf), 256, 0, s>>>(H, W, 0, Wf, m->color, crops[0]);
            GLIC_LAUNCH_CHECK();
            img_fit = crops[0];
            dL_fit = crops[2];
        }
        MAP_TRY(photometric_loss(m, H, Wf, img_fit, gt_fit, use_expo ? st->E : nullptr, &st->loss, dL_fit, st->dE, false, fit_mask, fit_valid));
        if (split) {
            pad_columns_kernel<<<plane_blocks((size_t)3 * H * W), 256, 0, s>>>(H, W, Wf, crops[2], m->dL_dpix);
            GLIC_LAUNCH_CHECK();
        }
        MAP_TRY(backward_view(m, v, col, cg, nullptr));
        MAP_TRY(launch_pose_kernel(m, 1, b, st->pose_grad, st->T, st->pose_f, st->pose_m, st->pose_v, &st->pose_t, p.lr_translation,
                                   p.lr_rotation, skip));
        if (p.exposure_lr > 0.0f)
            MAP_TRY(launch_exposure_adam(1, slot_kf, st->dE, st->E, st->expo_m, st->expo_v, &st->expo_t, p.exposure_lr, skip, s));
        align_tally_kernel<<<1, 1, 0, s>>>(ghdr, st);
        GLIC_LAUNCH_CHECK();
    }
    GLIC_CUDA_TRY(cudaMemcpyAsync(&h, st, sizeof(h), cudaMemcpyDeviceToHost, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    if (h.skipped) MAP_TRY(regrow_after_skip(m, h.max_pairs));
    // scoring at the fitted camera: the full clamped (exposed) frame, then with split its score columns
    MAP_TRY(forward_settled(m, v, 0));
    MAP_TRY(eval_psnr_ssim(3, H, W, m->color, m->gt_dev[0], use_expo ? st->E : nullptr, m->eval_out, m->eval_scratch, m->eval_scratch.bytes(), s,
                           m->deterministic ? m->det_sums.raw() : nullptr, full_mask, kf.mask_valid));
    if (rgb_host) MAP_TRY(scored_image_to_host(m, rgb_host));
    if (split) {
        for (int q = 0; q < 2; ++q) {
            crop_columns_kernel<<<plane_blocks((size_t)3 * H * Ws), 256, 0, s>>>(H, W, x_score, Ws, eval_clamped(m->eval_scratch, 3, H, W, q), crops[q]);
            GLIC_LAUNCH_CHECK();
        }
        MAP_TRY(eval_psnr_ssim(3, H, Ws, crops[0], crops[1], nullptr, m->eval_out, m->eval_scratch, m->eval_scratch.bytes(), s,
                               m->deterministic ? m->det_sums.raw() : nullptr, score_mask, score_valid));
    }
    if (m->lpips_w) MAP_TRY(scored_lpips(m, Ws));
    float out3[3] = {0.f, 0.f, std::numeric_limits<float>::quiet_NaN()};
    MAP_TRY(read_eval_out(m, out3, m->lpips_w ? 3 : 2));
    glic_align_result& r = *out;
    std::memcpy(r.R_wc, h.pose_f, sizeof(r.R_wc)); std::memcpy(r.t_wc, h.pose_f + 9, sizeof(r.t_wc));
    std::memcpy(r.E, h.E, sizeof(r.E));
    r.psnr = out3[0]; r.ssim = out3[1]; r.lpips = out3[2];
    r.first_loss = h.first_loss; r.last_loss = h.last_loss;
    std::memcpy(r.pose_exp_avg, h.pose_m, sizeof(r.pose_exp_avg)); std::memcpy(r.pose_exp_avg_sq, h.pose_v, sizeof(r.pose_exp_avg_sq));
    std::memcpy(r.expo_exp_avg, h.expo_m, sizeof(r.expo_exp_avg)); std::memcpy(r.expo_exp_avg_sq, h.expo_v, sizeof(r.expo_exp_avg_sq));
    r.steps = h.steps; r.skipped = h.skipped;
    return GLIC_OK;
}

// The workspace of glic_mapper_render_camera: the camera block (view16 | proj16 | campos4) | an image workspace | glic_render's
// colour, final T, depth and median depth planes | the scored colour
size_t render_carve(void* ws, int W, int H, RenderPlanes* out) {
    const size_t HW = (size_t)W * H;
    Carver c(ws);
    RenderPlanes r;
    r.cam = c.take<float>(36);
    r.image_ws = c.take<char>(glic_image_bytes(W, H));
    r.color = c.take<float>(3 * HW);
    r.T = c.take<float>(HW);
    r.depth = c.take<float>(HW);
    r.median = c.take<float>(HW);
    r.rgb = c.take<float>(3 * HW);
    if (out) *out = r;
    return c.total();
}

// rows [first, P) drawn with glic_render from v into r's colour and final T planes and, where given, depth and median depth; an
// overflow regrows the binning workspace alone (grow_render_binning)
int draw_rows(glic_mapper* m, size_t first, const glic_view& v, const RenderPlanes& r, float* depth, float* median) {
    // the groups are planar: rows [first, P) are the same call on every group pointer offset by `first` rows (rest stays null
    // when M = 0)
    const ArenaRows a = arena_rows(m->params, m->Pcap, m->M);
    return draw_settled(m, [&](long long* cnt) {
        return glic_render((int)(m->P - first), m->D, m->M, a.xyz + 3 * first, m->act_scales + 3 * first, 1.0f, m->act_rots + 4 * first,
                           m->act_opacity + first, a.dc + 3 * first, a.rest + (size_t)3 * m->M * first, &v, m->radii + first, m->geom_ws,
                           m->geom_ws.bytes(), r.image_ws, glic_image_bytes(v.width, v.height), m->binning_ws, m->binning_ws.bytes(), r.color,
                           r.T, depth, median, (int64_t*)cnt, m->stream);
    }, [&](int64_t pairs) { return grow_render_binning(m, pairs); });
}

// glic_mapper_render_camera after its checks: out = rgb, final_T, depth, median_depth (each may be NULL)
int render_camera(glic_mapper* m, const glic_render_camera& c, int exposure_index, int with_sky, float* const out[4]) {
    const int W = c.width, H = c.height;
    const size_t HW = (size_t)W * H;
    cudaStream_t s = m->stream;
    MAP_TRY(poll_ring(m, true));
    MAP_TRY(reserve(m, m->render_ws, render_carve(nullptr, W, H, nullptr)));
    RenderPlanes r;
    render_carve(m->render_ws, W, H, &r);
    CamBlock cb;
    camera_block(W, H, c.fx, c.fy, c.cx, c.cy, c.R_wc, c.t_wc, cb);
    GLIC_CUDA_TRY(cudaMemcpyAsync(r.cam, cb.view, 36 * sizeof(float), cudaMemcpyHostToDevice, s));
    const glic_view v = make_view(cb, r.cam, W, H);
    MAP_TRY(activate(m));
    MAP_TRY(draw_rows(m, with_sky ? 0 : m->n_sky, v, r, out[2] ? r.depth : nullptr, out[3] ? r.median : nullptr));
    if (out[0]) MAP_TRY(launch_scored_image(H, W, r.color, exposure_index >= 0 ? m->expo_E + 12 * (size_t)exposure_index : nullptr, r.rgb, s));
    const float* src[4] = {r.rgb, r.T, r.depth, r.median};
    for (int q = 0; q < 4; ++q)
        if (out[q]) GLIC_CUDA_TRY(cudaMemcpyAsync(out[q], src[q], sizeof(float) * (q ? HW : 3 * HW), cudaMemcpyDefault, s));
    GLIC_CUDA_TRY(cudaStreamSynchronize(s));
    return GLIC_OK;
}

}  // namespace mapper_impl

extern "C" {

int glic_mapper_align(glic_mapper* m, int is_train, int index, const glic_align_params* p, glic_align_result* out, float* rgb_host) {
    if (!m || !p || !out) { set_error("mapper_align: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const Keyframe* kf = nullptr;
    MAP_TRY(keyframe_at(m, is_train, index, "mapper_align", kf));
    if (p->iterations < 0 || !finite_at_least_zero(p->lr_translation) || !finite_at_least_zero(p->lr_rotation) ||
        !finite_at_least_zero(p->exposure_lr) || (p->split != 0 && p->split != 1)) {
        set_error("mapper_align: iterations must be >= 0, the rates finite and >= 0, split 0 or 1"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    const int W = m->cfg.width, H = m->cfg.height, Ws = W - (p->split ? W / 2 : 0);
    if (p->split && W < 2) { set_error("mapper_align: split needs a frame at least 2 columns wide"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (m->lpips_w && !glic_lpips_scratch_bytes(H, Ws)) { set_error("mapper_align: LPIPS needs a score region of at least 31x31"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (m->P == 0) { set_error("mapper_align: the map has no rows to align against"); return GLIC_ERR_INVALID_ARGUMENT; }
    return align(m, *kf, is_train != 0, index, *p, out, rgb_host);
}

int glic_mapper_render_camera(glic_mapper* m, const glic_render_camera* cam, int exposure_index, int with_sky, float* rgb, float* final_T,
                              float* depth, float* median_depth) {
    if (!m || !cam || (!rgb && !final_T && !depth && !median_depth)) { set_error("mapper_render_camera: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const glic_render_camera c = *cam;
    if (c.width < 1 || c.height < 1) { set_error("mapper_render_camera: width and height must be >= 1"); return GLIC_ERR_INVALID_ARGUMENT; }
    const int64_t tiles = (((int64_t)c.width + TILE - 1) / TILE) * (((int64_t)c.height + TILE - 1) / TILE);
    if (tiles > GLIC_MAX_TILES) {
        set_error("mapper_render_camera: " + std::to_string(c.width) + "x" + std::to_string(c.height) + " has " + std::to_string(tiles) +
                  " tiles of 16x16, more than GLIC_MAX_TILES = " + std::to_string(GLIC_MAX_TILES));
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!(std::isfinite(c.fx) && c.fx > 0.0f) || !(std::isfinite(c.fy) && c.fy > 0.0f) || !std::isfinite(c.cx) || !std::isfinite(c.cy)) {
        set_error("mapper_render_camera: fx and fy must be finite and > 0, cx and cy finite"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    MAP_TRY(pose_check(c.R_wc, c.t_wc, "mapper_render_camera"));
    if (exposure_index != -1 && (!m->expo_on || exposure_index < 0 || exposure_index >= (int)m->train.size())) {
        set_error("mapper_render_camera: exposure_index must be -1 or a training keyframe index with exposure enabled"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (with_sky != 0 && with_sky != 1) { set_error("mapper_render_camera: with_sky must be 0 or 1"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (m->P == 0) { set_error("mapper_render_camera: the mapper has no rows"); return GLIC_ERR_INVALID_ARGUMENT; }
    float* const out[4] = {rgb, final_T, depth, median_depth};
    return render_camera(m, c, exposure_index, with_sky, out);
}

}  // extern "C"

// torch_shim.cpp -- the reference's LibTorch operator surface on top of the glic_b200 C ABI.
//
// Exports, with the reference's exact C++ signatures, the six free functions that Gaussian-LIC's
// host code links against (SURVEY.md 8b):
//   RasterizeGaussiansCUDA / RasterizeGaussiansBackwardCUDA / adamUpdate
//       (/root/reference/src/rasterizer/rasterize_points.h:25-96)
//   fusedssim / fusedssim_backward          (/root/reference/src/fused-ssim/ssim.h:7-26)
//   distCUDA2                               (/root/reference/src/simple-knn/spatial.h:14)
// so that the reference's unchanged rasterizer.cpp (autograd Function), loss_utils.h
// (FusedSSIMMap) and optim_utils.h (SparseGaussianAdam) link against this library instead of the
// reference's rasterize_points.cu / ssim.cu / spatial.cu.  Only tensor plumbing lives here: every
// byte of compute happens in libglic_b200.so (hand-written sm_90a CUDA).  There is NO fallback:
// a non-OK status from the C ABI becomes a c10::Error.
#include <torch/extension.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime_api.h>
#include <algorithm>

#include <tuple>

#include "../../include/glic_b200.h"

#define GLIC_SHIM_EXPORT __attribute__((visibility("default")))

namespace {

void* cur_stream() { return static_cast<void*>(c10::cuda::getCurrentCUDAStream().stream()); }

void check(int status, const char* what) {
    TORCH_CHECK(status == GLIC_OK, "glic_b200 ", what, " failed (", status, "): ", glic_last_error());
}

torch::Tensor f32c(const torch::Tensor& t) {
    TORCH_CHECK(t.is_cuda(), "glic_b200: expected a CUDA tensor");
    TORCH_CHECK(t.scalar_type() == torch::kFloat32, "glic_b200: expected a float32 tensor");
    return t.contiguous();
}

struct ViewHold {
    torch::Tensor v, p, c;
    glic_view view;
};

ViewHold make_view(const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const torch::Tensor& campos,
                   float tan_fovx, float tan_fovy, float limx_neg, float limx_pos, float limy_neg, float limy_pos, int H,
                   int W) {
    ViewHold h;
    h.v = f32c(viewmatrix); h.p = f32c(projmatrix); h.c = f32c(campos);
    TORCH_CHECK(h.v.numel() == 16 && h.p.numel() == 16 && h.c.numel() >= 3, "glic_b200: bad camera tensors");
    h.view.viewmatrix = h.v.data_ptr<float>();
    h.view.projmatrix = h.p.data_ptr<float>();
    h.view.campos = h.c.data_ptr<float>();
    h.view.tan_fovx = tan_fovx; h.view.tan_fovy = tan_fovy;
    h.view.limx_neg = limx_neg; h.view.limx_pos = limx_pos; h.view.limy_neg = limy_neg; h.view.limy_pos = limy_pos;
    h.view.width = W; h.view.height = H;
    return h;
}

}  // namespace

// rasterize_points.h:25-50 / rasterize_points.cu:50-149
GLIC_SHIM_EXPORT
std::tuple<int, int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                       const torch::Tensor& opacity, const torch::Tensor& scales, const torch::Tensor& rotations,
                       const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                       const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const int image_height,
                       const int image_width, const float limx_neg, const float limx_pos, const float limy_neg,
                       const float limy_pos, const torch::Tensor& dc, const torch::Tensor& sh, const int degree,
                       const torch::Tensor& campos, const bool prefiltered, const bool debug, const bool no_color) {
    (void)background; (void)colors; (void)cov3D_precomp; (void)prefiltered;   // dead on this path (SURVEY App. C.4)
    if (means3D.ndimension() != 2 || means3D.size(1) != 3) {
        AT_ERROR("means3D must have dimensions (num_points, 3)");
    }
    const int P = means3D.size(0);
    const int H = image_height, W = image_width;
    int M = 0;
    if (sh.size(0) != 0) M = sh.size(1);

    auto fopt = means3D.options().dtype(torch::kFloat32);
    auto iopt = means3D.options().dtype(torch::kInt32);
    auto bopt = means3D.options().dtype(torch::kByte);
    torch::Tensor out_color = P ? torch::empty({3, H, W}, fopt) : torch::zeros({3, H, W}, fopt);
    torch::Tensor out_final_T = P ? torch::empty({H, W}, fopt) : torch::zeros({H, W}, fopt);
    if (P && no_color) out_color.zero_();
    torch::Tensor radii = torch::empty({P}, iopt);
    torch::Tensor geomBuffer = torch::empty({(int64_t)glic_geom_bytes(P)}, bopt);
    torch::Tensor imgBuffer = torch::empty({(int64_t)glic_image_bytes(W, H)}, bopt);
    torch::Tensor binningBuffer = torch::empty({0}, bopt);
    torch::Tensor sampleBuffer = torch::empty({0}, bopt);
    int64_t rendered = 0, buckets = 0;
    if (P != 0) {
        auto m = f32c(means3D), s = f32c(scales), r = f32c(rotations), o = f32c(opacity), d = f32c(dc);
        torch::Tensor shc = M > 0 ? f32c(sh) : torch::Tensor();
        ViewHold vh = make_view(viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, limx_neg, limx_pos, limy_neg, limy_pos, H, W);
        void* st = cur_stream();
        // Two stages split exactly where the reference reads num_rendered back (rasterizer_impl.cu:398): the host waits
        // only for the preprocess kernel (R travels to pinned memory while the GPU already sorts by depth), sizes the
        // binning / sample buffers EXACTLY, enqueues the rest and returns -- the render is still running when the caller
        // starts enqueuing its loss.  num_buckets would need a second wait (rasterizer_impl.cu:446); the backward here
        // reads it from the image header on the device, so the int handed back is the analytic upper bound.
        check(glic_forward_preprocess(P, degree, M, m.data_ptr<float>(), s.data_ptr<float>(), scale_modifier, r.data_ptr<float>(),
                                      o.data_ptr<float>(), d.data_ptr<float>(), M > 0 ? shc.data_ptr<float>() : nullptr, &vh.view,
                                      no_color ? 1 : 0, radii.data_ptr<int>(), geomBuffer.data_ptr(), (size_t)geomBuffer.numel(),
                                      imgBuffer.data_ptr(), (size_t)imgBuffer.numel(), &rendered, st),
              "forward_preprocess");
        binningBuffer = torch::empty({(int64_t)glic_binning_bytes(rendered)}, bopt);
        if (!no_color) sampleBuffer = torch::empty({(int64_t)glic_sample_bytes(rendered, W, H)}, bopt);
        check(glic_forward_render(P, &vh.view, no_color ? 1 : 0, rendered, geomBuffer.data_ptr(), imgBuffer.data_ptr(),
                                  binningBuffer.data_ptr(), (size_t)binningBuffer.numel(), no_color ? nullptr : sampleBuffer.data_ptr(),
                                  (size_t)sampleBuffer.numel(), out_color.data_ptr<float>(), out_final_T.data_ptr<float>(),
                                  /*num_buckets_host=*/nullptr, st),
              "forward_render");
        buckets = no_color ? 0 : glic_max_buckets(rendered, W, H);
    }
    return std::make_tuple((int)rendered, (int)buckets, out_color, out_final_T, radii, geomBuffer, binningBuffer, imgBuffer,
                           sampleBuffer);
}

// rasterize_points.h:52-82 / rasterize_points.cu:151-246
GLIC_SHIM_EXPORT
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBackwardCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
                               const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations,
                               const float scale_modifier, const torch::Tensor& cov3D_precomp,
                               const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                               const float tan_fovy, const float limx_neg, const float limx_pos, const float limy_neg,
                               const float limy_pos, const torch::Tensor& dL_dout_color, const torch::Tensor& dc,
                               const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
                               const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
                               const torch::Tensor& imageBuffer, const int B, const torch::Tensor& sampleBuffer,
                               const float lambda_erank, const bool debug) {
    (void)background; (void)colors; (void)cov3D_precomp; (void)B; (void)debug;
    const int P = means3D.size(0);
    const int H = dL_dout_color.size(1);
    const int W = dL_dout_color.size(2);
    int M = 0;
    if (sh.size(0) != 0) M = sh.size(1);
    auto opt = means3D.options().dtype(torch::kFloat32);
    // every element of every output is written by glic_backward: no zero-fill here
    torch::Tensor dL_dmeans3D = torch::empty({P, 3}, opt);
    torch::Tensor dL_dmeans2D = torch::empty({P, 3}, opt);
    torch::Tensor dL_dcolors = torch::empty({P, 3}, opt);
    torch::Tensor dL_dconic = torch::empty({P, 2, 2}, opt);
    torch::Tensor dL_dopacities = torch::empty({P, 1}, opt);
    torch::Tensor dL_dcov3Ds = torch::empty({P, 6}, opt);
    torch::Tensor dL_ddc = torch::empty({P, 1, 3}, opt);
    torch::Tensor dL_dsh = torch::empty({P, M, 3}, opt);
    torch::Tensor dL_dscales = torch::empty({P, 3}, opt);
    torch::Tensor dL_drotations = torch::empty({P, 4}, opt);
    if (P != 0) {
        auto m = f32c(means3D), s = f32c(scales), r = f32c(rotations), d = f32c(dc), g = f32c(dL_dout_color);
        torch::Tensor shc = M > 0 ? f32c(sh) : torch::Tensor();
        auto rad = radii.contiguous();
        auto gb = geomBuffer.contiguous(), bb = binningBuffer.contiguous(), ib = imageBuffer.contiguous(), sb = sampleBuffer.contiguous();
        ViewHold vh = make_view(viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, limx_neg, limx_pos, limy_neg, limy_pos, H, W);
        // R is the exact num_rendered the forward carved its workspaces with (ctx round trip, rasterizer.cpp)
        const int64_t cap = R;
        if (at::globalContext().deterministicAlgorithms()) {
            // torch.use_deterministic_algorithms(True): the fixed-order render backward, its workspace from the caching allocator
            torch::Tensor det = torch::empty({(int64_t)glic_deterministic_bytes(cap, W, H)}, means3D.options().dtype(torch::kByte));
            check(glic_backward_deterministic(P, degree, M, m.data_ptr<float>(), s.data_ptr<float>(), scale_modifier, r.data_ptr<float>(),
                                              d.data_ptr<float>(), M > 0 ? shc.data_ptr<float>() : nullptr, &vh.view, rad.data_ptr<int>(),
                                              cap, gb.data_ptr(), bb.data_ptr(), ib.data_ptr(), sb.data_ptr(), g.data_ptr<float>(),
                                              lambda_erank, dL_dmeans2D.data_ptr<float>(), dL_dconic.data_ptr<float>(),
                                              dL_dopacities.data_ptr<float>(), dL_dcolors.data_ptr<float>(), dL_dmeans3D.data_ptr<float>(),
                                              dL_dcov3Ds.data_ptr<float>(), dL_ddc.data_ptr<float>(), M > 0 ? dL_dsh.data_ptr<float>() : nullptr,
                                              dL_dscales.data_ptr<float>(), dL_drotations.data_ptr<float>(), det.data_ptr(),
                                              (size_t)det.numel(), cur_stream()),
                  "backward_deterministic");
        } else {
            check(glic_backward(P, degree, M, m.data_ptr<float>(), s.data_ptr<float>(), scale_modifier, r.data_ptr<float>(),
                                d.data_ptr<float>(), M > 0 ? shc.data_ptr<float>() : nullptr, &vh.view, rad.data_ptr<int>(),
                                cap, gb.data_ptr(), bb.data_ptr(), ib.data_ptr(), sb.data_ptr(), g.data_ptr<float>(), lambda_erank,
                                dL_dmeans2D.data_ptr<float>(), dL_dconic.data_ptr<float>(), dL_dopacities.data_ptr<float>(),
                                dL_dcolors.data_ptr<float>(), dL_dmeans3D.data_ptr<float>(), dL_dcov3Ds.data_ptr<float>(),
                                dL_ddc.data_ptr<float>(), M > 0 ? dL_dsh.data_ptr<float>() : nullptr,
                                dL_dscales.data_ptr<float>(), dL_drotations.data_ptr<float>(), cur_stream()),
                  "backward");
        }
    }
    return std::make_tuple(dL_dmeans2D, dL_dcolors, dL_dopacities, dL_dmeans3D, dL_dcov3Ds, dL_ddc, dL_dsh, dL_dscales,
                           dL_drotations);
}

// rasterize_points.h:84-96 / rasterize_points.cu:248-273
GLIC_SHIM_EXPORT
void adamUpdate(torch::Tensor& param, torch::Tensor& param_grad, torch::Tensor& exp_avg, torch::Tensor& exp_avg_sq,
                torch::Tensor& visible, const float lr, const float b1, const float b2, const float eps, const uint32_t N,
                const uint32_t M) {
    TORCH_CHECK(param.is_contiguous() && exp_avg.is_contiguous() && exp_avg_sq.is_contiguous(),
                "glic_b200 adamUpdate: param / exp_avg / exp_avg_sq must be contiguous (updated in place)");
    auto g = f32c(param_grad);
    auto vis = visible.contiguous();
    TORCH_CHECK(vis.scalar_type() == torch::kBool || vis.scalar_type() == torch::kByte, "glic_b200 adamUpdate: visible must be bool");
    check(glic_adam_update(param.data_ptr<float>(), g.data_ptr<float>(), exp_avg.data_ptr<float>(),
                           exp_avg_sq.data_ptr<float>(), static_cast<const uint8_t*>(vis.data_ptr()), lr, b1, b2, eps, N, M,
                           cur_stream()),
          "adam_update");
}

// fused-ssim/ssim.h:7-14 / ssim.cu:367-402
GLIC_SHIM_EXPORT
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
fusedssim(float C1, float C2, torch::Tensor& img1, torch::Tensor& img2, bool train) {
    const int B = img1.size(0), CH = img1.size(1), H = img1.size(2), W = img1.size(3);
    auto a = f32c(img1), b = f32c(img2);
    torch::Tensor target = torch::empty_like(a);
    torch::Tensor dm_dmu1 = train ? torch::empty_like(a) : torch::empty({0}, a.options());
    torch::Tensor dm_dsigma1_sq = train ? torch::empty_like(a) : torch::empty({0}, a.options());
    torch::Tensor dm_dsigma12 = train ? torch::empty_like(a) : torch::empty({0}, a.options());
    check(glic_fused_ssim(B, CH, H, W, C1, C2, a.data_ptr<float>(), b.data_ptr<float>(), target.data_ptr<float>(),
                          train ? dm_dmu1.data_ptr<float>() : nullptr, train ? dm_dsigma1_sq.data_ptr<float>() : nullptr,
                          train ? dm_dsigma12.data_ptr<float>() : nullptr, cur_stream()),
          "fused_ssim");
    return std::make_tuple(target, dm_dmu1, dm_dsigma1_sq, dm_dsigma12);
}

// fused-ssim/ssim.h:16-26 / ssim.cu:404-441
GLIC_SHIM_EXPORT
torch::Tensor fusedssim_backward(float C1, float C2, torch::Tensor& img1, torch::Tensor& img2, torch::Tensor& dL_dmap,
                                 torch::Tensor& dm_dmu1, torch::Tensor& dm_dsigma1_sq, torch::Tensor& dm_dsigma12) {
    const int B = img1.size(0), CH = img1.size(1), H = img1.size(2), W = img1.size(3);
    auto a = f32c(img1), b = f32c(img2), g = f32c(dL_dmap), d1 = f32c(dm_dmu1), d2 = f32c(dm_dsigma1_sq), d3 = f32c(dm_dsigma12);
    torch::Tensor out = torch::empty_like(a);
    check(glic_fused_ssim_backward(B, CH, H, W, C1, C2, a.data_ptr<float>(), b.data_ptr<float>(), g.data_ptr<float>(),
                                   d1.data_ptr<float>(), d2.data_ptr<float>(), d3.data_ptr<float>(), out.data_ptr<float>(),
                                   cur_stream()),
          "fused_ssim_backward");
    return out;
}

// simple-knn/spatial.h:14 / spatial.cu:15-26
GLIC_SHIM_EXPORT
torch::Tensor distCUDA2(const torch::Tensor& points) {
    const int P = points.size(0);
    auto p = f32c(points);
    torch::Tensor means = torch::zeros({P}, p.options());
    if (P > 0) {
        torch::Tensor temp = torch::empty({(int64_t)glic_knn_temp_bytes(P)}, p.options().dtype(torch::kByte));
        check(glic_knn_mean_dist2(P, p.data_ptr<float>(), means.data_ptr<float>(), temp.data_ptr(), (size_t)temp.numel(),
                                  cur_stream()),
              "knn_mean_dist2");
    }
    return means;
}

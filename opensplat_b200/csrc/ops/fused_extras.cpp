// fused_extras.cpp -- see fused_extras.hpp.  Thin libtorch wrappers over the C ABI (gsb_ssim_l1_loss, gsb_adam_step,
// gsb_densify_stats_*); Python has the same through opensplat_b200/ops.py and model.py.
#include "fused_extras.hpp"

#include <cmath>

#include "gsb_torch.hpp"

namespace gsb {

torch::Tensor MainLoss::forward(torch::autograd::AutogradContext *ctx, torch::Tensor rgb, torch::Tensor gt,
                                double ssimWeight) {
    TORCH_CHECK(rgb.dim() == 3 && rgb.size(2) == 3 && rgb.sizes() == gt.sizes(), "rgb and gt must be [H,W,3]");
    c10::cuda::CUDAGuard guard(rgb.device());
    const int H = (int)rgb.size(0), W = (int)rgb.size(1);
    torch::Tensor r = f32(rgb), g = f32(gt);
    torch::Tensor v = torch::empty_like(r);
    torch::Tensor out = torch::empty({3}, like(r, torch::kFloat32));
    const size_t wsBytes = gsb_ssim_workspace_bytes(H, W);
    torch::Tensor ws = torch::empty({(int64_t)wsBytes + 256}, like(r, torch::kUInt8));
    uint8_t *wp = ws.data_ptr<uint8_t>();
    const size_t off = (256 - ((uintptr_t)wp % 256)) % 256;
    check(gsb_ssim_l1_loss(H, W, fp(r), fp(g), (float)ssimWeight, fpw(v), fpw(out), wp + off, wsBytes, stream()),
          "gsb_ssim_l1_loss");
    ctx->save_for_backward({v});
    return out[0].clone();
}

torch::autograd::tensor_list MainLoss::backward(torch::autograd::AutogradContext *ctx,
                                                torch::autograd::tensor_list grad_outputs) {
    torch::Tensor v = ctx->get_saved_variables()[0];
    return {v * grad_outputs[0], torch::Tensor(), torch::Tensor()};
}

namespace {
int degFromBases(int64_t k) {   // spherical_harmonics.cpp:3-16
    switch (k) {
        case 1: return 0;
        case 4: return 1;
        case 9: return 2;
        case 16: return 3;
        default: return 4;
    }
}
torch::Tensor orZeros(const torch::Tensor &g, const torch::Tensor &like_) {
    return g.defined() ? f32(g) : torch::zeros_like(like_);
}
}  // namespace

torch::autograd::tensor_list ActivateGaussians::forward(torch::autograd::AutogradContext *ctx, torch::Tensor means,
                                                        torch::Tensor logScales, torch::Tensor rawQuats,
                                                        torch::Tensor opacityLogits, torch::Tensor camPos) {
    c10::cuda::CUDAGuard guard(means.device());
    const int n = (int)means.size(0);
    torch::Tensor m = f32(means), ls = f32(logScales), rq = f32(rawQuats), ol = f32(opacityLogits).reshape({-1});
    torch::Tensor cp = camPos.to(means.device(), torch::kFloat32).reshape({3}).contiguous();
    torch::Tensor scales = torch::empty_like(ls), quats = torch::empty_like(rq);
    torch::Tensor opac = torch::empty({n, 1}, like(m, torch::kFloat32)), vd = torch::empty_like(m);
    check(gsb_activate_forward(n, fp(m), fp(ls), fp(rq), fp(ol), fp(cp), fpw(scales), fpw(quats), fpw(opac), fpw(vd),
                               stream()),
          "gsb_activate_forward");
    ctx->save_for_backward({scales, rq, opac});
    ctx->mark_non_differentiable({vd});
    return {scales, quats, opac, vd};
}

torch::autograd::tensor_list ActivateGaussians::backward(torch::autograd::AutogradContext *ctx,
                                                         torch::autograd::tensor_list g) {
    auto saved = ctx->get_saved_variables();
    torch::Tensor scales = saved[0], rq = saved[1], opac = saved[2];
    c10::cuda::CUDAGuard guard(scales.device());
    const int n = (int)scales.size(0);
    torch::Tensor vS = orZeros(g[0], scales), vQ = orZeros(g[1], rq), vO = orZeros(g[2], opac);
    torch::Tensor vLs = torch::empty_like(scales), vRq = torch::empty_like(rq), vOl = torch::empty_like(opac);
    check(gsb_activate_backward(n, fp(scales), fp(rq), fp(opac), fp(vS), fp(vQ), fp(vO), fpw(vLs), fpw(vRq), fpw(vOl),
                                stream()),
          "gsb_activate_backward");
    return {torch::Tensor(), vLs, vRq, vOl, torch::Tensor()};
}

torch::Tensor SphericalHarmonicsRgb::forward(torch::autograd::AutogradContext *ctx, int64_t degreesToUse,
                                             torch::Tensor means, torch::Tensor camPos, torch::Tensor featuresDc,
                                             torch::Tensor featuresRest) {
    c10::cuda::CUDAGuard guard(means.device());
    const int n = (int)means.size(0);
    const int degree = degFromBases(featuresRest.size(-2) + 1);
    TORCH_CHECK(featuresDc.dim() == 2 && featuresDc.size(1) == 3 && featuresRest.dim() == 3 &&
                    featuresRest.size(2) == 3 && featuresRest.size(0) == n,
                "SphericalHarmonicsRgb: featuresDc [N,3], featuresRest [N,K-1,3]");
    TORCH_CHECK(degreesToUse >= 0 && degreesToUse <= degree, "SphericalHarmonicsRgb: degreesToUse out of range");
    torch::Tensor m = f32(means), dc = f32(featuresDc), rest = f32(featuresRest);
    torch::Tensor cp = camPos.to(means.device(), torch::kFloat32).reshape({3}).contiguous();
    torch::Tensor rgbs = torch::empty({n, 3}, like(m, torch::kFloat32));
    check(gsb_sh_forward_split(n, degree, (int)degreesToUse, fp(m), fp(cp), fp(dc), fp(rest), 0.5f, fpw(rgbs),
                               stream()),
          "gsb_sh_forward_split");
    ctx->saved_data["degreesToUse"] = degreesToUse;
    ctx->saved_data["degree"] = (int64_t)degree;
    ctx->saved_data["restBases"] = featuresRest.size(-2);
    ctx->save_for_backward({m, cp, rgbs});
    return rgbs;
}

torch::autograd::tensor_list SphericalHarmonicsRgb::backward(torch::autograd::AutogradContext *ctx,
                                                             torch::autograd::tensor_list g) {
    auto saved = ctx->get_saved_variables();
    torch::Tensor m = saved[0], cp = saved[1], rgbs = saved[2];
    c10::cuda::CUDAGuard guard(m.device());
    const int n = (int)m.size(0);
    const int degree = (int)ctx->saved_data["degree"].toInt();
    torch::Tensor v = f32(g[0]);
    torch::Tensor vDc = torch::empty({n, 3}, like(m, torch::kFloat32));
    torch::Tensor vRest = torch::empty({n, ctx->saved_data["restBases"].toInt(), 3}, like(m, torch::kFloat32));
    check(gsb_sh_backward_split(n, degree, (int)ctx->saved_data["degreesToUse"].toInt(), fp(m), fp(cp), fp(rgbs), fp(v),
                                fpw(vDc), fpw(vRest), stream()),
          "gsb_sh_backward_split");
    return {torch::Tensor(), torch::Tensor(), torch::Tensor(), vDc, vRest};
}

// The body of ProjectGaussiansActivated[Antialiased]: `aa` picks the anti-aliased kernels (DESIGN D19), whose backward
// takes the opacity logits where the plain one takes the saved sigmoid.
static torch::autograd::variable_list projectActivatedForward(
    torch::autograd::AutogradContext *ctx, bool aa, torch::Tensor means, torch::Tensor logScales, double globScale,
    torch::Tensor rawQuats, torch::Tensor opacityLogits, torch::Tensor viewMat, torch::Tensor projMat, double fx,
    double fy, double cx, double cy, int64_t imgHeight, int64_t imgWidth, std::tuple<int, int, int> tileBounds,
    double clipThresh) {
    const int n = (int)means.size(0);
    c10::cuda::CUDAGuard guard(means.device());
    TORCH_CHECK(opacityLogits.numel() == n, "ProjectGaussiansActivated: opacityLogits must hold one value per Gaussian");
    torch::Tensor m = f32(means), ls = f32(logScales), rq = f32(rawQuats), ol = f32(opacityLogits).reshape({-1});
    torch::Tensor V = f32(viewMat), P = f32(projMat);
    torch::Tensor cov3d = torch::empty({n, 6}, like(m, torch::kFloat32));
    torch::Tensor xys = torch::empty({n, 2}, like(m, torch::kFloat32));
    torch::Tensor depths = torch::empty({n}, like(m, torch::kFloat32));
    torch::Tensor radii = torch::empty({n}, like(m, torch::kInt32));
    torch::Tensor conics = torch::empty({n, 3}, like(m, torch::kFloat32));
    torch::Tensor numTilesHit = torch::empty({n}, like(m, torch::kInt32));
    torch::Tensor opac = torch::empty({n, 1}, like(m, torch::kFloat32));
    check((aa ? gsb_project_forward_activated_aa : gsb_project_forward_activated)(
              n, fp(m), fp(ls), (float)globScale, fp(rq), fp(ol), fp(V), fp(P), (float)fx, (float)fy, (float)cx,
              (float)cy, (int)imgHeight, (int)imgWidth, std::get<0>(tileBounds), std::get<1>(tileBounds),
              (float)clipThresh, fpw(cov3d), fpw(xys), fpw(depths), radii.data_ptr<int32_t>(), fpw(conics),
              numTilesHit.data_ptr<int32_t>(), fpw(opac), stream()),
          aa ? "gsb_project_forward_activated_aa" : "gsb_project_forward_activated");
    ctx->saved_data["imgHeight"] = imgHeight;
    ctx->saved_data["imgWidth"] = imgWidth;
    ctx->saved_data["globScale"] = globScale;
    ctx->saved_data["fx"] = fx;
    ctx->saved_data["fy"] = fy;
    ctx->saved_data["logitSizes"] = opacityLogits.sizes().vec();
    ctx->saved_data["aa"] = aa;
    ctx->save_for_backward({m, ls, rq, V, P, radii, conics, aa ? ol : opac});
    ctx->mark_non_differentiable({radii, numTilesHit});
    return {xys, depths, radii, conics, numTilesHit, cov3d, opac};
}

static torch::autograd::tensor_list projectActivatedBackward(torch::autograd::AutogradContext *ctx,
                                                             torch::autograd::tensor_list g) {
    auto saved = ctx->get_saved_variables();
    torch::Tensor m = saved[0], ls = saved[1], rq = saved[2], V = saved[3], P = saved[4];
    torch::Tensor radii = saved[5], conics = saved[6], opac = saved[7];   // opac: the logits when aa
    const bool aa = ctx->saved_data["aa"].toBool();
    const int n = (int)m.size(0);
    c10::cuda::CUDAGuard guard(m.device());
    // cotangents of xys (0), depths (1), conics (3), opacities (6); undefined == zeros
    torch::Tensor v_xy = g[0].defined() ? f32(g[0]) : torch::zeros({n, 2}, like(m, torch::kFloat32));
    torch::Tensor v_depth = g[1].defined() ? f32(g[1]) : torch::Tensor();
    torch::Tensor v_conic = g[3].defined() ? f32(g[3]) : torch::zeros({n, 3}, like(m, torch::kFloat32));
    torch::Tensor v_opac = g[6].defined() ? f32(g[6]) : torch::Tensor();
    torch::Tensor v_mean = torch::empty({n, 3}, like(m, torch::kFloat32));
    torch::Tensor v_ls = torch::empty({n, 3}, like(m, torch::kFloat32));
    torch::Tensor v_rq = torch::empty({n, 4}, like(m, torch::kFloat32));
    torch::Tensor v_ol = torch::empty({n}, like(m, torch::kFloat32));
    check((aa ? gsb_project_backward_activated_aa : gsb_project_backward_activated)(
              n, fp(m), fp(ls), (float)ctx->saved_data["globScale"].toDouble(), fp(rq), fp(opac), fp(V), fp(P),
              (float)ctx->saved_data["fx"].toDouble(), (float)ctx->saved_data["fy"].toDouble(),
              (int)ctx->saved_data["imgHeight"].toInt(), (int)ctx->saved_data["imgWidth"].toInt(),
              radii.data_ptr<int32_t>(), fp(conics), fp(v_xy), v_depth.defined() ? fp(v_depth) : nullptr, fp(v_conic),
              v_opac.defined() ? fp(v_opac) : nullptr, fpw(v_mean), fpw(v_ls), fpw(v_rq), fpw(v_ol), stream()),
          aa ? "gsb_project_backward_activated_aa" : "gsb_project_backward_activated");
    torch::Tensor none;
    return {v_mean, v_ls, none, v_rq, v_ol.reshape(ctx->saved_data["logitSizes"].toIntVector()),
            none, none, none, none, none, none, none, none, none, none};
}

torch::autograd::variable_list ProjectGaussiansActivated::forward(
    torch::autograd::AutogradContext *ctx, torch::Tensor means, torch::Tensor logScales, double globScale,
    torch::Tensor rawQuats, torch::Tensor opacityLogits, torch::Tensor viewMat, torch::Tensor projMat, double fx,
    double fy, double cx, double cy, int64_t imgHeight, int64_t imgWidth, std::tuple<int, int, int> tileBounds,
    double clipThresh) {
    return projectActivatedForward(ctx, false, means, logScales, globScale, rawQuats, opacityLogits, viewMat, projMat,
                                   fx, fy, cx, cy, imgHeight, imgWidth, tileBounds, clipThresh);
}

torch::autograd::tensor_list ProjectGaussiansActivated::backward(torch::autograd::AutogradContext *ctx,
                                                                 torch::autograd::tensor_list g) {
    return projectActivatedBackward(ctx, g);
}

torch::autograd::variable_list ProjectGaussiansActivatedAntialiased::forward(
    torch::autograd::AutogradContext *ctx, torch::Tensor means, torch::Tensor logScales, double globScale,
    torch::Tensor rawQuats, torch::Tensor opacityLogits, torch::Tensor viewMat, torch::Tensor projMat, double fx,
    double fy, double cx, double cy, int64_t imgHeight, int64_t imgWidth, std::tuple<int, int, int> tileBounds,
    double clipThresh) {
    return projectActivatedForward(ctx, true, means, logScales, globScale, rawQuats, opacityLogits, viewMat, projMat,
                                   fx, fy, cx, cy, imgHeight, imgWidth, tileBounds, clipThresh);
}

torch::autograd::tensor_list ProjectGaussiansActivatedAntialiased::backward(torch::autograd::AutogradContext *ctx,
                                                                            torch::autograd::tensor_list g) {
    return projectActivatedBackward(ctx, g);
}

torch::Tensor RasterizeGaussiansClamped::forward(torch::autograd::AutogradContext *ctx, torch::Tensor xys,
                                                 torch::Tensor depths, torch::Tensor radii, torch::Tensor conics,
                                                 torch::Tensor numTilesHit, torch::Tensor colors,
                                                 torch::Tensor opacity, int imgHeight, int imgWidth,
                                                 torch::Tensor background) {
    return rasterizeForward(ctx, GSB_RASTER_CLAMP_MAX_ONE, xys, depths, radii, conics, numTilesHit, colors, opacity,
                            imgHeight, imgWidth, background);
}

torch::autograd::tensor_list RasterizeGaussiansClamped::backward(torch::autograd::AutogradContext *ctx,
                                                                 torch::autograd::tensor_list grad_outputs) {
    return rasterizeBackward(ctx, grad_outputs);
}

torch::autograd::variable_list RasterizeGaussiansDepth::forward(torch::autograd::AutogradContext *ctx,
                                                                torch::Tensor xys, torch::Tensor depths,
                                                                torch::Tensor radii, torch::Tensor conics,
                                                                torch::Tensor numTilesHit, torch::Tensor colors,
                                                                torch::Tensor opacity, int imgHeight, int imgWidth,
                                                                torch::Tensor background) {
    DepthMaps maps;
    torch::Tensor rgb = rasterizeForward(ctx, 0u, xys, depths, radii, conics, numTilesHit, colors, opacity, imgHeight,
                                         imgWidth, background, &maps);
    return {rgb, maps.depth, maps.alpha};
}

torch::autograd::tensor_list RasterizeGaussiansDepth::backward(torch::autograd::AutogradContext *ctx,
                                                               torch::autograd::tensor_list grad_outputs) {
    return rasterizeBackward(ctx, grad_outputs);
}

torch::autograd::variable_list RasterizeGaussiansDepthClamped::forward(
    torch::autograd::AutogradContext *ctx, torch::Tensor xys, torch::Tensor depths, torch::Tensor radii,
    torch::Tensor conics, torch::Tensor numTilesHit, torch::Tensor colors, torch::Tensor opacity, int imgHeight,
    int imgWidth, torch::Tensor background) {
    DepthMaps maps;
    torch::Tensor rgb = rasterizeForward(ctx, GSB_RASTER_CLAMP_MAX_ONE, xys, depths, radii, conics, numTilesHit,
                                         colors, opacity, imgHeight, imgWidth, background, &maps);
    return {rgb, maps.depth, maps.alpha};
}

torch::autograd::tensor_list RasterizeGaussiansDepthClamped::backward(torch::autograd::AutogradContext *ctx,
                                                                      torch::autograd::tensor_list grad_outputs) {
    return rasterizeBackward(ctx, grad_outputs);
}

ModelForwardResult modelForward(const torch::Tensor &means, const torch::Tensor &logScales,
                                const torch::Tensor &rawQuats, const torch::Tensor &featuresDc,
                                const torch::Tensor &featuresRest, const torch::Tensor &opacityLogits,
                                const torch::Tensor &backgroundColor, const torch::Tensor &camToWorld, float fx,
                                float fy, float cx, float cy, int height, int width, int degreesToUse) {
    TORCH_CHECK(camToWorld.dim() == 2 && camToWorld.size(0) >= 3 && camToWorld.size(1) == 4,
                "modelForward: camToWorld must be [3|4, 4]");
    c10::cuda::CUDAGuard guard(means.device());
    // host side of model.cpp:92-113: R = c2w[:3,:3] diag(1,-1,-1) (gsplat's axis convention), worldToCam = [R^T | -R^T T],
    // OpenGL-style projection from the fields of view, projMat @ viewMat; plus the camera centre for the SH pass
    torch::Tensor c2w = camToWorld.to(torch::kCPU, torch::kFloat32).contiguous();
    auto a = c2w.accessor<float, 2>();
    const float flip[3] = {1.f, -1.f, -1.f};
    float V[4][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 1}};
    for (int i = 0; i < 3; ++i) {
        float t = 0.f;
        for (int j = 0; j < 3; ++j) {
            V[i][j] = a[j][i] * flip[i];                  // (R^T)[i][j] = R[j][i] = c2w[j][i] * flip[i]
            t += -V[i][j] * a[j][3];
        }
        V[i][3] = t;
    }
    const float zNear = 0.001f, zFar = 1000.0f;
    const float fovX = 2.0f * std::atan(width / (2.0f * fx)), fovY = 2.0f * std::atan(height / (2.0f * fy));
    const float top = zNear * std::tan(0.5f * fovY), right = zNear * std::tan(0.5f * fovX);
    const float P[4][4] = {{2.0f * zNear / (2.0f * right), 0.f, 0.f, 0.f},
                           {0.f, 2.0f * zNear / (2.0f * top), 0.f, 0.f},
                           {0.f, 0.f, (zFar + zNear) / (zFar - zNear), -1.0f * zFar * zNear / (zFar - zNear)},
                           {0.f, 0.f, 1.f, 0.f}};
    torch::Tensor host = torch::empty({35}, torch::TensorOptions().dtype(torch::kFloat32));
    float *h = host.data_ptr<float>();
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            h[4 * i + j] = V[i][j];
            float acc = 0.f;
            for (int k = 0; k < 4; ++k) acc += P[i][k] * V[k][j];
            h[16 + 4 * i + j] = acc;
        }
    for (int i = 0; i < 3; ++i) h[32 + i] = a[i][3];
    torch::Tensor devBuf = host.to(means.device());
    torch::Tensor viewMat = devBuf.slice(0, 0, 16).view({4, 4}), fullProj = devBuf.slice(0, 16, 32).view({4, 4});
    torch::Tensor camPos = devBuf.slice(0, 32, 35);

    const std::tuple<int, int, int> tileBounds = std::make_tuple((width + 15) / 16, (height + 15) / 16, 1);
    auto p = ProjectGaussiansActivated::apply(means, logScales, 1.0, rawQuats, opacityLogits, viewMat, fullProj,
                                              (double)fx, (double)fy, (double)cx, (double)cy, (int64_t)height,
                                              (int64_t)width, tileBounds, 0.01);
    ModelForwardResult r;
    r.xys = p[0];
    r.radii = p[2];
    r.xys.retain_grad();
    if (r.radii.sum().item<float>() == 0.0f) {       // model.cpp:173-174
        r.rgb = backgroundColor.repeat({height, width, 1});
        return r;
    }
    torch::Tensor rgbs = SphericalHarmonicsRgb::apply((int64_t)degreesToUse, means.detach(), camPos, featuresDc,
                                                      featuresRest);
    r.rgb = RasterizeGaussiansClamped::apply(p[0], p[1], p[2], p[3], p[4], rgbs, p[6], height, width, backgroundColor);
    return r;
}

void adamStep(torch::Tensor param, const torch::Tensor &grad, torch::Tensor expAvg, torch::Tensor expAvgSq, double lr,
              int64_t step, double beta1, double beta2, double eps) {
    TORCH_CHECK(param.is_cuda() && param.is_contiguous() && param.scalar_type() == torch::kFloat32,
                "adamStep: param must be a contiguous fp32 CUDA tensor");
    TORCH_CHECK(expAvg.is_contiguous() && expAvgSq.is_contiguous() && expAvg.numel() == param.numel() &&
                    expAvgSq.numel() == param.numel() && grad.numel() == param.numel(),
                "adamStep: moment / gradient size mismatch");
    TORCH_CHECK(step >= 1, "adamStep: step is 1-based");
    c10::cuda::CUDAGuard guard(param.device());
    torch::NoGradGuard noGrad;
    torch::Tensor g = f32(grad);
    check(gsb_adam_step(param.numel(), param.data_ptr<float>(), fp(g), expAvg.data_ptr<float>(),
                        expAvgSq.data_ptr<float>(), (float)lr, (float)beta1, (float)beta2, (float)eps,
                        (float)(1.0 - std::pow(beta1, (double)step)), (float)(1.0 - std::pow(beta2, (double)step)),
                        stream()),
          "gsb_adam_step");
}

void densifyStats(const torch::Tensor &xysGrad, const torch::Tensor &radii, int imgHeight, int imgWidth, bool first,
                  torch::Tensor xysGradNorm, torch::Tensor visCounts, torch::Tensor max2DSize) {
    const int n = (int)radii.numel();
    TORCH_CHECK(xysGradNorm.numel() == n && visCounts.numel() == n && max2DSize.numel() == n,
                "densifyStats: statistics tensors must have one entry per Gaussian");
    c10::cuda::CUDAGuard guard(radii.device());
    torch::Tensor g = f32(xysGrad), r = i32(radii);
    auto fn = first ? gsb_densify_stats_init : gsb_densify_stats_update;
    check(fn(n, fp(g), r.data_ptr<int32_t>(), imgHeight, imgWidth, xysGradNorm.data_ptr<float>(),
             visCounts.data_ptr<float>(), max2DSize.data_ptr<float>(), stream()),
          "gsb_densify_stats");
}

}  // namespace gsb

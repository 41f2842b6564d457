// fused_extras.hpp -- OPTIONAL one-line replacements for the ATen glue around the three operators in the reference's
// Model (SURVEY.md 8f rows 2-3).  Nothing in model.cpp needs them (it compiles and runs unchanged on this back end);
// a maintainer who wants the fused kernels swaps, e.g.,
//     torch::Tensor ssimLoss = 1.0f - ssim.eval(rgb, gt); ... return (1-w)*l1Loss + w*ssimLoss;   (model.cpp:780-784)
// for
//     return gsb::MainLoss::apply(rgb, gt, ssimWeight);
// and the six `xxxOpt->step()` calls (model.cpp:236-243) for gsb::adamStep on each parameter.
#pragma once
#include <torch/torch.h>
#include <tuple>

namespace gsb {

// Model::mainLoss = (1-w) * mean|rgb - gt| + w * (1 - SSIM(rgb, gt)) with the reference's SSIM (ssim.cpp:8-47),
// forward + gradient w.r.t. rgb in two fused tile kernels.  rgb, gt: [H,W,3] CUDA tensors.  Returns a scalar.
class MainLoss : public torch::autograd::Function<MainLoss> {
public:
    static torch::Tensor forward(torch::autograd::AutogradContext *ctx, torch::Tensor rgb, torch::Tensor gt,
                                 double ssimWeight);
    static torch::autograd::tensor_list backward(torch::autograd::AutogradContext *ctx,
                                                 torch::autograd::tensor_list grad_outputs);
};

// The parameter activations of Model::forward in one pass each way (model.cpp:148-150,176-177,200):
//   {scales = exp(logScales), quats = rawQuats / |rawQuats|, opacities [N,1] = sigmoid(opacityLogits),
//    viewDirs = normalize(means - camPos)  (detached: no gradient)}.       camPos: 3-element tensor (any device).
//   auto a = gsb::ActivateGaussians::apply(means, scales, quats, opacities, camPos);   // a[0..3]
class ActivateGaussians : public torch::autograd::Function<ActivateGaussians> {
public:
    static torch::autograd::tensor_list forward(torch::autograd::AutogradContext *ctx, torch::Tensor means,
                                                torch::Tensor logScales, torch::Tensor rawQuats,
                                                torch::Tensor opacityLogits, torch::Tensor camPos);
    static torch::autograd::tensor_list backward(torch::autograd::AutogradContext *ctx,
                                                 torch::autograd::tensor_list grad_outputs);
};

// The colour pass of Model::forward without its ATen glue (model.cpp:176-177,186-192):
//   rgbs = clamp_min(SphericalHarmonics(degreesToUse, means - camPos, cat(featuresDc[:,None,:], featuresRest)) + 0.5, 0)
// reading featuresDc [N,3] / featuresRest [N,K-1,3] where they lie (no 12K-byte/Gaussian cat, no split in autograd)
// and writing their two gradients directly.
//   torch::Tensor rgbs = gsb::SphericalHarmonicsRgb::apply(degreesToUse, means, camPos, featuresDc, featuresRest);
class SphericalHarmonicsRgb : public torch::autograd::Function<SphericalHarmonicsRgb> {
public:
    static torch::Tensor forward(torch::autograd::AutogradContext *ctx, int64_t degreesToUse, torch::Tensor means,
                                 torch::Tensor camPos, torch::Tensor featuresDc, torch::Tensor featuresRest);
    static torch::autograd::tensor_list backward(torch::autograd::AutogradContext *ctx,
                                                 torch::autograd::tensor_list grad_outputs);
};

// ProjectGaussians on the model's RAW parameters -- model.cpp:148-150 (`exp(scales)`, `quats / quats.norm()`),
// model.cpp:200 (`sigmoid(opacities)`) and model.cpp:152-165 as one operator; the activations run as the projection
// kernels' prologue / epilogue, gradients come back w.r.t. the raw parameters:
//   auto p = gsb::ProjectGaussiansActivated::apply(means, scales, 1, quats, opacities, viewMat, projMat @ viewMat,
//                                                  fx, fy, cx, cy, height, width, tileBounds);
//   // p[0..5] = xys, depths, radii, conics, numTilesHit, cov3d (as ProjectGaussians), p[6] = sigmoid(opacities) [N,1]
class ProjectGaussiansActivated : public torch::autograd::Function<ProjectGaussiansActivated> {
public:
    static torch::autograd::variable_list forward(torch::autograd::AutogradContext *ctx, torch::Tensor means,
                                                  torch::Tensor logScales, double globScale, torch::Tensor rawQuats,
                                                  torch::Tensor opacityLogits, torch::Tensor viewMat,
                                                  torch::Tensor projMat, double fx, double fy, double cx, double cy,
                                                  int64_t imgHeight, int64_t imgWidth,
                                                  std::tuple<int, int, int> tileBounds, double clipThresh = 0.01);
    static torch::autograd::tensor_list backward(torch::autograd::AutogradContext *ctx,
                                                 torch::autograd::tensor_list grad_outputs);
};

// ProjectGaussiansActivated with the anti-aliased opacity (DESIGN D19, gsplat's "antialiased" mode): same arguments
// and outputs, but p[6] = sigmoid(opacities) * sqrt(max(0, det0 / det)) with det0 / det the determinants of the
// screen covariance before / after the 0.3 px^2 blur (0 for a culled Gaussian); p[0..5] are bit-identical.
class ProjectGaussiansActivatedAntialiased : public torch::autograd::Function<ProjectGaussiansActivatedAntialiased> {
public:
    static torch::autograd::variable_list forward(torch::autograd::AutogradContext *ctx, torch::Tensor means,
                                                  torch::Tensor logScales, double globScale, torch::Tensor rawQuats,
                                                  torch::Tensor opacityLogits, torch::Tensor viewMat,
                                                  torch::Tensor projMat, double fx, double fy, double cx, double cy,
                                                  int64_t imgHeight, int64_t imgWidth,
                                                  std::tuple<int, int, int> tileBounds, double clipThresh = 0.01);
    static torch::autograd::tensor_list backward(torch::autograd::AutogradContext *ctx,
                                                 torch::autograd::tensor_list grad_outputs);
};

// `rgb = RasterizeGaussians::apply(...); rgb = torch::clamp_max(rgb, 1.0f);` (model.cpp:213-222) as one operator:
// the blend kernel writes the clamped image, the backward blend kernel applies clamp_max's gradient mask.
// Same arguments and gradient slots as RasterizeGaussians.
class RasterizeGaussiansClamped : public torch::autograd::Function<RasterizeGaussiansClamped> {
public:
    static torch::Tensor forward(torch::autograd::AutogradContext *ctx, torch::Tensor xys, torch::Tensor depths,
                                 torch::Tensor radii, torch::Tensor conics, torch::Tensor numTilesHit,
                                 torch::Tensor colors, torch::Tensor opacity, int imgHeight, int imgWidth,
                                 torch::Tensor background);
    static torch::autograd::tensor_list backward(torch::autograd::AutogradContext *ctx,
                                                 torch::autograd::tensor_list grad_outputs);
};

// RasterizeGaussians with the depth and opacity maps (DESIGN D18): same arguments, returns {rgb [H,W,3], depth [H,W],
// alpha [H,W]}: depth = sum alpha T z over the pairs the colour blend blends (z = `depths`, the projection's view-space
// depth; background 0, not normalised), alpha = 1 - T_final.  rgb is bit-identical to RasterizeGaussians'.  Gradients
// for xys (0), depths (1), conics (3), colors (5), opacity (6): composed with ProjectGaussians[Activated], a depth loss
// reaches the means.
class RasterizeGaussiansDepth : public torch::autograd::Function<RasterizeGaussiansDepth> {
public:
    static torch::autograd::variable_list forward(torch::autograd::AutogradContext *ctx, torch::Tensor xys,
                                                  torch::Tensor depths, torch::Tensor radii, torch::Tensor conics,
                                                  torch::Tensor numTilesHit, torch::Tensor colors,
                                                  torch::Tensor opacity, int imgHeight, int imgWidth,
                                                  torch::Tensor background);
    static torch::autograd::tensor_list backward(torch::autograd::AutogradContext *ctx,
                                                 torch::autograd::tensor_list grad_outputs);
};

// RasterizeGaussiansDepth with rgb = clamp_max(rgb, 1) fused as in RasterizeGaussiansClamped (what Model::forward
// renders); depth and alpha are never clamped.
class RasterizeGaussiansDepthClamped : public torch::autograd::Function<RasterizeGaussiansDepthClamped> {
public:
    static torch::autograd::variable_list forward(torch::autograd::AutogradContext *ctx, torch::Tensor xys,
                                                  torch::Tensor depths, torch::Tensor radii, torch::Tensor conics,
                                                  torch::Tensor numTilesHit, torch::Tensor colors,
                                                  torch::Tensor opacity, int imgHeight, int imgWidth,
                                                  torch::Tensor background);
    static torch::autograd::tensor_list backward(torch::autograd::AutogradContext *ctx,
                                                 torch::autograd::tensor_list grad_outputs);
};

// Model::forward (model.cpp:82-225) with every glue op fused, on plain tensors -- what a maintainer calls from the
// body of Model::forward to opt in (INTEGRATION.md):
//     auto r = gsb::modelForward(means, scales, quats, featuresDc, featuresRest, opacities, backgroundColor,
//                                cam.camToWorld, fx, fy, cx, cy, height, width, degreesToUse);
//     xys = r.xys; radii = r.radii; lastHeight = height; lastWidth = width; return r.rgb;
// = ProjectGaussiansActivated -> (nothing visible: background, as model.cpp:173-174) -> SphericalHarmonicsRgb ->
// RasterizeGaussiansClamped; the camera matrices (model.cpp:92-113) are formed on the host and uploaded in one copy.
// fx, fy, cx, cy, height, width are the already down-scaled values (model.cpp:84-90).  xys has retain_grad() set
// (model.cpp:171) so that afterTrain finds xys.grad().
struct ModelForwardResult {
    torch::Tensor rgb, xys, radii;
};
ModelForwardResult modelForward(const torch::Tensor &means, const torch::Tensor &logScales,
                                const torch::Tensor &rawQuats, const torch::Tensor &featuresDc,
                                const torch::Tensor &featuresRest, const torch::Tensor &opacityLogits,
                                const torch::Tensor &backgroundColor, const torch::Tensor &camToWorld, float fx,
                                float fy, float cx, float cy, int height, int width, int degreesToUse);

// One torch::optim::Adam step (no weight decay / amsgrad) on `param` in place with caller-held moments;
// `step` is the 1-based step count of this parameter (AdamParamState::step after the increment).
void adamStep(torch::Tensor param, const torch::Tensor &grad, torch::Tensor expAvg, torch::Tensor expAvgSq, double lr,
              int64_t step, double beta1 = 0.9, double beta2 = 0.999, double eps = 1e-8);

// Model::afterTrain statistics (model.cpp:317-337) in one pass; `first` = the three tensors are being (re)created.
void densifyStats(const torch::Tensor &xysGrad, const torch::Tensor &radii, int imgHeight, int imgWidth, bool first,
                  torch::Tensor xysGradNorm, torch::Tensor visCounts, torch::Tensor max2DSize);

}  // namespace gsb

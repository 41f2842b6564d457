// register.cpp -- exposes the C++ autograd operators to Python as torch.ops.opensplat_b200.* so that the
// parity tests and bench.py's e2e arm can drive the SAME libtorch operator classes a C++ caller
// (model.cpp / simple_trainer.cpp) uses.
#include <torch/library.h>
#include "project_gaussians.hpp"
#include "rasterize_gaussians.hpp"
#include "spherical_harmonics.hpp"
#include "fused_extras.hpp"

static std::vector<torch::Tensor> op_project(torch::Tensor means, torch::Tensor scales, double globScale,
                                             torch::Tensor quats, torch::Tensor viewMat, torch::Tensor projMat,
                                             double fx, double fy, double cx, double cy, int64_t imgHeight,
                                             int64_t imgWidth, double clipThresh) {
    TileBounds tb = std::make_tuple((int)(imgWidth + BLOCK_X - 1) / BLOCK_X, (int)(imgHeight + BLOCK_Y - 1) / BLOCK_Y, 1);
    return ProjectGaussians::apply(means, scales, (float)globScale, quats, viewMat, projMat, (float)fx, (float)fy,
                                   (float)cx, (float)cy, (int)imgHeight, (int)imgWidth, tb, (float)clipThresh);
}

static torch::Tensor op_rasterize(torch::Tensor xys, torch::Tensor depths, torch::Tensor radii,
                                  torch::Tensor conics, torch::Tensor numTilesHit, torch::Tensor colors,
                                  torch::Tensor opacity, int64_t imgHeight, int64_t imgWidth,
                                  torch::Tensor background) {
    return RasterizeGaussians::apply(xys, depths, radii, conics, numTilesHit, colors, opacity, (int)imgHeight,
                                     (int)imgWidth, background);
}

static torch::Tensor op_sh(int64_t degreesToUse, torch::Tensor viewDirs, torch::Tensor coeffs) {
    return SphericalHarmonics::apply((int)degreesToUse, viewDirs, coeffs);
}

static std::vector<torch::Tensor> op_bin_and_sort(int64_t numPoints, int64_t numIntersects, torch::Tensor xys,
                                                  torch::Tensor depths, torch::Tensor radii,
                                                  torch::Tensor cumTilesHit, int64_t tilesX, int64_t tilesY) {
    auto t = binAndSortGaussians((int)numPoints, (int)numIntersects, xys, depths, radii, cumTilesHit,
                                 std::make_tuple((int)tilesX, (int)tilesY, 1));
    return {std::get<0>(t), std::get<1>(t), std::get<2>(t), std::get<3>(t), std::get<4>(t)};
}

static torch::Tensor op_main_loss(torch::Tensor rgb, torch::Tensor gt, double ssimWeight) {
    return gsb::MainLoss::apply(rgb, gt, ssimWeight);
}

static void op_adam_step(torch::Tensor param, torch::Tensor grad, torch::Tensor expAvg, torch::Tensor expAvgSq,
                         double lr, int64_t step, double beta1, double beta2, double eps) {
    gsb::adamStep(param, grad, expAvg, expAvgSq, lr, step, beta1, beta2, eps);
}

static void op_densify_stats(torch::Tensor xysGrad, torch::Tensor radii, int64_t imgHeight, int64_t imgWidth,
                             bool first, torch::Tensor xysGradNorm, torch::Tensor visCounts, torch::Tensor max2DSize) {
    gsb::densifyStats(xysGrad, radii, (int)imgHeight, (int)imgWidth, first, xysGradNorm, visCounts, max2DSize);
}

static std::vector<torch::Tensor> op_activate(torch::Tensor means, torch::Tensor logScales, torch::Tensor rawQuats,
                                              torch::Tensor opacityLogits, torch::Tensor camPos) {
    return gsb::ActivateGaussians::apply(means, logScales, rawQuats, opacityLogits, camPos);
}

static torch::Tensor op_sh_rgb(int64_t degreesToUse, torch::Tensor means, torch::Tensor camPos, torch::Tensor featuresDc,
                               torch::Tensor featuresRest) {
    return gsb::SphericalHarmonicsRgb::apply(degreesToUse, means, camPos, featuresDc, featuresRest);
}

static std::vector<torch::Tensor> op_project_activated(torch::Tensor means, torch::Tensor logScales, double globScale,
                                                       torch::Tensor rawQuats, torch::Tensor opacityLogits,
                                                       torch::Tensor viewMat, torch::Tensor projMat, double fx,
                                                       double fy, double cx, double cy, int64_t imgHeight,
                                                       int64_t imgWidth, double clipThresh) {
    TileBounds tb = std::make_tuple((int)(imgWidth + BLOCK_X - 1) / BLOCK_X, (int)(imgHeight + BLOCK_Y - 1) / BLOCK_Y, 1);
    return gsb::ProjectGaussiansActivated::apply(means, logScales, globScale, rawQuats, opacityLogits, viewMat,
                                                 projMat, fx, fy, cx, cy, imgHeight, imgWidth, tb, clipThresh);
}

static std::vector<torch::Tensor> op_project_activated_antialiased(
    torch::Tensor means, torch::Tensor logScales, double globScale, torch::Tensor rawQuats, torch::Tensor opacityLogits,
    torch::Tensor viewMat, torch::Tensor projMat, double fx, double fy, double cx, double cy, int64_t imgHeight,
    int64_t imgWidth, double clipThresh) {
    TileBounds tb = std::make_tuple((int)(imgWidth + BLOCK_X - 1) / BLOCK_X, (int)(imgHeight + BLOCK_Y - 1) / BLOCK_Y, 1);
    return gsb::ProjectGaussiansActivatedAntialiased::apply(means, logScales, globScale, rawQuats, opacityLogits,
                                                            viewMat, projMat, fx, fy, cx, cy, imgHeight, imgWidth, tb,
                                                            clipThresh);
}

static torch::Tensor op_rasterize_clamped(torch::Tensor xys, torch::Tensor depths, torch::Tensor radii,
                                          torch::Tensor conics, torch::Tensor numTilesHit, torch::Tensor colors,
                                          torch::Tensor opacity, int64_t imgHeight, int64_t imgWidth,
                                          torch::Tensor background) {
    return gsb::RasterizeGaussiansClamped::apply(xys, depths, radii, conics, numTilesHit, colors, opacity,
                                                 (int)imgHeight, (int)imgWidth, background);
}

static std::vector<torch::Tensor> op_rasterize_depth(torch::Tensor xys, torch::Tensor depths, torch::Tensor radii,
                                                     torch::Tensor conics, torch::Tensor numTilesHit,
                                                     torch::Tensor colors, torch::Tensor opacity, int64_t imgHeight,
                                                     int64_t imgWidth, torch::Tensor background) {
    return gsb::RasterizeGaussiansDepth::apply(xys, depths, radii, conics, numTilesHit, colors, opacity, (int)imgHeight,
                                               (int)imgWidth, background);
}

static std::vector<torch::Tensor> op_rasterize_depth_clamped(torch::Tensor xys, torch::Tensor depths,
                                                             torch::Tensor radii, torch::Tensor conics,
                                                             torch::Tensor numTilesHit, torch::Tensor colors,
                                                             torch::Tensor opacity, int64_t imgHeight,
                                                             int64_t imgWidth, torch::Tensor background) {
    return gsb::RasterizeGaussiansDepthClamped::apply(xys, depths, radii, conics, numTilesHit, colors, opacity,
                                                      (int)imgHeight, (int)imgWidth, background);
}

TORCH_LIBRARY(opensplat_b200, m) {
    m.def("project_gaussians_activated", &op_project_activated);
    m.def("project_gaussians_activated_antialiased", &op_project_activated_antialiased);
    m.def("rasterize_gaussians_clamped", &op_rasterize_clamped);
    m.def("rasterize_gaussians_depth", &op_rasterize_depth);
    m.def("rasterize_gaussians_depth_clamped", &op_rasterize_depth_clamped);
    m.def("activate_gaussians", &op_activate);
    m.def("spherical_harmonics_rgb", &op_sh_rgb);
    m.def("project_gaussians", &op_project);
    m.def("rasterize_gaussians", &op_rasterize);
    m.def("spherical_harmonics", &op_sh);
    m.def("bin_and_sort_gaussians", &op_bin_and_sort);
    m.def("main_loss", &op_main_loss);
    m.def("adam_step_(Tensor(a!) param, Tensor grad, Tensor(b!) exp_avg, Tensor(c!) exp_avg_sq, float lr, int step, "
          "float beta1, float beta2, float eps) -> ()", &op_adam_step);
    m.def("densify_stats_(Tensor xys_grad, Tensor radii, int img_height, int img_width, bool first, "
          "Tensor(a!) xys_grad_norm, Tensor(b!) vis_counts, Tensor(c!) max_2d_size) -> ()", &op_densify_stats);
}

// tests/native/points_driver.cpp -- TEST INFRASTRUCTURE ONLY.
// Constructs the UNMODIFIED reference Model (model.cpp / model.hpp, compiled from the reference checkout by
// oracle/build_points_ref.py into oracle/_ref/libopensplat_ref_points.so) through its own constructor
// (model.hpp:23-57) on the CPU, and returns its six parameter tensors: torch.ops.opensplat_ref_points.init_model.
//
// The reference's PointsTensor::scales() is a nanoflann k-d tree search (kdtree_tensor.cpp), and nanoflann is not
// available offline.  This driver's stand-in returns the caller's mean_dist [n,1] instead, so the constructor's
// `.repeat({1, 3}).log()`, the seeded randomQuatTensor, rgb2sh and logit all run as the reference's own code; the
// nearest-neighbour distances themselves are pinned by the two restatements in oracle/points_init.py.
#include <torch/torch.h>
#include <torch/library.h>

#include "model.hpp"

namespace {
thread_local torch::Tensor g_mean_dist;   // what PointsTensor::scales() returns during init_model
}

torch::Tensor PointsTensor::scales() {
    TORCH_CHECK(g_mean_dist.defined() && g_mean_dist.size(0) == tensor.size(0), "init_model: mean_dist not set");
    return g_mean_dist.reshape({tensor.size(0), 1}).to(torch::kFloat32).clone();
}
PointsTensor::~PointsTensor() {}

namespace {

using torch::Tensor;

// Model(inputData{xyz, rgb}, ..., shDegree, ..., device = CPU) -> {means, scales, quats, featuresDc, featuresRest,
// opacities}
std::vector<Tensor> init_model(Tensor xyz, Tensor rgb, int64_t sh_degree, Tensor mean_dist) {
    InputData in;
    in.scale = 1.0f;
    in.translation = torch::zeros({3}, torch::kFloat32);
    in.points.xyz = xyz.contiguous();
    in.points.rgb = rgb.contiguous();
    g_mean_dist = mean_dist.contiguous();
    const torch::Device device(torch::kCPU);
    auto m = std::make_unique<Model>(in, /*numCameras*/ 1, /*numDownscales*/ 0, /*resolutionSchedule*/ 3000,
                                     (int)sh_degree, /*shDegreeInterval*/ 1000, /*refineEvery*/ 100,
                                     /*warmupLength*/ 500, /*resetAlphaEvery*/ 30, /*densifyGradThresh*/ 0.0002f,
                                     /*densifySizeThresh*/ 0.01f, /*stopScreenSizeAt*/ 4000,
                                     /*splitScreenSize*/ 0.05f, /*maxSteps*/ 30000, /*keepCrs*/ false, device);
    g_mean_dist = Tensor();
    return {m->means.detach().clone(),      m->scales.detach().clone(),       m->quats.detach().clone(),
            m->featuresDc.detach().clone(), m->featuresRest.detach().clone(), m->opacities.detach().clone()};
}

}  // namespace

TORCH_LIBRARY(opensplat_ref_points, m) {
    m.def("init_model", &init_model);
}

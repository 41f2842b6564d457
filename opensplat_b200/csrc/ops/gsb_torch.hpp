// gsb_torch.hpp -- glue between libtorch tensors and the C ABI (device pointers, current stream,
// error propagation).  torch supplies memory, streams and autograd; all compute is in libgsplat_b200.
#pragma once
#include <torch/torch.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include "../../../include/gsplat_b200.h"

namespace gsb {

inline void check(int code, const char *what) {
    TORCH_CHECK(code == 0, what, " failed: ", gsb_last_error());
}

// contiguous fp32 view of a CUDA tensor (the reference's bindings call .contiguous() themselves,
// bindings.cu:179-195, so non-contiguous operator inputs are legal)
inline torch::Tensor f32(const torch::Tensor &t) {
    TORCH_CHECK(t.is_cuda(), "gsplat_b200: expected a CUDA tensor (this back end has no CPU path)");
    return t.to(torch::kFloat32).contiguous();
}
inline torch::Tensor i32(const torch::Tensor &t) {
    TORCH_CHECK(t.is_cuda(), "gsplat_b200: expected a CUDA tensor (this back end has no CPU path)");
    return t.to(torch::kInt32).contiguous();
}
inline const float *fp(const torch::Tensor &t) { return t.data_ptr<float>(); }
inline float *fpw(torch::Tensor &t) { return t.data_ptr<float>(); }
inline gsb_stream_t stream() { return (gsb_stream_t)c10::cuda::getCurrentCUDAStream().stream(); }
inline torch::TensorOptions like(const torch::Tensor &t, torch::ScalarType dt) {
    return torch::TensorOptions().dtype(dt).device(t.device());
}


// Bodies of RasterizeGaussians::forward / backward with the GSB_RASTER_* flags of the blend kernels
// (rasterize_gaussians.cpp); shared with gsb::RasterizeGaussiansClamped and gsb::RasterizeGaussiansDepth[Clamped]
// (fused_extras.cpp).  Given depthOut, the forward also renders the depth and opacity maps into depthOut->depth /
// depthOut->alpha (DESIGN D18) and the backward then takes grad_outputs {rgb, depth, alpha} and returns v_depths in
// slot 1.
struct DepthMaps {
    torch::Tensor depth, alpha;
};
torch::Tensor rasterizeForward(torch::autograd::AutogradContext *ctx, unsigned flags, torch::Tensor xys,
                               torch::Tensor depths, torch::Tensor radii, torch::Tensor conics,
                               torch::Tensor numTilesHit, torch::Tensor colors, torch::Tensor opacity, int imgHeight,
                               int imgWidth, torch::Tensor background, DepthMaps *depthOut = nullptr);
torch::autograd::tensor_list rasterizeBackward(torch::autograd::AutogradContext *ctx,
                                               torch::autograd::tensor_list grad_outputs);

}  // namespace gsb

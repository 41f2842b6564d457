// rasterize_gaussians.cpp -- RasterizeGaussians / binAndSortGaussians over the C ABI.
// Replaces the reference's rasterize_gaussians.cpp:6-140 + bindings.cu:279-632 and the ATen calls in
// between (torch::cumsum :62, .item<int>() :63, torch::sort :25, torch::gather :32).
#include "rasterize_gaussians.hpp"
#include "gsplat.hpp"
#include "gsb_torch.hpp"
#include <ATen/cuda/CUDAEvent.h>
#include <algorithm>
#include <climits>
#include <mutex>

namespace {

struct Binned {
    torch::Tensor isectIds, gaussianIds, isectIdsSorted, sortedIndex, gaussianIdsSorted, tileBins;
};

Binned bin_and_sort(int numPoints, int numIntersects, const torch::Tensor &xys, const torch::Tensor &depths,
                    const torch::Tensor &radii, const torch::Tensor &cumTilesHit, TileBounds tileBounds) {
    const int tilesX = std::get<0>(tileBounds), tilesY = std::get<1>(tileBounds);
    const int numTiles = tilesX * tilesY, m = numIntersects;
    torch::Tensor x = gsb::f32(xys), d = gsb::f32(depths), r = gsb::i32(radii), cum = gsb::i32(cumTilesHit);
    Binned b;
    b.isectIds = torch::empty({m}, gsb::like(x, torch::kInt64));
    b.gaussianIds = torch::empty({m}, gsb::like(x, torch::kInt32));
    b.isectIdsSorted = torch::empty({m}, gsb::like(x, torch::kInt64));
    b.sortedIndex = torch::empty({m}, gsb::like(x, torch::kInt32));
    b.gaussianIdsSorted = torch::empty({m}, gsb::like(x, torch::kInt32));
    b.tileBins = torch::empty({numTiles, 2}, gsb::like(x, torch::kInt32));
    gsb::check(gsb_map_gaussian_to_intersects(numPoints, m, gsb::fp(x), gsb::fp(d), r.data_ptr<int32_t>(),
                                              cum.data_ptr<int32_t>(), tilesX, tilesY,
                                              b.isectIds.data_ptr<int64_t>(), b.gaussianIds.data_ptr<int32_t>(),
                                              gsb::stream()),
               "gsb_map_gaussian_to_intersects");
    const size_t wsBytes = gsb_sort_workspace_bytes(m);
    torch::Tensor ws = torch::empty({(int64_t)wsBytes + 256}, gsb::like(x, torch::kUInt8));
    char *wsPtr = (char *)ws.data_ptr();
    wsPtr += (256 - ((uintptr_t)wsPtr % 256)) % 256;
    gsb::check(gsb_sort_intersects(m, numTiles, b.isectIds.data_ptr<int64_t>(),
                                   b.isectIdsSorted.data_ptr<int64_t>(), b.sortedIndex.data_ptr<int32_t>(), wsPtr,
                                   wsBytes, gsb::stream()),
               "gsb_sort_intersects");
    gsb::check(gsb_gather_bin_edges(m, numTiles, b.isectIdsSorted.data_ptr<int64_t>(),
                                    b.sortedIndex.data_ptr<int32_t>(), b.gaussianIds.data_ptr<int32_t>(),
                                    b.gaussianIdsSorted.data_ptr<int32_t>(), b.tileBins.data_ptr<int32_t>(),
                                    gsb::stream()),
               "gsb_gather_bin_edges");
    return b;
}

}  // namespace

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
binAndSortGaussians(int numPoints, int numIntersects, torch::Tensor xys, torch::Tensor depths,
                    torch::Tensor radii, torch::Tensor cumTilesHit, TileBounds tileBounds) {
    c10::cuda::CUDAGuard guard(xys.device());
    Binned b = bin_and_sort(numPoints, numIntersects, xys, depths, radii, cumTilesHit, tileBounds);
    return std::make_tuple(b.isectIds, b.gaussianIds, b.isectIdsSorted, b.gaussianIdsSorted, b.tileBins);
}

// ---- capacity plan of the fast binning path ----------------------------------------------------
// The reference blocks on `cumTilesHit[-1].item<int>()` (rasterize_gaussians.cpp:63) in the middle of the forward
// pass.  Here the M-dependent buffers are sized from high-water marks of earlier frames (per device, grow-only,
// 25 % headroom), the kernels are enqueued against those capacities and flag a frame that outgrows them, and the
// read-back is waited for only after the whole forward pass has been enqueued; the rare overflowing frame (and the
// very first one) is redone with larger buffers.
namespace {

struct BinPlan {
    int64_t mCap = 0;
    int lenCap = 0;
};
std::mutex gPlanMutex;
BinPlan gPlans[64];

BinPlan getPlan(int dev) {
    std::lock_guard<std::mutex> lock(gPlanMutex);
    return gPlans[dev & 63];
}

void growPlan(int dev, int m, int maxLen) {
    std::lock_guard<std::mutex> lock(gPlanMutex);
    BinPlan &p = gPlans[dev & 63];
    if (m > p.mCap) p.mCap = (int64_t)m + m / 4 + 4096;
    if (maxLen > p.lenCap) {
        const int64_t want = (int64_t)maxLen + maxLen / 4;
        int64_t cap = 64;
        while (cap < want) cap <<= 1;
        if (cap > 64 && cap < 256) cap = 256;
        p.lenCap = (int)std::min<int64_t>(cap, gsb_bucket_max_tile_len());
    }
}

// pinned landing buffer of the stats read-back, one per (thread, device)
torch::Tensor &statsHostFor(int dev) {
    static thread_local torch::Tensor bufs[64];
    torch::Tensor &b = bufs[dev & 63];
    if (!b.defined()) b = torch::zeros({4}, torch::TensorOptions().dtype(torch::kInt32).pinned_memory(true));
    return b;
}

inline char *align256(torch::Tensor &t) {
    char *p = (char *)t.data_ptr();
    return p + (256 - ((uintptr_t)p % 256)) % 256;
}

}  // namespace

namespace gsb {

// Body of RasterizeGaussians::forward; `flags` = GSB_RASTER_* (gsb::RasterizeGaussiansClamped passes
// GSB_RASTER_CLAMP_MAX_ONE: clamp_max(rgb, 1) fused into the blend kernels, fused_extras.hpp); depthOut: see
// gsb_torch.hpp.
torch::Tensor rasterizeForward(AutogradContext *ctx, unsigned flags, torch::Tensor xys, torch::Tensor depths,
                               torch::Tensor radii, torch::Tensor conics, torch::Tensor numTilesHit,
                               torch::Tensor colors, torch::Tensor opacity, int imgHeight, int imgWidth,
                               torch::Tensor background, DepthMaps *depthOut) {
    const int n = (int)xys.size(0);
    TORCH_CHECK(colors.size(-1) == 3, "RasterizeGaussians: only 3 colour channels are supported");
    c10::cuda::CUDAGuard guard(xys.device());
    const int dev = xys.device().index();
    const TileBounds tileBounds =
        std::make_tuple((imgWidth + BLOCK_X - 1) / BLOCK_X, (imgHeight + BLOCK_Y - 1) / BLOCK_Y, 1);
    const int tilesX = std::get<0>(tileBounds), tilesY = std::get<1>(tileBounds);
    const int numTiles = tilesX * tilesY;
    torch::Tensor x = gsb::f32(xys), con = gsb::f32(conics), col = gsb::f32(colors), op = gsb::f32(opacity);
    torch::Tensor bg = gsb::f32(background), d = gsb::f32(depths), r = gsb::i32(radii);

    torch::Tensor cum = torch::empty({n}, gsb::like(x, torch::kInt32));
    torch::Tensor tileBins = torch::empty({numTiles, 2}, gsb::like(x, torch::kInt32));
    torch::Tensor tileOrder = torch::empty({numTiles}, gsb::like(x, torch::kInt32));   // longest list first
    bool ordered = true;
    torch::Tensor stats = torch::empty({4}, gsb::like(x, torch::kInt32));
    torch::Tensor outImg = torch::empty({imgHeight, imgWidth, 3}, gsb::like(x, torch::kFloat32));
    torch::Tensor finalTs = torch::empty({imgHeight, imgWidth}, gsb::like(x, torch::kFloat32));
    torch::Tensor finalIdx = torch::empty({imgHeight, imgWidth}, gsb::like(x, torch::kInt32));
    torch::Tensor records;
    // depth output: the sorted Gaussian ids and the per-record depth stream gathered from them
    const bool depth = depthOut != nullptr;
    torch::Tensor gidsSorted, recordDepths;
    if (depth) {
        depthOut->depth = torch::empty({imgHeight, imgWidth}, gsb::like(x, torch::kFloat32));
        depthOut->alpha = torch::empty({imgHeight, imgWidth}, gsb::like(x, torch::kFloat32));
    }
    // the blend of the frame: the plain or the DEPTH kernel on the same records
    auto blend = [&](int m, const int32_t *bins, const int32_t *order, const int32_t *st) {
        if (depth)
            gsb::check(gsb_rasterize_forward_packed_depth(
                           imgHeight, imgWidth, tilesX, tilesY, m, bins, order, st, gsb::fp(bg), records.data_ptr(),
                           gsb::fpw(outImg), gsb::fpw(finalTs), finalIdx.data_ptr<int32_t>(), flags,
                           gsb::fp(recordDepths), gsb::fpw(depthOut->depth), gsb::fpw(depthOut->alpha), gsb::stream()),
                       "gsb_rasterize_forward_packed_depth");
        else
            gsb::check(gsb_rasterize_forward_packed(imgHeight, imgWidth, tilesX, tilesY, m, bins, order, st,
                                                    gsb::fp(bg), records.data_ptr(), gsb::fpw(outImg),
                                                    gsb::fpw(finalTs), finalIdx.data_ptr<int32_t>(), flags,
                                                    gsb::stream()),
                       "gsb_rasterize_forward_packed");
    };
    torch::Tensor &statsHost = statsHostFor(dev);
    const int limit = gsb_bucket_max_tile_len();
    int mRaster = 0;   // what the records buffer is sized with (the blend kernels' scratch words sit behind it)
    const int cull = 1;
    while (true) {
        const BinPlan plan = getPlan(dev);
        const int mCap = (int)std::min<int64_t>(plan.mCap, INT32_MAX - 1024), lenCap = plan.lenCap;
        const size_t wsBytes = gsb_bucket_workspace_bytes(n, mCap, numTiles);
        torch::Tensor ws = torch::empty({(int64_t)wsBytes + 256}, gsb::like(x, torch::kUInt8));
        char *wp = align256(ws);
        records = torch::empty({(int64_t)gsb_raster_records_bytes(mCap)}, gsb::like(x, torch::kUInt8));
        gsb::check(gsb_bucket_tile_ranges(n, gsb::fp(x), r.data_ptr<int32_t>(), gsb::fp(con), gsb::fp(col),
                                          gsb::fp(op), cull, tilesX, tilesY, mCap, lenCap, wp, wsBytes,
                                          cum.data_ptr<int32_t>(), tileBins.data_ptr<int32_t>(),
                                          tileOrder.data_ptr<int32_t>(), stats.data_ptr<int32_t>(), gsb::stream()),
                   "gsb_bucket_tile_ranges");
        statsHost.copy_(stats, /*non_blocking=*/true);
        at::cuda::CUDAEvent statsReady;
        statsReady.record(c10::cuda::getCurrentCUDAStream());
        if (depth) {
            gidsSorted = torch::empty({std::max(mCap, 1)}, gsb::like(x, torch::kInt32));
            recordDepths = torch::empty({std::max(mCap, 1)}, gsb::like(x, torch::kFloat32));
        }
        if (mCap > 0)
            gsb::check(gsb_bucket_sort_pack(n, mCap, lenCap, gsb::fp(d), r.data_ptr<int32_t>(),
                                            cum.data_ptr<int32_t>(), cull, tilesX, tilesY,
                                            tileBins.data_ptr<int32_t>(), stats.data_ptr<int32_t>(), wp, wsBytes,
                                            records.data_ptr(), nullptr,
                                            depth ? gidsSorted.data_ptr<int32_t>() : nullptr, gsb::stream()),
                       "gsb_bucket_sort_pack");
        if (depth && n > 0)   // the ids past M hold nothing valid: the gather reads M from the stats
            gsb::check(gsb_gather_record_depths(mCap, gidsSorted.data_ptr<int32_t>(), gsb::fp(d),
                                                stats.data_ptr<int32_t>(), gsb::fpw(recordDepths), gsb::stream()),
                       "gsb_gather_record_depths");
        blend(mCap, tileBins.data_ptr<int32_t>(), tileOrder.data_ptr<int32_t>(), stats.data_ptr<int32_t>());
        // the path's single device->host read-back (rasterize_gaussians.cpp:63), waited for with the GPU busy
        statsReady.synchronize();
        const int32_t *sh = statsHost.data_ptr<int32_t>();
        const int m = sh[0], maxLen = sh[1];
        const bool overflow = sh[2] != 0;
        mRaster = mCap;
        if (!overflow) break;
        if (maxLen <= limit) {
            growPlan(dev, m, maxLen);
            continue;
        }
        // pathological tile lists: generic global radix sort on the reference's own (unculled) intersection lists
        torch::Tensor nth = gsb::i32(numTilesHit);
        const size_t sb = gsb_cumsum_workspace_bytes(n);
        torch::Tensor sws = torch::empty({(int64_t)sb + 256}, gsb::like(x, torch::kUInt8));
        char *swsPtr = (char *)sws.data_ptr();
        swsPtr += (256 - ((uintptr_t)swsPtr % 256)) % 256;
        gsb::check(gsb_cumsum_tiles_hit(n, nth.data_ptr<int32_t>(), cum.data_ptr<int32_t>(), swsPtr, sb,
                                        gsb::stream()),
                   "gsb_cumsum_tiles_hit");
        const int mRef = cum[n - 1].item<int>();
        Binned b = bin_and_sort(n, mRef, x, d, r, cum, tileBounds);
        tileBins = b.tileBins;
        records = torch::empty({(int64_t)gsb_raster_records_bytes(mRef)}, gsb::like(x, torch::kUInt8));
        gsb::check(gsb_pack_records(mRef, b.gaussianIdsSorted.data_ptr<int32_t>(), b.sortedIndex.data_ptr<int32_t>(),
                                    gsb::fp(x), gsb::fp(con), gsb::fp(col), gsb::fp(op), records.data_ptr(),
                                    gsb::stream()),
                   "gsb_pack_records");
        if (depth) {
            recordDepths = torch::empty({std::max(mRef, 1)}, gsb::like(x, torch::kFloat32));
            gsb::check(gsb_gather_record_depths(mRef, b.gaussianIdsSorted.data_ptr<int32_t>(), gsb::fp(d), nullptr,
                                                gsb::fpw(recordDepths), gsb::stream()),
                       "gsb_gather_record_depths");
        }
        blend(mRef, b.tileBins.data_ptr<int32_t>(), nullptr, nullptr);
        mRaster = mRef;
        ordered = false;
        break;
    }

    ctx->saved_data["imgWidth"] = imgWidth;
    ctx->saved_data["imgHeight"] = imgHeight;
    ctx->saved_data["numIntersects"] = mRaster;
    ctx->saved_data["ordered"] = ordered;
    ctx->saved_data["flags"] = (int64_t)flags;
    ctx->saved_data["depth"] = depth;
    if (depth)
        ctx->save_for_backward({tileBins, con, op, records, cum, bg, finalTs, finalIdx, tileOrder, recordDepths});
    else
        ctx->save_for_backward({tileBins, con, op, records, cum, bg, finalTs, finalIdx, tileOrder});
    return outImg;
}

namespace {

// rasterizeBackward of a frame rendered with the depth and opacity maps: grad_outputs {rgb, depth, alpha}, any of
// them undefined (zeros); gradients for xys (0), depths (1), conics (3), colors (5), opacity (6).
tensor_list rasterizeBackwardDepth(AutogradContext *ctx, const variable_list &saved, const tensor_list &grad_outputs) {
    const unsigned flags = (unsigned)ctx->saved_data["flags"].toInt();
    const int imgHeight = (int)ctx->saved_data["imgHeight"].toInt();
    const int imgWidth = (int)ctx->saved_data["imgWidth"].toInt();
    const int m = (int)ctx->saved_data["numIntersects"].toInt();
    torch::Tensor tileBins = saved[0], con = saved[1], op = saved[2], records = saved[3], cum = saved[4];
    torch::Tensor bg = saved[5], finalTs = saved[6], finalIdx = saved[7], tileOrder = saved[8], recordDepths = saved[9];
    const bool ordered = ctx->saved_data["ordered"].toBool();
    const int n = (int)con.size(0);
    torch::Tensor v_out = grad_outputs[0].defined() ? gsb::f32(grad_outputs[0])
                                                    : torch::zeros({imgHeight, imgWidth, 3}, gsb::like(con, torch::kFloat32));
    torch::Tensor v_depth = grad_outputs[1].defined() ? gsb::f32(grad_outputs[1]) : torch::Tensor();
    torch::Tensor v_alpha = grad_outputs[2].defined() ? gsb::f32(grad_outputs[2]) : torch::Tensor();
    torch::Tensor rows = torch::empty({(int64_t)gsb_raster_grad_rows_bytes(m)}, gsb::like(con, torch::kUInt8));
    torch::Tensor v_xy = torch::empty({n, 2}, gsb::like(con, torch::kFloat32));
    torch::Tensor v_conic = torch::empty({n, 3}, gsb::like(con, torch::kFloat32));
    torch::Tensor v_colors = torch::empty({n, 3}, gsb::like(con, torch::kFloat32));
    torch::Tensor v_opacity = torch::empty({n, 1}, gsb::like(con, torch::kFloat32));
    torch::Tensor v_depths = torch::empty({n}, gsb::like(con, torch::kFloat32));
    gsb::check(gsb_rasterize_backward_depth(
                   imgHeight, imgWidth, (imgWidth + BLOCK_X - 1) / BLOCK_X, (imgHeight + BLOCK_Y - 1) / BLOCK_Y, n, m,
                   tileBins.data_ptr<int32_t>(), ordered ? tileOrder.data_ptr<int32_t>() : nullptr, gsb::fp(con),
                   gsb::fp(op), records.data_ptr(), cum.data_ptr<int32_t>(), gsb::fp(bg), gsb::fp(finalTs),
                   finalIdx.data_ptr<int32_t>(), gsb::fp(v_out), v_alpha.defined() ? gsb::fp(v_alpha) : nullptr,
                   rows.data_ptr(), gsb::fpw(v_xy), gsb::fpw(v_conic), gsb::fpw(v_colors), gsb::fpw(v_opacity), flags,
                   gsb::fp(recordDepths), v_depth.defined() ? gsb::fp(v_depth) : nullptr, gsb::fpw(v_depths),
                   gsb::stream()),
               "gsb_rasterize_backward_depth");
    torch::Tensor none;
    return {v_xy, v_depths, none, v_conic, none, v_colors, v_opacity, none, none, none};
}

}  // namespace

tensor_list rasterizeBackward(AutogradContext *ctx, tensor_list grad_outputs) {
    const unsigned flags = (unsigned)ctx->saved_data["flags"].toInt();
    const int imgHeight = (int)ctx->saved_data["imgHeight"].toInt();
    const int imgWidth = (int)ctx->saved_data["imgWidth"].toInt();
    const int m = (int)ctx->saved_data["numIntersects"].toInt();
    variable_list saved = ctx->get_saved_variables();
    torch::Tensor tileBins = saved[0], con = saved[1], op = saved[2], records = saved[3], cum = saved[4];
    torch::Tensor bg = saved[5], finalTs = saved[6], finalIdx = saved[7], tileOrder = saved[8];
    const bool ordered = ctx->saved_data["ordered"].toBool();
    const int n = (int)con.size(0);
    c10::cuda::CUDAGuard guard(con.device());
    if (ctx->saved_data["depth"].toBool()) return rasterizeBackwardDepth(ctx, saved, grad_outputs);
    torch::Tensor v_out = gsb::f32(grad_outputs[0]);  // may arrive as an expanded (stride-0) tensor
    torch::Tensor rows = torch::empty({(int64_t)gsb_raster_grad_rows_bytes(m)}, gsb::like(con, torch::kUInt8));
    torch::Tensor v_xy = torch::empty({n, 2}, gsb::like(con, torch::kFloat32));
    torch::Tensor v_conic = torch::empty({n, 3}, gsb::like(con, torch::kFloat32));
    torch::Tensor v_colors = torch::empty({n, 3}, gsb::like(con, torch::kFloat32));
    torch::Tensor v_opacity = torch::empty({n, 1}, gsb::like(con, torch::kFloat32));
    // v_output_alpha is identically zero in the reference (rasterize_gaussians.cpp:108) -> NULL
    gsb::check(gsb_rasterize_backward(imgHeight, imgWidth, (imgWidth + BLOCK_X - 1) / BLOCK_X,
                                      (imgHeight + BLOCK_Y - 1) / BLOCK_Y, n, m, tileBins.data_ptr<int32_t>(),
                                      ordered ? tileOrder.data_ptr<int32_t>() : nullptr, gsb::fp(con), gsb::fp(op),
                                      records.data_ptr(), cum.data_ptr<int32_t>(), gsb::fp(bg), gsb::fp(finalTs),
                                      finalIdx.data_ptr<int32_t>(), gsb::fp(v_out), nullptr, rows.data_ptr(),
                                      gsb::fpw(v_xy), gsb::fpw(v_conic), gsb::fpw(v_colors), gsb::fpw(v_opacity),
                                      flags, gsb::stream()),
               "gsb_rasterize_backward");
    torch::Tensor none;
    return {v_xy, none, none, v_conic, none, v_colors, v_opacity, none, none, none};
}

}  // namespace gsb

torch::Tensor RasterizeGaussians::forward(AutogradContext *ctx, torch::Tensor xys, torch::Tensor depths,
                                          torch::Tensor radii, torch::Tensor conics, torch::Tensor numTilesHit,
                                          torch::Tensor colors, torch::Tensor opacity, int imgHeight,
                                          int imgWidth, torch::Tensor background) {
    return gsb::rasterizeForward(ctx, 0u, xys, depths, radii, conics, numTilesHit, colors, opacity, imgHeight,
                                 imgWidth, background);
}

tensor_list RasterizeGaussians::backward(AutogradContext *ctx, tensor_list grad_outputs) {
    return gsb::rasterizeBackward(ctx, grad_outputs);
}

torch::Tensor RasterizeGaussiansCPU::forward(AutogradContext *, torch::Tensor, torch::Tensor, torch::Tensor,
                                             torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, int, int,
                                             torch::Tensor) {
    TORCH_CHECK(false, "RasterizeGaussiansCPU: the gsplat_b200 back end has no CPU path; link the reference's "
                       "rasterizer/gsplat-cpu for CPU execution");
    return {};
}

tensor_list RasterizeGaussiansCPU::backward(AutogradContext *, tensor_list) {
    TORCH_CHECK(false, "RasterizeGaussiansCPU: no CPU path in the gsplat_b200 back end");
    return {};
}

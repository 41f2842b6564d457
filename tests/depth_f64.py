"""Float64 reference of the depth and opacity maps (DESIGN D18), built from tests/blend_f64.blend without changing it.

The blend's decisions (which pairs blend, where a pixel terminates) do not depend on the colours, so the depth map is
the same blend run on one more colour: z broadcast to three channels with background 0, and the VJP of the three
outputs is the sum of two blend() backward passes over the same certificates:
  * blend(colours, background) with v_out and v_output_alpha -- the image, alpha = 1 - final_Ts, and their gradient;
  * blend(z, 0) with v_out = (v_depth, 0, 0) -- the depth map (channel 0) and its gradient; its v_colors[:, 0] is
    v_depths.
The geometry gradients (v_xy, v_conic, v_opacity) and their error scales A / B are the sums of the two.
"""
import torch

import blend_f64 as bf


def blend_depth(gaussian_ids_sorted, tile_bins, xys, conics, colors, opacities, depths, background, img_h, img_w,
                v_output=None, v_output_depth=None, v_output_alpha=None, clamp=False, depth_background=None,
                budget=1 << 24):
    """blend() plus out_depth / A_depth / B_depth [H,W], out_alpha [H,W] and, with the cotangents, v_depths [N,1] with
    its A_ / B_.  pix_cert / gauss_cert are those of both passes.  depth_background (default 0) exists to show what a
    wrong background convention would give."""
    dev = xys.device
    H, W = int(img_h), int(img_w)
    bwd = v_output is not None
    r = bf.blend(gaussian_ids_sorted, tile_bins, xys, conics, colors, opacities, background, H, W,
                 v_output=v_output, v_output_alpha=v_output_alpha, clamp=clamp, budget=budget)
    z3 = depths.reshape(-1, 1).to(torch.float64).expand(-1, 3).contiguous()
    vd = None
    if bwd:
        v0 = (v_output_depth.to(dev, torch.float64).reshape(H, W) if v_output_depth is not None
              else torch.zeros(H, W, dtype=torch.float64, device=dev))
        vd = torch.stack([v0, torch.zeros_like(v0), torch.zeros_like(v0)], -1)
    dbg = torch.zeros(3, dtype=torch.float64) if depth_background is None else \
        torch.as_tensor(depth_background, dtype=torch.float64).expand(3)
    d = bf.blend(gaussian_ids_sorted, tile_bins, xys, conics, z3, opacities, dbg, H, W, v_output=vd, budget=budget)
    r["out_depth"], r["A_depth"], r["B_depth"] = d["out_img"][..., 0], d["A_out"][..., 0], d["B_out"][..., 0]
    r["out_alpha"] = 1.0 - r["final_Ts"]
    r["pix_cert"] = r["pix_cert"] & d["pix_cert"]
    r["gauss_cert"] = r["gauss_cert"] & d["gauss_cert"]
    if bwd:
        for k in ("v_xy", "v_conic", "v_opacity"):
            for p in ("", "A_", "B_"):
                r[p + k] = r[p + k] + d[p + k]
        for p in ("", "A_", "B_"):
            r[p + "v_depths"] = d[p + "v_colors"][:, :1].clone()
    return r

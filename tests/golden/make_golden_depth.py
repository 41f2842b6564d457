"""Generates tests/golden/depth_*.npz -- the depth and opacity maps of DESIGN D18 and their gradients -- by running the
REFERENCE ITSELF (oracle/_ref: the unmodified CPU ProjectGaussians / RasterizeGaussians with autograd).  Run in the
build container only (needs /root/reference to have built oracle/_ref):

    python tests/golden/make_golden_depth.py

The reference has no depth output, so one projection is rasterized three times under the chain conventions of
make_golden.py (distinct depths, dense camDepths, tight opacities except the opaque case):
  * the RGB image;
  * the depth map: colours = the view-space z broadcast to 3 channels, background 0 (channel 0 is the map);
  * the transmittance: colours 0, background 1, so alpha = 1 - image (channel 0).
The CPU back end's camDepths is the PROJECTED z (it orders the blend), not the view-space z the CUDA projection's
`depths` hold, so z is formed here as (viewmat [means, 1])_z with differentiable torch ops.  One weighted sum of the
three outputs is back-propagated into means, scales, quats, colours and opacities (the gradients w.r.t. xys, conics and
z are kept too, for the float64 check of the blend alone).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref  # noqa: E402
from opensplat_b200.scene import make_scene  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def depth_case(name, n, W, H, scale, opacity, background, seed, unit_quats=True):
    sc = make_scene(n, W, H, scale=scale, sh_degree=0, opacity=opacity, seed=seed)
    rng = np.random.default_rng(seed + 2000)
    quats = sc["quats"] if unit_quats else (sc["quats"] * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    wgt = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    wgt_depth = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    wgt_alpha = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    t = lambda a, g=False: torch.from_numpy(np.ascontiguousarray(a)).requires_grad_(g)
    means, scales, q = t(sc["means"], True), t(sc["scales"], True), t(quats, True)
    col, op = t(colors, True), t(sc["opacities"], True)
    viewmat = t(sc["viewmat"])
    o = ref.ops()
    xys, radii, conics, cov2d, camd = o.project_cpu(means, scales, 1.0, q, viewmat, t(sc["projmat"]), sc["fx"],
                                                    sc["fy"], sc["cx"], sc["cy"], H, W, 0.01)
    xys.retain_grad(); conics.retain_grad()
    camd = camd.contiguous()
    z = means @ viewmat[2, :3] + viewmat[2, 3]            # view-space depth, differentiable in the means
    z.retain_grad()
    raster = lambda c, bg: o.rasterize_cpu(xys, radii, conics, c, op, cov2d, camd, H, W, torch.tensor(bg))
    img = raster(col, np.asarray(background, np.float32))
    depth = raster(z[:, None].expand(n, 3).contiguous(), np.zeros(3, np.float32))[..., 0]
    alpha = 1.0 - raster(torch.zeros(n, 3), np.ones(3, np.float32))[..., 0]
    loss = (img * t(wgt)).sum() + (depth * t(wgt_depth)).sum() + (alpha * t(wgt_alpha)).sum()
    loss.backward()
    np.savez_compressed(
        os.path.join(OUT, name + ".npz"),
        means=sc["means"], scales=sc["scales"], quats=quats, colors=colors, opacities=sc["opacities"],
        viewmat=sc["viewmat"], projmat=sc["projmat"],
        intrins=np.array([sc["fx"], sc["fy"], sc["cx"], sc["cy"]], np.float64), hw=np.array([H, W]),
        background=np.asarray(background, np.float32), wgt=wgt, wgt_depth=wgt_depth, wgt_alpha=wgt_alpha,
        ref_xys=xys.detach().numpy(), ref_radii=radii.numpy(), ref_conics=conics.detach().numpy(),
        ref_z=z.detach().numpy(),
        ref_img=img.detach().numpy(), ref_depth=depth.detach().numpy(), ref_alpha=alpha.detach().numpy(),
        ref_v_xy=xys.grad.numpy(), ref_v_conic=conics.grad.numpy(), ref_v_z=z.grad.numpy(),
        ref_v_colors=col.grad.numpy(), ref_v_opacity=op.grad.numpy(), ref_v_means=means.grad.numpy(),
        ref_v_scales=scales.grad.numpy(), ref_v_quats=q.grad.numpy())
    print(name, "depth max", float(depth.detach().max()), "alpha mean", float(alpha.detach().mean()),
          "radii max", int(radii.max()))


if __name__ == "__main__":
    torch.manual_seed(0)
    # ragged image (partial tiles), low opacity, black background
    depth_case("depth_tight_100x72", 600, 100, 72, 0.6, (0.05, 0.35), [0, 0, 0], seed=11)
    # magenta background (model.hpp:54), raw (non-unit) quats
    depth_case("depth_bg_quat_128x96", 800, 128, 96, 0.5, (0.05, 0.35), [0.6130, 0.0101, 0.3984], seed=12,
               unit_quats=False)
    # high opacity: saturating pixels (T <= 1e-4 early-out) and the D5 fringe -> looser tolerance
    depth_case("depth_opaque_96x96", 1500, 96, 96, 0.6, (0.5, 0.95), [0, 0, 0], seed=13)

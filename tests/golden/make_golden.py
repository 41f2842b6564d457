"""Generates tests/golden/*.npz by running the REFERENCE ITSELF (oracle/_ref: unmodified
rasterizer/gsplat-cpu + operator .cpp files compiled from /root/reference).  Run in the build
container only (needs /root/reference to have built oracle/_ref):

    python tests/golden/make_golden.py

The vectors pin oracle/gsplat_oracle.c (tests/test_oracle_vs_golden.py) and are also compared
directly against the CUDA path (tests/test_gpu_parity.py).  Conventions that make the reference CPU
back end a valid oracle for the CUDA tile semantics (SURVEY.md 8c): simple_trainer camera (w == 1,
centred principal point), strictly distinct depths, dense camDepths (D0), contiguous upstream
gradient, opacity <= 0.35 for the "tight" cases (D5).
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


def chain_case(name, n, W, H, scale, opacity, background, seed, unit_quats=True):
    sc = make_scene(n, W, H, scale=scale, sh_degree=0, opacity=opacity, seed=seed)
    rng = np.random.default_rng(seed + 1000)
    quats = sc["quats"] if unit_quats else (sc["quats"] * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    wgt = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    t = lambda a, g=False: torch.from_numpy(np.ascontiguousarray(a)).requires_grad_(g)
    means, scales, q = t(sc["means"], True), t(sc["scales"], True), t(quats, True)
    col, op = t(colors, True), t(sc["opacities"], True)
    o = ref.ops()
    p = o.project_cpu(means, scales, 1.0, q, t(sc["viewmat"]), t(sc["projmat"]), sc["fx"], sc["fy"],
                      sc["cx"], sc["cy"], H, W, 0.01)
    xys, radii, conics, cov2d, camd = p
    xys.retain_grad(); conics.retain_grad()
    img = o.rasterize_cpu(xys, radii, conics, col, op, cov2d, camd.contiguous(), H, W, t(background))
    (img * t(wgt)).sum().backward()
    np.savez_compressed(
        os.path.join(OUT, name + ".npz"),
        means=sc["means"], scales=sc["scales"], quats=quats, colors=colors, opacities=sc["opacities"],
        viewmat=sc["viewmat"], projmat=sc["projmat"],
        intrins=np.array([sc["fx"], sc["fy"], sc["cx"], sc["cy"]], np.float64), hw=np.array([H, W]),
        background=np.asarray(background, np.float32), wgt=wgt,
        ref_xys=xys.detach().numpy(), ref_radii=radii.numpy(), ref_conics=conics.detach().numpy(),
        ref_cov2d=cov2d.detach().numpy(), ref_depths=camd.detach().contiguous().numpy(),
        ref_img=img.detach().numpy(),
        ref_v_xy=xys.grad.numpy(), ref_v_conic=conics.grad.numpy(), ref_v_colors=col.grad.numpy(),
        ref_v_opacity=op.grad.numpy(), ref_v_means=means.grad.numpy(), ref_v_scales=scales.grad.numpy(),
        ref_v_quats=q.grad.numpy())
    print(name, "img mean", float(img.detach().mean()), "radii max", int(radii.max()))


def sh_case(name, n, degree, seed):
    rng = np.random.default_rng(seed)
    K = (degree + 1) ** 2
    vd = rng.standard_normal((n, 3)).astype(np.float32)
    vd /= np.linalg.norm(vd, axis=-1, keepdims=True)
    coeffs = rng.standard_normal((n, K, 3)).astype(np.float32)
    wgt = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    out = dict(viewdirs=vd, coeffs=coeffs, wgt=wgt, degree=np.array(degree))
    o = ref.ops()
    for d in range(degree + 1):
        c = torch.from_numpy(coeffs).requires_grad_(True)
        col = o.sh_cpu(d, torch.from_numpy(vd), c)
        (col * torch.from_numpy(wgt)).sum().backward()
        out[f"ref_colors_d{d}"] = col.detach().numpy()
        out[f"ref_v_coeffs_d{d}"] = c.grad.numpy()
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **out)
    print(name, "ok")


def loss_case(name, H, W, ssim_weight, seed, ties=False):
    """Model::mainLoss (model.cpp:780-784) through the reference's SSIM class (ssim.cpp).  ties: the content of
    loss_f64.tie_images -- u8/255 ground truth with saturated 0 and 1 blocks, rendered == gt on about 30 % of the
    pixels and constant blocks wider than the window -- which pins sgn(0) = 0 and the flat regions."""
    rng = np.random.default_rng(seed)
    gt = rng.uniform(0, 1, (H, W, 3)).astype(np.float32)
    rend = np.clip(gt + 0.15 * rng.standard_normal((H, W, 3)).astype(np.float32), 0, 1).astype(np.float32)
    if ties:
        sys.path.insert(0, os.path.dirname(OUT))
        from loss_f64 import tie_images
        rend, gt = tie_images(H, W, seed)
    r = torch.from_numpy(rend).requires_grad_()
    loss = ref.ops().main_loss_cpu(r, torch.from_numpy(gt), ssim_weight)
    loss.backward()
    np.savez_compressed(os.path.join(OUT, name + ".npz"), rendered=rend, gt=gt, ssim_weight=np.array(ssim_weight),
                        ref_loss=np.array(float(loss.detach())), ref_v_rendered=r.grad.numpy())
    print(name, "loss", float(loss.detach()))


if __name__ == "__main__":
    torch.manual_seed(0)
    # tight: low opacity (no D5 fringe), ragged image size (partial tiles), black background
    chain_case("chain_tight_100x72", 600, 100, 72, 0.6, (0.05, 0.35), [0, 0, 0], seed=1)
    # magenta background (model.hpp:54), raw (non-unit) quats exercise the normalisation Jacobian (D11)
    chain_case("chain_bg_quat_128x96", 800, 128, 96, 0.5, (0.05, 0.35), [0.6130, 0.0101, 0.3984], seed=2,
               unit_quats=False)
    # high opacity: saturating pixels (T <= 1e-4 early-out) and the D5 fringe -> looser tolerance
    chain_case("chain_opaque_96x96", 1500, 96, 96, 0.6, (0.5, 0.95), [0, 0, 0], seed=3)
    sh_case("sh_deg3", 500, 3, seed=4)
    sh_case("sh_deg4", 200, 4, seed=5)
    loss_case("loss_45x70", 45, 70, 0.2, seed=6)
    loss_case("loss_ties_48x80", 48, 80, 0.2, seed=7, ties=True)

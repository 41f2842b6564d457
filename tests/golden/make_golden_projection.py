"""Generates tests/golden/projection_*.npz by running the REFERENCE ITSELF: the CPU back end's project_cpu
(oracle/_ref, built by `make -C oracle ref` where the reference checkout exists) and torch autograd through it.

    python tests/golden/make_golden_projection.py

Unlike chain_*.npz these use general cameras, so the fov clamp (D8), the perspective divide (D12) and the rotation in
T = J V all carry weight:
  projection_general  camera from model.camera_setup with a rotated and translated camToWorld, fx != fy and an
                      off-centre principal point (w = t.z), glob_scale 1.3, raw quaternions, Gaussians beyond the clamp
                      on all four sides and in the corners with footprints that enter the image, a tenth with t.z in
                      (0.02, 0.2];
  projection_ties     an axis-aligned camera with Gaussians exactly on +-lim in x, in y and in the corners (t and
                      t.x / t.z exact in fp32 in both the reference's order and the kernels'), among ordinary ones.
The cotangents v_xy and v_conic are random for the Gaussians the CUDA semantics keep (oracle/gsplat_oracle.c) and 0
for the rest.  There is no v_depth: the CPU back end's depth output is NDC z, not view z."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref, oracle as orc  # noqa: E402
from opensplat_b200.model import Camera  # noqa: E402
import project_f64 as pf  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def case(name, cam, means, scales, quats, glob_scale, seed):
    assert cam.lim_x == cam.lim_x_cpu and cam.lim_y == cam.lim_y_cpu, "the two ways of forming lim must agree"
    n = means.shape[0]
    rng = np.random.default_rng(seed)
    o = orc.project_forward(means, scales, glob_scale, quats, *cam.args())
    keep = (o["radii"] > 0)[:, None]
    v_xy = (rng.standard_normal((n, 2)) * keep).astype(np.float32)
    v_conic = (rng.standard_normal((n, 3)) * keep).astype(np.float32)
    t = lambda a, g=False: torch.from_numpy(np.ascontiguousarray(a)).requires_grad_(g)
    m, s, q = t(means, True), t(scales, True), t(quats, True)
    V, P = cam.args()[:2]
    xys, radii, conics, cov2d, camd = ref.ops().project_cpu(m, s, glob_scale, q, t(V), t(P), cam.fx, cam.fy, cam.cx,
                                                           cam.cy, cam.H, cam.W, cam.clip)
    ((xys * t(v_xy)).sum() + (conics * t(v_conic)).sum()).backward()
    np.savez_compressed(
        os.path.join(OUT, name + ".npz"),
        means=means, scales=scales, quats=quats, glob_scale=np.array(glob_scale, np.float32), viewmat=V, projmat=P,
        intrins=np.array([cam.fx, cam.fy, cam.cx, cam.cy], np.float64), hw=np.array([cam.H, cam.W]),
        clip_thresh=np.array(cam.clip, np.float32), v_xy=v_xy, v_conic=v_conic,
        ref_xys=xys.detach().numpy(), ref_radii=radii.numpy(), ref_conics=conics.detach().numpy(),
        ref_cov2d=cov2d.detach().numpy(), ref_depths=camd.detach().numpy(), ref_v_means=m.grad.numpy(),
        ref_v_scales=s.grad.numpy(), ref_v_quats=q.grad.numpy())
    print(name, "n", n, "kept", int(keep.sum()), "radii max", int(o["radii"].max()))


def general():
    cam = pf.camera_from_setup(pf.general_camera(160, 120, seed=11))
    means, scales, quats = pf.random_gaussians(cam, 1200, seed=12)
    case("projection_general", cam, means, scales, quats, 1.3, seed=13)


def ties():
    W, H = 128, 96
    c2w = np.diag([1.0, -1.0, -1.0, 1.0]).astype(np.float32)      # camera_setup's y/z flip makes the view identity
    cam = pf.camera_from_setup(Camera(W, H, 100.0, 80.0, 0.5 * W + 7.0, 0.5 * H - 5.0, c2w))
    mt, st, qt = pf.tie_gaussians(cam, seed=21)
    mg, sg, qg = pf.random_gaussians(cam, 200, seed=22)
    case("projection_ties", cam, np.concatenate([mt, mg]), np.concatenate([st, sg]), np.concatenate([qt, qg]), 1.0,
         seed=23)


if __name__ == "__main__":
    torch.manual_seed(0)
    general()
    ties()

"""GPU: the data-parallel trainer.SplatTrainer over the fused NVLink exchange.
 * `gsb_sh_backward_multiview_cams` / `gsb_exchange_gradients_cams` (camera centres read through a device array of
   per-view pointers, as the peers' symmetric trailers are) with emulated peers -- the kernels take plain pointer
   arrays, so local buffers stand in for the peers' -- bit-identical to the entry points that read a [V,3] array;
 * a view that hits nothing: the trainer's backward pass writes exact zeros (what such a rank contributes);
 * tools/check_parallel_trainer.py under torch.distributed.run against model.GaussianModel under the same group: at
   world size 1 everywhere (symmetric memory, the camera trailer, set_camera, the SH degree schedule, resize after a
   refinement, both exchange paths), at world size 2 when two GPUs are present (both all-reduce flavours)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from opensplat_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _views(n, num_views, seed):
    rng = np.random.default_rng(seed)
    means = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    cams = (rng.standard_normal((num_views, 3)) * 6 + np.array([0, 0, -8])).astype(np.float32)
    v = rng.standard_normal((num_views, n, 3)).astype(np.float32)
    v[rng.uniform(size=(num_views, n)) < 0.3] = 0.0     # Gaussians not visible in a view contribute nothing
    if num_views > 1:
        v[num_views // 2] = 0.0                         # a view that hit nothing: a zero colour gradient throughout
    return means, cams, v


def _cam_pointers(cams):
    """One 16-byte trailer per view, in separate allocations (as on separate GPUs), and the device pointer array."""
    trailers = []
    for c in cams:
        t = torch.full((4,), float("nan"), device=DEV)
        t[:3] = cu(c)
        trailers.append(t)
    return trailers, torch.tensor([t.data_ptr() for t in trailers], dtype=torch.int64, device=DEV)


@pytest.mark.parametrize("num_views,n,deg,use", [(1, 1000, 3, 3), (3, 5003, 3, 3), (8, 4097, 3, 2), (9, 777, 3, 3),
                                                 (2, 129, 4, 4), (5, 300, 1, 1), (8, 1, 0, 0), (9, 2000, 4, 2)])
def test_per_view_camera_pointers_match_the_camera_array_bit_for_bit(num_views, n, deg, use):
    L = capi.lib()
    K = (deg + 1) ** 2
    means, cams, v = _views(n, num_views, 31 * num_views + n)
    bufs = [cu(v[r]) for r in range(num_views)]
    ptrs = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=DEV)
    means_d, cams_d = cu(means), cu(cams)
    trailers, cam_ptrs = _cam_pointers(cams)
    scale = 1.0 / num_views
    ref = torch.full((n, K, 3), 9.0, device=DEV)
    got = torch.full((n, K, 3), -9.0, device=DEV)
    capi.check(L.gsb_sh_backward_multiview(n, deg, use, capi.ptr(means_d), num_views, capi.ptr(cams_d),
                                           ptrs.data_ptr(), scale, capi.ptr(ref), capi.stream()))
    capi.check(L.gsb_sh_backward_multiview_cams(n, deg, use, capi.ptr(means_d), num_views, cam_ptrs.data_ptr(),
                                                ptrs.data_ptr(), scale, capi.ptr(got), capi.stream()))
    assert torch.equal(got, ref)
    assert bool((got[:, (use + 1) ** 2:, :] == 0).all())     # bases above degrees_to_use are written as zeros
    # the centres matter: moving one view's centre changes exactly the Gaussians that view sees
    if use > 0 and num_views > 1:
        trailers[0][:3] += 0.5
        moved = torch.empty_like(got)
        capi.check(L.gsb_sh_backward_multiview_cams(n, deg, use, capi.ptr(means_d), num_views, cam_ptrs.data_ptr(),
                                                    ptrs.data_ptr(), scale, capi.ptr(moved), capi.stream()))
        seen = torch.from_numpy((v[0] != 0).any(-1)).to(DEV)
        changed = (moved != got).flatten(1).any(1)
        assert bool(changed[seen].any()) and not bool(changed[~seen].any())


def test_exchange_launch_with_per_view_camera_pointers_does_both_roles():
    """One launch of gsb_exchange_gradients_cams: the multi-view SH VJP and the all-reduce role (world = 1 here, so
    the reduction is the identity times scale), both as gsb_exchange_gradients computes them."""
    L = capi.lib()
    n, deg, use, views = 3001, 3, 1, 4
    means, cams, v = _views(n, views, 5)
    bufs = [cu(v[r]) for r in range(views)]
    ptrs = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=DEV)
    means_d, cams_d = cu(means), cu(cams)
    _trailers, cam_ptrs = _cam_pointers(cams)
    out_a, out_b = torch.empty((n, 16, 3), device=DEV), torch.empty((n, 16, 3), device=DEV)
    geom_a = torch.randn(4 * 5000, device=DEV)
    g0 = geom_a.clone()
    geom_b = g0.clone()
    gpa = torch.tensor([geom_a.data_ptr()], dtype=torch.int64, device=DEV)
    gpb = torch.tensor([geom_b.data_ptr()], dtype=torch.int64, device=DEV)
    capi.check(L.gsb_exchange_gradients(n, deg, use, capi.ptr(means_d), views, capi.ptr(cams_d), ptrs.data_ptr(),
                                        0.5, capi.ptr(out_a), 0, 1, geom_a.numel(), gpa.data_ptr(), None,
                                        capi.stream()))
    capi.check(L.gsb_exchange_gradients_cams(n, deg, use, capi.ptr(means_d), views, cam_ptrs.data_ptr(),
                                             ptrs.data_ptr(), 0.5, capi.ptr(out_b), 0, 1, geom_b.numel(),
                                             gpb.data_ptr(), None, capi.stream()))
    assert torch.equal(out_a, out_b) and torch.equal(geom_b, g0 * 0.5) and torch.equal(geom_a, geom_b)
    # n = 0: the all-reduce role alone, as ViewParallelExchange.finish launches it
    capi.check(L.gsb_exchange_gradients_cams(0, deg, use, None, 1, cam_ptrs.data_ptr(), None, 2.0, None, 0, 1,
                                             geom_b.numel(), gpb.data_ptr(), None, capi.stream()))
    assert torch.equal(geom_b, g0)


def test_empty_view_backward_helpers_write_exact_zeros():
    """What a rank whose view hits nothing contributes to the data-parallel exchange: the trainer's per-view backward
    pass (rasterize-backward, project-backward) and its SH backward on such a view write zeros into the whole
    gradient buffer and the colour gradient."""
    from opensplat_b200.model import Camera
    from opensplat_b200.trainer import SplatTrainer
    from test_gpu_trainer import _cams, make_problem, refine_config
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, refine_config(), device=DEV,
                      sh_degree_interval=1)
    for step in range(1, 4):
        tr.step(cams[(step - 1) % 3], gt[(step - 1) % 3], step)
    away = c2w[0].copy()
    away[:3, :3] = away[:3, :3] @ np.diag([-1.0, 1.0, -1.0]).astype(np.float32)
    pp = tr.pipe
    tr.step(Camera(W, H, *intr, away), gt[0], 4)
    assert pp.plan.visible == 0
    pp.grad_flat.fill_(float("nan"))
    pp.v_rgbs.fill_(float("nan"))
    tr._backward_view(0, 1, intr[0], intr[1])
    tr._sh_backward(1)
    torch.cuda.synchronize()
    for name, (o, c, _) in pp.offs.items():
        assert bool((pp.grad_flat[o:o + c] == 0).all()), name
    assert bool((pp.v_rgbs == 0).all())


def _run(nproc, port, env=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tools", "check_parallel_trainer.py")], capture_output=True, text=True,
                       timeout=900, env=e)
    print(r.stdout[-4000:])
    if r.returncode != 0:
        print(r.stderr[-6000:])
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert "check_ok=True" in r.stdout
    return r.stdout


@pytest.mark.parametrize("overlap", ["1", "0"])
def test_parallel_trainer_world1_follows_gaussian_model(overlap):
    out = _run(1, 29541 if overlap == "1" else 29543, {"GSB_EXCHANGE_OVERLAP": overlap})
    assert f"overlap={overlap == '1'}" in out and "steady_allocs=0 steady_waits=10" in out


def test_parallel_trainer_2gpu_follows_gaussian_model():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run(2, 29545)
    out = _run(2, 29547, {"GSB_EXCHANGE_MULTICAST": "0"})
    assert "multicast=False" in out

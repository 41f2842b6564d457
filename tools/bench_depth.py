"""Cost of the depth and opacity maps (DESIGN D18): times the forward and backward blend launches of the plain and the
DEPTH instantiations on the same binned frame, plus the per-record depth gather, alternating the arms within one run,
and prints the medians with the card's name and power limit.
usage: python tools/bench_depth.py [workload ...] [--reps N]      (default: c2_1M_1080p_sh3 c5_5M_1440p_dense)"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import WORKLOADS  # noqa: E402
from opensplat_b200 import capi  # noqa: E402
from opensplat_b200.pipeline import SplatPipeline  # noqa: E402
from opensplat_b200.scene import make_scene  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        return q or torch.cuda.get_device_name(0)
    except Exception:
        return torch.cuda.get_device_name(0)


def run(wl, reps):
    n, W, H, scale, opac = WORKLOADS[wl]
    sc = make_scene(n, W, H, scale=scale, sh_degree=3, opacity=opac, seed=0)
    pp = SplatPipeline(n, W, H, device="cuda:0")
    pp.load_scene(sc)
    pp.target.copy_(torch.from_numpy(np.random.default_rng(1).uniform(0, 1, (H, W, 3)).astype(np.float32)))
    pp.forward_backward()
    pp.forward_backward()
    d, f32 = pp.dev, torch.float32
    od, oa = torch.empty((H, W), dtype=f32, device=d), torch.empty((H, W), dtype=f32, device=d)
    vd = torch.randn((H, W), dtype=f32, device=d)
    v_depths = torch.empty(n, dtype=f32, device=d)
    # one depth frame: the same binning as the plain frame, plus the ids and the depth stream
    pp._bin_blend(pp.p["opacities"], 0, out_depth=od, out_alpha=oa)
    L, P, s = pp.L, capi.ptr, capi.stream()
    capi.check(L.gsb_mse_loss_grad(H * W * 3, P(pp.out_img), P(pp.target), P(pp.v_img), P(pp.loss),
                                   1.0 / (H * W * 3), s))
    tb, m, order = pp.tb, pp.m_raster, P(pp.tile_order)
    common = (H, W, tb[0], tb[1], m, P(pp.tile_bins), order, P(pp.stats_dev), P(pp.background), P(pp.records),
              P(pp.out_img), P(pp.final_Ts), P(pp.final_idx), 0)
    bwd = (H, W, tb[0], tb[1], pp.n, m, P(pp.tile_bins), order, P(pp.conics), P(pp.p["opacities"]), P(pp.records),
           P(pp.cum), P(pp.background), P(pp.final_Ts), P(pp.final_idx), P(pp.v_img), None, P(pp.grad_rows),
           P(pp.v_xy), P(pp.v_conic), P(pp.v_rgbs), P(pp.g["opacities"]), 0)
    arms = {
        "fwd_plain": lambda: L.gsb_rasterize_forward_packed(*common, s),
        "fwd_depth": lambda: L.gsb_rasterize_forward_packed_depth(*common, P(pp.record_depths), P(od), P(oa), s),
        "bwd_plain": lambda: L.gsb_rasterize_backward(*bwd, s),
        "bwd_depth": lambda: L.gsb_rasterize_backward_depth(*bwd, P(pp.record_depths), P(vd), P(v_depths), s),
        "gather": lambda: L.gsb_gather_record_depths(m, P(pp.gids_sorted), P(pp.depths), P(pp.stats_dev),
                                                     P(pp.record_depths), s),
    }
    times = {k: [] for k in arms}
    for _ in range(3):
        for f in arms.values():
            capi.check(f())
    torch.cuda.synchronize()
    for r in range(reps):
        for k, f in (list(arms.items()) if r % 2 == 0 else list(arms.items())[::-1]):   # alternate the order
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            capi.check(f())
            e1.record()
            times[k].append((e0, e1))
    torch.cuda.synchronize()
    med = {k: float(np.median([a.elapsed_time(b) for a, b in v])) for k, v in times.items()}
    print(f"{wl}: n={n} {W}x{H} M={pp.m} reps={reps}  " + "  ".join(f"{k}={v:.4f} ms" for k, v in med.items())
          + f"  fwd +{100 * (med['fwd_depth'] / med['fwd_plain'] - 1):.1f}%"
          + f"  bwd +{100 * (med['bwd_depth'] / med['bwd_plain'] - 1):.1f}%")


if __name__ == "__main__":
    args = sys.argv[1:]
    reps = 30
    if "--reps" in args:
        i = args.index("--reps")
        reps = int(args[i + 1])
        del args[i:i + 2]
    print("card:", card())
    for wl in args or ["c2_1M_1080p_sh3", "c5_5M_1440p_dense"]:
        run(wl, reps)
        torch.cuda.empty_cache()

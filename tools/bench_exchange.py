"""torchrun --nproc-per-node N tools/bench_exchange.py [--n 1000000] [--reps 30]
Times the data-parallel exchange step ALONE on N GPUs (CUDA events on the launching stream, max over ranks):
  * the fused launch `gsb_exchange_gradients` (multi-view SH backward over peer loads + two-shot all-reduce of the
    geometry gradients), with and without its two cross-rank barriers, multimem and peer-pointer flavours;
  * the baseline: sh_backward + ONE NCCL all-reduce of the flat gradient buffer;
and reports the achieved NVLink rate against the bytes the design says must cross the links
((G-1) x 12 B colour gradients pulled + the geometry slices), plus the NVLink byte counters nvidia-smi exposes
(`nvidia-smi nvlink -gt d`), read before and after the fused loop on rank 0's GPU.  ncu cannot wrap a multi-rank
command, so this is the exchange kernel's evidence."""
import argparse, json, os, re, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist
from opensplat_b200 import capi
from opensplat_b200.multigpu import ViewParallelExchange
from opensplat_b200.pipeline import SplatPipeline
from opensplat_b200.scene import make_scene, cube_view_camera


def nvlink_kib(gpu):
    """Sum of the per-link data counters (tx, rx) in KiB, or None if the tool / counters are unavailable."""
    try:
        out = subprocess.run(["nvidia-smi", "nvlink", "-gt", "d", "-i", str(gpu)], capture_output=True, text=True,
                             timeout=20).stdout
        tx = sum(int(v) for v in re.findall(r"Data Tx:\s*(\d+)\s*KiB", out))
        rx = sum(int(v) for v in re.findall(r"Data Rx:\s*(\d+)\s*KiB", out))
        return (tx, rx) if (tx or rx) else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    n, W, H = a.n, 1920, 1080
    sc = make_scene(n, W, H, scale=0.02, sh_degree=3, opacity=(0.05, 0.95), seed=0)
    cam = cube_view_camera(W, H, rank)
    pipe = SplatPipeline(n, W, H, device=dev)
    pipe.load_scene(sc)
    pipe.set_camera(cam)
    vd = sc["means"] - cam["cam_pos"]
    pipe.viewdirs.copy_(torch.from_numpy((vd / np.linalg.norm(vd, axis=-1, keepdims=True)).astype(np.float32)).to(dev))
    res = {"world": world, "gaussians": n}
    L = capi.lib()

    def timed(fn, reps):
        dist.barrier(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        dist.barrier(); torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1) / reps], device=dev)
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms[0])

    for flavour in ("multimem", "peer"):
        os.environ["GSB_EXCHANGE_MULTICAST"] = "1" if flavour == "multimem" else "0"
        ex = ViewParallelExchange(pipe, cam["cam_pos"])
        if flavour == "multimem" and not ex.multicast_ptr:
            res[flavour] = "no multicast mapping on this box"
            continue
        g = torch.Generator(device=dev).manual_seed(rank)
        ex.v_rgb.copy_(torch.randn(n, 3, device=dev, generator=g))
        pipe.grad_flat[:pipe.geom_numel].copy_(torch.randn(pipe.geom_numel, device=dev, generator=g))
        pipe.rgbs.fill_(1.0)

        def launch_only():
            capi.check(L.gsb_exchange_gradients(
                n, pipe.deg, pipe.deg, capi.ptr(pipe.p["means"]), world, capi.ptr(ex.cam_positions),
                ex.rgb_ptrs.data_ptr(), 1.0, capi.ptr(pipe.g["coeffs"]), rank, world, ex.geom_numel,
                ex.geom_ptrs.data_ptr(), ex.multicast_ptr if ex.multicast_ptr else None, capi.stream()))

        def geom_only():
            capi.check(L.gsb_exchange_gradients(
                0, pipe.deg, pipe.deg, None, 1, capi.ptr(ex.cam_positions), None, 1.0, None, rank, world,
                ex.geom_numel, ex.geom_ptrs.data_ptr(), ex.multicast_ptr if ex.multicast_ptr else None, capi.stream()))

        def two_streams():     # the pipeline's form: colour half on a side stream, geometry half on the main one
            cur = torch.cuda.current_stream()
            ex.side.wait_stream(cur)
            capi.check(L.gsb_sh_backward_multiview(n, pipe.deg, pipe.deg, capi.ptr(pipe.p["means"]), world,
                                                   capi.ptr(ex.cam_positions), ex.rgb_ptrs.data_ptr(), 1.0,
                                                   capi.ptr(pipe.g["coeffs"]), ex.side.cuda_stream))
            geom_only()
            cur.wait_stream(ex.side)

        def sh_only():
            capi.check(L.gsb_sh_backward_multiview(n, pipe.deg, pipe.deg, capi.ptr(pipe.p["means"]), world,
                                                   capi.ptr(ex.cam_positions), ex.rgb_ptrs.data_ptr(), 1.0,
                                                   capi.ptr(pipe.g["coeffs"]), capi.stream()))
        for _ in range(3):
            ex.exchange(average=False)
        before = nvlink_kib(local) if rank == 0 else None
        full = timed(lambda: ex.exchange(average=False), a.reps)        # mask + barrier + launch + barrier
        after = nvlink_kib(local) if rank == 0 else None
        k_only = timed(launch_only, a.reps)                               # (values grow; timing only)
        sh = timed(sh_only, a.reps)
        go = timed(geom_only, a.reps)
        ts = timed(two_streams, a.reps)
        bar = timed(lambda: ex.hdl.barrier(channel=0), a.reps)
        rgb_bytes = (world - 1) * 12 * n
        geom_bytes = ex.geom_numel * 4
        # bytes this rank RECEIVES: peers' colour gradients + its reduced slice (summed in the switch or pulled from
        # G-1 peers) + the other ranks' reduced slices
        recv = rgb_bytes + (geom_bytes if flavour == "multimem" else geom_bytes // world * (world - 1) * 2)
        r = {"step_ms_mask_barrier_launch_barrier": full, "launch_only_ms": k_only, "sh_half_only_ms": sh,
             "geometry_half_only_ms": go, "two_streams_ms": ts, "barrier_ms": bar, "bytes_received_per_rank_model": recv,
             "nvlink_GBps_achieved_launch_only": recv / (k_only * 1e-3) / 1e9,
             "nvlink_GBps_colour_pull_only": rgb_bytes / (sh * 1e-3) / 1e9,
             "nvlink_reference_GBps": 450.0,   # H100 SXM data sheet: NVLink 4, 450 GB/s per direction
             "local_hbm_write_bytes": 192 * n}
        if before and after:
            r["nvidia_smi_nvlink_rx_bytes_per_step"] = (after[1] - before[1]) * 1024 / a.reps
            r["nvidia_smi_nvlink_tx_bytes_per_step"] = (after[0] - before[0]) * 1024 / a.reps
        res[flavour] = r
        del ex
    # baseline: sh_backward + one NCCL all-reduce of the flat gradient buffer
    def baseline():
        capi.check(L.gsb_sh_backward_rgb(n, pipe.deg, pipe.deg, capi.ptr(pipe.viewdirs), capi.ptr(pipe.rgbs),
                                         capi.ptr(pipe.v_rgbs), capi.ptr(pipe.g["coeffs"]), capi.stream()))
        dist.all_reduce(pipe.grad_flat, op=dist.ReduceOp.SUM)
    for _ in range(3):
        baseline()
    res["nccl_flat_allreduce"] = {"step_ms": timed(baseline, a.reps), "bytes_allreduced": pipe.numel * 4}
    if rank == 0:
        print(json.dumps(res))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

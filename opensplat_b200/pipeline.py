"""Allocation-free driver of the full render path (SH -> project -> bin/sort -> blend -> loss ->
blend bwd -> project bwd -> SH bwd [-> allreduce -> Adam]) on top of the C ABI.

This is host-side plumbing: it owns the device buffers (torch tensors), sizes the M-dependent
workspaces from a high-water mark, and issues the C-ABI calls on the current stream in the order the
reference's simple_trainer.cpp:150-203 / model.cpp:83-225 issue their operators.  It is what bench.py
times for `value`; the autograd operators in ops.py give the same numbers through torch.autograd.

Gradients of all per-Gaussian parameters are written into slices of ONE flat fp32 buffer
(`grad_flat`, 59 floats per Gaussian at SH degree 3) so that data-parallel training needs a single
NCCL all-reduce per step (SURVEY.md section 8e).
"""
import os

import torch

from . import capi, ops
from .ops import tile_bounds, num_sh_bases, BinPlan
from .parallel import flat_layout


class SplatPipeline:
    def __init__(self, n, W, H, sh_degree=3, device="cuda:0", m_capacity=None, stage_timing=False):
        self.n, self.W, self.H, self.deg = int(n), int(W), int(H), int(sh_degree)
        self.K = num_sh_bases(sh_degree)
        self.dev = torch.device(device)
        self.tb = tile_bounds(W, H)
        self.T = self.tb[0] * self.tb[1]
        self.L = capi.lib()
        d, f32, i32 = self.dev, torch.float32, torch.int32
        self._alloc_gaussians(self.n)
        # ---- per-pixel ----
        self.out_img = torch.empty((H, W, 3), dtype=f32, device=d)
        self.final_Ts = torch.empty((H, W), dtype=f32, device=d)
        self.final_idx = torch.empty((H, W), dtype=i32, device=d)
        self.v_img = torch.empty((H, W, 3), dtype=f32, device=d)
        self.target = torch.zeros((H, W, 3), dtype=f32, device=d)
        self.background = torch.zeros(3, dtype=f32, device=d)
        self.loss = torch.zeros(1, dtype=f32, device=d)
        self.tile_bins = torch.empty((self.T, 2), dtype=i32, device=d)
        self.tile_order = torch.empty((self.T,), dtype=i32, device=d)   # longest-first tile order (fast path)
        self.stats_dev = torch.zeros(4, dtype=i32, device=d)
        self.plan = BinPlan()   # capacities of the M-dependent buffers, carried from frame to frame
        # ---- camera ----
        self.viewmat = torch.eye(4, dtype=f32, device=d)
        self.projmat = torch.eye(4, dtype=f32, device=d)
        self.intr = (1.0, 1.0, 0.0, 0.0)
        # ---- M-dependent (grown on demand) ----
        self.m = 0
        self.m_raster = 0
        if m_capacity:
            self.plan.grow(int(m_capacity), 0)
        self.nvtx = os.environ.get("GSB_NVTX", "0") == "1"
        self._nvtx_open = False
        self.exchange = None  # multigpu.ViewParallelExchange (fused SH backward + NVLink exchange)
        self.stage_timing = stage_timing
        self.stage_ms = {}
        self._ev = []
        self._steps_ev = []

    def _alloc_gaussians(self, n):
        """(Re)allocates everything sized by the Gaussian count: the flat parameter / gradient buffers with their
        per-tensor views, Adam state (dropped), and the per-Gaussian intermediates.  Called by __init__ and after a
        refinement changed the count (resize_gaussians)."""
        self.n = n = int(n)
        d, f32, i32 = self.dev, torch.float32, torch.int32
        # ---- parameters: one flat buffer, views per tensor (same layout for grads / Adam state); every slice
        # starts on a 16-byte boundary (parallel.flat_layout) whatever n is, so the 128-bit accesses of the
        # projection kernels stay legal after a refinement left an odd Gaussian count
        self.offs, self.numel = flat_layout(n, self.K)
        self.sizes = [(name, shp) for name, (o, c, shp) in self.offs.items()]
        self.geom_numel = self.offs["coeffs"][0]   # means, scales, quats, opacities: the prefix before the SH block
        self.param_flat = torch.zeros(self.numel, dtype=f32, device=d)
        self.grad_flat = self._alloc_grad_flat(self.numel)
        self.p, self.g = {}, {}
        for name, (o, c, shp) in self.offs.items():
            self.p[name] = self.param_flat[o:o + c].view(shp)
            self.g[name] = self.grad_flat[o:o + c].view(shp)
        self.adam_m = self.adam_v = None
        self.adam_t = 0
        # ---- per-Gaussian intermediates ----
        self.viewdirs = torch.zeros((n, 3), dtype=f32, device=d)
        self.colors = torch.empty((n, 3), dtype=f32, device=d)
        self.rgbs = torch.empty((n, 3), dtype=f32, device=d)
        self.cov3d = torch.empty((n, 6), dtype=f32, device=d)
        self.xys = torch.empty((n, 2), dtype=f32, device=d)
        self.depths = torch.empty((n,), dtype=f32, device=d)
        self.radii = torch.empty((n,), dtype=i32, device=d)
        self.conics = torch.empty((n, 3), dtype=f32, device=d)
        self.nth = torch.empty((n,), dtype=i32, device=d)
        self.cum = torch.empty((n,), dtype=i32, device=d)
        self.v_xy = torch.empty((n, 2), dtype=f32, device=d)
        self.v_conic = torch.empty((n, 3), dtype=f32, device=d)
        self.v_rgbs = torch.empty((n, 3), dtype=f32, device=d)
        self.max_len = 0
        self.m_cap = -1   # the M-sized buffers (and the n-sized bucket workspace) are (re)built by the next forward

    def _alloc_grad_flat(self, numel):
        """The flat gradient buffer; multigpu.ViewParallelExchange re-binds it to symmetric (peer-mapped) memory."""
        return torch.zeros(numel, dtype=torch.float32, device=self.dev)

    def rebind_grad_flat(self, flat):
        """Adopt `flat` (same numel; e.g. a symmetric-memory tensor) as the gradient buffer."""
        assert flat.numel() == self.numel and flat.dtype == torch.float32
        self.grad_flat = flat
        for name, (o, c, shp) in self.offs.items():
            self.g[name] = self.grad_flat[o:o + c].view(shp)

    # ------------------------------------------------------------------------------------------
    def _grow(self, m_cap):
        """(Re)allocates the buffers sized by the intersection capacity of the fast path."""
        d = self.dev
        self.records = torch.empty(self.L.gsb_raster_records_bytes(m_cap), dtype=torch.uint8, device=d)
        self.grad_rows = torch.empty(self.L.gsb_raster_grad_rows_bytes(m_cap), dtype=torch.uint8, device=d)
        self.bucket_ws = torch.empty(self.L.gsb_bucket_workspace_bytes(self.n, m_cap, self.T) + 256,
                                     dtype=torch.uint8, device=d)
        self.m_cap = m_cap

    def load_scene(self, sc):
        """sc: dict from opensplat_b200.scene.make_scene (numpy)."""
        for k in ("means", "scales", "quats", "opacities", "coeffs"):
            self.p[k].copy_(torch.from_numpy(sc[k]).to(self.dev))
        self.viewdirs.copy_(torch.from_numpy(sc["viewdirs"]).to(self.dev))
        self.set_camera(sc)

    def set_camera(self, cam):
        self.viewmat.copy_(torch.as_tensor(cam["viewmat"]).to(self.dev))
        self.projmat.copy_(torch.as_tensor(cam["projmat"]).to(self.dev))
        self.intr = (float(cam["fx"]), float(cam["fy"]), float(cam["cx"]), float(cam["cy"]))

    # ------------------------------------------------------------------------------------------
    def _stage(self, name):
        if self.nvtx:   # GSB_NVTX=1: one NVTX range per stage (nsys / ncu --nvtx)
            if self._nvtx_open:
                torch.cuda.nvtx.range_pop()
            self._nvtx_open = not name.startswith("end_")
            if self._nvtx_open:
                torch.cuda.nvtx.range_push("gsb:" + name)
        if self.stage_timing:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self._ev.append((name, e))

    def _collect(self):
        """End of one step: park this step's events; they are resolved by resolve_stage_times() after
        the timed region (no synchronisation inside it)."""
        if self.stage_timing and len(self._ev) >= 2:
            self._steps_ev.append(self._ev)
        self._ev = []

    def resolve_stage_times(self):
        torch.cuda.synchronize()
        for ev in self._steps_ev:
            for (n0, e0), (_, e1) in zip(ev[:-1], ev[1:]):
                self.stage_ms.setdefault(n0, []).append(e0.elapsed_time(e1))
        self._steps_ev = []
        return {k: sum(v) / len(v) for k, v in self.stage_ms.items() if not k.startswith("end_")}

    def forward(self):
        L, P, s = self.L, capi.ptr, capi.stream()
        n, W, H = self.n, self.W, self.H
        fx, fy, cx, cy = self.intr
        p = self.p
        self._stage("sh_fwd")
        # SH colour with the glue of model.cpp:192 fused: rgbs = clamp_min(colors + 0.5, 0)
        capi.check(L.gsb_sh_forward_rgb(n, self.deg, self.deg, P(self.viewdirs), P(p["coeffs"]), 0.5, P(self.rgbs), s))
        self._stage("project_fwd")
        capi.check(L.gsb_project_forward(n, P(p["means"]), P(p["scales"]), 1.0, P(p["quats"]), P(self.viewmat),
                                         P(self.projmat), fx, fy, cx, cy, H, W, self.tb[0], self.tb[1], 0.01,
                                         P(self.cov3d), P(self.xys), P(self.depths), P(self.radii), P(self.conics),
                                         P(self.nth), s))
        limit = L.gsb_bucket_max_tile_len()
        plan = self.plan
        # Everything below is sized by capacities planned from earlier frames and enqueued WITHOUT waiting for the
        # path's one device->host read-back (M, rasterize_gaussians.cpp:63): the host looks at it after the blend
        # kernel has been enqueued (the GPU never idles) and redoes a frame that outgrew the plan.
        while True:
            if plan.m_cap != self.m_cap:
                self._grow(plan.m_cap)
            m_cap, len_cap = plan.m_cap, plan.len_cap
            boff = (-self.bucket_ws.data_ptr()) % 256
            wsp, wsb = self.bucket_ws.data_ptr() + boff, self.bucket_ws.numel() - boff
            self._stage("scan")
            # cull = 1: bin only (Gaussian, tile) pairs whose extent box touches the tile
            capi.check(L.gsb_bucket_tile_ranges(n, P(self.xys), P(self.radii), P(self.conics), P(self.rgbs),
                                                P(p["opacities"]), 1, self.tb[0], self.tb[1], m_cap, len_cap, wsp, wsb,
                                                P(self.cum), P(self.tile_bins), P(self.tile_order), P(self.stats_dev),
                                                s))
            plan.read_back(self.stats_dev)
            if m_cap > 0:
                self._stage("bucket_sort_pack")
                capi.check(L.gsb_bucket_sort_pack(n, m_cap, len_cap, P(self.depths), P(self.radii), P(self.cum), 1,
                                                  self.tb[0], self.tb[1], P(self.tile_bins), P(self.stats_dev), wsp,
                                                  wsb, P(self.records), None, None, s))
            self._stage("raster_fwd")
            capi.check(L.gsb_rasterize_forward_packed(H, W, self.tb[0], self.tb[1], m_cap, P(self.tile_bins),
                                                      P(self.tile_order), P(self.stats_dev), P(self.background),
                                                      P(self.records), P(self.out_img), P(self.final_Ts),
                                                      P(self.final_idx), 0, s))
            self._stage("end_fwd")
            self.m, self.max_len, overflow = plan.wait()
            if not overflow:
                self.m_raster = m_cap
                self._ordered = True
                return self.out_img
            self._ev = []            # the frame is redone: drop its stage events
            if self.max_len > limit:
                break                # pathological tile lists: generic path below
            plan.grow(self.m, self.max_len)
        # ---- generic path: reference-exact global sort (binAndSortGaussians) of the unculled lists, with the M
        # read-back in the middle
        self._stage("generic_bin")
        self.cum = ops.cumsum_tiles_hit(self.nth)
        m = self.m = int(self.cum[-1])
        if L.gsb_raster_records_bytes(m) > self.records.numel():
            self._grow(int(m * 1.25) + 1024)
            self.plan.m_cap = self.m_cap
        _, _, _, gids_sorted, self.tile_bins, sorted_index = ops.binAndSortGaussians(
            n, m, self.xys, self.depths, self.radii, self.cum, self.tb, return_index=True)
        self._stage("raster_fwd")
        capi.check(L.gsb_pack_records(m, P(gids_sorted), P(sorted_index), P(self.xys), P(self.conics), P(self.rgbs),
                                      P(p["opacities"]), P(self.records), s))
        capi.check(L.gsb_rasterize_forward_packed(H, W, self.tb[0], self.tb[1], m, P(self.tile_bins), None, None,
                                                  P(self.background), P(self.records), P(self.out_img),
                                                  P(self.final_Ts), P(self.final_idx), 0, s))
        self.m_raster = m
        self._ordered = False
        self._stage("end_fwd")
        return self.out_img

    def backward(self):
        """MSE loss against self.target + the whole backward path; grads land in self.grad_flat."""
        L, P, s = self.L, capi.ptr, capi.stream()
        n, W, H, m = self.n, self.W, self.H, self.m_raster   # m: what the records buffer was sized with
        fx, fy, cx, cy = self.intr
        p, g = self.p, self.g
        cnt = H * W * 3
        self._stage("loss")
        capi.check(L.gsb_mse_loss_grad(cnt, P(self.out_img), P(self.target), P(self.v_img), P(self.loss), 1.0 / cnt, s))
        v_rgbs = self.exchange.v_rgbs_buffer() if self.exchange is not None else self.v_rgbs
        self._stage("raster_bwd")
        capi.check(L.gsb_rasterize_backward(H, W, self.tb[0], self.tb[1], n, m, P(self.tile_bins),
                                    P(self.tile_order) if self._ordered else None, P(self.conics),
                                    P(p["opacities"]), P(self.records), P(self.cum), P(self.background),
                                    P(self.final_Ts), P(self.final_idx),
                                    P(self.v_img), None, P(self.grad_rows), P(self.v_xy), P(self.v_conic),
                                    P(v_rgbs), P(g["opacities"]), 0, s))
        if self.exchange is not None and self.exchange.overlap:
            self.exchange.start_colour(average=True)   # colour pulls + SH expansion start now, on a side stream
        self._stage("project_bwd")
        capi.check(L.gsb_project_backward(n, P(p["means"]), P(p["scales"]), 1.0, P(p["quats"]), P(self.viewmat),
                                          P(self.projmat), fx, fy, cx, cy, H, W, None, P(self.radii), P(self.conics),
                                          P(self.v_xy), None, P(self.v_conic), P(g["means"]), P(g["scales"]),
                                          P(g["quats"]), s))
        self._stage("sh_bwd")
        if self.exchange is not None:
            # data-parallel: SH VJP fused with the cross-GPU exchange (also all-reduces the geometry grads)
            if self.exchange.overlap:
                self.exchange.finish()
            else:
                self.exchange.exchange(average=True)
        else:
            # SH VJP with the gradient of the clamp fused (mask = forward rgbs > 0)
            capi.check(L.gsb_sh_backward_rgb(n, self.deg, self.deg, P(self.viewdirs), P(self.rgbs), P(self.v_rgbs),
                                             P(g["coeffs"]), s))
        self._stage("end_bwd")
        return self.loss

    def forward_backward(self):
        self.forward()
        loss = self.backward()
        self._collect()
        return loss

    def adam_step(self, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8):
        if self.adam_m is None:
            self.adam_m = torch.zeros_like(self.param_flat)
            self.adam_v = torch.zeros_like(self.param_flat)
        self.adam_t += 1
        t = self.adam_t
        capi.check(self.L.gsb_adam_step(self.numel, capi.ptr(self.param_flat), capi.ptr(self.grad_flat),
                                        capi.ptr(self.adam_m), capi.ptr(self.adam_v), lr, b1, b2, eps,
                                        1.0 - b1 ** t, 1.0 - b2 ** t, capi.stream()))

    def train_step(self, world_size=1, lr=1e-3):
        """fwd + bwd (+ one NCCL all-reduce of the flat per-Gaussian gradient buffer) + fused Adam."""
        self.forward()
        loss = self.backward()
        if world_size > 1 and self.exchange is None:
            import torch.distributed as dist
            dist.all_reduce(self.grad_flat, op=dist.ReduceOp.SUM)
            self.grad_flat.mul_(1.0 / world_size)
        self.adam_step(lr=lr)
        self._collect()
        return loss

    # ---- changing the Gaussian count (after topology edits, densify.Densifier / model.GaussianModel) ------------
    def resize_gaussians(self, params, adam_m=None, adam_v=None):
        """Adopts a new Gaussian set (dicts keyed like self.p; leading dimension = new count): re-allocates the
        n-sized buffers and copies parameters and Adam moments into the new flat layout."""
        t = self.adam_t
        self._alloc_gaussians(params["means"].shape[0])
        self.adam_t = t
        for k in self.p:
            self.p[k].copy_(params[k].view(self.p[k].shape))
        if adam_m is not None and adam_v is not None:
            self.adam_m = torch.zeros_like(self.param_flat)
            self.adam_v = torch.zeros_like(self.param_flat)
            for name, (o, c, shp) in self.offs.items():
                self.adam_m[o:o + c].copy_(adam_m[name].reshape(-1))
                self.adam_v[o:o + c].copy_(adam_v[name].reshape(-1))
        if self.exchange is not None:
            self.exchange.resize(self)

    def tile_occupancy(self, nbins=16):
        """Diagnostic (SURVEY.md section 5): histogram of the tile-list lengths of the last frame (binned lists).
        Host-side, outside any timed region."""
        tb = self.tile_bins.cpu().numpy()
        lens = (tb[:, 1] - tb[:, 0]).astype("int64")
        import numpy as np
        mx = int(lens.max()) if lens.size else 0
        edges = np.linspace(0, max(mx, 1), nbins + 1)
        hist, _ = np.histogram(lens, bins=edges)
        q = np.percentile(lens, [50, 90, 99]) if lens.size else [0, 0, 0]
        return {"tiles": int(lens.size), "empty_tiles": int((lens == 0).sum()), "mean": float(lens.mean()),
                "p50": float(q[0]), "p90": float(q[1]), "p99": float(q[2]), "max": mx,
                "hist_edges": [round(float(e), 1) for e in edges], "hist": [int(h) for h in hist]}

    # algorithmic HBM bytes of the path for the last step (SURVEY.md 8d / BASELINE.md section 4)
    def algorithmic_bytes(self):
        n, m, P, T, K = self.n, self.m, self.W * self.H, self.T, self.K
        tile_bits = max(1, (T - 1).bit_length())
        passes = (32 + tile_bits + 7) // 8
        stages = {
            "sh_fwd": n * (12 + 12 * K + 12),
            "project_fwd": 96 * n,
            "scan": 8 * n,
            "emit": 20 * n + 12 * m,
            "sort": 8 * m + passes * 24 * m,
            "bins": 8 * m + 8 * T,
            "raster_fwd": 40 * m + 20 * P,
            "raster_bwd": 40 * m + 20 * P + 36 * n,
            "project_bwd": 144 * n,
            "sh_bwd": n * (12 + 12 * K + 12),
        }
        return stages, passes

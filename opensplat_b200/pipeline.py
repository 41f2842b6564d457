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

from . import capi
from .ops import tile_bounds, num_sh_bases, BinFrame, BinPlan
from .parallel import flat_layout


class SplatPipeline(BinFrame):
    """One BinFrame reused from frame to frame, on a plan of its own, plus every buffer of the render path."""

    def __init__(self, n, W, H, sh_degree=3, device="cuda:0", m_capacity=None, stage_timing=False):
        super().__init__(BinPlan(), device)
        self.n, self.deg = int(n), int(sh_degree)
        self.K = num_sh_bases(sh_degree)
        d, f32 = self.dev, torch.float32
        self._alloc_gaussians(self.n)
        self._alloc_pixels(W, H)
        self.background = torch.zeros(3, dtype=f32, device=d)
        self.loss = torch.zeros(1, dtype=f32, device=d)
        # ---- camera ----
        self.viewmat = torch.eye(4, dtype=f32, device=d)
        self.projmat = torch.eye(4, dtype=f32, device=d)
        self.intr = (1.0, 1.0, 0.0, 0.0)
        if m_capacity:
            self.plan.grow(int(m_capacity), 0)
        self.nvtx = os.environ.get("GSB_NVTX", "0") == "1"
        self._nvtx_open = False
        self.exchange = None  # multigpu.ViewParallelExchange (fused SH backward + NVLink exchange)
        self.stage_timing = stage_timing
        self.stage_ms = {}
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
        self.v_xy = torch.empty((n, 2), dtype=f32, device=d)
        self.v_conic = torch.empty((n, 3), dtype=f32, device=d)
        self.v_rgbs = torch.empty((n, 3), dtype=f32, device=d)
        self.max_len = 0
        self.m_cap = -1   # the frame's n-sized buffers are (re)built by the next forward

    def _alloc_pixels(self, W, H):
        """(Re)allocates everything sized by the image: the per-pixel buffers (the frame's tile-sized ones follow).
        Called by __init__ and when a trainer's downscale schedule changes the render resolution."""
        self.W, self.H = int(W), int(H)
        self.tb = tile_bounds(self.W, self.H)
        self.T = self.tb[0] * self.tb[1]
        d, f32, i32 = self.dev, torch.float32, torch.int32
        H, W = self.H, self.W
        self.out_img = torch.empty((H, W, 3), dtype=f32, device=d)
        self.final_Ts = torch.empty((H, W), dtype=f32, device=d)
        self.final_idx = torch.empty((H, W), dtype=i32, device=d)
        self.v_img = torch.empty((H, W, 3), dtype=f32, device=d)
        self.target = torch.zeros((H, W, 3), dtype=f32, device=d)
        self.m_cap = -1   # the frame's tile-sized buffers are (re)built by the next forward

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
    def _grow(self, m_cap, n, T):
        """The frame's buffers and the backward blend kernel's per-record gradient rows (_raster_backward)."""
        super()._grow(m_cap, n, T)
        self.grad_rows = torch.empty(self.L.gsb_raster_grad_rows_bytes(m_cap), dtype=torch.uint8, device=self.dev)

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
        return self._bin_blend(p["opacities"], 0)

    def _bin_blend(self, opacities, flags, count_visible=False, rgbs=None, out_img=None, out_depth=None,
                   out_alpha=None, depth_values=None):
        """bin_blend on the pipeline's projection and pixel buffers.  opacities: the [n] opacities the blend uses;
        rgbs: the [n,3] colours the records carry (default self.rgbs; a trainer with several views per step passes the
        view's); out_img: the image (default self.out_img); out_depth / out_alpha / depth_values: bin_blend's depth
        output and the per-Gaussian value it blends (default self.depths)."""
        return self.bin_blend(self.xys, self.radii, self.conics, self.depths, self.nth,
                              self.rgbs if rgbs is None else rgbs, opacities, self.background,
                              self.out_img if out_img is None else out_img, self.final_Ts, self.final_idx, flags,
                              count_visible, out_depth=out_depth, out_alpha=out_alpha, depth_values=depth_values)

    def _raster_backward(self, opacities, v_opacities, v_rgbs, flags):
        """The blend kernel's backward of the last frame (_bin_blend's), from the gradient of its image in self.v_img
        into self.v_xy / self.v_conic, `v_rgbs` ([n,3]) and `v_opacities` ([n]).  opacities: the ones the blend used;
        flags: the ones it was launched with.  The frame's binning state is read here, so callers need not know it:
        which path produced the frame (only the fast path leaves a tile order), the records and the capacity they
        were sized with, the per-pixel state of the blend."""
        P = capi.ptr
        capi.check(self.L.gsb_rasterize_backward(
            self.H, self.W, self.tb[0], self.tb[1], self.n, self.m_raster, P(self.tile_bins),
            P(self.tile_order) if self._ordered else None, P(self.conics), P(opacities), P(self.records), P(self.cum),
            P(self.background), P(self.final_Ts), P(self.final_idx), P(self.v_img), None, P(self.grad_rows),
            P(self.v_xy), P(self.v_conic), P(v_rgbs), P(v_opacities), flags, capi.stream()))

    def _raster_backward_depth(self, opacities, v_opacities, v_rgbs, flags, v_output_depth, v_depths):
        """_raster_backward of a depth frame (_bin_blend with out_depth): the same outputs plus, from the gradient of
        its depth map in `v_output_depth` ([H,W]), the gradient of the per-Gaussian value it blended into `v_depths`
        ([n]), through the frame's record_depths.  The opacity map gets no cotangent."""
        P = capi.ptr
        capi.check(self.L.gsb_rasterize_backward_depth(
            self.H, self.W, self.tb[0], self.tb[1], self.n, self.m_raster, P(self.tile_bins),
            P(self.tile_order) if self._ordered else None, P(self.conics), P(opacities), P(self.records), P(self.cum),
            P(self.background), P(self.final_Ts), P(self.final_idx), P(self.v_img), None, P(self.grad_rows),
            P(self.v_xy), P(self.v_conic), P(v_rgbs), P(v_opacities), flags, P(self.record_depths),
            P(v_output_depth), P(v_depths), capi.stream()))

    def backward(self):
        """MSE loss against self.target + the whole backward path; grads land in self.grad_flat."""
        L, P, s = self.L, capi.ptr, capi.stream()
        n, W, H = self.n, self.W, self.H
        fx, fy, cx, cy = self.intr
        p, g = self.p, self.g
        cnt = H * W * 3
        self._stage("loss")
        capi.check(L.gsb_mse_loss_grad(cnt, P(self.out_img), P(self.target), P(self.v_img), P(self.loss), 1.0 / cnt, s))
        v_rgbs = self.exchange.v_rgbs_buffer() if self.exchange is not None else self.v_rgbs
        self._stage("raster_bwd")
        self._raster_backward(p["opacities"], g["opacities"], v_rgbs, 0)
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
            # SH VJP with the gradient of the clamp fused (mask = forward rgbs > 0 or -0, the exact tie: D17)
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

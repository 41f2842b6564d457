"""Times the stages of one step for a given library variant (GSB_LIB=path) -- used to A/B kernel variants.
usage: GSB_LIB=... python tools/bench_blend.py [workload] [reps]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from bench import WORKLOADS
from opensplat_b200.pipeline import SplatPipeline
from opensplat_b200.scene import make_scene

wl = sys.argv[1] if len(sys.argv) > 1 else "c2_1M_1080p_sh3"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
n, W, H, scale, opac = WORKLOADS[wl]
sc = make_scene(n, W, H, scale=scale, sh_degree=3, opacity=opac, seed=0)
pipe = SplatPipeline(n, W, H, device="cuda:0", stage_timing=True)
pipe.load_scene(sc)
pipe.target.copy_(torch.from_numpy(np.random.default_rng(1).uniform(0, 1, (H, W, 3)).astype(np.float32)))
for _ in range(5):
    pipe.forward_backward()
pipe.resolve_stage_times(); pipe.stage_ms.clear()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    pipe.forward_backward()
e1.record()
st = pipe.resolve_stage_times()
print(os.environ.get("GSB_LIB", "default"), wl, f"step {e0.elapsed_time(e1)/reps:.4f} ms  M={pipe.m}",
      " ".join(f"{k}={v:.4f}" for k, v in st.items()))

"""Builds oracle/_ref/libopensplat_ref_points.so (test artefact, not product): the reference's UNMODIFIED Model
constructor (model.cpp / model.hpp, CPU build) with the driver tests/native/points_driver.cpp, exposed as
torch.ops.opensplat_ref_points.init_model.  It pins oracle/points_init.py's restatement of the constructor.

The reference objects are the ones oracle/Makefile already compiles into oracle/_ref/obj/ (model.o and the
translation units it links against); only the driver is compiled here.  Only possible where the reference checkout
exists; the library travels with oracle/_ref/."""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OBJ = os.path.join(ROOT, "oracle", "_ref", "obj")
OUT = os.path.join(ROOT, "oracle", "_ref", "libopensplat_ref_points.so")
REF_OBJS = ["model.o", "tensor_math.o", "optim_scheduler.o", "gsplat_cpu.o", "project_gaussians.o",
            "rasterize_gaussians.o", "spherical_harmonics.o", "ssim.o"]


def build(force=False):
    if not os.path.exists(os.path.join(REF, "model.cpp")):
        return OUT if os.path.exists(OUT) else None
    sys.path.insert(0, ROOT)
    from oracle import ref
    ref.build()                                   # oracle/Makefile: the reference objects
    objs = [os.path.join(OBJ, o) for o in REF_OBJS]
    missing = [o for o in objs if not os.path.exists(o)]
    if missing:
        raise RuntimeError(f"reference objects not built: {missing}")
    driver = os.path.join(ROOT, "tests", "native", "points_driver.cpp")
    deps = objs + [driver, __file__]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    from opensplat_b200 import build_ops
    T = os.path.dirname(torch.__file__)
    flags = ["-std=c++17", "-O2", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1", "-w", f"-I{T}/include",
             f"-I{T}/include/torch/csrc/api/include", f"-I{os.path.join(ROOT, 'shims', 'model_deps')}", f"-I{REF}",
             f"-I{REF}/rasterizer"]
    cxx = os.environ.get("CXX", "g++")
    drv_obj = os.path.join(OBJ, "points_driver.o")
    r = subprocess.run([cxx] + flags + ["-c", driver, "-o", drv_obj], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"compile failed for {driver}:\n{r.stderr[-6000:]}")
    cmd = [cxx, "-shared", "-o", OUT] + objs + [drv_obj] + build_ops.shared_stdcxx_flags() + [
        f"-L{T}/lib", f"-Wl,-rpath,{T}/lib", "-ltorch", "-ltorch_cpu", "-lc10"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stderr[-6000:])
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))

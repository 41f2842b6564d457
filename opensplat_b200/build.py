"""In-tree build of libgsplat_b200.so (sm_90a only) with nvcc.  `python -m opensplat_b200.build`.

The kernels are torch-free .cu files behind the C ABI in include/gsplat_b200.h, so each translation
unit compiles in seconds.  project.cu is built with --fmad=false (bit-exact integer artefacts, see the
file header)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(OUT_DIR, "libgsplat_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
SOURCES = {
    "error.cu": [],
    "sh.cu": [],
    "project.cu": ["--fmad=false"],
    "binning.cu": [],
    "bucket.cu": [],
    "raster_fwd.cu": [],
    "raster_bwd.cu": [],
    "fused.cu": [],
    "ssim.cu": [],
    "densify.cu": [],
    "mcmc.cu": [],
    "bilagrid.cu": [],
    "pose.cu": [],
    "depth.cu": ["--fmad=false"],
    "filter3d.cu": ["--fmad=false"],
    "export.cu": ["--fmad=false"],
    "knn.cu": ["--fmad=false"],
    "image.cu": ["--fmad=false"],
}


def _deps():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "gsplat_b200.h")]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in _deps() if os.path.exists(p))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    obj_dir = os.path.join(HERE, "build")
    os.makedirs(obj_dir, exist_ok=True)
    srcs = {k: v for k, v in SOURCES.items() if os.path.exists(os.path.join(CSRC, k))}

    def compile_one(item):
        name, extra = item
        obj = os.path.join(obj_dir, name.replace(".cu", ".o"))
        cmd = [NVCC] + ARCH + COMMON + extra + ["-c", os.path.join(CSRC, name), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {name}:\n{r.stdout}\n{r.stderr}")
        with open(obj + ".ptxas.log", "w") as f:
            f.write(r.stderr)
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(compile_one, srcs.items()))
    cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

"""In-tree build of libr3dg_b200.so with nvcc for sm_90a (no torch headers, so a full rebuild is
about a minute; nvcc cross-compiles without a GPU).  `python -m relightable3dgaussian_b200.build`."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "libr3dg_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


# shading.cu (and pixel_shading.cu, lights.cu and pixel_lights.cu, which share its per-sample and GGX code in shading_eval.cuh and brdf.cuh) mirrors a chain of separate PyTorch elementwise kernels (each op rounded on its own);
# without FMA contraction the fused kernel reproduces that rounding instead of a differently
# (if slightly better) rounded result of an ill-conditioned GGX denominator.
# denoise.cu: the backward recomputes each of the forward's weights, and must round it alike in another kernel.
# adam.cu: flush-to-zero arithmetic.  Real gradients span the whole fp32 range (g^2 of a barely visible Gaussian is a
# denormal); IEEE sqrt / division take a slow subroutine for denormal operands, and one such lane stalls its warp.
# With -ftz the results are unchanged for every normal number (torch's own CUDA kernels are compiled the same way).
PER_FILE_FLAGS = {"shading.cu": ["-fmad=false"], "pixel_shading.cu": ["-fmad=false"], "lights.cu": ["-fmad=false"],
                  "pixel_lights.cu": ["-fmad=false"], "denoise.cu": ["-fmad=false"], "adam.cu": ["-ftz=true"]}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime():
    m = 0.0
    for d in (CSRC, os.path.join(ROOT, "include")):
        for f in os.listdir(d):
            if f.endswith((".cuh", ".h")):
                m = max(m, os.path.getmtime(os.path.join(d, f)))
    return m


def build(force=False, verbose=False):
    hdr = _deps_mtime()
    objs, jobs = [], []
    for s in sources():
        src = os.path.join(CSRC, s)
        obj = os.path.join(CSRC, s[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr):
            extra = PER_FILE_FLAGS.get(s, [])
            jobs.append([NVCC] + FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj])
    if jobs:
        def run(cmd):
            r = subprocess.run(cmd, capture_output=True, text=True)
            return cmd, r
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for cmd, r in ex.map(run, jobs):
                if verbose or r.returncode != 0:
                    sys.stderr.write(" ".join(cmd[-3:]) + "\n" + r.stdout + r.stderr)
                if r.returncode != 0:
                    raise RuntimeError("nvcc failed for " + cmd[-3])
    if jobs or not os.path.exists(LIB):
        subprocess.check_call([NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

"""Several views per call against one call per view, on one GPU.

For V in {1, 2, 4, 8} views (synth.make_camera(k), k = 0..V-1) of the same scene, times the rasterizer forward +
backward as ONE rasterize_views call pair against V sequential rasterize_gaussians / _backward pairs, at the headline
configuration (1M Gaussians, 800x800, S=5) and at the stage-2 shape (1.5M, 1600x1200, S=16).  Each timing is CUDA
events around `iters` steps; the two arms alternate round by round and the median over `rounds` is reported, with the
per-stage times of the library's stage profiler (ms per step, summed over the step's calls) for both arms.  Prints one
JSON line that starts with the device name and power limit read in the same run.

In a several-view call every view is projected, depth-sorted and binned on its own and the compositors run once over
all views; the profiler's front-end marks are those of the last view, so the batched arm's `project` stage also holds
the earlier views' sort and binning (the front-end total is exact).

    python tools/bench_views.py [--rounds 3] [--iters 5]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relightable3dgaussian_b200 import _C_raster, _lib, synth  # noqa: E402

STAGES = ("project", "depth_sort", "bin_count", "bin_offsets", "bin_scatter", "composite", "normal", "composite_bwd",
          "project_bwd")


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        info["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"unavailable ({e})"
    return info


def steps(P, W, H, S, V):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    cams = [synth.make_camera(k, W, H) for k in range(V)]
    d = lambda t: t.cuda().contiguous()
    means, feats, opac, scales, rots, shs = (d(t) for t in (sc.means3D, sc.features, sc.opacities, sc.scales,
                                                            sc.rotations, sc.shs))
    bgs = [d(torch.tensor([0.0, 0.5, 1.0])) for _ in range(V)]
    views = [d(c.viewmatrix) for c in cams]
    projs = [d(c.projmatrix) for c in cams]
    campos = [d(c.campos) for c in cams]
    gen = torch.Generator(device="cuda").manual_seed(1)
    cots = [torch.randn(V, c, H, W, device="cuda", generator=gen) for c in (3, 1, 1, S)]
    empty = torch.empty(0, device="cuda")
    table = [(c.tanfovx, c.tanfovy, c.cx, c.cy) for c in cams]
    bg_all, view_all, proj_all, cam_all = (torch.stack(x) for x in (bgs, views, projs, campos))

    def batched():
        o = _C_raster.rasterize_views(bg_all, means, feats, empty, opac, scales, rots, 1.0, empty, view_all, proj_all,
                                      table, H, W, shs, 3, cam_all, False, True)
        _C_raster.rasterize_views_backward(bg_all, means, feats, empty, scales, rots, 1.0, empty, view_all, proj_all,
                                           table, *cots, shs, 3, cam_all, o[10], o[11], o[12], True)

    def sequential():
        for v, c in enumerate(cams):
            o = _C_raster.rasterize_gaussians(bgs[v], means, feats, empty, opac, scales, rots, 1.0, empty, views[v],
                                              projs[v], c.tanfovx, c.tanfovy, c.cx, c.cy, H, W, shs, 3, campos[v],
                                              False, True, False)
            _C_raster.rasterize_gaussians_backward(bgs[v], means, feats, o[9], empty, scales, rots, 1.0, empty, views[v],
                                                   projs[v], c.tanfovx, c.tanfovy, *(t[v] for t in cots), shs, 3,
                                                   campos[v], o[10], o[0], o[11], o[12], True, False)
    return batched, sequential


def timed(step, iters):
    step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def stage_times(step, iters, calls_per_step):
    lib = _lib.load()
    lib.r3dg_prof_begin(iters * calls_per_step)
    for _ in range(iters):
        step()
    torch.cuda.synchronize()
    arr = (ctypes.c_float * 9)()
    nf, nb = ctypes.c_int(0), ctypes.c_int(0)
    lib.r3dg_prof_end(arr, ctypes.byref(nf), ctypes.byref(nb))
    return {k: round(arr[i] / iters, 4) for i, k in enumerate(STAGES)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--views", type=str, default="1,2,4,8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_views.py needs a CUDA GPU")
    configs = {"1M_800x800_S5": (1_000_000, 800, 800, 5), "1.5M_1600x1200_S16": (1_500_000, 1600, 1200, 16)}
    res = device_info()
    for name, (P, W, H, S) in configs.items():
        for V in (int(x) for x in args.views.split(",")):
            batched, sequential = steps(P, W, H, S, V)
            ms = {"batched": [], "sequential": []}
            for _ in range(args.rounds):
                ms["batched"].append(timed(batched, args.iters))
                ms["sequential"].append(timed(sequential, args.iters))
            b, s = statistics.median(ms["batched"]), statistics.median(ms["sequential"])
            res[f"{name}_V{V}"] = {"batched_ms": round(b, 3), "sequential_ms": round(s, 3), "speedup": round(s / b, 4),
                                   "batched_stages_ms": stage_times(batched, args.iters, 1),
                                   "sequential_stages_ms": stage_times(sequential, args.iters, V)}
            del batched, sequential
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Cost of anchoring the deterministic mode's fixed point to the cotangent scale.

In deterministic mode the rasterizer backward reduces the largest |cotangent| of each view's planes before the
compositor (det_scale_reduce in csrc/composite_bwd.cu), inside the kernel that zeroes the composited gradient rows
(zero_composited_rows_kernel<true>), after a 2 V-word memset.  At the headline configuration (1M Gaussians, 800x800,
S=5, training-scale cotangents) this times, after warm-up:
  * that kernel: torch.profiler with CUDA activities, its device time per call (a run of its own);
  * the deterministic backward: CUDA events around `iters` backward calls over one forward, the median over `rounds`
    (profiler off).
The reduction reads (3 + S + 2) H W floats once; that read's HBM floor at 3.35 TB/s is printed beside it.  Run it once
more with R3DG_LIB_PATH pointing at a build without the reduction: the difference of the two kernel times is its cost.

Prints one JSON line that starts with the device name and power limit read in the same run.

    python tools/bench_det_scale.py [--rounds 5] [--iters 10]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_views import device_info, timed  # noqa: E402
from relightable3dgaussian_b200 import _C_raster, synth  # noqa: E402


def backward_step(P, W, H, S):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    cam = synth.make_camera(1, W, H)
    d = lambda t: t.cuda().contiguous()                                                 # noqa: E731
    means, feats, opac, scales, rots, shs = (d(t) for t in (sc.means3D, sc.features, sc.opacities, sc.scales,
                                                            sc.rotations, sc.shs))
    bg, view, proj, campos = d(torch.tensor([0.0, 0.5, 1.0])), d(cam.viewmatrix), d(cam.projmatrix), d(cam.campos)
    gen = torch.Generator(device="cuda").manual_seed(1)
    cots = [torch.randn(c, H, W, device="cuda", generator=gen) * 2.0 ** -21 for c in (3, 1, 1, S)]
    empty = torch.empty(0, device="cuda")
    o = _C_raster.rasterize_gaussians(bg, means, feats, empty, opac, scales, rots, 1.0, empty, view, proj,
                                      cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, H, W, shs, 3, campos, False, True, False)

    def run():
        _C_raster.rasterize_gaussians_backward(bg, means, feats, o[9], empty, scales, rots, 1.0, empty, view, proj,
                                               cam.tanfovx, cam.tanfovy, *cots, shs, 3, campos, o[10], o[0], o[11],
                                               o[12], True, False)
    return run


def kernel_us(run, iters, name="zero_composited_rows_kernel"):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            run()
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if name in e.key]
    if not ev:
        raise SystemExit(f"bench_det_scale.py: no {name} launch in the trace")
    total = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in ev)
    calls = sum(e.count for e in ev)
    return total / calls, calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_det_scale.py needs a CUDA GPU")
    res = device_info()
    P, W, H, S = 1_000_000, 800, 800, 5
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        run = backward_step(P, W, H, S)
        ms = [timed(run, args.iters) for _ in range(args.rounds)]
        us, calls = kernel_us(run, args.iters)
    finally:
        torch.use_deterministic_algorithms(prev)
    floor_us = (3 + S + 2) * W * H * 4 / 3.35e12 * 1e6
    bwd = statistics.median(ms)
    res["1M_800x800_S5"] = {"det_backward_ms": round(bwd, 3), "spread_ms": round(max(ms) - min(ms), 3),
                            "zero_rows_kernel_us": round(us, 2), "profiled_calls": calls,
                            "hbm_floor_us": round(floor_us, 2), "share_of_backward": round(us / 1e3 / bwd, 5)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

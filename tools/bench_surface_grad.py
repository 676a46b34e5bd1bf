"""Cost of the pseudo-normal / surface-xyz gradients: rasterizer forward + backward with and without them, on one GPU.

At the headline configuration (1M Gaussians, 800x800, S=5) and at the stage-2 shape (1.5M, 1600x1200, S=16), times
one rasterize_gaussians / rasterize_gaussians_backward pair without a surface cotangent (the default: the cotangent
of the pseudo-normal is ignored) against the same pair with a cotangent on the pseudo-normal and the surface_xyz (one
more launch in front of the backward compositor).  Each timing is CUDA events around `iters` steps; the two arms
alternate round by round and the median over `rounds` is reported, with the backward-compositor stage time of the
library's stage profiler (which includes the surface pass) for both arms.  Prints one JSON line that starts with the
device name and power limit read in the same run.

    python tools/bench_surface_grad.py [--rounds 5] [--iters 10]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_views import device_info, stage_times, timed  # noqa: E402
from relightable3dgaussian_b200 import _C_raster, synth  # noqa: E402


def step(P, W, H, S, surface):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    cam = synth.make_camera(1, W, H)
    d = lambda t: t.cuda().contiguous()
    means, feats, opac, scales, rots, shs = (d(t) for t in (sc.means3D, sc.features, sc.opacities, sc.scales,
                                                            sc.rotations, sc.shs))
    bg, view, proj, campos = d(torch.tensor([0.0, 0.5, 1.0])), d(cam.viewmatrix), d(cam.projmatrix), d(cam.campos)
    gen = torch.Generator(device="cuda").manual_seed(1)
    cots = [torch.randn(c, H, W, device="cuda", generator=gen) for c in (3, 1, 1, S)]
    g_normal, g_xyz = (torch.randn(3, H, W, device="cuda", generator=gen) for _ in range(2))
    empty = torch.empty(0, device="cuda")

    def run():
        o = _C_raster.rasterize_gaussians(bg, means, feats, empty, opac, scales, rots, 1.0, empty, view, proj,
                                          cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, H, W, shs, 3, campos, False, True,
                                          False)
        kw = dict(surface=(g_normal, g_xyz, o[3], o[4], cam.cx, cam.cy)) if surface else {}
        _C_raster.rasterize_gaussians_backward(bg, means, feats, o[9], empty, scales, rots, 1.0, empty, view, proj,
                                               cam.tanfovx, cam.tanfovy, *cots, shs, 3, campos, o[10], o[0], o[11],
                                               o[12], True, False, **kw)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_surface_grad.py needs a CUDA GPU")
    configs = {"1M_800x800_S5": (1_000_000, 800, 800, 5), "1.5M_1600x1200_S16": (1_500_000, 1600, 1200, 16)}
    res = device_info()
    for name, (P, W, H, S) in configs.items():
        arms = {"without": step(P, W, H, S, False), "with": step(P, W, H, S, True)}
        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, run in arms.items():
                ms[k].append(timed(run, args.iters))
        a, b = statistics.median(ms["without"]), statistics.median(ms["with"])
        res[name] = {"without_ms": round(a, 3), "with_ms": round(b, 3), "delta_us": round((b - a) * 1e3, 1),
                     "overhead": round(b / a - 1.0, 4),
                     "composite_bwd_ms": {k: stage_times(run, args.iters, 1)["composite_bwd"] for k, run in arms.items()}}
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

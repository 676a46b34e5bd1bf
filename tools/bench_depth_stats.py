"""Cost of the rasterizer's depth statistics (depth_stats=True: depth2 and the median depth, with gradients).

Rasterizer forward + backward at the headline configuration (1M Gaussians, 800x800, S=5) and at the stage-2 shape
(1.5M, 1600x1200, S=16), the statistics off and on over the same inputs, with the ray-depth mode on (the plane depth the
statistics are meant for) and once with it off.  Each timing is CUDA events around `iters` fwd+bwd pairs; the arms
alternate round by round in one process and the median over `rounds` is reported, with the forward and backward
compositors' stage times of the library's stage profiler in a separate run.  The statistics add one accumulator, the
running median and its position per pixel in the forward, and three per-pixel values and a few FMAs per
(pixel, entry) in the backward's entry phase.

Prints one JSON line that starts with the device name and power limit read in the same run.

    python tools/bench_depth_stats.py [--rounds 5] [--iters 10]
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
from bench_views import device_info, stage_times, timed  # noqa: E402
from relightable3dgaussian_b200 import _C_raster, synth  # noqa: E402


def raster_step(P, W, H, S, ray_depth, depth_stats):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    cam = synth.make_camera(1, W, H)
    d = lambda t: t.cuda().contiguous()                                      # noqa: E731
    means, feats, opac, scales, rots, shs = (d(t) for t in (sc.means3D, sc.features, sc.opacities, sc.scales,
                                                            sc.rotations, sc.shs))
    bg, view, proj, campos = d(torch.tensor([0.0, 0.5, 1.0])), d(cam.viewmatrix), d(cam.projmatrix), d(cam.campos)
    gen = torch.Generator(device="cuda").manual_seed(1)
    cots = [torch.randn(c, H, W, device="cuda", generator=gen) for c in (3, 1, 1, S)]
    stat_cots = [torch.randn(1, H, W, device="cuda", generator=gen) for _ in range(2)]
    empty = torch.empty(0, device="cuda")
    kw = {"ray_depth": ray_depth}
    fkw, bkw = dict(kw), dict(kw)
    if depth_stats:
        fkw["depth_stats"] = True
        bkw.update(depth_stats=True, dL_dout_depth2=stat_cots[0], dL_dout_median_depth=stat_cots[1])

    def run():
        o = _C_raster.rasterize_gaussians(bg, means, feats, empty, opac, scales, rots, 1.0, empty, view, proj,
                                          cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, H, W, shs, 3, campos, False, True,
                                          False, **fkw)
        _C_raster.rasterize_gaussians_backward(bg, means, feats, o[9], empty, scales, rots, 1.0, empty, view, proj,
                                               cam.tanfovx, cam.tanfovy, *cots, shs, 3, campos, o[10], o[0], o[11],
                                               o[12], True, False, **bkw)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_depth_stats.py needs a CUDA GPU")
    res = device_info()
    configs = {"1M_800x800_S5": (1_000_000, 800, 800, 5), "1.5M_1600x1200_S16": (1_500_000, 1600, 1200, 16)}
    for name, (P, W, H, S) in configs.items():
        for rd in (True, False):
            arms = {"off": raster_step(P, W, H, S, rd, False), "on": raster_step(P, W, H, S, rd, True)}
            ms = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, run in arms.items():
                    ms[k].append(timed(run, args.iters))
            st = {k: stage_times(run, args.iters, 1) for k, run in arms.items()}
            a, b = statistics.median(ms["off"]), statistics.median(ms["on"])
            res[f"{name}_{'ray_depth' if rd else 'centre_depth'}"] = {
                "fwd_bwd_off_ms": round(a, 3), "fwd_bwd_on_ms": round(b, 3), "ratio_on_off": round(b / a, 4),
                "spread_ms": {k: round(max(v) - min(v), 3) for k, v in ms.items()},
                **{f"{s}_ms": {k: t[s] for k, t in st.items()} for s in ("composite", "composite_bwd")}}
            del arms
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

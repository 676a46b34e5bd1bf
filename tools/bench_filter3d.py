"""Cost of Mip-Splatting's 3D filter: compute_3d_filter against Mip-Splatting's per-camera PyTorch loop, and the
filtered rasterizer mode (filter_3d=f) against the mode off.

  * compute: P in {1M, 3M} x V in {100, 300} cameras with mixed intrinsics, the CUDA pass (two launches) against a
    PyTorch restatement of Mip-Splatting's compute_3D_filter loop (~20 elementwise launches over P per camera);
  * rasterizer forward + backward at 1M / 800x800 / S = 5 and 1.5M / 1600x1200 / S = 16, the mode off and on over the
    same inputs.
Each timing is CUDA events around `iters` calls; the arms alternate round by round and the median over `rounds` is
reported.  Prints one JSON line that starts with the device name and power limit read in the same run.

    python tools/bench_filter3d.py [--rounds 5] [--iters 10]
"""
import argparse
import json
import math
import os
import statistics
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_views import device_info, timed  # noqa: E402
from relightable3dgaussian_b200 import _C_raster, filter3d, synth  # noqa: E402


def cameras(V, seed=0):
    g = np.random.default_rng(seed)
    cams = []
    for i in range(V):
        W, H = int(g.integers(400, 1600)), int(g.integers(300, 1200))
        c = synth.make_camera(i % 16 + 1, W, H, radius=float(4.0 * g.uniform(0.6, 1.6)))
        cams.append(SimpleNamespace(world_view_transform=c.viewmatrix.float().cuda().contiguous(), image_width=W,
                                    image_height=H, fx=float(g.uniform(0.5, 2.0) * W), fy=float(g.uniform(0.5, 2.0) * H),
                                    cx=W / 2, cy=H / 2))
    return cams


def torch_loop(xyz, cams):
    """Mip-Splatting's compute_3D_filter as a PyTorch loop over the cameras (with each camera's view matrix)."""
    distance = torch.ones((xyz.shape[0]), device=xyz.device) * 100000.0
    valid_points = torch.zeros((xyz.shape[0]), device=xyz.device, dtype=torch.bool)
    focal_length = 0.
    for c in cams:
        V = c.world_view_transform
        xyz_cam = xyz @ V[:3, :3] + V[3, :3][None, :]
        valid_depth = xyz_cam[:, 2] > 0.2
        x, y, z = xyz_cam[:, 0], xyz_cam[:, 1], xyz_cam[:, 2]
        z = torch.clamp(z, min=0.001)
        x = x / z * c.fx + c.image_width / 2.0
        y = y / z * c.fy + c.image_height / 2.0
        in_screen = torch.logical_and(torch.logical_and(x >= -0.15 * c.image_width, x <= c.image_width * 1.15),
                                      torch.logical_and(y >= -0.15 * c.image_height, y <= 1.15 * c.image_height))
        valid = torch.logical_and(valid_depth, in_screen)
        distance[valid] = torch.min(distance[valid], z[valid])
        valid_points = torch.logical_or(valid_points, valid)
        focal_length = max(focal_length, c.fx)
    distance[~valid_points] = distance[valid_points].max()
    return (distance / focal_length * (0.2 ** 0.5))[..., None]


def raster_step(P, W, H, S, filtered):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    cam = synth.make_camera(1, W, H)
    d = lambda t: t.cuda().contiguous()
    means, feats, opac, scales, rots, shs = (d(t) for t in (sc.means3D, sc.features, sc.opacities, sc.scales,
                                                            sc.rotations, sc.shs))
    bg, view, proj, campos = d(torch.tensor([0.0, 0.5, 1.0])), d(cam.viewmatrix), d(cam.projmatrix), d(cam.campos)
    gen = torch.Generator(device="cuda").manual_seed(1)
    cots = [torch.randn(c, H, W, device="cuda", generator=gen) for c in (3, 1, 1, S)]
    empty = torch.empty(0, device="cuda")
    tc = SimpleNamespace(world_view_transform=view, image_width=W, image_height=H, FoVx=2 * math.atan(cam.tanfovx),
                         FoVy=2 * math.atan(cam.tanfovy), fx=None)
    f = filter3d.compute_3d_filter(means, [tc]) if filtered else None
    fkw = {"filter_3d": f} if filtered else {}
    bkw = {"filter_3d": f, "opacities": opac} if filtered else {}

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
        raise SystemExit("bench_filter3d.py needs a CUDA GPU")
    res = device_info()
    for P in (1_000_000, 3_000_000):
        xyz = synth.make_scene(P, "shell-v1", 0, 0).means3D.float().cuda().contiguous()
        for V in (100, 300):
            cams = cameras(V)
            arms = {"cuda": lambda: filter3d.compute_3d_filter(xyz, cams), "torch_loop": lambda: torch_loop(xyz, cams)}
            ms = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, run in arms.items():
                    ms[k].append(timed(run, 2 if k == "torch_loop" else args.iters))
            a, b = statistics.median(ms["cuda"]), statistics.median(ms["torch_loop"])
            res[f"compute_{P // 1_000_000}M_V{V}"] = {"cuda_ms": round(a, 3), "torch_loop_ms": round(b, 2),
                                                      "speedup": round(b / a, 1)}
        del xyz
        torch.cuda.empty_cache()
    configs = {"1M_800x800_S5": (1_000_000, 800, 800, 5), "1.5M_1600x1200_S16": (1_500_000, 1600, 1200, 16)}
    for name, (P, W, H, S) in configs.items():
        arms = {"off": raster_step(P, W, H, S, False), "on": raster_step(P, W, H, S, True)}
        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, run in arms.items():
                ms[k].append(timed(run, args.iters))
        a, b = statistics.median(ms["off"]), statistics.median(ms["on"])
        res[name] = {"fwd_bwd_off_ms": round(a, 3), "fwd_bwd_on_ms": round(b, 3), "ratio_on_off": round(b / a, 4),
                     "spread_ms": {k: round(max(v) - min(v), 3) for k, v in ms.items()}}
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

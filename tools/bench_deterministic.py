"""Cost of the deterministic mode (torch.use_deterministic_algorithms(True)) on one GPU.

Times, alternating the two modes round by round, the rasterizer forward + backward at the headline configuration
(1M Gaussians, 800x800, S=5) and at the stage-2 shape (1.5M, 1600x1200, S=16), and the shading backward at N=32
(1M Gaussians, DirectLightMap 16x32).  Each timing is CUDA events around `iters` calls after a warm-up.
Prints one JSON line: device name and power limit, per configuration and mode the median over `rounds`.

    python tools/bench_deterministic.py [--rounds 5] [--iters 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relightable3dgaussian_b200 import _C_raster, synth  # noqa: E402
from relightable3dgaussian_b200.shading import _RenderEquation  # noqa: E402


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        info["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"unavailable ({e})"
    return info


def raster_step(P, W, H, S, view):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    cam = synth.make_camera(view, W, H)
    d = lambda t: t.cuda().contiguous()
    bg, means, feats, opac, scales, rots, shs = (d(t) for t in (torch.tensor([0.0, 0.5, 1.0]), sc.means3D, sc.features,
                                                               sc.opacities, sc.scales, sc.rotations, sc.shs))
    view_m, proj, campos = d(cam.viewmatrix), d(cam.projmatrix), d(cam.campos)
    gen = torch.Generator(device="cuda").manual_seed(1)
    cots = [torch.randn(c, H, W, device="cuda", generator=gen) for c in (3, 1, 1, S)]
    empty = torch.empty(0, device="cuda")

    def step():
        o = _C_raster.rasterize_gaussians(bg, means, feats, empty, opac, scales, rots, 1.0, empty, view_m, proj,
                                          cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, H, W, shs, 3, campos, False, True, False)
        _C_raster.rasterize_gaussians_backward(bg, means, feats, o[9], empty, scales, rots, 1.0, empty, view_m, proj,
                                               cam.tanfovx, cam.tanfovy, *cots, shs, 3, campos, o[10], o[0], o[11], o[12],
                                               True, False)
    return step


def shade_step(P, N):
    g = torch.Generator(device="cuda").manual_seed(2)
    base, rough = torch.rand(P, 3, device="cuda", generator=g), torch.rand(P, 1, device="cuda", generator=g)
    normals = F.normalize(torch.randn(P, 3, device="cuda", generator=g), dim=-1)
    viewdirs, incidents = torch.randn(P, 3, device="cuda", generator=g), 0.1 * torch.randn(P, 16, 3, device="cuda", generator=g)
    env = F.softplus(torch.randn(16, 32, 3, device="cuda", generator=g))
    vis, dirs = torch.rand(P, N, 1, device="cuda", generator=g), F.normalize(torch.randn(P, N, 3, device="cuda", generator=g), dim=-1)
    areas = torch.full((P, N, 1), 0.4, device="cuda")
    leaves = [t.requires_grad_(True) for t in (base, rough, viewdirs, incidents, env)]
    pbr, diffuse, _ = _RenderEquation.apply(*leaves, normals, vis, dirs, areas, None, False)
    cot_p, cot_d = torch.randn_like(pbr), torch.randn_like(diffuse)

    def step():
        torch.autograd.grad((pbr, diffuse), leaves, (cot_p, cot_d), retain_graph=True)
    return step


def timed(step, iters, det):
    torch.use_deterministic_algorithms(det)
    try:
        step()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            step()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / iters
    finally:
        torch.use_deterministic_algorithms(False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic.py needs a CUDA GPU")
    configs = {"raster_fwd_bwd_1M_800x800_S5": lambda: raster_step(1_000_000, 800, 800, 5, 0),
               "raster_fwd_bwd_1.5M_1600x1200_S16": lambda: raster_step(1_500_000, 1600, 1200, 16, 3),
               "shade_bwd_1M_N32_env16x32": lambda: shade_step(1_000_000, 32)}
    res = device_info()
    for name, make in configs.items():
        step = make()
        for det in (False, True):          # warm up both modes (module load, workspace sizes)
            timed(step, 1, det)
        ms = {False: [], True: []}
        for _ in range(args.rounds):
            for det in (False, True):
                ms[det].append(timed(step, args.iters, det))
        d, n = statistics.median(ms[False]), statistics.median(ms[True])
        res[name] = {"default_ms": round(d, 4), "deterministic_ms": round(n, 4), "overhead": round(n / d - 1.0, 4)}
        del step
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Time `shading.rendering_equation_views` (V views in one call) against V sequential `rendering_equation` calls.

Each configuration at V = 1, 2, 4, 8:
  * training:   forward + backward, 1M Gaussians, N = 32, a DirectLightMap-style 16x32 environment (softplus);
  * relighting: forward only with the means, 1.5M Gaussians, N = 384, an EnvLight 128x256 with one transform per view
    (and, as `relighting_shared`, the same with one transform for all views).
The two arms alternate inside each of 3 rounds (CUDA events around `--iters` calls each); the median round is
reported, with the HBM floor of the baked reads (20 B per sample: direction, visibility, area) of each arm at the
data-sheet 3.35 TB/s.  Prints one JSON line that starts with the device name and its power limit.

    python tools/bench_shade_views.py [--iters 10] [--views 1,2,4,8] [--only training|relighting|relighting_shared]
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

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


class SoftplusLight:
    def __init__(self, env_raw):
        self.env = env_raw

    @property
    def get_env(self):
        return F.softplus(self.env)


class FixedLight:
    def __init__(self, envmap, transform):
        self.envmap, self.transform = envmap, transform


def device_info():
    name, limit = torch.cuda.get_device_name(0), None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = float(out) if out else None
    except (OSError, ValueError, subprocess.TimeoutExpired):
        pass
    return name, limit


def make_inputs(P, N, He, V, seed=0):
    from relightable3dgaussian_b200 import raytracer
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = dict(device="cuda", generator=g)
    n = F.normalize(torch.randn(P, 3, **dev), dim=-1)
    dirs, areas = raytracer.sample_incident_rays(n, False, N)            # baked on the GPU
    vis = torch.where(torch.rand(P, N, 1, **dev) < 0.4, 0.0, 0.95).float()
    c = dict(base_color=torch.rand(P, 3, **dev) * 0.77 + 0.03, roughness=torch.rand(P, 1, **dev) * 0.9 + 0.09,
             normals=n, incidents=torch.randn(P, 16, 3, **dev) * 0.3, env_raw=torch.randn(1, He, 2 * He, 3, **dev),
             visibility=vis.contiguous(), incident_dirs=dirs.contiguous(), incident_areas=areas.contiguous(),
             viewdirs=F.normalize(torch.randn(V, P, 3, **dev), dim=-1))
    c["rot"] = torch.linalg.qr(torch.randn(V, 3, 3, device="cuda", generator=g, dtype=torch.float64))[0].float()
    c["cot"] = torch.randn(V, P, 3, **dev)
    return c


def training_arms(c, V):
    from relightable3dgaussian_b200.shading import rendering_equation, rendering_equation_views
    leaves = {k: c[k].clone().requires_grad_(True) for k in ("base_color", "roughness", "incidents", "env_raw")}
    vd = c["viewdirs"][:V].clone().requires_grad_(True)
    light = SoftplusLight(leaves["env_raw"])
    baked = (c["visibility"], c["incident_dirs"], c["incident_areas"])

    def batched():
        pbr, _ = rendering_equation_views(leaves["base_color"], leaves["roughness"], c["normals"], vd, leaves["incidents"],
                                          light, *baked)
        pbr.backward(c["cot"][:V])

    def sequential():
        for v in range(V):
            pbr, _ = rendering_equation(leaves["base_color"], leaves["roughness"], c["normals"], vd[v], leaves["incidents"],
                                        light, *baked)
            pbr.backward(c["cot"][v])
    return batched, sequential


def relighting_arms(c, V, per_view=True):
    from relightable3dgaussian_b200.shading import _RenderEquation, rendering_equation_views
    tex = F.softplus(c["env_raw"])[0].contiguous()
    baked = (c["visibility"], c["incident_dirs"], c["incident_areas"])

    def batched():
        with torch.no_grad():
            rendering_equation_views(c["base_color"], c["roughness"], c["normals"], c["viewdirs"][:V], c["incidents"],
                                     FixedLight(tex, c["rot"][:V] if per_view else c["rot"][0]), *baked, means=True)

    def sequential():               # rendering_equation's mean outputs (the eval pack) through its autograd function
        with torch.no_grad():
            for v in range(V):
                _RenderEquation.apply(c["base_color"], c["roughness"], c["viewdirs"][v], c["incidents"], tex, c["normals"],
                                      *baked, c["rot"][v] if per_view else c["rot"][0], True)
    return batched, sequential


def time_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def run(name, P, N, He, views, make_arms, iters, rounds=3):
    c = make_inputs(P, N, He, max(views))
    floor_one = 20.0 * P * N / HBM_BYTES_PER_S * 1e3        # ms: one pass over the baked tensors
    res = {}
    for V in views:
        batched, sequential = make_arms(c, V)
        for fn in (batched, sequential):                    # warm-up: modules, allocator, attributes
            fn()
        torch.cuda.synchronize()
        b, s = [], []
        for _ in range(rounds):
            b.append(time_ms(batched, iters))
            s.append(time_ms(sequential, iters))
        mb, ms = statistics.median(b), statistics.median(s)
        res[f"V{V}"] = dict(batched_ms=round(mb, 3), sequential_ms=round(ms, 3), speedup=round(ms / mb, 3),
                            hbm_floor_batched_ms=round(floor_one, 3), hbm_floor_sequential_ms=round(V * floor_one, 3))
        print(f"[{name}] V={V}: batched {mb:.3f} ms, sequential {ms:.3f} ms, x{ms / mb:.2f}", file=sys.stderr)
    del c
    torch.cuda.empty_cache()
    return dict(P=P, N=N, env=f"{He}x{2 * He}", **res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--views", default="1,2,4,8")
    ap.add_argument("--only", choices=("training", "relighting", "relighting_shared"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shade_views.py needs a CUDA device")
    name, limit = device_info()
    views = [int(v) for v in args.views.split(",")]
    out = dict(device=name, power_limit_w=limit)
    if args.only in (None, "training"):
        out["training"] = run("training", 1_000_000, 32, 16, views, training_arms, args.iters)
    if args.only in (None, "relighting"):
        out["relighting"] = run("relighting", 1_500_000, 384, 128, views, relighting_arms, args.iters)
    if args.only in (None, "relighting_shared"):
        out["relighting_shared"] = run("relighting_shared", 1_500_000, 384, 128, views,
                                       lambda c, V: relighting_arms(c, V, per_view=False), args.iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

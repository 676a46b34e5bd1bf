"""Time the shading step's filtered environment lookup (env_filter=True) against the point lookup (env_filter=False).

Configurations:
  * relighting: forward with the means, 1M Gaussians, N = 64 and 384, an EnvLight of 1024x512 and of 2000x1000, one
    view and 4 views with one transform per view;
  * pyramid:    r3dg_env_pyramid_build on its own at those two sizes;
  * training:   forward + backward, 1M Gaussians, N = 32, a softplus env of 16x32 and of 64x128.
The off and on arms alternate inside each of 3 rounds (CUDA events around `--iters` calls each); the median round is
reported in ms per call.  Prints one JSON line that starts with the device name and its power limit.

    python tools/bench_env_filter.py [--iters 10] [--gaussians 1000000]
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


def make_inputs(P, N, V, seed=0):
    from relightable3dgaussian_b200 import raytracer
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = dict(device="cuda", generator=g)
    n = F.normalize(torch.randn(P, 3, **dev), dim=-1)
    dirs, areas = raytracer.sample_incident_rays(n, False, N)            # baked on the GPU
    vis = torch.where(torch.rand(P, N, 1, **dev) < 0.4, 0.0, 0.95).float()
    c = dict(base_color=torch.rand(P, 3, **dev) * 0.77 + 0.03, roughness=torch.rand(P, 1, **dev) * 0.9 + 0.09,
             normals=n, incidents=torch.randn(P, 16, 3, **dev) * 0.3, visibility=vis.contiguous(),
             incident_dirs=dirs.contiguous(), incident_areas=areas.contiguous(),
             viewdirs=F.normalize(torch.randn(V, P, 3, **dev), dim=-1))
    c["rot"] = torch.linalg.qr(torch.randn(V, 3, 3, device="cuda", generator=g, dtype=torch.float64))[0].float()
    c["cot"] = torch.randn(P, 3, **dev)
    return c


def hdr(He, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    env = torch.rand(He, 2 * He, 3, device="cuda", generator=g) + 0.1
    bright = torch.rand(He, 2 * He, 1, device="cuda", generator=g) > 0.9995
    return (env + 200.0 * bright).contiguous()


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def compare(arms, iters):
    """{arm: median ms} over 3 rounds with the arms alternating in each."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(3):
        for k, fn in arms.items():
            times[k].append(timed(fn, iters))
    return {k: round(statistics.median(v), 4) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    args = ap.parse_args()
    from relightable3dgaussian_b200 import shading
    from relightable3dgaussian_b200.shading import rendering_equation, rendering_equation_views
    name, limit = device_info()
    P = args.gaussians
    res = {"device": name, "power_limit_w": limit, "gaussians": P}
    envs = {512: hdr(512), 1000: hdr(1000)}
    for N in (64, 384):
        for V in (1, 4):
            c = make_inputs(P, N, V)
            for He, env in envs.items():
                light = FixedLight(env, c["rot"][0] if V == 1 else c["rot"])
                base = (c["base_color"], c["roughness"], c["normals"], c["viewdirs"][0] if V == 1 else c["viewdirs"],
                        c["incidents"], light, c["visibility"], c["incident_dirs"], c["incident_areas"])

                def arm(f, base=base):
                    def run():
                        with torch.no_grad():
                            rendering_equation_views(*base[:3], base[3] if V > 1 else base[3][None], *base[4:], means=True,
                                                     env_filter=f)
                    return run
                r = compare({"off": arm(False), "on": arm(True)}, args.iters)
                res[f"relight_N{N}_V{V}_{2 * He}x{He}"] = r
                print(f"relight N={N} V={V} env {2 * He}x{He}: {r}", file=sys.stderr)
            del c
            torch.cuda.empty_cache()
    for He, env in envs.items():
        res[f"pyramid_{2 * He}x{He}"] = compare({"build": lambda env=env: shading.env_pyramid(env)}, args.iters)["build"]
    c = make_inputs(P, 32, 1)
    for He in (16, 64):
        g = torch.Generator(device="cuda").manual_seed(He)
        env_raw = torch.randn(1, He, 2 * He, 3, device="cuda", generator=g).requires_grad_(True)
        leaves = {k: c[k].clone().requires_grad_(True) for k in ("base_color", "roughness", "incidents")}
        vd = c["viewdirs"][0].clone().requires_grad_(True)

        def train(f, env_raw=env_raw, leaves=leaves, vd=vd):
            def run():
                pbr, ex = rendering_equation(leaves["base_color"], leaves["roughness"], c["normals"], vd, leaves["incidents"],
                                             SoftplusLight(env_raw), c["visibility"], c["incident_dirs"], c["incident_areas"],
                                             env_filter=f)
                pbr.backward(c["cot"])
            return run
        r = compare({"off": train(False), "on": train(True)}, args.iters)
        res[f"train_N32_{2 * He}x{He}"] = r
        print(f"train env {2 * He}x{He}: {r}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

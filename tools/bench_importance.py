"""Importance-sampled environment lighting on the GPU: the env table build, the sampler, the importance bake (sampler +
trace) against the Fibonacci bake (bake_visibility) of the same Gaussians and N, and the per-pixel trace and shading
(trace_pixels / shade_pixels forward and forward + backward) with and without a sampler on bench_pixel_shading's
synthetic G-buffers at 800 x 800 and 1920 x 1080.

    python tools/bench_importance.py [--P 1000000] [--out result.json]

Envs: 1024 x 512 and 2000 x 1000 (We x He) HDR maps with a small bright source.  Scenes: synth's shell-v1 and cube-v1
at P Gaussians, N = 32 and 64, the default mix (0.5, 0.25, 0.25) with random view directions and roughness.  Prints
one JSON line per case, then the card's name and power limit, and writes them all to --out when given."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relightable3dgaussian_b200 import synth  # noqa: E402
from relightable3dgaussian_b200.raytracer import RayTracer, inverse_covariance  # noqa: E402
from relightable3dgaussian_b200.shading import EnvSampler, importance_sample, shade_pixels  # noqa: E402
from bench_pixel_shading import gbuffer, timed  # noqa: E402


class FixedLight:
    def __init__(self, envmap, transform=None):
        self.envmap, self.transform = envmap, transform


def hdr_env(He, We, seed=0):
    g = torch.Generator().manual_seed(seed)
    env = torch.rand(He, We, 3, generator=g) * 0.2
    env[He // 5:He // 5 + max(He // 100, 1), We // 3:We // 3 + max(We // 100, 1)] = 2000.0
    return env.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_importance needs a CUDA GPU")
    results = []
    for He, We in ((512, 1024), (1000, 2000)):
        env = hdr_env(He, We)
        ms, _ = timed(lambda: EnvSampler(FixedLight(env)), 20)
        results.append(dict(case="table build", He=He, We=We, ms=ms))
        print(json.dumps(results[-1]), flush=True)
    sampler_env = hdr_env(1000, 2000)
    sampler = EnvSampler(FixedLight(sampler_env))
    for recipe in ("shell-v1", "cube-v1"):
        sc = synth.make_scene(args.P, recipe, 0, 0)
        m, s, r, o, nr = (t.cuda() for t in (sc.means3D, sc.scales, sc.rotations, sc.opacities[:, 0].contiguous(), sc.normals))
        inv = inverse_covariance(s, r).contiguous()
        rt = RayTracer(m, s, r)
        g = torch.Generator().manual_seed(1)
        view = torch.randn(args.P, 3, generator=g).cuda()
        rough = (torch.rand(args.P, 1, generator=g) * 0.9 + 0.08).cuda()
        for N in (32, 64):
            res = dict(case="bake", recipe=recipe, P=args.P, N=N)
            res["sample_ms"], _ = timed(lambda: importance_sample(nr, sampler, N, view, rough), 5)
            res["bake_importance_ms"], res["bake_importance_peak_mb"] = timed(
                lambda: rt.bake_importance(m, inv, o, nr, sampler, N, view, rough), 3)
            res["bake_fibonacci_ms"], res["bake_fibonacci_peak_mb"] = timed(lambda: rt.bake_visibility(m, inv, o, nr, N), 3)
            res["rays_per_s_importance"] = args.P * N / (res["bake_importance_ms"] / 1e3)
            results.append(res)
            print(json.dumps(res), flush=True)
        light = FixedLight(sampler_env)
        for H, W in ((800, 800), (1080, 1920)):
            g = gbuffer(recipe, H, W)
            for N in (32, 64):
                for smp in (None, sampler):
                    res = dict(case="pixels", recipe=recipe, P=args.P, H=H, W=W, N=N, sampler=smp is not None)
                    trace = lambda: rt.trace_pixels(g["points"], g["normal"], N, m, inv, o, nr, sampler=smp,
                                                    roughness=g["rough"], campos=g["campos"])
                    res["trace_ms"], _ = timed(trace, 1)
                    T = trace()
                    fwd = lambda: shade_pixels(g["base"], g["rough"], g["normal"], g["points"], g["campos"], T, light,
                                               sampler=smp)
                    res["shade_fwd_ms"], _ = timed(torch.no_grad()(fwd), 5)
                    base = g["base"].clone().requires_grad_()

                    def fwd_bwd():
                        out = shade_pixels(base, g["rough"], g["normal"], g["points"], g["campos"], T, light, sampler=smp)
                        out["pbr"].sum().backward()
                    res["shade_fwd_bwd_ms"], _ = timed(fwd_bwd, 5)
                    results.append(res)
                    print(json.dumps(res), flush=True)
        del rt
        torch.cuda.empty_cache()
    meta = {"gpu": torch.cuda.get_device_name()}
    try:
        meta["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                             capture_output=True, text=True).stdout.strip()
    except OSError:
        pass
    print(json.dumps(meta))
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"meta": meta, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()

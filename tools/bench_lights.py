#!/usr/bin/env python3
"""Time of the point and directional lights (RayTracer.trace_lights, lights.shade) at 1M Gaussians of synth's scene,
with the shading step's rendering_equation (forward + backward at N = 32) as a yardstick.

  python tools/bench_lights.py [--recipe shell-v1] [--P 1000000] [--lights 1 4 32] [--views 1 8] [--iters 20]

Half the lights are directional, half point lights inside the scene (K = 1: one directional light).  Timings are
CUDA-event medians over --iters calls after a warm-up: the shadow trace (tree packing included, tree build excluded),
the shading forward and forward + backward at each V.  The shading kernels' HBM floor is computed from the shapes:
forward 40 B per Gaussian (base colour, roughness, normal, mean) + 4 K B of shadows + 36 B per view (view direction
in, three [3] outputs); the backward reads that plus 36 B of cotangents per view and writes 40 B + 12 B per view of
gradient rows.  Achieved bytes/s = floor bytes / time.  The device name and power limit are read in the same run.
Ends with one JSON line of everything."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from relightable3dgaussian_b200 import lights as lt  # noqa: E402
from relightable3dgaussian_b200 import shading, synth  # noqa: E402
from relightable3dgaussian_b200.raytracer import RayTracer, inverse_covariance  # noqa: E402

DEV = torch.device("cuda")


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [s.strip() for s in out.split(",")]
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        info["power_limit"] = f"unavailable ({e})"
    return info


def median_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def floor_bytes(P, K, V, backward):
    fwd = P * (40 + 4 * K + 36 * V)
    return fwd + (P * (36 * V + 40 + 12 * V) if backward else 0)


def make_lights(means, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    nd = max(K // 2, 1) if K > 1 else 1
    dirs = torch.nn.functional.normalize(torch.randn(nd, 3, generator=g), dim=-1)
    m = means.cpu()
    pos = m[torch.randint(0, m.shape[0], (K - nd,), generator=g)] + 0.1 * torch.randn(K - nd, 3, generator=g)
    d = lt.Lights.directional(dirs.to(DEV), torch.rand(nd, 3, generator=g).to(DEV) * 2)
    if K == nd:
        return d
    return lt.Lights.cat(d, lt.Lights.point(pos.to(DEV), torch.rand(K - nd, 3, generator=g).to(DEV)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recipe", default="shell-v1")
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--lights", nargs="+", type=int, default=[1, 4, 32])
    ap.add_argument("--views", nargs="+", type=int, default=[1, 8])
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lights.py needs a GPU")
    info = device_info()
    sc = synth.make_scene(args.P, args.recipe, 0, 0)
    d = lambda t: t.to(DEV).contiguous()
    means, scales, rots = d(sc.means3D), d(sc.scales), d(sc.rotations)
    normals = d(-sc.normals if args.recipe == "shell-v1" else sc.normals)
    opacity = d(sc.opacities[:, 0])
    inv = inverse_covariance(scales, rots)
    P = args.P
    g = torch.Generator().manual_seed(1)
    base = torch.rand(P, 3, generator=g).to(DEV).requires_grad_(True)
    rough = torch.rand(P, 1, generator=g).to(DEV).requires_grad_(True)
    rt = RayTracer(means, scales, rots)
    print(f"# {info['device']}, power limit {info.get('power_limit')}; P = {P} ({args.recipe}); CUDA-event medians of "
          f"{args.iters} calls")
    results = []

    # yardstick: the shading step at N = 32, forward + backward
    N = 32
    vis = rt.bake_visibility(means, inv, opacity, normals, N)
    inc = torch.zeros(P, 16, 3, device=DEV, requires_grad=True)

    class Env:
        envmap = torch.rand(16, 32, 3, device=DEV).requires_grad_(True)
    view1 = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1).to(DEV).requires_grad_(True)

    def re_fb():
        pbr, _ = shading.rendering_equation(base, rough, normals, view1, inc, Env, vis["visibility"], vis["incident_dirs"],
                                            vis["incident_areas"])
        pbr.sum().backward()
    t_re = median_ms(re_fb, args.iters)
    print(f"rendering_equation N={N} fwd+bwd: {t_re:.3f} ms")
    del vis
    torch.cuda.empty_cache()

    for K in args.lights:
        lights = make_lights(means, K)
        lights = lt.Lights(lights.kind, lights.vec.requires_grad_(True), lights.color.requires_grad_(True))
        t_trace = median_ms(lambda: rt.trace_lights(means, inv, opacity, normals, lights), args.iters)
        T = rt.trace_lights(means, inv, opacity, normals, lights)
        row = {"K": K, "trace_ms": t_trace, "trace_rays_per_s": P * K / (t_trace * 1e-3),
               "shadowed": float((T < 1).double().mean()), "views": {}}
        print(f"K={K:2d}: shadow trace {t_trace:9.3f} ms ({P * K / t_trace / 1e3:8.1f} Mray/s, "
              f"{row['shadowed']:.1%} of pairs shadowed)")
        for V in args.views:
            vd = torch.nn.functional.normalize(torch.randn(V, P, 3, generator=g), dim=-1).to(DEV).requires_grad_(True)

            def fwd():
                with torch.no_grad():
                    lt.shade(base, rough, normals, vd, means, lights, T)

            def fb():
                pbr, extra = lt.shade(base, rough, normals, vd, means, lights, T)
                torch.autograd.backward((pbr, extra["diffuse_light"], extra["specular"]),
                                        [torch.ones_like(pbr)] * 3)
            t_f, t_fb = median_ms(fwd, args.iters), median_ms(fb, args.iters)
            bf, bfb = floor_bytes(P, K, V, False), floor_bytes(P, K, V, True)
            row["views"][V] = {"fwd_ms": t_f, "fwd_bwd_ms": t_fb, "fwd_GBps": bf / (t_f * 1e6),
                               "fwd_bwd_GBps": bfb / (t_fb * 1e6), "fwd_bwd_over_rendering_equation": t_fb / t_re}
            print(f"       V={V}: shade fwd {t_f:8.3f} ms ({bf / (t_f * 1e6):7.1f} GB/s of the floor), "
                  f"fwd+bwd {t_fb:8.3f} ms ({bfb / (t_fb * 1e6):7.1f} GB/s), {t_fb / t_re:.2f}x rendering_equation N=32",
                  flush=True)
        results.append(row)
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "lights", **info, "P": P, "recipe": args.recipe, "iters": args.iters,
                      "rendering_equation_n32_fwd_bwd_ms": t_re, "results": results}))


if __name__ == "__main__":
    main()

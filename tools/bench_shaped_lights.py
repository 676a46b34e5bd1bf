#!/usr/bin/env python3
"""Time of the spot and rect lights (RayTracer.trace_shaped_lights, lights.shade_shaped) at 1M Gaussians of synth's
scene, against lights.shade with the same K point lights and the shading step's rendering_equation at N = 32.

  python tools/bench_shaped_lights.py [--recipe shell-v1] [--P 1000000] [--lights 1 4] [--M 2 4 8] [--views 1 8]
                                      [--iters 10]

Rect lights (and, per K, a set of K spots) sit inside the scene.  Timings are CUDA-event medians over --iters calls
after a warm-up: the shadow trace (tree packing included, tree build excluded) with its rays/s, the shading forward
and forward + backward at each V.  The device name and power limit are read in the same run.  Ends with one JSON line."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_lights import device_info, median_ms  # noqa: E402
from relightable3dgaussian_b200 import lights as lt  # noqa: E402
from relightable3dgaussian_b200 import shading, synth  # noqa: E402
from relightable3dgaussian_b200.raytracer import RayTracer, inverse_covariance  # noqa: E402

DEV = torch.device("cuda")


def make_set(means, kind, K, M, seed=0):
    g = torch.Generator().manual_seed(seed)
    m = means.cpu()
    pos = m[torch.randint(0, m.shape[0], (K,), generator=g)] + 0.1 * torch.randn(K, 3, generator=g)
    a = torch.randn(K, 3, generator=g) * (0.05 if kind == lt.RECT else 1.0)
    b = torch.randn(K, 3, generator=g) * 0.05
    color = torch.rand(K, 3, generator=g) * 2
    cone = torch.tensor([[0.9, 0.7]]).expand(K, 2)
    return lt.ShapedLights(torch.full((K,), kind, dtype=torch.int32), *(t.to(DEV).contiguous().requires_grad_(True)
                                                                       for t in (pos, a, b, color, cone)), M=M, seed=seed)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recipe", default="shell-v1")
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--lights", nargs="+", type=int, default=[1, 4])
    ap.add_argument("--M", nargs="+", type=int, default=[2, 4, 8])
    ap.add_argument("--views", nargs="+", type=int, default=[1, 8])
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_shaped_lights.py needs a GPU")
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

    def shade_times(shade, lights, T, V):
        vd = torch.nn.functional.normalize(torch.randn(V, P, 3, generator=g), dim=-1).to(DEV).requires_grad_(True)

        def fwd():
            with torch.no_grad():
                shade(base, rough, normals, vd, means, lights, T)

        def fb():
            pbr, extra = shade(base, rough, normals, vd, means, lights, T)
            torch.autograd.backward((pbr, extra["diffuse_light"], extra["specular"]), [torch.ones_like(pbr)] * 3)
        return median_ms(fwd, args.iters), median_ms(fb, args.iters)

    results = []
    for K in args.lights:
        cases = [("spot", 1, make_set(means, lt.SPOT, K, 1))] + [("rect", M, make_set(means, lt.RECT, K, M)) for M in args.M]
        point = lt.Lights.point(cases[0][2].pos.detach().requires_grad_(True), cases[0][2].color.detach().requires_grad_(True))
        Tp = rt.trace_lights(means, inv, opacity, normals, point)
        for name, M, lights in cases:
            R = lights.num_rays()
            t_trace = median_ms(lambda: rt.trace_shaped_lights(means, inv, opacity, normals, lights), args.iters)
            T = rt.trace_shaped_lights(means, inv, opacity, normals, lights)
            row = {"kind": name, "K": K, "M": M, "R": R, "trace_ms": t_trace, "trace_rays_per_s": P * R / (t_trace * 1e-3),
                   "views": {}}
            print(f"K={K} {name:4s} M={M}: shadow trace {t_trace:9.3f} ms ({P * R / t_trace / 1e3:8.1f} Mray/s)", flush=True)
            for V in args.views:
                t_f, t_fb = shade_times(lt.shade_shaped, lights, T, V)
                p_f, p_fb = shade_times(lt.shade, point, Tp, V)
                row["views"][V] = {"fwd_ms": t_f, "fwd_bwd_ms": t_fb, "point_fwd_ms": p_f, "point_fwd_bwd_ms": p_fb,
                                   "fwd_bwd_over_rendering_equation": t_fb / t_re}
                print(f"       V={V}: shade fwd {t_f:8.3f} ms, fwd+bwd {t_fb:8.3f} ms  (K point lights: {p_f:.3f} / "
                      f"{p_fb:.3f} ms; {t_fb / t_re:.2f}x rendering_equation N=32)", flush=True)
            results.append(row)
            del T
            torch.cuda.empty_cache()
    print(json.dumps({"bench": "shaped_lights", **info, "P": P, "recipe": args.recipe, "iters": args.iters,
                      "rendering_equation_n32_fwd_bwd_ms": t_re, "results": results}))


if __name__ == "__main__":
    main()

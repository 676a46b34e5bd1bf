"""Per-pixel point, directional, spot and rect lights on the GPU: shadow-trace time and rate, shading forward and
forward + backward, and the peak memory of each, against the per-Gaussian path for the same lights (trace_lights /
trace_shaped_lights over the Gaussians + shade / shade_shaped).

    python tools/bench_pixel_lights.py [--P 1000000] [--out result.json]

Light sets: 1 point light, 8 point lights and one softbox (a rect light at M = 4, 16 rays per pixel).  The G-buffer is
synthetic, as tools/bench_pixel_shading.py's: surface points on the scene, random normals and materials.  Prints one
JSON line per case, then the card's name and power limit, and writes them all to --out when given."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relightable3dgaussian_b200 import lights as lt  # noqa: E402
from relightable3dgaussian_b200 import synth  # noqa: E402
from relightable3dgaussian_b200.raytracer import RayTracer, inverse_covariance  # noqa: E402
from bench_pixel_shading import gbuffer, timed  # noqa: E402


def light_sets():
    dev = "cuda"
    g = torch.Generator().manual_seed(7)
    eight = torch.randn(8, 3, generator=g) * 0.5 + torch.tensor([0.0, -1.5, 2.0])
    return {
        "1 point": lt.Lights.point(torch.tensor([[0.3, -1.8, 2.2]], device=dev), torch.full((1, 3), 8.0, device=dev)),
        "8 point": lt.Lights.point(eight.to(dev), torch.full((8, 3), 2.0, device=dev)),
        "softbox M=4": lt.ShapedLights.rect(torch.tensor([[0.0, -2.0, 2.0]], device=dev),
                                            torch.tensor([[0.6, 0.0, 0.0]], device=dev),
                                            torch.tensor([[0.0, 0.3, 0.4]], device=dev), torch.full((1, 3), 3.0, device=dev),
                                            M=4, seed=1),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pixel_lights needs a CUDA GPU")
    results = []
    for recipe in ("shell-v1", "cube-v1"):
        sc = synth.make_scene(args.P, recipe, 0, 0)
        m, s, r, o, nr = (t.cuda() for t in (sc.means3D, sc.scales, sc.rotations, sc.opacities[:, 0].contiguous(), sc.normals))
        inv = inverse_covariance(s, r).contiguous()
        rt = RayTracer(m, s, r)
        g_base, g_rough = torch.full((args.P, 3), 0.5, device="cuda"), torch.full((args.P, 1), 0.3, device="cuda")
        for H, W in ((800, 800), (1080, 1920)):
            g = gbuffer(recipe, H, W)
            for name, lights in light_sets().items():
                R = lt.num_rays(lights)
                res = dict(recipe=recipe, P=args.P, H=H, W=W, lights=name, rays_per_pixel=R)
                trace = lambda: rt.trace_pixel_lights(g["points"], lights, m, inv, o, nr)
                res["trace_ms"], res["trace_peak_mb"] = timed(trace, 1)
                res["trace_rays_per_s"] = H * W * R / (res["trace_ms"] / 1e3)
                T = trace()
                fwd = lambda: lt.shade_pixels(g["base"], g["rough"], g["normal"], g["points"], g["campos"], lights, T)
                res["shade_fwd_ms"], res["shade_fwd_peak_mb"] = timed(torch.no_grad()(fwd), 5)
                base = g["base"].clone().requires_grad_()
                cot = torch.randn(3, H, W, device="cuda")

                def fwd_bwd():
                    out = lt.shade_pixels(base, g["rough"], g["normal"], g["points"], g["campos"], lights, T)
                    out["pbr"].backward(cot)
                res["shade_fwd_bwd_ms"], res["shade_fwd_bwd_peak_mb"] = timed(fwd_bwd, 5)
                del T

                def per_gaussian():      # the same lights per Gaussian: trace over the Gaussians, then shade them
                    if isinstance(lights, lt.Lights):
                        Tg = rt.trace_lights(m, inv, o, nr, lights)
                        with torch.no_grad():
                            lt.shade(g_base, g_rough, nr, g["campos"][None] - m, m, lights, Tg)
                    else:
                        Tg = rt.trace_shaped_lights(m, inv, o, nr, lights)
                        with torch.no_grad():
                            lt.shade_shaped(g_base, g_rough, nr, g["campos"][None] - m, m, lights, Tg)
                res["per_gaussian_trace_shade_ms"], res["per_gaussian_peak_mb"] = timed(per_gaussian, 1)
                print(json.dumps(res), flush=True)
                results.append(res)
    meta = dict(device=torch.cuda.get_device_properties(0).name)
    try:
        meta["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                             capture_output=True, text=True).stdout.strip()
    except OSError:
        pass
    print(json.dumps(meta))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(meta=meta, results=results), f, indent=1)


if __name__ == "__main__":
    main()

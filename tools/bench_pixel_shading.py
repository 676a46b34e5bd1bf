"""Per-pixel (deferred) shading on the GPU: trace rate, shading forward and forward + backward, against the row-wise
composition of existing kernels (sampler + explicit-ray trace + rendering_equation on the transposed G-buffer) and the
per-Gaussian path (visibility bake + rendering_equation over the Gaussians), with the peak memory of each.

    python tools/bench_pixel_shading.py [--P 1000000] [--out result.json]

The G-buffer is synthetic: surface points on the scene (the shell's sphere, or uniform in the cube), normals along the
shell's radius (random for the cube), random materials, zero incidents (the common case).  Prints one JSON line per
case and writes them all to --out when given."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relightable3dgaussian_b200 import synth  # noqa: E402
from relightable3dgaussian_b200.raytracer import RayTracer, fibonacci_sphere_sampling, inverse_covariance  # noqa: E402
from relightable3dgaussian_b200.shading import rendering_equation, shade_pixels  # noqa: E402


class Light:
    def __init__(self, envmap):
        self.envmap, self.transform = envmap, None


def timed(fn, reps=3):
    """Median device time of fn() in ms over `reps` runs after one warm-up, and the peak memory above the start (MB)."""
    fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2], (torch.cuda.max_memory_allocated() - base) / 2**20


def gbuffer(recipe, H, W, seed=1):
    g = torch.Generator().manual_seed(seed)
    if recipe == "shell-v1":
        n = F.normalize(torch.randn(3, H, W, generator=g), dim=0)
        pts = n * 1.03
    else:
        pts = torch.rand(3, H, W, generator=g) * 2.6 - 1.3
        n = F.normalize(torch.randn(3, H, W, generator=g), dim=0)
    return dict(points=pts.cuda(), normal=n.cuda(), base=(torch.rand(3, H, W, generator=g) * 0.8 + 0.1).cuda(),
                rough=(torch.rand(1, H, W, generator=g) * 0.8 + 0.1).cuda(), campos=torch.tensor([0.0, -4.0, 1.5]).cuda())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pixel_shading needs a CUDA GPU")
    env = (torch.rand(256, 512, 3, generator=torch.Generator().manual_seed(3)) * 2).cuda()
    light = Light(env)
    results = []
    for recipe in ("shell-v1", "cube-v1"):
        sc = synth.make_scene(args.P, recipe, 0, 0)
        m, s, r, o, nr = (t.cuda() for t in (sc.means3D, sc.scales, sc.rotations, sc.opacities[:, 0].contiguous(), sc.normals))
        inv = inverse_covariance(s, r).contiguous()
        rt = RayTracer(m, s, r)
        for H, W in ((800, 800), (1080, 1920)):
            g = gbuffer(recipe, H, W)
            for N in (32, 64):
                res = dict(recipe=recipe, P=args.P, H=H, W=W, N=N)
                trace = lambda: rt.trace_pixels(g["points"], g["normal"], N, m, inv, o, nr)
                res["trace_ms"], res["trace_peak_mb"] = timed(trace, 1)
                res["trace_rays_per_s"] = H * W * N / (res["trace_ms"] / 1e3)
                T = trace()
                fwd = lambda: shade_pixels(g["base"], g["rough"], g["normal"], g["points"], g["campos"], T, light)
                res["shade_fwd_ms"], res["shade_fwd_peak_mb"] = timed(torch.no_grad()(fwd), 5)
                base = g["base"].clone().requires_grad_()
                cot = torch.randn(3, H, W, device="cuda")

                def fwd_bwd():
                    out = shade_pixels(base, g["rough"], g["normal"], g["points"], g["campos"], T, light)
                    out["pbr"].backward(cot)
                res["shade_fwd_bwd_ms"], res["shade_fwd_bwd_peak_mb"] = timed(fwd_bwd, 5)
                del T

                def rowwise():      # the same frame from existing kernels on the transposed G-buffer
                    n = g["normal"].reshape(3, -1).T
                    nh = n / torch.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2]).clamp_min(1e-12)[:, None]
                    dirs, areas = fibonacci_sphere_sampling(nh, N, random_rotate=False)
                    p = g["points"].reshape(3, -1).T
                    vis = rt.trace_visibility(p[:, None, :].expand(-1, N, -1), dirs, m, inv, o, nr)["visibility"]
                    with torch.no_grad():
                        rendering_equation(g["base"].reshape(3, -1).T, g["rough"].reshape(1, -1).T, n, g["campos"][None] - p,
                                           torch.zeros(H * W, 16, 3, device="cuda"), light, vis, dirs, areas)
                res["rowwise_ms"], res["rowwise_peak_mb"] = timed(rowwise, 1)

                def per_gaussian():  # the per-Gaussian path's shading work: bake + rendering_equation over the Gaussians
                    vis, dirs, areas = (rt.bake_visibility(m, inv, o, nr, N)[k] for k in ("visibility", "incident_dirs", "incident_areas"))
                    with torch.no_grad():
                        rendering_equation(sc_base, sc_rough, nr, g["campos"][None] - m, torch.zeros(args.P, 16, 3, device="cuda"),
                                           light, vis, dirs, areas)
                sc_base, sc_rough = torch.full((args.P, 3), 0.5, device="cuda"), torch.full((args.P, 1), 0.3, device="cuda")
                res["per_gaussian_bake_shade_ms"], res["per_gaussian_peak_mb"] = timed(per_gaussian, 1)
                print(json.dumps(res), flush=True)
                results.append(res)
    dev = torch.cuda.get_device_properties(0)
    meta = dict(device=dev.name)
    try:
        import subprocess
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

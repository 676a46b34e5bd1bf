#!/usr/bin/env python3
"""Time of the ray-traced indirect light (RayTracer.bake_radiance + fit_incident_sh) beside the LBVH build and the
visibility bake it shares rays and hits with.

  python tools/bench_indirect.py [--recipes shell-v1 cube-v1] [--sizes 300000 1000000] [--samples 32 64 384]
                                 [--rounds 3] [--ridge 1e-3]

Scenes are synth's, with the shell's normals turned inward so that its bake rays cross the shell (outward rays of a
convex shell meet nothing); the payload is the scene's degree-3 SH, fitted back into degree-3 incident SH.  Each round
runs build, visibility bake, radiance bake and fit once, one after the other (so the variants alternate), each timed
with CUDA events; the first round is a warm-up and the table shows medians of the others.

Per configuration it prints rays/s of both bakes, the radiance bake's time over the visibility bake's (which stops at
T < 0.9), the mean hits composited per ray and the mean k-buffer rounds per ray (derived exactly from each ray's hit
count and final T: a ray that ran out of hits needed hits // K + 1 rounds, one stopped by T < 1e-4 ceil(hits / K)),
and the relative RMS error of the fit: the shading step's local light of the fitted incidents at the bake directions
against the traced radiance, on the first 50k Gaussians.  The device name and power limit are read in the same run.
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
from relightable3dgaussian_b200 import shading, synth  # noqa: E402
from relightable3dgaussian_b200.raytracer import RayTracer, fit_incident_sh, inverse_covariance  # noqa: E402

K = 16                                  # RAD_K of csrc/indirect.cu
T_MIN = 1e-4
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


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return out, a.elapsed_time(b)


class _Env:
    def __init__(self):
        self.envmap = torch.zeros(8, 16, 3, device=DEV)


def fit_error(L, inc, normals, dirs, areas, sub=50_000):
    """Relative RMS of the shading step's local light of `inc` against the radiance it was fitted to."""
    s = slice(0, min(sub, L.shape[0]))
    P = inc[s].shape[0]
    _, extra = shading.rendering_equation(torch.full((P, 3), 0.5, device=DEV), torch.full((P, 1), 0.5, device=DEV),
                                          normals[s], normals[s], inc[s], _Env(), torch.ones_like(areas[s]), dirs[s], areas[s])
    loc = extra["local_incident_lights"]
    return float(((loc - L[s]) ** 2).sum().sqrt() / (L[s] ** 2).sum().sqrt())


def run(recipe, P, N, rounds, ridge):
    sc = synth.make_scene(P, recipe, 0, 0)
    d = lambda t: t.to(DEV).contiguous()
    means, scales, rots, shs = d(sc.means3D), d(sc.scales), d(sc.rotations), d(sc.shs)
    normals = d(-sc.normals if recipe == "shell-v1" else sc.normals)
    opacity = d(sc.opacities[:, 0])
    inv = inverse_covariance(scales, rots)
    times = {"build": [], "visibility": [], "radiance": [], "fit": []}
    for r in range(rounds + 1):
        rt, t_build = timed(lambda: RayTracer(means, scales, rots))
        vis, t_vis = timed(lambda: rt.bake_visibility(means, inv, opacity, normals, N))
        rad, t_rad = timed(lambda: rt.bake_radiance(means, inv, opacity, normals, shs, 3, N, want_hits=True))
        inc, t_fit = timed(lambda: fit_incident_sh(rad["radiance"], normals, 3, ridge))
        if r > 0:
            for k, t in zip(times, (t_build, t_vis, t_rad, t_fit)):
                times[k].append(t)
        if r < rounds:
            del vis, rad, inc
    med = {k: statistics.median(v) for k, v in times.items()}
    h, T = rad["num_hits"], rad["transmittance"][..., 0]
    stopped = T < T_MIN
    rounds_per_ray = torch.where(stopped, (h + K - 1) // K, h // K + 1).double().mean().item()
    err = fit_error(rad["radiance"], inc, normals, vis["incident_dirs"], vis["incident_areas"])
    rays = P * N
    return {"recipe": recipe, "P": P, "N": N, "ms": {k: round(v, 3) for k, v in med.items()},
            "rays_per_s": {"visibility": rays / (med["visibility"] * 1e-3), "radiance": rays / (med["radiance"] * 1e-3)},
            "radiance_over_visibility": med["radiance"] / med["visibility"],
            "hits_per_ray": h.double().mean().item(), "rounds_per_ray": rounds_per_ray,
            "stopped_by_T": stopped.double().mean().item(), "fit_rel_rms": err, "ridge": ridge}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recipes", nargs="+", default=["shell-v1", "cube-v1"])
    ap.add_argument("--sizes", nargs="+", type=int, default=[300_000, 1_000_000])
    ap.add_argument("--samples", nargs="+", type=int, default=[32, 64, 384])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ridge", type=float, default=1e-3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_indirect.py needs a GPU")
    info = device_info()
    print(f"# {info['device']}, power limit {info.get('power_limit')}; medians of {args.rounds} rounds (CUDA events)")
    print(f"{'recipe':9} {'P':>8} {'N':>4} | {'build':>8} {'vis':>9} {'radiance':>9} {'fit':>8} ms | "
          f"{'vis Mray/s':>10} {'rad Mray/s':>10} {'rad/vis':>7} | {'hits':>6} {'rounds':>6} {'T<1e-4':>7} | fit err")
    results = []
    for recipe in args.recipes:
        for P in args.sizes:
            for N in args.samples:
                r = run(recipe, P, N, args.rounds, args.ridge)
                results.append(r)
                m = r["ms"]
                print(f"{recipe:9} {P:>8} {N:>4} | {m['build']:8.2f} {m['visibility']:9.2f} {m['radiance']:9.2f} "
                      f"{m['fit']:8.2f}    | {r['rays_per_s']['visibility'] / 1e6:10.0f} {r['rays_per_s']['radiance'] / 1e6:10.0f} "
                      f"{r['radiance_over_visibility']:7.2f} | {r['hits_per_ray']:6.2f} {r['rounds_per_ray']:6.3f} "
                      f"{r['stopped_by_T']:7.2%} | {r['fit_rel_rms']:.4f}", flush=True)
                torch.cuda.empty_cache()
    print(json.dumps({"bench": "indirect", **info, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

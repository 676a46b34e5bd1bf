#!/usr/bin/env python3
"""Forward + backward time of the fused multi-view consistency losses (relightable3dgaussian_b200.multiview) against
the fp32 PyTorch formulation of the same definition (tests/multiview_oracle.py, autograd), and, for scale, a stage-1
rasterizer forward + backward of the two views (rasterize_views, ray_depth=True, 1M Gaussians).

  python tools/bench_multiview.py [--iters 20] [--warmup 3] [--rounds 3] [--skip-torch]

Prints one JSON line: device name and power limit (read in the same run), and per size and pair count the median
milliseconds of each variant over `rounds` alternating rounds, with two floors computed from the shapes: HBM bytes
(per pixel and pair: depth, normal and grey of the reference read and the gradients written, fwd + bwd) over the
3.35 TB/s data sheet, and the per-pixel fp32 work (~49 taps x ~60 flops forward, ~2x that backward) over 67 TFLOP/s."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import multiview_oracle as mo  # noqa: E402
from relightable3dgaussian_b200 import multiview, synth  # noqa: E402
from relightable3dgaussian_b200 import rasterizer as R  # noqa: E402

SIZES = [(800, 800), (1200, 1600), (1080, 1920)]         # (H, W)
PAIRS = {1: [(0, 1)], 4: [(0, 1), (1, 0), (0, 2), (2, 0)]}
HBM_BPS, FP32_FLOPS = 3.35e12, 67e12                     # H100 SXM data sheet (not reached; the floors use it)
FLOPS_PER_PIXEL = 49 * 60 * 3                            # forward + recomputing backward, per pixel and pair
BYTES_PER_PIXEL = 4 * (5 + 1 + 5)                        # fwd: depth, normal, grey; bwd: + tap depth, grads written


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [s.strip() for s in out.split(",")]
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        info["power_limit"] = f"unavailable ({e})"
    return info


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-torch", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multiview needs a GPU")
    dev = torch.device("cuda")
    res = {"tool": "bench_multiview", **device_info(), "cases": []}
    sc = synth.make_scene(1_000_000, "shell-v1", 0, 5)
    leaf = lambda t: t.to(dev).requires_grad_(True)
    g3 = [leaf(t) for t in (sc.means3D, sc.opacities, sc.shs, sc.scales, sc.rotations, sc.features)]
    for H, W in SIZES:
        depth, normal, gray, cams = mo.random_scene(W, H, 3, seed=1)
        d = depth.float().to(dev).requires_grad_()
        n = normal.float().to(dev).requires_grad_()
        g = gray.float().to(dev)
        settings = [R.GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, torch.zeros(3, device=dev),
                                                    1.0, c.viewmatrix.to(dev), torch.eye(4, device=dev), 0,
                                                    torch.zeros(3, device=dev), False, True, True, False) for c in cams]
        rcams = [synth.make_camera(0, W, H), synth.make_camera(0, W, H, elevation_deg=34.0)]
        rset = [R.GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, torch.zeros(3, device=dev), 1.0,
                                                c.viewmatrix.to(dev), c.projmatrix.to(dev), 3, c.campos.to(dev), False,
                                                True, True, False) for c in rcams]

        def raster():
            m2 = torch.zeros(2, g3[0].shape[0], 3, device=dev, requires_grad=True)
            out = R.rasterize_views(g3[0], m2, g3[1], settings=rset, shs=g3[2], scales=g3[3], rotations=g3[4],
                                    features=g3[5], ray_depth=True)
            (out[2].sum() + out[4].sum()).backward()

        for B, pairs in PAIRS.items():
            def fused():
                geo, photo = multiview.consistency_loss(d, n, g, settings, pairs)
                (geo.sum() + photo.sum()).backward()

            def eager():
                geo, photo = mo.consistency(d, n, g, cams, pairs)
                (geo.sum() + photo.sum()).backward()

            variants = {"fused": fused, "raster_2views": raster}
            if not args.skip_torch:
                variants["torch_fp32"] = eager
            times = {k: [] for k in variants}
            for _ in range(args.rounds):                 # alternating rounds
                for k, fn in variants.items():
                    times[k].append(time_ms(fn, args.iters if k != "torch_fp32" else max(args.iters // 10, 2),
                                            args.warmup))
            med = {k: statistics.median(v) for k, v in times.items()}
            px = B * H * W
            floor_hbm = px * BYTES_PER_PIXEL / HBM_BPS * 1e3
            floor_fp32 = px * FLOPS_PER_PIXEL / FP32_FLOPS * 1e3
            case = {"H": H, "W": W, "B": B, **{f"{k}_ms": round(v, 4) for k, v in med.items()},
                    "floor_hbm_ms": round(floor_hbm, 4), "floor_fp32_ms": round(floor_fp32, 4),
                    "fused_share_of_floor": round(max(floor_hbm, floor_fp32) / med["fused"], 4)}
            if "torch_fp32" in med:
                case["speedup_vs_torch"] = round(med["torch_fp32"] / med["fused"], 2)
            res["cases"].append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

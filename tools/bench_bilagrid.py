#!/usr/bin/env python3
"""Forward and forward + backward time of the fused bilateral-grid slice (relightable3dgaussian_b200.bilagrid.slice)
against the torch formulation (F.grid_sample on the grids, align_corners=True, padding_mode="border", then the per-pixel
3x4 matmul; tests/bilagrid_oracle.py torch_slice), both on the GPU in fp32, with gsplat's default 16x16x8 grids.  The
backward asks for the gradients of both the image and the grids, as in training.

  python tools/bench_bilagrid.py [--iters 100] [--warmup 10] [--rounds 3]

Prints one JSON line: device name and power limit (read in the same run), and per size and batch the median
milliseconds of each variant over `rounds` alternating rounds, the byte floors (forward 24 B per pixel: rgb in, out;
backward 36 B per pixel: rgb and dL/dout in, dL/drgb out, plus the grids' partials written and read) and the fused
kernels' share of the 3.35 TB/s data-sheet HBM bandwidth."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import bilagrid_oracle as bo  # noqa: E402
from relightable3dgaussian_b200 import _lib, bilagrid  # noqa: E402

SIZES = [(800, 800), (1200, 1600), (1080, 1920)]         # (H, W)
BATCHES = [1, 8]
GRID = (16, 16, 8)                                      # GX, GY, L
HBM_BPS = 3.35e12                                       # H100 SXM data sheet (not reached; the floors use it)


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [s.strip() for s in out.split(",")]
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        info["power_limit"] = f"unavailable ({e})"
    return info


def time_ms(step, iters, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        step()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_bilagrid.py measures on a CUDA GPU"
    GX, GY, L = GRID
    res = dict(device_info(), iters=args.iters, rounds=args.rounds, grid=[GX, GY, L], sizes=[])
    variants = {"fused": lambda g, x, ids: bilagrid.slice(g, x, ids),
                "torch_grid_sample": lambda g, x, ids: bo.torch_slice(g, x, ids)}
    for H, W in SIZES:
        for N in BATCHES:
            G = N
            grids, rgb = bo.random_case(G, N, H, W, L, GY, GX, seed=0, noise=0.1)
            g = torch.from_numpy(grids).cuda().requires_grad_(True)
            x = torch.from_numpy(rgb).cuda().requires_grad_(True)
            ids = list(range(N))
            dout = torch.randn_like(x)

            def fwd(fn):
                def step():
                    with torch.no_grad():
                        fn(g, x, ids)
                return step

            def fwd_bwd(fn):
                def step():
                    g.grad = x.grad = None
                    fn(g, x, ids).backward(dout)
                return step

            times = {f"{k}_{m}": [] for k in variants for m in ("fwd", "fwd_bwd")}
            for _ in range(args.rounds):          # alternate the variants so that drift hits all of them alike
                for k, fn in variants.items():
                    times[f"{k}_fwd"].append(time_ms(fwd(fn), args.iters, args.warmup))
                    times[f"{k}_fwd_bwd"].append(time_ms(fwd_bwd(fn), args.iters, args.warmup))
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            px = N * H * W
            part = _lib.load().r3dg_bilagrid_tmp_bytes(G, N, H, W, GX, GY, L)
            floor_fwd_us = 24 * px / HBM_BPS * 1e6
            floor_bwd_us = (36 * px + 2 * part) / HBM_BPS * 1e6       # partials: an upper bound, written once, read once
            res["sizes"].append(dict(
                H=H, W=W, N=N, ms={k: round(v, 4) for k, v in med.items()},
                ms_all={k: [round(t, 4) for t in v] for k, v in times.items()},
                speedup_fwd=round(med["torch_grid_sample_fwd"] / med["fused_fwd"], 2),
                speedup_fwd_bwd=round(med["torch_grid_sample_fwd_bwd"] / med["fused_fwd_bwd"], 2),
                floor_us=dict(fwd=round(floor_fwd_us, 2), fwd_bwd=round(floor_fwd_us + floor_bwd_us, 2)),
                hbm_share_fused=dict(fwd=round(floor_fwd_us / (med["fused_fwd"] * 1e3), 3),
                                     fwd_bwd=round((floor_fwd_us + floor_bwd_us) / (med["fused_fwd_bwd"] * 1e3), 3))))
            print(json.dumps(res["sizes"][-1]), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

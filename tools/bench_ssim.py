#!/usr/bin/env python3
"""Forward + backward time of the fused SSIM loss (relightable3dgaussian_b200.losses.ssim) against the
reference formula (utils/loss_utils.py:32-63, restated in tests/ssim_oracle.py) run the way the reference
runs it (cuDNN defaults: TF32 convolutions) and with IEEE fp32 convolutions.  The loss is differentiated
with respect to img1 only, as in training (the ground-truth image needs no gradient).

  python tools/bench_ssim.py [--iters 200] [--warmup 20] [--rounds 3]

Prints one JSON line: device name and power limit (read in the same run), per size the median
milliseconds per forward+backward of each variant over `rounds` alternating rounds, the fused forward
and backward alone, and the byte and FLOP floors computed from the shape."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import ssim_oracle as oss  # noqa: E402
from relightable3dgaussian_b200 import losses  # noqa: E402

SIZES = [(3, 800, 800), (3, 1200, 1600), (3, 1080, 1920)]
HBM_BPS, FP32_FLOPS = 3.35e12, 67e12          # H100 SXM data sheet (not reached; the floors use them)
FWD_FMA, BWD_FMA = 5 * 22, 3 * 22             # per element: 5 separable blurs forward, 3 transposed blurs backward
BYTES = 8 + 8 + 4                             # per element: read x, y forward; read x, y and write dL/dx backward


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
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ssim.py measures on a CUDA GPU"
    res = dict(device_info(), iters=args.iters, rounds=args.rounds, sizes=[])
    variants = {
        "fused": lambda x, y: losses.ssim(x, y),
        "reference_tf32": lambda x, y: oss.ssim(x, y, ieee=False),
        "reference_ieee": lambda x, y: oss.ssim(x, y, ieee=True),
    }
    for shape in SIZES:
        a, b, _ = oss.ssim_case("rendered", shape, seed=0)
        x, y = a.cuda().requires_grad_(True), b.cuda()

        def fwd_bwd(fn):
            def step():
                x.grad = None
                fn(x, y).backward()
            return step

        times = {k: [] for k in variants}
        for _ in range(args.rounds):              # alternate the variants so that drift hits all of them alike
            for k, fn in variants.items():
                times[k].append(time_ms(fwd_bwd(fn), args.iters, args.warmup))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        with torch.no_grad():
            fwd = time_ms(lambda: losses.ssim(x, y), args.iters, args.warmup)
        loss = losses.ssim(x, y)
        bwd = time_ms(lambda: loss.backward(retain_graph=True), args.iters, args.warmup)
        n = a.numel()
        floor_bytes_us = BYTES * n / HBM_BPS * 1e6
        floor_flop_us = 2 * (FWD_FMA + BWD_FMA) * n / FP32_FLOPS * 1e6
        res["sizes"].append(dict(
            shape=list(shape), ms={k: round(v, 4) for k, v in med.items()}, ms_all={k: [round(t, 4) for t in v] for k, v in times.items()},
            fused_fwd_ms=round(fwd, 4), fused_bwd_ms=round(bwd, 4),
            speedup_vs_tf32=round(med["reference_tf32"] / med["fused"], 2),
            speedup_vs_ieee=round(med["reference_ieee"] / med["fused"], 2),
            floor_us=dict(hbm=round(floor_bytes_us, 1), fp32=round(floor_flop_us, 1)),
            floor_share_of_fused=round(max(floor_bytes_us, floor_flop_us) / (med["fused"] * 1e3), 3)))
    print(json.dumps(res))


if __name__ == "__main__":
    main()

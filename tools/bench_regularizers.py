#!/usr/bin/env python3
"""Forward + backward time of the fused smoothness regularisers (relightable3dgaussian_b200.losses
first_order_edge_aware_loss and tv_loss) against the reference formula (utils/loss_utils.py:104-105,113-117 on
kornia's spatial_gradient, restated in tests/smooth_oracle.py) run the way the reference runs it (cuDNN defaults:
TF32 convolutions) and with IEEE fp32 convolutions.

The call forms are the four regularisers a stage-2 step adds (gaussian_renderer/neilf.py), each differentiated
with respect to what the reference differentiates:
  base      EA(base_color * mask, gt)      :284  gradient to base_color (3 x 3 channels)
  rough     EA(roughness * mask, gt)       :291  gradient to roughness (1 x 3)
  diffuse   EA(diffuse * mask, normal)     :299  gradients to diffuse and to the rendered normal (3 x 3)
  tv_normal tv(normal * mask)              :312  gradient to the normal
and `sum`, all four in one loss with one backward.  The mask product is the caller's and is not timed.  The env TV
(:306, tv(env[0].permute(2, 0, 1)) on the default 1 x 16 x 32 x 3 env map) is timed on its own.

  python tools/bench_regularizers.py [--iters 200] [--warmup 20] [--rounds 3]

Prints one JSON line: device name and power limit (read in the same run), per size the median milliseconds per
forward+backward of each variant and call form over `rounds` alternating rounds (CUDA events: what a training step
pays, host launch overhead included), the GPU busy time of the same calls (torch.profiler, a separate pass), and the
HBM floor of each fused call form computed from the shapes."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import smooth_oracle as so  # noqa: E402
from bench_ssim import HBM_BPS, device_info, time_ms  # noqa: E402
from relightable3dgaussian_b200 import losses  # noqa: E402

SIZES = [(800, 800), (1200, 1600), (1080, 1920)]
ENV_SHAPE = (1, 16, 32, 3)                       # DirectLightMap(H=16): arguments/__init__.py env_resolution
FORMS = ["base", "rough", "diffuse", "tv_normal", "sum"]


def variants():
    return {
        "fused": (losses.first_order_edge_aware_loss, losses.tv_loss),
        "reference_tf32": (lambda d, i: so.first_order_edge_aware_loss(d, i, ieee=False), so.tv_loss),
        "reference_ieee": (lambda d, i: so.first_order_edge_aware_loss(d, i, ieee=True), so.tv_loss),
    }


def hbm_floor_us(H, W):
    """Bytes the fused kernels must move per call form (read the inputs forward, read them again and write the
    requested gradients backward), over the data-sheet bandwidth."""
    hw4 = 4.0 * H * W
    b = {"base": hw4 * (2 * (3 + 3) + 3), "rough": hw4 * (2 * (1 + 3) + 1), "diffuse": hw4 * (2 * (3 + 3) + 6),
         "tv_normal": hw4 * 3 * 3}
    b["sum"] = sum(b.values())
    return {k: round(v / HBM_BPS * 1e6, 1) for k, v in b.items()}


def device_ms(run, iters):
    """GPU busy time per call: the summed duration of every kernel and memory operation torch.profiler records over
    `iters` calls.  Unlike the event timing it excludes host-side gaps between launches."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            run()
        torch.cuda.synchronize()
    us = sum(e.self_device_time_total for e in prof.key_averages() if e.device_type == DeviceType.CUDA)
    return us / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_regularizers.py measures on a CUDA GPU"
    res = dict(device_info(), iters=args.iters, rounds=args.rounds, sizes=[])
    var = variants()
    for H, W in SIZES:
        g = torch.Generator().manual_seed(0)
        m, _ = so._mask(H, W, g)
        leaf = lambda t: t.cuda().requires_grad_(True)
        base, rough, diffuse = (leaf(so._rendered(c, H, W, g) * m) for c in (3, 1, 3))
        normal = leaf(torch.nn.functional.normalize(so._rendered(3, H, W, g) * 2 - 1, dim=0) * m)
        gt = so._rendered(3, H, W, g).cuda()
        leaves = (base, rough, diffuse, normal)

        def step(form, ea, tv):
            terms = {"base": lambda: ea(base, gt), "rough": lambda: ea(rough, gt),
                     "diffuse": lambda: ea(diffuse, normal), "tv_normal": lambda: tv(normal)}
            parts = list(terms.values()) if form == "sum" else [terms[form]]

            def run():
                for t in leaves:
                    t.grad = None
                sum(p() for p in parts).backward()
            return run

        times = {k: {f: [] for f in FORMS} for k in var}
        for _ in range(args.rounds):             # alternate the variants so that drift hits all of them alike
            for k, (ea, tv) in var.items():
                for f in FORMS:
                    times[k][f].append(time_ms(step(f, ea, tv), args.iters, args.warmup))
        med = {k: {f: round(sorted(v)[len(v) // 2], 4) for f, v in t.items()} for k, t in times.items()}
        dev = {k: {f: round(device_ms(step(f, ea, tv), 20), 4) for f in FORMS} for k, (ea, tv) in var.items()}
        res["sizes"].append(dict(
            shape=[3, H, W], ms=med, device_ms=dev,
            speedup_vs_tf32={f: round(med["reference_tf32"][f] / med["fused"][f], 2) for f in FORMS},
            speedup_vs_ieee={f: round(med["reference_ieee"][f] / med["fused"][f], 2) for f in FORMS},
            hbm_floor_us=hbm_floor_us(H, W)))
    env = torch.rand(ENV_SHAPE, generator=torch.Generator().manual_seed(1)).cuda().requires_grad_(True)
    env_ms = {k: [] for k in var}
    for _ in range(args.rounds):
        for k, (_, tv) in var.items():
            def run(tv=tv):
                env.grad = None
                tv(env[0].permute(2, 0, 1)).backward()
            env_ms[k].append(time_ms(run, args.iters, args.warmup))
    res["env_tv"] = dict(shape=list(ENV_SHAPE), ms={k: round(sorted(v)[len(v) // 2], 4) for k, v in env_ms.items()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Time of the similarity transform of Gaussian models (compose.transform_gaussians) at 1M Gaussians, against the
same transform written as PyTorch einsums.

  python tools/bench_compose.py [--P 1000000] [--objects 1 16] [--iters 20]

Workload: the full PBR model's transformed tensors: xyz, normal, rotation, scaling, f_rest and incidents_rest at
degree 3 (C = 3), and visibility_rest at degree 3 and at degree 4 (C = 1; relighting.py pads composed visibility to
degree 4), for K objects of equal size.  Timings are CUDA-event medians over --iters calls after a warm-up: the
forward, and the forward + backward.  The bytes the pass must move are computed from the shapes (every input row read
once and every output row written once; the backward reads the inputs and the output cotangents and writes the input
gradients), and the share of the 3.35 TB/s HBM3 bound is those bytes over the time.  The device name and power limit
are read in the same run.  Ends with one JSON line of everything."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from relightable3dgaussian_b200 import compose  # noqa: E402

DEV = torch.device("cuda")
HBM_BYTES_PER_S = 3.35e12


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


def sh_rotations(quat, L):
    """D^l(R) of each object (fp64 least squares, as tests/compose64.py), for the einsum comparison."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import compose64
    R = compose64.build_rotation(quat.double())
    return [compose64.sh_rotation(R, l).float() for l in range(1, L + 1)]


def einsum_transform(rows, shs, quat, t, s, obj, Ds):
    """The forward as PyTorch ops: per-row pose gathered by object id, bands rotated with einsum."""
    xyz, normal, rotation, scaling = rows
    R = compose.build_rotation(quat)[obj]
    out = [s[obj, None] * torch.einsum("pij,pj->pi", R, xyz) + t[obj], torch.einsum("pij,pj->pi", R, normal)]
    q = (quat / quat.norm(dim=-1, keepdim=True))[obj]
    w1, x1, y1, z1 = q.unbind(-1)
    w2, x2, y2, z2 = rotation.unbind(-1)
    out.append(torch.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                            w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1))
    out.append(scaling + s.log()[obj, None])
    for sh in shs:
        L = int(round((sh.shape[1] + 1) ** 0.5)) - 1
        out.append(torch.cat([torch.einsum("pij,pjc->pic", Ds[l - 1][obj], sh[:, l * l - 1:(l + 1) ** 2 - 1])
                              for l in range(1, L + 1)], 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--objects", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_compose.py needs a CUDA GPU")
    info = device_info()
    P = args.P
    g = torch.Generator().manual_seed(0)
    rows = [torch.randn(P, w, generator=g).to(DEV) for w in (3, 3, 4, 3)]
    results = []
    for vis_deg in (3, 4):
        shs = [torch.randn(P, 15, 3, generator=g).to(DEV), torch.randn(P, 15, 3, generator=g).to(DEV),
               torch.randn(P, (vis_deg + 1) ** 2 - 1, 1, generator=g).to(DEV)]
        floats = sum(r.shape[1] for r in rows) + sum(x[0].numel() for x in shs)
        fwd_bytes = 2 * 4 * P * floats                        # read every input row, write every output row
        bwd_bytes = 3 * 4 * P * floats                        # read inputs and cotangents, write input gradients
        for K in args.objects:
            quat = torch.randn(K, 4, generator=g).to(DEV)
            t, s = torch.randn(K, 3, generator=g).to(DEV), (torch.rand(K, generator=g) + 0.5).to(DEV)
            offsets = [P * k // K for k in range(K + 1)]
            leaves = [x.clone().requires_grad_(True) for x in rows + shs]
            cots = None

            def fwd():
                with torch.no_grad():
                    return compose.transform_gaussians(*rows, shs, quat, t, s, offsets)

            def fwd_bwd():
                nonlocal cots
                outs = compose.transform_gaussians(*leaves[:4], leaves[4:], quat.requires_grad_(True),
                                                   t.requires_grad_(True), s.requires_grad_(True), offsets)
                outs = list(outs[:4]) + outs[4]
                if cots is None:
                    cots = [torch.randn_like(o) for o in outs]
                torch.autograd.backward(outs, cots)

            obj = torch.repeat_interleave(torch.arange(K, device=DEV), torch.tensor([b - a for a, b in zip(offsets, offsets[1:])], device=DEV))
            Ds = sh_rotations(quat, vis_deg)
            ms_f = median_ms(fwd, args.iters)
            ms_fb = median_ms(fwd_bwd, args.iters)
            ms_e = median_ms(lambda: einsum_transform(rows, shs, quat, t, s, obj, Ds), args.iters)
            r = dict(P=P, K=K, visibility_degree=vis_deg, fwd_ms=round(ms_f, 4), fwd_bwd_ms=round(ms_fb, 4),
                     einsum_fwd_ms=round(ms_e, 4), fwd_bytes=fwd_bytes, bwd_bytes=bwd_bytes,
                     fwd_hbm_share=round(fwd_bytes / HBM_BYTES_PER_S / (ms_f * 1e-3), 3),
                     fwd_bwd_hbm_share=round((fwd_bytes + bwd_bytes) / HBM_BYTES_PER_S / (ms_fb * 1e-3), 3))
            print(f"K={K:3d} vis deg {vis_deg}: forward {ms_f:.3f} ms ({r['fwd_hbm_share']:.0%} of HBM), "
                  f"forward + backward {ms_fb:.3f} ms ({r['fwd_bwd_hbm_share']:.0%}), einsum forward {ms_e:.3f} ms")
            results.append(r)
    print(json.dumps(dict(info, results=results)))


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Time of the fused densify_and_prune (relightable3dgaussian_b200.densify) against the reference's semantics as
PyTorch runs them (the restatement in tests/densify_oracle.py: boolean indexing and torch.cat), at P in
{300k, 1M, 3M} with the stage-1 (7) and PBR (13) parameter groups, about 2 % clone, 1 % split, 3 % prune; and one
add_densification_stats call at 1M.  Each densify call needs fresh inputs, so every timed call starts from a copy
of the model made beforehand; CUDA-event time covers the call and host wall time includes its syncs.

  python tools/bench_densify.py [--iters 5] [--rounds 3]

Prints one JSON line: device name and power limit, per configuration the median over `rounds` alternating rounds."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import densify_oracle as do  # noqa: E402
from relightable3dgaussian_b200 import densify  # noqa: E402

SIZES = [300_000, 1 << 20, 3 << 20]
HBM_BPS = 3.35e12                                # H100 SXM data sheet


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"] = out
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit"] = f"unavailable ({e})"
    return info


def time_call(make, fn, iters):
    """Median (CUDA-event ms, host wall ms) of fn(model) over `iters` fresh models."""
    ev, wall = [], []
    for _ in range(iters):
        m = make()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        w0 = time.perf_counter()
        t0.record()
        with contextlib.redirect_stdout(io.StringIO()):
            fn(m)
        t1.record()
        w1 = time.perf_counter()
        t1.synchronize()
        ev.append(t0.elapsed_time(t1))
        wall.append((w1 - w0) * 1e3)
        del m
    return sorted(ev)[len(ev) // 2], sorted(wall)[len(wall) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_densify.py measures on a CUDA GPU"
    res = dict(device_info(), iters=args.iters, rounds=args.rounds, densify=[], stats={})
    for pbr in (False, True):
        for P in SIZES:
            do.LARGE[f"bench_{P}_{pbr}"] = (P, pbr, "real", {})
            case = do.densify_case(f"bench_{P}_{pbr}", device="cuda")
            base = do.build_model(case, do.StandIn, device="cuda")

            def make():
                return clone_model(base)
            variants = {"fused": lambda m: densify.densify_and_prune(m, **case["args"]),
                        "reference": lambda m: do.restate_densify_and_prune(m, **case["args"])}
            times = {k: [] for k in variants}
            for _ in range(args.rounds):
                for k, fn in variants.items():
                    times[k].append(time_call(make, fn, args.iters))
            med = {k: (sorted(t[0] for t in v)[len(v) // 2], sorted(t[1] for t in v)[len(v) // 2]) for k, v in times.items()}
            nbytes = sum(t.numel() * 4 for t in do.output_tensors(base).values())
            res["densify"].append(dict(P=P, groups=13 if pbr else 7, old_bytes=nbytes,
                                       fused_ms=round(med["fused"][0], 3), fused_wall_ms=round(med["fused"][1], 3),
                                       reference_ms=round(med["reference"][0], 3),
                                       reference_wall_ms=round(med["reference"][1], 3),
                                       speedup_wall=round(med["reference"][1] / med["fused"][1], 2),
                                       hbm_floor_ms=round(2 * nbytes / HBM_BPS * 1e3, 3)))
            print(json.dumps(res["densify"][-1]), file=sys.stderr)
            del base, case
            torch.cuda.empty_cache()
    P = 1 << 20
    case = do.densify_case("s1_p1m", device="cuda")
    m = do.build_model(case, do.StandIn, device="cuda")
    vpt = torch.zeros((P, 3), device="cuda", requires_grad=True)
    vpt.grad = torch.randn((P, 3), device="cuda")
    m._normal.grad = torch.randn((P, 3), device="cuda")
    filt = torch.rand(P, device="cuda") < 0.7
    w = torch.rand((P, 1), device="cuda")
    radii = torch.randint(0, 30, (P,), device="cuda", dtype=torch.int32)
    variants = {"fused": lambda: densify.add_densification_stats(m, vpt, filt, w, radii=radii),
                "reference": lambda: (do.restate_add_densification_stats(m, vpt, filt, w, radii=radii))}
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            w0 = time.perf_counter()
            t0.record()
            for _ in range(50):
                fn()
            t1.record()
            w1 = time.perf_counter()
            t1.synchronize()
            times[k].append((t0.elapsed_time(t1) / 50, (w1 - w0) * 1e3 / 50))
    for k, v in times.items():
        res["stats"][f"{k}_ms"] = round(sorted(t[0] for t in v)[len(v) // 2], 4)
        res["stats"][f"{k}_wall_ms"] = round(sorted(t[1] for t in v)[len(v) // 2], 4)
    print(json.dumps(res))


def clone_model(base):
    """A deep copy of the model's tensors and optimizer (a densify call replaces them)."""
    m = do.StandIn.__new__(do.StandIn)
    m.use_pbr, m.percent_dense = base.use_pbr, base.percent_dense
    groups = []
    for g in base.optimizer.param_groups:
        p = torch.nn.Parameter(g["params"][0].detach().clone())
        setattr(m, do.ATTRS[g["name"]], p)
        groups.append({"params": [p], "lr": g["lr"], "name": g["name"]})
    m.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    for g, gb in zip(m.optimizer.param_groups, base.optimizer.param_groups):
        st = base.optimizer.state.get(gb["params"][0])
        if st is not None:
            m.optimizer.state[g["params"][0]] = {k: v.clone() for k, v in st.items()}
    for n in do.STATS + ("max_radii2D",):
        setattr(m, n, getattr(base, n).clone())
    return m


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Time of the MCMC densification (relightable3dgaussian_b200.mcmc) against PyTorch implementations of the same
semantics, at P in {1M, 3M} with the stage-1 (7) and PBR (13) parameter groups and about 5 % dead rows.

* noise, per optimiser step: `inject_noise` (torch.randn + one kernel) and the kernel alone, against the usual PyTorch
  form (gsplat's: covariance by bmm of the scale-rotation factor, sigmoid gate, bmm with the noise; fp32).  The noise
  touches 4 tensors whatever the groups, so it is timed once per P.
* relocation and growth, per call: `relocate_and_grow(cap_max = 2P)` (relocation, then 5 % growth) against the
  restatement in tests/mcmc_oracle.py (boolean indexing, torch.searchsorted on an fp64 cumsum, torch.cat).  Each call
  needs fresh inputs, so every timed call starts from a model built beforehand.

CUDA events; the median of each configuration over `rounds` rounds that alternate fused and PyTorch.  Bytes are
computed from shapes: the noise kernel reads 56 B and writes 12 B a row (torch.randn writes 12 B more); growth reads
every old row of every tensor and writes every new one.

  python tools/bench_mcmc.py [--iters 5] [--rounds 3] [--sizes 1048576,3145728]

Prints one JSON line: device name and power limit, then the results."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import densify_oracle as do  # noqa: E402
import mcmc_oracle as mo  # noqa: E402
from relightable3dgaussian_b200 import _lib, mcmc  # noqa: E402

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


def event_ms(fn, iters, prepare=None):
    """Median CUDA-event ms of fn(state) over `iters` calls, state = prepare() made outside the timed window."""
    ts = []
    for _ in range(iters):
        st = prepare() if prepare else None
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fn(st)
        t1.record()
        t1.synchronize()
        ts.append(t0.elapsed_time(t1))
        del st
    return sorted(ts)[len(ts) // 2]


def torch_noise(m, noise_lr=5e5, k=100, t=0.005):
    """gsplat's inject_noise_to_position in fp32 PyTorch ops."""
    lr = m.optimizer.param_groups[0]["lr"]
    with torch.no_grad():
        R = do.rotation_matrices(m._rotation)
        L = R * torch.exp(m._scaling)[:, None, :]
        cov = torch.bmm(L, L.transpose(1, 2))
        gate = 1 / (1 + torch.exp(-(-k * (torch.sigmoid(m._opacity) - t))))
        noise = torch.randn_like(m._xyz) * gate * noise_lr * lr
        m._xyz.add_(torch.bmm(cov, noise.unsqueeze(-1)).squeeze(-1))


def pbr_case(name):
    """The stage-1 case `name` plus the six PBR groups, seeded here, with moments as densify_oracle.densify_case draws
    them (the seeded PBR tables stop at 1M rows)."""
    c = mo.mcmc_case(name, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0x9b2)
    P = c["P"]
    for n, shape in do.PBR.items():
        c["params"][n] = torch.randn((P,) + shape, generator=g, device="cuda")
        c["moments"][n] = (torch.randn((P,) + shape, generator=g, device="cuda") * 1e-3,
                           torch.rand((P,) + shape, generator=g, device="cuda") * 1e-6)
    return dict(c, pbr=True, name=name.replace("s1_", "pbr_"))


def row_bytes(m):
    n = 0
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        n += p[0].numel() * 4 * (3 if p in m.optimizer.state else 1)
    return n + 4 * len(mo.STATS)


def median(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default=f"{1 << 20},{3 << 20}")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mcmc needs a GPU"
    res = dict(device_info(), noise=[], relocate_and_grow=[])
    for P in [int(s) for s in a.sizes.split(",")]:
        name = "s1_p1m" if P == 1 << 20 else "s1_p3m" if P == 3 << 20 else None
        assert name, "sizes: 1048576 and / or 3145728 (the seeded densify_oracle cases)"
        case = mo.mcmc_case(name, device="cuda")
        m = do.build_model(case, mo.StandIn, device="cuda")
        z = torch.randn((P, 3), device="cuda")
        scale = 5e5 * m.optimizer.param_groups[0]["lr"]
        kernel = lambda _: _lib.call("r3dg_mcmc_noise", m._xyz.device, P, m._xyz.data_ptr(), m._rotation.data_ptr(),
                                     m._scaling.data_ptr(), m._opacity.data_ptr(), z.data_ptr(), scale, 100.0, 0.005)
        for f in (kernel, lambda _: mcmc.inject_noise(m), lambda _: torch_noise(m)):
            f(None)                                                        # warm-up
        r = {"fused_call": [], "fused_kernel": [], "torch": []}
        for _ in range(a.rounds):
            r["fused_kernel"].append(event_ms(kernel, 20 * a.iters))
            r["fused_call"].append(event_ms(lambda _: mcmc.inject_noise(m), 20 * a.iters))
            r["torch"].append(event_ms(lambda _: torch_noise(m), 20 * a.iters))
        med = {k: median(v) for k, v in r.items()}
        res["noise"].append(dict(P=P, **{f"{k}_ms": round(v, 4) for k, v in med.items()},
                                 kernel_bytes=68 * P, kernel_hbm_fraction=round(68 * P / HBM_BPS / (med["fused_kernel"] * 1e-3), 3),
                                 speedup=round(med["torch"] / med["fused_call"], 2)))
        print(json.dumps(res["noise"][-1]), file=sys.stderr)
        del m, case, z
        for pbr in (False, True):
            case = pbr_case(name) if pbr else mo.mcmc_case(name, device="cuda")
            n_new = mcmc.growth_count(P, 2 * P)
            make = lambda: do.build_model(case, mo.StandIn, device="cuda")
            uniforms = lambda: (torch.rand(P, device="cuda"), torch.rand(n_new, device="cuda"))

            def fused(st):
                mcmc.relocate_and_grow(st, 2 * P)

            def restated(st):
                mo.restate_relocate_and_grow(st, 2 * P, u_reloc=st.u[0], u_grow=st.u[1])

            def prep():
                mdl = make()
                mdl.u = uniforms()
                return mdl
            fused(make())
            restated(prep())
            r = {"fused": [], "torch": []}
            for _ in range(a.rounds):
                r["fused"].append(event_ms(fused, a.iters, make))
                r["torch"].append(event_ms(restated, a.iters, prep))
            med = {k: median(v) for k, v in r.items()}
            mdl = make()
            nbytes = row_bytes(mdl) * (2 * P + n_new)
            del mdl
            res["relocate_and_grow"].append(dict(P=P, groups=13 if pbr else 7, n_new=n_new,
                                                 **{f"{k}_ms": round(v, 3) for k, v in med.items()},
                                                 growth_bytes=nbytes,
                                                 growth_hbm_floor_ms=round(nbytes / HBM_BPS * 1e3, 3),
                                                 speedup=round(med["torch"] / med["fused"], 2)))
            print(json.dumps(res["relocate_and_grow"][-1]), file=sys.stderr)
            del case
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

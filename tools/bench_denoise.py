"""The a-trous denoiser on the GPU: forward and forward + backward of `denoise.atrous` against an fp32 PyTorch
formulation of the same filter (pad, shift and sum, differentiated by autograd), with each pass's HBM byte floor.

    python tools/bench_denoise.py [--iters 20] [--out result.json]

Sizes 800 x 800, 1200 x 1600 and 1920 x 1080; V = 1 and 4 views; C = 3 channels with one feature guide (the specular
term's roughness); L = 3 and 5 passes.  The G-buffer is synthetic: a ground plane, a 90 degree crease and a depth step
with seeded noise, and 15 % of the pixels masked.  Prints one JSON line: the card's name and power limit and every
case."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relightable3dgaussian_b200.denoise import atrous  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM HBM3, data sheet
H5 = (1 / 16, 4 / 16, 6 / 16, 4 / 16, 1 / 16)


def gbuffer(V, H, W, F, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ys, xs = torch.meshgrid((torch.arange(H, device="cuda") + 0.5) / H, (torch.arange(W, device="cuda") + 0.5) / W,
                            indexing="ij")
    crease = xs > 0.6
    pts = torch.stack([torch.where(crease, 0.6, xs), ys, torch.where(crease, xs - 0.6, torch.where(ys < 0.3, 0.5, 0.0))])
    nrm = torch.stack([crease.float(), torch.zeros_like(xs), (~crease).float()])
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda")
    return dict(normal=nrm[None] + 0.04 * rnd(V, 3, H, W), points=pts[None] + (0.1 / max(H, W)) * rnd(V, 3, H, W),
                mask=torch.rand(V, H, W, generator=g, device="cuda") > 0.15,
                features=0.3 + 0.05 * rnd(V, F, H, W), x=0.5 + 0.2 * rnd(V, 3, H, W))


def _tap(t, dy, dx):
    H, W = t.shape[-2], t.shape[-1]
    out = torch.zeros_like(t)
    ys, yd = slice(max(dy, 0), H + min(dy, 0)), slice(max(-dy, 0), H + min(-dy, 0))
    xs, xd = slice(max(dx, 0), W + min(dx, 0)), slice(max(-dx, 0), W + min(-dx, 0))
    if ys.start < ys.stop and xs.start < xs.stop:
        out[..., yd, xd] = t[..., ys, xs]
    return out


def torch_atrous(x, normal, points, mask, features, passes, sigma_normal=128.0, sigma_plane=0.1, sigma_features=0.1):
    """The same filter in fp32 PyTorch ops: every tap's weight and shifted image materialised"""
    nh = normal / normal.norm(dim=1, keepdim=True).clamp_min(1e-12)
    valid = mask.float()
    y = torch.where(mask[:, None], x, 0.0)
    for k in range(passes):
        s = 2 ** k
        acc, wsum = 0.0, 0.0
        for oy in range(-2, 3):
            for ox in range(-2, 3):
                dy, dx = oy * s, ox * s
                if oy == 0 and ox == 0:
                    w = H5[2] * H5[2] * valid
                else:
                    d = _tap(points, dy, dx) - points
                    dn = d.norm(dim=1)
                    t = torch.where(dn > 0, (nh * d).sum(1).abs() / dn.clamp_min(1e-30), 0.0)
                    w = (H5[oy + 2] * H5[ox + 2] * (nh * _tap(nh, dy, dx)).sum(1).clamp(0, 1) ** sigma_normal *
                         torch.exp(-t / sigma_plane - ((_tap(features, dy, dx) - features) ** 2).sum(1) / sigma_features ** 2) *
                         _tap(valid, dy, dx) * valid)
                acc = acc + w[:, None] * _tap(y, dy, dx)
                wsum = wsum + w
        y = torch.where(mask[:, None], acc / torch.where(mask, wsum, 1.0)[:, None], 0.0)
    return y


def timed(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def floor_bytes(V, H, W, C, F, L):
    """HBM bytes the kernels cannot avoid: the pack reads the guides and mask once and writes the records; each
    forward pass reads its image and the records and writes its image and 1 / W; each backward pass reads its
    gradient, the records and 1 / W and writes its gradient."""
    npix, planes = V * H * W, 2 if F <= 1 else 2 + (F + 2) // 4
    pack = npix * (4 * (6 + F) + 1 + 16 * planes)
    fwd_pass = npix * (8 * C + 16 * planes + 4)
    bwd_pass = npix * (8 * C + 16 * planes + 4)
    return pack, fwd_pass, bwd_pass, pack + L * fwd_pass, L * bwd_pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_denoise needs a CUDA GPU")
    meta = dict(device=torch.cuda.get_device_properties(0).name)
    try:
        meta["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                             capture_output=True, text=True).stdout.strip()
    except OSError:
        meta["power_limit"] = "unknown"
    results, C, F = [], 3, 1
    for H, W in ((800, 800), (1200, 1600), (1080, 1920)):
        for V in (1, 4):
            g = gbuffer(V, H, W, F)
            cot = torch.randn_like(g["x"])
            for L in (3, 5):
                res = dict(V=V, H=H, W=W, C=C, F=F, L=L)
                guides = (g["normal"], g["points"], g["mask"], g["features"])
                with torch.no_grad():
                    res["cuda_fwd_ms"] = timed(lambda: atrous(g["x"], *guides, passes=L), args.iters)
                    res["torch_fwd_ms"] = timed(lambda: torch_atrous(g["x"], *guides, L), max(args.iters // 4, 3))
                    y_cuda, y_torch = atrous(g["x"], *guides, passes=L), torch_atrous(g["x"], *guides, L)
                    res["max_rel_diff"] = float(((y_cuda - y_torch).abs().max() / y_torch.abs().max()))
                x = g["x"].clone().requires_grad_()

                def fwd_bwd(fn):
                    def run():
                        x.grad = None
                        fn().backward(cot)
                    return run
                res["cuda_fwd_bwd_ms"] = timed(fwd_bwd(lambda: atrous(x, *guides, passes=L)), args.iters)
                res["torch_fwd_bwd_ms"] = timed(fwd_bwd(lambda: torch_atrous(x, *guides, L)), max(args.iters // 4, 3))
                pack, fwd_pass, bwd_pass, fwd, bwd = floor_bytes(V, H, W, C, F, L)
                res["floor_bytes_per_pass"] = fwd_pass
                res["floor_fwd_ms"] = fwd / HBM_BYTES_PER_S * 1e3
                res["floor_fwd_bwd_ms"] = (fwd + bwd) / HBM_BYTES_PER_S * 1e3
                res["speedup_fwd"] = res["torch_fwd_ms"] / res["cuda_fwd_ms"]
                res["speedup_fwd_bwd"] = res["torch_fwd_bwd_ms"] / res["cuda_fwd_bwd_ms"]
                results.append({k: (float(f"{v:.4g}") if isinstance(v, float) and math.isfinite(v) else v) for k, v in res.items()})
            del g, cot
            torch.cuda.empty_cache()
    line = dict(meta, cases=results, cuda_faster_everywhere=all(r["speedup_fwd"] > 1 and r["speedup_fwd_bwd"] > 1
                                                               for r in results))
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Time of TSDF fusion (relightable3dgaussian_b200.tsdf) against the vectorised PyTorch integration a user without
the module would write, and of marching-cubes extraction, on the shell scene.

  python tools/bench_tsdf.py [--sizes 512 1024] [--views 320] [--per-call 64] [--torch-views 4] [--rounds 2]

The shell-v1 scene (1M Gaussians, a unit-radius shell) is rendered once with rasterize_views at 800 x 800 for
`views` cameras (8 azimuths x views/8 elevations in [-60, 60] degrees); depth = out_depth / opacity, zeroed where
opacity < 0.5, and colour = the image.  Each round fuses all views into a fresh grid over [-1.2, 1.2]^3 with
sdf_trunc = 4 voxels in calls of `per-call` views (with and without colour), then runs the PyTorch integration of the
same definition on `torch-views` views (it walks the grid in slabs of 64 x N x N points to bound its temporaries), so
the two alternate in one process.  Extraction is timed on the fused volume.

Prints one JSON line: device name and power limit (read in the same run) and, per grid size and colour mode, the
median time per call and per view of each variant, and the effective HBM rate of the fused kernel with bytes from the
shapes: every grid point read once per call and written once (8 B, 20 B with colour; an upper bound on the writes)
plus the call's depth (and colour) maps, over the 3.35 TB/s data sheet."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from relightable3dgaussian_b200 import synth, tsdf  # noqa: E402
from relightable3dgaussian_b200 import rasterizer as R  # noqa: E402

HBM_BPS = 3.35e12                                        # H100 SXM data sheet (not reached; the floor uses it)
DEV = torch.device("cuda")
LO, HI = -1.2, 1.2


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [s.strip() for s in out.split(",")]
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        info["power_limit"] = f"unavailable ({e})"
    return info


def render(views, W=800, H=800, P=1_000_000, chunk=16):
    sc = synth.make_scene(P, "shell-v1", 0, 0)
    els = torch.linspace(-60.0, 60.0, views // 8).tolist()
    cams = [synth.make_camera(k, W, H, elevation_deg=e) for e in els for k in range(8)]
    settings = [R.GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, torch.zeros(3, device=DEV), 1.0,
                                                c.viewmatrix.to(DEV), c.projmatrix.to(DEV), 3, c.campos.to(DEV),
                                                False, True, True, False) for c in cams]
    d = lambda t: t.to(DEV)
    depth = torch.empty(len(cams), 1, H, W, device=DEV)
    color = torch.empty(len(cams), 3, H, W, device=DEV)
    with torch.no_grad():
        for s in range(0, len(cams), chunk):
            n = min(chunk, len(cams) - s)
            out = R.rasterize_views(d(sc.means3D), torch.zeros(n, P, 3, device=DEV), d(sc.opacities),
                                    settings=settings[s:s + n], shs=d(sc.shs), scales=d(sc.scales),
                                    rotations=d(sc.rotations))
            op = out[3]
            depth[s:s + n] = torch.where(op > 0.5, out[4] / op.clamp_min(1e-5), torch.zeros_like(op))
            color[s:s + n] = out[2].clamp(0, 1)
    return settings, depth, color


def torch_integrate(vol, depth, settings, color, slab=64):
    """The definition in PyTorch, one view at a time over slabs of the grid (in place on vol's tensors)."""
    NX, NY, NZ = vol.dims
    vs, st = vol.voxel_size, vol.sdf_trunc
    o = torch.tensor(vol.origin, device=DEV)
    jj, kk = torch.meshgrid(torch.arange(NY, device=DEV), torch.arange(NZ, device=DEV), indexing="ij")
    for v, s in enumerate(settings):
        H, W = s.image_height, s.image_width
        fx, fy = W / (2 * s.tanfovx), H / (2 * s.tanfovy)
        M = s.viewmatrix.float()
        dv = depth[v, 0].reshape(-1)
        for i0 in range(0, NX, slab):
            i1 = min(NX, i0 + slab)
            ii = torch.arange(i0, i1, device=DEV).view(-1, 1, 1).expand(-1, NY, NZ)
            pts = torch.stack([o[0] + vs * ii, o[1] + vs * jj.expand_as(ii), o[2] + vs * kk.expand_as(ii)], -1)
            p = pts @ M[:3, :3] + M[3, :3]
            Z = p[..., 2]
            u = torch.floor(fx * p[..., 0] / Z + s.cx + 0.5)
            w_ = torch.floor(fy * p[..., 1] / Z + s.cy + 0.5)
            ok = (Z > 0) & (u >= 0) & (u < W) & (w_ >= 0) & (w_ < H)
            pix = torch.where(ok, w_ * W + u, torch.zeros_like(u)).long()
            D = dv[pix]
            sdf = D - Z
            ok &= torch.isfinite(D) & (D > 0) & (sdf >= -st)
            obs = torch.clamp(sdf / st, max=1.0)
            t, w = vol.tsdf[i0:i1], vol.weight[i0:i1]
            w1 = w + 1
            t.copy_(torch.where(ok, (t * w + obs) / w1, t))
            if color is not None:
                rgb = color[v].reshape(3, -1)[:, pix].permute(1, 2, 3, 0)
                c = vol.color[i0:i1]
                c.copy_(torch.where(ok[..., None], (c * w[..., None] + rgb) / w1[..., None], c))
            w.copy_(torch.where(ok, w1, w))


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--views", type=int, default=320)
    ap.add_argument("--per-call", type=int, default=64)
    ap.add_argument("--torch-views", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    info = device_info()
    settings, depth, color = render(args.views)
    V, _, H, W = depth.shape
    res = {"bench": "tsdf", **info, "views": V, "per_call": args.per_call, "image": [H, W], "results": []}
    for n in args.sizes:
        vs = (HI - LO) / (n - 1)
        for use_color in (False, True):
            vol_bytes = 20 if use_color else 8
            calls, views_ms, torch_ms, ex_ms = [], [], [], []
            vol = None
            for _ in range(args.rounds + 1):                 # the first round warms up
                vol = None
                torch.cuda.empty_cache()
                vol = tsdf.TSDFVolume((LO,) * 3, (HI,) * 3, vs, 4 * vs, color=use_color, device=DEV)
                assert vol.dims == (n, n, n)
                ms = []
                for s in range(0, V, args.per_call):
                    e = min(V, s + args.per_call)
                    t, _ = timed(lambda: vol.integrate(depth[s:e], settings[s:e], color[s:e] if use_color else None))
                    ms.append(t)
                calls.append(statistics.median(ms))
                views_ms.append(sum(ms) / V)
                t, mesh = timed(vol.extract)
                ex_ms.append(t)
                nv, nf = mesh[0].shape[0], mesh[1].shape[0]
                del mesh
                tv = tsdf.TSDFVolume((LO,) * 3, (HI,) * 3, vs, 4 * vs, color=use_color, device=DEV)
                k = args.torch_views
                t, _ = timed(lambda: torch_integrate(tv, depth[:k], settings[:k], color[:k] if use_color else None))
                torch_ms.append(t / k)
                del tv
            N = n ** 3
            pc = args.per_call
            call_bytes = 2 * N * vol_bytes + pc * H * W * 4 * (4 if use_color else 1)
            call_ms = statistics.median(calls[1:])
            res["results"].append({
                "grid": n, "color": use_color, "points": N,
                "fused_ms_per_call": round(call_ms, 3), "fused_ms_per_view": round(statistics.median(views_ms[1:]), 4),
                "torch_ms_per_view": round(statistics.median(torch_ms[1:]), 3),
                "speedup_per_view": round(statistics.median(torch_ms[1:]) / statistics.median(views_ms[1:]), 1),
                "call_bytes": call_bytes, "effective_TBps": round(call_bytes / (call_ms * 1e-3) / 1e12, 3),
                "hbm_floor_ms_per_call": round(call_bytes / HBM_BPS * 1e3, 3),
                "extract_ms": round(statistics.median(ex_ms[1:]), 2), "mesh_vertices": nv, "mesh_faces": nf,
                "observed_points": int((vol.weight > 0).sum())})
            del vol
            print(json.dumps(res["results"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

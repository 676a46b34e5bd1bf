"""Cost of the full rasterizer backward against the appearance-only backward a frozen-geometry step takes.

1. Rasterizer forward + backward at the headline configuration (1M Gaussians, 800x800, S=5) and at the stage-2 shape
   (1.5M, 1600x1200, S=16): the full backward (what a step whose geometry requires grad runs) against the
   appearance-only backward with only dL/dfeatures requested (the stage-2 case: every geometry leaf and the SH
   coefficients frozen), and with dL/dfeatures and the dense dL/dsh requested (SH learnt under frozen geometry).  Each
   timing is CUDA events around `iters` fwd+bwd pairs; the arms alternate round by round and the median over `rounds`
   is reported, with the composite_bwd and project_bwd stage times of the library's stage profiler in a separate run.
2. The stage-2 step of bench_stage2.py (its model, cameras, shading, fused feature pack, rasterizer, unpremultiply,
   L1 loss and FusedAdam step, 1.5M Gaussians at 1600x1200, S=16, N=32) with the geometry leaves requiring grad at
   learning rate 0 (the reference's stage 2) against the same step with them frozen (requires_grad off, means2D
   without grad).

Prints one JSON line that starts with the device name and power limit read in the same run.

    python tools/bench_frozen_geometry.py [--rounds 5] [--iters 10] [--step-iters 10]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_views import device_info, stage_times, timed  # noqa: E402
from relightable3dgaussian_b200 import _C_raster, synth  # noqa: E402


def raster_step(P, W, H, S, geometry, sh=False):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    cam = synth.make_camera(1, W, H)
    d = lambda t: t.cuda().contiguous()
    means, feats, opac, scales, rots, shs = (d(t) for t in (sc.means3D, sc.features, sc.opacities, sc.scales,
                                                            sc.rotations, sc.shs))
    bg, view, proj, campos = d(torch.tensor([0.0, 0.5, 1.0])), d(cam.viewmatrix), d(cam.projmatrix), d(cam.campos)
    gen = torch.Generator(device="cuda").manual_seed(1)
    cots = [torch.randn(c, H, W, device="cuda", generator=gen) for c in (3, 1, 1, S)]
    empty = torch.empty(0, device="cuda")
    kw = {} if geometry else dict(geometry=False, appearance=(True, False, sh))

    def run():
        o = _C_raster.rasterize_gaussians(bg, means, feats, empty, opac, scales, rots, 1.0, empty, view, proj,
                                          cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, H, W, shs, 3, campos, False, True,
                                          False)
        _C_raster.rasterize_gaussians_backward(bg, means, feats, o[9], empty, scales, rots, 1.0, empty, view, proj,
                                               cam.tanfovx, cam.tanfovy, *cots, shs, 3, campos, o[10], o[0], o[11],
                                               o[12], True, False, **kw)
    return run


def stage2_arms():
    """The two stage-2 step functions over one model (bench_stage2.py's), and the learnt leaves."""
    import bench_stage2 as b2
    from relightable3dgaussian_b200 import raytracer, shading
    from relightable3dgaussian_b200.optim import FusedAdam
    from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, pack_features,
                                                        unpremultiply)
    dev = torch.device("cuda")
    cfg = b2.CONFIG4
    P, W, H, N = cfg["P"], cfg["W"], cfg["H"], cfg["N"]
    m, lrs = b2.make_model(cfg, dev)
    cams, camd = b2.make_cameras(cfg, dev)
    g = torch.Generator().manual_seed(11)
    gts = [torch.rand(3, H, W, generator=g).to(dev) for _ in cams]
    bg = torch.zeros(3, device=dev)
    with torch.no_grad():
        a = b2.activated(m)
        icov = raytracer.inverse_covariance(a["scaling"], a["rotation"])
        vis, dirs, areas = raytracer.update_visibility(a["xyz"], a["scaling"], a["rotation"], icov,
                                                       a["opacity"][:, 0].contiguous(), a["normal"], N)
        vis_mean = vis.mean(-2)
    learnt = [k for k, lr in lrs.items() if lr > 0]
    frozen_m = {k: (t if k in learnt else t.detach()) for k, t in m.items()}

    def make(model, names, means2d_grad):
        light = b2.Light(model["env"])
        opt = FusedAdam([{"params": [model[k]], "lr": lrs[k], "name": k} for k in names], lr=0.0, eps=1e-15)
        it = [0]

        def step():
            v = it[0] % len(cams)
            it[0] += 1
            c, cd = cams[v], camd[v]
            base_color, roughness, nrm, viewdirs, incidents = b2._shade_inputs(model, cd)
            brdf, extra = shading.rendering_equation(base_color, roughness, nrm.detach(), viewdirs, incidents, light,
                                                     visibility_precompute=vis, incident_dirs_precompute=dirs,
                                                     incident_areas_precompute=areas)
            feats = b2.neilf_features(model, cd, brdf, extra, vis_mean, pack=pack_features)
            rs = GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, bg, 1.0, cd["view"], cd["proj"], 3,
                                               cd["pos"], False, True, True, False)
            act = b2.activated(model)
            means2D = torch.zeros(P, 3, device=dev, requires_grad=means2d_grad)
            out = GaussianRasterizer(rs)(means3D=act["xyz"], means2D=means2D, opacities=act["opacity"],
                                         shs=torch.cat([model["f_dc"], model["f_rest"]], dim=1), scales=act["scaling"],
                                         rotations=act["rotation"], features=feats)
            loss = b2.loss_fn(out[2], out[5], out[3], out[1], gts[v], bg, unpremultiply)
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
        return step

    return {"full": make(m, list(lrs), True), "frozen": make(frozen_m, learnt, False)}, P, W, H


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--step-iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frozen_geometry.py needs a CUDA GPU")
    res = device_info()
    configs = {"1M_800x800_S5": (1_000_000, 800, 800, 5), "1.5M_1600x1200_S16": (1_500_000, 1600, 1200, 16)}
    for name, (P, W, H, S) in configs.items():
        arms = {"full": raster_step(P, W, H, S, True), "appearance": raster_step(P, W, H, S, False),
                "appearance_sh": raster_step(P, W, H, S, False, sh=True)}
        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, run in arms.items():
                ms[k].append(timed(run, args.iters))
        st = {k: stage_times(run, args.iters, 1) for k, run in arms.items()}
        a, b = statistics.median(ms["full"]), statistics.median(ms["appearance"])
        c = statistics.median(ms["appearance_sh"])
        res[name] = {"fwd_bwd_full_ms": round(a, 3), "fwd_bwd_appearance_ms": round(b, 3), "speedup": round(a / b, 4),
                     "fwd_bwd_appearance_sh_ms": round(c, 3), "speedup_sh": round(a / c, 4),
                     "spread_ms": {k: round(max(v) - min(v), 3) for k, v in ms.items()},
                     "composite_bwd_ms": {k: s["composite_bwd"] for k, s in st.items()},
                     "project_bwd_ms": {k: s["project_bwd"] for k, s in st.items()}}
        del arms
        torch.cuda.empty_cache()
    arms, P, W, H = stage2_arms()
    ms = {k: [] for k in arms}
    for run in arms.values():          # warm-up: the first forwards of a shape learn its instance counts
        for _ in range(10):
            run()
    for _ in range(args.rounds):
        for k, run in arms.items():
            ms[k].append(timed(run, args.step_iters))
    st = {k: stage_times(run, args.step_iters, 1) for k, run in arms.items()}
    a, b = statistics.median(ms["full"]), statistics.median(ms["frozen"])
    res[f"stage2_step_{P // 1000}k_{W}x{H}_S16"] = {
        "step_full_ms": round(a, 3), "step_frozen_ms": round(b, 3), "speedup": round(a / b, 4),
        "spread_ms": {k: round(max(v) - min(v), 3) for k, v in ms.items()},
        "composite_bwd_ms": {k: s["composite_bwd"] for k, s in st.items()},
        "project_bwd_ms": {k: s["project_bwd"] for k, s in st.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""bench.py --workload stage2: the reference's stage-2 ("neilf") TRAINING STEP at the BASELINE.json
configs #4 (DTU shape: 1.5M Gaussians, 1600x1200, 1 GPU) and #5 (TnT shape: 2M, 1920x1080, one view
per GPU on N GPUs), assembled exactly like the reference assembles it:

    gaussian_renderer/neilf.py:87-147    activations -> rendering_equation (BRDF shading with the baked
                                         BVH visibility) -> 16-channel feature pack -> GaussianRasterizer
                                         (S = 16) -> un-premultiply -> pbr composite
    train.py:115-127                     loss -> backward
    scene/gaussian_model.py:465-497      Adam over the 12 per-Gaussian groups + the environment map
                                         (script/run_dtu.sh:27-46: geometry learning rates are 0)
    scene/gaussian_model.py:312-342      the one-off visibility bake (LBVH build + N rays per Gaussian),
                                         run once before the loop and reported beside the step

Two arms over the SAME seeded model, cameras and targets:
  * ours       — fused shading kernels, this project's rasterizer through the GaussianRasterizer mirror (deferred
                 count), FusedAdam, LBVH bake with in-kernel direction sampling;
  * reference  — the reference's PyTorch rendering_equation formulation (oracle/oracle_shading.py, pinned
                 to the reference's own function bodies), its own rasterizer (stock wrapper + pybind module
                 from oracle/_ref/ext when built, else the raw-pointer shim over the same kernels),
                 torch.optim.Adam, its own BVH kernels for the bake.
The loss is a plain L1 on the radiance and PBR images plus a light regulariser on both arms (the
reference's SSIM / smoothness terms are host PyTorch outside the hot path, SURVEY.md §2).
"""
import ctypes
import gc
import json
import os
import statistics
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))

CONFIG4 = dict(P=1_500_000, W=1600, H=1200, N=32, views=8, recipe="shell-v1", seed=0)      # DTU_scan24 shape
CONFIG5 = dict(P=2_000_000, W=1920, H=1080, N=32, views=8, recipe="shell-v1", seed=0)      # TnT-Barn shape
S2 = 16                                                                                     # neilf.py:115-118
RASTER_STAGES = ["project", "depth_sort", "bin_count", "bin_offsets", "bin_scatter", "composite_fwd",
                 "surface_normal", "composite_bwd", "project_bwd"]


class Light:                     # duck-types scene/direct_light_map.py:DirectLightMap (get_env = softplus(env))
    def __init__(self, env_raw):
        self.env = env_raw

    @property
    def get_env(self):
        return F.softplus(self.env)


def make_model(cfg, dev):
    """Seeded raw (pre-activation) parameters, activations as in scene/gaussian_model.py:76-110."""
    from relightable3dgaussian_b200 import synth
    P = cfg["P"]
    sc = synth.make_scene(P, cfg["recipe"], cfg["seed"], 0)
    g = torch.Generator().manual_seed(7)
    leaf = lambda t: t.to(dev).contiguous().requires_grad_(True)
    m = dict(
        xyz=leaf(sc.means3D), normal=leaf(sc.normals), rotation=leaf(sc.rotations), scaling=leaf(sc.scales.log()),
        opacity=leaf(torch.logit(sc.opacities.clamp(1e-4, 1 - 1e-4))),
        f_dc=leaf(sc.shs[:, :1]), f_rest=leaf(sc.shs[:, 1:]),
        base_color=leaf(torch.randn(P, 3, generator=g)), roughness=leaf(torch.randn(P, 1, generator=g)),
        incidents_dc=leaf(torch.randn(P, 1, 3, generator=g) * 0.3), incidents_rest=leaf(torch.randn(P, 15, 3, generator=g) * 0.1),
        env=leaf(torch.randn(1, 16, 32, 3, generator=g)))
    # learning rates: arguments/__init__.py defaults with script/run_dtu.sh:27-46 overrides (frozen geometry)
    lrs = dict(xyz=0.0, normal=0.0, rotation=0.0, scaling=0.0, opacity=0.0, f_dc=0.0, f_rest=0.0, base_color=0.01,
               roughness=0.01, incidents_dc=0.0025, incidents_rest=0.000125, env=0.1)
    return m, lrs


def activated(m):
    return dict(xyz=m["xyz"], scaling=torch.exp(m["scaling"]), rotation=F.normalize(m["rotation"]),
                opacity=torch.sigmoid(m["opacity"]), normal=F.normalize(m["normal"], dim=-1))


def make_cameras(cfg, dev):
    from relightable3dgaussian_b200 import synth
    cams = [synth.make_camera(k, cfg["W"], cfg["H"]) for k in range(cfg["views"])]
    camd = [dict(view=c.viewmatrix.to(dev), proj=c.projmatrix.to(dev), pos=c.campos.to(dev), c=c) for c in cams]
    return cams, camd


def neilf_features(m, cd, brdf, extra, vis_mean, pack=None):
    """neilf.py:110-118 (training branch): depth, depth^2, brdf, normal, base_color, roughness, diffuse, visibility.
    `pack`: the optional fused operator (rasterizer.pack_features, SURVEY.md §8(f)2) instead of the PyTorch expression."""
    xyz = m["xyz"]
    if pack is not None:
        base_color = torch.sigmoid(m["base_color"]) * 0.77 + 0.03
        roughness = torch.sigmoid(m["roughness"]) * 0.9 + 0.09
        nrm = F.normalize(m["normal"], dim=-1)
        return pack([brdf, nrm, base_color, roughness, extra["diffuse_light"], vis_mean], means3D=xyz, viewmatrix=cd["view"])
    depths = (torch.cat([xyz, torch.ones_like(xyz[:, :1])], dim=-1) @ cd["view"])[:, 2:3]
    base_color = torch.sigmoid(m["base_color"]) * 0.77 + 0.03          # gaussian_model.py base_color_activation
    roughness = torch.sigmoid(m["roughness"]) * 0.9 + 0.09
    nrm = F.normalize(m["normal"], dim=-1)
    return torch.cat([depths, depths.square(), brdf, nrm, base_color, roughness, extra["diffuse_light"], vis_mean], dim=-1)


def loss_fn(color, feature, opacity, num_contrib, gt, bg, unpremultiply):
    feature = unpremultiply(feature, opacity, num_contrib)            # neilf.py:136-137
    pbr = feature[2:5] * opacity + (1 - opacity) * bg[:, None, None]  # neilf.py:167-168
    return (color - gt).abs().mean() + (pbr - gt).abs().mean() + 0.01 * feature[12:15].mean()


def _shade_inputs(m, cd):
    base_color = torch.sigmoid(m["base_color"]) * 0.77 + 0.03
    roughness = torch.sigmoid(m["roughness"]) * 0.9 + 0.09
    incidents = torch.cat([m["incidents_dc"], m["incidents_rest"]], dim=1)
    viewdirs = F.normalize(cd["pos"] - m["xyz"], dim=-1)
    nrm = F.normalize(m["normal"], dim=-1)
    return base_color, roughness, nrm, viewdirs, incidents


def _median_ms(events):
    return statistics.median(a.elapsed_time(b) for a, b in events)


def run_ours(args, cfg, rank, local, world):
    from relightable3dgaussian_b200 import _lib, dist as rdist, raytracer, shading
    from relightable3dgaussian_b200.optim import FusedAdam
    from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, pack_features, set_deferred_count,
                                                        unpremultiply, set_grad_exchange)
    from bench import ClockSampler, alg_bytes, measured_peak
    import torch.distributed as tdist
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    lib = _lib.load()
    P, W, H, N = cfg["P"], cfg["W"], cfg["H"], cfg["N"]
    m, lrs = make_model(cfg, dev)
    cams, camd = make_cameras(cfg, dev)
    g = torch.Generator().manual_seed(11)
    gts_host = [torch.rand(3, H, W, generator=g).pin_memory() for _ in cams]
    bg = torch.zeros(3, device=dev)
    light = Light(m["env"])
    opt = FusedAdam([{"params": [m[k]], "lr": lr, "name": k} for k, lr in lrs.items()], lr=0.0, eps=1e-15)

    # ---- one-off visibility bake (gaussian_model.py:312-342), sharded over the ranks when world > 1 ----
    with torch.no_grad():
        a = activated(m)
        icov = raytracer.inverse_covariance(a["scaling"], a["rotation"])
        # untimed warm-up on a small prefix: CUDA module loading / first-launch setup is not part of the bake
        raytracer.update_visibility(a["xyz"][:2048], a["scaling"][:2048], a["rotation"][:2048], icov[:2048], a["opacity"][:2048, 0].contiguous(),
                                    a["normal"][:2048], N, shard_group=True if world > 1 else None)
        torch.cuda.synchronize(dev)
        t0 = time.time()
        vis, dirs, areas = raytracer.update_visibility(a["xyz"], a["scaling"], a["rotation"], icov, a["opacity"][:, 0].contiguous(),
                                                       a["normal"], N, shard_group=True if world > 1 else None)
        torch.cuda.synchronize(dev)
        bake_s = time.time() - t0
        vis_mean = vis.mean(-2)
        blocked = float((vis == 0).float().mean())

    # ---- multi-GPU: SH factor inside backward, everything else averaged at the leaves ---------------
    exchange = bucket = None
    exchange_kind = None
    if world > 1:
        leaves = [m[k] for k in m if k not in ("f_dc", "f_rest")]
        if args.exchange in ("p2p", "auto"):
            try:                                             # one-kernel NVLink exchange (symmetric memory + NVLS)
                exchange = rdist.P2PGradExchange(P, S2, 16, dev)
                bucket = rdist.LeafGradBucket(leaves, dev, symmetric=True)
                exchange_kind = "p2p"
            except Exception as e:
                if args.exchange == "p2p":
                    raise
                print(f"[bench] P2P exchange unavailable ({type(e).__name__}: {e}); using NCCL", file=sys.stderr)
                exchange = bucket = None
        if exchange is None:
            exchange = rdist.FactoredGradExchange(P, S2, 16, dev)
            bucket = rdist.LeafGradBucket(leaves, dev)
            exchange_kind = "factored"
    gt_dev = [torch.empty(3, H, W, device=dev) for _ in range(2)]
    loss_host = torch.zeros(64).pin_memory()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    marks = []

    def step(i, record=False):
        v = rdist.view_for_rank(i, rank, world, cfg["views"])
        c, cd = cams[v], camd[v]
        e = [ev() for _ in range(6)] if record else None
        mark = (lambda k: e[k].record()) if record else (lambda k: None)
        mark(0)
        gt = gt_dev[i % 2]
        gt.copy_(gts_host[v], non_blocking=True)                          # per-step H2D of the target image
        if bucket is not None:
            bucket.zero()
        base_color, roughness, nrm, viewdirs, incidents = _shade_inputs(m, cd)
        brdf, extra = shading.rendering_equation(base_color, roughness, nrm.detach(), viewdirs, incidents, light,
                                                 visibility_precompute=vis, incident_dirs_precompute=dirs, incident_areas_precompute=areas)
        mark(1)
        feats = neilf_features(m, cd, brdf, extra, vis_mean, pack=pack_features)
        rs = GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, bg, 1.0, cd["view"], cd["proj"], 3, cd["pos"],
                                           False, True, True, False)
        a = activated(m)
        means2D = torch.zeros_like(m["xyz"], requires_grad=True)
        out = GaussianRasterizer(rs)(means3D=a["xyz"], means2D=means2D, opacities=a["opacity"], shs=torch.cat([m["f_dc"], m["f_rest"]], dim=1),
                                     scales=a["scaling"], rotations=a["rotation"], features=feats)
        mark(2)
        loss = loss_fn(out[2], out[5], out[3], out[1], gt, bg, unpremultiply)
        mark(3)
        if exchange is not None:
            campos_all = torch.stack([camd[rdist.view_for_rank(i, r, world, cfg["views"])]["pos"] for r in range(world)]).contiguous()
            set_grad_exchange(exchange, campos_all)
        loss.backward()
        if bucket is not None:
            bucket.allreduce_mean()
        mark(4)
        opt.step()
        opt.zero_grad(set_to_none=bucket is None)
        loss_host[i % 64:i % 64 + 1].copy_(loss.detach().reshape(1), non_blocking=True)   # per-step D2H of the loss
        mark(5)
        if record:
            marks.append(e)
        return out

    set_deferred_count(True)
    warm = max(args.warmup, 10)          # the first _LEARN forwards of a shape take the synchronous count path
    for i in range(warm):
        step(i)
    gc.collect()
    gc.disable()              # as timeit does (both arms); before the barrier so that the ranks enter the region together
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
    lib.r3dg_prof_begin(args.steps)
    torch.cuda.synchronize(dev)
    if world > 1:
        tdist.barrier()
    torch.cuda.synchronize(dev)
    l0 = lib.r3dg_launch_count()
    e0, e1 = ev(), ev()
    e0.record()
    for i in range(args.steps):
        out = step(warm + i, record=True)
    e1.record()
    gc.enable()
    torch.cuda.synchronize(dev)
    if world > 1:
        tdist.barrier()
    torch.cuda.synchronize(dev)
    clocks = sampler.stop() if sampler else None
    ms = e0.elapsed_time(e1)
    arr = (ctypes.c_float * 9)(); nf = ctypes.c_int(); nb = ctypes.c_int()
    lib.r3dg_prof_end(arr, ctypes.byref(nf), ctypes.byref(nb))
    stage = {n: arr[k] / max(nf.value if k < 7 else nb.value, 1) for k, n in enumerate(RASTER_STAGES)}
    launches = lib.r3dg_launch_count() - l0
    set_deferred_count(False)
    set_grad_exchange(None)
    if world > 1:
        t = torch.tensor([ms], device=dev)
        tdist.all_reduce(t, op=tdist.ReduceOp.MAX)
        ms = float(t.item())
    phases = {name: _median_ms([(mk[k], mk[k + 1]) for mk in marks]) for k, name in
              enumerate(["h2d_shading_fwd", "pack_raster_fwd", "unpremultiply_loss", "backward_exchange", "adam_d2h"])}
    # start-to-start intervals of consecutive steps: a host hiccup (allocator, GC) shows up as an outlier here, not in the phases
    gaps = sorted(marks[k][0].elapsed_time(marks[k + 1][0]) for k in range(len(marks) - 1))
    step_stats = {"median": gaps[len(gaps) // 2], "min": gaps[0], "max": gaps[-1]} if gaps else None
    if rank != 0:
        return None
    R = int(out[0]); Pv = int((out[9] > 0).sum().item())
    T = ((W + 15) // 16) * ((H + 15) // 16)
    ab = alg_bytes(P, Pv, R, H * W, T, S2)
    ab["shading_fwd"] = P * N * 20 + P * (3 + 1 + 3 + 3 + 48 + 9) * 4          # baked tensors once + per-Gaussian operands/results
    ab["shading_bwd"] = P * N * 20 + P * (3 + 1 + 3 + 3 + 48 + 9 + 3 + 1 + 3 + 48) * 4
    dom = max(stage, key=lambda k: stage[k])
    peak, peak_src = measured_peak()
    achieved = ab[dom] / (stage[dom] * 1e-3) / 1e9
    value = world * args.steps / (ms / 1e3)
    h2d = 3 * H * W * 4
    return {
        "workload": "stage2",
        "metric": f"stage-2 (neilf) training steps/sec, {P} Gaussians {W}x{H}, render_equation N={N} + BVH-baked visibility, S=16 raster fwd+bwd, Adam",
        "value": value, "unit": "views/s", "n_gpus": world, "steps": args.steps, "warmup": warm, "ms_per_step": ms / args.steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"stage-2 neilf training step (BASELINE config #{'5' if world > 1 else '4'} shape): shading N={N} -> 16-channel pack -> raster fwd -> "
                               f"un-premultiply + L1 -> backward -> FusedAdam (optional fused operators used: pack_features, unpremultiply, FusedAdam); {cfg['recipe']} seed {cfg['seed']}, P={P}, {W}x{H}, {cfg['views']}-camera ring",
                   "P": P, "W": W, "H": H, "S": S2, "N": N, "num_rendered": R, "P_visible": Pv,
                   "parallelism": "single GPU" if world == 1 else (
                       f"view-parallel x{world} ({exchange_kind}): SH gradient rebuilt inside backward from the ranks' factors "
                       f"({'P2P loads over NVLink' if exchange_kind == 'p2p' else 'NCCL all-gather'}), all other leaf gradients averaged in one "
                       f"{bucket.bytes() / 1e6:.0f} MB {'NVLS multimem kernel' if exchange_kind == 'p2p' else 'NCCL all-reduce'} after backward; bake sharded over ranks"),
                   "l2": "inputs larger than L2 (P x N x 20 B baked tensors + 236 B/Gaussian parameters vs 126 MB)"},
        "e2e": {"value": value, "unit": "views/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
                "what": "the step IS the public-API path (rendering_equation + GaussianRasterizer mirrors + autograd + FusedAdam); the per-step H2D of the "
                        "target image from pinned memory and the D2H of the loss are inside the timed region"},
        "gpu_launches": int(launches), "clocks": clocks,
        "phase_ms_median": phases, "step_interval_ms": step_stats, "raster_stage_ms": stage,
        "bake": {"seconds": bake_s, "rays": P * N, "mrays_per_s": P * N / bake_s / 1e6, "blocked_fraction": blocked,
                 "what": "LBVH build + in-kernel Fibonacci direction sampling + opacity trace, once before the loop (not in ms_per_step)"},
        "roofline": {"bound": "hbm", "kernel": dom, "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                     "traffic": None, "peak_source": peak_src, "alg_bytes_per_launch": ab[dom],
                     "per_kernel": {k: {"ms": stage[k], "alg_GBps": ab[k] / (stage[k] * 1e-3) / 1e9 if stage[k] > 0 else None} for k in stage}},
        "peak_mem_GB": torch.cuda.max_memory_allocated(dev) / 1e9,
    }


def run_reference(args, cfg, rank, local, world):
    """The reference's formulation of the same step on one GPU (rank 0 only)."""
    if rank != 0:
        return None
    from oracle import oracle_sampling, oracle_shading as osh, ref_gpu
    from bench import ClockSampler
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    P, W, H, N = cfg["P"], cfg["W"], cfg["H"], cfg["N"]
    m, lrs = make_model(cfg, dev)
    cams, camd = make_cameras(cfg, dev)
    g = torch.Generator().manual_seed(11)
    gts_host = [torch.rand(3, H, W, generator=g).pin_memory() for _ in cams]
    bg = torch.zeros(3, device=dev)
    opt = torch.optim.Adam([{"params": [m[k]], "lr": lr, "name": k} for k, lr in lrs.items()], lr=0.0, eps=1e-15)
    raster, raster_kind = ref_gpu.reference_rasterizer()        # stock wrapper + pybind module when built, else the shim

    # bake with the reference's own BVH kernels, driven like gaussian_model.py:312-342
    with torch.no_grad():
        a = activated(m)
        icov = oracle_sampling.inverse_covariance(a["scaling"], a["rotation"])
        ref_gpu.reference_update_visibility(a["xyz"][:2048], a["scaling"][:2048], a["rotation"][:2048], icov[:2048], a["opacity"][:2048, 0].contiguous(),
                                            a["normal"][:2048], N)                      # untimed warm-up (module loading)
        torch.cuda.synchronize()
        t0 = time.time()
        vis, dirs, areas, bake_kind = ref_gpu.reference_update_visibility(a["xyz"], a["scaling"], a["rotation"], icov,
                                                                          a["opacity"][:, 0].contiguous(), a["normal"], N)
        torch.cuda.synchronize()
        bake_s = time.time() - t0
        vis_mean = vis.mean(-2)
    gt_dev = [torch.empty(3, H, W, device=dev) for _ in range(2)]
    loss_host = torch.zeros(64).pin_memory()
    unpre = lambda f, o, n: f / o.clamp_min(1e-5) * (n > 0)       # neilf.py:136-137
    ev = lambda: torch.cuda.Event(enable_timing=True)
    marks = []

    def step(i, record=False):
        v = i % cfg["views"]
        c, cd = cams[v], camd[v]
        e = [ev() for _ in range(6)] if record else None
        mark = (lambda k: e[k].record()) if record else (lambda k: None)
        mark(0)
        gt = gt_dev[i % 2]
        gt.copy_(gts_host[v], non_blocking=True)
        base_color, roughness, nrm, viewdirs, incidents = _shade_inputs(m, cd)
        brdf, extra = osh.rendering_equation(base_color, roughness, nrm.detach(), viewdirs, incidents, F.softplus(m["env"])[0], vis, dirs, areas)
        mark(1)
        feats = neilf_features(m, cd, brdf, extra, vis_mean)
        a = activated(m)
        out = raster(c, cd, bg, a["xyz"], a["opacity"], torch.cat([m["f_dc"], m["f_rest"]], dim=1), a["scaling"], a["rotation"], feats)
        mark(2)
        loss = loss_fn(out["color"], out["feature"], out["opacity"], out["num_contrib"], gt, bg, unpre)
        mark(3)
        loss.backward()
        mark(4)
        opt.step()
        opt.zero_grad()
        loss_host[i % 64:i % 64 + 1].copy_(loss.detach().reshape(1), non_blocking=True)
        mark(5)
        if record:
            marks.append(e)
        return out

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    sampler = ClockSampler(local); sampler.start()
    e0, e1 = ev(), ev()
    gc.collect()
    gc.disable()
    e0.record()
    for i in range(args.steps):
        out = step(args.warmup + i, record=True)
    e1.record()
    gc.enable()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    ms = e0.elapsed_time(e1)
    v = args.steps / (ms / 1e3)
    phases = {name: _median_ms([(mk[k], mk[k + 1]) for mk in marks]) for k, name in
              enumerate(["h2d_shading_fwd", "pack_raster_fwd", "unpremultiply_loss", "backward_exchange", "adam_d2h"])}
    return {"impl": "reference", "workload": "stage2",
            "metric": f"stage-2 (neilf) training steps/sec, {P} Gaussians {W}x{H}, render_equation N={N} + BVH-baked visibility, S=16 raster fwd+bwd, Adam",
            "value": v, "unit": "views/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "clocks": clocks,
            "config": {"workload": f"reference formulation of the stage-2 step: PyTorch rendering_equation (neilf.py:339-406 restated, pinned) + {raster_kind} + torch.optim.Adam; "
                                   f"same model / cameras / targets, P={P}, {W}x{H}, N={N}", "num_rendered": int(out["num_rendered"])},
            "phase_ms_median": phases,
            "bake": {"seconds": bake_s, "rays": P * N, "mrays_per_s": P * N / bake_s / 1e6, "what": bake_kind},
            "cpu_baseline": {"value": v, "unit": "views/s", "cores": os.cpu_count(), "kind": "reference",
                             "sample": "not a CPU run: the reference has no CPU path for this step; its own CUDA kernels + PyTorch on the same GPU"},
            "e2e": {"value": v, "unit": "views/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "peak_mem_GB": torch.cuda.max_memory_allocated(dev) / 1e9}

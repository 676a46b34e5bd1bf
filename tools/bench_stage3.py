#!/usr/bin/env python3
"""Stage-3 measurements on one H100 (development / evidence, not the headline bench):
  * BVH build + visibility bake (update_visibility) vs the unmodified reference kernels
    (oracle/_ref/libref_bvh.so driven like bvh/__init__.py + scene/gaussian_model.py:312-342);
  * fused rendering_equation fwd+bwd vs the reference's PyTorch formulation (oracle_shading on GPU).
Prints one JSON line per measurement."""
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import shading_case  # noqa: E402
from relightable3dgaussian_b200 import raytracer, shading, synth  # noqa: E402
from oracle import oracle_shading as osh, ref_gpu  # noqa: E402


def timeit(fn, n=3, warm=1):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def bvh(P, N, recipe="shell-v1", ref=True):
    """LBVH build + the visibility bake (one launch, in-kernel direction sampling) vs the reference's own kernels driven
    like scene/gaussian_model.py:312-342.  `cube-v1` (random normals inside a cube) exercises the T < 0.9 early exit;
    `shell-v1` (outward normals on a sphere) never blocks, every ray walks the tree to the end."""
    sc = synth.make_scene(P, recipe, 0, 0)
    d = lambda t: t.cuda()
    xyz, s, r, op, nrm = d(sc.means3D), d(sc.scales), d(sc.rotations), d(sc.opacities[:, 0].contiguous()), d(sc.normals)
    icov = raytracer.inverse_covariance(s, r)
    t_build = timeit(lambda: raytracer.RayTracer(xyz, s, r))
    rt = raytracer.RayTracer(xyz, s, r)
    t_trace = timeit(lambda: rt.bake_visibility(xyz, icov, op, nrm, N), n=3)
    t_bake = timeit(lambda: raytracer.update_visibility(xyz, s, r, icov, op, nrm, N), n=2)
    vis_o = raytracer.update_visibility(xyz, s, r, icov, op, nrm, N)[0]
    out = dict(what="bvh", recipe=recipe, P=P, N=N, rays=P * N, ours_build_ms=t_build, ours_trace_ms=t_trace, ours_bake_ms=t_bake,
               ours_Mrays_per_s=P * N / t_trace / 1e3, blocked_fraction=float((vis_o == 0).float().mean()))
    if ref and ref_gpu.bvh_available():
        t_rbake = timeit(lambda: ref_gpu.reference_update_visibility(xyz, s, r, icov, op, nrm, N), n=1, warm=1)
        rvis = ref_gpu.reference_update_visibility(xyz, s, r, icov, op, nrm, N)[0]
        flip = float(((vis_o == 0) != (rvis == 0)).float().mean())
        out.update(ref_bake_ms=t_rbake, ref_Mrays_per_s=P * N / t_rbake / 1e3, bake_speedup=t_rbake / t_bake, flip_rate_vs_reference=flip)
    print(json.dumps(out), flush=True)


class Light:
    def __init__(self, env_raw):
        self.env = env_raw

    @property
    def get_env(self):
        return F.softplus(self.env)


def shade(P, N):
    c = {k: v.cuda() for k, v in shading_case(P, N, 16, seed=2).items()}

    def run(ours):
        leaves = {k: c[k].clone().requires_grad_(True) for k in ("base_color", "roughness", "viewdirs", "incidents")}
        env_raw = c["env_raw"].clone().requires_grad_(True)
        if ours:
            pbr, ex = shading.rendering_equation(leaves["base_color"], leaves["roughness"], c["normals"], leaves["viewdirs"],
                                                 leaves["incidents"], Light(env_raw), c["visibility"], c["incident_dirs"], c["incident_areas"])
        else:
            pbr, ex = osh.rendering_equation(leaves["base_color"], leaves["roughness"], c["normals"], leaves["viewdirs"],
                                             leaves["incidents"], F.softplus(env_raw)[0], c["visibility"], c["incident_dirs"], c["incident_areas"])
        ((pbr * c["cot_pbr"]).sum() + (ex["diffuse_light"] * c["cot_diffuse"]).sum()).backward()
    t_o = timeit(lambda: run(True), n=5)
    torch.cuda.reset_peak_memory_stats(); run(True); mem_o = torch.cuda.max_memory_allocated()
    t_r = timeit(lambda: run(False), n=3)
    torch.cuda.reset_peak_memory_stats(); run(False); mem_r = torch.cuda.max_memory_allocated()
    print(json.dumps(dict(what="shading fwd+bwd", P=P, N=N, ours_ms=t_o, pytorch_ms=t_r, speedup=t_r / t_o,
                          ours_peak_GB=mem_o / 1e9, pytorch_peak_GB=mem_r / 1e9,
                          ours_GBps_of_baked_tensors=2 * P * N * 20 / t_o / 1e6)), flush=True)


def shade_kernels(P, N):
    """Kernel-only timing of r3dg_render_equation_forward / _backward (no autograd glue) for every
    kernel variant (r3dg_tune): lanes per Gaussian x env-gradient mode."""
    import ctypes
    from relightable3dgaussian_b200 import _lib
    from relightable3dgaussian_b200.shading import _shade_args
    lib = _lib.load()
    c = {k: v.cuda() for k, v in shading_case(P, N, 16, seed=2).items()}
    env = F.softplus(c["env_raw"])[0].contiguous()
    f = dict(dtype=torch.float32, device="cuda")
    outs = [torch.empty((P, 3), **f) for _ in range(3)]
    grads = dict(d_base=torch.empty((P, 3), **f), d_rough=torch.empty((P, 1), **f), d_view=torch.empty((P, 3), **f),
                 d_inc=torch.empty((P, 16, 3), **f), d_env=torch.empty(env.shape, **f))
    a, _, _ = _shade_args([c[k] for k in ("base_color", "roughness", "normals", "viewdirs", "incidents")] + [env] +
                          [c[k] for k in ("visibility", "incident_dirs", "incident_areas")], None)
    a.pbr, a.diffuse_light, a.specular = [t.data_ptr() for t in outs]
    a.dL_dpbr, a.dL_ddiffuse_light = c["cot_pbr"].data_ptr(), c["cot_diffuse"].data_ptr()
    a.dL_dbase_color, a.dL_droughness, a.dL_dviewdirs = grads["d_base"].data_ptr(), grads["d_rough"].data_ptr(), grads["d_view"].data_ptr()
    a.dL_dincidents, a.dL_denv = grads["d_inc"].data_ptr(), grads["d_env"].data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    ref = None
    for group, mode, fv, bv in ((8, 2, 0, 0), (8, 2, 1, 1), (8, 2, 1, 2), (8, 1, 1, 2), (8, 1, 1, 1), (32, 1, 0, 0)):
        old = _lib.tune("shade_group", group), _lib.tune("shade_env_mode", mode), _lib.tune("shade_fwd_variant", fv), _lib.tune("shade_bwd_variant", bv)
        t_f = timeit(lambda: _lib.check(lib.r3dg_render_equation_forward(ctypes.byref(a), st), "fwd"), n=10, warm=2)
        t_b = timeit(lambda: _lib.check(lib.r3dg_render_equation_backward(ctypes.byref(a), st), "bwd"), n=10, warm=2)
        sig = [float(outs[0].double().sum()), float(grads["d_inc"].double().abs().sum()), float(grads["d_env"].double().abs().sum())]
        ref = ref or sig
        for k, v in zip(("shade_group", "shade_env_mode", "shade_fwd_variant", "shade_bwd_variant"), old):
            _lib.tune(k, v)
        print(json.dumps(dict(what="shading kernels", P=P, N=N, group=group, env_mode=mode, fwd_variant=fv, bwd_variant=bv, fwd_ms=t_f, bwd_ms=t_b,
                              fwd_GBps=P * N * 20 / t_f / 1e6, bwd_GBps=P * N * 20 / t_b / 1e6,
                              checksum_rel=[abs(x - y) / (abs(y) + 1e-30) for x, y in zip(sig, ref)])), flush=True)


def adam_stage2(P):
    """FusedAdam over the stage-2 parameter groups (114 floats per Gaussian, bench_stage2.make_model)."""
    from relightable3dgaussian_b200.optim import FusedAdam
    shapes = [(3,), (3,), (4,), (3,), (1,), (1, 3), (15, 3), (3,), (1,), (1, 3), (15, 3)]
    ps = [torch.randn((P,) + s, device="cuda").requires_grad_(True) for s in shapes]
    for q in ps:
        q.grad = torch.randn_like(q) * 1e-3
    opt = FusedAdam([{"params": [q], "lr": 1e-3} for q in ps], lr=0.0, eps=1e-15)
    t = timeit(opt.step, n=10, warm=3)
    elems = P * 114
    print(json.dumps(dict(what="adam step (stage-2 groups)", P=P, elems=elems, ours_ms=t, ours_GBps=elems * 28 / t / 1e6)), flush=True)


def shade_once(P, N):
    """One fused rendering_equation forward + backward (ncu target)."""
    c = {k: v.cuda() for k, v in shading_case(P, N, 16, seed=2).items()}
    leaves = {k: c[k].clone().requires_grad_(True) for k in ("base_color", "roughness", "viewdirs", "incidents")}
    env_raw = c["env_raw"].clone().requires_grad_(True)
    for _ in range(2):
        pbr, ex = shading.rendering_equation(leaves["base_color"], leaves["roughness"], c["normals"], leaves["viewdirs"],
                                             leaves["incidents"], Light(env_raw), c["visibility"], c["incident_dirs"], c["incident_areas"])
        ((pbr * c["cot_pbr"]).sum() + (ex["diffuse_light"] * c["cot_diffuse"]).sum()).backward()
    torch.cuda.synchronize()


def adam(P):
    """Fused optimiser step over the reference's stage-1 parameter groups (62 floats per Gaussian)
    vs torch.optim.Adam (foreach) and torch's own fused implementation."""
    from relightable3dgaussian_b200.optim import FusedAdam
    shapes = [(3,), (3,), (4,), (3,), (1,), (1, 3), (15, 3)]
    res = {}
    for name, cls, kw in (("ours", FusedAdam, {}), ("torch_foreach", torch.optim.Adam, {}), ("torch_fused", torch.optim.Adam, {"fused": True})):
        ps = [torch.randn((P,) + s, device="cuda").requires_grad_(True) for s in shapes]
        for q in ps:
            q.grad = torch.randn_like(q) * 1e-3
        opt = cls([{"params": [q], "lr": 1e-3} for q in ps], lr=0.0, eps=1e-15, **kw)
        res[name] = timeit(opt.step, n=20, warm=3)
        del opt, ps
    elems = P * 62
    print(json.dumps(dict(what="adam step", P=P, elems=elems, ours_ms=res["ours"], torch_foreach_ms=res["torch_foreach"],
                          torch_fused_ms=res["torch_fused"], ours_GBps=elems * 28 / res["ours"] / 1e6,
                          speedup_vs_foreach=res["torch_foreach"] / res["ours"], speedup_vs_torch_fused=res["torch_fused"] / res["ours"])), flush=True)


if __name__ == "__main__":
    which = sys.argv[1:] or ["bvh", "shade", "kernels", "adam"]
    if "bvh" in which:
        bvh(300_000, 64)
        bvh(300_000, 64, "cube-v1")
        bvh(1_500_000, 32, "cube-v1")
    if "bvh_fast" in which:                       # ncu target: one configuration, no reference
        bvh(300_000, 64, "cube-v1", ref=False)
    if "shade" in which:
        shade(300_000, 64)
        shade(1_000_000, 32)
    if "kernels" in which:
        shade_kernels(300_000, 64)
        shade_kernels(1_000_000, 32)
        shade_kernels(100_000, 384)
    if "adam" in which:
        adam(1_000_000)
    if "adam2" in which:
        adam_stage2(1_500_000)
    if "shade_once" in which:
        shade_once(300_000, 64)

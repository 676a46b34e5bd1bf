#!/usr/bin/env python3
"""Generates tests/golden/shade_edge.npz by EXECUTING the reference's own function bodies on the CPU, in fp32 and in
fp64: `rendering_equation` + `GGX_specular` (/root/reference/gaussian_renderer/neilf.py:339-406),
`DirectLightMap.direct_light` / `get_env` (scene/direct_light_map.py:70-83,104-106) and `EnvLight.direct_light`
(scene/envmap.py:35-53; the method only, the module imports nvdiffrast and pyexr).  The sources are cut out of the
files with `ast` and compiled unmodified into a namespace that provides torch, numpy, F and the reference's eval_sh
(utils/sh_utils.py, imported by path).  Gradients come from autograd through those functions.

Every case is small, seeded and adversarial (see CASES), and asserts from its own inputs that it reaches the path it
is named for (tests/shading_edge.py: path_stats / assert_reaches).  Stored per case: the fp32 inputs (`in_*`; an
`in_transform` marks an EnvLight case, whose `in_env` is the fixed envmap, otherwise `in_env` is the raw map that
`get_env` passes through softplus), and for `32` and `64` the outputs, the computed `extra_results` entries and the
autograd gradients of every leaf.  Of the seven entries, `incident_dirs` / `incident_visibility` are the inputs
themselves (checked by identity here) and `incident_lights` is `local_incident_lights + global_incident_lights` in one
rounding (checked bit for bit here): shading_edge.load_cases rebuilds it, so it is not stored.  /root/reference is
absent on the GPU machine: only the outputs are committed."""
import ast
import importlib.util
import math
import os
import sys
import textwrap

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from helpers import shading_case  # noqa: E402
import shading_edge as se  # noqa: E402
from oracle.oracle_sampling import fibonacci_sphere_sampling  # noqa: E402

REF = "/root/reference"


def cut(path, names, cls=None):
    src = open(path).read()
    body = ast.parse(src).body
    if cls is not None:
        body = next(n for n in body if isinstance(n, ast.ClassDef) and n.name == cls).body
    out = []
    for n in body:
        if isinstance(n, ast.FunctionDef) and n.name in names:
            decos = "".join("@" + ast.get_source_segment(src, d) + "\n" for d in n.decorator_list)
            out.append(decos + ast.get_source_segment(src, n))
    assert len(out) == len(names), (path, names, cls)
    return out


def ref_namespace():
    spec = importlib.util.spec_from_file_location("ref_sh_utils", os.path.join(REF, "utils/sh_utils.py"))
    sh_utils = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sh_utils)
    ns = dict(torch=torch, np=np, F=F, eval_sh=sh_utils.eval_sh)
    for s in cut(os.path.join(REF, "gaussian_renderer/neilf.py"), ["rendering_equation", "GGX_specular"]):
        exec(compile(s, "neilf.py", "exec"), ns)
    for cls, path, names in (("DirectLightMap", "scene/direct_light_map.py", ["direct_light", "get_env"]),
                             ("EnvLight", "scene/envmap.py", ["direct_light"])):
        methods = cut(os.path.join(REF, path), names, cls=cls)
        exec(compile(f"class Ref{cls}:\n" + "\n".join(textwrap.indent(m, "    ") for m in methods), path, "exec"), ns)
    return ns


# ---- cases -----------------------------------------------------------------------------------------------------------
def _base(P, N, He, seed):
    """helpers.shading_case with the raw env map on a 1/16 grid and the SH coefficients on a 1/256 grid (keeps the
    fixture small), inputs keyed as stored."""
    c = shading_case(P, N, He, seed)
    c["env"] = torch.round(c.pop("env_raw") * 16) / 16
    c["incidents"] = torch.round(c["incidents"] * 256) / 256
    return c


def _fixed_env(c, g):
    """EnvLight inputs: a fixed non-negative envmap [He, We, 3] (no softplus)."""
    He, We = c["env"].shape[1:3]
    c["env"] = torch.round(torch.rand(He, We, 3, generator=g) * 64) / 32


def _unit(x):
    return F.normalize(x, dim=-1)


def case_zero_incidents():
    c = _base(29, 16, 16, 11)                      # the stage-2 initial state (scene/gaussian_model.py:394)
    c["incidents"].zero_()
    return c


def case_zero_incidents_dc():
    c = _base(31, 16, 16, 12)                      # only the DC term, never positive: local_raw is 0 or negative
    g = torch.Generator().manual_seed(12)
    inc = torch.zeros(31, 16, 3)
    inc[:, 0] = -torch.rand(31, 3, generator=g) * 0.5
    inc[::3, 0, 1] = 0.0
    inc[1::5, 0, :] = 0.0
    c["incidents"] = inc
    return c


def case_nom_clamp():
    P, N = 32, 16
    c = _base(P, N, 16, 13)
    g = torch.Generator().manual_seed(13)
    n = _unit(torch.randn(P, 3, generator=g))
    t = _unit(torch.cross(n, torch.randn(P, 3, generator=g), dim=-1))
    a = 0.3 + 0.9 * torch.rand(P, 1, generator=g)
    v = _unit(torch.cos(a) * n + torch.sin(a) * t)
    refl = 2 * (n * v).sum(-1, keepdim=True) * n - v
    dirs, _ = fibonacci_sphere_sampling(n, N, random_rotate=False)
    # 10 of 16 samples in a 0.01 rad cone around the mirror direction: H ~ N, nom below 1e-6 at roughness 0.09
    jit = torch.randn(P, 10, 3, generator=g)
    jit = jit - (jit * refl[:, None]).sum(-1, keepdim=True) * refl[:, None]
    dirs[:, :10] = _unit(refl[:, None] + 0.01 * torch.rand(P, 10, 1, generator=g) * _unit(jit))
    c.update(normals=n, viewdirs=v, incident_dirs=dirs.contiguous(), roughness=torch.full((P, 1), 0.09))
    return c


def case_v_perp_n():
    P, N = 30, 16
    c = _base(P, N, 16, 14)
    pairs = [((0, 0, 1), (1, 0, 0)), ((0, 0, 2), (0, -3, 0)), ((1, 0, 0), (0, 0.6, 0.8)), ((0, 1, 0), (-1, 0, 0)),
             ((0, 0, -1), (0.6, 0.8, 0)), ((0, -0.5, 0), (0, 0, 1))]
    n, v = c["normals"].clone(), c["viewdirs"].clone()
    for i in range(24):
        n[i], v[i] = torch.tensor(pairs[i % 6][0]), torch.tensor(pairs[i % 6][1])
    dirs, areas = fibonacci_sphere_sampling(_unit(n), N, random_rotate=False)
    c.update(normals=n, viewdirs=v, incident_dirs=dirs.contiguous(), incident_areas=areas.contiguous())
    return c


def case_back_facing():
    P, N = 32, 16
    c = _base(P, N, 16, 15)
    g = torch.Generator().manual_seed(15)
    n = c["normals"].clone()
    m = torch.where((torch.arange(P) % 2 == 0)[:, None], -n, torch.randn(P, 3, generator=g))
    dirs, _ = fibonacci_sphere_sampling(_unit(m), N, random_rotate=False)
    # n . d == 0 exactly: z normals (not unit length) against equatorial directions
    ang = torch.rand(8, 8, generator=g) * 2 * math.pi
    n[:8] = torch.tensor([0.0, 0.0, 1.0]) * (1 + 0.1 * torch.arange(8.0))[:, None]
    dirs[:8, :8] = torch.stack([torch.cos(ang), torch.sin(ang), torch.zeros_like(ang)], -1)
    c.update(normals=n, incident_dirs=dirs.contiguous())
    return c


def case_l_eq_minus_v():
    P, N = 22, 16
    c = _base(P, N, 16, 16)
    v = c["viewdirs"].clone()
    v[::2] = -_unit(c["normals"][::2] + 0.3 * torch.randn(P // 2, 3, generator=torch.Generator().manual_seed(16)))
    dirs = c["incident_dirs"].clone()
    dirs[:, 3] = -v                                # L = -V exactly: h = 0 and F.normalize takes its eps branch
    c.update(viewdirs=v, incident_dirs=dirs)
    return c


def _seam_pole_dirs(P, g):
    """12 directions per row: dx < 0 with dy = +0 / -0 (columns 0 / We-1), dz = +-1 exactly and +-(1 - 1 ulp)."""
    one_ulp = float(torch.nextafter(torch.tensor(1.0), torch.tensor(0.0)))
    out = torch.empty(P, 12, 3)
    for p in range(P):
        s = float(0.2 + 0.75 * torch.rand(1, generator=g))
        z = math.sqrt(1 - s * s)
        e = 1e-4 * (1 + float(torch.rand(1, generator=g)))
        out[p] = torch.tensor([[-s, 0.0, z], [-s, -0.0, z], [-s, 0.0, -z], [-s, -0.0, -z],
                               [0.0, 0.0, 1.0], [0.0, 0.0, -1.0], [e, -e, 1.0], [-e, 0.0, -1.0],
                               [e, e, one_ulp], [-e, e, -one_ulp], [-1.0, 0.0, 0.0], [-1.0, -0.0, 0.0]])
    return out


def case_seam_poles(He, seed):
    P, N = 24, 16
    c = _base(P, N, He, seed)
    g = torch.Generator().manual_seed(seed)
    dirs = c["incident_dirs"].clone()
    sp = _seam_pole_dirs(P, g)
    dirs[:, :12] = sp
    pick = sp[torch.arange(P), torch.arange(P) % 12]
    n = pick + 0.2 * torch.randn(P, 3, generator=g)             # each row lights one special direction
    vis = c["visibility"].clone()
    vis[:, :12] = 1.0
    c.update(normals=n, incident_dirs=dirs, visibility=vis)
    return c


def case_random_rotate():
    P, N = 24, 32
    c = _base(P, N, 24, 17)
    g = torch.Generator().manual_seed(17)
    n = _unit(torch.randn(P, 3, generator=g))
    dirs, _ = fibonacci_sphere_sampling(n, N, random_rotate=True, phase=torch.rand(P, generator=g))
    areas = 2 * math.pi * (0.5 + torch.rand(P, N, 1, generator=g))
    c.update(normals=(n + 0.3 * torch.randn(P, 3, generator=g)).contiguous(), incident_dirs=dirs.contiguous(),
             incident_areas=areas)
    return c


def case_envlight_perm():
    P, N = 24, 16
    c = _base(P, N, 16, 18)
    g = torch.Generator().manual_seed(18)
    _fixed_env(c, g)
    c["transform"] = torch.tensor(se.TO_OPENGL)
    dirs = c["incident_dirs"].clone()
    # in the env frame (x, z, -y): the seam for dz = +-0 and dx < 0, the poles for dy = -+1.  The second direction's
    # y row is three -0 products, which `@` (a BLAS product) sums to +0: column 0, not We-1
    dirs[:, :4] = torch.tensor([[-0.8, 0.6, 0.0], [-0.8, -0.6, -0.0], [0.0, -1.0, 0.0], [0.0, 1.0, 0.0]])
    n = c["normals"].clone()
    n[: P // 2] = dirs[: P // 2, 0] + 0.2 * torch.randn(P // 2, 3, generator=g)
    n[P // 2:] = dirs[P // 2:, 1] + 0.2 * torch.randn(P - P // 2, 3, generator=g)
    vis = c["visibility"].clone()
    vis[:, :4] = 1.0
    c.update(normals=n, incident_dirs=dirs, visibility=vis)
    return c


def case_envlight_rot():
    P, N = 24, 16
    c = _base(P, N, 16, 19)
    g = torch.Generator().manual_seed(19)
    _fixed_env(c, g)
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    T = q.float()
    # keep |e_z| < 0.99 in the env frame: acos of a rounded |e_z| > 1 is NaN in the reference as well
    dirs = c["incident_dirs"].clone()
    bad = (dirs @ T.T)[..., 2].abs() > 0.99
    dirs[bad] = _unit(dirs[bad] + torch.tensor([0.3, 0.3, 0.3]) @ T)
    assert ((dirs @ T.T)[..., 2].abs() <= 0.99).all()
    c.update(transform=T, incident_dirs=dirs.contiguous())
    return c


CASES = {"zero_incidents": case_zero_incidents, "zero_incidents_dc": case_zero_incidents_dc, "nom_clamp": case_nom_clamp,
         "v_perp_n": case_v_perp_n, "back_facing": case_back_facing, "l_eq_minus_v": case_l_eq_minus_v,
         "seam_poles": lambda: case_seam_poles(16, 20), "seam_poles_64": lambda: case_seam_poles(64, 21),
         "random_rotate": case_random_rotate, "envlight_perm": case_envlight_perm, "envlight_rot": case_envlight_rot}
INPUTS = ("base_color", "roughness", "normals", "viewdirs", "incidents", "env", "visibility", "incident_dirs",
          "incident_areas", "transform", "cot_pbr", "cot_diffuse", "cot_specular")


def run_reference(ns, c, dtype):
    t = {k: v.to(dtype) for k, v in c.items()}
    leaves = {k: t[k].clone().requires_grad_(True) for k in se.LEAVES}
    if "transform" in t:
        light = ns["RefEnvLight"]()
        light.envmap, light.transform = leaves["env"], t["transform"]
    else:
        light = ns["RefDirectLightMap"]()
        light.env = leaves["env"]
    pbr, extra = ns["rendering_equation"](leaves["base_color"], leaves["roughness"], t["normals"], leaves["viewdirs"],
                                          leaves["incidents"], light, visibility_precompute=t["visibility"],
                                          incident_dirs_precompute=t["incident_dirs"],
                                          incident_areas_precompute=t["incident_areas"])
    assert extra["incident_dirs"] is t["incident_dirs"] and extra["incident_visibility"] is t["visibility"]
    assert set(extra) == set(se.EXTRAS) | {"incident_dirs", "incident_visibility"}
    loss = (pbr * t["cot_pbr"]).sum() + (extra["diffuse_light"] * t["cot_diffuse"]).sum() + (extra["specular"] * t["cot_specular"]).sum()
    loss.backward()
    # incident_lights is local + global, one rounding: not stored, shading_edge.load_cases adds the two back
    assert torch.equal(extra["incident_lights"], extra["local_incident_lights"] + extra["global_incident_lights"])
    rec = {"pbr": pbr.detach().numpy()}
    rec.update({k: extra[k].detach().numpy() for k in se.EXTRAS if k != "incident_lights"})
    rec.update({"grad_" + k: v.grad.numpy() for k, v in leaves.items()})
    for k, v in rec.items():
        assert v.dtype == {torch.float32: np.float32, torch.float64: np.float64}[dtype] and np.isfinite(v).all(), k
    return rec


def main():
    torch.set_num_threads(1)
    ns = ref_namespace()
    rec = {}
    for name, make in CASES.items():
        c = {k: v.float().contiguous() for k, v in make().items()}
        assert set(c) <= set(INPUTS), set(c) - set(INPUTS)
        s = se.path_stats(c)
        se.assert_reaches(name, s)
        rec.update({f"{name}/in_{k}": v.numpy() for k, v in c.items()})
        for tag, dt in (("32", torch.float32), ("64", torch.float64)):
            rec.update({f"{name}/{tag}/{k}": v for k, v in run_reference(ns, c, dt).items()})
        print(f"{name:18s} P={c['base_color'].shape[0]:3d} N={c['incident_dirs'].shape[1]:2d} env={tuple(c['env'].shape[-3:-1])} "
              f"pbr mean {rec[f'{name}/64/pbr'].mean():.5f}  {s}")
    path = se.PATH
    np.savez_compressed(path, **rec)
    print(f"wrote {path}: {os.path.getsize(path) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()

"""Adversarial cases of the fused shading step (tests/golden/shade_edge.npz, written by
tests/golden/make_golden_shading_edge.py) and the fp64 pieces the CPU and GPU tests share: which
edge paths a case reaches, and the environment-map gradient as an explicit fp64 scatter of the four
bilinear taps of grid_sample(align_corners=True, zeros padding)."""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

from helpers import GOLDEN

EPS32 = float(np.finfo(np.float32).eps)
PATH = os.path.join(GOLDEN, "shade_edge.npz")
LEAVES = ("base_color", "roughness", "viewdirs", "incidents", "env")
EXTRAS = ("incident_lights", "local_incident_lights", "global_incident_lights", "diffuse_light", "specular")
# scene/envmap.py EnvLight.to_opengl: a signed permutation, so `dirs @ T.T` is exact in fp32
TO_OPENGL = [[1.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, -1.0, 0.0]]


def load_cases(path=PATH):
    """{case: {key: array}} with keys in_<input>, <32|64>/<output>; `in_transform` marks an EnvLight case."""
    g = np.load(path)
    out = {}
    for k in g.files:
        name, _, rest = k.partition("/")
        out.setdefault(name, {})[rest] = g[k]
    for c in out.values():              # incident_lights = local + global, the reference's one rounding in either dtype
        for tag in ("32", "64"):
            c[f"{tag}/incident_lights"] = c[f"{tag}/local_incident_lights"] + c[f"{tag}/global_incident_lights"]
    return out


def env_frame(dirs, transform):
    """[..., 3] directions in the env map's frame: `dirs @ transform.T` as in EnvLight.direct_light."""
    d = dirs.reshape(-1, 3)
    return d if transform is None else d @ transform.T


def path_stats(c):
    """Counts of the edge paths a case reaches, evaluated with the reference's own fp32 torch ops on its fp32 inputs
    (c: input name -> tensor).  Per sample unless noted."""
    from oracle import oracle_shading as osh
    dirs, n, v, r = c["incident_dirs"], c["normals"], c["viewdirs"], c["roughness"]
    P, N = dirs.shape[:2]
    He = c["env"].shape[-3]
    local = osh.eval_sh3(c["incidents"].transpose(1, 2).reshape(-1, 1, 3, 16), dirs)
    L, V, Nn = F.normalize(dirs, dim=-1), F.normalize(v, dim=-1), F.normalize(n, dim=-1)
    h = (L + V[:, None, :]) / 2.0
    nov = torch.sum(V * Nn, dim=-1, keepdim=True)
    Ns = Nn * nov.sign()
    H = F.normalize(h, dim=-1)
    NoL = torch.sum(Ns[:, None, :] * L, dim=-1, keepdim=True).clamp(1e-6, 1)
    NoV = torch.sum(Ns * V, dim=-1, keepdim=True).clamp(1e-6, 1)
    NoH = torch.sum(Ns[:, None, :] * H, dim=-1, keepdim=True).clamp(1e-6, 1)
    a2 = (r * r) * (r * r)
    k = (r * r + 2 * r + 1.0) / 8.0
    nom0 = NoH * NoH * (a2[:, None, :] - 1) + 1
    nom1 = NoV * (1 - k) + k
    nom2 = NoL * (1 - k[:, None, :]) + k[:, None, :]
    nom_r = 4 * np.pi * nom0 * nom0 * nom1[:, None, :] * nom2
    ndi = (n[:, None] * dirs).sum(-1)
    T = c.get("transform")
    e = env_frame(dirs, T)
    ex, ey, ez = e.unbind(-1)
    below1 = torch.nextafter(torch.tensor(1.0), torch.tensor(0.0)).to(ez)
    iy = ((torch.arccos(ez) - 1e-6) / np.pi * 2 - 1 + 1) / 2 * (He - 1)
    lit = (ndi > 0).reshape(-1)
    seam = (ex < 0) & (ey == 0)
    # seam samples whose transformed y is a sum of -0 terms: -0 left to right, +0 from `@`
    d = dirs.reshape(-1, 3)
    ey_sum = d[:, 0] * T[1, 0] + d[:, 1] * T[1, 1] + d[:, 2] * T[1, 2] if T is not None else ey
    return dict(samples=P * N, rows=P,
                local_zero=int((local == 0).sum()), local_neg=int((local < 0).sum()), local_pos=int((local > 0).sum()),
                nov_zero_rows=int((nov == 0).sum()), h_zero=int((h.norm(dim=-1) == 0).sum()),
                nom_clamp=int(((nom_r < 1e-6).reshape(-1) & lit).sum()), nom_free=int(((nom_r >= 1e-6).reshape(-1) & lit).sum()),
                back=int((ndi < 0).sum()), ndi_zero=int((ndi == 0).sum()),
                seam_pos=int((seam & ~torch.signbit(ey)).sum()), seam_neg=int((seam & torch.signbit(ey)).sum()),
                seam_pos_lit=int((seam & ~torch.signbit(ey) & lit).sum()), seam_neg_lit=int((seam & torch.signbit(ey) & lit).sum()),
                seam_neg_zero_sum=int((seam & ~torch.signbit(ey) & torch.signbit(ey_sum) & lit).sum()),
                pole=int((ez.abs() == 1).sum()), pole_ulp=int((ez.abs() == below1).sum()),
                pad_row=int(((iy < 0) | (iy > He - 1)).sum()), max_abs_ez=float(ez.abs().max()),
                areas_distinct=int(torch.unique(c["incident_areas"]).numel()))


def assert_reaches(name, s):
    """Each fixture case exists for one path; fail if its inputs no longer reach it."""
    if name == "zero_incidents":
        assert s["local_zero"] == 3 * s["samples"], s
    elif name == "zero_incidents_dc":
        assert s["local_pos"] == 0 and s["local_zero"] > 100 and s["local_neg"] > 100, s
    elif name == "nom_clamp":
        assert s["nom_clamp"] > s["samples"] // 4 and s["nom_free"] > s["samples"] // 4, s
    elif name == "v_perp_n":
        assert s["nov_zero_rows"] >= 24, s
    elif name == "back_facing":
        assert s["back"] > s["samples"] // 4 and s["ndi_zero"] >= 32, s
    elif name == "l_eq_minus_v":
        assert s["h_zero"] == s["rows"], s
    elif name.startswith("seam_poles"):
        assert min(s["seam_pos_lit"], s["seam_neg_lit"]) >= 8 and s["pole"] >= 4 * s["rows"] and s["pole_ulp"] >= 2 * s["rows"], s
        assert s["pad_row"] >= 2 * s["rows"], s
    elif name == "random_rotate":
        assert s["areas_distinct"] > 100 and s["back"] > 0, s
    elif name == "envlight_perm":
        assert s["seam_pos_lit"] >= 8 and s["seam_neg_zero_sum"] >= 4 and s["pole"] >= 2 * s["rows"], s
    elif name == "envlight_rot":
        assert s["max_abs_ez"] < 0.999, s
    else:
        raise KeyError(name)


def inputs(c, device="cpu"):
    """The fp32 inputs of a fixture case as tensors on `device`."""
    return {k[3:]: torch.from_numpy(v).to(device) for k, v in c.items() if k.startswith("in_")}


COTS = ("pbr", "diffuse", "specular")


def oracle_run(t, dtype, cots=COTS):
    """oracle_shading.rendering_equation on the inputs t (fp32, cast to dtype here), L = sum of <output, cot_output>
    over `cots`.  Returns the outputs, the five extras, grad_<leaf> (grad_env: of the raw map for a DirectLightMap case,
    of the envmap for an EnvLight case), grad_tex (of the texture the lookup reads) and g_light (of the looked-up light,
    per sample: what grid_sample's backward scatters)."""
    from oracle import oracle_shading as osh
    t = {k: v.to(dtype) for k, v in t.items()}
    leaves = {k: t[k].clone().requires_grad_(True) for k in LEAVES}
    T = t.get("transform")
    tex = leaves["env"] if T is not None else F.softplus(leaves["env"])[0]
    if T is None:
        tex.retain_grad()
    pbr, ex = osh.rendering_equation(leaves["base_color"], leaves["roughness"], t["normals"], leaves["viewdirs"],
                                     leaves["incidents"], tex, t["visibility"], t["incident_dirs"], t["incident_areas"],
                                     transform=T)
    ex["global_incident_lights"].retain_grad()
    outs = dict(pbr=pbr, diffuse=ex["diffuse_light"], specular=ex["specular"])
    sum((outs[k] * t["cot_" + k]).sum() for k in cots).backward()
    rec = {"pbr": pbr.detach(), **{k: ex[k].detach() for k in EXTRAS}}
    rec.update({"grad_" + k: v.grad for k, v in leaves.items()})
    rec["grad_tex"] = tex.grad
    rec["g_light"] = ex["global_incident_lights"].grad * t["visibility"]
    return rec


PER_ROW = ("base_color", "roughness", "normals", "viewdirs", "incidents", "cot_pbr", "cot_diffuse", "cot_specular")


def oracle_magnitudes(t, cots=COTS):
    """fp64 magnitudes of the sums behind each per-Gaussian result: for the outputs and leaf gradients, the mean over
    the N samples of |the sample's own term| (the case re-run with every sample as a Gaussian of its own, N = 1) under
    |cotangents|; for the env texture, sum over taps of |contribution| under |cotangents| (`tex`)."""
    P, N = t["incident_dirs"].shape[:2]
    a = {k: (v.abs() if k.startswith("cot_") else v) for k, v in t.items()}
    s = {k: (v.repeat_interleave(N, 0) if k in PER_ROW else v if k in ("env", "transform") else v.reshape(P * N, 1, -1))
         for k, v in a.items()}
    rec = oracle_run(s, torch.float64, cots)
    out = {}
    for k in ("pbr", "diffuse_light", "specular") + tuple("grad_" + k for k in LEAVES[:4]):
        x = rec[k]
        out[k] = None if x is None else x.abs().reshape(P, N, *x.shape[1:]).sum(1) / N
    full = oracle_run(a, torch.float64, cots)
    He, We = full["grad_tex"].shape[-3:-1]
    T = t.get("transform")
    out["tex"] = env_scatter64(env_frame(t["incident_dirs"].double(), None if T is None else T.double()),
                               full["g_light"], He, We)[1]
    return out


def env_scatter64(e, g, He, We):
    """grid_sample's adjoint written out: the fp64 gradient of an [He, We, 3] env texture from per-sample gradients
    g [S, 3] of the looked-up light at env-frame directions e [S, 3], and per texel the sum of |contribution|.
    Same coordinates as scene/direct_light_map.py direct_light: phi = acos(z) - 1e-6, theta = atan2(y, x)."""
    e, g = e.reshape(-1, 3).double(), g.reshape(-1, 3).double()
    phi = torch.arccos(e[:, 2]) - 1e-6
    theta = torch.atan2(e[:, 1], e[:, 0])
    ix = ((-theta / math.pi) + 1) / 2 * (We - 1)
    iy = ((phi / math.pi) * 2 - 1 + 1) / 2 * (He - 1)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    grad = torch.zeros(He * We, 3, dtype=torch.float64, device=e.device)
    mag = torch.zeros_like(grad)
    for xs, wx in ((x0, x0 + 1 - ix), (x0 + 1, ix - x0)):
        for ys, wy in ((y0, y0 + 1 - iy), (y0 + 1, iy - y0)):
            inside = (xs >= 0) & (xs < We) & (ys >= 0) & (ys < He)
            idx = (ys * We + xs).long()[inside]
            contrib = g[inside] * (wx * wy)[inside, None]
            grad.index_add_(0, idx, contrib)
            mag.index_add_(0, idx, contrib.abs())
    return grad.reshape(He, We, 3), mag.reshape(He, We, 3)

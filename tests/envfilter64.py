"""fp64 restatement of the shading step's filtered environment lookup (include/r3dg_b200.h, PREFILTERED ENVIRONMENT):
the lat-long mip pyramid, the level of detail and the trilinear taps, and the shading formula of
oracle/oracle_shading.py with that global light.  Written as dense torch operations, so autograd through it gives the
pyramid's adjoint without restating it."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import oracle_shading as osh

MAX_LEVELS = 16


def level_sizes(He, We):
    """[(H_l, W_l)]: level l+1 halves level l (ceil) while level l has at least 3 rows and 3 columns."""
    sizes = [(He, We)]
    while len(sizes) < MAX_LEVELS and sizes[-1][0] >= 3 and sizes[-1][1] >= 3:
        h, w = sizes[-1]
        sizes.append(((h + 1) // 2, (w + 1) // 2))
    return sizes


def band_weights(h, h2):
    """[h2, h]: solid angle per radian of azimuth shared by latitude band k of an h2-row level and band j of an h-row
    level (rows are the bands [(j - 1/2) dt, (j + 1/2) dt] clipped to [0, pi])."""
    d, d2 = math.pi / (h - 1), math.pi / (h2 - 1)
    j = torch.arange(h, dtype=torch.float64)[None, :]
    k = torch.arange(h2, dtype=torch.float64)[:, None]
    lo = torch.clamp(torch.maximum((j - 0.5) * d, (k - 0.5) * d2), min=0.0)
    hi = torch.clamp(torch.minimum((j + 0.5) * d, (k + 0.5) * d2), max=math.pi)
    return torch.where(hi > lo, torch.cos(lo) - torch.cos(hi), torch.zeros((), dtype=torch.float64))


def cell_weights(w, w2):
    """[w2, w]: azimuth shared by column cell i of a w2-column level and cell m of a w-column level, modulo 2 pi.
    Fine column w-1 (the seam copy of column 0) gets no weight; coarse column w2-1 repeats column 0."""
    d, d2 = 2 * math.pi / (w - 1), 2 * math.pi / (w2 - 1)
    m = torch.arange(w - 1, dtype=torch.float64)[None, :]
    i = torch.arange(w2 - 1, dtype=torch.float64)[:, None]
    out = torch.zeros(w2 - 1, w - 1, dtype=torch.float64)
    for shift in (-(w - 1), 0, w - 1):
        lo = torch.maximum((m + shift - 0.5) * d, (i - 0.5) * d2)
        hi = torch.minimum((m + shift + 0.5) * d, (i + 0.5) * d2)
        out = out + torch.clamp(hi - lo, min=0.0)
    out = torch.cat([out, out[:1]], 0)
    return torch.cat([out, torch.zeros(w2, 1, dtype=torch.float64)], 1)


def downsample(level):
    """The next coarser level of `level` [h,w,3] (fp64, differentiable)."""
    h, w = level.shape[0], level.shape[1]
    h2, w2 = (h + 1) // 2, (w + 1) // 2
    A, B = band_weights(h, h2), cell_weights(w, w2)
    An, Bn = A / A.sum(1, keepdim=True), B / B.sum(1, keepdim=True)
    out = torch.einsum("kj,jmc,im->kic", An, level, Bn)
    caps = torch.einsum("kj,jc->kc", An[[0, h2 - 1]], level[:, : w - 1].mean(1))      # the pole rows: cap means
    rows = [caps[0:1, None].expand(1, w2, 3), out[1:h2 - 1], caps[1:2, None].expand(1, w2, 3)]
    return torch.cat(rows, 0)


def pyramid(env):
    """[level 0 = env, level 1, ...] of the activated env [He,We,3], fp64."""
    levels = [env.double()]
    for _ in level_sizes(env.shape[0], env.shape[1])[1:]:
        levels.append(downsample(levels[-1]))
    return levels


def texel_weights(h, w):
    """[h, w] solid angle of each texel's cell, the seam column 0 (it repeats column 0)."""
    band = band_weights(h, h).diagonal()                       # each row's own band: cos(top) - cos(bottom)
    col = torch.full((w,), 2 * math.pi / (w - 1), dtype=torch.float64)
    col[-1] = 0.0
    return band[:, None] * col[None, :]


def sphere_mean(level):
    """The solid-angle-weighted mean of a level [h,w,3] over the sphere, per channel."""
    wt = texel_weights(level.shape[0], level.shape[1])
    return (level * wt[..., None]).sum((0, 1)) / wt.sum()


def bilinear(level, d):
    """grid_sample(align_corners=True) of level [h,w,3] at directions d [M,3] with the reference's lat-long map."""
    phi = torch.arccos(d[:, 2]) - 1e-6
    theta = torch.atan2(d[:, 1], d[:, 0])
    grid = torch.stack((-theta / np.pi, (phi / np.pi) * 2 - 1), -1)[None, None]
    return F.grid_sample(level.permute(2, 0, 1)[None], grid, align_corners=True)[0, :, 0].T


def lod(d, omega, He, We, L):
    """lambda = log2(omega / Omega0(theta)) / 2 clamped to [0, L-1], Omega0 = dt dp max(sin theta, sin(dt / 2))."""
    if L == 1:
        return torch.zeros(d.shape[0], dtype=torch.float64)
    dt, dp = math.pi / (He - 1), 2 * math.pi / (We - 1)
    st = torch.sqrt(torch.clamp(1 - d[:, 2] ** 2, min=0.0))
    om0 = dt * dp * torch.clamp(st, min=math.sin(dt / 2))
    return torch.clamp(0.5 * torch.log2(omega / om0), 0.0, L - 1.0)


def filtered_lookup(levels, d, lam):
    """Trilinear lookup: levels floor(lam) and floor(lam) + 1 with weights 1 - f and f."""
    L = len(levels)
    taps = torch.stack([bilinear(lv, d) for lv in levels])     # [L, M, 3]
    l0 = torch.clamp(torch.floor(lam).long(), max=L - 1)
    f = (lam - l0.double())[:, None]
    l1 = torch.clamp(l0 + 1, max=L - 1)
    idx = torch.arange(d.shape[0])
    return (1 - f) * taps[l0, idx] + f * taps[l1, idx]


def direct_light_filtered(env, dirs, areas, transform=None):
    """The filtered global light of dirs [P,N,3] with areas [P,N,1] (Omega = area / N), env [He,We,3] activated."""
    P, N = dirs.shape[0], dirs.shape[1]
    d = dirs.reshape(-1, 3).double()
    if transform is not None:
        d = d @ transform.double().T
    He, We = env.shape[0], env.shape[1]
    levels = pyramid(env)
    lam = lod(d, areas.reshape(-1).double() / N, He, We, len(levels))
    return filtered_lookup(levels, d, lam).reshape(P, N, 3)


def rendering_equation(base_color, roughness, normals, viewdirs, incidents, env_tex, visibility, incident_dirs,
                       incident_areas, transform=None):
    """oracle_shading.rendering_equation with the filtered global light, in fp64 (inputs are promoted)."""
    dd = lambda t: t.double()
    base_color, roughness, normals, viewdirs, incidents = map(dd, (base_color, roughness, normals, viewdirs, incidents))
    visibility, incident_dirs, incident_areas = map(dd, (visibility, incident_dirs, incident_areas))
    global_l = direct_light_filtered(env_tex.double(), incident_dirs, incident_areas, transform) * visibility
    local_l = osh.eval_sh3(incidents.transpose(1, 2).reshape(-1, 1, 3, 16), incident_dirs).clamp_min(0)
    lights = local_l + global_l
    n_d_i = (normals[:, None] * incident_dirs).sum(-1, keepdim=True).clamp(min=0)
    f_d = base_color[:, None] / np.pi
    f_s = osh.ggx_specular(normals, viewdirs, incident_dirs, roughness, fresnel=0.04)
    transport = lights * incident_areas * n_d_i
    extra = {"incident_lights": lights, "local_incident_lights": local_l, "global_incident_lights": global_l,
             "diffuse_light": transport.mean(dim=-2), "specular": (f_s * transport).mean(dim=-2)}
    return ((f_d + f_s) * transport).mean(dim=-2), extra

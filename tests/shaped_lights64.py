"""fp64 truth of the spot and rect lights (csrc/lights_trace.cu, csrc/lights.cu; include/r3dg_b200.h, SHAPED LIGHTS).

Sampling: the header's lowbias32 hash chain and the rect samples (s, t, y) reproduced in numpy with the kernels' fp32
op-by-op rounding, so the oracle sees the kernels' points.

Shading: per Gaussian g, light j and sample q, in torch float64 so that autograd gives every gradient (normals and T
get none; each rect sample's (s, t) is held fixed):
    spot:  w = pos - m,  l = w / max(|w|, 1e-12),  x = clamp((-l . a^ - cos_outer) / max(cos_inner - cos_outer, 1e-6), 0, 1),
           E = color x^2 (3 - 2x) / max(|w|^2, 1e-8)
    rect:  y = pos + s u + t v,  w = y - m,  l = w / max(|w|, 1e-12),  n_e = normalize(u x v),  A = 4 |u x v|,
           E = color max(-n_e . l, 0) A / (M^2 max(|w|^2, 1e-8))
    transport = E T[g, col] max(n . l, 0), f_s = GGX_specular along l, summed in light order, then sample order.

Shadows: lights64's brute force (the visibility bake's hit rule, the t_max margin and the `fragile` flags) with one
point light per ray at the ray's fp32 target point."""
import numpy as np
import torch

import lights64 as L64
from oracle.oracle_shading import ggx_specular

SPOT, RECT = 2, 3
EPS = 1e-12
R2_MIN = 1e-8
MASK = 0xFFFFFFFF
f32 = np.float32


def lowbias32(x):
    x &= MASK
    x ^= x >> 16
    x = (x * 0x7FEB352D) & MASK
    x ^= x >> 15
    x = (x * 0x846CA68B) & MASK
    x ^= x >> 16
    return x


def rect_hash(seed, g, j):
    return lowbias32(lowbias32(lowbias32(seed) ^ g) ^ j)


def xi(seed, g, j, q):
    """The jitter (xi1, xi2) of sample q of light j at Gaussian row g, exact in fp32."""
    h = rect_hash(seed, g, j)
    return tuple(f32(lowbias32(h ^ (2 * q + k)) >> 8) * f32(2.0 ** -24) for k in (0, 1))


def rect_sample(pos, u, v, M, seed, g, j, q):
    """(s, t, y [3]) of sample q = i M + k, s = -1 + (2i + 2 xi1) / M and t likewise, rounded op by op in fp32 as the
    kernels do."""
    i, k = divmod(q, M)
    x1, x2 = xi(seed, g, j, q)
    s = f32(f32(-1.0) + f32(f32(f32(2 * i) + f32(2 * x1)) / f32(M)))
    t = f32(f32(-1.0) + f32(f32(f32(2 * k) + f32(2 * x2)) / f32(M)))
    p, uu, vv = (np.asarray(x, np.float32) for x in (pos, u, v))
    y = np.array([f32(f32(p[c] + f32(s * uu[c])) + f32(t * vv[c])) for c in range(3)], np.float32)
    return s, t, y


def columns(kind, M):
    """[(light j, sample q)] of every shadow column, in order."""
    return [(j, q) for j, k in enumerate(kind) for q in range(M * M if k == RECT else 1)]


def ray_targets(kind, pos, a, b, M, seed, P, rows=None):
    """targets [P,R,3] (fp32) and (s, t) [P,R,2] of every ray: a spot's position, a rect's samples at each row."""
    cols = columns(list(kind), M)
    pos, a, b = (np.asarray(x, np.float32).reshape(-1, 3) for x in (pos, a, b))
    tg = np.zeros((P, len(cols), 3), np.float32)
    st = np.zeros((P, len(cols), 2), np.float32)
    for g in (range(P) if rows is None else rows):
        for c, (j, q) in enumerate(cols):
            if kind[j] == RECT:
                s, t, y = rect_sample(pos[j], a[j], b[j], M, seed, g, j, q)
                tg[g, c], st[g, c] = y, (s, t)
            else:
                tg[g, c] = pos[j]
    return tg, st


def shade(base_color, roughness, normals, viewdirs, means, kind, pos, a, b, color, cone, T, M, st):
    """viewdirs [V,P,3] -> (pbr, diffuse_light, specular), each [V,P,3]; st [P,R,2] the rect samples' (s, t) (from
    ray_targets).  Differentiable in every input but normals, T, kind and st."""
    normals = normals.detach()
    T = T.detach()
    st = torch.as_tensor(np.asarray(st, np.float64), dtype=means.dtype)
    rough = roughness.reshape(-1, 1)
    terms = []                                      # per column: (l [P,3], E [P,3])
    col = 0
    for j, k in enumerate(list(kind)):
        if k == SPOT:
            w = pos[j][None] - means
            r2 = (w * w).sum(-1, keepdim=True)
            l = w / w.norm(dim=-1, keepdim=True).clamp_min(EPS)
            ah = torch.nn.functional.normalize(a[j], dim=-1, eps=EPS)
            x = (((-(l * ah).sum(-1, keepdim=True)) - cone[j, 1]) / (cone[j, 0] - cone[j, 1]).clamp_min(1e-6)).clamp(0, 1)
            terms.append((l, color[j][None] * (x * x * (3 - 2 * x)) / r2.clamp_min(R2_MIN), col))
            col += 1
        else:
            c = torch.linalg.cross(a[j], b[j])
            ne = torch.nn.functional.normalize(c, dim=-1, eps=EPS)
            A = 4 * c.norm()
            for q in range(M * M):
                y = pos[j][None] + st[:, col, 0:1] * a[j][None] + st[:, col, 1:2] * b[j][None]
                w = y - means
                r2 = (w * w).sum(-1, keepdim=True)
                l = w / w.norm(dim=-1, keepdim=True).clamp_min(EPS)
                ce = (-(l * ne).sum(-1, keepdim=True)).clamp(min=0)
                terms.append((l, color[j][None] * ce * A / (M * M * r2.clamp_min(R2_MIN)), col))
                col += 1
    outs = []
    for v in range(viewdirs.shape[0]):
        pbr = diff = spec = torch.zeros_like(means)
        for l, E, c in terms:
            tr = E * T[:, c:c + 1] * (normals * l).sum(-1, keepdim=True).clamp(min=0)
            fs = ggx_specular(normals, viewdirs[v], l[:, None], rough)[:, 0]
            pbr, diff, spec = pbr + (base_color / np.pi + fs) * tr, diff + tr, spec + fs * tr
        outs.append((pbr, diff, spec))
    return tuple(torch.stack([o[k] for o in outs]) for k in range(3))


def shadows(means, inv_cov, opacity, normals, boxes, kind, pos, a, b, M, seed, pairs, lone_leaf=False):
    """T [P,R] and fragile [P,R] of the (g, column) rays in `pairs` (the others stay 1), each traced as lights64's point
    light at the ray's fp32 target."""
    P = np.asarray(means).shape[0]
    rows = sorted({g for g, _ in pairs})
    tg, _ = ray_targets(kind, pos, a, b, M, seed, P, rows)
    R = tg.shape[1]
    T, fr = np.ones((P, R)), np.zeros((P, R), bool)
    for g in rows:
        cs = [c for gg, c in pairs if gg == g]
        Tg, fg = L64.shadows(means, inv_cov, opacity, normals, boxes, np.ones(R, np.int32), tg[g], lone_leaf=lone_leaf,
                             pairs=[(g, c) for c in cs])
        T[g, cs], fr[g, cs] = Tg[g, cs], fg[g, cs]
    return T, fr


def polygon_irradiance(x, n, verts):
    """Lambert's formula: the cosine-weighted solid angle of the polygon `verts` [k,3] seen from x with normal n,
    (1/2) |sum_e theta_e n . (v_e x v_e+1) / |v_e x v_e+1||, v_e the unit directions to the vertices.  A Lambertian
    emitter of radiance L gives the irradiance L times this."""
    v = np.asarray(verts, np.float64) - np.asarray(x, np.float64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    s = 0.0
    for e in range(len(v)):
        a, b = v[e], v[(e + 1) % len(v)]
        c = np.cross(a, b)
        s += np.arccos(np.clip(a @ b, -1, 1)) * (np.asarray(n, np.float64) @ c) / np.linalg.norm(c)
    return 0.5 * abs(s)

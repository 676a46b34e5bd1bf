"""fp64 truth of the point and directional lights (csrc/lights_trace.cu, csrc/lights.cu; include/r3dg_b200.h, LIGHTS).

Shading: per Gaussian g and light j
    directional: l = vec_j / max(|vec_j|, 1e-12),  E = color_j
    point:       w = vec_j - m_g,  l = w / max(|w|, 1e-12),  E = color_j / max(|w|^2, R2_MIN)
    transport = E T[g,j] max(n . l, 0),  f_s = GGX_specular (oracle/oracle_shading.py) along l,
    diffuse_light = sum_j transport,  specular = sum_j f_s transport,  pbr = sum_j (base / pi + f_s) transport,
in torch float64 so that autograd gives every gradient (normals and T get none).

Shadows: brute force.  The ray from o = m + 0.05 l along l tests every Gaussian with the visibility bake's hit rule
(tests/indirect64.py), keeps those with peak t < (1 - 1e-5) t_max (t_max = +inf for a directional light, |vec - o| for a point light)
whose leaf box the segment [0, t_max] meets, and multiplies (1 - alpha) over all of them.  The kernel stops once T
< 1e-4, so a T below that is compared as "below 1e-4".  Each ray also gets a `fragile` flag: indirect64's flags (box
graze, t = 0.01, back-face, a t tie) plus a peak t within rounding of (1 - 1e-5) t_max or a box entry within rounding of t_max."""
import numpy as np
import torch

import indirect64 as ind
from oracle.oracle_shading import ggx_specular

R2_MIN = 1e-8
EPS = 1e-12
T_MIN = 1e-4
T_MAX_MARGIN = np.float32(1.0) - np.float32(1e-5)     # hits need peak t < (1 - 1e-5) t_max


def light_dirs(kind, vec, means):
    """(l [P,K,3], E-scale [P,K] = 1 or 1 / max(|w|^2, R2_MIN), w [P,K,3]) in the dtype of the torch inputs."""
    point = (torch.as_tensor(kind) == 1).to(means.device)[None, :, None]
    w = torch.where(point, vec[None] - means[:, None], vec[None].expand(means.shape[0], -1, -1))
    n = w.norm(dim=-1, keepdim=True)
    l = w / n.clamp_min(EPS)
    inv_r2 = torch.where(point[..., 0], 1.0 / (w * w).sum(-1).clamp_min(R2_MIN), torch.ones_like(n[..., 0]))
    return l, inv_r2, w


def shade(base_color, roughness, normals, viewdirs, means, kind, vec, color, T):
    """viewdirs [V,P,3] -> (pbr, diffuse_light, specular), each [V,P,3].  Differentiable in every input but normals,
    T and kind."""
    normals = normals.detach()
    l, inv_r2, _ = light_dirs(kind, vec, means)                 # [P,K,3], [P,K]
    E = color[None] * inv_r2[..., None]                          # [P,K,3]
    ndi = (normals[:, None] * l).sum(-1, keepdim=True).clamp(min=0)
    transport = E * T.detach()[..., None] * ndi                  # [P,K,3]
    rough = roughness.reshape(-1, 1)
    outs = []
    for v in range(viewdirs.shape[0]):
        fs = ggx_specular(normals, viewdirs[v], l, rough)        # [P,K,1]
        outs.append((((base_color[:, None] / np.pi + fs) * transport).sum(1), transport.sum(1), (fs * transport).sum(1)))
    return tuple(torch.stack([o[k] for o in outs]) for k in range(3))


def shadows(means, inv_cov, opacity, normals, boxes, kind, vec, lone_leaf=False, pairs=None):
    """T [P,K] and fragile [P,K] of the fp32 inputs (numpy): the rays are built in fp32 exactly as the kernel does
    (op-by-op rounding), then traced in fp64.  pairs: the (g, j) rays to trace (default all; the others stay 1)."""
    m32 = np.asarray(means, np.float32)
    v32 = np.asarray(vec, np.float32).reshape(-1, 3)
    kind = np.asarray(kind).reshape(-1)
    P, K = m32.shape[0], kind.size
    mu = m32.astype(np.float64)
    ci = np.asarray(inv_cov, np.float64)
    op = np.asarray(opacity, np.float32).reshape(-1)
    nr = np.asarray(normals, np.float64)
    bx = np.asarray(boxes, np.float64)
    c0, c1, c2, c3, c4, c5 = (ci[:, k] for k in range(6))
    ci32 = np.float32(inv_cov)
    T_out, fragile = np.ones((P, K)), np.zeros((P, K), bool)
    f32 = np.float32
    for g, j in (pairs if pairs is not None else [(g, j) for g in range(P) for j in range(K)]):
        if True:
            w = v32[j] - m32[g] if kind[j] == 1 else v32[j].copy()
            r2 = f32(f32(f32(w[0] * w[0]) + f32(w[1] * w[1])) + f32(w[2] * w[2]))
            l = (w / max(f32(np.sqrt(r2)), f32(EPS))).astype(np.float32)
            o32 = (m32[g] + l * f32(0.05)).astype(np.float32)
            if kind[j] == 1:
                e = v32[j] - o32
                tmax_seg = float(f32(np.sqrt(f32(f32(f32(e[0] * e[0]) + f32(e[1] * e[1])) + f32(e[2] * e[2])))))
                t_hit = float(f32(f32(tmax_seg) * T_MAX_MARGIN))
            else:
                tmax_seg = t_hit = np.inf
            o, d = o32.astype(np.float64), l.astype(np.float64)
            if not d.any():
                continue                     # a light at the Gaussian's centre: no direction, no hit
            if lone_leaf:
                box_hit, box_edge = np.ones(P, bool), np.zeros(P, bool)
            else:
                tmin, tmx = ind._slab(bx, o, d)
                box_hit = (tmin <= tmx) & (tmx > 0) & (tmin <= tmax_seg)
                scale = np.abs(tmin) + np.abs(tmx) + 1e-3
                box_edge = (np.abs(tmx - tmin) < 1e-6 * scale) | (np.abs(tmx) < 1e-6 * scale)
                if np.isfinite(tmax_seg):
                    box_edge |= (np.abs(tmin - tmax_seg) < 1e-6 * (np.abs(tmin) + tmax_seg + 1e-3)) & (tmin <= tmx)
            nd = nr @ d
            mm = mu - o
            t1 = c0 * mm[:, 0] * d[0] + c1 * (mm[:, 0] * d[1] + mm[:, 1] * d[0]) + c2 * (mm[:, 0] * d[2] + mm[:, 2] * d[0]) + \
                c3 * mm[:, 1] * d[1] + c4 * (mm[:, 1] * d[2] + mm[:, 2] * d[1]) + c5 * mm[:, 2] * d[2]
            t2 = c0 * d[0] * d[0] + 2 * c1 * d[0] * d[1] + 2 * c2 * d[0] * d[2] + c3 * d[1] * d[1] + \
                2 * c4 * d[1] * d[2] + c5 * d[2] * d[2]
            with np.errstate(divide="ignore", invalid="ignore"):
                t = t1 / t2
                t_err = np.abs(ind._t_fp32(ci32, m32 - o32, l) - t)
            ee = mu - (o + t[:, None] * d)
            power = -0.5 * (ee[:, 0] ** 2 * c0 + ee[:, 1] ** 2 * c3 + ee[:, 2] ** 2 * c5 + 2 * ee[:, 0] * ee[:, 1] * c1 +
                            2 * ee[:, 0] * ee[:, 2] * c2 + 2 * ee[:, 1] * ee[:, 2] * c4)
            live = box_hit & (op >= ind.OP_MIN) & ~(nd > 0)
            hit = live & (t >= 0.01) & ~(power > 0) & (t < t_hit)
            near = (box_hit | box_edge) & (op >= ind.OP_MIN)
            fr = box_edge & (op >= ind.OP_MIN) & (t >= 0.0095) & ~(nd > 1e-6)
            fr |= near & (np.abs(nd) < 1e-6)
            fr |= near & ~(nd > 0) & (np.abs(t - 0.01) < 4 * t_err + 1e-8)
            if np.isfinite(tmax_seg):
                fr |= near & ~(nd > 0) & (np.abs(t - t_hit) < 4 * t_err + 4e-7 * t_hit + 1e-8)
            alpha = op[hit].astype(np.float64) * np.exp(power[hit])
            T = float(np.prod(1.0 - alpha))
            T_out[g, j], fragile[g, j] = T, bool(fr.any())
    return T_out, fragile


def shadows_match(T, T64, fragile):
    """Per ray: the kernel's T agrees with the truth (tolerance 1e-5 + 1e-4 T), or both are below the stop 1e-4 (the
    kernel reports the T it reached, in traversal order).  Rays whose product passes within 1e-3 of the stop at some
    order are not decidable and count as fragile."""
    ok = np.abs(T - T64) <= 1e-5 + 1e-4 * T64
    ok |= (T64 < T_MIN) & (T < T_MIN)
    return ok, fragile | (np.abs(T64 / T_MIN - 1) < 1e-3)

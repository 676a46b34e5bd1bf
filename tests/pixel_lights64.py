"""fp64 truth of the per-pixel lights (csrc/lights_trace.cu, csrc/pixel_lights.cu; include/r3dg_b200.h, PIXEL LIGHTS),
restated on the row oracles: every valid pixel p = y W + x of view v is one row of lights64 / shaped_lights64 with
mean = its point, the raw normal, viewdir = campos_v - point (fp32) and row index p for the rect samples.

Shadows: the rays start at the pixels' points, not at Gaussian means.  The row oracles trace from their own rows, so
the points are appended to the scene as extra rows of zero opacity (never a hit, never fragile) and traced from there;
a rect's targets are hashed with the pixel's index p, not with that row."""
import numpy as np
import torch

import lights64 as L64
import shaped_lights64 as S64

D = torch.float64


def rows(img):
    """[C,H,W] -> [HW,C]."""
    return img.reshape(img.shape[0], -1).T


def columns(kind, M):
    """R and the light family of a set: (R, shaped)."""
    kind = [int(k) for k in kind]
    shaped = len(kind) > 0 and kind[0] in (S64.SPOT, S64.RECT)
    return (len(S64.columns(kind, M)) if shaped else len(kind)), shaped


def shade_pixels(base_color, roughness, normal, points, campos, T, kind, fields, M=1, seed=0, mask=None):
    """dict(pbr, diffuse_light, specular) [V,3,H,W] in fp64 for images [V,C,H,W], campos [V,3], T [V,R,H,W] and the
    set's fields (vec, color) or (pos, a, b, color, cone).  Differentiable in base_color, roughness and the fields."""
    V, _, H, W = base_color.shape
    R, shaped = columns(kind, M)
    out = {k: [] for k in ("pbr", "diffuse_light", "specular")}
    st = None
    if shaped:
        pos, a, b = (np.asarray(f.detach().cpu(), np.float32) for f in fields[:3])
        _, st = S64.ray_targets(list(kind), pos, a, b, M, seed, H * W)
    for v in range(V):
        pts = rows(points[v]).float()
        vd = (campos[v].float()[None] - pts).to(D)[None]             # one fp32 subtraction per component
        args = (rows(base_color[v]).to(D), rows(roughness[v]).to(D), rows(normal[v]).to(D), vd, pts.to(D), kind)
        Tv = rows(T[v]).to(D)
        if shaped:
            pbr, diff, spec = S64.shade(*args, *[f.to(D) for f in fields], Tv, M, st)
        else:
            pbr, diff, spec = L64.shade(*args, *[f.to(D) for f in fields], Tv)
        keep = torch.ones(H * W, dtype=torch.bool) if mask is None else mask[v].reshape(-1).cpu()
        for k, x in (("pbr", pbr), ("diffuse_light", diff), ("specular", spec)):
            out[k].append(torch.where(keep[:, None], x[0], torch.zeros_like(x[0])).T.reshape(3, H, W))
    return {k: torch.stack(x) for k, x in out.items()}


def shadows(points, means, inv_cov, opacity, normals, boxes, kind, fields, M, seed, pixels):
    """T [V,R,H,W] and fragile [V,R,H,W] (numpy) of the rays of `pixels` [(v, p)] (the others stay 1): the row oracles'
    rays from each pixel's point, through the P Gaussians (means, inv_cov, opacity, normals, leaf boxes)."""
    points = np.asarray(points, np.float32)
    V, _, H, W = points.shape
    R, shaped = columns(kind, M)
    P = means.shape[0]
    T, fr = np.ones((V, R, H * W)), np.zeros((V, R, H * W), bool)
    pts = points.reshape(V, 3, H * W)
    for v, p in pixels:
        m = np.concatenate([means, pts[v, :, p][None]]).astype(np.float32)
        ci = np.concatenate([inv_cov, np.asarray([[1, 0, 0, 1, 0, 1]], np.float32)])
        op = np.concatenate([opacity, [0.0]]).astype(np.float32)
        nr = np.concatenate([normals, [[0.0, 0.0, 1.0]]]).astype(np.float32)
        bx = np.concatenate([boxes, np.tile(pts[v, :, p], 2)[None]]).astype(np.float32)
        if shaped:
            pos, a, b = (np.asarray(f, np.float32) for f in fields[:3])
            tg, _ = S64.ray_targets(list(kind), pos, a, b, M, seed, p + 1, [p])
            Tp, fp = L64.shadows(m, ci, op, nr, bx, np.ones(R, np.int32), tg[p], pairs=[(P, c) for c in range(R)])
        else:
            Tp, fp = L64.shadows(m, ci, op, nr, bx, np.asarray(kind), np.asarray(fields[0], np.float32),
                                 pairs=[(P, c) for c in range(R)])
        T[v, :, p], fr[v, :, p] = Tp[P], fp[P]
    return T.reshape(V, R, H, W), fr.reshape(V, R, H, W)

"""fp64 restatement of Mip-Splatting's 3D filter as the library computes it (relightable3dgaussian_b200/filter3d.py,
csrc/filter3d.cu, the F3D path of csrc/projection.cu and csrc/projection_bwd.cu).

compute(means, views, intr, F): per (Gaussian, camera) pair the view-space position t = [m, 1] V, the pixel position
u = t.x / z fx + cx, v = t.y / z fy + cy, the valid test (z > 0.2 and u, v within 15 % of the image) and its distance
to the nearest boundary in units of that quantity's rounding scale; then d, and f = d / F sqrt(0.2).

dilate(s, o, f): s' = sqrt(s^2 + f^2) and coef = prod_k |s_k| / s'_k, differentiable (torch fp64 autograd);
coef_det(s, f): Mip-Splatting's sqrt(det1 / det2) form of the same coefficient; chain(...): dL/ds and dL/do from the
gradients of the filtered Gaussian."""
import torch

EPS32 = 2.0 ** -24


def compute(means, views, intr, F, chunk=20_000):
    """means [P,3], views [V,16] (the rasterizer's viewmatrix layout), intr [V,6] {fx, fy, cx, cy, W, H}, F: fp64
    tensors / float.  Returns (f [P], seen [P] bool, margin [P], cond [P]).  margin is the smallest distance, over the
    row's cameras, of z, u or v to its bound relative to that quantity's fp32 rounding scale (the sum of the magnitudes
    of its terms times eps32): a row with margin <= ~16 may be decided either way by fp32 rounding.  cond is the
    conditioning of the row's own least depth (sum of term magnitudes / |z|).  Rows are processed `chunk` at a time."""
    means, views, intr = means.double(), views.double(), intr.double()
    P, V = means.shape[0], views.shape[0]
    M = views.reshape(V, 4, 4)                           # row j is the j-th [m,1] coefficient: t_k = sum_j h_j M[j, k]
    fx, fy, cx, cy, W, H = (intr[:, k][None, :] for k in range(6))
    f32 = lambda x: torch.tensor(x.numpy(), dtype=torch.float32).double()
    lo_x, hi_x, lo_y, hi_y = f32(-0.15 * W), f32(W * 1.15), f32(-0.15 * H), f32(1.15 * H)
    zb = float(torch.tensor(0.2, dtype=torch.float32))
    ds, margins, conds = [], [], []
    for r0 in range(0, P, chunk):
        m = means[r0:r0 + chunk]
        h = torch.cat([m, torch.ones(m.shape[0], 1, dtype=torch.float64)], 1)
        t = torch.einsum("pj,vjk->pvk", h, M)
        ts = torch.einsum("pj,vjk->pvk", h.abs(), M.abs())
        x, y, z = t[..., 0], t[..., 1], t[..., 2]
        u = x / z * fx + cx
        v = y / z * fy + cy
        zs = ts[..., 2] * EPS32
        us = (ts[..., 0] / z.abs() + ts[..., 2] * x.abs() / z ** 2) * fx * EPS32 + u.abs() * EPS32
        vs = (ts[..., 1] / z.abs() + ts[..., 2] * y.abs() / z ** 2) * fy * EPS32 + v.abs() * EPS32
        valid = (z > zb) & (u >= lo_x) & (u <= hi_x) & (v >= lo_y) & (v <= hi_y)
        inf = torch.full_like(z, float("inf"))
        mz = (z - zb).abs() / zs.clamp_min(1e-300)
        front = z > 0.1                                  # u, v matter only in front of the camera
        mu = torch.where(front, torch.minimum((u - lo_x).abs(), (u - hi_x).abs()) / us.clamp_min(1e-300), inf)
        mv = torch.where(front, torch.minimum((v - lo_y).abs(), (v - hi_y).abs()) / vs.clamp_min(1e-300), inf)
        margin = torch.minimum(mz, torch.minimum(torch.nan_to_num(mu, nan=0.0), torch.nan_to_num(mv, nan=0.0)))
        zv = torch.where(valid, z, inf)
        d, arg = zv.min(1)
        ds.append(d)
        margins.append(margin.min(1).values)
        conds.append(torch.gather(ts[..., 2] / z.abs(), 1, arg[:, None])[:, 0])
    d, margin, cond = torch.cat(ds), torch.cat(margins), torch.cat(conds)
    seen = torch.isfinite(d)
    cond = torch.where(seen, cond, torch.ones_like(cond))
    if bool(seen.any()):
        d = torch.where(seen, d, d[seen].max())
        f = d / F * (0.2 ** 0.5)
    else:
        f = torch.zeros(P, dtype=torch.float64)
    return f, seen, margin, cond


def dilate(s, o, f):
    """(s', o', coef) in fp64: s' = sqrt(s^2 + f^2), coef = prod_k |s_k| / s'_k (1 for an axis with s' = 0)."""
    g = (f.reshape(-1, 1) ** 2)
    sp = torch.sqrt(s * s + g)
    ratio = torch.where(sp > 0, s.abs() / torch.where(sp > 0, sp, torch.ones_like(sp)), torch.ones_like(sp))
    coef = ratio.prod(1)
    return sp, o.reshape(-1) * coef, coef


def coef_det(s, f):
    """Mip-Splatting's form: sqrt(det(S^2) / det(S^2 + f^2 I)) = sqrt(prod s^2 / prod (s^2 + f^2))."""
    g = (f.reshape(-1, 1) ** 2)
    return torch.sqrt((s * s).prod(1) / (s * s + g).prod(1))


def dcoef(s, f):
    """d coef / d s_k in the cancellation-free form (prod_{j != k} |s_j| / s'_j) sign(s_k) (g / e_k) / s'_k, fp64."""
    g = (f.reshape(-1, 1) ** 2)
    e = s * s + g
    sp = torch.sqrt(e)
    pos = sp > 0
    safe = torch.where(pos, sp, torch.ones_like(sp))
    a = torch.where(pos, s.abs() / safe, torch.ones_like(sp))
    h = torch.where(pos, torch.sign(s) * (g / torch.where(pos, e, torch.ones_like(e))) / safe, torch.zeros_like(sp))
    h = torch.where(pos & (s == 0), g / torch.where(pos, e, torch.ones_like(e)) / safe, h)   # sign(0) -> +
    other = torch.stack([a[:, 1] * a[:, 2], a[:, 0] * a[:, 2], a[:, 0] * a[:, 1]], 1)
    return other * h


def chain(s, o, f, g_sp, g_op):
    """dL/ds and dL/do from dL/ds' and dL/do' (the gradients of the filtered Gaussian), fp64; and the per-entry
    magnitude |dL/ds' s/s'| + |o dL/do' dcoef/ds| the rounding of dL/ds scales with."""
    s, o, f, g_sp, g_op = (t.double() for t in (s, o, f, g_sp, g_op))
    sp, _, coef = dilate(s, o, f)
    ratio = torch.where(sp > 0, s / torch.where(sp > 0, sp, torch.ones_like(sp)), torch.ones_like(sp))
    t1 = g_sp * ratio
    t2 = (o.reshape(-1, 1) * g_op.reshape(-1, 1)) * dcoef(s, f)
    return t1 + t2, coef * g_op.reshape(-1), t1.abs() + t2.abs()

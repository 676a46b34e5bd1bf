"""fp64 NumPy truth of the radiance bake and the incident-SH fit (csrc/indirect.cu).

Brute force: every ray tests every Gaussian whose leaf box it hits with the visibility trace's hit rule, sorts the hits
by (t, Gaussian index) and composites them front to back until T < 1e-4.  Alongside the result each ray gets a
`fragile` flag: some input sits within fp32 rounding of a decision (box graze, t = 0.01, back-face, opacity 1/255, a t
tie, the T < 1e-4 stop), so the fp32 kernel may legitimately decide it the other way."""
import numpy as np

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)
T_MIN = 1e-4
OP_MIN = np.float32(1.0) / np.float32(255.0)


def sh_basis(deg, v):
    """Real SH basis [..., (deg+1)^2] of unit vectors v [..., 3] (utils/sh_utils.py eval_sh), fp64."""
    x, y, z = (np.asarray(v, np.float64)[..., k] for k in range(3))
    w = [np.full_like(x, C0)]
    if deg > 0:
        w += [-C1 * y, C1 * z, -C1 * x]
    if deg > 1:
        xx, yy, zz = x * x, y * y, z * z
        w += [C2[0] * x * y, C2[1] * y * z, C2[2] * (2 * zz - xx - yy), C2[3] * x * z, C2[4] * (xx - yy)]
    if deg > 2:
        w += [C3[0] * y * (3 * xx - yy), C3[1] * x * y * z, C3[2] * y * (4 * zz - xx - yy),
              C3[3] * z * (2 * zz - 3 * xx - 3 * yy), C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy),
              C3[6] * x * (xx - 3 * yy)]
    return np.stack(w, axis=-1)


def bake_origins(means, dirs, offset=0.05):
    """The kernel's fp32 ray origins mean + offset * d (two separately rounded fp32 ops)."""
    return (np.float32(means)[:, None, :] + np.float32(dirs) * np.float32(offset)).astype(np.float32)


def _t_fp32(ci, m, d):
    """The peak t of every Gaussian in plain fp32 arithmetic: its distance to the fp64 t estimates the kernel's
    rounding error (which contracts to FMAs, so it is not bit-equal to this)."""
    c0, c1, c2, c3, c4, c5 = (ci[:, k] for k in range(6))
    t1 = c0 * m[:, 0] * d[0] + c1 * m[:, 0] * d[1] + c2 * m[:, 0] * d[2] + c1 * m[:, 1] * d[0] + c3 * m[:, 1] * d[1] + \
        c4 * m[:, 1] * d[2] + c2 * m[:, 2] * d[0] + c4 * m[:, 2] * d[1] + c5 * m[:, 2] * d[2]
    t2 = c0 * d[0] * d[0] + c1 * d[0] * d[1] + c2 * d[0] * d[2] + c1 * d[1] * d[0] + c3 * d[1] * d[1] + \
        c4 * d[1] * d[2] + c2 * d[2] * d[0] + c4 * d[2] * d[1] + c5 * d[2] * d[2]
    return (t1 / t2).astype(np.float64)


def _slab(boxes, o, d):
    """fp64 slab test of every box against one ray: (tmin, tmax); a miss has tmin > tmax."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t0 = (boxes[:, :3] - o) * inv
        t1 = (boxes[:, 3:] - o) * inv
    lo, hi = np.minimum(t0, t1), np.maximum(t0, t1)
    return np.nanmax(lo, axis=1), np.nanmin(hi, axis=1)


def bake_radiance(means, inv_cov, opacity, normals, shs, deg, boxes, origins, dirs, lone_leaf=False):
    """Radiance bake of rays (origins [R,3], dirs [R,3]) through Gaussians (means [P,3], inverse covariances [P,6],
    opacity [P], normals [P,3], payload shs [P,M,3] of degree deg, leaf boxes [P,6] = lo3, hi3).  `lone_leaf`: a
    one-Gaussian tree has no box test (its root is the leaf).  Returns (radiance [R,3], T [R], hits [R], fragile [R])."""
    mu = np.asarray(means, np.float64)
    ci = np.asarray(inv_cov, np.float64)
    op = np.asarray(opacity, np.float32).reshape(-1)
    nr = np.asarray(normals, np.float64)
    sh = np.asarray(shs, np.float64)
    bx = np.asarray(boxes, np.float64)
    P, n = mu.shape[0], (deg + 1) ** 2
    R = origins.shape[0]
    rad, T_out, hits_out, fragile = np.zeros((R, 3)), np.ones(R), np.zeros(R, np.int64), np.zeros(R, bool)
    if P == 0:
        return rad, T_out, hits_out, fragile
    c0, c1, c2, c3, c4, c5 = (ci[:, k] for k in range(6))
    ci32, mu32 = np.float32(inv_cov), np.float32(means)
    for r in range(R):
        o, d = np.asarray(origins[r], np.float64), np.asarray(dirs[r], np.float64)
        if lone_leaf:
            box_hit, box_edge = np.ones(P, bool), np.zeros(P, bool)
        else:
            tmin, tmax = _slab(bx, o, d)
            box_hit = (tmin <= tmax) & (tmax > 0)
            scale = np.abs(tmin) + np.abs(tmax) + 1e-3
            box_edge = (np.abs(tmax - tmin) < 1e-6 * scale) | (np.abs(tmax) < 1e-6 * scale)
        nd = nr @ d
        m = mu - o
        t1 = c0 * m[:, 0] * d[0] + c1 * (m[:, 0] * d[1] + m[:, 1] * d[0]) + c2 * (m[:, 0] * d[2] + m[:, 2] * d[0]) + \
            c3 * m[:, 1] * d[1] + c4 * (m[:, 1] * d[2] + m[:, 2] * d[1]) + c5 * m[:, 2] * d[2]
        t2 = c0 * d[0] * d[0] + 2 * c1 * d[0] * d[1] + 2 * c2 * d[0] * d[2] + c3 * d[1] * d[1] + \
            2 * c4 * d[1] * d[2] + c5 * d[2] * d[2]
        with np.errstate(divide="ignore", invalid="ignore"):
            t = t1 / t2
            t_err = np.abs(_t_fp32(ci32[:, :], mu32 - np.float32(origins[r]), np.float32(dirs[r])) - t)
        e = mu - (o + t[:, None] * d)
        power = -0.5 * (e[:, 0] ** 2 * c0 + e[:, 1] ** 2 * c3 + e[:, 2] ** 2 * c5 + 2 * e[:, 0] * e[:, 1] * c1 +
                        2 * e[:, 0] * e[:, 2] * c2 + 2 * e[:, 1] * e[:, 2] * c4)
        live = box_hit & (op >= OP_MIN) & ~(nd > 0)
        hit = live & (t >= 0.01) & ~(power > 0)
        # decisions within fp32 rounding of their threshold, on Gaussians that matter (box hit or grazed)
        near = (box_hit | box_edge) & (op >= OP_MIN)
        fr = box_edge & (op >= OP_MIN) & (t >= 0.0095) & ~(nd > 1e-6)
        fr |= near & (np.abs(nd) < 1e-6)
        fr |= near & ~(nd > 0) & (np.abs(t - 0.01) < 4 * t_err + 1e-8)
        idx = np.nonzero(hit)[0]
        order = idx[np.lexsort((idx, t[idx]))]
        ts = t[order]
        te = 4 * t_err[order] + 2e-7 * ts                 # fp32 error bound of each hit's t
        flag = fr.any() or (len(ts) > 1 and (np.diff(ts) <= te[1:] + te[:-1]).any())
        L, T, h = np.zeros(3), 1.0, 0
        for g in order:
            alpha = float(op[g]) * np.exp(power[g])
            v = mu[g] - o
            v = v / np.linalg.norm(v)
            c = np.maximum(sh_basis(deg, v) @ sh[g, :n] + 0.5, 0.0)
            L += T * alpha * c
            T *= 1 - alpha
            h += 1
            if abs(T / T_MIN - 1) < 1e-3:
                flag = True
            if T < T_MIN:
                break
        rad[r], T_out[r], hits_out[r], fragile[r] = L, T, h, flag
    return rad, T_out, hits_out, fragile


def fit_incident_sh(radiance, dirs, deg, ridge):
    """Per Gaussian: argmin_c (1/N) sum_i |Y(w_i)^T c - L_i|^2 + ridge |c|^2 (numpy.linalg.solve of the normal
    equations).  radiance [P,N,3], dirs [P,N,3] -> [P,(deg+1)^2,3]."""
    L = np.asarray(radiance, np.float64)
    Y = sh_basis(deg, dirs)                              # [P,N,n]
    N, n = L.shape[1], Y.shape[-1]
    G = np.einsum("pik,pil->pkl", Y, Y) / N + ridge * np.eye(n)
    b = np.einsum("pik,pic->pkc", Y, L) / N
    return np.linalg.solve(G, b)


def fit_residual(radiance, dirs, coeffs):
    """Relative RMS error of the fitted local light sum_k Y_k c_k against the radiance it was fitted to."""
    Y = sh_basis(int(round(np.sqrt(coeffs.shape[1]))) - 1, dirs)
    pred = np.einsum("pik,pkc->pic", Y, np.asarray(coeffs, np.float64))
    L = np.asarray(radiance, np.float64)
    return float(np.sqrt(((pred - L) ** 2).sum() / max((L ** 2).sum(), 1e-30)))

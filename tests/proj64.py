"""fp64 truth of the projection backward (csrc/projection_bwd.cu): the leaf gradients of one Gaussian from its record's.

The projection turns each Gaussian's leaves (means3D, scales, rotations, opacity and SH, or cov3D_precomp /
colors_precomp) and one camera into the record the compositors read.  record() restates that map in fp64 per
Gaussian, with these outputs (REC):
  ndc x, ndc y   the projected mean in the units of the compositor's dL_dmeans2D (0.5 W and 0.5 H per pixel)
  depth          the view-space z
  conic a, b, c  the inverse of cov2D + 0.3 I (b: the true derivative, twice the reference's dL_dconic.y)
  opacity        o, o rho (antialiased), o coef (3D filter) or o coef rho
  r, g, b        the colour; SH colours with the forward's clamp flags taken as given

The truth is the reference's BACKWARD DEFINITION, which departs from the derivative of its forward in three places:
  * frustum clamp: with t0 = clamp(tx / tz, +-1.3 tan fov) tz, the reference zeroes dL/dtx of a clamped row but keeps
    2 h_x t0 tz^-3 dL/dJ02 in dL/dtz.  That is autograd of J02 = -h_x t0 / tz^2 with t0 = (L tz).detach() where the row
    is clamped (tx where not): for clamped rows twice the true tz-derivative of that term.  Parity with the reference
    is the specification; the kernel must not be "fixed" towards plain autograd.
  * conic inverse: differentiated with 1 / (denom^2 + 1e-7) in place of 1 / denom^2 (linearised here: value N / D,
    derivative (dN D - N dD) / (D^2 + 1e-7));
  * projected mean: ndc = h / (w + 1e-7).
and it keeps two conventions: dL_dscales is dL/d(s scale_modifier) (the chain omits the modifier's factor), and the
quaternion is used as given, not normalised.

leaf_truth() restates record() as a chain of stages whose Jacobian entries are single products (_stages), forms each
stage's per-Gaussian fp64 Jacobian (torch.func.jacrev under vmap, in chunks) and returns, for every leaf,
g64 = J^T g_rec (J the chain's product: the Jacobian of record()) and m_row = |J_1|^T ... |J_n|^T m_rec, where
(g_rec, m_rec) are the signed and magnitude sums of the record's gradient (raster64.row_truth).  So every sum the
backward forms counts with the magnitudes of its terms, not of the sum: the SH colour's derivative in the mean per
coefficient (a colour flat in the view direction), the conic's 1/det - a c / det^2, the basis values' x^2 - y^2,
the view direction's |d|^2 - d_x^2.  Otherwise a row whose sum cancels gets a bound below the kernel's own rounding.

ambiguous_rows() names the rows whose fp32 decisions or conditioning the comparison cannot judge."""
import torch
from torch.func import jacrev, vmap

import aa_oracle
import filter3d_oracle

REC = ("ndc_x", "ndc_y", "depth", "conic_a", "conic_b", "conic_c", "opacity", "r", "g", "b")
EPS_CONIC = 1e-7
EPS_W = 1e-7
SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def sh_basis(D, d):
    """The real SH basis [16] at the unit direction d (zero above (D + 1)^2), the reference's constants and signs."""
    x, y, z = d[0], d[1], d[2]
    w = [torch.ones_like(x) * SH_C0]
    if D > 0:
        w += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if D > 1:
        xx, yy, zz = x * x, y * y, z * z
        w += [SH_C2[0] * x * y, SH_C2[1] * y * z, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * x * z, SH_C2[4] * (xx - yy)]
    if D > 2:
        xx, yy, zz = x * x, y * y, z * z
        w += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * x * y * z, SH_C3[2] * y * (4 * zz - xx - yy),
              SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * z * (xx - yy),
              SH_C3[6] * x * (xx - 3 * yy)]
    w += [torch.zeros_like(x)] * (16 - len(w))
    return torch.stack(w)


MONOMIALS = ("x", "y", "z", "xx", "yy", "zz", "xy", "yz", "xz", "xxy", "yyy", "xyz", "yzz", "zzz", "xxz", "yyz", "xzz",
             "xxx", "xyy")
NMON = len(MONOMIALS)
# the basis as sums of (constant, monomial) terms (sh_basis with its products expanded)
SH_TERMS = [[(SH_C0, None)], [(-SH_C1, "y")], [(SH_C1, "z")], [(-SH_C1, "x")],
            [(SH_C2[0], "xy")], [(SH_C2[1], "yz")], [(2 * SH_C2[2], "zz"), (-SH_C2[2], "xx"), (-SH_C2[2], "yy")],
            [(SH_C2[3], "xz")], [(SH_C2[4], "xx"), (-SH_C2[4], "yy")],
            [(3 * SH_C3[0], "xxy"), (-SH_C3[0], "yyy")], [(SH_C3[1], "xyz")],
            [(4 * SH_C3[2], "yzz"), (-SH_C3[2], "xxy"), (-SH_C3[2], "yyy")],
            [(2 * SH_C3[3], "zzz"), (-3 * SH_C3[3], "xxz"), (-3 * SH_C3[3], "yyz")],
            [(4 * SH_C3[4], "xzz"), (-SH_C3[4], "xxx"), (-SH_C3[4], "xyy")], [(SH_C3[5], "xxz"), (-SH_C3[5], "yyz")],
            [(SH_C3[6], "xxx"), (-3 * SH_C3[6], "xyy")]]


def monomials(d):
    """The monomials of the unit direction d that the basis up to degree 3 is made of (MONOMIALS)."""
    v = {"x": d[0], "y": d[1], "z": d[2]}
    return torch.stack([torch.stack([v[c] for c in name]).prod() for name in MONOMIALS])


def sh_from_monomials(D, mon, magnitude=False):
    """sh_basis from the monomials [NMON] (zero above (D + 1)^2); `magnitude`: the sum of each value's terms'
    magnitudes instead."""
    at = {n: mon[i] for i, n in enumerate(MONOMIALS)}
    out = []
    for k, terms in enumerate(SH_TERMS):
        if k >= (D + 1) ** 2:
            out.append(torch.zeros_like(mon[0]))
            continue
        vals = [c * (at[n] if n else torch.ones_like(mon[0])) for c, n in terms]
        out.append(sum(v.abs() for v in vals) if magnitude else sum(vals))
    return torch.stack(out)


class Camera:
    """One view in fp64: viewmatrix / projmatrix [4,4] in the rasterizer's layout (t = [m,1] V), campos [3]."""

    def __init__(self, viewmatrix, projmatrix, campos, W, H, tan_fovx, tan_fovy, scale_modifier=1.0):
        f64 = lambda t: torch.as_tensor(t).double().reshape(-1)                          # noqa: E731
        self.V, self.P = f64(viewmatrix).view(4, 4), f64(projmatrix).view(4, 4)
        self.campos = f64(campos)
        self.W, self.H, self.tanfovx, self.tanfovy = W, H, float(tan_fovx), float(tan_fovy)
        self.mod = float(scale_modifier)

    def to(self, dev):
        self.V, self.P, self.campos = self.V.to(dev), self.P.to(dev), self.campos.to(dev)
        return self


def _clamp_t(t, tz, L):
    """t0 of the reference's backward: the clamped t as a constant on clamped rows (see the module notes)."""
    r = t / tz
    return torch.where(r.abs() > L, (r.clamp(-L, L) * tz).detach(), t)


def cov2d(m, sigma, cam):
    """(a0, b, c0, tz) of one Gaussian: T Sigma T^T before the 0.3 px^2 dilation, with the reference's J."""
    t = m @ cam.V[:3, :3] + cam.V[3, :3]
    tx, ty, tz = t[0], t[1], t[2]
    hx, hy = cam.W / (2.0 * cam.tanfovx), cam.H / (2.0 * cam.tanfovy)
    t0x = _clamp_t(tx, tz, 1.3 * cam.tanfovx)
    t0y = _clamp_t(ty, tz, 1.3 * cam.tanfovy)
    zero = torch.zeros_like(tz)
    J = torch.stack([hx / tz, zero, -hx * t0x / (tz * tz), zero, hy / tz, -hy * t0y / (tz * tz)]).view(2, 3)
    T = J @ cam.V[:3, :3].T
    C = T @ sigma @ T.T
    return C[0, 0], C[0, 1], C[1, 1], tz


def _lin_div(n, d):
    """n / d with the reference's derivative (dn d - n dd) / (d^2 + 1e-7) (first order only)."""
    n0, d0 = n.detach(), d.detach()
    return n0 / d0 + (n * d0 - n0 * d) / (d0 * d0 + EPS_CONIC)


def _modified(x, mod):
    """mod x in value, with the derivative of x: dL/d(mod x) is what the kernel reports as dL/dx."""
    return x + (mod - 1.0) * x.detach()


def record(leaves, const, cam, D, aa=False, f3d=False):
    """The record of ONE Gaussian ([10], REC) and, with SH, its colour's per-coefficient terms [16, 3] (the colour is
    0.5 + their sum over k, times the clamp gates).  leaves: means3D [3], opacities [1], scales [3] + rotations [4] or
    cov3D [6], shs [M,3] or colors [3].  const: clamped [3] (0 / 1), filter_3d [] (f3d)."""
    m = leaves["means3D"]
    o = leaves["opacities"].reshape(())
    if "cov3D" in leaves:
        sigma = aa_oracle.cov3d_from_six(leaves["cov3D"][None])[0]
    else:
        s = leaves["scales"]
        if f3d:
            sp, _, coef = filter3d_oracle.dilate(s[None], o.reshape(1), const["filter_3d"].reshape(1))
            s, o = sp[0], o * coef[0]
        sc = _modified(s, cam.mod)
        sigma = aa_oracle.cov3d_of(sc[None], leaves["rotations"][None])[0]
    a0, b, c0, tz = cov2d(m, sigma, cam)
    a, c = a0 + aa_oracle.DILATION, c0 + aa_oracle.DILATION
    det = a * c - b * b
    conic = [_lin_div(c, det), _lin_div(-b, det), _lin_div(a, det)]
    if aa:
        o = o * aa_oracle.rho_of_cov2d(a0, b, c0)
    h = m @ cam.P[:3, :] + cam.P[3, :]
    ndc = h[:2] / (h[3] + EPS_W)
    if "shs" in leaves:
        d = m - cam.campos
        d = d / torch.sqrt((d * d).sum())
        M = leaves["shs"].shape[0]
        gate = 1.0 - const["clamped"]
        terms = sh_basis(D, d)[:M, None] * leaves["shs"] * gate
        col = 0.5 * gate + terms.sum(0)
    else:
        terms, col = None, leaves["colors"]
    rec = torch.cat([ndc, tz[None], torch.stack(conic), o[None], col])
    return rec, terms


def _rotation(q):
    """R(q) [3,3] of the unnormalised quaternion (r, x, y, z), aa_oracle.cov3d_of's layout."""
    r, x, y, z = q[0], q[1], q[2], q[3]
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]).view(3, 3)


def _sym6(S):
    return torch.stack([S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2]])


def _stages(names, sizes, cam, D, aa, f3d):
    """record() as a chain of stages, each a map of flat per-Gaussian vectors whose Jacobian entries are single
    products (no sum of terms that can cancel inside one entry): leaves -> (t, m, o, M = R diag(s) or cov6,
    appearance) -> (T, Sigma, ndc, depth, o, colour terms) -> (T, V = Sigma T^T, ...) -> (a0, b, c0, ...) ->
    (a, b, c, det, o rho, colour) -> record.  The product of their absolute Jacobians bounds the rounding of a kernel
    that evaluates the same chain (leaf_truth)."""
    offs = {}
    o0 = 0
    for n, k in zip(names, sizes):
        offs[n] = slice(o0, o0 + k)
        o0 += k
    sh = "shs" in offs
    cov = "cov3D" in offs
    Vm = cam.V

    def A(x, cs):
        m, o = x[offs["means3D"]], x[offs["opacities"]]
        t = m @ Vm[:3, :3] + Vm[3, :3]
        if cov:
            Mm = x[offs["cov3D"]]
        else:
            s = x[offs["scales"]]
            if f3d:
                sp, _, coef = filter3d_oracle.dilate(s[None], o, cs["filter_3d"].reshape(1))
                s, o = sp[0], o * coef
            Mm = (_rotation(x[offs["rotations"]]) * _modified(s, cam.mod)[None, :]).reshape(9)
        app = x[offs["shs"]] if sh else x[offs["colors"]]
        return torch.cat([t, m, o, Mm, app])

    nM = 6 if cov else 9

    def B(y, cs):
        t, m, o, Mm, app = y[:3], y[3:6], y[6:7], y[7:7 + nM], y[7 + nM:]
        if cov:
            S6 = Mm
        else:
            Mq = Mm.view(3, 3)
            S6 = _sym6(Mq @ Mq.T)
        hx, hy = cam.W / (2.0 * cam.tanfovx), cam.H / (2.0 * cam.tanfovy)
        tx, ty, tz = t[0], t[1], t[2]
        t0x = _clamp_t(tx, tz, 1.3 * cam.tanfovx)
        t0y = _clamp_t(ty, tz, 1.3 * cam.tanfovy)
        zero = torch.zeros_like(tz)
        J = torch.stack([hx / tz, zero, -hx * t0x / (tz * tz), zero, hy / tz, -hy * t0y / (tz * tz)]).view(2, 3)
        T = (J @ Vm[:3, :3].T).reshape(6)
        h = m @ cam.P[:3, :] + cam.P[3, :]
        ndc = h[:2] / (h[3] + EPS_W)
        if sh:
            d = m - cam.campos
            return torch.cat([T, S6, ndc, tz[None], o, d, (d * d).sum()[None], app])
        return torch.cat([T, S6, ndc, tz[None], o, app])

    # SH colour (with shs): the view direction d / |d|, its monomials, then the colour terms w_k(monomials) sh_k
    def B2(y, cs):
        head, d, s2, app = y[:16], y[16:19], y[19], y[20:]
        return torch.cat([head, d / torch.sqrt(s2), app])

    def B3(y, cs):
        head, d, app = y[:16], y[16:19], y[19:]
        return torch.cat([head, monomials(d), app])

    def B4(y, cs):
        head, mon, app = y[:16], y[16:16 + NMON], y[16 + NMON:]
        shs = app.view(-1, 3)
        col = (sh_from_monomials(D, mon)[:shs.shape[0], None] * shs * (1.0 - cs["clamped"])).reshape(-1)
        return torch.cat([head, col])

    def C(z, cs):
        T, S6, rest = z[:6].view(2, 3), z[6:12], z[12:]
        Sg = aa_oracle.cov3d_from_six(S6[None])[0]
        VT = (Sg @ T.T).reshape(6)
        return torch.cat([T.reshape(6), VT, rest])

    def Dst(z, cs):
        T, VT, rest = z[:6].view(2, 3), z[6:12].view(3, 2), z[12:]
        a0, b, c0 = T[0] @ VT[:, 0], T[1] @ VT[:, 0], T[1] @ VT[:, 1]
        return torch.cat([torch.stack([a0, b, c0]), rest])

    def E(z, cs):
        a0, b, c0 = z[0], z[1], z[2]
        ndc, depth, o, col = z[3:5], z[5:6], z[6:7], z[7:]
        a, c = a0 + aa_oracle.DILATION, c0 + aa_oracle.DILATION
        det = a * c - b * b
        if aa:
            o = o * aa_oracle.rho_of_cov2d(a0, b, c0)
        if sh:
            col = 0.5 * (1.0 - cs["clamped"]) + col.view(-1, 3).sum(0)
        return torch.cat([ndc, depth, torch.stack([a, b, c, det]), o, col])

    def F(z, cs):
        ndc, depth, a, b, c, det, o, col = z[0:2], z[2:3], z[3], z[4], z[5], z[6], z[7:8], z[8:11]
        conic = torch.stack([_lin_div(c, det), _lin_div(-b, det), _lin_div(a, det)])
        return torch.cat([ndc, depth, conic, o, col])

    return offs, ([A, B, B2, B3, B4] if sh else [A, B]) + [C, Dst, E, F]


def leaf_truth(leaves, const, cam, D, g_rec, m_rec, aa=False, f3d=False, chunk=4096):
    """{leaf: (g64 [P,*], m_row [P,*])} for leaves {name: [P,*] tensors} (made fp64 here), the per-row constants
    `const` {name: [P,*]} and the record's signed / magnitude gradient sums g_rec, m_rec [P,10] (REC order).
    g64 = J^T g_rec with J the Jacobian of record() (the stages of _stages chained); m_row = |J_1|^T ... |J_6|^T m_rec
    over the stages' Jacobians, so that every term the chain sums counts with its magnitude (the SH colour's
    derivative in the mean per coefficient, the conic's 1/det - a c / det^2 per term, ...)."""
    names = list(leaves)
    P = g_rec.shape[0]
    X = torch.cat([leaves[k].double().reshape(P, -1) for k in names], 1)
    sizes = [leaves[k].reshape(P, -1).shape[1] for k in names]
    const = {k: v.double() for k, v in const.items()}
    offs, stages = _stages(names, sizes, cam, D, aa, f3d)
    jacs = [vmap(jacrev(f)) for f in stages]
    g_out, m_out = [], []
    for r0 in range(0, P, chunk):
        sl = slice(r0, min(P, r0 + chunk))
        x = X[sl]
        cs = {k: v[sl] for k, v in const.items()}
        Js = []
        for f, jf in zip(stages, jacs):
            J = jf(x, cs)
            A = J.abs()
            if f.__name__ == "B4":
                # d(w_k sh_kc) / d(sh_kc) is the basis value w_k, itself a sum of monomial terms that can cancel
                # (x^2 - y^2): its magnitude is the sum of theirs
                wmag = vmap(lambda mon: sh_from_monomials(D, mon, magnitude=True))(x[:, 16:16 + NMON])
                M = (x.shape[1] - 16 - NMON) // 3
                diag = (wmag[:, :M, None] * (1.0 - cs["clamped"])[:, None, :]).reshape(x.shape[0], -1)
                idx = torch.arange(3 * M, device=x.device)
                A[:, 16 + idx, 16 + NMON + idx] = diag
            Js.append((J, A))
            x = vmap(f)(x, cs)
        g, m = g_rec[sl].double(), m_rec[sl].double()
        for J, A in reversed(Js):
            g = torch.einsum("nr,nrl->nl", g, J)
            m = torch.einsum("nr,nrl->nl", m, A)
        g_out.append(g)
        m_out.append(m)
    g, m = torch.cat(g_out), torch.cat(m_out)
    return {k: (g[:, offs[k]], m[:, offs[k]]) for k in names}


def rec_grad_from_rows(truth):
    """(g_rec, m_rec) [P,10] in REC order from raster64.row_truth's outputs (dL_dmeans2D, dL_ddepth, dL_dconic,
    dL_dopacity, dL_dcolors)."""
    order = ("dL_dmeans2D", "dL_ddepth", "dL_dconic", "dL_dopacity", "dL_dcolors")
    return (torch.cat([truth[k][0] for k in order], 1), torch.cat([truth[k][1] for k in order], 1))


def ambiguous_rows(leaves, const, cam, D, aa=False, f3d=False, rel=1e-4, rho_margin=0.05, cond_max=1e4):
    """The rows whose fp32 decisions the fp64 restatement may take the other way, with the criterion that fires:
    frustum clamp within `rel` of 1.3 tan fov, a pre-clamp SH colour within `rel` of 0 (relative to its terms'
    magnitude), rho within `rho_margin` of the antialiasing floor, 2D conditioning (|a||c| + b^2) / |det| over
    `cond_max`.  -> {criterion: [P] bool}."""
    m = leaves["means3D"].double()
    t = m @ cam.V[:3, :3] + cam.V[3, :3]
    crit = {}
    for i, tf in ((0, cam.tanfovx), (1, cam.tanfovy)):
        r = (t[:, i] / t[:, 2]).abs()
        crit["frustum-" + "xy"[i]] = ((r / (1.3 * tf)) - 1.0).abs() <= rel
    if "shs" in leaves:
        d = m - cam.campos
        d = d / d.norm(dim=1, keepdim=True)
        sh = leaves["shs"].double()
        w = vmap(lambda dd: sh_basis(D, dd))(d)[:, :sh.shape[1], None] * sh
        raw = 0.5 + w.sum(1)
        mag = 0.5 + w.abs().sum(1)
        crit["sh-clamp"] = (raw.abs() <= rel * mag).any(1)
    if "cov3D" in leaves:
        sig = aa_oracle.cov3d_from_six(leaves["cov3D"].double())
    else:
        s = leaves["scales"].double()
        if f3d:
            s = filter3d_oracle.dilate(s, leaves["opacities"].double(), const["filter_3d"].double())[0]
        sig = aa_oracle.cov3d_of(s * cam.mod, leaves["rotations"].double())
    a0, b, c0 = vmap(lambda mm, ss: torch.stack(cov2d(mm, ss, cam)[:3]))(m, sig).unbind(1)
    a, c = a0 + aa_oracle.DILATION, c0 + aa_oracle.DILATION
    crit["conditioning"] = (a.abs() * c.abs() + b * b) > cond_max * (a * c - b * b).abs()
    if aa:
        r = aa_oracle.ratio(a0, b, c0)
        crit["aa-floor"] = (r / aa_oracle.FLOOR - 1.0).abs() <= rho_margin * 2      # rho within 5 %: r within ~10 %
    return crit

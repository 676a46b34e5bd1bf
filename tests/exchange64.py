"""fp64 truth of the multi-GPU SH-gradient rebuild (include/r3dg_b200.h: r3dg_sh_grad_from_factors, r3dg_exchange_p2p).

    dL_dsh[g,k,c] = (1 / world) sum_v basis_k(normalize(mean_g - campos_v)) f_v[g,c]    for k < (D + 1)^2,

and exactly 0 for k >= (D + 1)^2.  A view in which row g's factor is all zeros contributes exactly 0, whatever the
direction: the kernel skips such rows, so a Gaussian culled in every view gets a row of exact zeros, and a Gaussian
culled in a view whose camera centre sits on its mean gets no NaN from that view.

bound() is the fp32 error bound of the kernel's result, per element:

    |g - g64| <= 8 eps32 (sum_v |basis_k| |f_v[g,c]|) / world + tiny,

with |basis_k| the sum of the magnitudes of basis_k's terms (x^2 + y^2 for x^2 - y^2; proj64.sh_from_monomials with
magnitude=True).  The kernel rounds each term of a basis value, so where the terms cancel its error is relative to
them, not to the value; with the value's own magnitude a direction on a nodal line of basis_k would get a bound below
the kernel's rounding.  Every term's error is a few ulps of the term (direction: difference, norm and division;
monomial: up to three products; then the FMA chain over the views and the final scale), well inside 8."""
import torch

import proj64

EPS32 = 2.0 ** -23
TINY = 1e-30


def monomials(u):
    """proj64.MONOMIALS of the unit directions u [3,N] (proj64.monomials for many directions): [NMON, N]."""
    at = {"x": u[0], "y": u[1], "z": u[2]}
    return torch.stack([torch.stack([at[c] for c in name]).prod(0) for name in proj64.MONOMIALS])


def sh_grad(means3D, campos, factors, D, M, rows=None):
    """(g64, mag) for the rows `rows` (a slice; all rows by default): g64 [n,M,3] the rebuilt gradient in fp64, mag
    [n,M,3] sum_v |basis_k| |f_v[g,c]| / world.  means3D [P,3], campos [world,3], factors [world,P,3]: any float
    dtype; computed on their device."""
    rows = slice(None) if rows is None else rows
    m = means3D[rows].double()
    f = factors[:, rows].double()
    cam = campos.double()
    world, n = f.shape[0], f.shape[1]
    g64 = torch.zeros((n, M, 3), dtype=torch.float64, device=m.device)
    mag = torch.zeros_like(g64)
    K = min((D + 1) ** 2, M)
    for v in range(world):
        d = m - cam[v]
        u = (d / d.norm(dim=1, keepdim=True)).T
        live = (f[v] != 0).any(1)[:, None, None]
        basis = proj64.sh_basis(D, u).T[:, :K, None]                                       # [n,K,1]
        bmag = proj64.sh_from_monomials(D, monomials(u), magnitude=True).T[:, :K, None]
        g64[:, :K] += torch.where(live, basis * f[v][:, None, :], 0.0)
        mag[:, :K] += torch.where(live, bmag * f[v].abs()[:, None, :], 0.0)
    return g64 / world, mag / world


def bound(mag):
    """The per-element fp32 error bound of the kernel from sh_grad()'s `mag`."""
    return 8 * EPS32 * mag + TINY


def check(got, means3D, campos, factors, D, M, chunk=1 << 17):
    """Asserts that `got` [P,M,3] (the kernel's dL_dsh) is within bound() of the fp64 truth, row chunk by row chunk on
    the device of `got`.  Returns the largest |got - g64| / bound seen."""
    dev = got.device
    means3D, campos, factors = (torch.as_tensor(t).to(dev) for t in (means3D, campos, factors))
    worst = 0.0
    for lo in range(0, got.shape[0], chunk):
        rows = slice(lo, min(lo + chunk, got.shape[0]))
        g64, mag = sh_grad(means3D, campos, factors, D, M, rows)
        err = (got[rows].double() - g64).abs()
        tol = bound(mag)
        bad = ~(err <= tol)
        if bad.any():
            i = int(bad.nonzero()[0, 0])
            raise AssertionError(f"{int(bad.sum())} elements outside the fp32 bound; first at row {lo + i}: "
                                 f"got {got[lo + i].tolist()}, fp64 {g64[i].tolist()}, bound {tol[i].tolist()}")
        worst = max(worst, float((err / tol).max()))
    return worst

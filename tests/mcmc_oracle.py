"""Test-side code for the MCMC densification (relightable3dgaussian_b200/mcmc.py, csrc/mcmc.cu).

* `mcmc_case(name, device, dead)`: densify_oracle's seeded case `name` with a fraction `dead` of the opacity logits
  pushed below logit(0.005) (opacities drawn in [1e-4, 4.9e-3]).
* `correction(o, N, min_opacity)`: the source update in fp64, as PyTorch operations.
* `restate_relocate_and_grow` / `restate_inject_noise`: a PyTorch restatement of mcmc.py's semantics, on any device,
  with boolean indexing, `torch.searchsorted` on an fp64 `torch.cumsum`, and the fp64 formulas.
* `StandIn`: densify_oracle's model stand-in plus the reference's `step` and `reset_opacity`.
"""
import hashlib
import math

import numpy as np
import torch

import densify_oracle as do

EPS32 = float(np.finfo(np.float32).eps)
STATS = do.STATS + ("max_radii2D",)
OMAX = 1.0 - 2.0 ** -23


def mcmc_case(name, device="cpu", dead=0.05):
    c = do.densify_case(name, device)
    P = c["P"]
    g = torch.Generator(device=device).manual_seed(int(hashlib.sha256(("mcmc/" + name).encode()).hexdigest()[:8], 16))
    sel = torch.rand(P, generator=g, device=device) < dead
    o = torch.rand(P, generator=g, device=device) * (4.9e-3 - 1e-4) + 1e-4
    op = c["params"]["opacity"]
    c["params"]["opacity"] = torch.where(sel[:, None], torch.log(o / (1 - o))[:, None], op).contiguous()
    return c


# C(n, j) for n, j <= 64, rounded once to fp64 from the exact integers, as the kernel's table
BINOM = torch.tensor([[float(math.comb(n, j)) for j in range(65)] for n in range(65)], dtype=torch.float64)


def correction(o, N, min_opacity):
    """o: fp64 opacities, N: int64 copies, same shape.  Returns (x, coef, new_logit fp64 before rounding)."""
    x = -torch.expm1(torch.log1p(-o) / N.double())
    s = torch.zeros_like(o)
    xp = torch.ones_like(o)
    for j in range(1, int(N.max()) + 1 if N.numel() else 1):
        xp = xp * x
        c = BINOM.to(o.device)[N, j]                   # C(N, j) = 0 for j > N
        term = c * xp / math.sqrt(j)
        s = s + term if j % 2 == 1 else s - term
    coef = torch.where(x > 0, o / torch.where(x > 0, s, torch.ones_like(s)), torch.ones_like(o))
    on = x.clamp(min_opacity, OMAX)
    return x, coef, torch.log(on / (1 - on))


def draw(opacity_logit, u, min_opacity, relocation):
    """Sources of the draws.  Returns (pick [len(u)] int64 or -1, cdf fp64, total, v fp64)."""
    o = torch.sigmoid(opacity_logit[:, 0])
    alive = o > min_opacity
    w = torch.where(alive, o, torch.zeros_like(o)).double()
    P = w.shape[0]
    cdf = torch.cumsum(w, 0)
    total = float(cdf[-1])
    if total > 0:
        v = u.double() * total
        pick = torch.searchsorted(cdf, v, right=True).clamp_max(P - 1)
    else:
        v = u.double() * P
        pick = torch.floor(v).long().clamp_max(P - 1)
    if relocation:
        pick = torch.where(~alive & (total > 0), pick, torch.full_like(pick, -1))
    return pick, cdf, total, v


def near_boundary(pick, cdf, total, v, tol=1e-12):
    """Draws whose target lies within tol * total of a CDF value they sit between."""
    ok = pick >= 0
    if total <= 0 or not bool(ok.any()):
        return 0
    p = pick[ok]
    hi = cdf[p]
    lo = torch.where(p > 0, cdf[(p - 1).clamp_min(0)], torch.zeros_like(hi))
    vv = v[ok]
    return int((((hi - vv).abs() <= tol * total) | ((vv - lo).abs() <= tol * total)).sum())


def _update(m, pick, n_max, min_opacity):
    """Counts and corrected (logit, scaling) of every source of `pick` (values of the current rows)."""
    P = m._xyz.shape[0]
    p = pick[pick >= 0]
    count = torch.bincount(p, minlength=P)
    src = count > 0
    o = torch.sigmoid(m._opacity[:, 0]).double()
    N = torch.clamp(count + 1, max=n_max)
    _, coef, lg = correction(o[src], N[src], min_opacity)
    new_l = m._opacity.detach().clone()
    new_s = m._scaling.detach().clone()
    new_l[src, 0] = lg.float()
    new_s[src] = (m._scaling.detach()[src].double() + torch.log(coef)[:, None]).float()
    return count, src, new_l, new_s


def _state(m, p):
    return m.optimizer.state.get(p, None)


def restate_relocate_and_grow(m, cap_max, min_opacity=0.005, growth_rate=0.05, n_max=51, u_reloc=None, u_grow=None):
    """mcmc.relocate_and_grow on `m`, with injected uniforms u_reloc [P] and u_grow [n_new].  Returns dict(reloc, grow)
    of (pick, cdf, total, v) plus the counts."""
    opt = m.optimizer
    P = m._xyz.shape[0]
    out = {}
    with torch.no_grad():
        pick, cdf, total, v = draw(m._opacity, u_reloc, min_opacity, True)
        out["reloc"] = (pick, cdf, total, v)
        count, src, new_l, new_s = _update(m, pick, n_max, min_opacity)
        dst = pick >= 0
        rew = dst | src
        srow = pick[dst]
        for g in opt.param_groups:
            n, p = g["name"], g["params"][0]
            if n == "opacity":
                p[src] = new_l[src]
                p[dst] = new_l[srow]
            elif n == "scaling":
                p[src] = new_s[src]
                p[dst] = new_s[srow]
            else:
                p[dst] = p[srow]
            st = _state(m, p)
            if st is not None:
                st["exp_avg"][rew] = 0
                st["exp_avg_sq"][rew] = 0
        for n in STATS:
            getattr(m, n)[rew] = 0
        out["reloc_count"] = count
        out["reloc_rewritten"] = rew
        for g in opt.param_groups:
            g["params"][0].grad = None
        n_new = max(0, min(cap_max, int(P * (1 + growth_rate))) - P)
        out["n_new"] = n_new
        if n_new == 0:
            return out
        pick, cdf, total, v = draw(m._opacity, u_grow, min_opacity, False)
        out["grow"] = (pick, cdf, total, v)
        count, src, new_l, new_s = _update(m, pick, n_max, min_opacity)
        out["grow_count"] = count
        out["grow_src"] = src
    for g in opt.param_groups:
        n, old = g["name"], g["params"][0]
        base = old.detach().clone()
        if n == "opacity":
            base[src] = new_l[src]
            ext = new_l[pick]
        elif n == "scaling":
            base[src] = new_s[src]
            ext = new_s[pick]
        else:
            ext = base[pick]
        newp = torch.nn.Parameter(torch.cat((base, ext), 0).requires_grad_(True))
        st = _state(m, old)
        if st is not None:
            for k in ("exp_avg", "exp_avg_sq"):
                t = st[k].clone()
                t[src] = 0
                st[k] = torch.cat((t, torch.zeros_like(ext)), 0)
            del opt.state[old]
            opt.state[newp] = st
        g["params"][0] = newp
        setattr(m, do.ATTRS[n], newp)
    for n in STATS:
        t = getattr(m, n).clone()
        t[src] = 0
        setattr(m, n, torch.cat((t, torch.zeros((n_new,) + tuple(t.shape[1:]), device=t.device)), 0))
    return out


def restate_inject_noise(m, z, noise_lr=5e5, k=100, t=0.005):
    """(expected xyz in fp64, per-component bound 4 eps32 (|x| + sum_jk |noise terms|)) for standard normals z."""
    lr = [g["lr"] for g in m.optimizer.param_groups if g["name"] == "xyz"][0]
    scale = noise_lr * lr
    o = torch.sigmoid(m._opacity.detach()[:, 0]).double()
    gate = scale / (1 + torch.exp(k * (o - t)))
    R = do.rotation_matrices(m._rotation.detach().double())
    e2 = torch.exp(m._scaling.detach().double()) ** 2
    zz = z.double()
    # terms[i, c, j, k] = R_ck e2_k R_jk z_j
    terms = R[:, :, None, :] * e2[:, None, None, :] * R[:, None, :, :] * zz[:, None, :, None]
    noise = gate[:, None] * terms.sum((2, 3))
    mag = gate[:, None] * terms.abs().sum((2, 3))
    x = m._xyz.detach().double()
    return x + noise, 4 * EPS32 * (x.abs() + mag)


class StandIn(do.StandIn):
    """densify_oracle.StandIn plus the reference's `step` (optimizer step, then zero_grad) and `reset_opacity`."""

    def step(self):
        self.optimizer.step()
        self.optimizer.zero_grad()

    def reset_opacity(self):
        with torch.no_grad():
            self._opacity.copy_(torch.logit(torch.clamp(torch.sigmoid(self._opacity), max=0.01)))

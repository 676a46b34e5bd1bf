"""MCMC densification (3DGS-MCMC, Kheradmand et al. 2024; gsplat's `MCMCStrategy`), backed by csrc/mcmc.cu.

MCMC replaces the clone / split / prune heuristic with a hard budget on the number of Gaussians:

* `relocate_and_grow` moves dead Gaussians (opacity <= min_opacity) onto live ones, drawn in proportion to opacity,
  with an opacity and scale correction that keeps the rendered result, then grows the model by `growth_rate` per call
  until it holds `cap_max` Gaussians.  It never prunes: with `cap_max <= P` it only relocates.
* `inject_noise` adds, after every optimiser step, opacity-gated noise shaped by each Gaussian's covariance to the
  positions, so that dead or transparent Gaussians keep exploring.

Relocation rewrites the rows in place; growth replaces every tensor by one with `P + n_new` rows: the relocated rows
(the drawn sources corrected), then one copy of the source per draw, in draw order.  Every rewritten row (each drawn
source and each copy) gets the source's values with the corrected opacity and scale, zero Adam moments in every group
that has state, and zero statistics (`weights_accum`, `xyz_gradient_accum`, `normal_gradient_accum`, `denom`,
`max_radii2D`); `state["step"]` is untouched, and a group without state grows only its parameter.  Every parameter's
`.grad` is dropped: the reference densifies between the backward pass and the step, and a gradient kept on a
rewritten row (zero moments) would drive a full-size Adam step computed for another Gaussian.

Sampling: row i is alive when sigmoid(l_i) > min_opacity (torch's fp32 sigmoid, min_opacity rounded to fp32, as torch
compares them) and weighs its opacity; the CDF is an fp64 prefix sum in a fixed order, and draw d picks the smallest i
with cdf[i] > u_d * total.  Relocation gives every row one uniform (`torch.rand(P)`; only dead rows use theirs), so the
number of dead rows is never needed on the host; growth draws `torch.rand(n_new)`, n_new =
max(0, min(cap_max, int(P (1 + growth_rate))) - P).  The draws of each source are counted with integer atomics, so a
call is deterministic given its uniforms: repeated calls, and ranks seeded alike, give bitwise-equal models.

Correction of a source drawn c times, N = min(c + 1, n_max), o its opacity in fp64: x = 1 - (1 - o)^(1/N) is the
opacity of each of the N Gaussians, and the scale is multiplied by coef = o / sum_{j=1..N} (-1)^(j-1) C(N,j) x^j /
sqrt(j), the paper's double sum folded into one by the hockey-stick identity.  The sum alternates; fp64 keeps its
relative error near 1e-12 for N <= 51, where fp32 loses 3.5e-4.  x is clamped to [min_opacity, 1 - 2^-23] before the
logit.  A source drawn more than n_max - 1 times gives all its copies the N = n_max values.

Edge cases: with no live row relocation does nothing and growth draws uniformly (every row weighs 1); a source whose
fp32 opacity underflowed to 0 gets x = 0 and coef = 1 (the limit), so nothing becomes NaN.

Neither entry point synchronises with the host.  `relocate_and_grow` is 6 launches, 12 with growth; `inject_noise` is 1
(0 when noise_lr * lr_xyz == 0, in which case nothing is drawn either).  There is no PyTorch fallback: CUDA float32
contiguous tensors only, anything else raises before a launch.  `install()` lets the reference's training loop train
with MCMC; `uninstall()` restores it.
"""
import ctypes

import torch

from . import _lib
from .densify import ATTRS, STATS, _check, _f32, _groups

KIND = {"copy": 0, "moment": 1, "opacity": 5, "scaling": 6}
MAX_N = 64


def _default_sampler(kind, shape, device):
    return torch.randn(shape, device=device) if kind == "randn" else torch.rand(shape, device=device)


# Draws the noise's [P,3] standard normals (kind "randn") and the draws' uniforms (kind "rand"); tests replace it to
# inject fixed samples.
_sampler = _default_sampler


def _sample(kind, shape, device):
    s = _sampler(kind, shape, device)
    if tuple(s.shape) != tuple(shape):
        raise ValueError(f"mcmc: sampler returned shape {tuple(s.shape)} for {kind}{tuple(shape)}")
    return _check(s, f"{kind} samples")


def growth_count(P, cap_max, growth_rate=0.05):
    """Rows one growth step adds: max(0, min(cap_max, int(P (1 + growth_rate))) - P)."""
    return max(0, min(int(cap_max), int(P * (1 + growth_rate))) - P)


def _xyz_lr(model):
    for g in model.optimizer.param_groups:
        if g.get("name") == "xyz":
            return float(g["lr"])
    raise KeyError("inject_noise: the optimizer has no 'xyz' group")


def inject_noise(model, noise_lr=5e5, k=100, t=0.005):
    """xyz += noise_lr * lr_xyz * sigmoid(-k (o - t)) * Sigma z in place, with o = sigmoid(opacity logit), Sigma =
    R diag(exp(s))^2 R^T the Gaussian's covariance, z ~ N(0, I) from `torch.randn` and lr_xyz the current lr of the
    optimizer's "xyz" group.  Call it after every optimiser step.  Adam moments are not touched.  One launch, no host
    sync; with noise_lr * lr_xyz == 0 nothing is drawn or launched."""
    scale = float(noise_lr) * _xyz_lr(model)
    P = model._xyz.shape[0]
    xyz = _check(model._xyz, "xyz", P, 3)
    rot = _check(model._rotation, "rotation", P, 4)
    scl = _check(model._scaling, "scaling", P, 3)
    opa = _check(model._opacity, "opacity", P, 1)
    dev = xyz.device
    if any(x.device != dev for x in (rot, scl, opa)):
        raise RuntimeError("inject_noise: all tensors must live on one device")
    if scale == 0.0 or P == 0:
        return
    z = _sample("randn", (P, 3), dev)
    _lib.call("r3dg_mcmc_noise", dev, P, xyz.data_ptr(), rot.data_ptr(), scl.data_ptr(), opa.data_ptr(), z.data_ptr(),
              scale, float(k), float(t), what="mcmc_noise")


def _desc(src, dst, kind, row_bytes):
    d = _lib.DensifyTensor()
    d.src, d.dst, d.row_bytes, d.kind = src.data_ptr(), dst.data_ptr(), row_bytes, KIND[kind]
    return d


def _phase(model, groups, P, n_new, min_opacity, n_max, tmp, dev):
    """One relocation (n_new == 0, in place) or growth (n_new > 0, new tensors) pass; returns the new tensors."""
    u = _sample("rand", (n_new if n_new else P,), dev)
    byname = {n: p for _, n, p, _ in groups}
    _lib.call("r3dg_mcmc_classify", dev, P, byname["opacity"].data_ptr(), _f32(min_opacity), tmp.data_ptr(), tmp.numel(),
              what="mcmc_classify")
    out = lambda t: t if n_new == 0 else torch.empty((P + n_new,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
    descs, new = [], []
    for g, name, p, st in groups:
        row_bytes = p[0].numel() * 4
        np_ = out(p)
        descs.append(_desc(p, np_, name if name in ("opacity", "scaling") else "copy", row_bytes))
        moms = None
        if st is not None:
            moms = (out(st["exp_avg"]), out(st["exp_avg_sq"]))
            descs += [_desc(st["exp_avg"], moms[0], "moment", row_bytes), _desc(st["exp_avg_sq"], moms[1], "moment", row_bytes)]
        new.append((g, name, p, st, np_, moms))
    stats = {}
    for n in STATS + ("max_radii2D",):
        t = getattr(model, n)
        stats[n] = out(t)
        descs.append(_desc(t, stats[n], "moment", 4))
    arr = (_lib.DensifyTensor * len(descs))(*descs)
    _lib.call("r3dg_mcmc_apply", dev, P, n_new, u.data_ptr(), byname["opacity"].data_ptr(), byname["scaling"].data_ptr(),
              float(min_opacity), n_max, len(descs), arr, tmp.data_ptr(), tmp.numel(), what="mcmc_apply")
    return new, stats


def relocate_and_grow(model, cap_max, min_opacity=0.005, growth_rate=0.05, n_max=51):
    """Relocate the dead Gaussians onto live ones, then grow by `growth_rate` up to `cap_max` rows; see the module
    docstring.  Every parameter is left without a gradient, so the next optimiser step skips them (the reference's
    densify_and_prune, which runs before the step, replaces every parameter to the same effect).  Returns the number
    of rows added.  No host sync."""
    if getattr(model, "_visibility_tracing", None) is not None:
        raise RuntimeError("relocate_and_grow: the model carries a baked visibility ([P, N] per Gaussian), which "
                           "relocation and growth would leave stale and mis-sized; densify before baking")
    if isinstance(n_max, bool) or not isinstance(n_max, int) or not 2 <= n_max <= MAX_N:
        raise ValueError(f"relocate_and_grow: n_max must be an integer in [2, {MAX_N}], got {n_max!r}")
    if isinstance(cap_max, bool) or not isinstance(cap_max, int) or cap_max < 0:
        raise ValueError(f"relocate_and_grow: cap_max must be a non-negative integer, got {cap_max!r}")
    P = model._xyz.shape[0]
    groups = _groups(model, P, "relocate_and_grow")
    byname = {n: p for _, n, p, _ in groups}
    _check(byname["scaling"], "scaling", P, 3)
    _check(byname["opacity"], "opacity", P, 1)
    for n in STATS:
        _check(getattr(model, n), n, P, 1)
    _check(model.max_radii2D, "max_radii2D", P, 1)
    dev = byname["xyz"].device
    tensors = list(byname.values()) + [getattr(model, n) for n in STATS + ("max_radii2D",)]
    if any(t.device != dev for t in tensors):
        raise RuntimeError("relocate_and_grow: all tensors must live on one device")
    if P == 0:
        return 0
    n_new = growth_count(P, cap_max, growth_rate)
    tmp = _lib.scratch(_lib.load().r3dg_mcmc_tmp_bytes(P, n_new), dev)
    with torch.no_grad():
        _phase(model, groups, P, 0, min_opacity, n_max, tmp, dev)
        # The gradients in place belong to the rows before relocation, and a rewritten row's zero moments would turn
        # any of them into a full-size Adam step; drop them all, as replacing the parameters does.
        for _, _, p, _ in groups:
            p.grad = None
        if n_new == 0:
            return 0
        new, stats = _phase(model, groups, P, n_new, min_opacity, n_max, tmp, dev)
    opt = model.optimizer
    for g, name, p, st, np_, moms in new:
        newp = torch.nn.Parameter(np_.requires_grad_(True))
        if st is not None:
            del opt.state[p]
            st["exp_avg"], st["exp_avg_sq"] = moms
            opt.state[newp] = st
        g["params"][0] = newp
        setattr(model, ATTRS[name], newp)
    for n, t in stats.items():
        setattr(model, n, t)
    return n_new


_saved = None


def installed_on():
    """The class install() rebound, or None."""
    return None if _saved is None else _saved[0]


def install(cls=None, *, cap_max, noise_lr=5e5, growth_rate=0.05, n_max=51):
    """Let the reference's training loop (train.py) train with MCMC: on `cls` (default: the reference's
    scene.gaussian_model.GaussianModel) `densify_and_prune(max_grad, min_opacity, ...)` becomes
    `relocate_and_grow(self, cap_max, min_opacity, growth_rate, n_max)` (the gradient thresholds are ignored),
    `add_densification_stats` and `reset_opacity` become no-ops (MCMC has no opacity reset), and `step` runs the
    original step, then `inject_noise(self, noise_lr)`.  The reference's schedule stays: relocation and growth every
    densification_interval iterations between densify_from_iter and densify_until_iter, noise on every step.
    Raises if already installed, or while densify.install() holds the same class."""
    global _saved
    if _saved is not None:
        raise RuntimeError("mcmc.install(): already installed; call uninstall() first")
    if isinstance(cap_max, bool) or not isinstance(cap_max, int) or cap_max < 0:
        raise ValueError(f"mcmc.install(): cap_max must be a non-negative integer, got {cap_max!r}")
    if isinstance(n_max, bool) or not isinstance(n_max, int) or not 2 <= n_max <= MAX_N:
        raise ValueError(f"mcmc.install(): n_max must be an integer in [2, {MAX_N}], got {n_max!r}")
    if cls is None:
        from scene.gaussian_model import GaussianModel as cls
    from . import densify
    if densify._saved is not None and densify._saved[0] is cls:
        raise RuntimeError(f"mcmc.install(): densify.install() holds {cls.__name__}; call densify.uninstall() first")
    step = cls.step
    names = ("densify_and_prune", "add_densification_stats", "reset_opacity", "step")
    _saved = (cls, {n: cls.__dict__.get(n) for n in names})

    def _dp(self, max_grad, min_opacity, extent, max_screen_size, max_grad_normal, weights_threshold=1e-4):
        return relocate_and_grow(self, cap_max, min_opacity, growth_rate, n_max)

    def _stats(self, viewspace_point_tensor, update_filter, weights):
        return None

    def _reset(self):
        return None

    def _step(self):
        step(self)
        inject_noise(self, noise_lr)

    cls.densify_and_prune, cls.add_densification_stats, cls.reset_opacity, cls.step = _dp, _stats, _reset, _step
    return cls


def uninstall():
    """Restore what install() replaced."""
    global _saved
    if _saved is None:
        return
    cls, fns = _saved
    for name, fn in fns.items():
        if fn is None:
            delattr(cls, name)
        else:
            setattr(cls, name, fn)
    _saved = None

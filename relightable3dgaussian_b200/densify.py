"""Stage-1 densification with the reference's signatures: `GaussianModel.add_densification_stats` and
`GaussianModel.densify_and_prune` (scene/gaussian_model.py:890-937), backed by csrc/densify.cu.

The reference clones, splits and prunes with boolean indexing and `torch.cat`: every per-Gaussian tensor and both
Adam moments are copied four times, with one host sync per boolean index.  Here `densify_and_prune` is four launches
(classify, scan, offsets, apply) and ONE host read-back of seven counts; the final tensors are written directly from
the old ones, so the peak is the old plus the final tensors (plus 17 B per old row of scratch).  The result is the
reference's on the same device:

* row order: kept originals, kept clones, kept split copy 1 of each split row, kept split copy 2, each in row order;
* clones are raw copies; split copies get xyz' = build_rotation(q) (z * exp(s)) + xyz and
  scaling' = log(exp(s) / 1.6), every other parameter raw; z is `torch.randn((2|S|, 3))` drawn where the reference
  calls `torch.normal`, which consumes the generator identically;
* new rows get zero Adam moments, `state["step"]` is untouched, a group without state grows only its parameter;
* the final prune sees `max_radii2D` already zeroed (the reference's `densification_postfix` does that before it),
  and on exit all five statistics are zero;
* the two lines the reference prints are printed with the same numbers.

Not reproduced: the reference's closing `torch.cuda.empty_cache()`, which would synchronise the device again.

`add_densification_stats` is one launch with no host sync; with `radii` it also does train.py's
`max_radii2D[filter] = max(max_radii2D[filter], radii[filter])`.

There is no PyTorch fallback: CUDA float32 contiguous tensors only, anything else raises before a launch.
`install()` rebinds both methods on the reference's `GaussianModel`, `uninstall()` restores them.
"""
import ctypes

import numpy as np
import torch

from . import _lib

STAGE1_GROUPS = ("xyz", "normal", "rotation", "scaling", "opacity", "f_dc", "f_rest")
PBR_GROUPS = ("base_color", "roughness", "incidents_dc", "incidents_rest", "visibility_dc", "visibility_rest")
# optimizer group name -> GaussianModel attribute
ATTRS = dict({"xyz": "_xyz", "normal": "_normal", "rotation": "_rotation", "scaling": "_scaling", "opacity": "_opacity",
              "f_dc": "_shs_dc", "f_rest": "_shs_rest"}, **{n: "_" + n for n in PBR_GROUPS})
STATS = ("weights_accum", "xyz_gradient_accum", "normal_gradient_accum", "denom")
KIND = {"copy": 0, "moment": 1, "xyz": 2, "scaling": 3, "zero": 4}


def _default_sampler(shape, device):
    return torch.randn(shape, device=device)


# Draws the [2|S|, 3] standard normals of the split copies; tests replace it to inject fixed samples.
_sampler = _default_sampler
_pinned = {}


def _f32(x):
    """A Python float as torch compares it with a float32 tensor: rounded to fp32."""
    return float(np.float32(x))


def _check(t, what, rows=None, cols=None):
    if not torch.is_tensor(t):
        raise TypeError(f"{what}: expected a tensor, got {type(t).__name__}")
    if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
        raise RuntimeError(f"{what}: must be a contiguous CUDA float32 tensor (no CPU path), got {t.dtype} on {t.device}"
                           f"{'' if t.is_contiguous() else ', non-contiguous'}")
    if rows is not None and (t.dim() == 0 or t.shape[0] != rows):
        raise ValueError(f"{what}: expected {rows} rows, got shape {tuple(t.shape)}")
    if cols is not None and t.numel() != rows * cols:
        raise ValueError(f"{what}: expected {cols} values per row, got shape {tuple(t.shape)}")
    return t


def add_densification_stats(model, viewspace_point_tensor, update_filter, weights, radii=None, absgrad=False):
    """`GaussianModel.add_densification_stats` (gaussian_model.py:931-937): weights_accum += weights and, for the rows
    in `update_filter`, xyz_gradient_accum += |grad[:, :2]|, normal_gradient_accum += |_normal.grad|, denom += 1.
    With `radii` it also folds in train.py:164-165's max_radii2D update over the same rows.  One launch, no sync.

    `absgrad=True` (AbsGS; not part of the reference surface): xyz_gradient_accum accumulates |absgrad| instead, the
    norm of `viewspace_point_tensor.absgrad` [P,2] that the rasterizer's backward sets in its absgrad mode
    (rasterizer.set_absgrad), the per-pixel magnitudes summed before cancelling.  That statistic is larger than
    |grad[:, :2]|, so it wants a larger densify_grad_threshold: gsplat defaults to grow_grad2d = 0.0008 with absgrad
    and 0.0002 without (gsplat's defaults, not a value tuned for this project).  A missing or mis-shaped `.absgrad` is
    refused before anything is launched."""
    P = model._xyz.shape[0]
    if absgrad:
        grad = getattr(viewspace_point_tensor, "absgrad", None)
        if grad is None:
            raise RuntimeError("add_densification_stats(absgrad=True): viewspace_point_tensor has no .absgrad (the "
                               "rasterizer sets it in its absgrad mode: rasterizer.set_absgrad(True) or absgrad=True)")
        if not torch.is_tensor(grad) or tuple(grad.shape) != (P, 2):
            raise ValueError(f"viewspace_point_tensor.absgrad: expected a [P, 2] = {(P, 2)} tensor, got "
                             f"{tuple(grad.shape) if torch.is_tensor(grad) else type(grad).__name__}")
        _check(grad, "viewspace_point_tensor.absgrad", P)
    else:
        grad = viewspace_point_tensor.grad
    if grad is None:
        raise RuntimeError("add_densification_stats: viewspace_point_tensor has no .grad")
    ngrad = model._normal.grad
    if ngrad is None:
        raise RuntimeError("add_densification_stats: _normal has no .grad")
    _check(grad, "viewspace_point_tensor.grad", P)
    if grad.dim() != 2 or grad.shape[1] < 2:
        raise ValueError(f"viewspace_point_tensor.grad: expected [P, >=2], got {tuple(grad.shape)}")
    _check(ngrad, "_normal.grad", P, 3)
    _check(weights, "weights", P, 1)
    for n in STATS:
        _check(getattr(model, n), n, P, 1)
    if not torch.is_tensor(update_filter) or update_filter.dtype != torch.bool or not update_filter.is_cuda \
            or update_filter.numel() != P or not update_filter.is_contiguous():
        raise RuntimeError("add_densification_stats: update_filter must be a contiguous CUDA bool tensor with P elements")
    mr = None
    if radii is not None:
        if not torch.is_tensor(radii) or radii.dtype != torch.int32 or not radii.is_cuda or radii.numel() != P \
                or not radii.is_contiguous():
            raise RuntimeError("add_densification_stats: radii must be a contiguous CUDA int32 tensor with P elements")
        mr = _check(model.max_radii2D, "max_radii2D", P, 1)
    devs = {grad.device, ngrad.device, weights.device, update_filter.device}
    if len(devs) != 1:
        raise RuntimeError("add_densification_stats: all tensors must live on one device")
    _lib.call("r3dg_densify_stats", grad.device, P, grad.data_ptr(), grad.shape[1], ngrad.data_ptr(),
              update_filter.view(torch.uint8).data_ptr(), weights.data_ptr(), radii.data_ptr() if radii is not None else None,
              model.weights_accum.data_ptr(), model.xyz_gradient_accum.data_ptr(), model.normal_gradient_accum.data_ptr(),
              model.denom.data_ptr(), mr.data_ptr() if mr is not None else None, what="densify_stats")


def _groups(model, P, what="densify_and_prune"):
    """[(group, name, param, state or None)] in param_groups order, validated; errors name the caller `what`."""
    opt = model.optimizer
    out = []
    for g in opt.param_groups:
        name = g.get("name")
        if len(g["params"]) != 1:
            raise ValueError(f"{what}: group {name!r} must hold exactly one parameter")
        if name not in ATTRS:
            raise KeyError(f"{what}: unknown parameter group {name!r}")
        p = _check(g["params"][0], f"parameter {name!r}", P)
        st = opt.state.get(p, None)
        if st is not None:
            if "exp_avg" not in st or "exp_avg_sq" not in st:
                raise ValueError(f"{what}: optimizer state of {name!r} has no Adam moments")
            for k in ("exp_avg", "exp_avg_sq"):
                _check(st[k], f"{k} of {name!r}", P)
                if st[k].shape != p.shape:
                    raise ValueError(f"{what}: {k} of {name!r} has shape {tuple(st[k].shape)}, parameter {tuple(p.shape)}")
        out.append((g, name, p, st))
    names = [n for _, n, _, _ in out]
    want = STAGE1_GROUPS + (PBR_GROUPS if getattr(model, "use_pbr", False) else ())
    if sorted(names) != sorted(want):
        raise ValueError(f"{what}: parameter groups {names} do not match the model's {list(want)}")
    return out


def densify_and_prune(model, max_grad, min_opacity, extent, max_screen_size, max_grad_normal, weights_threshold=1e-4):
    """`GaussianModel.densify_and_prune` (gaussian_model.py:890-914) with its clone, split and prune steps fused; see
    the module docstring for what is reproduced.  One host read-back; every tensor is replaced by a new one."""
    P = model._xyz.shape[0]
    groups = _groups(model, P)
    byname = {n: p for _, n, p, _ in groups}
    for n, cols in (("xyz", 3), ("scaling", 3), ("rotation", 4), ("opacity", 1)):
        _check(byname[n], n, P, cols)
    for n in STATS:
        _check(getattr(model, n), n, P, 1)
    _check(model.max_radii2D, "max_radii2D", P, 1)
    dev = byname["xyz"].device
    if any(p.device != dev for p in byname.values()):
        raise RuntimeError("densify_and_prune: all tensors must live on one device")
    split_recip = float(np.float32(1.0) / np.float32(0.8 * 2))   # torch's CUDA x / 1.6: x * fp32(1 / fp32(1.6))
    th = _lib.DensifyThresholds()
    th.max_grad, th.max_grad_normal = _f32(max_grad), _f32(max_grad_normal)
    th.dense_scale = _f32(model.percent_dense * extent)
    th.min_opacity, th.weights_threshold = _f32(min_opacity), _f32(weights_threshold)
    th.check_size = 1 if max_screen_size else 0
    th.max_screen_size = _f32(max_screen_size) if max_screen_size else 0.0
    th.big_scale = _f32(0.1 * extent)
    th.split_recip = split_recip
    key = dev.index
    if key not in _pinned:
        _pinned[key] = torch.zeros(8, dtype=torch.int32).pin_memory()
    totals_h = _pinned[key]
    tmp = _lib.scratch(_lib.load().r3dg_densify_tmp_bytes(P), dev)
    _lib.call("r3dg_densify_classify", dev, P, model.xyz_gradient_accum.data_ptr(), model.normal_gradient_accum.data_ptr(),
              model.denom.data_ptr(), model.weights_accum.data_ptr(), byname["scaling"].data_ptr(), byname["opacity"].data_ptr(),
              ctypes.byref(th), tmp.data_ptr(), tmp.numel(), totals_h.data_ptr(), what="densify_classify")
    torch.cuda.current_stream(dev).synchronize()                    # the one read-back
    tot = [int(v) for v in totals_h.tolist()]
    keep_a, keep_b, keep_c, n_split, n_clone, normal_sel, light = tot[:7]
    P1 = P + n_clone
    # clones enter the split test with a padded gradient of 0, and clones and split copies carry weights_accum = 1
    zero_f, one_f, thn, wt = np.float32(0), np.float32(1), np.float32(max_grad_normal), np.float32(weights_threshold)
    print("densify_and_split_normal:", normal_sel + (n_clone if zero_f >= thn else 0), "/", P1)
    print("weights_accum:", light + (n_clone + 2 * n_split if one_f < wt else 0), "/", P1 + n_split)
    z = _sampler((2 * n_split, 3), dev)
    if z.shape != (2 * n_split, 3):
        raise ValueError(f"densify_and_prune: sampler returned shape {tuple(z.shape)}, expected {(2 * n_split, 3)}")
    z = _check(z, "normal samples")
    Pn = keep_a + keep_b + 2 * keep_c
    descs, hold, new = [], [], []
    for g, name, p, st in groups:
        kind = {"xyz": "xyz", "scaling": "scaling"}.get(name, "copy")
        row_bytes = p[0].numel() * 4 if P > 0 else 4 * max(1, int(np.prod(p.shape[1:])))
        np_ = torch.empty((Pn,) + tuple(p.shape[1:]), dtype=torch.float32, device=dev)
        work = [(p, np_, kind)]
        moms = None
        if st is not None:
            moms = (torch.empty_like(np_), torch.empty_like(np_))
            work += [(st["exp_avg"], moms[0], "moment"), (st["exp_avg_sq"], moms[1], "moment")]
        for src, dst, k in work:
            d = _lib.DensifyTensor()
            d.src, d.dst, d.row_bytes, d.kind = src.data_ptr(), dst.data_ptr(), row_bytes, KIND[k]
            descs.append(d)
        new.append((g, name, p, st, np_, moms))
    stats = {n: torch.empty((Pn, 1), dtype=torch.float32, device=dev) for n in STATS}
    stats["max_radii2D"] = torch.empty((Pn,), dtype=torch.float32, device=dev)
    for t in stats.values():
        d = _lib.DensifyTensor()
        d.src, d.dst, d.row_bytes, d.kind = None, t.data_ptr(), 4, KIND["zero"]
        descs.append(d)
    arr = (_lib.DensifyTensor * len(descs))(*descs)
    tot_c = (ctypes.c_int * 7)(*tot[:7])
    rot = _lib.aligned16(byname["rotation"].detach())
    _lib.call("r3dg_densify_apply", dev, P, tot_c, len(descs), arr, rot.data_ptr(), byname["scaling"].data_ptr(),
              z.data_ptr(), split_recip, tmp.data_ptr(), tmp.numel(), what="densify_apply")
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


_saved = None


def install(cls=None, absgrad=False):
    """Rebind `cls.add_densification_stats` and `cls.densify_and_prune` (default: the reference's
    scene.gaussian_model.GaussianModel) to the fused versions.  Raises if already installed.  `absgrad=True`: the
    installed add_densification_stats accumulates the absgrad statistic (add_densification_stats(absgrad=True)); with
    rasterizer.set_absgrad(True) these are the two lines that give the reference's training loop AbsGS densification."""
    global _saved
    if _saved is not None:
        raise RuntimeError("densify.install(): already installed; call uninstall() first")
    if cls is None:
        from scene.gaussian_model import GaussianModel as cls
    from . import mcmc
    if mcmc.installed_on() is cls:
        raise RuntimeError(f"densify.install(): mcmc.install() holds {cls.__name__}; call mcmc.uninstall() first")
    _saved = (cls, cls.__dict__.get("add_densification_stats"), cls.__dict__.get("densify_and_prune"))

    def _stats(self, viewspace_point_tensor, update_filter, weights):
        return add_densification_stats(self, viewspace_point_tensor, update_filter, weights, absgrad=absgrad)

    def _dp(self, max_grad, min_opacity, extent, max_screen_size, max_grad_normal, weights_threshold=1e-4):
        return densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, max_grad_normal, weights_threshold)

    cls.add_densification_stats = _stats
    cls.densify_and_prune = _dp
    return cls


def uninstall():
    """Restore what install() replaced."""
    global _saved
    if _saved is None:
        return
    cls, stats, dp = _saved
    for name, fn in (("add_densification_stats", stats), ("densify_and_prune", dp)):
        if fn is None:
            delattr(cls, name)
        else:
            setattr(cls, name, fn)
    _saved = None

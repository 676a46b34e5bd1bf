"""The rasterizer's host layer, recorded: every library call that one-view and two-view forwards and backwards make
through the public entry points, over every combination of the opt-in modes, with the four `_C_raster` functions
replaced by stand-ins.  Each call is bound to the real function's signature with its defaults applied, so the record
holds the effective arguments, not their spelling.  A tensor argument is named after the leaf, settings tensor or
stand-in output it is (same storage, shape and strides), or else described by its shape, dtype and a digest of its
contents.  The gradient every leaf receives and `means2D.absgrad` complete the record.

tests/golden/raster_host_calls.json holds one digest per case; `python tests/golden/make_golden_raster_host.py`
rewrites it.  A change in how the host layer calls the library, or in what it hands back to autograd, shows up as
a changed digest; `record(case)` prints the full record of one case."""
import hashlib
import inspect
import itertools
import json
import os
import warnings

import pytest
import torch

from relightable3dgaussian_b200 import _C_raster
from relightable3dgaussian_b200 import rasterizer as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "raster_host_calls.json")
MODES = ("surface_grads", "antialiasing", "filter_3d", "ray_depth", "depth_stats", "absgrad")
P, S, M, H, W = 3, 2, 4, 4, 5
FNS = ("rasterize_gaussians", "rasterize_gaussians_backward", "rasterize_views", "rasterize_views_backward")


class FakeCuda(torch.Tensor):
    """A CPU tensor that passes the 3D filter's device check."""

    @property
    def is_cuda(self):
        return True


def cases():
    """(name, views, modes, geometry, defer, exchange): one view with and without the deferred count and a gradient
    exchange, two views without either; geometry inputs that need a gradient, or only appearance inputs."""
    out = []
    for bits in itertools.product((False, True), repeat=len(MODES)):
        modes = tuple(m for m, b in zip(MODES, bits) if b)
        for geometry in (True, False):
            for views, defer, exchange in ((1, False, False), (1, True, False), (1, False, True), (1, True, True),
                                           (2, False, False)):
                name = "-".join((f"v{views}", "geo" if geometry else "app", "defer" if defer else "sync",
                                 "ex" if exchange else "noex") + (modes or ("plain",)))
                out.append((name, views, modes, geometry, defer, exchange))
    return out


class _Overflowed(_C_raster.DeferredCount):
    """A deferred count that resolved above its buffer's capacity: the backward re-runs the forward."""

    def __init__(self, value):
        self._value, self.overflowed = value, True

    def resolve(self):
        return self._value

    __int__ = __index__ = resolve


class _Recorder:
    def __init__(self):
        self.named = []           # (name, tensor): leaves, settings tensors, stand-in outputs
        self.calls = []
        self.n = 0

    def name(self, name, t):
        self.named.append((name, t))
        return t

    def fresh(self, name, shape, dtype=torch.float32):
        """A tensor with contents no other tensor of the case has."""
        self.n += 1
        t = (torch.arange(int(torch.Size(shape).numel()), dtype=torch.float64).reshape(shape) * 0.01 + self.n)
        return self.name(name, t.to(dtype))

    def describe(self, v):
        if isinstance(v, _C_raster.DeferredCount):
            return {"deferred": int(v)}
        if isinstance(v, torch.Tensor):
            if v.numel() > 0:
                for name, t in self.named:
                    if (t.numel() > 0 and t.data_ptr() == v.data_ptr() and t.shape == v.shape and t.stride() == v.stride()
                            and t.dtype == v.dtype):
                        return name
            return _content(v)
        if isinstance(v, (tuple, list)):
            return [self.describe(x) for x in v]
        if isinstance(v, dict):
            return {k: self.describe(x) for k, x in sorted(v.items())}
        if isinstance(v, float):
            return repr(v)
        return v

    def fake(self, fn):
        sig = inspect.signature(getattr(_C_raster, fn))

        def call(*args, **kw):
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            a = b.arguments
            self.calls.append({"fn": fn, "args": {k: self.describe(v) for k, v in a.items()}})
            k = len(self.calls) - 1
            return (self._forward if fn in FNS[0::2] else self._backward)(fn, a, k)
        return call

    def _forward(self, fn, a, k):
        views = fn == "rasterize_views"
        V = len(a["cams"]) if views else 1
        lead = (V,) if views else ()
        f = lambda i, *s, dtype=torch.float32: self.fresh(f"call{k}.out{i}", lead + s, dtype)   # noqa: E731
        if views:
            rendered = [11 + v for v in range(V)]
        elif a["_defer"]:
            rendered = _Overflowed(11)
        else:
            rendered = 11
        out = (rendered, f(1, H, W, dtype=torch.int32), f(2, 3, H, W), f(3, 1, H, W), f(4, 1, H, W), f(5, S, H, W),
               f(6, 3, H, W), f(7, 3, H, W), f(8, P, 1), f(9, P, dtype=torch.int32))
        out += tuple(self.fresh(f"call{k}.out{i}", (16,), torch.uint8) for i in (10, 11, 12))
        if a["depth_stats"]:
            out += (f(13, 1, H, W), f(14, 1, H, W))
        return out

    def _backward(self, fn, a, k):
        views = fn == "rasterize_views_backward"
        V = len(a["cams"]) if views else 1
        geometry, (need_f, need_c, need_sh) = a["geometry"], a["appearance"]
        per_view = lambda t: t.dim() == 3                                   # noqa: E731
        shapes = [((V,) if views else ()) + (P, 3), a["colors"].shape if per_view(a["colors"]) else (P, 3), (P, 1),
                  (P, 3), a["features"].shape if per_view(a["features"]) else (P, S), (P, 6), (P, M, 3), (P, 3), (P, 4)]
        want = [geometry] * 9
        if not geometry:
            want[1], want[4], want[6] = need_c, need_f, need_sh
        out = a.get("_out")
        grads = []
        for i, (shape, w) in enumerate(zip(shapes, want)):
            if i == 6 and out is not None and "sh_factor" in out:
                out["sh_factor"].copy_(self.fresh(f"call{k}.sh_factor", (P, 3)))
                grads.append(torch.empty(0))
            else:
                grads.append(self.fresh(f"call{k}.grad{i}", shape) if w else None)
        grads = tuple(grads)
        if a["cam_grads"]:
            cam = tuple(self.fresh(f"call{k}.cam{i}", s) for i, s in enumerate(((V, 4, 4), (V, 4, 4), (V, 3))))
            grads += cam if views else tuple(t[0] for t in cam)
        if a["absgrad"]:
            grads += (self.fresh(f"call{k}.absgrad", ((V,) if views else ()) + (P, 2)) if geometry else None,)
        return grads


def _content(t):
    t = t.detach().contiguous()
    digest = hashlib.sha256(t.numpy().tobytes()).hexdigest()[:16] if t.numel() else ""
    return {"shape": list(t.shape), "dtype": str(t.dtype).replace("torch.", ""), "sha": digest}


class _Exchange:
    """Stand-in for dist.FactoredGradExchange: its factor buffer, the gather and the rebuild."""

    def __init__(self, rec):
        self.rec = rec
        self.factor = rec.name("exchange.factor", torch.zeros(P, 3))

    def gather_factors(self):
        self.rec.calls.append({"fn": "gather_factors"})

    def rebuild_sh(self, means3D, campos_all, degree):
        self.rec.calls.append({"fn": "rebuild_sh", "args": self.rec.describe([means3D, campos_all, degree])})
        return self.rec.fresh("exchange.sh", (P, M, 3))


def record(case, monkeypatch):
    """The record of one case: the library calls, then every leaf's gradient and means2D.absgrad."""
    name, views, modes, geometry, defer, exchange = case
    rec = _Recorder()
    for fn in FNS:
        monkeypatch.setattr(R._C, fn, rec.fake(fn))
    leaf = lambda n, *s, g=True: rec.fresh(n, s).requires_grad_(g)                     # noqa: E731
    means3D, opacities, scales, rotations = (leaf("means3D", P, 3, g=geometry), leaf("opacities", P, 1, g=geometry),
                                             leaf("scales", P, 3, g=geometry), leaf("rotations", P, 4, g=geometry))
    shs, features = leaf("shs", P, M, 3), leaf("features", P, S)
    means2D = leaf("means2D", *(((views,) if views > 1 else ()) + (P, 3)), g=geometry)
    cam_grad = geometry and not exchange
    settings = []
    for v in range(views):
        settings.append(R.GaussianRasterizationSettings(
            H, W, 0.8 + 0.1 * v, 0.6, 2.5 + v, 2.0, rec.fresh(f"bg{v}", (3,)), 1.0,
            leaf(f"viewmatrix{v}", 4, 4, g=cam_grad), leaf(f"projmatrix{v}", 4, 4, g=False), 1,
            leaf(f"campos{v}", 3, g=cam_grad), False, True, True, False))
    kw = {m: True for m in modes if m != "filter_3d"}
    if "filter_3d" in modes:
        kw["filter_3d"] = rec.name("filter_3d", (torch.arange(P, dtype=torch.float32) * 0.01 + 0.5).as_subclass(FakeCuda))
    R.set_deferred_count(defer)
    R.set_grad_exchange(_Exchange(rec) if exchange else None, rec.name("campos_all", torch.zeros(1, 3)))
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            if views > 1:
                out = R.rasterize_views(means3D, means2D, opacities, settings=settings, shs=shs, scales=scales,
                                        rotations=rotations, features=features, **kw)
            else:
                fkw = {"filter_3d": kw.pop("filter_3d")} if "filter_3d" in kw else {}
                out = R.GaussianRasterizer(settings[0], **kw)(means3D=means3D, means2D=means2D, opacities=opacities,
                                                              shs=shs, scales=scales, rotations=rotations,
                                                              features=features, **fkw)
            # the loss touches colour, depth, normal, surface_xyz and depth2, not opacity, features or the median
            loss = sum((out[i] * rec.fresh(f"weight{i}", out[i].shape)).sum() for i in (2, 4, 6, 7, 10) if i < len(out))
            loss.backward()
    finally:
        R.set_deferred_count(False)
        R.set_grad_exchange(None)
    leaves = dict(means3D=means3D, means2D=means2D, opacities=opacities, scales=scales, rotations=rotations, shs=shs,
                  features=features, **{f"{k}{v}": getattr(s, k) for v, s in enumerate(settings)
                                        for k in ("viewmatrix", "projmatrix", "campos")})
    grads = {k: None if t.grad is None else _content(t.grad) for k, t in leaves.items()}
    absgrad = getattr(means2D, "absgrad", None)
    return {"calls": rec.calls, "grads": grads, "absgrad": None if absgrad is None else _content(absgrad),
            "outputs": len(out)}


def digest(rec):
    return hashlib.sha256(json.dumps(rec, sort_keys=True).encode()).hexdigest()[:24]


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_host_layer_calls_the_library_as_recorded(case, monkeypatch):
    rec = record(case, monkeypatch)
    assert digest(rec) == _golden()[case[0]], json.dumps(rec, sort_keys=True, indent=1)


def test_golden_covers_every_case():
    assert sorted(_golden()) == sorted(c[0] for c in cases())

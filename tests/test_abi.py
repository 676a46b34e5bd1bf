"""C-ABI surface: the shared library loads and exports every symbol include/r3dg_b200.h declares,
struct layouts agree with the header, sizing functions are sane.  No GPU compute is issued."""
import ctypes
import os
import re

import pytest

from helpers import ROOT
from relightable3dgaussian_b200 import _lib


def _declared_functions():
    hdr = open(os.path.join(ROOT, "include", "r3dg_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = re.findall(r"\b(r3dg_[a-z0-9_]+)\s*\(", hdr)
    return sorted(set(n for n in names if not n.endswith("_t")))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    declared = _declared_functions()
    assert len(declared) >= 10
    bound = {n for n, _, _ in _lib.SYMBOLS}
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/r3dg_b200.h but not exported"
        assert name in bound, f"{name} is exported but not bound in _lib.SYMBOLS"
    assert b"sm_90a" in lib.r3dg_version()


def test_struct_field_order_matches_header():
    hdr = open(os.path.join(ROOT, "include", "r3dg_b200.h")).read()
    for cname, cls in (("r3dg_raster_fwd_args", _lib.RasterFwdArgs), ("r3dg_raster_bwd_args", _lib.RasterBwdArgs),
                       ("r3dg_shade_args", _lib.ShadeArgs), ("r3dg_adam_tensor", _lib.AdamTensor)):
        body = re.search(r"typedef struct " + cname + r" \{(.*?)\} " + cname + ";", hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            names = re.sub(r"^(const\s+)?(float|int|void|size_t|long long|double)\s*\**", "", decl)
            for n in names.split(","):
                fields.append(n.replace("*", "").strip())
        assert fields == [f[0] for f in cls._fields_], cname


def test_sizing_functions_monotone_and_aligned():
    lib = _lib.load()
    g1, g2 = lib.r3dg_raster_geom_bytes(1000, 5), lib.r3dg_raster_geom_bytes(2000, 5)
    assert 0 < g1 < g2 and g1 % 256 == 0
    assert lib.r3dg_raster_geom_bytes(1000, 16) > g1
    i1 = lib.r3dg_raster_img_bytes(800, 800)
    assert i1 >= 800 * 800 * 8 and i1 % 256 == 0
    off = lib.r3dg_raster_img_n_contrib_offset(800, 800)
    assert 0 < off < i1 and off % 256 == 0
    b1, b2 = lib.r3dg_raster_binning_bytes(10_000), lib.r3dg_raster_binning_bytes(20_000)
    assert 4 * 10_000 <= b1 < b2          # one u32 list entry per (tile, Gaussian) instance


def test_bad_arguments_are_rejected_without_touching_the_gpu():
    lib = _lib.load()
    a = _lib.RasterFwdArgs()
    a.P, a.W, a.H, a.S = 10, 0, 16, 0            # zero width
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001
    a.W, a.S = 16, 99                             # too many feature channels (forward.cu:312 F[33])
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10002
    b = _lib.RasterBwdArgs()
    b.P, b.W, b.H, b.S = 10, 16, 16, 25           # backward.cu:449 limit
    assert lib.r3dg_raster_backward(ctypes.byref(b), None) == -10002


def test_tune_keys_and_error_codes():
    """r3dg_tune: every documented key round-trips, unknown keys / out-of-range values are refused (host state only)."""
    lib = _lib.load()
    prev = ctypes.c_int(-5)
    for key, ok, bad in (("composite_bulk", 1, 2), ("composite_fwd_ctas", 4, 99), ("composite_bwd_ctas", 3, -1), ("shade_group", 16, 7)):
        assert lib.r3dg_tune(key.encode(), ok, ctypes.byref(prev)) == 0, key
        old = prev.value
        assert lib.r3dg_tune(key.encode(), bad, ctypes.byref(prev)) == -10001, key          # R3DG_ERR_BAD_ARG
        assert prev.value == ok
        assert lib.r3dg_tune(key.encode(), old, None) == 0
    assert lib.r3dg_tune(b"no_such_knob", 1, None) == -10002                                  # R3DG_ERR_UNSUPPORTED
    assert lib.r3dg_tune(None, 1, None) == -10001


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(ImportError):
        _lib.load()


def test_adam_step_argument_checks_and_host_mirror():
    """r3dg_adam_step validates its host descriptor table before any launch; FusedAdam mirrors
    torch.optim.Adam's constructor / state layout and has no CPU path."""
    import torch
    from relightable3dgaussian_b200.optim import FusedAdam, install, uninstall
    lib = _lib.load()
    assert lib.r3dg_adam_step(0, None, None) == 0
    assert lib.r3dg_adam_step(1, None, None) == -10001
    t = (_lib.AdamTensor * 1)()
    t[0].n, t[0].step, t[0].lr, t[0].beta1, t[0].beta2, t[0].eps = 8, 0, 1e-3, 0.9, 0.999, 1e-15
    assert lib.r3dg_adam_step(1, t, None) == -10001          # step counts from 1
    t[0].step = 1
    assert lib.r3dg_adam_step(1, t, None) == -10001          # null tensors with n > 0
    t[0].n = 0
    assert lib.r3dg_adam_step(1, t, None) == 0               # empty tensor: nothing launched
    p = torch.zeros(4, requires_grad=True)
    opt = FusedAdam([{"params": [p], "lr": 1e-3, "name": "xyz"}], lr=0.0, eps=1e-15)
    assert opt.param_groups[0]["name"] == "xyz" and opt.param_groups[0]["eps"] == 1e-15 and opt.param_groups[0]["betas"] == (0.9, 0.999)
    p.grad = torch.ones(4)
    with pytest.raises(RuntimeError):
        opt.step()
    with pytest.raises(ValueError):
        FusedAdam([p], betas=(1.0, 0.999))
    orig = torch.optim.Adam
    try:
        assert install() is FusedAdam and torch.optim.Adam is FusedAdam
    finally:
        uninstall()
    assert torch.optim.Adam is orig

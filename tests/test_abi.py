"""C-ABI surface: the shared library loads and exports every symbol include/r3dg_b200.h declares, the ctypes
bindings (struct layouts and function signatures) agree with the header, sizing functions are sane.  No GPU compute
is issued."""
import ctypes
import os
import re

import pytest

from helpers import ROOT
from relightable3dgaussian_b200 import _lib


C = ctypes
# header struct -> its ctypes class
STRUCTS = {"r3dg_raster_fwd_args": _lib.RasterFwdArgs, "r3dg_raster_bwd_args": _lib.RasterBwdArgs,
           "r3dg_exchange_args": _lib.ExchangeArgs, "r3dg_pack_src": _lib.PackSrc,
           "r3dg_compact_tensor": _lib.CompactTensor, "r3dg_densify_tensor": _lib.DensifyTensor,
           "r3dg_densify_thresholds": _lib.DensifyThresholds, "r3dg_shade_args": _lib.ShadeArgs,
           "r3dg_adam_tensor": _lib.AdamTensor}
SCALARS = {"int": C.c_int, "long long": C.c_longlong, "unsigned long long": C.c_ulonglong, "size_t": C.c_size_t,
           "float": C.c_float, "double": C.c_double, "uint8_t": C.c_uint8, "int32_t": C.c_int32, "uint64_t": C.c_uint64}


def _ctype_name(t):
    if isinstance(t, type) and issubclass(t, C.Array):
        return f"{_ctype_name(t._type_)}[{t._length_}]"
    if isinstance(t, type) and issubclass(t, C._Pointer):
        return f"POINTER({_ctype_name(t._type_)})"
    return getattr(t, "__name__", repr(t))


def _type(decl):
    """C type of a declaration without its name, normalised: no `const`, single spaces, `*` attached."""
    t = " ".join(decl.replace("const ", " ").replace("*", " * ").split())
    return t.replace(" *", "*")


def parse_header():
    """({struct: [(field, C type, array length or None)]}, {function: (return type, [parameter types])}) of
    include/r3dg_b200.h, comments stripped."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "r3dg_b200.h")).read(), flags=re.S)
    structs = {}
    for name, body, alias in re.findall(r"typedef struct (\w+) \{(.*?)\} (\w+);", src, re.S):
        assert name == alias, name
        fields = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            base, names = re.fullmatch(r"((?:const\s+)?(?:unsigned\s+)?(?:long\s+long|\w+))\s*(.*)", decl, re.S).groups()
            for n in names.split(","):
                stars, field, length = re.fullmatch(r"\s*(\**)\s*(\w+)\s*(?:\[(\d+)\])?\s*", n).groups()
                fields.append((field, _type(base + stars), int(length) if length else None))
        structs[name] = fields
    src = re.sub(r"^[ \t]*#.*$", ";", re.sub(r"typedef struct \w+ \{.*?\} \w+;", ";", src, flags=re.S), flags=re.M)
    protos = {}
    for ret, name, params in re.findall(r"([A-Za-z_][\w\s*]*?)\b(r3dg_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src):
        params = [p.strip() for p in params.split(",")]
        protos[name] = (_type(ret), [] if params == ["void"] else [_type(re.fullmatch(r"(.*?)\w+", p, re.S).group(1))
                                                                   for p in params])
    return structs, protos


def _expected_field(ctype, length):
    t = C.c_void_p if ctype.endswith("*") else SCALARS[ctype]
    return t * length if length else t


def _param_ok(ctype, bound):
    """Scalars exactly; a header struct by POINTER(its class); `const char*` as c_char_p; any other pointer and the
    stream as c_void_p or POINTER of the matching scalar."""
    if ctype in SCALARS:
        return bound is SCALARS[ctype]
    if ctype.endswith("*") and ctype[:-1] in STRUCTS:
        return bound is C.POINTER(STRUCTS[ctype[:-1]])
    if ctype == "char*":
        return bound is C.c_char_p
    if ctype.endswith("*") and ctype[:-1] in SCALARS and bound is C.POINTER(SCALARS[ctype[:-1]]):
        return True
    return bound is C.c_void_p and (ctype.endswith("*") or ctype == "r3dg_stream_t")


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    _, protos = parse_header()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "r3dg_b200.h")).read(), flags=re.S)
    assert set(protos) == {n for n in re.findall(r"\b(r3dg_[a-z0-9_]+)\s*\(", hdr) if not n.endswith("_t")}
    assert len(protos) >= 10
    bound = {n for n, _, _ in _lib.SYMBOLS}
    for name in sorted(protos):
        assert hasattr(lib, name), f"{name} declared in include/r3dg_b200.h but not exported"
        assert name in bound, f"{name} is exported but not bound in _lib.SYMBOLS"
    assert b"sm_90a" in lib.r3dg_version()


def test_struct_field_order_matches_header():
    """Every struct of the header has a ctypes class whose fields match it in order, name, type and array length."""
    structs, _ = parse_header()
    assert sorted(structs) == sorted(STRUCTS)
    for cname, fields in structs.items():
        cls = STRUCTS[cname]
        assert [f[0] for f in cls._fields_] == [f[0] for f in fields], cname
        for (field, ctype, length), (_, bound) in zip(fields, cls._fields_):
            want = _expected_field(ctype, length)
            assert bound is want, f"{cname}.{field}: header {ctype}{f'[{length}]' if length else ''}, bound as " \
                                  f"{_ctype_name(bound)} (expected {_ctype_name(want)})"
    for cls in (_lib.RasterFwdArgs, _lib.RasterBwdArgs, _lib.ShadeArgs):
        assert [f[0] for f in cls._fields_[-3:]] == ["deterministic", "det_work", "det_work_bytes"]


def test_symbols_match_prototypes():
    """Every _lib.SYMBOLS binding has its prototype's return type and the number and types of its parameters."""
    _, protos = parse_header()
    for name, restype, argtypes in _lib.SYMBOLS:
        assert name in protos, f"{name} is bound but not declared in include/r3dg_b200.h"
        ret, params = protos[name]
        assert _param_ok(ret, restype), f"{name} returns {ret}, bound as {_ctype_name(restype)}"
        assert len(argtypes) == len(params), f"{name} takes {len(params)} arguments ({params}), bound with {len(argtypes)}"
        for k, (ctype, bound) in enumerate(zip(params, argtypes)):
            assert _param_ok(ctype, bound), f"{name} argument {k}: header {ctype}, bound as {_ctype_name(bound)}"


# Shapes at the edges of the work-buffer layout: P = 0 (sized as one Gaussian), record widths of one to nine float4
# groups, images of one pixel, one tile row and more than 256 tile columns, capacities around the 64-instance granule.
SIZING_P, SIZING_S = (0, 1, 1000, 10**6), (0, 5, 16, 24, 33)
SIZING_WH = ((1, 1), (37, 1), (800, 800), (1920, 1080), (4100, 16))
SIZING_CAP = (0, 1, 63, 64, 10**6)


def _sizing(lib):
    return {"geom": [lib.r3dg_raster_geom_bytes(P, S) for P in SIZING_P for S in SIZING_S],
            "img": [lib.r3dg_raster_img_bytes(W, H) for W, H in SIZING_WH],
            "n_contrib": [lib.r3dg_raster_img_n_contrib_offset(W, H) for W, H in SIZING_WH],
            "binning": [lib.r3dg_raster_binning_bytes(c) for c in SIZING_CAP],
            "fwd_det": [lib.r3dg_raster_fwd_det_bytes(P) for P in SIZING_P],
            "bwd_det": [lib.r3dg_raster_bwd_det_bytes(P, S) for P in SIZING_P for S in SIZING_S]}


# The sizes callers allocate: any change here is a change of the work-buffer layout.
SIZING = {"geom": [11264, 11264, 11264, 11264, 11264,
                   11264, 11264, 11264, 11264, 11264,
                   142848, 174592, 270848, 334848, 398848,
                   134010112, 166010112, 262010112, 326010112, 390010112],
          "img": [6144, 14336, 15461376, 50338816, 1589248],
          "n_contrib": [256, 256, 2560000, 8294400, 262400],
          "binning": [1152, 1152, 1152, 1152, 6000768],
          "fwd_det": [256, 256, 8192, 8000000],
          "bwd_det": [768, 768, 1024, 1280, 1536,
                      768, 768, 1024, 1280, 1536,
                      291072, 388096, 679168, 873216, 1067008,
                      291000064, 388000000, 679000064, 873000192, 1067000064]}
# The same with R3DG_BIN_MAX_CHUNKS=3: only the binning matrix in the img buffer shrinks.
SIZING_IMG_3_CHUNKS = [2048, 2048, 5251328, 17013248, 539648]


def test_sizing_functions_monotone_and_aligned(monkeypatch):
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
    assert _sizing(lib) == SIZING
    monkeypatch.setenv("R3DG_BIN_MAX_CHUNKS", "3")
    assert _sizing(lib) == dict(SIZING, img=SIZING_IMG_3_CHUNKS)


FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued


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

    # work buffers smaller than the sizing functions ask for; 1151 bytes of binning buffer hold no instance
    P, S, W, H = 100, 5, 64, 48
    short = (("geom_bytes", lib.r3dg_raster_geom_bytes(P, S) - 1), ("img_bytes", lib.r3dg_raster_img_bytes(W, H) - 1),
             ("binning_bytes", 1151))
    for call, cls in ((lib.r3dg_raster_forward, _lib.RasterFwdArgs), (lib.r3dg_raster_backward, _lib.RasterBwdArgs)):
        for field, size in short:
            a = cls()
            a.P, a.S, a.W, a.H = P, S, W, H
            if cls is _lib.RasterFwdArgs:
                a.colors_precomp = a.cov3D_precomp = FAKE
            a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
            a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(W, H)
            a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
            setattr(a, field, size)
            assert call(ctypes.byref(a), None) == -10001, (call.__name__, field)
    b = _lib.RasterBwdArgs()
    b.P, b.S, b.W, b.H = 0, S, W, H               # no Gaussians: nothing to do, the buffers are not needed
    assert lib.r3dg_raster_backward(ctypes.byref(b), None) == 0

    def debug_copy(id_, max_bytes, binning_bytes):
        return lib.r3dg_raster_debug_copy(id_, P, S, W, H, FAKE, FAKE, FAKE, binning_bytes, FAKE, max_bytes, None)
    for id_, row_bytes in ((0, 4), (1, 3), (3, 8), (5, 16), (6, 12), (8, 4)):
        assert debug_copy(id_, row_bytes * P - 1, lib.r3dg_raster_binning_bytes(10_000)) == -1, id_
    for id_ in (-1, 2, 11, 21):
        assert debug_copy(id_, 1 << 20, lib.r3dg_raster_binning_bytes(10_000)) == -1, id_
    for id_ in (9, 10, 18, 19):                   # the binning lists need a binning buffer
        assert debug_copy(id_, 1 << 20, 0) == -1, id_


def test_misaligned_rotations_are_refused_before_any_launch():
    """rotations is read, and dL_drotations written, as float4: a base that is not 16-byte aligned is refused.  The
    aligned twin of each refused call is one that returns 0 without launching anything (P = 0)."""
    lib = _lib.load()
    odd = FAKE + 4
    a = _lib.RasterFwdArgs()
    a.P, a.S, a.W, a.H = 100, 0, 64, 48
    a.shs, a.scales, a.rotations = FAKE, FAKE, odd
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001
    for field in ("rotations", "dL_drotations"):
        for ptr, want in ((odd, -10001), (FAKE + 8, -10001), (FAKE, 0)):
            b = _lib.RasterBwdArgs()
            b.P, b.S, b.W, b.H = 0, 5, 64, 48
            setattr(b, field, ptr)
            assert lib.r3dg_raster_backward(ctypes.byref(b), None) == want, (field, hex(ptr))
    for ptr, want in ((odd, -10001), (FAKE, 0)):
        assert lib.r3dg_bvh_leaf_aabbs(0, None, None, ptr, None, None, None) == want
        totals = (ctypes.c_int * 7)()
        assert lib.r3dg_densify_apply(0, totals, 0, None, ptr, None, None, 0.625, FAKE, lib.r3dg_densify_tmp_bytes(0),
                                      None) == want


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

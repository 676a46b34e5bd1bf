"""The a-trous denoiser without a GPU: the fp64 oracle (tests/denoise64.py) is linear with the header's backward as its
exact transpose, keeps constants, honours the mask; the ctypes struct matches the header; the sizing function; and the
refusals of the C entry points and of the Python wrappers (nothing is launched)."""
import ctypes
import os
import re

import pytest
import torch

import denoise64 as D64
from helpers import ROOT
from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200 import denoise as dn

D = torch.float64


@pytest.mark.parametrize("V,H,W,C,F,L", [(1, 9, 11, 3, 0, 3), (2, 13, 7, 2, 2, 4), (1, 1, 6, 1, 1, 2), (1, 5, 5, 8, 8, 6)])
def test_oracle_transpose_is_the_adjoint(V, H, W, C, F, L):
    """<A x, g> = <x, A^T g> to 1e-12, with A^T the header's backward formula; it is also autograd's gradient."""
    normal, points, mask, feats = D64.gbuffer(V, H, W, F, seed=V * 7 + L)
    g = torch.Generator().manual_seed(L)
    x = torch.randn(V, C, H, W, generator=g, dtype=D).requires_grad_()
    cot = torch.randn(V, C, H, W, generator=g, dtype=D)
    kw = dict(passes=L, sigma_normal=64.0, sigma_plane=0.2, sigma_features=0.15)
    y = D64.atrous(x, normal, points, mask, feats, **kw)
    at = D64.transpose(cot, normal, points, mask, feats, **kw)
    lhs, rhs = float((y.detach() * cot).sum()), float((x.detach() * at).sum())
    assert abs(lhs - rhs) <= 1e-12 * (abs(lhs) + (y.abs() * cot.abs()).sum().item())
    (y * cot).sum().backward()
    assert torch.allclose(x.grad, at, rtol=1e-12, atol=1e-14)
    w = D64.weights(D64.guides(normal, points, mask, feats), 1, 64.0, 0.2, 0.15)
    off = sum(v for k, v in w.items() if k != (0, 0))
    assert float(off.max()) > 0.02                        # the guides leave real weight on the neighbours


def test_constant_on_a_connected_valid_region_stays_constant():
    """A constant on the valid pixels (garbage, NaN included, on the invalid ones) is kept exactly; invalid are 0."""
    normal, points, mask, feats = D64.gbuffer(2, 16, 20, 1, seed=3)
    x = torch.full((2, 2, 16, 20), 0.7, dtype=D)
    x[:, 1] = -2.5
    x[~mask[:, None].expand_as(x)] = float("nan")
    y = D64.atrous(x, normal, points, mask, feats, passes=5)
    keep = mask[:, None].expand_as(y)
    assert torch.allclose(y[:, 0][mask], torch.full_like(y[:, 0][mask], 0.7), rtol=1e-14)
    assert torch.allclose(y[:, 1][mask], torch.full_like(y[:, 1][mask], -2.5), rtol=1e-14)
    assert torch.all(y[~keep] == 0)


def test_mask_semantics():
    """Masked pixels output 0, get gradient 0, and their input values change nothing."""
    normal, points, mask, _ = D64.gbuffer(1, 12, 14, 0, seed=5)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 3, 12, 14, generator=g, dtype=D).requires_grad_()
    y = D64.atrous(x, normal, points, mask, passes=3)
    inv = ~mask[:, None].expand_as(y)
    assert torch.all(y[inv] == 0)
    x2 = x.detach().clone()
    x2[inv] = 1e6
    assert torch.equal(D64.atrous(x2, normal, points, mask, passes=3), y.detach())
    y.sum().backward()
    assert torch.all(x.grad[inv] == 0) and torch.all(x.grad[~inv] != 0)
    # a masked neighbour is not a tap: no mask is the same as a mask of all ones
    ones = torch.ones_like(mask)
    assert torch.equal(D64.atrous(x.detach(), normal, points, ones, passes=3), D64.atrous(x.detach(), normal, points, passes=3))


def test_edges_stop_the_filter():
    """Across the crease and the depth step the weights nearly vanish; on each plane they do not."""
    normal, points, _, _ = D64.gbuffer(1, 20, 20, 0, seed=2, masked=False)
    w = D64.weights(D64.guides(normal, points), 1, 128.0, 0.1, 0.1)
    # pixel (10, 11) sits on the ground left of the crease (x = 0.575), pixel (10, 13) on the wall
    assert float(w[(0, 2)][0, 10, 11]) < 1e-6 and float(w[(0, -2)][0, 10, 13]) < 1e-6
    assert float(w[(0, -1)][0, 10, 10]) > 0.005
    # the depth step: row 5 (y = 0.275) is the near ground, row 6 the far ground; normals are parallel
    assert float(w[(1, 0)][0, 5, 3]) < 1e-3 and float(w[(-1, 0)][0, 4, 3]) > 0.005


# ---- the ABI and the refusals -----------------------------------------------------------------------------------------
def test_ctypes_struct_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "r3dg_b200.h")).read(), flags=re.S)
    body = re.search(r"struct r3dg_denoise_args \{(.*?)\};", src, re.S).group(1)
    names = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names += [n.strip().lstrip("*") for n in re.sub(r"^(const\s+)?\w+\s*\**", "", decl).split(",")]
    assert names == [n for n, _ in _lib.DenoiseArgs._fields_]
    ptr = ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(_lib.DenoiseArgs) == 6 * 4 + 3 * 4 + 4 + 9 * ptr + 8      # 4 bytes of padding after the sigmas
    for name, value in (("R3DG_DENOISE_MAX_CHANNELS", dn.MAX_CHANNELS), ("R3DG_DENOISE_MAX_FEATURES", dn.MAX_FEATURES),
                        ("R3DG_DENOISE_MAX_PASSES", dn.MAX_PASSES), ("R3DG_MAX_VIEWS", dn.MAX_VIEWS)):
        assert re.search(rf"#define {name} (\d+)", src).group(1) == str(value)


def test_work_bytes():
    lib = _lib.load()
    a = lambda n: (n + 255) // 256 * 256
    npix = 3 * 17 * 29
    for F, planes in ((0, 2), (1, 2), (2, 3), (5, 3), (6, 4), (8, 4)):
        assert lib.r3dg_denoise_work_bytes(3, 17, 29, 5, F, 4) == a(planes * 16 * npix) + a(4 * 4 * npix) + a(5 * 4 * npix)
    for bad in ((0, 4, 4, 1, 0, 1), (1, 0, 4, 1, 0, 1), (1, 4, 4, 0, 0, 1), (1, 4, 4, 1, -1, 1), (1, 4, 4, 1, 0, 0)):
        assert lib.r3dg_denoise_work_bytes(*bad) == 0
    assert lib.r3dg_denoise_work_bytes(4, 1080, 1920, 3, 1, 5) == a(32 * 4 * 1080 * 1920) + a(4 * 5 * 4 * 1080 * 1920) + \
        a(4 * 3 * 4 * 1080 * 1920)


FAKE = 0x10000                 # never dereferenced: every call below is refused before anything is enqueued


def _fake_args(**kw):
    a = _lib.DenoiseArgs()
    a.V, a.H, a.W, a.C, a.F, a.L = 1, 8, 8, 3, 1, 4
    a.sigma_normal, a.sigma_plane, a.sigma_features = 128.0, 0.1, 0.1
    for f in ("normal", "points", "features", "x", "y", "dL_dy", "dL_dx", "work"):
        setattr(a, f, FAKE)
    a.work_bytes = 1 << 40
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _calls(a):
    lib = _lib.load()
    return lib.r3dg_denoise_forward(ctypes.byref(a), None), lib.r3dg_denoise_backward(ctypes.byref(a), None)


@pytest.mark.parametrize("kw,rc", [
    (dict(V=0), -10001), (dict(V=65), -10001), (dict(H=0), -10001), (dict(W=0), -10001),
    (dict(C=0), -10001), (dict(C=9), -10001), (dict(F=-1), -10001), (dict(F=9), -10001),
    (dict(L=0), -10001), (dict(L=7), -10001),
    (dict(sigma_normal=0.0), -10001), (dict(sigma_plane=-1.0), -10001), (dict(sigma_features=float("inf")), -10001),
    (dict(sigma_plane=float("nan")), -10001),
    (dict(work=None), -10001), (dict(work_bytes=100), -10001),
    (dict(V=64, H=2 ** 12, W=2 ** 12, C=2, F=0, work_bytes=1 << 62), -10002),      # V H W C = 2^31
    (dict(V=1, H=2 ** 14, W=2 ** 14, C=1, F=8, work_bytes=1 << 62), -10002),       # V H W F = 2^31
])
def test_c_entry_points_refuse_before_any_launch(kw, rc):
    assert _calls(_fake_args(**kw)) == (rc, rc)


def test_each_direction_refuses_its_own_missing_pointers():
    lib = _lib.load()
    for f in ("normal", "points", "features", "x", "y"):
        assert lib.r3dg_denoise_forward(ctypes.byref(_fake_args(**{f: None})), None) == -10001, f
    for f in ("dL_dy", "dL_dx"):
        assert lib.r3dg_denoise_backward(ctypes.byref(_fake_args(**{f: None})), None) == -10001, f
    short = lib.r3dg_denoise_work_bytes(1, 8, 8, 3, 1, 4) - 1
    assert _calls(_fake_args(work_bytes=short)) == (-10001, -10001)


def _images(V=None, H=6, W=7, C=3):
    lead = () if V is None else (V,)
    return dict(x=torch.rand(*lead, C, H, W), normal=torch.rand(*lead, 3, H, W), points=torch.rand(*lead, 3, H, W))


@pytest.mark.parametrize("change,err,match", [
    (dict(x=torch.rand(6, 7)), ValueError, "x must be"),
    (dict(x=torch.rand(1, 1, 3, 6, 7)), ValueError, "x must be"),
    (dict(x=torch.rand(9, 6, 7)), ValueError, "1 to 8 channels"),
    (dict(x=torch.rand(0, 6, 7)), ValueError, "1 to 8 channels"),
    (dict(x=torch.rand(65, 3, 2, 2), normal=torch.rand(65, 3, 2, 2), points=torch.rand(65, 3, 2, 2)), ValueError, "views"),
    (dict(normal=torch.rand(3, 6, 8)), ValueError, "does not match"),
    (dict(normal=torch.rand(2, 3, 6, 7)), ValueError, "does not match"),
    (dict(points=torch.rand(4, 6, 7)), ValueError, "3 channels"),
    (dict(features=torch.rand(9, 6, 7)), ValueError, "features"),
    (dict(features=torch.rand(1, 5, 7)), ValueError, "does not match"),
    (dict(mask=torch.ones(6, 7)), ValueError, "mask"),
    (dict(mask=torch.ones(6, 8, dtype=torch.bool)), ValueError, "mask"),
    (dict(passes=0), ValueError, "passes"),
    (dict(passes=7), ValueError, "passes"),
    (dict(passes=2.5), ValueError, "passes"),
    (dict(sigma_normal=0), ValueError, "sigma_normal"),
    (dict(sigma_plane=-0.1), ValueError, "sigma_plane"),
    (dict(sigma_features=float("nan")), ValueError, "sigma_features"),
    (dict(sigma_plane=float("inf")), ValueError, "sigma_plane"),
    (dict(), RuntimeError, "CUDA"),                                    # CPU tensors
])
def test_atrous_refuses(change, err, match):
    args = dict(_images(), mask=None, features=None)
    args.update(change)
    with pytest.raises(err, match=match):
        dn.atrous(args.pop("x"), args.pop("normal"), args.pop("points"), **args)


def test_atrous_refuses_the_32_bit_bound_without_allocating():
    big = lambda C: torch.zeros(1).expand(8, C, 2 ** 14, 2 ** 14)     # V H W C >= 2^31, no storage
    with pytest.raises(ValueError, match="2\\^31"):
        dn.atrous(big(2), big(3), big(3))
    with pytest.raises(ValueError, match="2\\^31"):
        dn.atrous(torch.zeros(1).expand(1, 1, 2 ** 14, 2 ** 14), torch.zeros(1).expand(1, 3, 2 ** 14, 2 ** 14),
                  torch.zeros(1).expand(1, 3, 2 ** 14, 2 ** 14), features=torch.zeros(1).expand(1, 8, 2 ** 14, 2 ** 14))


def test_denoise_shading_refuses_before_any_launch():
    im = _images()
    out = {"diffuse_light": im["x"], "specular": im["x"], "pbr": im["x"]}
    rough, base = torch.rand(1, 6, 7), torch.rand(3, 6, 7)
    with pytest.raises(ValueError, match="roughness"):
        dn.denoise_shading(out, base, torch.rand(2, 6, 7), im["normal"], im["points"])
    with pytest.raises(ValueError, match="base_color"):
        dn.denoise_shading(out, torch.rand(3, 6, 6), rough, im["normal"], im["points"])
    with pytest.raises(ValueError, match="specular"):
        dn.denoise_shading(dict(out, specular=torch.rand(3, 5, 7)), base, rough, im["normal"], im["points"])
    with pytest.raises(ValueError, match="passes"):
        dn.denoise_shading(out, base, rough, im["normal"], im["points"], passes=9)
    with pytest.raises(RuntimeError, match="CUDA"):
        dn.denoise_shading(out, base, rough, im["normal"], im["points"])

"""Per-pixel lights without a GPU: the fp64 pixel oracle (tests/pixel_lights64.py) against the row oracles of
lights64 and shaped_lights64, the ctypes struct against the header, the sizing function, and the refusals of the host
wrappers and of the C entry points (nothing is launched)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import lights64 as L64
import pixel_lights64 as PL64
import shaped_lights64 as S64
from helpers import ROOT
from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200 import lights as lt
from relightable3dgaussian_b200.raytracer import RayTracer

D = torch.float64


def _gbuffer(V, H, W, R, seed=0):
    g = torch.Generator().manual_seed(900 + seed)
    n = torch.randn(V, 3, H, W, generator=g)
    return dict(base_color=torch.rand(V, 3, H, W, generator=g) * 0.8 + 0.05,
                roughness=torch.rand(V, 1, H, W, generator=g) * 0.9 + 0.08,
                normal=n * (0.5 + torch.rand(V, 1, H, W, generator=g)),
                points=torch.randn(V, 3, H, W, generator=g) * 0.5,
                campos=torch.randn(V, 3, generator=g) * 0.3 + torch.tensor([0.0, -2.5, 1.7]),
                T=torch.rand(V, R, H, W, generator=g),
                mask=torch.rand(V, H, W, generator=g) < 0.7)


def _point_set():
    kind = np.array([0, 1, 1], np.int32)
    return kind, (torch.tensor([[0.3, 0.2, 1.0], [0.5, -0.4, 1.2], [-0.6, 0.1, 0.8]]), torch.rand(3, 3) * 2)


def _shaped_set(M):
    kind = np.array([3, 2, 3], np.int32)
    fields = (torch.tensor([[0.0, 0.0, 1.5], [0.6, -0.2, 1.1], [-0.5, 0.4, 1.3]]),
              torch.tensor([[0.3, 0.0, 0.0], [-0.3, 0.1, -1.0], [0.0, 0.2, 0.1]]),
              torch.tensor([[0.0, 0.2, 0.05], [0.0, 0.0, 0.0], [0.25, 0.0, 0.0]]),
              torch.rand(3, 3) * 2, torch.tensor([[0.0, 0.0], [0.9, 0.5], [0.0, 0.0]]))
    return kind, fields


@pytest.mark.parametrize("family", ["point", "shaped"])
@pytest.mark.parametrize("V,H,W", [(1, 1, 1), (2, 5, 7)])
def test_pixel_oracle_is_the_row_oracle_per_pixel(family, V, H, W):
    M, seed = 2, 31
    kind, fields = _point_set() if family == "point" else _shaped_set(M)
    R, shaped = PL64.columns(kind, M)
    c = _gbuffer(V, H, W, R)
    got = PL64.shade_pixels(c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], kind, fields,
                            M, seed, c["mask"])
    for v in range(V):
        pts = PL64.rows(c["points"][v])
        vd = (c["campos"][v][None] - pts).double()[None]
        args = (PL64.rows(c["base_color"][v]).double(), PL64.rows(c["roughness"][v]).double(),
                PL64.rows(c["normal"][v]).double(), vd, pts.double(), kind)
        Tv = PL64.rows(c["T"][v]).double()
        if shaped:
            _, st = S64.ray_targets(list(kind), *(f.numpy() for f in fields[:3]), M, seed, H * W)   # row g = pixel p
            want = S64.shade(*args, *[f.double() for f in fields], Tv, M, st)
        else:
            want = L64.shade(*args, *[f.double() for f in fields], Tv)
        keep = c["mask"][v].reshape(-1)
        for k, w in zip(("pbr", "diffuse_light", "specular"), want):
            x = PL64.rows(got[k][v])
            assert x.dtype == D and torch.equal(x[keep], w[0][keep]), k
            assert torch.all(x[~keep] == 0), k


def test_rect_samples_follow_the_pixel_index_not_the_view():
    """Two views of the same images give the same terms; moving a pixel to another index changes its rect samples."""
    M, seed = 2, 5
    kind, fields = _shaped_set(M)
    R, _ = PL64.columns(kind, M)
    c = _gbuffer(1, 3, 4, R)
    two = {k: torch.cat([c[k], c[k]]) for k in ("base_color", "roughness", "normal", "points", "T")}
    one = PL64.shade_pixels(c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], kind, fields, M, seed)
    both = PL64.shade_pixels(*(two[k] for k in ("base_color", "roughness", "normal", "points")), c["campos"].repeat(2, 1),
                             two["T"], kind, fields, M, seed)
    for k in one:
        assert torch.equal(both[k][0], one[k][0]) and torch.equal(both[k][1], one[k][0])
    flip = {k: c[k].flip(-1) for k in ("base_color", "roughness", "normal", "points", "T")}
    moved = PL64.shade_pixels(*(flip[k] for k in ("base_color", "roughness", "normal", "points")), c["campos"], flip["T"],
                              kind, fields, M, seed)
    assert not torch.equal(moved["pbr"].flip(-1), one["pbr"])


def _scene(P, seed):
    rng = np.random.default_rng(seed)
    means = (rng.standard_normal((P, 3)) * 0.4).astype(np.float32)
    s = rng.uniform(0.03, 0.12, (P, 3))
    inv_cov = np.stack([1 / s[:, 0] ** 2, 0 * s[:, 0], 0 * s[:, 0], 1 / s[:, 1] ** 2, 0 * s[:, 0], 1 / s[:, 2] ** 2], 1)
    normals = rng.standard_normal((P, 3)).astype(np.float32)
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    opacity = rng.uniform(0.3, 0.99, P).astype(np.float32)
    boxes = np.tile(np.array([[-1e3, -1e3, -1e3, 1e3, 1e3, 1e3]], np.float32), (P, 1))     # no culling
    return means, inv_cov.astype(np.float32), opacity, normals, boxes


@pytest.mark.parametrize("family", ["point", "shaped"])
def test_pixel_shadows_from_gaussian_means_are_the_row_shadows(family):
    """A G-buffer whose pixel p holds Gaussian p's mean: the pixel oracle's T equals the row oracle's row p."""
    M, seed = 2, 9
    kind, fields = _point_set() if family == "point" else _shaped_set(M)
    f = [x.numpy() for x in fields]
    R, shaped = PL64.columns(kind, M)
    P, H, W = 24, 4, 6
    means, inv_cov, opacity, normals, boxes = _scene(P, 3)
    pts = means.T.reshape(1, 3, H, W)
    pixels = [(0, p) for p in range(H * W)]
    T, fr = PL64.shadows(pts, means, inv_cov, opacity, normals, boxes, kind, f, M, seed, pixels)
    pairs = [(g, j) for g in range(P) for j in range(R)]
    if shaped:
        T64, fr64 = S64.shadows(means, inv_cov, opacity, normals, boxes, kind, *f[:3], M, seed, pairs)
    else:
        T64, fr64 = L64.shadows(means, inv_cov, opacity, normals, boxes, kind, f[0], pairs=pairs)
    assert np.array_equal(T.reshape(R, P).T, T64) and np.array_equal(fr.reshape(R, P).T, fr64)
    assert (T64 < 1).any() and (T64 > 0.5).any()


# ---- the ABI and the refusals -----------------------------------------------------------------------------------------
def test_ctypes_struct_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "r3dg_b200.h")).read(), flags=re.S)
    body = re.search(r"struct r3dg_pixel_light_args \{(.*?)\};", src, re.S).group(1)
    names = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names += [n.strip().lstrip("*") for n in re.sub(r"^(const\s+)?\w+\s*\**", "", decl).split(",")]
    assert names == [n for n, _ in _lib.PixelLightArgs._fields_]
    ptr = ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(_lib.PixelLightArgs) == 6 * 4 + 27 * ptr + 8
    lib = _lib.load()
    for name in ("r3dg_bvh_trace_pixel_lights", "r3dg_shade_pixel_lights_forward", "r3dg_shade_pixel_lights_backward"):
        assert hasattr(lib, name)


def test_work_bytes():
    lib = _lib.load()
    assert lib.r3dg_shade_pixel_lights_work_bytes(1, 4, 4, 0) == 0
    assert lib.r3dg_shade_pixel_lights_work_bytes(0, 4, 4, 3) == 0
    assert lib.r3dg_shade_pixel_lights_work_bytes(1, 1, 1, 1) == 16 * 4                 # one CTA, 16 slots per light
    assert lib.r3dg_shade_pixel_lights_work_bytes(1, 16, 16, 2) == 2 * 16 * 2 * 4      # 256 pixels: 2 CTAs of 128
    # the grid stops growing at 2048 CTAs, so the workspace of a large call is bounded
    assert lib.r3dg_shade_pixel_lights_work_bytes(64, 1080, 1920, 32) == 2048 * 16 * 32 * 4
    assert lib.r3dg_bvh_trace_pixel_lights_tmp_bytes(10) == lib.r3dg_bvh_trace_lights_tmp_bytes(10)


FAKE = 0x10000                 # never dereferenced: every call below is refused before anything is enqueued


def _fake_args(kind, **kw):
    keep = np.ascontiguousarray(kind, np.int32)
    a = _lib.PixelLightArgs()
    a.V, a.H, a.W, a.K, a.M = 1, 4, 4, keep.size, 2
    a.kind = keep.ctypes.data if keep.size else None
    for f in ("pos", "a", "b", "color", "cone", "base_color", "roughness", "normal", "points", "campos", "shadows", "pbr",
              "diffuse_light", "specular", "dL_dpbr", "dL_dbase_color", "dL_droughness", "dL_dpos", "dL_da", "dL_db",
              "dL_dcolor", "dL_dcone", "work"):
        setattr(a, f, FAKE)
    a.work_bytes = 1 << 30
    for k, v in kw.items():
        setattr(a, k, v)
    return a, keep


def _calls(a):
    lib = _lib.load()
    tmp = lib.r3dg_bvh_trace_pixel_lights_tmp_bytes(10)
    return (lib.r3dg_shade_pixel_lights_forward(ctypes.byref(a), None),
            lib.r3dg_shade_pixel_lights_backward(ctypes.byref(a), None),
            lib.r3dg_bvh_trace_pixel_lights(ctypes.byref(a), 10, *[FAKE] * 8, tmp, None))


@pytest.mark.parametrize("kind,kw,rc", [
    ([0, 2], {}, -10001),                                    # mixed families
    ([1, 3], {}, -10001),
    ([3, 1], {}, -10001),
    ([4], {}, -10001),                                       # no such kind
    ([-1], {}, -10001),
    ([1] * 33, {}, -10001),                                  # K > 32
    ([1], dict(M=0), -10001),                                # M outside 1..8, for either family
    ([3], dict(M=9), -10001),
    ([3] * 5, dict(M=8), -10001),                            # R = 320 > 256
    ([1], dict(V=0), -10001),
    ([1], dict(V=65), -10001),
    ([1], dict(H=0), -10001),
    ([1], dict(W=0), -10001),
    ([1], dict(points=None), -10001),
    ([1], dict(pos=None), -10001),
    ([3], dict(b=None), -10001),                             # a rect needs u and v
    ([1], dict(V=64, H=2 ** 13, W=2 ** 13), -10002),         # V H W > 2^31 - 1
])
def test_c_entry_points_refuse_before_any_launch(kind, kw, rc):
    a, keep = _fake_args(kind, **kw)
    assert _calls(a) == (rc, rc, rc)


def test_shading_and_trace_refuse_their_own_missing_pointers():
    lib = _lib.load()
    tmp = lib.r3dg_bvh_trace_pixel_lights_tmp_bytes(10)
    for f in ("color", "base_color", "roughness", "normal", "campos", "shadows"):
        a, keep = _fake_args([1], **{f: None})
        assert _calls(a)[:2] == (-10001, -10001), f
    a, keep = _fake_args([2], cone=None)                     # a spot's cone: shading only
    assert _calls(a)[:2] == (-10001, -10001)
    for f in ("pbr", "diffuse_light", "specular"):
        a, keep = _fake_args([1], **{f: None})
        assert lib.r3dg_shade_pixel_lights_forward(ctypes.byref(a), None) == -10001, f
    for f in ("dL_dpbr", "dL_dbase_color", "dL_droughness", "dL_dpos", "dL_dcolor"):
        a, keep = _fake_args([1], **{f: None})
        assert lib.r3dg_shade_pixel_lights_backward(ctypes.byref(a), None) == -10001, f
    for f in ("dL_da", "dL_db", "dL_dcone"):
        a, keep = _fake_args([3, 2], **{f: None})
        assert lib.r3dg_shade_pixel_lights_backward(ctypes.byref(a), None) == -10001, f
    a, keep = _fake_args([1], work_bytes=lib.r3dg_shade_pixel_lights_work_bytes(1, 4, 4, 1) - 1)
    assert lib.r3dg_shade_pixel_lights_backward(ctypes.byref(a), None) == -10001
    a, keep = _fake_args([1])
    assert lib.r3dg_bvh_trace_pixel_lights(ctypes.byref(a), 10, *[FAKE] * 8, tmp - 1, None) == -10001
    assert lib.r3dg_bvh_trace_pixel_lights(ctypes.byref(a), 0, *[FAKE] * 8, tmp, None) == -10001


def test_host_wrappers_refuse_cpu_tensors_and_bad_shapes():
    c = _gbuffer(1, 4, 4, 2)
    pts = lt.Lights.point(torch.zeros(2, 3), torch.ones(2, 3))
    img = lambda k: c[k][0]
    with pytest.raises(RuntimeError, match="CUDA"):
        lt.shade_pixels(img("base_color"), img("roughness"), img("normal"), img("points"), c["campos"][0], pts, img("T"))
    with pytest.raises(RuntimeError, match="GPU"):
        RayTracer.trace_pixel_lights(None, img("points"), pts, torch.zeros(4, 3), torch.zeros(4, 6), torch.zeros(4),
                                     torch.zeros(4, 3))
    with pytest.raises(TypeError, match="Lights"):
        lt.pixel_light_args(object(), img("points"), None)
    assert lt.num_rays(pts) == 2
    assert lt.num_rays(lt.ShapedLights.rect(torch.zeros(2, 3), torch.ones(2, 3), torch.ones(2, 3), torch.ones(2, 3), M=3)) == 18

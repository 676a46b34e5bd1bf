"""The lights' fp64 truth (tests/lights64.py) against the shading step's fp64 restatement and analytic shadows, and the
refusals of the C layer and of the Python layer that need no GPU."""
import ctypes

import numpy as np
import pytest
import torch

import lights64 as L64
from oracle import oracle_shading as osh
from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200.lights import Lights, shade

FAKE = 0x10000      # never dereferenced: every call below is refused (or does nothing) before anything is enqueued
D = torch.float64


def _material(P, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(P, 3, generator=g, dtype=D)
    rough = torch.rand(P, 1, generator=g, dtype=D) * 0.9 + 0.05
    normals = torch.nn.functional.normalize(torch.randn(P, 3, generator=g, dtype=D), dim=-1)
    means = torch.randn(P, 3, generator=g, dtype=D) * 0.3
    views = torch.nn.functional.normalize(torch.randn(1, P, 3, generator=g, dtype=D), dim=-1)
    return base, rough, normals, views, means


@pytest.mark.parametrize("kind", [0, 1])
def test_term_is_the_shading_step_with_one_sample(kind):
    """Each light equals oracle_shading.rendering_equation with N = 1 along l, area 1, visibility T, zero incidents
    and a constant env E."""
    P = 64
    base, rough, normals, views, means = _material(P, 1)
    g = torch.Generator().manual_seed(2)
    vec = torch.randn(1, 3, generator=g, dtype=D) * (3.0 if kind else 1.0)
    color = torch.rand(1, 3, generator=g, dtype=D) * 4
    T = torch.rand(P, 1, generator=g, dtype=D)
    pbr, diff, spec = L64.shade(base, rough, normals, views, means, [kind], vec, color, T)
    l, inv_r2, _ = L64.light_dirs([kind], vec, means)
    for p in range(P):                    # E differs per Gaussian for a point light: one constant env per row
        E = (color[0] * inv_r2[p, 0]).reshape(1, 1, 3).expand(4, 8, 3)
        r = [p, p]                        # two rows: the oracle's squeeze() needs more than one sample in all
        ref, extra = osh.rendering_equation(base[r], rough[r], normals[r], views[0, r], torch.zeros(2, 16, 3, dtype=D), E,
                                            T[r, None], l[r], torch.ones(2, 1, 1, dtype=D))
        torch.testing.assert_close(pbr[0, r], ref, rtol=1e-12, atol=1e-14)
        torch.testing.assert_close(diff[0, r], extra["diffuse_light"], rtol=1e-12, atol=1e-14)
        torch.testing.assert_close(spec[0, r], extra["specular"], rtol=1e-12, atol=1e-14)


def test_point_light_falls_off_with_the_squared_distance():
    base, rough, _, _, _ = _material(1, 3)
    means = torch.zeros(1, 3, dtype=D)
    normals = torch.tensor([[0.0, 0.0, 1.0]], dtype=D)
    views = torch.tensor([[[0.0, 0.6, 0.8]]], dtype=D)
    color = torch.tensor([[2.0, 1.0, 0.5]], dtype=D)
    T = torch.ones(1, 1, dtype=D)
    r = 1.7
    near = L64.shade(base, rough, normals, views, means, [1], torch.tensor([[0.0, 0.0, r]], dtype=D), color, T)
    far = L64.shade(base, rough, normals, views, means, [1], torch.tensor([[0.0, 0.0, 2 * r]], dtype=D), color, T)
    for a, b in zip(near, far):
        torch.testing.assert_close(b, a / 4, rtol=1e-14, atol=0)
    # the floor R2_MIN keeps a light at the centre finite
    at = L64.shade(base, rough, normals, views, means, [1], torch.zeros(1, 3, dtype=D), color, T)
    assert all(torch.isfinite(t).all() for t in at)


def _occluder(offset, op, sigma=0.05):
    """A receiver at the origin facing +z, an isotropic occluder 1 unit up (offset sideways by `offset`) facing down."""
    means = np.array([[0, 0, 0], [offset, 0, 1]], np.float32)
    inv = np.array([[1, 0, 0, 1, 0, 1], [1 / sigma ** 2, 0, 0, 1 / sigma ** 2, 0, 1 / sigma ** 2]], np.float32)
    opacity = np.array([0.9, op], np.float32)
    normals = np.array([[0, 0, 1], [0, 0, -1]], np.float32)
    boxes = np.concatenate([means - 3 * sigma, means + 3 * sigma], axis=1).astype(np.float32)
    return means, inv, opacity, normals, boxes


@pytest.mark.parametrize("kind, vec", [(0, (0, 0, 1)), (1, (0, 0, 3))])
def test_analytic_shadows(kind, vec):
    op = 0.6
    T, fr = L64.shadows(*_occluder(0.0, op), [kind], np.array([vec], np.float32))
    assert not fr[0, 0]
    assert abs(T[0, 0] - (1 - op)) < 1e-6
    d, sigma = 0.04, 0.05
    T, _ = L64.shadows(*_occluder(d, op, sigma), [kind], np.array([vec], np.float32))
    assert abs(T[0, 0] - (1 - op * np.exp(-d * d / (2 * sigma * sigma)))) < 1e-6
    assert T[1, 0] == 1.0                     # the occluder faces away from its own ray's direction: nothing behind it


def test_point_light_in_front_of_the_occluder_casts_no_shadow():
    T, fr = L64.shadows(*_occluder(0.0, 0.6), [1], np.array([[0, 0, 0.5]], np.float32))
    assert T[0, 0] == 1.0 and not fr[0, 0]


def test_box_met_only_beyond_t_max_is_not_a_hit():
    """The occluder's peak lies before the light, but its (shifted) leaf box is entered only beyond t_max."""
    means, inv, opacity, normals, boxes = _occluder(0.0, 0.6)
    vec = np.array([[0, 0, 1.5]], np.float32)
    T, _ = L64.shadows(means, inv, opacity, normals, boxes, [1], vec)
    assert abs(T[0, 0] - 0.4) < 1e-6
    boxes[1, 2], boxes[1, 5] = 1.6, 1.8
    T, _ = L64.shadows(means, inv, opacity, normals, boxes, [1], vec)
    assert T[0, 0] == 1.0


def test_shadow_matching_rule():
    ok, fr = L64.shadows_match(np.array([0.5, 5e-5, 2e-4]), np.array([0.5, 1e-7, 1e-7]), np.zeros(3, bool))
    assert ok.tolist() == [True, True, False] and not fr.any()


# ---- refusals ------------------------------------------------------------------------------------------------------
def _kinds(*k):
    return (ctypes.c_int32 * max(len(k), 1))(*k)


def _args(P=10, K=2, V=1, kind=None):
    a = _lib.LightArgs()
    a.P, a.K, a.V = P, K, V
    a.kind_buf = kind if kind is not None else _kinds(*([0] * max(K, 0)))       # alive as long as the struct
    a.kind = ctypes.cast(a.kind_buf, ctypes.c_void_p)
    for f in ("vec", "color", "means3D", "base_color", "roughness", "normals", "viewdirs", "shadows", "pbr", "diffuse_light",
              "specular", "dL_dpbr", "dL_dbase_color", "dL_droughness", "dL_dviewdirs", "dL_dmeans3D", "dL_dvec",
              "dL_dcolor", "work"):
        setattr(a, f, FAKE)
    a.work_bytes = _lib.load().r3dg_shade_lights_work_bytes(P, K)
    return a


def test_c_layer_refuses_bad_arguments():
    lib = _lib.load()
    fwd, bwd = lib.r3dg_shade_lights_forward, lib.r3dg_shade_lights_backward
    keep = []

    def run(call, a):
        keep.append(a)
        return call(ctypes.byref(a), None)
    for call in (fwd, bwd):
        assert call(None, None) == -10001
        for P, K, V in ((-1, 2, 1), (10, -1, 1), (10, 33, 1), (10, 2, 0), (10, 2, 65)):
            assert run(call, _args(P, K, V)) == -10001, (P, K, V)
        k = _kinds(0, 2)
        assert run(call, _args(kind=k)) == -10001                  # a kind other than 0 or 1
        a = _args()
        a.kind = None
        assert run(call, a) == -10001
        for field in ("vec", "color", "means3D", "base_color", "roughness", "normals", "viewdirs", "shadows"):
            a = _args()
            setattr(a, field, None)
            assert run(call, a) == -10001, field
    for field in ("pbr", "diffuse_light", "specular"):
        a = _args()
        setattr(a, field, None)
        assert run(fwd, a) == -10001, field
    for field in ("dL_dpbr", "dL_dbase_color", "dL_droughness", "dL_dviewdirs", "dL_dmeans3D", "dL_dvec", "dL_dcolor", "work"):
        a = _args()
        setattr(a, field, None)
        assert run(bwd, a) == -10001, field
    a = _args()
    a.work_bytes -= 1
    assert run(bwd, a) == -10001
    # P = 0: nothing to shade and no light gradient to zero-fill when K = 0 too
    assert run(fwd, _args(P=0, K=0)) == 0 and run(bwd, _args(P=0, K=0)) == 0
    assert lib.r3dg_shade_lights_work_bytes(0, 4) == 0 and lib.r3dg_shade_lights_work_bytes(1000, 0) == 0
    assert lib.r3dg_shade_lights_work_bytes(1000, 4) >= 1000 // 128 * 4 * 6 * 4


def test_c_layer_refuses_bad_trace_arguments():
    lib = _lib.load()
    P, K = 10, 2
    tmp = lib.r3dg_bvh_trace_lights_tmp_bytes(P)

    def trace(P=P, K=K, kind=None, tmp_bytes=tmp, **null):
        ptrs = {n: (None if n in null else FAKE) for n in ("vec", "nodes", "aabbs", "means3D", "covs3D", "opacities",
                                                            "normals", "shadows", "tmp")}
        kd = kind if kind is not None else _kinds(*([1] * max(K, 0)))
        return lib.r3dg_bvh_trace_lights(P, K, ctypes.cast(kd, ctypes.c_void_p), ptrs["vec"], ptrs["nodes"], ptrs["aabbs"],
                                         ptrs["means3D"], ptrs["covs3D"], ptrs["opacities"], ptrs["normals"],
                                         ptrs["shadows"], ptrs["tmp"], tmp_bytes, None)
    assert trace(P=-1) == -10001
    assert trace(K=33) == -10001 and trace(K=-1) == -10001
    assert trace(kind=_kinds(1, 5)) == -10001
    for n in ("vec", "nodes", "aabbs", "means3D", "covs3D", "opacities", "normals", "shadows", "tmp"):
        assert trace(**{n: None}) == -10001, n
    assert trace(tmp_bytes=tmp - 1) == -10001
    assert trace(P=0) == 0 and trace(K=0) == 0
    assert lib.r3dg_bvh_trace_lights(P, 1, None, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, tmp, None) == -10001


def test_python_layer_checks_before_launching():
    with pytest.raises(ValueError):
        Lights([0, 2], torch.zeros(2, 3), torch.zeros(2, 3))
    with pytest.raises(ValueError):
        Lights.point(torch.zeros(33, 3), torch.zeros(33, 3))
    with pytest.raises(ValueError):
        Lights([0], torch.zeros(2, 3), torch.zeros(2, 3))
    lt = Lights.cat(Lights.point(torch.zeros(2, 3), torch.ones(2, 3)), Lights.directional(torch.ones(1, 3), torch.ones(1, 3)))
    assert lt.kind.tolist() == [1, 1, 0] and len(lt) == 3
    P = 4
    z = torch.zeros(P, 3)
    with pytest.raises(ValueError):
        shade(z, torch.zeros(P, 1), z, torch.zeros(P, 2), z, lt, torch.zeros(P, 3))       # viewdirs
    with pytest.raises(ValueError):
        shade(z, torch.zeros(P, 1), z, torch.zeros(65, P, 3), z, lt, torch.zeros(P, 3))   # too many views
    with pytest.raises(ValueError):
        shade(z, torch.zeros(P, 1), z, z, z, lt, torch.zeros(P, 2))                       # shadows not [P,K]
    with pytest.raises(RuntimeError):
        shade(z, torch.zeros(P, 1), z, z, z, lt, torch.zeros(P, 3))                       # CPU tensors: no fallback

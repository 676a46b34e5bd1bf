"""The spot and rect lights' fp64 truth (tests/shaped_lights64.py) against closed forms and limits: a rect's estimate
against Lambert's polygon irradiance, a shrinking rect against a point light, a spot against a point light inside and
outside its cone, the falloff; the sample hash's golden values; and the refusals of the C and Python layers."""
import ctypes

import numpy as np
import pytest
import torch

import lights64 as L64
import shaped_lights64 as S64
from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200.lights import ShapedLights, shade_shaped
from relightable3dgaussian_b200.raytracer import RayTracer

FAKE = 0x10000      # never dereferenced: every call below is refused (or does nothing) before anything is enqueued
D = torch.float64


def _diffuse(means, normals, lights, M, seed, T=None):
    """diffuse_light [P,3] of the oracle for fp64 Gaussians (base 0 and any view: only the transport matters)."""
    P = means.shape[0]
    kind = lights["kind"]
    _, st = S64.ray_targets(kind, lights["pos"], lights["a"], lights["b"], M, seed, P)
    R = st.shape[1]
    T = torch.ones(P, R, dtype=D) if T is None else T
    views = torch.nn.functional.normalize(torch.ones(1, P, 3, dtype=D), dim=-1)
    _, diff, _ = S64.shade(torch.zeros(P, 3, dtype=D), torch.full((P, 1), 0.5, dtype=D), normals, views, means, kind,
                           *(torch.as_tensor(np.asarray(lights[f], np.float32), dtype=D)
                             for f in ("pos", "a", "b", "color", "cone")), T, M, st)
    return diff[0]


def _rect(center, u, v, color=(1.0, 1.0, 1.0)):
    return dict(kind=[3], pos=[center], a=[u], b=[v], color=[color], cone=[[0.0, 0.0]])


def _cell_oscillation_bound(x, n, center, u, v, M):
    """sum over the M x M strata of (max - min of the integrand on the stratum) x its area: the worst-case error of a
    one-sample-per-stratum estimate, the integrand evaluated on a 9 x 9 grid per stratum."""
    c, u, v = (np.asarray(t, np.float64) for t in (center, u, v))
    ne = np.cross(u, v)
    area = 4 * np.linalg.norm(ne)
    ne /= np.linalg.norm(ne)
    total = 0.0
    g = np.linspace(0, 1, 9)
    for i in range(M):
        for k in range(M):
            s = -1 + (2 * i + g[:, None]) / M
            t = -1 + (2 * k + g[None, :]) / M
            y = c + s[..., None] * u + t[..., None] * v
            w = y - x
            r2 = (w * w).sum(-1)
            l = w / np.sqrt(r2)[..., None]
            f = np.maximum(l @ n, 0) * np.maximum(-(l @ ne), 0) / r2
            total += (f.max() - f.min()) * area / (M * M)
    return total


def test_rect_converges_to_the_polygon_irradiance():
    """An unoccluded receiver under a tilted rect: the estimate converges to Lambert's closed form as M grows, within
    the stratified estimator's bound at every M (and 0.5 % at M = 8)."""
    x, n = np.zeros(3), np.array([0.0, 0.0, 1.0])
    center, u, v = [0.3, -0.2, 1.0], [0.4, 0.0, 0.1], [0.0, 0.25, 0.0]
    # the emitting side faces the receiver: n_e = normalize(u x v) must point down, so swap u and v
    lights = _rect(center, v, u, (2.0, 1.0, 0.5))
    ne = np.cross(v, u)
    assert ne[2] < 0
    corners = [np.add(np.add(center, su * np.asarray(v)), sv * np.asarray(u)) for su, sv in ((-1, -1), (1, -1), (1, 1), (-1, 1))]
    truth = S64.polygon_irradiance(x, n, corners)
    errs = []
    for M in (1, 2, 4, 8):
        est = np.mean([float(_diffuse(torch.zeros(1, 3, dtype=D), torch.tensor(n[None]), lights, M, seed)[0, 0]) / 2.0
                       for seed in range(4)])
        bound = _cell_oscillation_bound(x, n, center, v, u, M)
        errs.append(abs(est - truth))
        assert errs[-1] <= bound * 1.01 + 1e-9, (M, est, truth, bound)
    assert errs[-1] < 5e-3 * truth
    assert errs[-1] < errs[0]


def test_rect_with_the_receiver_behind_it_or_edge_on_gives_nothing():
    x = torch.zeros(1, 3, dtype=D)
    n = torch.tensor([[0.0, 0.0, 1.0]], dtype=D)
    back = _rect([0.0, 0.0, 1.0], [0.3, 0.0, 0.0], [0.0, 0.3, 0.0])          # u x v = +z: emits upwards, away
    assert float(_diffuse(x, n, back, 4, 0).abs().max()) == 0.0
    flat = _rect([0.0, 0.0, 1.0], [0.3, 0.0, 0.0], [0.6, 0.0, 0.0])          # degenerate: u x v = 0
    assert float(_diffuse(x, n, flat, 4, 0).abs().max()) == 0.0


def test_small_rect_is_a_point_light_times_its_emitter_cosine():
    """A rect shrunk at fixed color x A converges to a point light at its centre of intensity color x A, scaled by
    max(-n_e . l, 0)."""
    g = torch.Generator().manual_seed(3)
    P = 16
    means = torch.randn(P, 3, generator=g, dtype=D) * 0.3
    normals = torch.nn.functional.normalize(torch.randn(P, 3, generator=g, dtype=D), dim=-1)
    center = np.array([0.1, 0.2, 2.0])
    I = np.array([1.0, 2.0, 3.0])
    prev = None
    for h in (1e-1, 1e-2, 1e-3):
        u, v = np.array([0.0, h, 0.0]), np.array([h * 0.8, 0.0, 0.0])           # u x v = -z (towards the Gaussians)
        A = 4 * np.linalg.norm(np.cross(u, v))
        lights = _rect(center, u, v, I / A)
        est = _diffuse(means, normals, lights, 2, 7)
        l, inv_r2, _ = L64.light_dirs([1], torch.tensor([center]), means)
        ce = (l[:, 0] * torch.tensor([0.0, 0.0, 1.0], dtype=D)).sum(-1, keepdim=True).clamp(min=0)
        point = torch.tensor(I)[None] * inv_r2 * ce * (normals * l[:, 0]).sum(-1, keepdim=True).clamp(min=0)
        err = float((est - point).abs().max() / point.abs().max())
        assert prev is None or err < prev
        prev = err
    assert prev < 1e-3


def test_spot_is_a_point_light_inside_its_inner_cone_and_dark_outside():
    g = torch.Generator().manual_seed(4)
    P = 32
    base = torch.rand(P, 3, generator=g, dtype=D)
    rough = torch.rand(P, 1, generator=g, dtype=D) * 0.9 + 0.05
    normals = torch.nn.functional.normalize(torch.randn(P, 3, generator=g, dtype=D), dim=-1)
    means = torch.randn(P, 3, generator=g, dtype=D) * 0.05
    views = torch.nn.functional.normalize(torch.randn(1, P, 3, generator=g, dtype=D), dim=-1)
    pos = torch.tensor([[0.0, 0.0, 2.0]], dtype=D)
    color = torch.tensor([[3.0, 2.0, 1.0]], dtype=D)
    T = torch.rand(P, 1, generator=g, dtype=D)
    st = np.zeros((P, 1, 2))
    z = torch.zeros(1, 3, dtype=D)
    down = torch.tensor([[0.0, 0.0, -1.0]], dtype=D)
    inside = S64.shade(base, rough, normals, views, means, [2], pos, down, z, color, torch.tensor([[0.9, 0.8]], dtype=D), T, 1, st)
    point = L64.shade(base, rough, normals, views, means, [1], pos, color, T)
    for a, b in zip(inside, point):                 # E = color x 1 / r^2: the same up to fp64 rounding
        torch.testing.assert_close(a, b, rtol=1e-14, atol=0)
    up = torch.tensor([[0.0, 0.0, 1.0]], dtype=D)
    outside = S64.shade(base, rough, normals, views, means, [2], pos, up, z, color, torch.tensor([[0.9, 0.8]], dtype=D), T, 1, st)
    assert all(not t.any() for t in outside)


def test_spot_falloff_is_monotone_and_c1():
    """E along a receiver moving out of the cone: non-increasing, and the smoothstep's slope vanishes at both ends."""
    ci, co = 0.95, 0.85
    ang = np.linspace(0.0, 0.7, 2001)
    means = torch.tensor(np.stack([2 * np.tan(ang), np.zeros_like(ang), np.zeros_like(ang)], 1))
    normals = torch.tensor([[0.0, 0.0, 1.0]], dtype=D).expand(len(ang), 3)
    lights = dict(kind=[2], pos=[[0.0, 0.0, 2.0]], a=[[0.0, 0.0, -1.0]], b=[[0.0, 0.0, 0.0]], color=[[1.0, 1.0, 1.0]],
                  cone=[[ci, co]])
    E = _diffuse(means, normals, lights, 1, 0)[:, 0].numpy()
    r2 = 4 + (2 * np.tan(ang)) ** 2
    s = E * r2 / (2 / np.sqrt(r2))                     # divide out 1/r^2 and n . l
    assert np.all(np.diff(s) <= 1e-12)
    assert s[0] == pytest.approx(1.0, abs=1e-6) and s[-1] == 0.0
    cosang = np.cos(ang)
    x = np.clip((cosang - co) / (ci - co), 0, 1)
    assert np.allclose(s, x * x * (3 - 2 * x), atol=1e-5)
    # C1: the slope ds/dcos is continuous: it falls to 0 at both ends of the band, where the constant parts begin
    slope = np.abs(np.gradient(s, cosang))
    band = (cosang > co) & (cosang < ci)
    peak = slope[band].max()
    assert peak == pytest.approx(1.5 / (ci - co), rel=1e-2)           # the smoothstep's slope at x = 1/2
    for end in (co, ci):
        near = np.abs(cosang - end) < 2e-3 * (ci - co) + 1e-4
        assert near.any() and slope[near].max() < 0.05 * peak, end


# ---- the sample hash --------------------------------------------------------------------------------------------
GOLDEN_LOWBIAS32 = {0: 0x00000000, 1: 0x688990C0, 0xDEADBEEF: 0xE628C683, 0xFFFFFFFF: 0x6768824A}
# (seed, g, j, q) -> (xi1, xi2) bits of the fp32 jitter
GOLDEN_XI = {(0, 0, 0, 0): (0x00000000, 0x3ED11320), (12345, 999999, 31, 63): (0x3F35D7A6, 0x3EB0C62C)}


def test_hash_golden_values():
    for x, h in GOLDEN_LOWBIAS32.items():
        assert S64.lowbias32(x) == h, hex(S64.lowbias32(x))
    for key, bits in GOLDEN_XI.items():
        got = tuple(int(np.asarray(v, np.float32).view(np.uint32)) for v in S64.xi(*key))
        assert got == bits, (key, [hex(b) for b in got])
        assert all(0.0 <= v < 1.0 for v in S64.xi(*key))


def test_rect_samples_are_stratified():
    """Every (i, k) stratum of the parallelogram gets exactly one sample."""
    M = 8
    for g in (0, 17, 123456):
        ij = set()
        for q in range(M * M):
            s, t, _ = S64.rect_sample([0, 0, 0], [1, 0, 0], [0, 1, 0], M, 99, g, 2, q)
            assert -1 <= s <= 1 and -1 <= t <= 1
            ij.add((int((s + 1) * M / 2), int((t + 1) * M / 2)))
        assert len(ij) == M * M


# ---- refusals ------------------------------------------------------------------------------------------------------
def _kinds(*k):
    return (ctypes.c_int32 * max(len(k), 1))(*k)


FIELDS = ("pos", "a", "b", "color", "cone", "means3D", "base_color", "roughness", "normals", "viewdirs", "shadows", "pbr",
          "diffuse_light", "specular", "dL_dpbr", "dL_dbase_color", "dL_droughness", "dL_dviewdirs", "dL_dmeans3D",
          "dL_dpos", "dL_da", "dL_db", "dL_dcolor", "dL_dcone", "work")


def _args(P=10, K=2, V=1, M=4, kind=None):
    a = _lib.ShapedLightArgs()
    a.P, a.K, a.V, a.M, a.seed = P, K, V, M, 7
    a.kind_buf = kind if kind is not None else _kinds(*([2, 3] * 16)[:max(K, 0)])   # alive as long as the struct
    a.kind = ctypes.cast(a.kind_buf, ctypes.c_void_p)
    for f in FIELDS:
        setattr(a, f, FAKE)
    a.work_bytes = _lib.load().r3dg_shade_shaped_lights_work_bytes(P, K)
    return a


def test_c_layer_refuses_bad_shading_arguments():
    lib = _lib.load()
    fwd, bwd = lib.r3dg_shade_shaped_lights_forward, lib.r3dg_shade_shaped_lights_backward
    keep = []

    def run(call, a):
        keep.append(a)
        return call(ctypes.byref(a), None)
    for call in (fwd, bwd):
        assert call(None, None) == -10001
        for P, K, V, M in ((-1, 2, 1, 4), (10, -1, 1, 4), (10, 33, 1, 4), (10, 2, 0, 4), (10, 2, 65, 4), (10, 2, 1, 0),
                           (10, 2, 1, 9)):
            assert run(call, _args(P, K, V, M)) == -10001, (P, K, V, M)
        for bad in ((0, 3), (1, 3), (2, 5)):                                 # kinds of the other set, or none at all
            assert run(call, _args(kind=_kinds(*bad))) == -10001, bad
        assert run(call, _args(K=5, M=8, kind=_kinds(3, 3, 3, 3, 2))) == -10001      # R = 257
        a = _args(K=4, M=8, kind=_kinds(3, 3, 3, 3))                                  # R = 256 is fine: refused for
        a.pos = None                                                                  # the missing pointer only
        assert run(call, a) == -10001
        a = _args()
        a.kind = None
        assert run(call, a) == -10001
        for field in ("pos", "a", "b", "color", "cone", "means3D", "base_color", "roughness", "normals", "viewdirs", "shadows"):
            a = _args()
            setattr(a, field, None)
            assert run(call, a) == -10001, field
    for field in ("pbr", "diffuse_light", "specular"):
        a = _args()
        setattr(a, field, None)
        assert run(fwd, a) == -10001, field
    for field in ("dL_dpbr", "dL_dbase_color", "dL_droughness", "dL_dviewdirs", "dL_dmeans3D", "dL_dpos", "dL_da", "dL_db",
                  "dL_dcolor", "dL_dcone", "work"):
        a = _args()
        setattr(a, field, None)
        assert run(bwd, a) == -10001, field
    a = _args()
    a.work_bytes -= 1
    assert run(bwd, a) == -10001
    # b is read only by rects and cone only by spots
    a = _args(P=0, K=1, kind=_kinds(2))
    a.b = None
    assert run(fwd, a) == 0
    a = _args(P=0, K=1, kind=_kinds(3))
    a.cone = None
    assert run(fwd, a) == 0
    assert run(fwd, _args(P=0, K=0)) == 0 and run(bwd, _args(P=0, K=0)) == 0
    assert lib.r3dg_shade_shaped_lights_work_bytes(0, 4) == 0 and lib.r3dg_shade_shaped_lights_work_bytes(1000, 0) == 0
    assert lib.r3dg_shade_shaped_lights_work_bytes(1000, 4) >= 1000 // 128 * 4 * 16 * 4


def test_c_layer_refuses_bad_trace_arguments():
    lib = _lib.load()
    P = 10
    tmp = lib.r3dg_bvh_trace_shaped_lights_tmp_bytes(P)
    keep = []

    def trace(a, tmp_bytes=tmp, **null):
        keep.append(a)
        p = {n: (None if n in null else FAKE) for n in ("nodes", "aabbs", "covs3D", "opacities", "shadows", "tmp")}
        return lib.r3dg_bvh_trace_shaped_lights(ctypes.byref(a), p["nodes"], p["aabbs"], p["covs3D"], p["opacities"],
                                                p["shadows"], p["tmp"], tmp_bytes, None)
    assert lib.r3dg_bvh_trace_shaped_lights(None, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, tmp, None) == -10001
    for P_, K, M in ((-1, 2, 4), (P, 33, 4), (P, -1, 4), (P, 2, 0), (P, 2, 9)):
        assert trace(_args(P_, K, 1, M)) == -10001, (P_, K, M)
    for bad in ((0, 3), (1, 3), (2, 4)):
        assert trace(_args(kind=_kinds(*bad))) == -10001, bad
    assert trace(_args(K=5, M=8, kind=_kinds(3, 3, 3, 3, 2))) == -10001                  # R = 257
    for n in ("nodes", "aabbs", "covs3D", "opacities", "shadows", "tmp"):
        assert trace(_args(), **{n: None}) == -10001, n
    for field in ("pos", "a", "b", "means3D", "normals"):
        a = _args()
        setattr(a, field, None)
        assert trace(a) == -10001, field
    a = _args(K=1, kind=_kinds(2))                                                       # a spot reads no b
    a.b = None
    a.P = 0
    assert trace(a) == 0
    assert trace(_args(), tmp_bytes=tmp - 1) == -10001
    assert trace(_args(P=0)) == 0 and trace(_args(K=0)) == 0


def test_num_rays():
    lib = _lib.load()
    assert lib.r3dg_shaped_lights_num_rays(3, ctypes.cast(_kinds(2, 3, 3), ctypes.c_void_p), 4) == 33
    assert lib.r3dg_shaped_lights_num_rays(0, None, 1) == 0
    assert lib.r3dg_shaped_lights_num_rays(4, ctypes.cast(_kinds(3, 3, 3, 3), ctypes.c_void_p), 8) == 256
    assert lib.r3dg_shaped_lights_num_rays(5, ctypes.cast(_kinds(3, 3, 3, 3, 2), ctypes.c_void_p), 8) == -1
    assert lib.r3dg_shaped_lights_num_rays(1, ctypes.cast(_kinds(1), ctypes.c_void_p), 4) == -1
    assert lib.r3dg_shaped_lights_num_rays(1, ctypes.cast(_kinds(3), ctypes.c_void_p), 9) == -1
    assert S64.columns([2, 3, 2], 2) == [(0, 0), (1, 0), (1, 1), (1, 2), (1, 3), (2, 0)]


def test_python_layer_checks_before_launching():
    z3 = torch.zeros(1, 3)
    for kind in ([0], [1], [5]):
        with pytest.raises(ValueError):
            ShapedLights(kind, z3, z3, z3, z3, torch.zeros(1, 2))
    for M in (0, 9, 2.5):
        with pytest.raises(ValueError):
            ShapedLights.rect(z3, z3, z3, z3, M=M)
    with pytest.raises(ValueError):
        ShapedLights.spot(torch.zeros(33, 3), torch.zeros(33, 3), torch.zeros(33, 3), 0.9, 0.8)
    with pytest.raises(ValueError):
        ShapedLights([2], z3, z3, z3, z3, torch.zeros(1, 3))                     # cone not [K,2]
    with pytest.raises(ValueError):
        ShapedLights([3], torch.zeros(2, 3), z3, z3, z3, torch.zeros(1, 2))      # pos not [K,3]
    rects = ShapedLights.rect(torch.zeros(4, 3), torch.zeros(4, 3), torch.zeros(4, 3), torch.zeros(4, 3), M=8)
    assert rects.num_rays() == 256
    with pytest.raises(ValueError):                                              # R = 257
        ShapedLights.cat(rects, ShapedLights.spot(z3, z3, z3, 0.9, 0.8))
    lt = ShapedLights.cat(ShapedLights.spot(torch.zeros(2, 3), z3.expand(2, 3), torch.ones(2, 3), 0.9, torch.tensor([0.8, 0.7])),
                          ShapedLights.rect(z3, z3, z3, z3, M=3), seed=5)
    assert lt.kind.tolist() == [2, 2, 3] and len(lt) == 3 and lt.num_rays() == 18 and lt.M == 4 and lt.seed == 5
    assert lt.cone.tolist() == [[0.8999999761581421, 0.800000011920929], [0.8999999761581421, 0.699999988079071], [0.0, 0.0]]
    P, R = 4, lt.num_rays()
    z = torch.zeros(P, 3)
    with pytest.raises(ValueError):
        shade_shaped(z, torch.zeros(P, 1), z, torch.zeros(P, 2), z, lt, torch.zeros(P, R))       # viewdirs
    with pytest.raises(ValueError):
        shade_shaped(z, torch.zeros(P, 1), z, torch.zeros(65, P, 3), z, lt, torch.zeros(P, R))   # too many views
    with pytest.raises(ValueError):
        shade_shaped(z, torch.zeros(P, 1), z, z, z, lt, torch.zeros(P, 3))                       # shadows not [P,R]
    with pytest.raises(RuntimeError):
        shade_shaped(z, torch.zeros(P, 1), z, z, z, lt, torch.zeros(P, R))                       # CPU tensors
    with pytest.raises(RuntimeError):
        RayTracer.__new__(RayTracer).trace_shaped_lights(z, torch.zeros(P, 6), torch.zeros(P), z, lt)

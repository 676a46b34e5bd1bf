"""Per-pixel shading without a GPU: the fp64 pixel oracle (tests/pixel64.py) against the row formula of
oracle/oracle_shading.py, and the refusals of the host wrappers and of the C entry points (nothing is launched)."""
import ctypes
import math

import pytest
import torch

import pixel64
from oracle import oracle_sampling, oracle_shading
from relightable3dgaussian_b200 import _lib, shading
from relightable3dgaussian_b200.raytracer import RayTracer


def pixel_case(H, W, N, He=8, seed=0):
    g = torch.Generator().manual_seed(700 + seed)
    n = torch.randn(3, H, W, generator=g)
    return dict(base_color=torch.rand(3, H, W, generator=g) * 0.8 + 0.05,
                roughness=torch.rand(1, H, W, generator=g) * 0.9 + 0.08,
                normal=n * (0.5 + torch.rand(1, H, W, generator=g)),               # blended normals: not unit length
                points=torch.randn(3, H, W, generator=g) * 0.5,
                campos=torch.tensor([0.3, -2.5, 1.7]),
                T=torch.where(torch.rand(N, H, W, generator=g) < 0.3, torch.zeros(N, H, W), 0.9 + 0.1 * torch.rand(N, H, W, generator=g)),
                incidents=torch.randn(48, H, W, generator=g) * 0.3,
                env=torch.rand(He, 2 * He, 3, generator=g) * 2,
                transform=torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))[0].float(),
                mask=torch.rand(H, W, generator=g) < 0.7)


def rows_oracle(c, transform, incidents):
    """oracle_shading.rendering_equation (fp32) on the pixels as rows."""
    H, W = c["base_color"].shape[-2:]
    rows = lambda t: t.reshape(t.shape[0], H * W).T.contiguous()
    n = rows(c["normal"])
    nh = n / torch.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2]).clamp_min(1e-12)[:, None]
    dirs, areas = oracle_sampling.fibonacci_sphere_sampling(nh, c["T"].shape[0], random_rotate=False)
    inc = rows(incidents).reshape(-1, 16, 3) if incidents is not None else torch.zeros(H * W, 16, 3)
    pbr, extra = oracle_shading.rendering_equation(rows(c["base_color"]), rows(c["roughness"]), n,
                                                   c["campos"][None] - rows(c["points"]), inc, c["env"],
                                                   rows(c["T"])[..., None], dirs, areas, transform)
    back = lambda x: x.T.reshape(-1, H, W)
    return {"pbr": back(pbr), "diffuse_light": back(extra["diffuse_light"]), "specular": back(extra["specular"]),
            "visibility": back(rows(c["T"]).mean(1, keepdim=True))}


@pytest.mark.parametrize("H,W,N,with_inc,with_tr,with_mask", [(1, 1, 3, True, False, False), (5, 7, 16, True, True, True),
                                                              (9, 4, 32, False, False, True), (3, 11, 8, False, True, False)])
def test_pixel_oracle_agrees_with_row_formula(H, W, N, with_inc, with_tr, with_mask):
    c = pixel_case(H, W, N)
    inc = c["incidents"] if with_inc else None
    tr = c["transform"] if with_tr else None
    mask = c["mask"] if with_mask else None
    got = pixel64.shade_pixels(c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], c["env"],
                               tr, inc, mask)
    want = rows_oracle(c, tr, inc)
    keep = torch.ones(H, W, dtype=torch.bool) if mask is None else mask
    for k, x in got.items():
        assert x.dtype == torch.float64 and x.shape == want[k].shape
        assert torch.all(x[:, ~keep] == 0), k
        w = want[k].double()[:, keep]
        err = (x[:, keep] - w).abs().max().item()
        assert err <= 5e-5 * max(1.0, w.abs().max().item()), (k, err)     # the row formula runs in fp32


def test_zero_incidents_equal_no_incidents_and_transform_matters():
    c = pixel_case(6, 5, 16)
    args = (c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], c["env"])
    none = pixel64.shade_pixels(*args)
    zero = pixel64.shade_pixels(*args, None, torch.zeros(48, 6, 5))
    rotated = pixel64.shade_pixels(*args, c["transform"])
    for k in none:
        assert torch.equal(none[k], zero[k])
    assert (rotated["pbr"] - none["pbr"]).abs().max() > 1e-3
    assert torch.equal(rotated["visibility"], none["visibility"])


def test_sample_dirs_are_unit_and_in_the_hemisphere():
    n = torch.nn.functional.normalize(torch.randn(50, 3, dtype=torch.float64), dim=-1)
    n[0] = torch.tensor([0.0, 0.0, -1.0], dtype=torch.float64)
    d = pixel64.sample_dirs(n, 24)
    assert torch.allclose(d.norm(dim=-1), torch.ones(50, 24, dtype=torch.float64))
    assert ((d * n[:, None]).sum(-1) >= math.sin(math.radians(10)) - 1e-12).all()


# ---- refusals ----------------------------------------------------------------------------------------------------------
class Light:
    def __init__(self, envmap, transform=None):
        self.envmap, self.transform = envmap, transform


def test_host_wrappers_refuse_cpu_tensors_and_bad_shapes():
    c = pixel_case(4, 4, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        shading.shade_pixels(c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], Light(c["env"]))
    with pytest.raises(RuntimeError, match="GPU"):
        RayTracer.trace_pixels(None, c["points"], c["normal"], 8, torch.zeros(4, 3), torch.zeros(4, 6), torch.zeros(4),
                               torch.zeros(4, 3))
    with pytest.raises(ValueError, match=r"\[3,H,W\]"):
        shading._views(torch.zeros(2, 4, 4), 3, "normal")
    with pytest.raises(ValueError, match="does not match"):
        shading._views(torch.zeros(3, 4, 5), 3, "points", ((), 4, 4))
    with pytest.raises(ValueError, match="1 to 64 views"):
        shading._views(torch.zeros(65, 3, 4, 4), 3, "normal")
    with pytest.raises(ValueError, match="mask"):
        shading._mask(torch.ones(4, 5, dtype=torch.bool), ((), 4, 4))
    with pytest.raises(ValueError, match="mask"):
        shading._mask(torch.ones(4, 4), ((), 4, 4))


def _fake_args(**kw):
    a = _lib.PixelArgs()
    a.V, a.H, a.W, a.N, a.env_h, a.env_w = 1, 4, 4, 8, 8, 16
    FAKE = 0x10000                     # never dereferenced: every call below is refused before anything is enqueued
    for f in ("base_color", "roughness", "normal", "points", "campos", "env", "visibility", "pbr", "diffuse_light",
              "specular", "mean_visibility", "dL_dpbr", "dL_dbase_color", "dL_droughness", "dL_denv"):
        setattr(a, f, FAKE)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,rc", [(dict(V=0), -10001), (dict(V=65), -10001), (dict(H=0), -10001), (dict(N=0), -10001),
                                   (dict(N=2731), -10002), (dict(env_h=0), -10001), (dict(points=None), -10001),
                                   (dict(transform_per_view=1), -10001), (dict(V=64, H=2**13, W=2**13), -10002)])
def test_c_entry_points_refuse_before_any_launch(kw, rc):
    lib = _lib.load()
    a = _fake_args(**kw)
    assert lib.r3dg_shade_pixels_forward(ctypes.byref(a), None) == rc
    assert lib.r3dg_shade_pixels_backward(ctypes.byref(a), None) == rc
    if not {"env_h", "transform_per_view"} & set(kw):          # the trace reads no env
        tmp = lib.r3dg_bvh_trace_pixels_tmp_bytes(10)
        assert lib.r3dg_bvh_trace_pixels(ctypes.byref(a), 10, *[0x10000] * 8, tmp, None) == rc


def test_backward_refuses_missing_workspaces():
    lib = _lib.load()
    a = _fake_args(env_pyramid=0x10000)                       # pyramid without its gradient workspace
    assert lib.r3dg_shade_pixels_backward(ctypes.byref(a), None) == -10001
    a = _fake_args(deterministic=1, det_work=0x10000, det_work_bytes=lib.r3dg_shade_det_bytes(8, 16) - 1)
    assert lib.r3dg_shade_pixels_backward(ctypes.byref(a), None) == -10001
    a = _fake_args(incidents=0x10000)                         # incidents without their gradient
    assert lib.r3dg_shade_pixels_backward(ctypes.byref(a), None) == -10001
    a = _fake_args(pbr=None)
    assert lib.r3dg_shade_pixels_forward(ctypes.byref(a), None) == -10001
    tmp = lib.r3dg_bvh_trace_pixels_tmp_bytes(10)
    a = _fake_args()
    assert lib.r3dg_bvh_trace_pixels(ctypes.byref(a), 10, *[0x10000] * 8, tmp - 1, None) == -10001
    assert lib.r3dg_bvh_trace_pixels(ctypes.byref(a), 0, *[0x10000] * 8, tmp, None) == -10001

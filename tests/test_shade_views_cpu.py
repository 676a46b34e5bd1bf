"""rendering_equation_views refuses what it cannot shade before anything is launched (no GPU needed), and the C ABI
refuses several-view shading calls beyond the view limit, with per-sample outputs, or with per-view transforms in the
backward."""
import ctypes

import pytest
import torch

from helpers import shading_case
from relightable3dgaussian_b200 import _lib, shading
from relightable3dgaussian_b200.shading import rendering_equation_views


class FixedLight:               # duck-types EnvLight (envmap + transform)
    def __init__(self, envmap, transform=None):
        self.envmap, self.transform = envmap, transform


def _call(viewdirs, light=None, incidents=None, P=6, N=5):
    c = shading_case(P, N, 4, seed=1)
    light = light if light is not None else FixedLight(torch.nn.functional.softplus(c["env_raw"])[0])
    return rendering_equation_views(c["base_color"], c["roughness"], c["normals"], viewdirs,
                                    c["incidents"] if incidents is None else incidents, light, c["visibility"],
                                    c["incident_dirs"], c["incident_areas"])


def test_view_count_and_shape_refused():
    with pytest.raises(ValueError, match="1 to 64"):
        _call(torch.zeros(0, 6, 3))
    with pytest.raises(ValueError, match="1 to 64"):
        _call(torch.zeros(shading.MAX_VIEWS + 1, 6, 3))
    for bad in (torch.zeros(6, 3), torch.zeros(2, 5, 3), torch.zeros(2, 6, 4)):
        with pytest.raises(ValueError, match=r"\[V,P,3\]"):
            _call(bad)


def test_incidents_must_be_degree_3():
    with pytest.raises(RuntimeError, match=r"\[P,16,3\]"):
        _call(torch.zeros(2, 6, 3), incidents=torch.zeros(6, 9, 3))


def test_per_view_transform_count_and_backward_refused():
    env = torch.rand(4, 8, 3)
    with pytest.raises(ValueError, match=r"\[V,3,3\]"):
        _call(torch.zeros(2, 6, 3), light=FixedLight(env, torch.eye(3).repeat(3, 1, 1)))
    with pytest.raises(ValueError, match="forward-only"):
        _call(torch.zeros(2, 6, 3, requires_grad=True), light=FixedLight(env, torch.eye(3).repeat(2, 1, 1)))
    with pytest.raises(ValueError, match="forward-only"):
        _call(torch.zeros(2, 6, 3), light=FixedLight(env.requires_grad_(True), torch.eye(3).repeat(2, 1, 1)))


def _fake_args(V, P=10):
    fake = 0x10000                      # never dereferenced: every call below is refused before anything is enqueued
    a = _lib.ShadeArgs()
    a.P, a.N, a.sh_coeffs, a.env_h, a.env_w, a.V = P, 8, 16, 4, 8, V
    for name in ("base_color", "roughness", "normals", "viewdirs", "incidents", "env", "visibility", "incident_dirs",
                 "incident_areas", "pbr", "diffuse_light", "specular", "dL_dpbr", "dL_dbase_color", "dL_droughness",
                 "dL_dviewdirs", "dL_dincidents", "dL_denv"):
        setattr(a, name, fake)
    return a


def test_c_abi_refuses_bad_view_arguments():
    lib = _lib.load()
    fake = 0x10000
    assert lib.r3dg_render_equation_forward(ctypes.byref(_fake_args(shading.MAX_VIEWS + 1)), None) == -10001
    assert lib.r3dg_render_equation_backward(ctypes.byref(_fake_args(shading.MAX_VIEWS + 1)), None) == -10001
    assert lib.r3dg_render_equation_forward(ctypes.byref(_fake_args(-1)), None) == -10001
    a = _fake_args(2)                   # per-sample [P,N,3] lights exist for one view only
    a.incident_lights = a.local_incident_lights = a.global_incident_lights = fake
    assert lib.r3dg_render_equation_forward(ctypes.byref(a), None) == -10002
    b = _fake_args(2)                   # per-view transforms are forward-only
    b.env_transform, b.transform_per_view = fake, 1
    assert lib.r3dg_render_equation_backward(ctypes.byref(b), None) == -10002

"""Point and directional lights on top of the shading step's environment light (include/r3dg_b200.h, LIGHTS).

`Lights` holds K <= MAX_LIGHTS lights; `RayTracer.trace_lights` traces their shadows T [P,K] through the scene's BVH
once per light placement; `shade` evaluates their terms with the shading step's BRDF for one view or several, in the
shading step's conventions (pbr, diffuse_light and specular, [P,3] or [V,P,3]).  Add them to `rendering_equation`'s
outputs before packing the features:

    T = RayTracer(xyz, scaling, rotation).trace_lights(xyz, inv_cov, opacity, normal, lights)
    pbr_l, extra_l = lights.shade(base_color, roughness, normal, viewdirs, xyz, lights, T)
    pbr = pbr + pbr_l   (and the same for extra["diffuse_light"] and extra["specular"])

Gradients: base_color, roughness and viewdirs as in the shading step; means3D through the point lights; each light's
vec and color.  Normals and shadows get none, as in the shading step.  Every output is bitwise reproducible.
"""
import ctypes

import torch

from . import _lib

MAX_LIGHTS = 32          # R3DG_MAX_LIGHTS (include/r3dg_b200.h)
MAX_VIEWS = 64           # R3DG_MAX_VIEWS
DIRECTIONAL, POINT = 0, 1


class Lights:
    """K lights: kind [K] int32 (0 directional, 1 point; kept on the host), vec [K,3] (a directional light's direction
    towards the light, a point light's position) and color [K,3] (irradiance at normal incidence, or intensity
    divided by the squared distance).  vec and color may require grad."""

    def __init__(self, kind, vec, color):
        kind = torch.as_tensor(kind, dtype=torch.int32).detach().cpu().reshape(-1).contiguous()
        K = kind.numel()
        if K > MAX_LIGHTS:
            raise ValueError(f"at most {MAX_LIGHTS} lights per set (got {K})")
        if not bool(((kind == DIRECTIONAL) | (kind == POINT)).all()):
            raise ValueError("light kinds must be 0 (directional) or 1 (point)")
        if vec.shape != (K, 3) or color.shape != (K, 3):
            raise ValueError(f"vec and color must be [K,3] with K = {K} (got {tuple(vec.shape)}, {tuple(color.shape)})")
        if vec.device != color.device:
            raise ValueError("vec and color must be on the same device")
        self.kind, self.vec, self.color = kind, vec, color

    def __len__(self):
        return self.kind.numel()

    @staticmethod
    def point(positions, intensities):
        return Lights(torch.full((positions.shape[0],), POINT, dtype=torch.int32), positions, intensities)

    @staticmethod
    def directional(directions, irradiances):
        return Lights(torch.full((directions.shape[0],), DIRECTIONAL, dtype=torch.int32), directions, irradiances)

    @staticmethod
    def cat(*sets):
        return Lights(torch.cat([s.kind for s in sets]), torch.cat([s.vec for s in sets]), torch.cat([s.color for s in sets]))


def _args(P, K, V, kind, ts):
    """LightArgs over the contiguous float32 inputs ts = (vec, color, means3D, base_color, roughness, normals, viewdirs,
    shadows)."""
    a = _lib.LightArgs()
    a.P, a.K, a.V = P, K, V
    a.kind = kind.data_ptr() if K > 0 else None
    a.vec, a.color, a.means3D, a.base_color, a.roughness, a.normals, a.viewdirs, a.shadows = [_lib.ptr(t) for t in ts]
    return a


class _ShadeLights(torch.autograd.Function):
    """The lights' terms for V views (viewdirs [V,P,3]); one node for one view and for several."""

    @staticmethod
    def forward(ctx, base_color, roughness, viewdirs, means3D, vec, color, normals, shadows, kind):
        V, P = viewdirs.shape[0], viewdirs.shape[1]
        K = kind.numel()
        ts = [_lib.f32(t) for t in (vec, color, means3D, base_color, roughness, normals, viewdirs, shadows)]
        f = dict(dtype=torch.float32, device=viewdirs.device)
        outs = [torch.empty((V, P, 3), **f) for _ in range(3)]
        a = _args(P, K, V, kind, ts)
        a.pbr, a.diffuse_light, a.specular = [_lib.ptr(t) for t in outs]
        if P > 0:
            _lib.call("r3dg_shade_lights_forward", viewdirs.device, ctypes.byref(a), what="shade lights")
        ctx.save_for_backward(*ts)
        ctx.kind, ctx.rough_shape = kind, roughness.shape
        return tuple(outs)

    @staticmethod
    def backward(ctx, g_pbr, g_diffuse, g_specular):
        ts = ctx.saved_tensors
        vec, viewdirs = ts[0], ts[6]
        V, P, K = viewdirs.shape[0], viewdirs.shape[1], ctx.kind.numel()
        dev = viewdirs.device
        f = dict(dtype=torch.float32, device=dev)
        d_base, d_rough, d_view, d_mean = (torch.empty((P, 3), **f), torch.empty((P,), **f), torch.empty((V, P, 3), **f),
                                           torch.empty((P, 3), **f))
        d_vec, d_color = torch.empty((K, 3), **f), torch.empty((K, 3), **f)
        if P == 0:
            d_vec.zero_(); d_color.zero_()
        else:
            g = [None if t is None else _lib.f32(t) for t in (g_pbr, g_diffuse, g_specular)]
            if g[0] is None:
                g[0] = torch.zeros((V, P, 3), **f)
            a = _args(P, K, V, ctx.kind, ts)
            a.dL_dpbr, a.dL_ddiffuse_light, a.dL_dspecular = [_lib.ptr(t) for t in g]
            a.dL_dbase_color, a.dL_droughness, a.dL_dviewdirs, a.dL_dmeans3D = [_lib.ptr(t) for t in (d_base, d_rough, d_view, d_mean)]
            a.dL_dvec, a.dL_dcolor = _lib.ptr(d_vec), _lib.ptr(d_color)
            work = _lib.scratch(_lib.load().r3dg_shade_lights_work_bytes(P, K), dev)
            a.work, a.work_bytes = _lib.ptr(work), work.numel()
            _lib.call("r3dg_shade_lights_backward", dev, ctypes.byref(a), what="shade lights backward")
        return d_base, d_rough.view(ctx.rough_shape), d_view, d_mean, d_vec, d_color, None, None, None


def shade(base_color, roughness, normals, viewdirs, means3D, lights, shadows):
    """The terms of `lights` (Lights) under shadows T [P,K] (RayTracer.trace_lights): returns (pbr, {"diffuse_light",
    "specular"}), each [P,3] for viewdirs [P,3] or [V,P,3] for viewdirs [V,P,3] (1 <= V <= MAX_VIEWS; each view equals
    a one-view call bit for bit).  Inputs are checked before anything is launched."""
    P = base_color.shape[0]
    K = len(lights)
    one = viewdirs.dim() == 2
    vd = viewdirs.unsqueeze(0) if one else viewdirs
    if vd.dim() != 3 or vd.shape[1:] != (P, 3):
        raise ValueError(f"viewdirs must be [P,3] or [V,P,3] with P = {P} (got {tuple(viewdirs.shape)})")
    if not 1 <= vd.shape[0] <= MAX_VIEWS:
        raise ValueError(f"shade evaluates 1 to {MAX_VIEWS} views per call (got {vd.shape[0]})")
    if base_color.shape != (P, 3) or normals.shape != (P, 3) or means3D.shape != (P, 3) or roughness.numel() != P:
        raise ValueError("base_color, normals and means3D must be [P,3] and roughness [P] or [P,1]")
    if shadows.shape != (P, K):
        raise ValueError(f"shadows must be [P,K] = [{P},{K}] (got {tuple(shadows.shape)})")
    tensors = (base_color, roughness, normals, vd, means3D, shadows, lights.vec, lights.color)
    if not all(t.is_cuda for t in tensors):
        raise RuntimeError("lights.shade runs on the GPU only (no CPU path)")
    if len({t.device for t in tensors}) != 1:
        raise ValueError("every input of lights.shade must be on one device")
    pbr, diffuse, specular = _ShadeLights.apply(base_color, roughness, vd, means3D, lights.vec, lights.color, normals,
                                                shadows, lights.kind)
    if one:
        pbr, diffuse, specular = pbr[0], diffuse[0], specular[0]
    return pbr, {"diffuse_light": diffuse, "specular": specular}

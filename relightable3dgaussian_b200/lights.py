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

`ShapedLights` holds spot and rectangular area lights (SHAPED LIGHTS): `RayTracer.trace_shaped_lights` traces their
shadows T [P,R] (one ray per spot, M x M stratified rays per rect), `shade_shaped` their terms, in the same conventions.

Either set also shades every pixel of the per-pixel shading's G-buffer (PIXEL LIGHTS): `RayTracer.trace_pixel_lights`
traces T [R,H,W] from each pixel's surface point, and `shade_pixels` returns terms to add to `shading.shade_pixels`'
outputs.
"""
import ctypes

import torch

from . import _lib

MAX_LIGHTS = 32          # R3DG_MAX_LIGHTS (include/r3dg_b200.h)
MAX_VIEWS = 64           # R3DG_MAX_VIEWS
DIRECTIONAL, POINT = 0, 1
SPOT, RECT = 2, 3
MAX_RECT_SAMPLES = 8     # R3DG_MAX_RECT_SAMPLES
MAX_SHAPED_RAYS = 256    # R3DG_MAX_SHAPED_RAYS: shadow columns per set


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


# ---- spot and rect lights ----------------------------------------------------------------------------------------
class ShapedLights:
    """K spot and rect lights with M x M samples per rect and one sample seed (include/r3dg_b200.h, SHAPED LIGHTS).
    kind [K] int32 (2 spot, 3 rect; kept on the host) and, per light, pos [K,3] (spot position, rect centre), a [K,3]
    (spot axis, the direction it points; rect half-edge u), b [K,3] (rect half-edge v), color [K,3] (spot intensity,
    rect radiance) and cone [K,2] (spot cos_inner, cos_outer).  Fields a kind does not use are ignored and get a zero
    gradient.  pos, a, b, color and cone may require grad."""

    def __init__(self, kind, pos, a, b, color, cone, M=4, seed=0):
        kind = torch.as_tensor(kind, dtype=torch.int32).detach().cpu().reshape(-1).contiguous()
        K = kind.numel()
        if K > MAX_LIGHTS:
            raise ValueError(f"at most {MAX_LIGHTS} lights per set (got {K})")
        if not bool(((kind == SPOT) | (kind == RECT)).all()):
            raise ValueError("shaped light kinds must be 2 (spot) or 3 (rect)")
        if isinstance(M, bool) or int(M) != M or not 1 <= int(M) <= MAX_RECT_SAMPLES:
            raise ValueError(f"M must be an integer in 1..{MAX_RECT_SAMPLES} (got {M})")
        for name, t, w in (("pos", pos, 3), ("a", a, 3), ("b", b, 3), ("color", color, 3), ("cone", cone, 2)):
            if t.shape != (K, w):
                raise ValueError(f"{name} must be [K,{w}] with K = {K} (got {tuple(t.shape)})")
        if len({t.device for t in (pos, a, b, color, cone)}) != 1:
            raise ValueError("the fields of a light set must be on one device")
        self.kind, self.pos, self.a, self.b, self.color, self.cone = kind, pos, a, b, color, cone
        self.M, self.seed = int(M), int(seed) & 0xFFFFFFFF
        if self.num_rays() > MAX_SHAPED_RAYS:
            raise ValueError(f"a set traces at most {MAX_SHAPED_RAYS} shadow rays per Gaussian (got {self.num_rays()}: "
                             f"1 per spot, M^2 = {self.M * self.M} per rect)")

    def __len__(self):
        return self.kind.numel()

    def num_rays(self):
        """R: the shadow columns of the set, 1 per spot and M^2 per rect, in light order."""
        return int(((self.kind == SPOT).sum() + (self.kind == RECT).sum() * self.M * self.M).item())

    @staticmethod
    def spot(pos, axis, color, cos_inner, cos_outer, M=4, seed=0):
        """Spots at pos [K,3] pointing along axis [K,3]: full intensity color [K,3] inside cos_inner, none outside
        cos_outer, a smoothstep between.  cos_inner and cos_outer are numbers or [K] tensors."""
        K = pos.shape[0]
        ci, co = (torch.as_tensor(c, dtype=pos.dtype, device=pos.device).expand(K) for c in (cos_inner, cos_outer))
        return ShapedLights(torch.full((K,), SPOT, dtype=torch.int32), pos, axis, torch.zeros_like(pos), color,
                            torch.stack([ci, co], -1), M, seed)

    @staticmethod
    def rect(center, u, v, radiance, M=4, seed=0):
        """One-sided parallelograms center + s u + t v (s, t in [-1, 1]) emitting radiance [K,3] along u x v."""
        K = center.shape[0]
        return ShapedLights(torch.full((K,), RECT, dtype=torch.int32), center, u, v, radiance,
                            torch.zeros((K, 2), dtype=center.dtype, device=center.device), M, seed)

    @staticmethod
    def cat(*sets, M=None, seed=None):
        """The lights of `sets` in order, with M and seed of the first set unless given."""
        return ShapedLights(torch.cat([s.kind for s in sets]), *(torch.cat([getattr(s, f) for s in sets])
                                                                   for f in ("pos", "a", "b", "color", "cone")),
                            sets[0].M if M is None else M, sets[0].seed if seed is None else seed)


def _shaped_args(P, V, lights, ts):
    """ShapedLightArgs over the contiguous float32 inputs ts = (pos, a, b, color, cone, means3D, base_color, roughness,
    normals, viewdirs, shadows)."""
    a = _lib.ShapedLightArgs()
    a.P, a.K, a.V, a.M, a.seed = P, len(lights), V, lights.M, lights.seed
    a.kind = lights.kind.data_ptr() if len(lights) > 0 else None
    (a.pos, a.a, a.b, a.color, a.cone, a.means3D, a.base_color, a.roughness, a.normals, a.viewdirs,
     a.shadows) = [_lib.ptr(t) for t in ts]
    return a


class _ShadeShaped(torch.autograd.Function):
    """The shaped lights' terms for V views (viewdirs [V,P,3]); one node for one view and for several."""

    @staticmethod
    def forward(ctx, base_color, roughness, viewdirs, means3D, pos, a, b, color, cone, normals, shadows, lights):
        V, P = viewdirs.shape[0], viewdirs.shape[1]
        ts = [_lib.f32(t) for t in (pos, a, b, color, cone, means3D, base_color, roughness, normals, viewdirs, shadows)]
        f = dict(dtype=torch.float32, device=viewdirs.device)
        outs = [torch.empty((V, P, 3), **f) for _ in range(3)]
        args = _shaped_args(P, V, lights, ts)
        args.pbr, args.diffuse_light, args.specular = [_lib.ptr(t) for t in outs]
        if P > 0:
            _lib.call("r3dg_shade_shaped_lights_forward", viewdirs.device, ctypes.byref(args), what="shade shaped lights")
        ctx.save_for_backward(*ts)
        ctx.lights, ctx.rough_shape = lights, roughness.shape
        return tuple(outs)

    @staticmethod
    def backward(ctx, g_pbr, g_diffuse, g_specular):
        ts = ctx.saved_tensors
        viewdirs = ts[9]
        V, P, K = viewdirs.shape[0], viewdirs.shape[1], len(ctx.lights)
        dev = viewdirs.device
        f = dict(dtype=torch.float32, device=dev)
        d_base, d_rough, d_view, d_mean = (torch.empty((P, 3), **f), torch.empty((P,), **f), torch.empty((V, P, 3), **f),
                                           torch.empty((P, 3), **f))
        d_pos, d_a, d_b, d_color, d_cone = [torch.empty((K, w), **f) for w in (3, 3, 3, 3, 2)]
        if P == 0:
            for t in (d_pos, d_a, d_b, d_color, d_cone):
                t.zero_()
        else:
            g = [None if t is None else _lib.f32(t) for t in (g_pbr, g_diffuse, g_specular)]
            if g[0] is None:
                g[0] = torch.zeros((V, P, 3), **f)
            args = _shaped_args(P, V, ctx.lights, ts)
            args.dL_dpbr, args.dL_ddiffuse_light, args.dL_dspecular = [_lib.ptr(t) for t in g]
            args.dL_dbase_color, args.dL_droughness, args.dL_dviewdirs, args.dL_dmeans3D = [
                _lib.ptr(t) for t in (d_base, d_rough, d_view, d_mean)]
            args.dL_dpos, args.dL_da, args.dL_db, args.dL_dcolor, args.dL_dcone = [
                _lib.ptr(t) for t in (d_pos, d_a, d_b, d_color, d_cone)]
            work = _lib.scratch(_lib.load().r3dg_shade_shaped_lights_work_bytes(P, K), dev)
            args.work, args.work_bytes = _lib.ptr(work), work.numel()
            _lib.call("r3dg_shade_shaped_lights_backward", dev, ctypes.byref(args), what="shade shaped lights backward")
        return (d_base, d_rough.view(ctx.rough_shape), d_view, d_mean, d_pos, d_a, d_b, d_color, d_cone, None, None, None)


def shade_shaped(base_color, roughness, normals, viewdirs, means3D, lights, shadows):
    """The terms of `lights` (ShapedLights) under shadows T [P,R] (RayTracer.trace_shaped_lights): returns (pbr,
    {"diffuse_light", "specular"}), each [P,3] for viewdirs [P,3] or [V,P,3] for viewdirs [V,P,3] (1 <= V <= MAX_VIEWS;
    each view equals a one-view call bit for bit).  Inputs are checked before anything is launched."""
    P = base_color.shape[0]
    R = lights.num_rays()
    one = viewdirs.dim() == 2
    vd = viewdirs.unsqueeze(0) if one else viewdirs
    if vd.dim() != 3 or vd.shape[1:] != (P, 3):
        raise ValueError(f"viewdirs must be [P,3] or [V,P,3] with P = {P} (got {tuple(viewdirs.shape)})")
    if not 1 <= vd.shape[0] <= MAX_VIEWS:
        raise ValueError(f"shade_shaped evaluates 1 to {MAX_VIEWS} views per call (got {vd.shape[0]})")
    if base_color.shape != (P, 3) or normals.shape != (P, 3) or means3D.shape != (P, 3) or roughness.numel() != P:
        raise ValueError("base_color, normals and means3D must be [P,3] and roughness [P] or [P,1]")
    if shadows.shape != (P, R):
        raise ValueError(f"shadows must be [P,R] = [{P},{R}] (got {tuple(shadows.shape)})")
    tensors = (base_color, roughness, normals, vd, means3D, shadows, lights.pos, lights.a, lights.b, lights.color, lights.cone)
    if not all(t.is_cuda for t in tensors):
        raise RuntimeError("lights.shade_shaped runs on the GPU only (no CPU path)")
    if len({t.device for t in tensors}) != 1:
        raise ValueError("every input of lights.shade_shaped must be on one device")
    pbr, diffuse, specular = _ShadeShaped.apply(base_color, roughness, vd, means3D, lights.pos, lights.a, lights.b,
                                                lights.color, lights.cone, normals, shadows, lights)
    if one:
        pbr, diffuse, specular = pbr[0], diffuse[0], specular[0]
    return pbr, {"diffuse_light": diffuse, "specular": specular}


# ---- per-pixel lights --------------------------------------------------------------------------------------------
def _fields(lights):
    """The set's differentiable fields in the PIXEL LIGHTS order: (vec, color) of a Lights set, (pos, a, b, color,
    cone) of a ShapedLights set."""
    return (lights.vec, lights.color) if isinstance(lights, Lights) else (lights.pos, lights.a, lights.b, lights.color,
                                                                          lights.cone)


def num_rays(lights):
    """R: the shadow columns of a Lights set (one per light) or a ShapedLights set (lights.num_rays())."""
    return len(lights) if isinstance(lights, Lights) else lights.num_rays()


def pixel_light_args(lights, points, mask):
    """PixelLightArgs with the set, views, size, points and mask of a per-pixel light call, and the tensors it points to
    (which must outlive the launch): (args, lead, keep) with lead = (leading shape, H, W)."""
    from .shading import _mask, _views
    if not isinstance(lights, (Lights, ShapedLights)):
        raise TypeError(f"lights must be a Lights or a ShapedLights set (got {type(lights).__name__})")
    p, lead = _views(points, 3, "points")
    m = _mask(mask, lead)
    fs = [_lib.f32(t) for t in _fields(lights)]
    if not all(t.is_cuda for t in fs):
        raise RuntimeError("per-pixel lights run on the GPU only (the light set must be on the GPU)")
    a = _lib.PixelLightArgs()
    a.V, a.H, a.W, a.K = p.shape[0], lead[1], lead[2], len(lights)
    a.kind = lights.kind.data_ptr() if len(lights) > 0 else None
    a.points, a.mask = p.data_ptr(), _lib.ptr(m)
    if isinstance(lights, Lights):
        a.M, a.seed = 1, 0
        a.pos, a.color = [_lib.ptr(t) for t in fs]
    else:
        a.M, a.seed = lights.M, lights.seed
        a.pos, a.a, a.b, a.color, a.cone = [_lib.ptr(t) for t in fs]
    return a, lead, [p, m] + fs


class _ShadePixelLights(torch.autograd.Function):
    """The per-pixel light terms of V views: one node with gradients to base_color, roughness and the light fields."""

    @staticmethod
    def forward(ctx, base_color, roughness, normal, points, campos, shadows, mask, lights, *fields):
        from .shading import _views
        a, lead, keep = pixel_light_args(lights, points, mask)
        V, H, W = a.V, a.H, a.W
        b, _ = _views(base_color, 3, "base_color", lead)
        r, _ = _views(roughness, 1, "roughness", lead)
        n, _ = _views(normal, 3, "normal", lead)
        T, _ = _views(shadows, num_rays(lights), "shadows", lead)
        cp = _lib.f32(campos).reshape(-1, 3)
        if cp.shape[0] != V or not cp.is_cuda:
            raise ValueError(f"campos must be a CUDA [3] or [V,3] tensor with V = {V}, got {tuple(campos.shape)}")
        a.base_color, a.roughness, a.normal, a.campos, a.shadows = (t.data_ptr() for t in (b, r, n, cp, T))
        f = dict(dtype=torch.float32, device=b.device)
        outs = [torch.empty((V, 3, H, W), **f) for _ in range(3)]
        a.pbr, a.diffuse_light, a.specular = (t.data_ptr() for t in outs)
        _lib.call("r3dg_shade_pixel_lights_forward", b.device, ctypes.byref(a), what="shade_pixels (lights)")
        ctx.save_for_backward(b, r, n, cp, T)
        ctx.keep, ctx.lights, ctx.lead = keep, lights, lead
        return tuple(t.reshape(lead[0] + t.shape[1:]) for t in outs)

    @staticmethod
    def backward(ctx, g_pbr, g_diffuse, g_specular):
        b, r, n, cp, T = ctx.saved_tensors
        lights = ctx.lights
        a, lead, keep = pixel_light_args(lights, ctx.keep[0], None)
        a.mask = _lib.ptr(ctx.keep[1])
        V, H, W, K = a.V, a.H, a.W, len(lights)
        a.base_color, a.roughness, a.normal, a.campos, a.shadows = (t.data_ptr() for t in (b, r, n, cp, T))
        dev = b.device
        f = dict(dtype=torch.float32, device=dev)
        g = [None if t is None else _lib.f32(t).reshape(V, 3, H, W) for t in (g_pbr, g_diffuse, g_specular)]
        if g[0] is None:
            g[0] = torch.zeros((V, 3, H, W), **f)
        a.dL_dpbr, a.dL_ddiffuse_light, a.dL_dspecular = (_lib.ptr(t) for t in g)
        d_base, d_rough = torch.empty_like(b), torch.empty_like(r)
        d_fields = [torch.empty((K, t.shape[1]), **f) for t in _fields(lights)]
        a.dL_dbase_color, a.dL_droughness = d_base.data_ptr(), d_rough.data_ptr()
        if isinstance(lights, Lights):
            a.dL_dpos, a.dL_dcolor = (_lib.ptr(t) for t in d_fields)
        else:
            a.dL_dpos, a.dL_da, a.dL_db, a.dL_dcolor, a.dL_dcone = (_lib.ptr(t) for t in d_fields)
        work = _lib.scratch(_lib.load().r3dg_shade_pixel_lights_work_bytes(V, H, W, K), dev)
        a.work, a.work_bytes = _lib.ptr(work), work.numel()
        _lib.call("r3dg_shade_pixel_lights_backward", dev, ctypes.byref(a), what="shade_pixels (lights) backward")
        shape = lambda t: t.reshape(ctx.lead[0] + t.shape[1:])
        return (shape(d_base), shape(d_rough), None, None, None, None, None, None, *d_fields)


def shade_pixels(base_color, roughness, normal, points, campos, lights, shadows, mask=None):
    """The terms of `lights` (Lights or ShapedLights) at every pixel of the per-pixel shading's G-buffer (include/
    r3dg_b200.h, PIXEL LIGHTS).  One view: base_color [3,H,W], roughness [1,H,W], normal [3,H,W], points [3,H,W],
    campos [3], shadows T [R,H,W] from RayTracer.trace_pixel_lights and an optional mask [H,W] (bool or uint8).  V views
    (1 <= V <= MAX_VIEWS): a leading V on every image and campos [V,3].

    Each valid pixel is `shade` / `shade_shaped` of one row (mean = its point, the raw normal, viewdir = campos -
    point, row index y W + x for the rect samples), bit for bit.  Returns dict(pbr, diffuse_light, specular), each
    [.., 3,H,W], to add to shading.shade_pixels' outputs; masked pixels are 0.  Gradients: base_color, roughness and the
    light fields (vec, color, or pos, a, b, color, cone), summed over pixels and views; none for normal, points, campos
    or the shadows.  Every output is bitwise reproducible.  Inputs are checked before anything is launched."""
    pbr, diffuse, specular = _ShadePixelLights.apply(base_color, roughness, normal, points, campos, shadows, mask, lights,
                                                     *_fields(lights))
    return {"pbr": pbr, "diffuse_light": diffuse, "specular": specular}

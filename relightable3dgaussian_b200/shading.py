"""Host-side mirror of the reference's shading step: `rendering_equation(...)` with the signature,
return value (pbr, extra_results dict) and light-object duck typing of
gaussian_renderer/neilf.py:339-371, backed by the fused sm_90a kernels
(r3dg_render_equation_forward / _backward).

The reference function lives inside gaussian_renderer/neilf.py (pure PyTorch), so there is no
extension module to replace; `install()` rebinds `gaussian_renderer.neilf.rendering_equation` (a
3-line plug-in, see INTEGRATION.md) for callers that must stay unmodified.

Gradients: base_color, roughness, viewdirs, incidents and the light's environment map (through
`light.get_env`, i.e. softplus, in PyTorch); normals and the baked tensors receive none, exactly as
in the reference call (neilf.py:92-96).  Under torch.use_deterministic_algorithms(True), read at call
time, the backward accumulates the environment-map gradient in fixed point, so every gradient is
bitwise reproducible (the reference's grid_sample backward raises under that flag).  The per-sample entries of extra_results
(`incident_lights`, `local_incident_lights`, `global_incident_lights`) are materialised lazily on
first access (eval only) and carry no gradient.
"""
import ctypes

import torch

from . import _lib


def _env_texture(light):
    """DirectLightMap -> softplus(env)[0] (differentiable); EnvLight -> envmap (+ rotation)."""
    if hasattr(light, "get_env"):
        env = light.get_env
        return (env[0] if env.dim() == 4 else env), None
    if hasattr(light, "envmap"):
        return light.envmap, getattr(light, "transform", None)
    raise TypeError("direct_light_env_light must expose `get_env` (DirectLightMap) or `envmap` (EnvLight)")


def _args(P, N, He, We):
    a = _lib.ShadeArgs()
    a.P, a.N, a.sh_coeffs, a.env_h, a.env_w = P, N, 16, He, We
    return a


def _c(t):
    return t.detach().float().contiguous()


class _RenderEquation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, base_color, roughness, viewdirs, incidents, env, normals, visibility, dirs, areas, transform, want_means):
        lib = _lib.load()
        P, N = dirs.shape[0], dirs.shape[1]
        dev = dirs.device
        ts = [_c(t) for t in (base_color, roughness, normals, viewdirs, incidents, env, visibility, dirs, areas)]
        tr = None if transform is None else _c(transform)
        f = dict(dtype=torch.float32, device=dev)
        pbr, diffuse, specular = (torch.empty((P, 3), **f) for _ in range(3))
        a = _args(P, N, env.shape[0], env.shape[1])
        (a.base_color, a.roughness, a.normals, a.viewdirs, a.incidents, a.env, a.visibility, a.incident_dirs,
         a.incident_areas) = [t.data_ptr() for t in ts]
        a.env_transform = None if tr is None else tr.data_ptr()
        a.pbr, a.diffuse_light, a.specular = pbr.data_ptr(), diffuse.data_ptr(), specular.data_ptr()
        means = None
        if want_means:
            means = [torch.empty((P, 3), **f) for _ in range(3)] + [torch.empty((P, 1), **f)]
            a.mean_incident_lights, a.mean_local_lights, a.mean_global_lights, a.mean_visibility = [m.data_ptr() for m in means]
        if P > 0:
            with torch.cuda.device(dev):
                _lib.check(lib.r3dg_render_equation_forward(ctypes.byref(a), torch.cuda.current_stream(dev).cuda_stream),
                           "rendering_equation")
        ctx.save_for_backward(*ts)
        ctx.transform = tr
        ctx.mark_non_differentiable(*(means or []))
        return (pbr, diffuse, specular) + tuple(means or [])

    @staticmethod
    def backward(ctx, g_pbr, g_diffuse, g_specular, *_):
        lib = _lib.load()
        base_color, roughness, normals, viewdirs, incidents, env, visibility, dirs, areas = ctx.saved_tensors
        P, N = dirs.shape[0], dirs.shape[1]
        dev = dirs.device
        f = dict(dtype=torch.float32, device=dev)
        d_base, d_view = torch.empty((P, 3), **f), torch.empty((P, 3), **f)
        d_rough = torch.empty((P, 1), **f)
        d_inc = torch.empty((P, 16, 3), **f)
        d_env = torch.empty(env.shape, **f)
        a = _args(P, N, env.shape[0], env.shape[1])
        (a.base_color, a.roughness, a.normals, a.viewdirs, a.incidents, a.env, a.visibility, a.incident_dirs,
         a.incident_areas) = [t.data_ptr() for t in (base_color, roughness, normals, viewdirs, incidents, env, visibility, dirs, areas)]
        a.env_transform = None if ctx.transform is None else ctx.transform.data_ptr()
        gz = torch.zeros((P, 3), **f)
        g = [gz if t is None else _c(t) for t in (g_pbr, g_diffuse, g_specular)]
        a.dL_dpbr, a.dL_ddiffuse_light, a.dL_dspecular = [t.data_ptr() for t in g]
        a.dL_dbase_color, a.dL_droughness, a.dL_dviewdirs = d_base.data_ptr(), d_rough.data_ptr(), d_view.data_ptr()
        a.dL_dincidents, a.dL_denv = d_inc.data_ptr(), d_env.data_ptr()
        if torch.are_deterministic_algorithms_enabled():
            ws = torch.empty((lib.r3dg_shade_det_bytes(env.shape[0], env.shape[1]),), dtype=torch.uint8, device=dev)
            a.deterministic, a.det_work, a.det_work_bytes = 1, ws.data_ptr(), ws.numel()
        with torch.cuda.device(dev):
            _lib.check(lib.r3dg_render_equation_backward(ctypes.byref(a), torch.cuda.current_stream(dev).cuda_stream),
                       "rendering_equation backward")
        return d_base, d_rough, d_view, d_inc, d_env, None, None, None, None, None, None


class _LazyExtras(dict):
    """extra_results dict whose three per-sample [P,N,3] entries are computed on first access."""
    _LAZY = ("incident_lights", "local_incident_lights", "global_incident_lights")

    def __init__(self, eager, maker):
        super().__init__(eager)
        self._maker = maker

    def _fill(self):
        if self._maker is not None:
            super().update(self._maker())
            self._maker = None

    def __getitem__(self, k):
        if k in self._LAZY and not super().__contains__(k):
            self._fill()
        return super().__getitem__(k)

    def __contains__(self, k):
        return k in self._LAZY or super().__contains__(k)

    def keys(self):
        self._fill()
        return super().keys()

    def items(self):
        self._fill()
        return super().items()

    def __iter__(self):
        self._fill()
        return super().__iter__()


def rendering_equation(base_color, roughness, normals, viewdirs, incidents, direct_light_env_light=None,
                       visibility_precompute=None, incident_dirs_precompute=None, incident_areas_precompute=None):
    """Drop-in for gaussian_renderer/neilf.py:339-371: returns (pbr [P,3], extra_results)."""
    if incidents.shape[1] != 16:
        raise RuntimeError("incidents must be degree-3 SH coefficients [P,16,3]")
    env, transform = _env_texture(direct_light_env_light)
    dirs, areas, vis = incident_dirs_precompute, incident_areas_precompute, visibility_precompute
    pbr, diffuse, specular = _RenderEquation.apply(base_color, roughness, viewdirs, incidents, env, normals, vis, dirs,
                                                   areas, transform, False)

    def per_sample():
        lib = _lib.load()
        P, N = dirs.shape[0], dirs.shape[1]
        f = dict(dtype=torch.float32, device=dirs.device)
        outs = [torch.empty((P, N, 3), **f) for _ in range(3)]
        scratch = [torch.empty((P, 3), **f) for _ in range(3)]
        ts = [_c(t) for t in (base_color, roughness, normals, viewdirs, incidents, env, vis, dirs, areas)]
        tr = None if transform is None else _c(transform)
        a = _args(P, N, env.shape[0], env.shape[1])
        (a.base_color, a.roughness, a.normals, a.viewdirs, a.incidents, a.env, a.visibility, a.incident_dirs,
         a.incident_areas) = [t.data_ptr() for t in ts]
        a.env_transform = None if tr is None else tr.data_ptr()
        a.pbr, a.diffuse_light, a.specular = [t.data_ptr() for t in scratch]
        a.incident_lights, a.local_incident_lights, a.global_incident_lights = [t.data_ptr() for t in outs]
        if P > 0:
            with torch.cuda.device(dirs.device):
                _lib.check(lib.r3dg_render_equation_forward(ctypes.byref(a), torch.cuda.current_stream(dirs.device).cuda_stream),
                           "rendering_equation (per-sample lights)")
        return dict(zip(_LazyExtras._LAZY, outs))

    extra = _LazyExtras({"incident_dirs": dirs, "incident_visibility": vis, "diffuse_light": diffuse, "specular": specular},
                        per_sample)
    return pbr, extra


def install(module=None):
    """Rebind `rendering_equation` inside the reference's gaussian_renderer.neilf (or `module`)."""
    if module is None:
        import gaussian_renderer.neilf as module
    module.rendering_equation = rendering_equation
    return module

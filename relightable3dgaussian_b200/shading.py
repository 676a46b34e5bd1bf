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

Filtered environment lighting (opt-in: `env_filter=True`, or `set_env_filter(True)` for the process): each incident
sample reads the environment averaged over its own solid angle from a lat-long mip pyramid instead of one bilinear
tap (include/r3dg_b200.h, PREFILTERED ENVIRONMENT).  The pyramid is built from the activated env on every call, so
the env gradient flows through it (and softplus); at footprints below a texel the lookup is the point lookup, bit for
bit.
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


_ENV_FILTER = False      # process default of `env_filter` (set_env_filter)


def set_env_filter(enabled):
    """Process default of the filtered environment lookup for calls that pass env_filter=None (the reference's
    unmodified callers after install()).  Off by default.  Returns the previous setting."""
    global _ENV_FILTER
    prev, _ENV_FILTER = _ENV_FILTER, bool(enabled)
    return prev


def _filter_on(env_filter):
    return _ENV_FILTER if env_filter is None else bool(env_filter)


def env_pyramid(env):
    """The filtered mode's mip pyramid of the activated env [He,We,3] (all levels, level 0 = env, flattened), or None
    when the env has no coarser level (fewer than 3 rows or columns): the mode then changes nothing."""
    env = _lib.f32(env)
    He, We = env.shape[0], env.shape[1]
    lib = _lib.load()
    if lib.r3dg_env_pyramid_levels(He, We) <= 1:
        return None
    pyr = torch.empty((lib.r3dg_env_pyramid_floats(He, We),), dtype=torch.float32, device=env.device)
    _lib.call("r3dg_env_pyramid_build", env.device, env.data_ptr(), He, We, pyr.data_ptr(), what="env pyramid build")
    return pyr


def _args(P, N, He, We):
    a = _lib.ShadeArgs()
    a.P, a.N, a.sh_coeffs, a.env_h, a.env_w = P, N, 16, He, We
    return a


def _shade_args(inputs, transform):
    """ShadeArgs for the nine inputs (base_color, roughness, normals, viewdirs, incidents, env, visibility,
    incident_dirs, incident_areas) and the optional env transform, all as contiguous float32.  viewdirs [P,3] is one
    view; viewdirs [V,P,3] is V views, with a [3,3] transform or one [V,3,3] per view.  Returns the struct and the
    converted inputs and transform, which must outlive the launch."""
    ts = [_lib.f32(t) for t in inputs]
    tr = None if transform is None else _lib.f32(transform)
    viewdirs, env, dirs = ts[3], ts[5], ts[7]
    a = _args(dirs.shape[0], dirs.shape[1], env.shape[0], env.shape[1])
    (a.base_color, a.roughness, a.normals, a.viewdirs, a.incidents, a.env, a.visibility, a.incident_dirs,
     a.incident_areas) = [t.data_ptr() for t in ts]
    a.env_transform = None if tr is None else tr.data_ptr()
    if viewdirs.dim() == 3:
        a.V, a.transform_per_view = viewdirs.shape[0], int(tr is not None and tr.dim() == 3)
    return a, ts, tr


class _RenderEquation(torch.autograd.Function):
    """The shading step of one view (viewdirs [P,3], outputs [P,*]) or of V views (viewdirs [V,P,3], outputs [V,P,*])."""

    @staticmethod
    def forward(ctx, base_color, roughness, viewdirs, incidents, env, normals, visibility, dirs, areas, transform, want_means,
                env_filter=False):
        P = dirs.shape[0]
        lead = tuple(viewdirs.shape[:-2])
        f = dict(dtype=torch.float32, device=dirs.device)
        a, ts, tr = _shade_args((base_color, roughness, normals, viewdirs, incidents, env, visibility, dirs, areas), transform)
        pyr = env_pyramid(ts[5]) if env_filter and P > 0 else None
        a.env_pyramid = None if pyr is None else pyr.data_ptr()
        pbr, diffuse, specular = (torch.empty(lead + (P, 3), **f) for _ in range(3))
        a.pbr, a.diffuse_light, a.specular = pbr.data_ptr(), diffuse.data_ptr(), specular.data_ptr()
        means = []
        if want_means:
            means = [torch.empty(lead + (P, 3), **f) for _ in range(3)] + [torch.empty(lead + (P, 1), **f)]
            a.mean_incident_lights, a.mean_local_lights, a.mean_global_lights, a.mean_visibility = [m.data_ptr() for m in means]
        if P > 0:
            _lib.call("r3dg_render_equation_forward", dirs.device, ctypes.byref(a), what="rendering_equation")
        ctx.save_for_backward(*ts)
        ctx.transform, ctx.pyramid = tr, pyr
        ctx.mark_non_differentiable(*means)
        return (pbr, diffuse, specular) + tuple(means)

    @staticmethod
    def backward(ctx, g_pbr, g_diffuse, g_specular, *_):
        a, ts, _ = _shade_args(ctx.saved_tensors, ctx.transform)
        env, viewdirs, dirs = ts[5], ts[3], ts[7]
        P = dirs.shape[0]
        dev = dirs.device
        f = dict(dtype=torch.float32, device=dev)
        d_base, d_view = torch.empty((P, 3), **f), torch.empty(viewdirs.shape, **f)
        d_rough = torch.empty((P, 1), **f)
        d_inc = torch.empty((P, 16, 3), **f)
        d_env = torch.empty(env.shape, **f)
        if P == 0:                      # nothing to shade: empty gradients (no device pointers to pass)
            return d_base, d_rough, d_view, d_inc, d_env.zero_(), None, None, None, None, None, None, None
        gz = torch.zeros(viewdirs.shape, **f)
        g = [gz if t is None else _lib.f32(t) for t in (g_pbr, g_diffuse, g_specular)]
        a.dL_dpbr, a.dL_ddiffuse_light, a.dL_dspecular = [t.data_ptr() for t in g]
        a.dL_dbase_color, a.dL_droughness, a.dL_dviewdirs = d_base.data_ptr(), d_rough.data_ptr(), d_view.data_ptr()
        a.dL_dincidents, a.dL_denv = d_inc.data_ptr(), d_env.data_ptr()
        lib, pyr, g_pyr = _lib.load(), ctx.pyramid, None
        if pyr is not None:             # the gradient of every pyramid level, folded into dL/denv by the call
            a.env_pyramid, g_pyr = pyr.data_ptr(), torch.empty_like(pyr)
            a.dL_denv_pyramid = g_pyr.data_ptr()
        det_bytes = (lib.r3dg_shade_det_bytes if pyr is None else lib.r3dg_shade_filtered_det_bytes)(env.shape[0], env.shape[1])
        det_ws = _lib.det_workspace(a, det_bytes, dev)
        _lib.call("r3dg_render_equation_backward", dev, ctypes.byref(a), what="rendering_equation backward")
        return d_base, d_rough, d_view, d_inc, d_env, None, None, None, None, None, None, None


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
                       visibility_precompute=None, incident_dirs_precompute=None, incident_areas_precompute=None,
                       env_filter=None):
    """Drop-in for gaussian_renderer/neilf.py:339-371: returns (pbr [P,3], extra_results).  env_filter: True reads the
    environment filtered over each sample's footprint, False the point lookup, None the process default
    (set_env_filter)."""
    if incidents.shape[1] != 16:
        raise RuntimeError("incidents must be degree-3 SH coefficients [P,16,3]")
    env, transform = _env_texture(direct_light_env_light)
    dirs, areas, vis = incident_dirs_precompute, incident_areas_precompute, visibility_precompute
    filt = _filter_on(env_filter)
    pbr, diffuse, specular = _RenderEquation.apply(base_color, roughness, viewdirs, incidents, env, normals, vis, dirs,
                                                   areas, transform, False, filt)

    def per_sample():
        a, ts, tr = _shade_args((base_color, roughness, normals, viewdirs, incidents, env, vis, dirs, areas), transform)
        P, N = dirs.shape[0], dirs.shape[1]
        pyr = env_pyramid(ts[5]) if filt and P > 0 else None
        a.env_pyramid = None if pyr is None else pyr.data_ptr()
        f = dict(dtype=torch.float32, device=dirs.device)
        outs = [torch.empty((P, N, 3), **f) for _ in range(3)]
        scratch = [torch.empty((P, 3), **f) for _ in range(3)]
        a.pbr, a.diffuse_light, a.specular = [t.data_ptr() for t in scratch]
        a.incident_lights, a.local_incident_lights, a.global_incident_lights = [t.data_ptr() for t in outs]
        if P > 0:
            _lib.call("r3dg_render_equation_forward", dirs.device, ctypes.byref(a), what="rendering_equation (per-sample lights)")
        return dict(zip(_LazyExtras._LAZY, outs))

    extra = _LazyExtras({"incident_dirs": dirs, "incident_visibility": vis, "diffuse_light": diffuse, "specular": specular},
                        per_sample)
    return pbr, extra


MAX_VIEWS = 64          # R3DG_MAX_VIEWS (include/r3dg_b200.h)
_MEANS = ("mean_incident_lights", "mean_local_incident_lights", "mean_global_incident_lights", "mean_incident_visibility")


def rendering_equation_views(base_color, roughness, normals, viewdirs, incidents, direct_light_env_light=None,
                             visibility_precompute=None, incident_dirs_precompute=None, incident_areas_precompute=None,
                             means=False, env_filter=None, sampler=None):
    """`rendering_equation` for V view directions of the same Gaussians in one call: viewdirs [V,P,3], every other input
    as in `rendering_equation`.  The incident light of each sample is evaluated once for all views.

    Returns (pbr [V,P,3], extra) with extra = {incident_dirs, incident_visibility (the baked tensors), diffuse_light
    [V,P,3], specular [V,P,3]} and, with means=True, mean_incident_lights, mean_local_incident_lights,
    mean_global_incident_lights [V,P,3] and mean_incident_visibility [V,P,1] (the `.mean(-2)` of the per-sample lights;
    no gradient).  Each view's outputs equal a one-view call with that view's direction and transform bit for bit.

    An EnvLight `transform` may be [3,3] or [V,3,3] (one per view, forward only).  Gradients: viewdirs per view;
    base_color, roughness, incidents and the environment map summed over the views; none for normals and the baked
    tensors.  Refused before anything is launched: V outside 1..MAX_VIEWS, viewdirs not [V,P,3], incidents not [P,16,3],
    a [V',3,3] transform with V' != V, and per-view transforms when autograd would need a backward.  env_filter: as in
    `rendering_equation`; the filtered light is evaluated once per sample for all views (per view with per-view
    transforms).  sampler: the EnvSampler the directions and areas came from (importance_sample or
    RayTracer.bake_importance); the views share them, so it is refused when its mix has GGX samples (they depend on
    the view) or with per-view transforms (the env samples follow one transform)."""
    dirs, areas, vis = incident_dirs_precompute, incident_areas_precompute, visibility_precompute
    P = dirs.shape[0]
    if sampler is not None:
        transform = _env_texture(direct_light_env_light)[1]
        if sampler.counts(dirs.shape[1])[1] > 0:
            raise ValueError("rendering_equation_views shares its directions over the views: a sampler with GGX "
                             "samples (per-view directions) is refused; use mix=(m_env, 0, m_cos)")
        if transform is not None and transform.dim() == 3:
            raise ValueError("a sampler follows one env transform: per-view transforms are refused")
        sampler.check_light(direct_light_env_light, "rendering_equation_views")
    if viewdirs.dim() != 3 or viewdirs.shape[1:] != (P, 3):
        raise ValueError(f"viewdirs must be [V,P,3] with P = {P} (got {tuple(viewdirs.shape)})")
    V = viewdirs.shape[0]
    if not 1 <= V <= MAX_VIEWS:
        raise ValueError(f"rendering_equation_views shades 1 to {MAX_VIEWS} views per call (got {V})")
    if incidents.shape[1:] != (16, 3):
        raise RuntimeError("incidents must be degree-3 SH coefficients [P,16,3]")
    env, transform = _env_texture(direct_light_env_light)
    if transform is not None and transform.dim() == 3:
        if transform.shape != (V, 3, 3):
            raise ValueError(f"a per-view transform must be [V,3,3] with V = {V} (got {tuple(transform.shape)})")
        if torch.is_grad_enabled() and any(t.requires_grad for t in (base_color, roughness, viewdirs, incidents, env)):
            raise ValueError("per-view transforms are forward-only: call under torch.no_grad() or with detached inputs")
    outs = _RenderEquation.apply(base_color, roughness, viewdirs, incidents, env, normals, vis, dirs, areas, transform,
                                 bool(means), _filter_on(env_filter))
    pbr, diffuse, specular = outs[:3]
    extra = {"incident_dirs": dirs, "incident_visibility": vis, "diffuse_light": diffuse, "specular": specular}
    extra.update(zip(_MEANS, outs[3:]))
    return pbr, extra


class EnvSampler:
    """The importance sampler of an environment light (include/r3dg_b200.h, IMPORTANCE SAMPLING): a table built once
    from the detached activated env, the EnvLight transform it samples under, the strategy mix (env, GGX, cosine) and
    the seed.  Refused on the host: a mix that is negative or does not sum to 1, an env with fewer than 2 rows or
    columns, a transform that is not one orthonormal [3,3] (to 1e-4), a seed outside [0, 2^32).  The table follows
    the env as it was at construction; rebuilding it after an env update is the caller's choice."""

    def __init__(self, direct_light_env_light, mix=(0.5, 0.25, 0.25), seed=0):
        env, transform = _env_texture(direct_light_env_light)
        mix = tuple(float(m) for m in mix)
        if len(mix) != 3 or not all(m >= 0 for m in mix) or abs(sum(mix) - 1.0) > 1e-6:
            raise ValueError(f"mix must be three non-negative weights (env, ggx, cos) summing to 1, got {mix}")
        if not 0 <= int(seed) < 2 ** 32:
            raise ValueError(f"seed must be in [0, 2^32), got {seed}")
        env = _lib.f32(env)
        if env.dim() != 3 or env.shape[2] != 3 or env.shape[0] < 2 or env.shape[1] < 2:
            raise ValueError(f"the env must be [He,We,3] with He, We >= 2, got {tuple(env.shape)}")
        tr = None
        if transform is not None:
            tr = _lib.f32(transform)
            if tr.device != env.device:
                raise ValueError(f"the env transform must be on the env's device {env.device}, got {tr.device}")
            if tr.shape != (3, 3):
                raise ValueError(f"the sampler takes one [3,3] env transform, got {tuple(tr.shape)}")
            err = float((tr.double() @ tr.double().T - torch.eye(3, dtype=torch.float64, device=tr.device)).abs().max())
            if not err <= 1e-4:
                raise ValueError(f"the env transform must be orthonormal to 1e-4 (|T T^T - I| = {err:.3g})")
        if not env.is_cuda:
            raise RuntimeError("EnvSampler builds its table on the GPU only (no CPU path)")
        He, We = env.shape[0], env.shape[1]
        lib = _lib.load()
        self.table = torch.empty((lib.r3dg_env_sampler_floats(He, We),), dtype=torch.float32, device=env.device)
        _lib.call("r3dg_env_sampler_build", env.device, env.data_ptr(), He, We, self.table.data_ptr(), what="env sampler build")
        self.transform, self.mix, self.seed, self.env_shape = tr, mix, int(seed), (He, We)

    def counts(self, N):
        """(n_env, n_ggx, n_cos) of N samples: n_env = floor(N m_e + 1/2), n_env + n_ggx = floor(N (m_e + m_g) + 1/2).
        Refuses a split without a cosine sample (the cosine lobe is what keeps the estimator unbiased)."""
        N = int(N)
        n_env = int(N * self.mix[0] + 0.5)
        n_eg = int(N * (self.mix[0] + self.mix[1]) + 0.5)
        if N - n_eg < 1:
            raise ValueError(f"mix {self.mix} leaves no cosine sample of N = {N}: at least one is required")
        return n_env, n_eg - n_env, N - n_eg

    def check_light(self, direct_light_env_light, what):
        """Refuse a light whose env size or (one [3,3]) transform differs from the sampler's: its areas would be wrong."""
        env, transform = _env_texture(direct_light_env_light)
        if tuple(env.shape[:2]) != self.env_shape:
            raise ValueError(f"{what}: the light's env is {tuple(env.shape[:2])}, the sampler's {self.env_shape}")
        if transform is not None and transform.dim() == 3:
            return
        same = (transform is None) == (self.transform is None) and (
            transform is None or torch.equal(_lib.f32(transform).to(self.transform.device), self.transform))
        if not same:
            raise ValueError(f"{what}: the light's env transform is not the one the sampler was built with")

    def fill(self, args, N):
        """Enter the sampler into a PixelArgs record for N samples per pixel."""
        n_env, n_ggx, _ = self.counts(N)
        args.sampler_table, args.n_env, args.n_ggx, args.seed = self.table.data_ptr(), n_env, n_ggx, self.seed
        args.sampler_transform = _lib.ptr(self.transform)
        return n_ggx


def importance_sample(normals, sampler, N, viewdirs=None, roughness=None):
    """N importance-sampled incident directions per Gaussian row (r3dg_sample_importance_dirs): (dirs [P,N,3],
    areas [P,N,1]), the `incident_dirs_precompute` / `incident_areas_precompute` of `rendering_equation` shaded under
    the sampler's light.  normals [P,3]; viewdirs [P,3] and roughness [P,1] are required when the mix has GGX samples.
    Row g's numbers are hashed with g.  No gradient."""
    n = _lib.f32(normals).reshape(-1, 3)
    P = n.shape[0]
    n_env, n_ggx, _ = sampler.counts(N)
    if n_ggx > 0 and (viewdirs is None or roughness is None):
        raise ValueError("GGX samples need viewdirs and roughness")
    if not n.is_cuda:
        raise RuntimeError("importance_sample runs on the GPU only (no CPU path)")
    if n.device != sampler.table.device:
        raise ValueError(f"normals are on {n.device}, the sampler on {sampler.table.device}")
    v = None if n_ggx == 0 else _lib.f32(viewdirs).reshape(-1, 3)
    r = None if n_ggx == 0 else _lib.f32(roughness).reshape(-1)
    if v is not None and (v.shape[0] != P or r.shape[0] != P):
        raise ValueError(f"viewdirs and roughness must hold P = {P} rows")
    if v is not None and (v.device != n.device or r.device != n.device):
        raise ValueError(f"viewdirs and roughness must be on the normals' device {n.device}")
    f = dict(dtype=torch.float32, device=n.device)
    dirs, areas = torch.empty((P, int(N), 3), **f), torch.empty((P, int(N), 1), **f)
    _lib.call("r3dg_sample_importance_dirs", n.device, P, int(N), _lib.ptr(n), _lib.ptr(v), _lib.ptr(r),
              sampler.table.data_ptr(), _lib.ptr(sampler.transform), n_env, n_ggx, sampler.seed, _lib.ptr(dirs),
              _lib.ptr(areas), what="importance_sample")
    return dirs, areas


def install(module=None):
    """Rebind `rendering_equation` inside the reference's gaussian_renderer.neilf (or `module`).  Its callers pass no
    env_filter, so set_env_filter decides their lookup."""
    if module is None:
        import gaussian_renderer.neilf as module
    module.rendering_equation = rendering_equation
    return module


# ---- per-pixel (deferred) shading ------------------------------------------------------------------------------------
def _views(t, C, name, lead=None):
    """A planar image `t` [C,H,W] (one view) or [V,C,H,W] as contiguous float32 [V,C,H,W], and (leading shape, H, W).
    lead: the call's (leading shape, H, W) to match."""
    if t.dim() not in (3, 4) or t.shape[-3] != C:
        raise ValueError(f"{name} must be [{C},H,W] or [V,{C},H,W], got {tuple(t.shape)}")
    shape = (tuple(t.shape[:-3]), t.shape[-2], t.shape[-1])
    if lead is not None and shape != lead:
        raise ValueError(f"{name} {tuple(t.shape)} does not match the images' views and size {lead}")
    if not 1 <= (t.shape[0] if t.dim() == 4 else 1) <= MAX_VIEWS:
        raise ValueError(f"per-pixel shading takes 1 to {MAX_VIEWS} views per call (got {t.shape[0]})")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (per-pixel shading runs on the GPU only)")
    x = _lib.f32(t)
    return (x if x.dim() == 4 else x.unsqueeze(0)), shape


def _mask(mask, lead):
    """The optional validity mask [H,W] or [V,H,W] (bool or uint8) as contiguous uint8 [V,H,W]."""
    if mask is None:
        return None
    if mask.dtype not in (torch.bool, torch.uint8) or tuple(mask.shape) != lead[0] + (lead[1], lead[2]):
        raise ValueError(f"mask must be bool or uint8 {lead[0] + (lead[1], lead[2])}, got {mask.dtype} {tuple(mask.shape)}")
    if not mask.is_cuda:
        raise RuntimeError("mask must be a CUDA tensor (per-pixel shading runs on the GPU only)")
    m = mask.detach().contiguous()
    m = m.view(torch.uint8) if m.dtype == torch.bool else m
    return m.reshape(-1, lead[1], lead[2])


def pixel_args(normal, points, N, mask):
    """PixelArgs with the views, size, samples, normal, points and mask of a per-pixel call, and the tensors it points
    to (which must outlive the launch): (args, lead, [normal, points, mask]) with lead = (leading shape, H, W)."""
    n, lead = _views(normal, 3, "normal")
    p, _ = _views(points, 3, "points", lead)
    m = _mask(mask, lead)
    if not 1 <= int(N):
        raise ValueError(f"sample_num must be >= 1 (got {N})")
    a = _lib.PixelArgs()
    a.V, a.H, a.W, a.N = n.shape[0], lead[1], lead[2], int(N)
    a.normal, a.points, a.mask = n.data_ptr(), p.data_ptr(), _lib.ptr(m)
    return a, lead, [n, p, m]


class _ShadePixels(torch.autograd.Function):
    """The per-pixel shading of V views: one node with gradients to base_color, roughness, incidents and env."""

    @staticmethod
    def forward(ctx, base_color, roughness, incidents, env, normal, points, campos, visibility, mask, transform, env_filter,
                sampler=None):
        a, lead, keep = pixel_args(normal, points, visibility.shape[-3], mask)
        if sampler is not None:
            if sampler.table.device != normal.device:
                raise ValueError(f"the sampler is on {sampler.table.device}, the images on {normal.device}")
            sampler.fill(a, a.N)
        V, H, W = a.V, a.H, a.W
        b, _ = _views(base_color, 3, "base_color", lead)
        r, _ = _views(roughness, 1, "roughness", lead)
        vis, _ = _views(visibility, a.N, "visibility", lead)
        inc = None if incidents is None else _views(incidents, 48, "incidents", lead)[0]
        cp = _lib.f32(campos).reshape(-1, 3)
        if cp.shape[0] != V or not cp.is_cuda:
            raise ValueError(f"campos must be a CUDA [3] or [V,3] tensor with V = {V}, got {tuple(campos.shape)}")
        e = _lib.f32(env)
        tr = None if transform is None else _lib.f32(transform)
        if tr is not None and tr.shape not in ((3, 3), (V, 3, 3)):
            raise ValueError(f"the env transform must be [3,3] or [V,3,3] with V = {V}, got {tuple(tr.shape)}")
        a.env_h, a.env_w = e.shape[0], e.shape[1]
        a.base_color, a.roughness, a.campos, a.incidents, a.env = b.data_ptr(), r.data_ptr(), cp.data_ptr(), _lib.ptr(inc), e.data_ptr()
        a.env_transform, a.transform_per_view = _lib.ptr(tr), int(tr is not None and tr.dim() == 3)
        a.visibility = vis.data_ptr()
        pyr = env_pyramid(e) if env_filter else None
        a.env_pyramid = _lib.ptr(pyr)
        f = dict(dtype=torch.float32, device=b.device)
        pbr, diffuse, specular = (torch.empty((V, 3, H, W), **f) for _ in range(3))
        mean_vis = torch.empty((V, 1, H, W), **f)
        a.pbr, a.diffuse_light, a.specular, a.mean_visibility = (t.data_ptr() for t in (pbr, diffuse, specular, mean_vis))
        _lib.call("r3dg_shade_pixels_forward", b.device, ctypes.byref(a), what="shade_pixels")
        ctx.save_for_backward(b, r, inc, e, vis, cp, tr, pyr, *keep[:2])
        ctx.mask, ctx.lead, ctx.sampler = keep[2], lead, sampler
        ctx.mark_non_differentiable(mean_vis)
        shape = lambda t: t.reshape(lead[0] + t.shape[1:])
        return shape(pbr), shape(diffuse), shape(specular), shape(mean_vis)

    @staticmethod
    def backward(ctx, g_pbr, g_diffuse, g_specular, _):
        b, r, inc, e, vis, cp, tr, pyr, n, p = ctx.saved_tensors
        V, H, W = b.shape[0], b.shape[2], b.shape[3]
        a = _lib.PixelArgs()
        a.V, a.H, a.W, a.N, a.env_h, a.env_w = V, H, W, vis.shape[1], e.shape[0], e.shape[1]
        a.base_color, a.roughness, a.normal, a.points, a.campos = (t.data_ptr() for t in (b, r, n, p, cp))
        a.incidents, a.mask, a.env, a.visibility = _lib.ptr(inc), _lib.ptr(ctx.mask), e.data_ptr(), vis.data_ptr()
        a.env_transform, a.transform_per_view = _lib.ptr(tr), int(tr is not None and tr.dim() == 3)
        if ctx.sampler is not None:
            ctx.sampler.fill(a, a.N)
        dev = b.device
        f = dict(dtype=torch.float32, device=dev)
        g = [None if t is None else _lib.f32(t).reshape(V, 3, H, W) for t in (g_pbr, g_diffuse, g_specular)]
        if g[0] is None:
            g[0] = torch.zeros((V, 3, H, W), **f)
        a.dL_dpbr, a.dL_ddiffuse_light, a.dL_dspecular = (_lib.ptr(t) for t in g)
        d_base, d_rough, d_env = torch.empty_like(b), torch.empty_like(r), torch.empty_like(e)
        d_inc = None if inc is None else torch.empty_like(inc)
        a.dL_dbase_color, a.dL_droughness, a.dL_dincidents, a.dL_denv = d_base.data_ptr(), d_rough.data_ptr(), _lib.ptr(d_inc), d_env.data_ptr()
        lib, g_pyr = _lib.load(), None
        if pyr is not None:
            a.env_pyramid, g_pyr = pyr.data_ptr(), torch.empty_like(pyr)
            a.dL_denv_pyramid = g_pyr.data_ptr()
        det_bytes = (lib.r3dg_shade_det_bytes if pyr is None else lib.r3dg_shade_filtered_det_bytes)(e.shape[0], e.shape[1])
        det_ws = _lib.det_workspace(a, det_bytes, dev)
        _lib.call("r3dg_shade_pixels_backward", dev, ctypes.byref(a), what="shade_pixels backward")
        shape = lambda t: None if t is None else t.reshape(ctx.lead[0] + t.shape[1:])
        return shape(d_base), shape(d_rough), shape(d_inc), d_env, None, None, None, None, None, None, None, None


def shade_pixels(base_color, roughness, normal, points, campos, visibility, direct_light_env_light, incidents=None,
                 mask=None, env_filter=None, sampler=None):
    """The shading step at every pixel of rasterized material images (deferred shading; include/r3dg_b200.h, PIXEL
    SHADING).  One view: base_color [3,H,W], roughness [1,H,W], normal [3,H,W] (un-premultiplied material channels),
    points [3,H,W] world-space surface points, campos [3], visibility [N,H,W] from RayTracer.trace_pixels, optional
    incidents [48,H,W] (channel 3k + c = SH coefficient k of colour c) and mask [H,W] (bool or uint8).  V views: a
    leading V on every image, campos [V,3], and an EnvLight transform of [3,3] or [V,3,3].

    Per valid pixel: the N samples of the sampler around normalize(normal) (area 2 pi), viewdir = campos - points,
    and the formula of `rendering_equation`, so each output equals that function on the pixel as a row bit for bit.
    Returns dict(pbr, diffuse_light, specular [.., 3,H,W], visibility [.., 1,H,W] = mean_i T); masked pixels are 0.
    Gradients: base_color, roughness, incidents and the environment map; none for normal, points, campos or the
    visibility.  env_filter: as in `rendering_equation` (None: set_env_filter's default).

    sampler: a shading.EnvSampler of this light (same env size and transform; a per-view transform is allowed, the env
    samples then follow the sampler's).  The N samples of pixel p = y W + x are the sampler's directions of row p with
    their areas (importance_sample of the pixels as rows), and `visibility` must be RayTracer.trace_pixels' T traced
    with the same sampler: this call cannot tell.  The returned visibility is then mean_i T over those directions."""
    env, transform = _env_texture(direct_light_env_light)
    if sampler is not None:
        sampler.check_light(direct_light_env_light, "shade_pixels")
    pbr, diffuse, specular, vis = _ShadePixels.apply(base_color, roughness, incidents, env, normal, points, campos, visibility,
                                                     mask, transform, _filter_on(env_filter), sampler)
    return {"pbr": pbr, "diffuse_light": diffuse, "specular": specular, "visibility": vis}

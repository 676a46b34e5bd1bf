"""Host-side mirror of the reference's BVH operator surface — `RayTracer` (bvh/__init__.py:28-71),
`sample_incident_rays` / `fibonacci_sphere_sampling` (scene/gaussian_model.py:20-28,
utils/graphics_utils.py:9-37, utils/sh_utils.py:36-68) and the visibility bake `update_visibility`
(scene/gaussian_model.py:312-342) — as thin marshalling over this project's CUDA kernels.  No sampling or
tracing arithmetic lives in this file: directions come from `r3dg_sample_incident_dirs`, the bake
from `r3dg_bvh_bake_visibility` (directions generated inside the trace kernel, written once).

Differences from the reference that are not observable in the results:
  * the ~60 small PyTorch kernels of RayTracer.__init__ are one fused kernel (same fp32 rounding);
  * trace_visibility does not materialise `rays_o + 0.05 * rays_d` nor the expanded origins;
  * update_visibility is ONE launch over all Gaussians in Morton order instead of the reference's
    chunk loop (the chunks only bound the size of its [chunk,N,3] PyTorch temporaries); the
    `[P,N,3]` ray-origin / ray-direction inputs of the reference's trace call never exist.

Beyond the reference: `RayTracer.bake_radiance` / `fit_incident_sh` / `update_incidents` compute each Gaussian's
incident-light SH (`incidents`) from the scene itself — the bake's rays composited front to back through the
other Gaussians (r3dg_bvh_bake_radiance), then a per-Gaussian ridge fit (r3dg_fit_incident_sh).
`RayTracer.trace_lights` traces the shadows of point and directional lights (lights.py), `trace_shaped_lights` those
of spot and rect lights.  `RayTracer.trace_pixels` traces the visibility of the per-pixel
shading (shading.shade_pixels) from the surface points of rasterized G-buffer images.
"""
import ctypes

import torch

from . import _C_bvh as _C
from . import _lib


def fibonacci_sphere_sampling(normals, sample_num, random_rotate=True):
    """utils/graphics_utils.py:9-37: (incident_dirs [...,N,3], incident_areas [...,N,1]).  With
    random_rotate the per-Gaussian phase is drawn here with torch.rand (as the reference does) and
    applied in the kernel."""
    pre_shape = normals.shape[:-1]
    n = _lib.f32(normals).reshape(-1, 3)
    P, N = n.shape[0], int(sample_num)
    if not n.is_cuda:
        raise RuntimeError("fibonacci_sphere_sampling runs on the GPU only (no CPU path)")
    dirs = torch.empty((P, N, 3), dtype=torch.float32, device=n.device)
    areas = torch.empty((P, N, 1), dtype=torch.float32, device=n.device)
    phase = torch.rand(P, device=n.device) if random_rotate else None
    if P > 0 and N > 0:
        _lib.call("r3dg_sample_incident_dirs", n.device, P, N, n.data_ptr(), _lib.ptr(phase), dirs.data_ptr(),
                  areas.data_ptr(), what="sample_incident_dirs")
    return dirs.reshape(*pre_shape, N, 3), areas.reshape(*pre_shape, N, 1)


def sample_incident_rays(normals, is_training=False, sample_num=24):
    """scene/gaussian_model.py:20-28."""
    return fibonacci_sphere_sampling(normals, sample_num, random_rotate=bool(is_training))


def inverse_covariance(scaling, rotation, scaling_modifier=1.0):
    """`GaussianModel.get_inverse_covariance` (scene/gaussian_model.py:257-260): the symmetric 6-vector of
    L L^T with L = R(q) diag(1 / (s / modifier))  (utils/general_utils.py:66-79,151-160).  Init-time host
    PyTorch in the reference too (a handful of [P,3,3] ops, once per bake)."""
    q = torch.nn.functional.normalize(rotation.float(), dim=-1)
    r, x, y, z = q.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1).view(-1, 3, 3)
    L = R * ((1.0 / scaling.float()) * (1.0 / scaling_modifier)).unsqueeze(1)
    cov = L @ L.transpose(1, 2)
    return torch.stack([cov[:, 0, 0], cov[:, 0, 1], cov[:, 0, 2], cov[:, 1, 1], cov[:, 1, 2], cov[:, 2, 2]], dim=-1).contiguous()


class RayTracer:
    """bvh/__init__.py:28-71: builds the LBVH in __init__, `trace_visibility` bakes T in {0} U [0.9,1]."""

    def __init__(self, means3D, scales, rotations):
        P = means3D.shape[0]
        dev = means3D.device
        nodes = torch.empty((2 * P - 1, 5), dtype=torch.int32, device=dev)
        aabbs = torch.empty((2 * P - 1, 6), dtype=torch.float32, device=dev)
        m, s, r = _lib.f32(means3D), _lib.f32(scales), _lib.aligned16(_lib.f32(rotations))
        _lib.call("r3dg_bvh_leaf_aabbs", dev, P, m.data_ptr(), s.data_ptr(), r.data_ptr(), nodes.data_ptr(), aabbs.data_ptr(),
                  what="RayTracer leaf boxes")
        self.tree, self.aabb, self.morton = _C.create_bvh(m, s, r, nodes, aabbs)

    @torch.no_grad()
    def trace_visibility(self, rays_o, rays_d, means3D, symm_inv, opacity, normals):
        # origins that are an expand() over the sample dimension are passed un-expanded
        group = 1
        if rays_o.dim() >= 2 and rays_o.shape == rays_d.shape and rays_o.stride(-2) == 0 and rays_d.is_contiguous():
            group = rays_o.shape[-2]
            rays_o = rays_o[..., 0, :]
        cotrib, opa = _C._trace(self.tree, self.aabb, rays_o, group, 0.05, rays_d, means3D, symm_inv, opacity, normals)
        return {"visibility": opa.unsqueeze(-1), "contribute": cotrib.unsqueeze(-1)}

    @torch.no_grad()
    def bake_visibility(self, means3D, symm_inv, opacity, normals, sample_num, first_slot=0, count=None, out=None,
                        want_contribute=False, write_dirs=True):
        """The whole of the reference's bake loop body for leaf slots [first_slot, first_slot + count) in one
        launch (r3dg_bvh_bake_visibility).  Returns dict(visibility [P,N,1], incident_dirs [P,N,3],
        incident_areas [P,N,1][, contribute]); rows of Gaussians outside the slot range keep the content of
        `out` (zero-initialised when not given) — that is what the sharded bake sums over the ranks."""
        P, N = means3D.shape[0], int(sample_num)
        dev = means3D.device
        count = P - first_slot if count is None else count
        f = dict(dtype=torch.float32, device=dev)
        if out is None:
            partial = first_slot != 0 or count != P
            mk = torch.zeros if partial else torch.empty
            out = {"visibility": mk((P, N, 1), **f)}
            if write_dirs:
                out.update(incident_dirs=mk((P, N, 3), **f), incident_areas=mk((P, N, 1), **f))
            if want_contribute:
                out["contribute"] = mk((P, N, 1), dtype=torch.int32, device=dev)
        m, ci, op, nr = _lib.f32(means3D), _lib.f32(symm_inv), _lib.f32(opacity), _lib.f32(normals)
        tmp = _lib.scratch(_lib.load().r3dg_bvh_trace_tmp_bytes(P), dev)
        if P > 0 and N > 0 and count > 0:
            _lib.call("r3dg_bvh_bake_visibility", dev, P, int(first_slot), int(count), N, self.tree.data_ptr(),
                      self.aabb.data_ptr(), m.data_ptr(), ci.data_ptr(), op.data_ptr(), nr.data_ptr(), 0.05,
                      _lib.ptr(out.get("contribute")), out["visibility"].data_ptr(), _lib.ptr(out.get("incident_dirs")),
                      _lib.ptr(out.get("incident_areas")), tmp.data_ptr(), tmp.numel(), what="bake_visibility")
        return out

    @torch.no_grad()
    def bake_importance(self, means3D, symm_inv, opacity, normals, sampler, sample_num, viewdirs=None, roughness=None):
        """The visibility bake along importance-sampled directions (shading.EnvSampler): shading.importance_sample's
        directions and areas for every Gaussian, then trace_visibility's T of the rays from each mean + 0.05 d
        (r3dg_bvh_trace_opacity, the bake's hit rule).  Returns dict(visibility [P,N,1], incident_dirs [P,N,3],
        incident_areas [P,N,1]) in bake_visibility's shapes, for `rendering_equation` under the sampler's light."""
        from .shading import importance_sample
        dirs, areas = importance_sample(normals, sampler, sample_num, viewdirs, roughness)
        P, N = dirs.shape[0], dirs.shape[1]
        if P == 0:
            return {"visibility": torch.empty((0, N, 1), dtype=torch.float32, device=dirs.device), "incident_dirs": dirs,
                    "incident_areas": areas}
        _, opa = _C._trace(self.tree, self.aabb, _lib.f32(means3D), N, 0.05, dirs, means3D, symm_inv, opacity, normals)
        return {"visibility": opa.unsqueeze(-1), "incident_dirs": dirs, "incident_areas": areas}

    @torch.no_grad()
    def bake_radiance(self, means3D, symm_inv, opacity, normals, shs, sh_degree, sample_num, want_hits=False):
        """What each of the bake's rays (those of `bake_visibility`) sees of the other Gaussians, composited front to
        back in ascending (t, Gaussian index) until T < 1e-4 (r3dg_bvh_bake_radiance).  The payload `shs` [P,M,3]
        is coloured like the rasterizer does from the ray origin; a view-independent radiance L [P,3] goes in as
        degree 0 with shs = ((L - 0.5) / C0)[:, None].  Returns dict(radiance [P,N,3], transmittance [P,N,1]
        [, num_hits i32[P,N]])."""
        P, N, deg = means3D.shape[0], int(sample_num), int(sh_degree)
        dev = means3D.device
        if not all(t.is_cuda for t in (means3D, symm_inv, opacity, normals, shs)):
            raise RuntimeError("bake_radiance runs on the GPU only (no CPU path)")
        sh = _lib.f32(shs)
        if sh.dim() != 3 or sh.shape[0] != P or sh.shape[2] != 3:
            raise ValueError(f"shs must be [P, M, 3] with P = {P}, got {tuple(sh.shape)}")
        out = {"radiance": torch.empty((P, N, 3), dtype=torch.float32, device=dev),
               "transmittance": torch.empty((P, N, 1), dtype=torch.float32, device=dev)}
        if want_hits:
            out["num_hits"] = torch.empty((P, N), dtype=torch.int32, device=dev)
        m, ci, op, nr = _lib.f32(means3D), _lib.f32(symm_inv), _lib.f32(opacity), _lib.f32(normals)
        tmp = _lib.scratch(_lib.load().r3dg_bvh_bake_radiance_tmp_bytes(P), dev)
        _lib.call("r3dg_bvh_bake_radiance", dev, P, N, self.tree.data_ptr(), self.aabb.data_ptr(), m.data_ptr(),
                  ci.data_ptr(), op.data_ptr(), nr.data_ptr(), sh.data_ptr(), sh.shape[1], deg, 0.05,
                  out["radiance"].data_ptr(), out["transmittance"].data_ptr(), _lib.ptr(out.get("num_hits")),
                  tmp.data_ptr(), tmp.numel(), what="bake_radiance")
        return out

    @torch.no_grad()
    def trace_lights(self, means3D, symm_inv, opacity, normals, lights):
        """Shadow transmittance T [P,K] of every (Gaussian, light) pair of `lights` (lights.Lights) through this tree
        (r3dg_bvh_trace_lights): the ray from mean + 0.05 l towards the light, the bake's hit rule, hits only before
        a point light, T multiplied until it falls below 1e-4.  No gradient.  A static light is traced once and its T
        reused for every view."""
        P, K = means3D.shape[0], len(lights)
        dev = means3D.device
        if not all(t.is_cuda for t in (means3D, symm_inv, opacity, normals, lights.vec)):
            raise RuntimeError("trace_lights runs on the GPU only (no CPU path)")
        kind, vec = lights.kind, _lib.f32(lights.vec)
        out = torch.empty((P, K), dtype=torch.float32, device=dev)
        m, ci, op, nr = _lib.f32(means3D), _lib.f32(symm_inv), _lib.f32(opacity), _lib.f32(normals)
        tmp = _lib.scratch(_lib.load().r3dg_bvh_trace_lights_tmp_bytes(P), dev)
        _lib.call("r3dg_bvh_trace_lights", dev, P, K, kind.data_ptr() if K else None, _lib.ptr(vec), self.tree.data_ptr(),
                  self.aabb.data_ptr(), m.data_ptr(), ci.data_ptr(), op.data_ptr(), nr.data_ptr(), _lib.ptr(out),
                  tmp.data_ptr(), tmp.numel(), what="trace_lights")
        return out

    @torch.no_grad()
    def trace_shaped_lights(self, means3D, symm_inv, opacity, normals, lights):
        """Shadow transmittance T [P,R] of the spot and rect lights `lights` (lights.ShapedLights) through this tree
        (r3dg_bvh_trace_shaped_lights): a spot's column is trace_lights' T of a point light at its position, a rect's
        M^2 columns those of point lights at its hashed stratified samples (the points shade_shaped uses).  No
        gradient.  A static light set is traced once and its T reused for every view."""
        from .lights import _shaped_args
        P, R = means3D.shape[0], lights.num_rays()
        dev = means3D.device
        if not all(t.is_cuda for t in (means3D, symm_inv, opacity, normals, lights.pos, lights.a, lights.b)):
            raise RuntimeError("trace_shaped_lights runs on the GPU only (no CPU path)")
        if means3D.shape != (P, 3) or normals.shape != (P, 3) or symm_inv.shape != (P, 6) or opacity.numel() != P:
            raise ValueError("means3D and normals must be [P,3], symm_inv [P,6] and opacity [P]")
        out = torch.empty((P, R), dtype=torch.float32, device=dev)
        m, ci, op, nr = _lib.f32(means3D), _lib.f32(symm_inv), _lib.f32(opacity), _lib.f32(normals)
        ts = [_lib.f32(t) for t in (lights.pos, lights.a, lights.b, lights.color, lights.cone)] + [m, None, None, nr, None, None]
        args = _shaped_args(P, 1, lights, ts)
        tmp = _lib.scratch(_lib.load().r3dg_bvh_trace_shaped_lights_tmp_bytes(P), dev)
        _lib.call("r3dg_bvh_trace_shaped_lights", dev, ctypes.byref(args), self.tree.data_ptr(), self.aabb.data_ptr(),
                  ci.data_ptr(), op.data_ptr(), _lib.ptr(out), tmp.data_ptr(), tmp.numel(), what="trace_shaped_lights")
        return out

    @torch.no_grad()
    def trace_pixels(self, points, normals, sample_num, means3D, symm_inv, opacity, gaussian_normals, mask=None, sampler=None,
                     roughness=None, campos=None):
        """Visibility T [N,H,W] (or [V,N,H,W]) of the per-pixel shading (shading.shade_pixels) through this tree
        (r3dg_bvh_trace_pixels): for every valid pixel of points / normals [3,H,W] (or [V,3,H,W]; world-space surface
        points and the rasterized normals) and sample i, trace_visibility's T of the ray from the point along the
        sampler's direction i around normalize(normal), bit for bit.  Pixels outside `mask` ([H,W] or [V,H,W], bool
        or uint8) trace nothing and get 0.  No gradient.  A view is traced once and shaded under any number of envs.
        sampler: a shading.EnvSampler; the directions are then its directions of pixel p = y W + x as row p (those of
        importance_sample), and roughness [1,H,W] / [V,1,H,W] and campos [3] / [V,3] are required when its mix has GGX
        samples.  Shade the result with shading.shade_pixels(..., sampler=) and the same sampler."""
        from .shading import pixel_args
        P = means3D.shape[0]
        if not all(t.is_cuda for t in (means3D, symm_inv, opacity, gaussian_normals)):
            raise RuntimeError("trace_pixels runs on the GPU only (no CPU path)")
        if means3D.shape != (P, 3) or gaussian_normals.shape != (P, 3) or symm_inv.shape != (P, 6) or opacity.numel() != P:
            raise ValueError("means3D and gaussian_normals must be [P,3], symm_inv [P,6] and opacity [P]")
        a, lead, keep = pixel_args(normals, points, sample_num, mask)
        if sampler is not None:
            if sampler.table.device != points.device:
                raise ValueError(f"the sampler is on {sampler.table.device}, the images on {points.device}")
            if sampler.fill(a, a.N) > 0:
                if roughness is None or campos is None:
                    raise ValueError("a sampler with GGX samples needs roughness and campos")
                r = _lib.f32(roughness).reshape(a.V, 1, a.H, a.W)
                cp = _lib.f32(campos).reshape(a.V, 3)
                if r.device != points.device or cp.device != points.device:
                    raise ValueError(f"roughness and campos must be on the images' device {points.device}")
                a.roughness, a.campos = r.data_ptr(), cp.data_ptr()
                keep += [r, cp]
        out = torch.empty((a.V, a.N, a.H, a.W), dtype=torch.float32, device=points.device)
        m, ci, op, nr = _lib.f32(means3D), _lib.f32(symm_inv), _lib.f32(opacity), _lib.f32(gaussian_normals)
        tmp = _lib.scratch(_lib.load().r3dg_bvh_trace_pixels_tmp_bytes(P), points.device)
        _lib.call("r3dg_bvh_trace_pixels", points.device, ctypes.byref(a), P, self.tree.data_ptr(), self.aabb.data_ptr(),
                  m.data_ptr(), ci.data_ptr(), op.data_ptr(), nr.data_ptr(), out.data_ptr(), tmp.data_ptr(), tmp.numel(),
                  what="trace_pixels")
        return out.reshape(lead[0] + out.shape[1:])

    @torch.no_grad()
    def trace_pixel_lights(self, points, lights, means3D, symm_inv, opacity, gaussian_normals, mask=None):
        """Shadow transmittance T [R,H,W] (or [V,R,H,W]) of `lights` (lights.Lights, R = K, or lights.ShapedLights,
        R = num_rays(), trace_shaped_lights' column order) at every valid pixel of points [3,H,W] (or [V,3,H,W];
        world-space surface points) through this tree (r3dg_bvh_trace_pixel_lights): column c is trace_lights' /
        trace_shaped_lights' ray of a Gaussian whose mean is the pixel's point, a rect's samples hashed with the
        pixel's index y W + x (the points lights.shade_pixels uses).  Pixels outside `mask` ([H,W] or [V,H,W]) trace
        nothing and get 0.  No gradient.  A light placement is traced once per view."""
        from .lights import num_rays, pixel_light_args
        P = means3D.shape[0]
        if not all(t.is_cuda for t in (means3D, symm_inv, opacity, gaussian_normals)):
            raise RuntimeError("trace_pixel_lights runs on the GPU only (no CPU path)")
        if means3D.shape != (P, 3) or gaussian_normals.shape != (P, 3) or symm_inv.shape != (P, 6) or opacity.numel() != P:
            raise ValueError("means3D and gaussian_normals must be [P,3], symm_inv [P,6] and opacity [P]")
        a, lead, keep = pixel_light_args(lights, points, mask)
        out = torch.empty((a.V, num_rays(lights), a.H, a.W), dtype=torch.float32, device=points.device)
        m, ci, op, nr = _lib.f32(means3D), _lib.f32(symm_inv), _lib.f32(opacity), _lib.f32(gaussian_normals)
        tmp = _lib.scratch(_lib.load().r3dg_bvh_trace_pixel_lights_tmp_bytes(P), points.device)
        _lib.call("r3dg_bvh_trace_pixel_lights", points.device, ctypes.byref(a), P, self.tree.data_ptr(), self.aabb.data_ptr(),
                  m.data_ptr(), ci.data_ptr(), op.data_ptr(), nr.data_ptr(), out.data_ptr(), tmp.data_ptr(), tmp.numel(),
                  what="trace_pixel_lights")
        return out.reshape(lead[0] + out.shape[1:])


@torch.no_grad()
def fit_incident_sh(radiance, normals, degree=3, ridge=1e-3):
    """Per Gaussian, the SH c [(degree+1)^2, 3] minimising (1/N) sum_i |Y(w_i)^T c - L_i|^2 + ridge |c|^2 over the
    bake's N directions w_i around its normal (r3dg_fit_incident_sh): the local incident light of the shading step,
    in the layout of `get_incidents()` (dc first).  radiance [P,N,3] -> [P,(degree+1)^2,3]."""
    L, n = _lib.f32(radiance), _lib.f32(normals).reshape(-1, 3)
    if not (L.is_cuda and n.is_cuda):
        raise RuntimeError("fit_incident_sh runs on the GPU only (no CPU path)")
    if L.dim() != 3 or L.shape[2] != 3 or L.shape[0] != n.shape[0]:
        raise ValueError(f"radiance must be [P, N, 3] matching normals [P, 3], got {tuple(L.shape)}")
    P, N, deg = L.shape[0], L.shape[1], int(degree)
    out = torch.empty((P, max(deg + 1, 0) ** 2, 3), dtype=torch.float32, device=L.device)
    _lib.call("r3dg_fit_incident_sh", L.device, P, N, L.data_ptr(), n.data_ptr(), deg, float(ridge), out.data_ptr(),
              what="fit_incident_sh")
    return out


@torch.no_grad()
def update_incidents(xyz, scaling, rotation, inverse_covariance, opacity, normal, shs, sh_degree, sample_num,
                     incident_degree=3, ridge=1e-3):
    """The analogue of `update_visibility` for the local half of the incident light: bake what each Gaussian's N
    incident rays see of the others (payload `shs` of degree `sh_degree`, see RayTracer.bake_radiance) and fit it
    into incident SH of degree `incident_degree`.  Returns incidents [P,(incident_degree+1)^2,3], to be written into
    `_incidents_dc` (coefficient 0) and `_incidents_rest` (the others)."""
    if xyz.shape[0] == 0:                   # no tree to build; the fit of nothing is empty
        return fit_incident_sh(torch.zeros((0, int(sample_num), 3), device=xyz.device), normal, incident_degree, ridge)
    raytracer = RayTracer(xyz, scaling, rotation)
    out = raytracer.bake_radiance(xyz, inverse_covariance, opacity, normal, shs, sh_degree, sample_num)
    return fit_incident_sh(out["radiance"], normal, incident_degree, ridge)


@torch.no_grad()
def update_visibility(xyz, scaling, rotation, inverse_covariance, opacity, normal, sample_num, shard_group=None):
    """scene/gaussian_model.py:312-342 as a free function of the activated Gaussian tensors.
    Returns (visibility [P,N,1], incident_dirs [P,N,3], incident_areas [P,N,1]).

    `shard_group` (a torch.distributed process group, or True for the default group) shards the one-off
    bake over the ranks (SURVEY.md §8e): the model is replicated, so every rank builds the same LBVH,
    traces only its contiguous range of ceil(P / world) leaf slots into a zero-initialised full-size
    visibility tensor, and ONE sum all-reduce restores the complete tensor on every rank (each row is
    written by exactly one rank); directions / areas are deterministic and cheap, so every rank
    generates all of them locally (r3dg_sample_incident_dirs) instead of exchanging 16 B per ray.
    The reference is single-GPU; without `shard_group` this is its loop as one launch."""
    import torch.distributed as tdist
    P = xyz.shape[0]
    world, rank, group = 1, 0, None
    if shard_group is not None and shard_group is not False and tdist.is_available() and tdist.is_initialized():
        group = None if shard_group is True else shard_group
        world, rank = tdist.get_world_size(group), tdist.get_rank(group)
    raytracer = RayTracer(xyz, scaling, rotation)
    per_rank = -(-P // world)
    lo, hi = min(rank * per_rank, P), min((rank + 1) * per_rank, P)
    if world == 1:
        out = raytracer.bake_visibility(xyz, inverse_covariance, opacity, normal, sample_num)
        return out["visibility"], out["incident_dirs"], out["incident_areas"]
    out = raytracer.bake_visibility(xyz, inverse_covariance, opacity, normal, sample_num, first_slot=lo, count=hi - lo, write_dirs=False)
    tdist.all_reduce(out["visibility"], op=tdist.ReduceOp.SUM, group=group)
    dirs, areas = sample_incident_rays(normal, False, sample_num)
    return out["visibility"], dirs, areas

"""TEST INFRASTRUCTURE — not product code.

ctypes driver for oracle/_ref/libref_raster.so: the UNMODIFIED reference rasterizer kernels
(/root/reference/r3dg-rasterization/cuda_rasterizer/*.cu) compiled for sm_90 by
oracle/build_ref.sh behind the raw-pointer shim oracle/ref_shim_raster.cu.  It is the parity
oracle on the GPU box (bit-exact checks of radii / point_list / ranges / n_contrib, tolerance
checks of images and gradients) and the timed `--impl reference` arm of bench.py.

Only tests/, __graft_entry__.smoke() and bench.py may import this module.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libref_raster.so")
_lib = None


def available():
    return os.path.exists(LIB_PATH) and torch.cuda.is_available()


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.ref_ctx_create.restype = ctypes.c_void_p
        _lib.ref_copy_out.restype = ctypes.c_longlong
    return _lib


def _p(t):
    return None if t is None or t.numel() == 0 else ctypes.c_void_p(t.data_ptr())


_IDS = {"depths": (0, torch.float32, 1), "clamped": (1, torch.uint8, 3), "radii": (2, torch.int32, 1),
        "means2D": (3, torch.float32, 2), "cov3D": (4, torch.float32, 6),
        "conic_opacity": (5, torch.float32, 4), "rgb": (6, torch.float32, 3),
        "tiles_touched": (7, torch.int32, 1), "point_offsets": (8, torch.int32, 1)}


class RefRasterizer:
    """One reference rasterizer context (three growable device buffers, like the torch glue of
    rasterize_points.cu:28-34,83-90)."""

    def __init__(self):
        self.ctx = ctypes.c_void_p(lib().ref_ctx_create())

    def __del__(self):
        try:
            lib().ref_ctx_destroy(self.ctx)
        except Exception:
            pass

    def forward(self, *, means3D, opacities, viewmatrix, projmatrix, campos, bg, W, H, tan_fovx,
                tan_fovy, cx, cy, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, features=None, sh_degree=3, scale_modifier=1.0,
                prefiltered=False, computer_pseudo_normal=True, debug=False):
        dev = means3D.device
        P = means3D.shape[0]
        S = 0 if features is None else features.shape[1]
        M = 0 if shs is None else shs.shape[1]
        z = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)   # rasterize_points.cu:74-81
        out = dict(color=z(3, H, W), opacity=z(1, H, W), depth=z(1, H, W), feature=z(S, H, W),
                   normal=z(3, H, W), surface_xyz=z(3, H, W), weights=z(P, 1),
                   radii=torch.zeros(P, dtype=torch.int32, device=dev))
        # no synchronize: the reference launches on the legacy default stream, which is torch's default stream
        R = lib().ref_raster_forward(
            self.ctx, P, S, int(sh_degree), M, _p(bg), W, H, _p(means3D), _p(shs), _p(colors_precomp),
            _p(features), _p(opacities), _p(scales), ctypes.c_float(scale_modifier), _p(rotations),
            _p(cov3D_precomp), _p(viewmatrix), _p(projmatrix), _p(campos), ctypes.c_float(tan_fovx),
            ctypes.c_float(tan_fovy), ctypes.c_float(cx), ctypes.c_float(cy), int(prefiltered),
            int(computer_pseudo_normal), _p(out["color"]), _p(out["opacity"]), _p(out["depth"]),
            _p(out["feature"]), _p(out["normal"]), _p(out["surface_xyz"]), _p(out["weights"]),
            _p(out["radii"]), int(debug))
        if R < 0:
            raise RuntimeError("reference forward failed")
        self.P, self.S, self.M, self.W, self.H, self.R = P, S, M, W, H, R
        out["num_rendered"] = R
        return out

    def intermediate(self, name):
        P, R, HW = self.P, self.R, self.W * self.H
        T = ((self.W + 15) // 16) * ((self.H + 15) // 16)
        dev = torch.device("cuda")
        if name in _IDS:
            i, dt, k = _IDS[name]
            t = torch.empty((P, k) if k > 1 else (P,), dtype=dt, device=dev)
        elif name == "point_list":
            i, t = 9, torch.empty(R, dtype=torch.int32, device=dev)
        elif name == "point_list_keys":
            i, t = 10, torch.empty(R, dtype=torch.int64, device=dev)
        elif name == "point_list_unsorted":
            i, t = 11, torch.empty(R, dtype=torch.int32, device=dev)
        elif name == "point_list_keys_unsorted":
            i, t = 12, torch.empty(R, dtype=torch.int64, device=dev)
        elif name == "final_T":
            i, t = 13, torch.empty(HW, dtype=torch.float32, device=dev)
        elif name == "n_contrib":
            i, t = 14, torch.empty(HW, dtype=torch.int32, device=dev)
        elif name == "ranges":
            i, t = 15, torch.empty((T, 2), dtype=torch.int32, device=dev)
        else:
            raise KeyError(name)
        if t.numel():
            torch.cuda.synchronize()
            n = lib().ref_copy_out(self.ctx, i, _p(t), ctypes.c_longlong(t.numel() * t.element_size()))
            if n < 0:
                raise RuntimeError(f"ref_copy_out({name}) failed: {n}")
            torch.cuda.synchronize()
        return t

    def backward(self, fwd_out, *, means3D, viewmatrix, projmatrix, campos, bg, tan_fovx, tan_fovy,
                 dL_dcolor, dL_dopacity, dL_ddepth, dL_dfeature, shs=None, colors_precomp=None,
                 scales=None, rotations=None, cov3D_precomp=None, features=None, sh_degree=3,
                 scale_modifier=1.0, backward_geometry=True, debug=False):
        dev = means3D.device
        P, S, M, W, H = self.P, self.S, self.M, self.W, self.H
        z = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)   # rasterize_points.cu:183-192
        g = dict(dL_dmeans3D=z(P, 3), dL_dmeans2D=z(P, 3), dL_dfeatures=z(P, S), dL_dcolors=z(P, 3),
                 dL_dconic=z(P, 2, 2), dL_dopacity=z(P, 1), dL_dcov3D=z(P, 6), dL_dsh=z(P, M, 3),
                 dL_dscales=z(P, 3), dL_drotations=z(P, 4))
        rc = lib().ref_raster_backward(
            self.ctx, P, S, int(sh_degree), M, self.R, _p(bg), W, H, _p(means3D), _p(shs),
            _p(features), _p(colors_precomp), _p(scales), ctypes.c_float(scale_modifier),
            _p(rotations), _p(cov3D_precomp), _p(viewmatrix), _p(projmatrix), _p(campos),
            ctypes.c_float(tan_fovx), ctypes.c_float(tan_fovy), _p(fwd_out["radii"]),
            _p(dL_dcolor.contiguous()), _p(dL_dopacity.contiguous()), _p(dL_ddepth.contiguous()),
            _p(dL_dfeature.contiguous()), _p(g["dL_dmeans2D"]), _p(g["dL_dconic"]),
            _p(g["dL_dopacity"]), _p(g["dL_dcolors"]), _p(g["dL_dfeatures"]), _p(g["dL_dmeans3D"]),
            _p(g["dL_dcov3D"]), _p(g["dL_dsh"]), _p(g["dL_dscales"]), _p(g["dL_drotations"]),
            int(backward_geometry), int(debug))
        if rc != 0:
            raise RuntimeError("reference backward failed")
        return g


# ----------------------------------------------------------------------------------------------
# reference BVH (oracle/_ref/libref_bvh.so)
# ----------------------------------------------------------------------------------------------
BVH_LIB_PATH = os.path.join(_HERE, "_ref", "libref_bvh.so")
_bvh = None


def bvh_available():
    return os.path.exists(BVH_LIB_PATH) and torch.cuda.is_available()


def bvh_lib():
    global _bvh
    if _bvh is None:
        _bvh = ctypes.CDLL(BVH_LIB_PATH)
    return _bvh


def ref_leaf_init(means3D, scales, rotations):
    """bvh/__init__.py:29-57 in PyTorch (build_rotation: utils/general_utils.py:82-103), verbatim op order."""
    P = means3D.shape[0]
    r = rotations
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    rot = torch.zeros((q.size(0), 3, 3), device=r.device)
    rr, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    rot[:, 0, 0] = 1 - 2 * (y * y + z * z); rot[:, 0, 1] = 2 * (x * y - rr * z); rot[:, 0, 2] = 2 * (x * z + rr * y)
    rot[:, 1, 0] = 2 * (x * y + rr * z); rot[:, 1, 1] = 1 - 2 * (x * x + z * z); rot[:, 1, 2] = 2 * (y * z - rr * x)
    rot[:, 2, 0] = 2 * (x * z - rr * y); rot[:, 2, 1] = 2 * (y * z + rr * x); rot[:, 2, 2] = 1 - 2 * (x * x + y * y)
    nodes = torch.full((2 * P - 1, 5), -1, device=r.device).int()
    nodes[:P - 1, 4] = 0
    nodes[P - 1:, 4] = 1
    aabbs = torch.zeros(2 * P - 1, 6, device=r.device).float()
    aabbs[:, :3] = 100000
    aabbs[:, 3:] = -100000
    a, b, c = rot[:, :, 0], rot[:, :, 1], rot[:, :, 2]
    m = 3
    sa, sb, sc = m * scales[:, 0], m * scales[:, 1], m * scales[:, 2]
    xs = [means3D + s0 * a * sa[:, None] + s1 * b * sb[:, None] + s2 * c * sc[:, None]
          for s0 in (1, -1) for s1 in (1, -1) for s2 in (1, -1)]
    # (means +- a*sa) +- b*sb +- c*sc : multiplying by +-1 is exact, so this is the reference's rounding
    aabb_min = xs[0]
    aabb_max = xs[0]
    for t in xs[1:]:
        aabb_min = torch.minimum(aabb_min, t)
        aabb_max = torch.maximum(aabb_max, t)
    aabbs[P - 1:] = torch.cat([aabb_min, aabb_max], dim=-1)
    return nodes.contiguous(), aabbs.contiguous()


def ref_bvh_create(means3D, scales, rotations):
    nodes, aabbs = ref_leaf_init(means3D, scales, rotations)
    P = means3D.shape[0]
    morton = torch.zeros(P, dtype=torch.int64, device=means3D.device)
    torch.cuda.synchronize()
    rc = bvh_lib().ref_bvh_create(P, _p(means3D.contiguous()), _p(scales.contiguous()), _p(rotations.contiguous()),
                                  _p(nodes), _p(aabbs), _p(morton))
    if rc != 0:
        raise RuntimeError("reference create_bvh failed")
    return nodes, aabbs, morton


def ref_bvh_trace_opacity(nodes, aabbs, rays_o, rays_d, means3D, covs3D, opacities, normals):
    shape = rays_d.shape[:-1]
    n = rays_d.numel() // 3
    contrib = torch.zeros(shape, dtype=torch.int32, device=rays_d.device)
    opa = torch.ones(shape, dtype=torch.float32, device=rays_d.device)
    ts = [t.contiguous() for t in (rays_o, rays_d, means3D, covs3D, opacities, normals)]
    torch.cuda.synchronize()
    rc = bvh_lib().ref_bvh_trace_opacity(n, _p(nodes), _p(aabbs), *[_p(t) for t in ts], _p(contrib), _p(opa))
    if rc != 0:
        raise RuntimeError("reference trace_bvh_opacity failed")
    return contrib, opa


# ----------------------------------------------------------------------------------------------
# The STOCK code path: the reference's own Python wrappers (git-ignored copies under oracle/_ref/py,
# made by oracle/build_ref_ext.sh) over either the reference's own pybind modules (oracle/_ref/ext)
# or this repo's drop-in packages (dropin/) — the latter is how tests/test_dropin_gpu.py proves that
# the reference's files run unmodified on this project's kernels.
# ----------------------------------------------------------------------------------------------
import importlib.util
import sys

_REF_PY = os.path.join(_HERE, "_ref", "py")
_REF_EXT = os.path.join(_HERE, "_ref", "ext")
_DROPIN = os.path.join(os.path.dirname(_HERE), "dropin")
_WRAPPERS = {"raster": ("gaussian_renderer/r3dg_rasterization.py", "r3dg_rasterization"),
             "bvh": ("bvh/__init__.py", "bvh_tracing")}
_loaded = {}


def ext_available(which="raster"):
    name = _WRAPPERS[which][1]
    return (os.path.exists(os.path.join(_REF_EXT, name, "_C.so")) and
            os.path.exists(os.path.join(_REF_PY, _WRAPPERS[which][0])) and torch.cuda.is_available())


def wrappers_available(which="raster"):
    return os.path.exists(os.path.join(_REF_PY, _WRAPPERS[which][0]))


def load_reference_wrapper(which, backend):
    """Import the reference's wrapper file `which` ("raster" | "bvh") BY PATH with its extension package
    (`r3dg_rasterization` / `bvh_tracing`) resolving to backend "ref" (the reference's own build) or "dropin"
    (this repo).  Returns the module; both backends can be loaded side by side."""
    key = (which, backend)
    if key in _loaded:
        return _loaded[key]
    rel, pkg = _WRAPPERS[which]
    root = _REF_EXT if backend == "ref" else _DROPIN
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == pkg or k.startswith(pkg + ".") or k == "utils" or k.startswith("utils.")}
    sys.path[:0] = [root, _REF_PY]
    try:
        spec = importlib.util.spec_from_file_location(f"_refwrap_{which}_{backend}", os.path.join(_REF_PY, rel))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        origin = os.path.realpath(getattr(mod._C, "__file__", ""))
        allowed = [os.path.realpath(_REF_EXT)] if backend == "ref" else [os.path.realpath(_DROPIN), os.path.realpath(
            os.path.join(os.path.dirname(_HERE), "relightable3dgaussian_b200"))]
        if not any(origin.startswith(a) for a in allowed):
            raise ImportError(f"{pkg}._C resolved to {origin}, not under {allowed}")
        mod._C_origin = origin
    finally:
        del sys.path[:2]
        for k in [k for k in sys.modules if k == pkg or k.startswith(pkg + ".") or k == "utils" or k.startswith("utils.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    _loaded[key] = mod
    return mod


class _ShimRasterize(torch.autograd.Function):
    """Fallback when the reference's own pybind module is not built: its unmodified kernels + rasterizer_impl.cu
    orchestration behind the raw-pointer shim, with the zero-fills of rasterize_points.cu reproduced."""

    @staticmethod
    def forward(ctx, ref, means3D, opacities, shs, scales, rotations, features, cam, cd, bg, W, H):
        kw = dict(means3D=means3D.detach().contiguous(), shs=shs.detach().contiguous(), scales=scales.detach().contiguous(),
                  rotations=rotations.detach().contiguous(), features=features.detach().contiguous())
        o = ref.forward(bg=bg, W=W, H=H, tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy, viewmatrix=cd["view"],
                        projmatrix=cd["proj"], campos=cd["pos"], opacities=opacities.detach().contiguous(), **kw)
        ctx.ref, ctx.o, ctx.kw, ctx.cam, ctx.cd, ctx.bg = ref, o, kw, cam, cd, bg
        n_contrib = ref.intermediate("n_contrib").view(H, W)
        ctx.mark_non_differentiable(n_contrib)
        return o["color"], o["opacity"], o["depth"], o["feature"], n_contrib

    @staticmethod
    def backward(ctx, g_color, g_opacity, g_depth, g_feature, _):
        z = lambda g, like: torch.zeros_like(like) if g is None else g
        o = ctx.o
        g = ctx.ref.backward(o, bg=ctx.bg, tan_fovx=ctx.cam.tanfovx, tan_fovy=ctx.cam.tanfovy, viewmatrix=ctx.cd["view"],
                             projmatrix=ctx.cd["proj"], campos=ctx.cd["pos"], dL_dcolor=z(g_color, o["color"]),
                             dL_dopacity=z(g_opacity, o["opacity"]), dL_ddepth=z(g_depth, o["depth"]),
                             dL_dfeature=z(g_feature, o["feature"]), **ctx.kw)
        return (None, g["dL_dmeans3D"], g["dL_dopacity"], g["dL_dsh"], g["dL_dscales"], g["dL_drotations"], g["dL_dfeatures"],
                None, None, None, None, None)


def reference_rasterizer():
    """-> (raster(cam, cd, bg, xyz, opacity, shs, scales, rotations, features) -> dict, description).  Differentiable
    through torch autograd.  Prefers the stock code path (reference wrapper + reference pybind module)."""
    if ext_available("raster"):
        mod = load_reference_wrapper("raster", "ref")

        def raster(cam, cd, bg, xyz, opacity, shs, scales, rotations, features):
            rs = mod.GaussianRasterizationSettings(
                image_height=cam.image_height, image_width=cam.image_width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, cx=cam.cx, cy=cam.cy,
                bg=bg, scale_modifier=1.0, viewmatrix=cd["view"], projmatrix=cd["proj"], sh_degree=3, campos=cd["pos"], prefiltered=False,
                backward_geometry=True, computer_pseudo_normal=True, debug=False)
            means2D = torch.zeros_like(xyz, requires_grad=True)
            (num_rendered, num_contrib, color, opac, depth, feature, normal, surface_xyz, weights, radii) = mod.GaussianRasterizer(rs)(
                means3D=xyz, means2D=means2D, shs=shs, colors_precomp=None, opacities=opacity, scales=scales, rotations=rotations,
                cov3D_precomp=None, features=features)
            return dict(num_rendered=num_rendered, num_contrib=num_contrib, color=color, opacity=opac, depth=depth, feature=feature,
                        radii=radii, means2D=means2D)
        return raster, ("the reference's own rasterizer, stock code path: gaussian_renderer/r3dg_rasterization.py -> r3dg_rasterization._C "
                        "(rasterize_points.cu + cuda_rasterizer/*.cu built for sm_90 by oracle/build_ref_ext.sh)")
    ref = RefRasterizer()

    def raster(cam, cd, bg, xyz, opacity, shs, scales, rotations, features):
        color, opac, depth, feature, n_contrib = _ShimRasterize.apply(ref, xyz, opacity, shs, scales, rotations, features, cam, cd, bg,
                                                                      cam.image_width, cam.image_height)
        return dict(num_rendered=ref.R, num_contrib=n_contrib, color=color, opacity=opac, depth=depth, feature=feature, radii=None)
    return raster, "the reference's unmodified kernels + rasterizer_impl.cu behind the raw-pointer shim (its pybind module is not built)"


@torch.no_grad()
def reference_update_visibility(xyz, scaling, rotation, icov, opacity, normal, sample_num):
    """scene/gaussian_model.py:312-342 driven exactly like the reference drives it (chunk loop, PyTorch direction
    sampling, RayTracer.trace_visibility) on the reference's own BVH kernels."""
    from . import oracle_sampling
    P = xyz.shape[0]
    chunk_size = max(1, P // ((sample_num - 1) // 24 + 1))
    vis, dirs, areas = [], [], []
    if ext_available("bvh"):
        mod = load_reference_wrapper("bvh", "ref")
        rt = mod.RayTracer(xyz, scaling, rotation)
        kind = "reference RayTracer (bvh/__init__.py) + bvh_tracing._C built for sm_90, PyTorch direction sampling, the reference's chunk loop"
        trace = lambda o, d: rt.trace_visibility(o, d, xyz, icov, opacity, normal)["visibility"]
    else:
        nodes, aabbs, _ = ref_bvh_create(xyz, scaling, rotation)
        kind = "reference BVH kernels behind the raw-pointer shim, PyTorch direction sampling, the reference's chunk loop"
        trace = lambda o, d: ref_bvh_trace_opacity(nodes, aabbs, (o + d * 0.05).contiguous(), d, xyz, icov, opacity, normal)[1].unsqueeze(-1)
    for off in range(0, P, chunk_size):
        d, a = oracle_sampling.sample_incident_rays(normal[off:off + chunk_size], False, sample_num)
        vis.append(trace(xyz[off:off + chunk_size, None].expand_as(d), d))
        dirs.append(d); areas.append(a)
    return torch.cat(vis, 0), torch.cat(dirs, 0), torch.cat(areas, 0), kind

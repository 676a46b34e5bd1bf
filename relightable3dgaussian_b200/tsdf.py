"""TSDF fusion and marching-cubes mesh extraction for sm_90a (csrc/tsdf.cu): the mesh step of 2DGS, PGSR, RaDe-GS and
GOF.  Not part of the reference surface.

  vol = TSDFVolume(bbox_min, bbox_max, voxel_size, sdf_trunc, color=True, device="cuda")
  vol.integrate(depth, settings, color=None, depth_trunc=float("inf"))   # depth [V,1,H,W], color [V,3,H,W]
  verts, faces, colors = vol.extract()    # [N,3] float32, [F,3] int32, [N,3] float32 or None
  formats.save_mesh_ply(path, verts, faces, colors)

The volume is a dense grid of points origin + voxel_size * (i, j, k) covering the box, with `tsdf` (initialised to 1),
`weight` (0) and optionally `color` [NX,NY,NZ,3] (0) as public float32 tensors.  `integrate` fuses V <= 64 rendered
views in order, Open3D's projective TSDF with unit weights: a grid point in front of a view whose nearest pixel has a
finite depth D with 0 < D <= depth_trunc and D - z >= -sdf_trunc averages min(1, (D - z) / sdf_trunc) into its tsdf
(and the pixel's colour into its colour).  Depth <= 0, NaN and Inf are skipped, so mask pixels by zeroing them.  One
launch, no host synchronisation, bitwise reproducible; V views in one call give the same bits as V one-view calls.
`extract` runs marching cubes over the cells whose 8 corners all have weight > 0 (inside: tsdf < 0) with a crack-free
table and returns a welded mesh whose normals point from inside to outside; its order is a function of the volume.  It
synchronises once, to size its outputs.  The exact definition is in include/r3dg_b200.h (r3dg_tsdf_*).  No gradients.
"""
import ctypes
import math
import numbers

import torch

from . import _lib
from .multiview import check_settings, view_matrices

MAX_VIEWS = 64          # R3DG_MAX_VIEWS (include/r3dg_b200.h)
MAX_POINTS = 2 ** 31    # grid points per volume (exclusive)


def _finite(x):
    return isinstance(x, numbers.Real) and not isinstance(x, bool) and math.isfinite(float(x))


def _vec3(fn, name, v):
    v = list(v.tolist() if isinstance(v, torch.Tensor) else v)
    if len(v) != 3 or not all(_finite(x) for x in v):
        raise ValueError(f"{fn}: {name} must be three finite numbers (got {v!r})")
    return [float(x) for x in v]


def _positive(fn, name, x):
    if not (_finite(x) and float(x) > 0.0):
        raise ValueError(f"{fn}: {name} must be a finite number > 0 (got {x!r})")
    return float(x)


class TSDFVolume:
    """A dense TSDF grid over the box [bbox_min, bbox_max]: NX x NY x NZ points with NX = ceil((max - min) / voxel_size)
    + 1 (so the last point reaches bbox_max) and the same for y and z; origin = bbox_min.  sdf_trunc is the
    truncation distance in world units (2DGS uses 4-5 voxels).  color=False keeps no colour grid."""

    def __init__(self, bbox_min, bbox_max, voxel_size, sdf_trunc, color=True, device="cuda"):
        fn = "TSDFVolume"
        lo, hi = _vec3(fn, "bbox_min", bbox_min), _vec3(fn, "bbox_max", bbox_max)
        if not all(h > l for l, h in zip(lo, hi)):
            raise ValueError(f"{fn}: bbox_max {hi} must exceed bbox_min {lo} on every axis")
        vs = _positive(fn, "voxel_size", voxel_size)
        self.sdf_trunc = _positive(fn, "sdf_trunc", sdf_trunc)
        dims = tuple(int(math.ceil((h - l) / vs - 1e-6)) + 1 for l, h in zip(lo, hi))
        if math.prod(dims) >= MAX_POINTS:
            raise ValueError(f"{fn}: {dims} is {math.prod(dims)} grid points, the limit is 2^31 - 1")
        if not isinstance(color, bool):
            raise TypeError(f"{fn}: color must be a bool (got {color!r})")
        self.origin, self.voxel_size, self.dims = lo, vs, dims
        dev = torch.device(device)
        self.tsdf = torch.ones(dims, dtype=torch.float32, device=dev)
        self.weight = torch.zeros(dims, dtype=torch.float32, device=dev)
        self.color = torch.zeros(dims + (3,), dtype=torch.float32, device=dev) if color else None

    @property
    def device(self):
        return self.tsdf.device

    def _check_volume(self, fn):
        vol = [("tsdf", self.tsdf, self.dims), ("weight", self.weight, self.dims)]
        if self.color is not None:
            vol.append(("color", self.color, self.dims + (3,)))
        for name, t, shape in vol:
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) != shape \
                    or not t.is_contiguous() or t.device != self.tsdf.device:
                raise ValueError(f"{fn}: vol.{name} must stay a contiguous float32 {list(shape)} tensor on the "
                                 "volume's device")

    def _grid(self, a):
        a.NX, a.NY, a.NZ = self.dims
        a.origin[:] = self.origin
        a.voxel_size = self.voxel_size
        a.tsdf, a.weight = self.tsdf.data_ptr(), self.weight.data_ptr()
        a.color = self.color.data_ptr() if self.color is not None else None

    def integrate(self, depth, settings, color=None, depth_trunc=float("inf")):
        """Fuse V rendered views: depth [V,1,H,W] float32 (camera z; pixels <= 0, NaN or Inf are skipped), the V
        GaussianRasterizationSettings they were rendered with (viewmatrix, tanfovx, tanfovy, cx, cy and the image size
        are read; one settings object stands for V = 1), and color [V,3,H,W] float32, required exactly when the volume
        keeps colour.  Depths beyond depth_trunc are skipped.  1 <= V <= 64 per call; call again for more views."""
        fn = "TSDFVolume.integrate"
        if not isinstance(depth, torch.Tensor):
            raise TypeError(f"{fn}: depth must be a tensor")
        if depth.dtype != torch.float32:
            raise TypeError(f"{fn}: depth must be float32 (got {depth.dtype})")
        if depth.dim() != 4 or depth.shape[1] != 1:
            raise ValueError(f"{fn}: depth must be [V,1,H,W] (got {tuple(depth.shape)})")
        V, _, H, W = depth.shape
        if not 1 <= V <= MAX_VIEWS:
            raise ValueError(f"{fn}: 1..{MAX_VIEWS} views per call (got {V})")
        if H == 0 or W == 0:
            raise ValueError(f"{fn}: empty maps {tuple(depth.shape)}")
        if H * W >= MAX_POINTS:
            raise ValueError(f"{fn}: {H}x{W} maps have 2^31 pixels or more")
        if (color is None) != (self.color is None):
            raise ValueError(f"{fn}: color is required exactly when the volume keeps colour "
                             f"(volume color={self.color is not None}, color given={color is not None})")
        if color is not None:
            if not isinstance(color, torch.Tensor):
                raise TypeError(f"{fn}: color must be a tensor")
            if color.dtype != torch.float32:
                raise TypeError(f"{fn}: color must be float32 (got {color.dtype})")
            if tuple(color.shape) != (V, 3, H, W):
                raise ValueError(f"{fn}: color must be [V,3,H,W] = {[V, 3, H, W]} (got {tuple(color.shape)})")
        if hasattr(settings, "viewmatrix"):
            settings = [settings]
        settings = check_settings(fn, settings, V, H, W)
        for v, s in enumerate(settings):
            if not all(_finite(x) for x in (s.tanfovx, s.tanfovy, s.cx, s.cy)):
                raise ValueError(f"{fn}: settings[{v}] has a non-finite tanfovx, tanfovy, cx or cy")
        if not (isinstance(depth_trunc, numbers.Real) and float(depth_trunc) > 0.0):
            raise ValueError(f"{fn}: depth_trunc must be > 0 (got {depth_trunc!r})")
        self._check_volume(fn)
        for name, t in (("volume", self.tsdf), ("depth", depth), ("color", color)):
            if t is not None and not t.is_cuda:
                raise ValueError(f"{fn}: {name} must be on a CUDA device (got {t.device})")
            if t is not None and t.device != self.tsdf.device:
                raise ValueError(f"{fn}: {name} is on {t.device}, the volume on {self.tsdf.device}")
        cams = (ctypes.c_float * (4 * V))()
        for v, s in enumerate(settings):
            cams[4 * v: 4 * v + 4] = [s.tanfovx, s.tanfovy, s.cx, s.cy]
        d = depth.detach().contiguous()
        rgb = color.detach().contiguous() if color is not None else None
        view = view_matrices(settings, self.tsdf.device)
        a = _lib.TsdfIntegrateArgs()
        self._grid(a)
        a.sdf_trunc, a.depth_trunc = self.sdf_trunc, float(depth_trunc)
        a.V, a.H, a.W = V, H, W
        a.depth, a.rgb, a.viewmatrix, a.cams = d.data_ptr(), _lib.ptr(rgb), view.data_ptr(), ctypes.addressof(cams)
        _lib.call("r3dg_tsdf_integrate", self.tsdf.device, ctypes.byref(a), what="TSDFVolume.integrate")

    def extract(self):
        """Marching cubes over the observed cells: (verts [N,3] float32, faces [F,3] int32, colors [N,3] float32 or
        None), on the volume's device.  Reads the two totals back to the host once."""
        fn = "TSDFVolume.extract"
        self._check_volume(fn)
        if not self.tsdf.is_cuda:
            raise ValueError(f"{fn}: the volume must be on a CUDA device (got {self.tsdf.device})")
        dev = self.tsdf.device
        work = _lib.scratch(_lib.load().r3dg_tsdf_extract_work_bytes(*self.dims), dev)
        totals = (ctypes.c_longlong * 2)()
        a = _lib.TsdfExtractArgs()
        self._grid(a)
        a.work, a.work_bytes, a.totals_host = work.data_ptr(), work.numel(), ctypes.addressof(totals)
        _lib.call("r3dg_tsdf_extract_count", dev, ctypes.byref(a), what=fn)
        nv, nf = totals[0], totals[1]
        verts = torch.empty((nv, 3), dtype=torch.float32, device=dev)
        faces = torch.empty((nf, 3), dtype=torch.int32, device=dev)
        colors = torch.empty((nv, 3), dtype=torch.float32, device=dev) if self.color is not None else None
        a.n_verts, a.n_faces = nv, nf
        a.verts, a.faces, a.vert_colors = _lib.ptr(verts), _lib.ptr(faces), _lib.ptr(colors)
        _lib.call("r3dg_tsdf_extract_emit", dev, ctypes.byref(a), what=fn)
        return verts, faces, colors

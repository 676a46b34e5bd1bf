"""Seeded synthetic scenes and cameras (BASELINE.md §2.2) shared by tests and bench.py.

Everything is generated on the CPU with a seeded torch.Generator so that the GPU box and this
container see bit-identical inputs.  Camera matrices follow the reference's conventions
(scene/cameras.py:62-77, utils/graphics_utils.py:148-189): `viewmatrix` is the world->view
matrix stored transposed (row-vector convention), `projmatrix` = viewmatrix @ projection^T.
"""
import math
from typing import NamedTuple, Optional

import torch

SH_C0 = 0.28209479177387814


class Scene(NamedTuple):
    means3D: torch.Tensor      # [P,3]
    scales: torch.Tensor       # [P,3]   (activated, positive)
    rotations: torch.Tensor    # [P,4]   (normalised quaternion, r,x,y,z)
    opacities: torch.Tensor    # [P,1]   (activated, (0,1))
    shs: torch.Tensor          # [P,16,3]
    normals: torch.Tensor      # [P,3]
    features: Optional[torch.Tensor]  # [P,S]


class Camera(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    cx: float
    cy: float
    viewmatrix: torch.Tensor   # [4,4]
    projmatrix: torch.Tensor   # [4,4]
    campos: torch.Tensor       # [3]


def make_scene(P: int, recipe: str = "shell-v1", seed: int = 0, S: int = 5) -> Scene:
    g = torch.Generator().manual_seed(seed)
    if recipe == "shell-v1":
        n = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
        xyz = n * (1.0 + 0.02 * torch.randn(P, 1, generator=g))
    elif recipe == "cube-v1":   # scene/dataset_readers.py:294 random init
        xyz = torch.rand(P, 3, generator=g) * 2.6 - 1.3
        n = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    else:
        raise ValueError(recipe)
    lo, hi = math.log(0.003), math.log(0.03)
    scales = torch.exp(torch.rand(P, 3, generator=g) * (hi - lo) + lo)
    rot = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1)
    opac = torch.sigmoid(torch.randn(P, 1, generator=g) * 2.0)
    shs = torch.randn(P, 16, 3, generator=g) * 0.1
    shs[:, 0] = torch.randn(P, 3, generator=g) * 0.5 / SH_C0
    feats = None
    if S > 0:
        feats = torch.randn(P, S, generator=g) * 0.5
        feats[:, : min(3, S)] = n[:, : min(3, S)]
    return Scene(xyz.float().contiguous(), scales.float().contiguous(), rot.float().contiguous(),
                 opac.float().contiguous(), shs.float().contiguous(), n.float().contiguous(),
                 None if feats is None else feats.float().contiguous())


def _projection(znear, zfar, left, right, top, bottom):
    Pm = torch.zeros(4, 4)
    Pm[0, 0] = 2.0 * znear / (right - left)
    Pm[1, 1] = 2.0 * znear / (top - bottom)
    Pm[0, 2] = (right + left) / (right - left)
    Pm[1, 2] = (top + bottom) / (top - bottom)
    Pm[3, 2] = 1.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    return Pm


def make_camera(k: int, W: int, H: int, radius: float = 4.0311, elevation_deg: float = 30.0,
                fovx: float = 0.6911112070083618, center_shift: bool = False) -> Camera:
    """View k of the 8-view ring (azimuth k*45 deg), looking at the origin."""
    az = math.radians(45.0 * k)
    el = math.radians(elevation_deg)
    C = torch.tensor([radius * math.cos(el) * math.cos(az), radius * math.cos(el) * math.sin(az),
                      radius * math.sin(el)], dtype=torch.float64)
    fwd = -C / C.norm()
    up = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
    right = torch.linalg.cross(fwd, up)
    right = right / right.norm()
    down = torch.linalg.cross(fwd, right)
    Rc = torch.stack([right, down, fwd], dim=1)          # camera-to-world rotation (columns)
    W2C = torch.eye(4, dtype=torch.float64)
    W2C[:3, :3] = Rc.t()
    W2C[:3, 3] = -Rc.t() @ C
    view = W2C.float().t().contiguous()                  # stored transposed (cameras.py:62)
    znear, zfar = 0.01, 100.0
    fovy = 2.0 * math.atan(math.tan(fovx / 2.0) * H / W)
    if center_shift:
        fx = W / (2.0 * math.tan(fovx / 2.0))
        fy = H / (2.0 * math.tan(fovy / 2.0))
        cx, cy = W / 2.0 + 7.3, H / 2.0 - 4.1
        proj = _projection(znear, zfar, -(W - cx) / fx * znear, cx / fx * znear, cy / fy * znear,
                           -(H - cy) / fy * znear)
    else:
        t, r = math.tan(fovy / 2.0) * znear, math.tan(fovx / 2.0) * znear
        proj = _projection(znear, zfar, -r, r, t, -t)
        cx, cy = W / 2.0, H / 2.0
    full = (view.unsqueeze(0).bmm(proj.t().unsqueeze(0))).squeeze(0).contiguous()
    campos = view.inverse()[3, :3].contiguous()
    return Camera(H, W, math.tan(fovx / 2.0), math.tan(fovy / 2.0), float(cx), float(cy), view, full,
                  campos)


def make_axis_camera(W: int, H: int, fovx: float = 0.6911112070083618) -> Camera:
    """Camera at the origin looking down +z: identity view rotation, zero translation.  The view-space
    depth of a point is then its z coordinate, bit for bit, so a scene can place depths exactly (sort
    keys, the z = 0.2 cull plane)."""
    view = torch.eye(4)
    znear, zfar = 0.01, 100.0
    fovy = 2.0 * math.atan(math.tan(fovx / 2.0) * H / W)
    t, r = math.tan(fovy / 2.0) * znear, math.tan(fovx / 2.0) * znear
    full = _projection(znear, zfar, -r, r, t, -t).t().contiguous()
    return Camera(H, W, math.tan(fovx / 2.0), math.tan(fovy / 2.0), W / 2.0, H / 2.0, view, full,
                  torch.zeros(3))

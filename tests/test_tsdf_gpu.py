"""TSDF fusion and marching cubes on the GPU against the fp64 oracle (tests/tsdf_oracle.py): integration of analytic
sphere views with colour, its invariances (call splitting, reruns, skipped pixels, grid points outside every
frustum), extraction on the device-made volume and on a random field with unobserved holes, empty volumes, and the
chain from rasterize_views to a mesh."""
import math

import numpy as np
import pytest
import torch

import tsdf_oracle as O
from relightable3dgaussian_b200 import synth, tsdf
from relightable3dgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
VS = 2.4 / 95
ORIGIN = (-1.2, -1.2, -1.2)
SPHERE = [((0.0, 0.0, 0.0), 0.8)]
TWO = [((-0.55, 0.0, 0.0), 0.4), ((0.55, 0.0, 0.0), 0.4)]


def _views(spheres, W=256, H=256, seed=0):
    cams = O.ring_cameras(W, H)
    dep = np.stack([O.sphere_depth(c, spheres) for c in cams]).astype(np.float32)
    rgb = torch.rand(len(cams), 3, H, W, generator=torch.Generator().manual_seed(seed)).numpy()
    return cams, dep, rgb


def _volume(color=True):
    vol = tsdf.TSDFVolume((-1.2,) * 3, (1.2,) * 3, VS, 4 * VS, color=color, device=DEV)
    assert vol.dims == (96, 96, 96)
    return vol


def _integrate(vol, cams, dep, rgb, per_call=16, depth_trunc=math.inf):
    for s in range(0, len(cams), per_call):
        d = torch.from_numpy(dep[s:s + per_call]).unsqueeze(1).to(DEV)
        c = None if rgb is None else torch.from_numpy(rgb[s:s + per_call]).to(DEV)
        vol.integrate(d, cams[s:s + per_call], c, depth_trunc=depth_trunc)
    torch.cuda.synchronize()
    return vol


def _state(vol):
    return [t.cpu().clone() for t in (vol.tsdf, vol.weight, vol.color) if t is not None]


def _bits_equal(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


@pytest.fixture(scope="module")
def sphere_case():
    cams, dep, rgb = _views(SPHERE)
    vol = _integrate(_volume(), cams, dep, rgb)
    return cams, dep, rgb, vol


def test_integrate_matches_oracle(sphere_case):
    cams, dep, rgb, vol = sphere_case
    dims = vol.dims
    t, w, c, near = O.integrate(np.ones(dims, np.float32), np.zeros(dims, np.float32), np.zeros(dims + (3,), np.float32),
                                ORIGIN, VS, 4 * VS, dep, rgb, O.cam_rows(cams))
    keep = ~near
    assert near.mean() < 0.01
    gt, gw, gc = (x.cpu().double().numpy() for x in (vol.tsdf, vol.weight, vol.color))
    assert np.array_equal(gw[keep], w[keep])
    assert np.abs(gt - t)[keep].max() < 1e-5
    assert np.abs(gc - c)[keep].max() < 1e-5
    assert (w > 0).sum() > 100000


def test_one_call_equals_one_view_calls_and_reruns(sphere_case):
    cams, dep, rgb, vol = sphere_case
    ref = _state(vol)
    assert _bits_equal(ref, _state(_integrate(_volume(), cams, dep, rgb, per_call=1)))
    assert _bits_equal(ref, _state(_integrate(_volume(), cams, dep, rgb)))
    assert _bits_equal(ref, _state(_integrate(_volume(), cams, dep, rgb, per_call=5)))


def test_skipped_pixels_change_nothing():
    cams, dep, rgb = _views(SPHERE, W=128, H=128, seed=1)
    mask = torch.rand(dep.shape, generator=torch.Generator().manual_seed(2)).numpy() < 0.3
    trunc = 5.0
    base = dep.copy()
    base[mask] = 0.0
    ref = _state(_integrate(_volume(), cams, base, rgb, depth_trunc=trunc))
    for bad in (-1.0, -np.inf, np.nan, np.inf, 7.5, 0.0):
        d = dep.copy()
        d[mask] = bad
        assert _bits_equal(ref, _state(_integrate(_volume(), cams, d, rgb, depth_trunc=trunc))), bad
    far = dep.copy()
    far[mask & (dep > 0)] += trunc                            # real surfaces pushed beyond depth_trunc
    assert _bits_equal(ref, _state(_integrate(_volume(), cams, np.where(mask & (dep > 0), far, base), rgb,
                                              depth_trunc=trunc)))


def test_points_outside_every_frustum_keep_their_bytes():
    cams, dep, rgb = _views(SPHERE, W=96, H=64, seed=3)
    full = np.where(dep > 0, dep, 3.0).astype(np.float32)      # every pixel observed
    vol = tsdf.TSDFVolume((-6.0,) * 3, (6.0,) * 3, 0.25, 0.5, device=DEV)
    init = [torch.full(vol.dims, 1.0), torch.zeros(vol.dims), torch.zeros(vol.dims + (3,))]
    _integrate(vol, cams, full, rgb)
    pts = O.grid_points(vol.origin, vol.voxel_size, vol.dims).reshape(-1, 3)
    seen = np.zeros(len(pts), dtype=bool)
    for vm, fx, fy, cx, cy, W, H in O.cam_rows(cams):
        p = pts @ vm[:3, :3] + vm[3, :3]
        Z = p[:, 2]
        Zs = np.where(Z > 1e-3, Z, 1.0)
        u, v = fx * p[:, 0] / Zs + cx, fy * p[:, 1] / Zs + cy
        seen |= (Z > -1e-3) & (u > -1.5) & (u < W + 0.5) & (v > -1.5) & (v < H + 0.5)
    out = torch.from_numpy(~seen.reshape(vol.dims))
    assert out.sum() > 1000 and (~out).sum() > 1000
    for got, want in zip(_state(vol), init):
        assert torch.equal(got[out].view(torch.int32), want[out].view(torch.int32))
    assert (vol.weight.cpu()[~out] > 0).any()


def _check_extract(vol):
    v, f, c = vol.extract()
    ov, of, oc = O.marching_cubes(vol.tsdf.cpu().numpy(), vol.weight.cpu().numpy(),
                                  None if vol.color is None else vol.color.cpu().numpy(), vol.origin, vol.voxel_size)
    assert v.dtype == torch.float32 and f.dtype == torch.int32 and tuple(v.shape) == (len(ov), 3)
    assert np.array_equal(f.cpu().numpy(), of)
    assert np.abs(v.cpu().double().numpy() - ov).max(initial=0) < 1e-6
    if vol.color is not None:
        assert np.abs(c.cpu().double().numpy() - oc).max(initial=0) < 1e-6
    else:
        assert c is None
    v2, f2, c2 = vol.extract()
    assert torch.equal(v.view(torch.int32), v2.view(torch.int32)) and torch.equal(f, f2)
    if c is not None:
        assert torch.equal(c.view(torch.int32), c2.view(torch.int32))
    if len(f):
        assert np.array_equal(np.unique(of), np.arange(len(ov))), "unreferenced vertex"
    return v.cpu().double().numpy(), f.cpu().numpy()


def test_extract_sphere(sphere_case):
    v, f = _check_extract(sphere_case[3])
    assert O.is_closed_oriented_manifold(f) and O.euler(len(v), f) == 2 and O.signed_volume(v, f) > 0
    assert (np.abs(np.linalg.norm(v, axis=1) - 0.8) < 0.5 * VS).all()


def test_extract_two_spheres():
    cams, dep, rgb = _views(TWO, seed=4)
    v, f = _check_extract(_integrate(_volume(), cams, dep, rgb))
    assert O.is_closed_oriented_manifold(f) and O.components(len(v), f) == 2 and O.euler(len(v), f) == 4


def test_extract_random_field_with_holes():
    g = torch.Generator().manual_seed(5)
    vol = tsdf.TSDFVolume((0.0,) * 3, (1.0, 1.4, 0.6), 0.02, 0.08, device=DEV)
    field = torch.randn(vol.dims, generator=g)
    field[torch.rand(vol.dims, generator=g) < 0.1] = 0.0
    weight = torch.randint(1, 5, vol.dims, generator=g).float()
    for _ in range(6):                                        # unobserved boxes
        lo = [int(torch.randint(0, n - 4, (1,), generator=g)) for n in vol.dims]
        weight[lo[0]:lo[0] + 6, lo[1]:lo[1] + 9, lo[2]:lo[2] + 4] = 0.0
    vol.tsdf.copy_(field)
    vol.weight.copy_(weight)
    vol.color.copy_(torch.rand(vol.dims + (3,), generator=g))
    v, f = _check_extract(vol)
    assert len(f) > 1000 and O.directed_edges_unique(f) and not O.is_closed_oriented_manifold(f)


def test_extract_empty_volumes():
    vol = _volume()
    for _ in range(2):
        v, f, c = vol.extract()
        assert tuple(v.shape) == (0, 3) and tuple(f.shape) == (0, 3) and tuple(c.shape) == (0, 3)
        vol.tsdf.copy_(torch.randn(vol.dims, generator=torch.Generator().manual_seed(6)))   # unobserved: weight 0
    vol = tsdf.TSDFVolume((0,) * 3, (1,) * 3, 0.5, 1.0, color=False, device=DEV)
    vol.weight.fill_(1.0)                                     # observed but no sign change
    v, f, c = vol.extract()
    assert len(v) == 0 and len(f) == 0 and c is None


# Radial bound of the mesh fused from the shell below: the same pipeline (P = 100000, 16 views of 128 x 128, centre
# depth / opacity masked at opacity > 0.5, 96^3 over [-1.2, 1.2]^3, sdf_trunc 4 voxels) through the CPU
# oracle.rasterize_forward and tests/tsdf_oracle.py gave max |r - 1| = 0.0935 (p99 0.068) over 36,611 vertices.
E2E_RADIAL_BOUND = 0.12


def test_end_to_end_from_rasterize_views():
    P, W, H = 100000, 128, 128
    sc = synth.make_scene(P, "shell-v1", 0, 0)
    cams = O.ring_cameras(W, H)
    settings = [R.GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, torch.zeros(3, device=DEV), 1.0,
                                                c.viewmatrix.to(DEV), c.projmatrix.to(DEV), 3, c.campos.to(DEV),
                                                False, True, True, False) for c in cams]
    d = lambda t: t.to(DEV)
    with torch.no_grad():
        out = R.rasterize_views(d(sc.means3D), torch.zeros(len(cams), P, 3, device=DEV), d(sc.opacities),
                                settings=settings, shs=d(sc.shs), scales=d(sc.scales), rotations=d(sc.rotations))
        opacity, depth_img, image = out[3], out[4], out[2]
        depth = torch.where(opacity > 0.5, depth_img / opacity.clamp_min(1e-5), torch.zeros_like(depth_img))
        assert (opacity > 0.5).float().mean() > 0.4
        vol = _volume()
        vol.integrate(depth, settings, image.clamp(0, 1))
    dims = vol.dims
    t, w, c, near = O.integrate(np.ones(dims, np.float32), np.zeros(dims, np.float32), np.zeros(dims + (3,), np.float32),
                                ORIGIN, VS, 4 * VS, depth[:, 0].cpu().numpy(), image.clamp(0, 1).cpu().numpy(),
                                O.cam_rows(settings))
    keep = ~near
    assert np.array_equal(vol.weight.cpu().double().numpy()[keep], w[keep])
    assert np.abs(vol.tsdf.cpu().double().numpy() - t)[keep].max() < 1e-5
    assert np.abs(vol.color.cpu().double().numpy() - c)[keep].max() < 1e-5
    v, f = _check_extract(vol)
    r = np.linalg.norm(v, axis=1)
    assert len(v) > 10000 and np.abs(r - 1.0).max() < E2E_RADIAL_BOUND

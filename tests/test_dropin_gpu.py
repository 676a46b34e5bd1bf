"""The drop-in boundary (SURVEY.md §8b): this repo's `dropin/` packages (`r3dg_rasterization`, `bvh_tracing`) against
what the reference's OWN code path computed on the same seeded inputs — its wrapper files
(gaussian_renderer/r3dg_rasterization.py, bvh/__init__.py) over its own pybind modules (rasterize_points.cu / bvh.cu
glue + its kernels).  Those results are stored in tests/golden/live_dropin.npz (tests/golden/make_golden_live.py):
integer outputs as sha256 digests, images at a seeded pixel sample and as random-sign sketches, gradients as sketches, visibility at
a seeded ray sample.  Outputs and gradients must agree to the north_star tolerances.  Also: the full visibility bake
(own tree + in-kernel sampling + own trace) against the reference's bake (its tree + PyTorch sampling + its trace),
and the sampling kernel against the reference's own `fibonacci_sphere_sampling`."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN, ROOT, case_inputs, digest, fixed_sample, npy, rel_l2_sketch, sketch

pytestmark = pytest.mark.gpu
DROPIN_CASES = [(60_000, 400, 304, 16), (300_000, 800, 800, 5)]
BAKE_CASES = [(100_000, 32), (40_000, 64)]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "live_dropin.npz"))


def dropin(pkg):
    if os.path.join(ROOT, "dropin") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "dropin"))
    return importlib.import_module(pkg)


def render_through_wrapper(mod, sc, cam, S, bg, cots):
    d = lambda t: t.cuda()
    leaves = [d(t).requires_grad_(True) for t in (sc.means3D, sc.opacities, sc.shs, sc.scales, sc.rotations, sc.features)]
    xyz, opac, shs, scales, rots, feats = leaves
    rs = mod.GaussianRasterizationSettings(
        image_height=cam.image_height, image_width=cam.image_width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, cx=cam.cx, cy=cam.cy,
        bg=d(bg), scale_modifier=1.0, viewmatrix=d(cam.viewmatrix), projmatrix=d(cam.projmatrix), sh_degree=3, campos=d(cam.campos),
        prefiltered=False, backward_geometry=True, computer_pseudo_normal=True, debug=False)
    means2D = torch.zeros_like(xyz, requires_grad=True)
    rast = mod.GaussianRasterizer(rs)
    out = rast(means3D=xyz, means2D=means2D, shs=shs, colors_precomp=None, opacities=opac, scales=scales, rotations=rots,
               cov3D_precomp=None, features=feats)
    (num_rendered, num_contrib, color, opacity, depth, feature, normal, surface_xyz, weights, radii) = out
    # the reference returns num_contrib as a NON-OWNING from_blob view of imgBuffer (rasterize_points.cu:136-139): it dangles
    # once autograd frees the saved buffers, so it is copied before backward
    num_contrib = num_contrib.clone()
    loss = sum((o * d(c)).sum() for o, c in zip((color, opacity, depth, feature), cots))
    loss.backward()
    torch.cuda.synchronize()
    vis = rast.markVisible(xyz)
    res = dict(num_rendered=int(num_rendered), num_contrib=num_contrib, color=color, opacity=opacity, depth=depth, feature=feature,
               normal=normal, surface_xyz=surface_xyz, weights=weights, radii=radii, visible=vis)
    grads = dict(means3D=xyz.grad, opacity=opac.grad, shs=shs.grad, scales=scales.grad, rotations=rots.grad, features=feats.grad,
                 means2D=means2D.grad)
    return res, grads


@pytest.mark.parametrize("P,W,H,S", DROPIN_CASES, ids=["60k-S16", "300k-S5"])
def test_dropin_rasterizer_matches_reference_wrapper_golden(golden, P, W, H, S):
    mod = dropin("r3dg_rasterization")
    assert os.path.realpath(mod._C.__file__).startswith(os.path.join(os.path.realpath(ROOT), "relightable3dgaussian_b200"))
    key = f"raster_P{P}_S{S}__"
    sc, cam = case_inputs(P, W, H, S, view=4, center_shift=True)
    g = torch.Generator().manual_seed(3)
    cots = [torch.randn(c, H, W, generator=g) for c in (3, 1, 1, S)]
    oo, og = render_through_wrapper(mod, sc, cam, S, torch.tensor([0.3, 0.1, 0.7]), cots)
    assert oo["num_rendered"] == int(golden[key + "num_rendered"])
    for n in ("radii", "num_contrib", "visible"):
        assert digest(oo[n]) == str(golden[key + "dig_" + n]), n
    pix = torch.from_numpy(golden[key + "pix"].astype(np.int64)).cuda()
    for n in ("color", "opacity", "depth", "feature", "normal", "surface_xyz"):
        t = oo[n]
        assert np.abs(npy(t.reshape(t.shape[0], -1)[:, pix]) - golden[key + "img_" + n]).max() <= 1e-4, n
        assert rel_l2_sketch(sketch(t), golden[key + "sk_img_" + n]) < 1e-4, n
    for n in og:
        assert og[n] is not None, n
        assert rel_l2_sketch(sketch(og[n]), golden[key + "sk_" + n]) < 1e-3, n


def bvh_scene(P):
    sc, _ = case_inputs(P, 64, 64, 0)
    d = lambda t: t.cuda()
    return d(sc.means3D), d(sc.scales), d(sc.rotations), d(sc.opacities[:, 0].contiguous()), d(sc.normals)


def test_dropin_raytracer_matches_reference_golden(golden):
    from oracle import oracle_sampling
    ours = dropin("bvh_tracing")
    xyz, s, r, op, nrm = bvh_scene(30_000)
    icov = oracle_sampling.inverse_covariance(s, r)
    a = ours.RayTracer(xyz, s, r)
    for name in ("tree", "morton"):                                   # topology + Morton codes bit-exact
        if "tracer__dig_" + name in golden.files:
            assert digest(getattr(a, name)) == str(golden["tracer__dig_" + name]), name
    dirs, _ = oracle_sampling.sample_incident_rays(nrm, False, 24)
    ro = xyz[:, None].expand_as(dirs)
    va = npy(a.trace_visibility(ro, dirs, xyz, icov, op, nrm)["visibility"]).reshape(-1)[golden["tracer__ray_idx"]]
    vb = golden["tracer__visibility"]
    flips = ((va == 0) != (vb == 0)).mean()
    same = (va == 0) == (vb == 0)
    assert flips <= 1e-3, flips
    assert np.abs(va - vb)[same].max() <= 1e-4


def sampling_normals():
    g = torch.Generator().manual_seed(1)
    nrm = torch.nn.functional.normalize(torch.randn(50_000, 3, generator=g), dim=-1).cuda()
    nrm[0] = torch.tensor([0.0, 0.0, -1.0]); nrm[1] = torch.tensor([0.0, 0.0, 1.0])      # the -I fallback and the identity
    return nrm


def sampling_pairs(P, N):
    """Flat (normal, direction) indices: every direction of the two special normals + a seeded sample of the rest."""
    return np.concatenate([np.arange(2 * N), fixed_sample(P * N - 2 * N, 2048, N) + 2 * N])


def test_sampling_kernel_vs_reference_function(golden):
    """r3dg_sample_incident_dirs vs the reference's own fibonacci_sphere_sampling (utils/graphics_utils.py:9-37),
    deterministic and random-rotate variants."""
    from relightable3dgaussian_b200 import raytracer
    nrm = sampling_normals()
    for N in (24, 32, 384):
        d, a = raytracer.sample_incident_rays(nrm, False, N)
        assert tuple(d.shape) == tuple(golden[f"sampling__shape_{N}"]) and a.shape == d.shape[:-1] + (1,)
        assert digest(a.contiguous().view(torch.int32)) == str(golden[f"sampling__dig_areas_{N}"])
        dd = npy(d).reshape(-1, 3)[golden[f"sampling__idx_{N}"]]
        assert np.abs(dd - golden[f"sampling__dirs_{N}"]).max() <= 5e-7, N                    # unit vectors: a few ulp at most
        print(f"[sampling] N={N}: bit-equal fraction {(dd == golden[f'sampling__dirs_{N}']).mean():.6f}")
    # random rotation: same phase numbers through both
    torch.manual_seed(5)
    d, _ = raytracer.fibonacci_sphere_sampling(nrm, 32, random_rotate=True)
    assert np.abs(npy(d).reshape(-1, 3)[sampling_pairs(nrm.shape[0], 32)] - golden["sampling__dirs_rot32"]).max() <= 5e-6


@pytest.mark.parametrize("P,N", BAKE_CASES)
def test_full_bake_parity_own_tree_vs_reference_tree(golden, P, N):
    """update_visibility end to end: OUR tree (exact refit) + in-kernel sampling + our trace, against the REFERENCE's
    bake (its racy-refit tree, PyTorch sampling, its trace kernel, its chunk loop).  Visibility is a step function of T
    at 0.9, so the flip rate across that cliff is the meaningful figure (north_star)."""
    from oracle import oracle_sampling
    from relightable3dgaussian_b200 import raytracer
    key = f"bake_P{P}_N{N}__"
    xyz, s, r, op, nrm = bvh_scene(P)
    icov = oracle_sampling.inverse_covariance(s, r)
    assert (raytracer.inverse_covariance(s, r) - icov).abs().max().item() <= 1e-3 * icov.abs().max().item()
    vis, dirs, areas = raytracer.update_visibility(xyz, s, r, icov, op, nrm, N)
    assert vis.shape == (P, N, 1) and dirs.shape == (P, N, 3)
    assert digest(areas.contiguous().view(torch.int32)) == str(golden[key + "dig_areas"])
    idx = golden[key + "ray_idx"]
    assert np.abs(npy(dirs).reshape(-1, 3)[idx] - golden[key + "dirs"]).max() <= 5e-7
    v, rv = npy(vis).reshape(-1)[idx], golden[key + "visibility"]
    flip = ((v == 0) != (rv == 0)).mean()
    same = (v == 0) == (rv == 0)
    print(f"[bake] P={P} N={N}: blocked {float(golden[key + 'blocked']):.3f}, flip rate {flip:.2e}, max-abs on agreeing rays {np.abs(v - rv)[same].max():.2e}")
    assert flip <= 1e-3
    assert np.abs(v - rv)[same].max() <= 1e-4

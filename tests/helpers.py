"""Shared test utilities: seeded cases, conversions, comparison helpers."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from relightable3dgaussian_b200 import synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def sh_case(P, seed):
    """Inputs of BASELINE.json config #1: sh [P,3,16] (channel-major, utils/sh_utils.py:77), unit dirs."""
    g = torch.Generator().manual_seed(1000 + seed)
    sh = torch.randn(P, 3, 16, generator=g) * 0.3
    dirs = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    return sh, dirs


def npy(t):
    return None if t is None else t.detach().cpu().numpy()


def case_inputs(P, W, H, S, view=1, recipe="shell-v1", seed=0, scale_boost=1.0, center_shift=False):
    sc = synth.make_scene(P, recipe, seed, S)
    if scale_boost != 1.0:
        sc = sc._replace(scales=sc.scales * scale_boost)
    cam = synth.make_camera(view, W, H, center_shift=center_shift)
    return sc, cam


def oracle_kwargs(sc, cam, bg):
    return dict(means3D=npy(sc.means3D), opacities=npy(sc.opacities), viewmatrix=npy(cam.viewmatrix),
                projmatrix=npy(cam.projmatrix), campos=npy(cam.campos), bg=npy(bg),
                W=cam.image_width, H=cam.image_height, tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy,
                cx=cam.cx, cy=cam.cy)


def rel_l2(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def max_rel_above_floor(a, b, floor=1e-6):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    m = np.abs(b) > floor * (np.abs(b).max() + 1e-30)
    if not m.any():
        return 0.0
    return float((np.abs(a - b)[m] / np.abs(b)[m]).max())


def digest(t):
    """sha256 of an integer array's values (as int64): bit-exact comparison against a stored fixture."""
    import hashlib
    a = t.detach().cpu().long().numpy() if isinstance(t, torch.Tensor) else np.asarray(t).astype(np.int64)
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def sketch(t, k=32):
    """k random +-1 projections of a float array (a Johnson-Lindenstrauss sketch, float64).  The rows are a
    fixed integer hash of (row, element index), identical on every device, so the sketches of two arrays
    estimate their relative L2 difference over ALL elements: rel_l2_sketch(sketch(a), sketch(b))."""
    x = t.detach().reshape(-1).double()
    j = torch.arange(x.numel(), dtype=torch.int64, device=x.device)
    out = np.empty(k)
    for i in range(k):
        h = (j + ((i + 1) * 0x9E3779B1 & 0xFFFFFFFF)) & 0xFFFFFFFF
        h = (((h >> 16) ^ h) * 0x45D9F3B) & 0xFFFFFFFF
        h = (((h >> 16) ^ h) * 0x45D9F3B) & 0xFFFFFFFF
        h = (h >> 16) ^ h
        out[i] = float((x * ((h & 1).double() * 2 - 1)).sum())
    return out


def rel_l2_sketch(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / (np.linalg.norm(b) + 1e-30))


def raster_key(P, W, H, S, view, shift, bwd, deg=3, M=16, boost=1.0):
    """Name of a rasterizer parity case in tests/golden/live_raster.npz."""
    return f"P{P}_{W}x{H}_S{S}_v{view}_c{int(shift)}_b{int(bwd)}_d{deg}_M{M}_x{boost:g}"


def fixed_sample(n, k, seed):
    """Seeded sorted sample of min(n, k) indices out of n."""
    return np.sort(np.random.default_rng(seed).choice(n, min(n, k), replace=False))


def inverse_covariance(scales, rotations):
    """scene/gaussian_model.py:257-260 + utils/general_utils.py:151-160 (strip_symmetric of
    L L^T with L = R diag(1/s)); torch ops, device of the inputs."""
    r = rotations
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = torch.zeros((q.size(0), 3, 3), device=r.device)
    rr, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - rr * z); R[:, 0, 2] = 2 * (x * z + rr * y)
    R[:, 1, 0] = 2 * (x * y + rr * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - rr * x)
    R[:, 2, 0] = 2 * (x * z - rr * y); R[:, 2, 1] = 2 * (y * z + rr * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    L = torch.zeros((q.size(0), 3, 3), dtype=torch.float, device=r.device)
    inv_s = 1 / scales
    L[:, 0, 0] = inv_s[:, 0]; L[:, 1, 1] = inv_s[:, 1]; L[:, 2, 2] = inv_s[:, 2]
    L = R @ L
    cov = L @ L.transpose(1, 2)
    return torch.stack([cov[:, 0, 0], cov[:, 0, 1], cov[:, 0, 2], cov[:, 1, 1], cov[:, 1, 2], cov[:, 2, 2]], dim=-1).contiguous()


def bvh_case(recipe, P, n_src, N, boost, seed=3):
    """Seeded BVH / visibility case: P Gaussians, rays from the first n_src of them along N
    Fibonacci directions around the FLIPPED normal (so that they run through the scene),
    origins pre-offset by 0.05 d like bvh/__init__.py:63."""
    from oracle.oracle_sampling import fibonacci_sphere_sampling
    sc = synth.make_scene(P, recipe, seed, 0)
    scales = sc.scales * boost
    normals = sc.normals
    dirs, _ = fibonacci_sphere_sampling(-normals[:n_src], N, random_rotate=False)
    rays_o = (sc.means3D[:n_src, None] + dirs * 0.05).contiguous()
    return dict(means3D=sc.means3D, scales=scales.contiguous(), rotations=sc.rotations, opacity=sc.opacities[:, 0].contiguous(),
                normals=normals, inv_cov=inverse_covariance(scales, sc.rotations), rays_o=rays_o, rays_d=dirs.contiguous())


def shading_case(P, N, He, seed):
    """Seeded inputs of `rendering_equation` (neilf.py:339): activated material parameters, SH
    incident light, raw env map (softplus applied by the light object), baked visibility / dirs."""
    from oracle.oracle_sampling import fibonacci_sphere_sampling
    g = torch.Generator().manual_seed(500 + seed)
    n = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    dirs, areas = fibonacci_sphere_sampling(n, N, random_rotate=False)
    vis = torch.where(torch.rand(P, N, 1, generator=g) < 0.4, torch.zeros(P, N, 1), 0.9 + 0.1 * torch.rand(P, N, 1, generator=g))
    return dict(base_color=torch.sigmoid(torch.randn(P, 3, generator=g)) * 0.77 + 0.03,
                roughness=torch.sigmoid(torch.randn(P, 1, generator=g)) * 0.9 + 0.09,
                normals=(n + 0.05 * torch.randn(P, 3, generator=g)).contiguous(),       # deliberately not unit length
                viewdirs=torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1),
                incidents=(torch.randn(P, 16, 3, generator=g) * 0.3).contiguous(),
                env_raw=torch.randn(1, He, 2 * He, 3, generator=g),
                visibility=vis.contiguous(), incident_dirs=dirs.contiguous(), incident_areas=areas.contiguous(),
                cot_pbr=torch.randn(P, 3, generator=g), cot_diffuse=torch.randn(P, 3, generator=g),
                cot_specular=torch.randn(P, 3, generator=g))


def adam_case():
    """Seeded optimiser case shared by tests/golden/make_golden_adam.py and the tests: three parameter
    groups shaped like the reference's (xyz [P,3], f_rest [P,15,3], opacity [P,1]) with its learning
    rates (arguments/__init__.py), 7 steps of gradients (exact zeros for half of the f_rest rows: never
    seen Gaussians, eps = 1e-15 decides; an all-zero step for xyz), one lr edit at step 5."""
    g = torch.Generator().manual_seed(3)
    shapes, lrs = [(500, 3), (500, 15, 3), (500, 1)], [1.6e-4, 2.5e-3 / 20, 5e-2]
    params = [torch.randn(s, generator=g).numpy() for s in shapes]

    def grads_for_step(step):
        gg = torch.Generator().manual_seed(100 + step)
        gs = [torch.randn(s, generator=gg) * (0.0 if (step == 3 and i == 0) else 1e-3) for i, s in enumerate(shapes)]
        gs[1][::2] = 0.0
        return [t.numpy() for t in gs]
    return params, lrs, grads_for_step, {5: [(0, 1.0e-4)]}

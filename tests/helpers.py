"""Shared test utilities: seeded cases, conversions, comparison helpers."""
import math
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


def _axis_points(n, g, W, H, tanfovx, z, margin=0.9):
    """n points at depths z (tensor [n]) whose projections fall inside the image of make_axis_camera."""
    tanfovy = tanfovx * H / W
    u = (torch.rand(n, 2, generator=g) * 2 - 1) * margin
    return torch.stack([u[:, 0] * tanfovx * z, u[:, 1] * tanfovy * z, z], dim=1)


def _edge_scene(name, P=None):
    """-> (Scene-like dict of torch inputs, Camera, S).  See EDGE_CASES.  `P` overrides the size of a depth case."""
    family, _, arg = name.partition("-")
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    if family == "inside":                                  # camera inside a cube of random Gaussians
        sc = synth.make_scene(30_000, "cube-v1", 4, 5)
        cam = synth.make_camera(3, 320, 240, radius=0.3, fovx=1.8)
        return dict(means3D=sc.means3D, opacities=sc.opacities, shs=sc.shs, scales=sc.scales * 3.0, rotations=sc.rotations,
                    features=sc.features, scale_modifier=float(arg[1:])), cam, 5
    if family == "needles":                                 # per-axis scale ratios up to ~1e4 : 1
        P = 2_500
        sc = synth.make_scene(P, "shell-v1", 6, 0)
        stretch = torch.exp((torch.rand(P, 3, generator=g) * 2 - 1) * math.log(100.0))
        scales = sc.scales * stretch * torch.tensor([3.0, 1.0, 0.3])
        opac = 1.0 - torch.rand(P, 1, generator=g)          # (0, 1]
        return dict(means3D=sc.means3D, opacities=opac, shs=sc.shs, scales=scales, rotations=sc.rotations,
                    features=None), synth.make_camera(2, 320, 232), 0
    if family == "opaque":                                  # stacks of near-coincident, nearly opaque Gaussians
        S = int(arg[1:])
        k = torch.randint(8, 65, (260,), generator=g)
        centre = torch.repeat_interleave(synth.make_scene(260, "shell-v1", 7, 0).means3D, k, dim=0)
        P = centre.shape[0]
        sc = synth.make_scene(P, "shell-v1", 8, S)
        means = centre + 2e-3 * torch.randn(P, 3, generator=g)
        scales = 0.02 + 0.04 * torch.rand(P, 3, generator=g)
        opac = 0.97 + 0.03 * torch.rand(P, 1, generator=g)
        return dict(means3D=means, opacities=opac, shs=sc.shs, scales=scales, rotations=sc.rotations,
                    features=sc.features), synth.make_camera(1, 208, 144), S
    if family == "depth":                                   # depth-key bit patterns of every radix-sort plan
        P, W, H = P or 6_500, 128, 96
        cam = synth.make_axis_camera(W, H)
        z = {"equal": torch.full((P,), 2.0),
             "adjacent": torch.where(torch.rand(P, generator=g) < 0.5, torch.tensor(2.0),
                                     torch.nextafter(torch.tensor(2.0), torch.tensor(3.0))),
             "narrow": 1.0 + torch.randint(0, 2 ** 15, (P,), generator=g).float() * 2.0 ** -23,
             "w7": 1.0 + torch.randint(0, 2 ** 20, (P,), generator=g).float() * 2.0 ** -23,
             "3to5": 3.0 + 2.0 * torch.rand(P, generator=g),
             "wide": torch.exp(math.log(0.25) + math.log(240.0) * torch.rand(P, generator=g))}[arg].float()
        # exact ties: a third of the Gaussians copy the depth of another one
        tie = torch.rand(P, generator=g) < 0.33
        z = torch.where(tie, z[torch.randint(0, P, (P,), generator=g)], z)
        means = _axis_points(P, g, W, H, cam.tanfovx, z)
        scales = z[:, None] * torch.exp(torch.rand(P, 3, generator=g) * 2.3 - 5.0)
        sc = synth.make_scene(P, "shell-v1", 9, 3)
        return dict(means3D=means, opacities=sc.opacities, shs=sc.shs, scales=scales, rotations=sc.rotations,
                    features=sc.features), cam, 3
    if family == "thresholds":                              # the z = 0.2 cull plane and the alpha = 1/255 threshold
        W, H = 65, 49                                       # odd: the principal point is a pixel centre
        cam = synth.make_axis_camera(W, H)
        z02 = torch.tensor(0.2, dtype=torch.float32)
        zs = torch.stack([torch.nextafter(z02, torch.tensor(0.0)), z02, torch.nextafter(z02, torch.tensor(1.0)),
                          torch.tensor(0.5), torch.tensor(1.5)])
        a = torch.tensor(1.0 / 255.0, dtype=torch.float32)
        ops = torch.stack([torch.nextafter(a, torch.tensor(0.0)), a, torch.nextafter(a, torch.tensor(1.0)),
                           torch.tensor(0.99), torch.tensor(1.0)])
        zz, oo = torch.meshgrid(zs, ops, indexing="ij")
        zz, oo = zz.reshape(-1).repeat(12), oo.reshape(-1).repeat(12)
        P = zz.numel()
        means = _axis_points(P, g, W, H, cam.tanfovx, zz)
        means[:25, :2] = 0.0                                 # centred on the principal point: alpha == opacity there
        scales = zz[:, None] * torch.exp(torch.rand(P, 3, generator=g) * 1.5 - 4.5)
        sc = synth.make_scene(P, "shell-v1", 10, 2)
        return dict(means3D=means, opacities=oo[:, None].contiguous(), shs=sc.shs, scales=scales,
                    rotations=sc.rotations, features=sc.features), cam, 2
    if family == "strip":                                   # degenerate image shapes
        W, H = map(int, arg.split("x"))
        sc = synth.make_scene(3_000, "shell-v1", 11, 1)
        return dict(means3D=sc.means3D, opacities=sc.opacities, shs=sc.shs, scales=sc.scales * 2.0,
                    rotations=sc.rotations, features=sc.features), synth.make_camera(4, W, H), 1
    if family == "precomp":                                 # colours + covariances given, some indefinite / singular
        P, W, H = 4_000, 160, 120
        sc = synth.make_scene(P, "shell-v1", 12, 0)
        cam = synth.make_axis_camera(W, H)
        means = _axis_points(P, g, W, H, cam.tanfovx, 1.0 + 3.0 * torch.rand(P, generator=g))
        A = torch.randn(P, 3, 3, generator=g) * 0.03
        cov = A @ A.transpose(1, 2)
        kind = torch.arange(P) % 5
        ev = torch.randn(P, 3, generator=g).abs() * 1e-3
        ev = torch.where((kind == 1)[:, None], ev * torch.tensor([1.0, -1.0, 1.0]), ev)        # indefinite
        ev = torch.where((kind == 2)[:, None], ev * torch.tensor([1.0, 1e-7, 1e-7]), ev)       # nearly rank 1
        ev = torch.where((kind == 3)[:, None], ev * torch.tensor([1.0, 1.0, 1e-7]), ev)        # nearly rank 2
        # (no negative-definite covariances: their 2D radius is NaN -> 0 while they still touch a tile, and the
        # reference then leaves those list entries unwritten, rasterizer_impl.cu:85)
        Q = torch.linalg.qr(torch.randn(P, 3, 3, generator=g))[0]
        cov = torch.where((kind == 0)[:, None, None], cov, Q @ torch.diag_embed(ev) @ Q.transpose(1, 2))
        c6 = torch.stack([cov[:, 0, 0], cov[:, 0, 1], cov[:, 0, 2], cov[:, 1, 1], cov[:, 1, 2], cov[:, 2, 2]], 1)
        # det(cov2D) == 0 exactly: a centred Gaussian whose projected x variance cancels the +0.3 low-pass term
        fx = W / (2.0 * cam.tanfovx)
        means[:8] = torch.tensor([0.0, 0.0, 1.0])
        c6[:8] = torch.tensor([-0.3 / fx ** 2, 0.0, 0.0, 1e-3, 0.0, 1e-3])
        colors = torch.rand(P, 3, generator=g)
        return dict(means3D=means, opacities=sc.opacities, colors_precomp=colors, cov3D_precomp=c6.float(),
                    features=None), cam, 0
    raise KeyError(name)


# Adversarial rasterizer cases (tests/test_raster_gpu.py, tests/golden/make_golden_live.py --only edge).  Small enough
# for the CPU oracle; every one asserts that it reaches the path it is named for (edge_coverage).
EDGE_CASES = (["inside-x1", "inside-x0.6", "inside-x1.8", "needles", "opaque-S0", "opaque-S5", "opaque-S16"] +
              [f"depth-{k}" for k in ("equal", "adjacent", "narrow", "w7", "3to5", "wide")] +
              ["thresholds"] +
              [f"strip-{s}" for s in ("1x1", "1x37", "37x1", "7x5", "9x4", "17x33", "4100x16", "16x2050")] +
              ["precomp"])


def edge_case(name, P=None):
    """Seeded inputs of one EDGE_CASES entry as numpy arrays: (oracle / run_ours keyword arguments, cotangents).
    `P` overrides the size of a depth case (the default is the fixture's)."""
    d, cam, S = _edge_scene(name, P)
    bg = torch.tensor([0.0, 0.5, 1.0])
    kw = dict(means3D=d["means3D"], opacities=d["opacities"], viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix,
              campos=cam.campos, bg=bg, W=cam.image_width, H=cam.image_height, tan_fovx=cam.tanfovx,
              tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy, features=d["features"],
              scale_modifier=d.get("scale_modifier", 1.0))
    for k in ("shs", "scales", "rotations", "colors_precomp", "cov3D_precomp"):
        if k in d:
            kw[k] = d[k]
    kw = {k: (np.ascontiguousarray(npy(v.float())) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    gen = torch.Generator().manual_seed(2)
    H, W = cam.image_height, cam.image_width
    cots = [npy(torch.randn(c, H, W, generator=gen)) for c in (3, 1, 1, S)]
    return kw, cots


def edge_stats(kw, radii, depths, conic_opacity, n_contrib, final_T, ranges):
    """What an edge case reaches, from a rasterizer's intermediates (ours or the oracle's): the radix-sort plan of the
    visible depth keys (common.cuh sort_plan), the fraction of visible Gaussians whose x / y view direction is clamped
    to 1.3 tan(fov), the trace^2 / det range of the visible conics, and how many pixels stop early."""
    vis = np.asarray(radii) > 0
    bits = np.asarray(depths, np.float32).view(np.uint32)[vis]
    diff = (int(np.bitwise_or.reduce(bits)) & int(np.bitwise_or.reduce(~bits))) if bits.size else 0
    nb = diff.bit_length()
    passes = (nb + 7) // 8
    w = -(-nb // passes) if passes else 0
    V = np.asarray(kw["viewmatrix"], np.float64)
    t = np.c_[np.asarray(kw["means3D"], np.float64), np.ones(len(vis))] @ V
    t = t[vis]
    cx = np.abs(t[:, 0] / t[:, 2]) > 1.3 * kw["tan_fovx"]
    cy = np.abs(t[:, 1] / t[:, 2]) > 1.3 * kw["tan_fovy"]
    co = np.asarray(conic_opacity, np.float64)[vis]
    with np.errstate(divide="ignore", invalid="ignore"):
        cond = (co[:, 0] + co[:, 2]) ** 2 / (co[:, 0] * co[:, 2] - co[:, 1] ** 2)
    pd = (co[:, 0] > 0) & (co[:, 2] > 0) & np.isfinite(cond) & (cond > 0)
    W, H = kw["W"], kw["H"]
    gx = (W + 15) // 16
    rg = np.asarray(ranges, np.int64).reshape(-1, 2)
    lens = rg[:, 1] - rg[:, 0]
    tile = (np.arange(H)[:, None] // 16) * gx + np.arange(W)[None, :] // 16
    nc = np.asarray(n_contrib, np.int64).reshape(H, W)
    fT = np.asarray(final_T, np.float32).reshape(H, W)
    early = nc < lens[tile]
    sat = early & (fT < 1e-2)
    return dict(P=len(vis), visible=int(vis.sum()), passes=passes, w=w, clamp_x=float(cx.mean()) if vis.any() else 0.0,
                clamp_y=float(cy.mean()) if vis.any() else 0.0, near=int((t[:, 2] < 0.3).sum()),
                cond_min=float(cond[pd].min()) if pd.any() else 0.0, cond_max=float(cond[pd].max()) if pd.any() else 0.0,
                cond_over=int((cond[pd] > 6000).sum()), cond_under=int((cond[pd] <= 6000).sum()), not_pd=int((~pd).sum()),
                max_radius=int(np.asarray(radii).max()) if len(vis) else 0, early=int(early.sum()), saturated=int(sat.sum()),
                sat_stop_residues=sorted(set((nc[sat] % 4).tolist())), sat_min_contrib=int(nc[sat].min()) if sat.any() else -1)


def edge_coverage(name, s):
    """Assert that edge case `name` still reaches the path it exists for (stats from edge_stats)."""
    family, _, arg = name.partition("-")
    assert s["visible"] > 0, s
    if family == "inside":
        assert s["passes"] == 4 and s["clamp_x"] > 0.004 and s["clamp_y"] > 0.004 and s["near"] > 100, s
    elif family == "needles":
        assert s["cond_over"] > 50 and s["cond_under"] > 50 and s["max_radius"] > 200, s
    elif family == "opaque":
        assert s["saturated"] > 1000 and s["sat_stop_residues"] == [0, 1, 2, 3] and s["sat_min_contrib"] <= 3, s
    elif family == "depth":
        assert (s["passes"], s["w"]) == {"equal": (0, 0), "adjacent": (1, 1), "narrow": (2, 8), "w7": (3, 7),
                                         "3to5": (3, 8), "wide": (4, 8)}[arg], s
    elif family == "precomp":
        assert s["not_pd"] > 100, s


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


# every shading kernel variant r3dg_tune can select: lanes per Gaussian, env-gradient accumulation mode, SH operands /
# gradient accumulators in shared memory (csrc/shading.cu g_knobs)
SHADE_KNOBS = [dict(shade_group=16), dict(shade_group=32), dict(shade_env_mode=1), dict(shade_env_mode=0),
               dict(shade_group=32, shade_env_mode=1), dict(shade_fwd_variant=1, shade_bwd_variant=1),
               dict(shade_fwd_variant=1, shade_bwd_variant=2), dict(shade_bwd_variant=2, shade_env_mode=1),
               dict(shade_fwd_variant=0, shade_bwd_variant=0, shade_env_mode=2), dict(shade_bwd_variant=1, shade_env_mode=2),
               dict(shade_bwd_variant=2, shade_env_mode=2)]


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


def fake_raster_library(monkeypatch, overflow=False):
    """Replaces the four library functions behind rasterizer._C with stand-ins that record each call as (name, keyword
    arguments) in the list returned, and give zero outputs and gradients of the right shapes (None for the geometry
    gradients of an appearance-only backward).  With `overflow`, a deferred forward's count overflows its buffer, so
    the backward re-runs the forward."""
    import inspect
    from relightable3dgaussian_b200 import _C_raster
    from relightable3dgaussian_b200 import rasterizer as R

    class Overflowed(_C_raster.DeferredCount):
        def __init__(self):
            self._value, self.overflowed = 10, True

        def resolve(self):
            return 10

        __int__ = __index__ = resolve
    calls = []

    def stand_in(name):
        sig = inspect.signature(getattr(_C_raster, name))

        def call(*args, **kw):
            calls.append((name, kw))
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            a = b.arguments
            P, S = a["means3D"].shape[0], a["features"].shape[-1]
            V = len(a["cams"]) if "views" in name else 1
            lead = (V,) if "views" in name else ()
            z = lambda *s: torch.zeros(*s)                                       # noqa: E731
            if not name.endswith("backward"):
                H, W = a["image_height"], a["image_width"]
                count = [1] * V if lead else (Overflowed() if overflow and a["_defer"] else 1)
                return ((count, z(lead + (H, W)).int()) + tuple(z(lead + (c, H, W)) for c in (3, 1, 1, S, 3, 3)) +
                        (z(lead + (P, 1)), z(lead + (P,)).int()) + tuple(z(8).byte() for _ in range(3)) +
                        ((z(lead + (1, H, W)), z(lead + (1, H, W))) if a["depth_stats"] else ()))
            geo = a["geometry"]
            M = a["sh"].shape[1] if a["sh"].numel() else 0
            grads = (z(lead + (P, 3)) if geo else None, z(P, 3), z(P, 1) if geo else None, z(P, 3) if geo else None,
                     z(tuple(a["features"].shape)), z(P, 6) if geo else None, z(P, M, 3), z(P, 3) if geo else None,
                     z(P, 4) if geo else None)
            if a["cam_grads"]:
                grads += (z(lead + (4, 4)), z(lead + (4, 4)), z(lead + (3,)))
            return grads + ((z(lead + (P, 2)) if geo else None,) if a["absgrad"] else ())
        return call
    for name in ("rasterize_gaussians", "rasterize_gaussians_backward", "rasterize_views", "rasterize_views_backward"):
        monkeypatch.setattr(R._C, name, stand_in(name))
    return calls

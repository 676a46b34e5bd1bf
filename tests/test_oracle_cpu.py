"""The CPU oracle pinned against reference-owned data (no GPU needed):
  * eval_sh restatement vs outputs of the Python reference (config #1, tests/golden/sh_eval.npz);
  * the C rasterizer restatement vs outputs of the unmodified reference CUDA kernels
    (tests/golden/raster_*.npz, generated on a GPU by tests/golden/make_golden.py);
  * internal invariants of the binning (sortedness, ranges partition, stability)."""
import glob
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import GOLDEN, case_inputs, max_rel_above_floor, npy, oracle_kwargs, rel_l2, sh_case
from oracle import oracle

RASTER_CASES = sorted(glob.glob(os.path.join(GOLDEN, "raster_*.npz")))


def test_sh_config1_matches_python_reference():
    gold = np.load(os.path.join(GOLDEN, "sh_eval.npz"))
    for deg in (0, 1, 2, 3):
        sh, dirs = sh_case(10_000 if deg == 3 else 1_000, seed=deg)
        got = oracle.eval_sh(deg, sh.numpy(), dirs.numpy())
        assert got.shape == gold[f"deg{deg}"].shape
        # same float32 op order as the torch expression; allow 2 ulp of slack for fused scalars
        np.testing.assert_allclose(got, gold[f"deg{deg}"], rtol=0, atol=3e-7)
    rgb = np.maximum(oracle.eval_sh(3, *[t.numpy() for t in sh_case(10_000, 3)]) + np.float32(0.5), 0)
    np.testing.assert_allclose(rgb, gold["deg3_rgb"], rtol=0, atol=3e-7)
    sh4 = torch.randn(256, 3, 25, generator=torch.Generator().manual_seed(9))
    d4 = torch.nn.functional.normalize(torch.randn(256, 3, generator=torch.Generator().manual_seed(10)), dim=-1)
    np.testing.assert_allclose(oracle.eval_sh(4, sh4.numpy(), d4.numpy()), gold["deg4_small"], rtol=0, atol=2e-6)


def _run_oracle_on_golden(g):
    P, W, H, S, view, deg, R = [int(x) for x in g["meta"]]
    tfx, tfy, cx, cy = [float(x) for x in g["tanfov"]]
    mode = str(g["mode"])
    kw = dict(means3D=g["in_means3D"], opacities=g["in_opacities"], viewmatrix=g["in_viewmatrix"],
              projmatrix=g["in_projmatrix"], campos=g["in_campos"], bg=g["in_bg"], W=W, H=H, tan_fovx=tfx,
              tan_fovy=tfy, cx=cx, cy=cy, features=g["in_features"] if S else None, sh_degree=deg)
    if mode == "sh_sr":
        kw.update(shs=g["in_shs"], scales=g["in_scales"], rotations=g["in_rotations"])
    else:
        kw.update(colors_precomp=g["in_colors_precomp"], cov3D_precomp=g["in_cov3D_precomp"])
    f = oracle.rasterize_forward(**kw)
    bkw = {k: v for k, v in kw.items() if k in ("means3D", "viewmatrix", "projmatrix", "campos", "bg", "W", "H",
                                                 "tan_fovx", "tan_fovy", "shs", "scales", "rotations",
                                                 "cov3D_precomp", "features", "sh_degree")}
    gr = oracle.rasterize_backward(f, dL_dcolor=g["cot_color"], dL_dopacity=g["cot_opacity"],
                                   dL_ddepth=g["cot_depth"], dL_dfeature=g["cot_feature"], **bkw)
    return f, gr, (P, W, H, S, R, mode)


@pytest.mark.parametrize("path", RASTER_CASES, ids=[os.path.basename(p)[7:-4] for p in RASTER_CASES])
def test_oracle_matches_reference_cuda_golden(path):
    g = np.load(path)
    f, gr, (P, W, H, S, R, mode) = _run_oracle_on_golden(g)
    pre, b, img = f["pre"], f["binned"], f["img"]
    vis = g["out_radii"] > 0
    # ---- integer / index work: bit-exact -----------------------------------------------------
    assert np.array_equal(pre["radii"], g["out_radii"])
    assert np.array_equal(pre["tiles_touched"], g["mid_tiles_touched"].view(np.uint32))
    assert b["num_rendered"] == R
    assert np.array_equal(b["point_offsets"], g["mid_point_offsets"].view(np.uint32))
    assert np.array_equal(b["keys"], g["mid_point_list_keys"].view(np.uint64))
    assert np.array_equal(b["point_list"], g["mid_point_list"].view(np.uint32))
    T = b["ranges"].shape[0]
    assert np.array_equal(b["ranges"], g["mid_ranges"].view(np.uint32)[:T])
    # ---- IEEE-exact floats that feed the keys: bit-exact (visible Gaussians only; the reference
    # leaves culled rows uninitialised) ---------------------------------------------------------
    for name in ("depths", "means2D", "conic_opacity"):
        a, r = pre[name][vis], g["mid_" + name][vis]
        assert np.array_equal(a.view(np.uint32), r.view(np.uint32)), name
    if mode == "sh_sr":
        assert np.array_equal(pre["cov3D"][vis].view(np.uint32), g["mid_cov3D"][vis].view(np.uint32))
        np.testing.assert_allclose(pre["rgb"][vis], g["mid_rgb"][vis], atol=2e-6, rtol=0)
        assert np.array_equal(pre["clamped"][vis], g["mid_clamped"][vis])
    # ---- images: CUDA expf vs glibc expf differ by ~1 ulp -> 1e-5; tolerance of the task 1e-4 --
    for name, tol in (("color", 1e-5), ("opacity", 1e-5), ("depth", 5e-5), ("feature", 5e-5)):
        if g["out_" + name].size:
            assert np.abs(img[name] - g["out_" + name]).max() < tol, name
    assert np.abs(img["weights"] - g["out_weights"]).max() < 1e-4
    assert (img["n_contrib"] != g["mid_n_contrib"].view(np.uint32)).mean() < 2e-3
    assert np.abs(f["surface_xyz"] - g["out_surface_xyz"]).max() < 1e-3
    # normals amplify 1-ulp depth differences where the surface is nearly flat: compare robustly
    dn = np.abs(f["normal"] - g["out_normal"]).max(axis=0)
    assert np.quantile(dn, 0.99) < 1e-3
    # ---- gradients (tolerance 1e-3 rel of the task; the reference itself is atomics-ordered) ---
    names = ["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D"]
    names += ["dL_dsh", "dL_dscales", "dL_drotations"] if mode == "sh_sr" else []
    names += ["dL_dfeatures"] if S else []
    for n in names:
        assert rel_l2(gr[n], g["grad_" + n]) < 2e-4, (n, rel_l2(gr[n], g["grad_" + n]))


def test_binning_invariants_and_stability():
    sc, cam = case_inputs(3000, 96, 80, 0, view=2, scale_boost=3.0)
    bg = torch.zeros(3)
    kw = oracle_kwargs(sc, cam, bg)
    f = oracle.rasterize_forward(shs=npy(sc.shs), scales=npy(sc.scales), rotations=npy(sc.rotations), **kw)
    b, pre = f["binned"], f["pre"]
    keys, pl, ranges = b["keys"], b["point_list"], b["ranges"]
    R = b["num_rendered"]
    assert R == int(pre["tiles_touched"].sum()) == len(keys)
    assert np.all(keys[1:] >= keys[:-1])                                   # sortedness
    same = keys[1:] == keys[:-1]
    assert np.all(pl[1:][same] > pl[:-1][same])                            # stable: ties by Gaussian index
    tiles = (keys >> np.uint64(32)).astype(np.int64)
    lens = (ranges[:, 1].astype(np.int64) - ranges[:, 0].astype(np.int64))
    assert lens.sum() == R and np.array_equal(np.bincount(tiles, minlength=len(ranges)), lens)
    dbits = (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    assert np.array_equal(dbits, pre["depths"].view(np.uint32)[pl])        # key low word = depth bits


def test_edge_cases_empty_and_culled():
    cam = case_inputs(4, 40, 24, 0)[1]
    z = lambda *s: np.zeros(s, np.float32)
    # P = 0
    f = oracle.rasterize_forward(z(0, 3), z(0, 1), npy(cam.viewmatrix), npy(cam.projmatrix), npy(cam.campos),
                                 np.array([.5, .25, 1], np.float32), 40, 24, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                 shs=z(0, 16, 3), scales=z(0, 3), rotations=z(0, 4))
    assert f["binned"]["num_rendered"] == 0
    assert np.allclose(f["img"]["color"][1], 0.25) and np.all(f["img"]["n_contrib"] == 0)
    # everything behind the camera -> culled by the z <= 0.2 test (auxiliary.h:154)
    sc, cam = case_inputs(50, 40, 24, 0)
    behind = (sc.means3D + cam.campos * 3.0)
    f = oracle.rasterize_forward(npy(behind), npy(sc.opacities), npy(cam.viewmatrix), npy(cam.projmatrix),
                                 npy(cam.campos), z(3), 40, 24, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                 shs=npy(sc.shs), scales=npy(sc.scales), rotations=npy(sc.rotations))
    assert f["binned"]["num_rendered"] == 0 and np.all(f["pre"]["radii"] == 0)
    assert not oracle.mark_visible(npy(behind), npy(cam.viewmatrix)).any()
    assert oracle.mark_visible(npy(sc.means3D), npy(cam.viewmatrix)).all()


BVH_CASES = sorted(glob.glob(os.path.join(GOLDEN, "bvh_*.npz")))


@pytest.mark.parametrize("path", BVH_CASES, ids=[os.path.basename(p)[4:-4] for p in BVH_CASES])
def test_bvh_oracle_matches_reference_cuda_golden(path):
    """LBVH restatement vs the unmodified reference kernels: topology + Morton codes + leaf boxes
    bit-exact, internal boxes contain the reference's (whose refit is racy, see oracle_bvh.c),
    traced visibility on the reference's own tree within 1e-4 with a bounded flip rate."""
    g = np.load(path)
    nodes, aabbs, morton = oracle.bvh_build(g["in_means3D"], g["in_scales"], g["in_rotations"])
    P = morton.shape[0]
    assert np.array_equal(morton, g["morton"].view(np.uint64))
    assert np.array_equal(nodes, g["nodes"])
    assert np.array_equal(aabbs[P - 1:].view(np.uint32), g["aabbs"][P - 1:].view(np.uint32))
    assert (aabbs[:P - 1, :3] <= g["aabbs"][:P - 1, :3]).all() and (aabbs[:P - 1, 3:] >= g["aabbs"][:P - 1, 3:]).all()
    assert nodes[0, 4] == P and (nodes[1:, 0] >= 0).all() and (np.diff(morton.astype(np.int64)) > 0).all()
    cont, vis = oracle.bvh_trace_opacity(g["nodes"], g["aabbs"], g["in_rays_o"], g["in_rays_d"], g["in_means3D"],
                                         g["in_inv_cov"], g["in_opacity"], g["in_normals"])
    flips = ((vis == 0) != (g["visibility"] == 0)).mean()
    same = (vis == 0) == (g["visibility"] == 0)
    assert flips <= 5e-3, flips
    assert np.abs(vis - g["visibility"])[same].max() <= 1e-4
    assert (cont != g["contribute"])[same].mean() <= 5e-3


SHADING_CASES = sorted(glob.glob(os.path.join(GOLDEN, "shading_*.npz")))


@pytest.mark.parametrize("path", SHADING_CASES, ids=[os.path.basename(p)[8:-4] for p in SHADING_CASES])
def test_shading_oracle_matches_reference_function_golden(path):
    """PyTorch restatement of rendering_equation / GGX_specular / direct_light vs outputs and autograd
    gradients of the reference's own function bodies (make_golden_shading.py)."""
    from oracle import oracle_shading as osh
    g = np.load(path)
    t = lambda k: torch.from_numpy(g["in_" + k])
    leaves = {k: t(k).clone().requires_grad_(True) for k in ("base_color", "roughness", "viewdirs", "incidents", "env_raw")}
    env_tex = F.softplus(leaves["env_raw"])[0]
    pbr, ex = osh.rendering_equation(leaves["base_color"], leaves["roughness"], t("normals"), leaves["viewdirs"],
                                     leaves["incidents"], env_tex, t("visibility"), t("incident_dirs"), t("incident_areas"))
    np.testing.assert_allclose(pbr.detach().numpy(), g["pbr"], rtol=1e-5, atol=1e-6)
    for k in ("incident_lights", "local_incident_lights", "global_incident_lights", "diffuse_light", "specular"):
        np.testing.assert_allclose(ex[k].detach().numpy(), g["x_" + k], rtol=1e-5, atol=1e-6)
    ((pbr * t("cot_pbr")).sum() + (ex["diffuse_light"] * t("cot_diffuse")).sum() + (ex["specular"] * t("cot_specular")).sum()).backward()
    for k, v in leaves.items():
        assert rel_l2(v.grad.numpy(), g["grad_" + k]) < 1e-5, k


def test_adam_oracle_matches_torch_adam():
    """oracle_adam restates torch's `_single_tensor_adam`; pin it against torch.optim.Adam run here
    on CPU with the reference's settings (lr per group, eps=1e-15; scene/gaussian_model.py:489)."""
    import torch
    from oracle import oracle_adam
    g = torch.Generator().manual_seed(3)
    shapes, lrs = [(1000, 3), (1000, 15, 3), (1000, 1)], [1.6e-4, 2.5e-3 / 20, 5e-2]
    params = [torch.randn(s, generator=g).requires_grad_(True) for s in shapes]
    opt = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(params, lrs)], lr=0.0, eps=1e-15)
    ours = [(p.detach().numpy().copy(), np.zeros(s, np.float32), np.zeros(s, np.float32)) for p, s in zip(params, shapes)]
    p0 = [o[0].copy() for o in ours]
    for step in range(1, 8):
        grads = [torch.randn(s, generator=g) * (0.0 if (step == 3 and i == 0) else 1e-3) for i, s in enumerate(shapes)]
        grads[1][::2] = 0.0                                  # never-seen Gaussians: exp_avg_sq stays 0, eps decides
        if step == 5:
            opt.param_groups[0]["lr"] = lrs[0] = 1.0e-4      # update_learning_rate (gaussian_model.py:499-505)
        for p, gr in zip(params, grads):
            p.grad = gr.clone()
        opt.step()
        ours = [oracle_adam.adam_step(o[0], gr.numpy(), o[1], o[2], step, lr, eps=1e-15) for o, gr, lr in zip(ours, grads, lrs)]
    for p, o, q0 in zip(params, ours, p0):
        st = opt.state[p]
        # parameters are O(1): a last-ulp difference of one update is 6e-8 absolute, 7 updates accumulate a few
        np.testing.assert_allclose(o[0], p.detach().numpy(), rtol=1e-6, atol=1e-7)
        assert np.linalg.norm(o[0] - p.detach().numpy()) <= 1e-5 * np.linalg.norm(p.detach().numpy() - q0)
        np.testing.assert_allclose(o[1], st["exp_avg"].numpy(), rtol=2e-6, atol=1e-6 * float(st["exp_avg"].abs().max()))   # a signed sum: cancellation
        np.testing.assert_allclose(o[2], st["exp_avg_sq"].numpy(), rtol=2e-6, atol=1e-18)


def test_sh_gradient_factorisation_identity():
    """The multi-GPU exchange rebuilds mean_v(dL_dsh_v) from per-view factors: check the identity on
    the C oracle's own backward for two views (dense per-view dL_dsh vs the rebuilt one)."""
    from relightable3dgaussian_b200 import synth
    P, W, H, S = 3000, 96, 64, 2
    sc = synth.make_scene(P, "shell-v1", 0, S)
    n = lambda t: t.numpy()
    bg = np.zeros(3, np.float32)
    rng = np.random.default_rng(5)
    dense, factors, campos = 0, [], []
    for v in (1, 5):
        cam = synth.make_camera(v, W, H)
        f = oracle.rasterize_forward(n(sc.means3D), n(sc.opacities), n(cam.viewmatrix), n(cam.projmatrix), n(cam.campos), bg, W, H,
                                     cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, shs=n(sc.shs), scales=n(sc.scales),
                                     rotations=n(sc.rotations), features=n(sc.features))
        cots = [rng.standard_normal((c, H, W)).astype(np.float32) for c in (3, 1, 1, S)]
        g = oracle.rasterize_backward(f, n(sc.means3D), n(cam.viewmatrix), n(cam.projmatrix), n(cam.campos), bg, W, H,
                                      cam.tanfovx, cam.tanfovy, *cots, shs=n(sc.shs), scales=n(sc.scales),
                                      rotations=n(sc.rotations), features=n(sc.features))
        dense = dense + g["dL_dsh"] / 2
        factors.append(oracle.sh_grad_factor(g, f)); campos.append(n(cam.campos))
        assert (f["pre"]["clamped"] != 0).any() and (f["pre"]["radii"] > 0).any()       # the gate is exercised
    rebuilt = oracle.sh_grad_from_factors(n(sc.means3D), campos, factors, 3, 16, 0.5)
    assert np.abs(dense).max() > 0
    np.testing.assert_allclose(rebuilt, dense, rtol=2e-5, atol=1e-6 * np.abs(dense).max())


def test_adam_oracle_matches_committed_torch_fixture():
    """Same pin as above, against the committed fixture (tests/golden/make_golden_adam.py ran
    torch.optim.Adam here): travels to boxes regardless of their torch build."""
    from helpers import adam_case
    from oracle import oracle_adam
    g = np.load(os.path.join(GOLDEN, "adam_steps.npz"))
    params, lrs, grads_for_step, lr_edits = adam_case()
    st = [(p.copy(), np.zeros_like(p), np.zeros_like(p)) for p in params]
    lrs = list(lrs)
    for step in range(1, 8):
        for gi, lr in lr_edits.get(step, []):
            lrs[gi] = lr
        st = [oracle_adam.adam_step(s[0], gr, s[1], s[2], step, lr, eps=1e-15) for s, gr, lr in zip(st, grads_for_step(step), lrs)]
    for i, s in enumerate(st):
        assert float(g[f"step{i}"]) == 7.0
        np.testing.assert_allclose(s[0], g[f"p{i}"], rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(s[1], g[f"m{i}"], rtol=2e-6, atol=1e-6 * float(np.abs(g[f"m{i}"]).max()))
        np.testing.assert_allclose(s[2], g[f"v{i}"], rtol=2e-6, atol=1e-18)


def test_sampling_oracle_pinned_to_reference_functions():
    """oracle/oracle_sampling.py == the reference's own rotation_between_z / fibonacci_sphere_sampling
    (tests/golden/sampling.npz, generated by executing the reference modules: make_golden_sampling.py)."""
    from oracle import oracle_sampling as osamp
    g = np.load(os.path.join(GOLDEN, "sampling.npz"))
    n = torch.from_numpy(g["normals"])
    assert np.array_equal(osamp.rotation_between_z(n).numpy(), g["R"])
    for N in (24, 32, 100):
        d, a = osamp.fibonacci_sphere_sampling(n, N, random_rotate=False)
        assert np.array_equal(d.numpy(), g[f"dirs_{N}"]) and np.array_equal(a.numpy(), g[f"areas_{N}"])
    d, _ = osamp.fibonacci_sphere_sampling(n, 32, random_rotate=True, phase=torch.from_numpy(g["phase"]))
    assert np.array_equal(d.numpy(), g["dirs_32_random"])
    # inverse covariance: Sigma^-1 Sigma == I for the restated helper
    s = torch.rand(50, 3) * 0.5 + 0.1
    q = torch.nn.functional.normalize(torch.randn(50, 4), dim=-1)
    ic = osamp.inverse_covariance(s, q)
    R = osamp.build_rotation(q)
    cov = R @ torch.diag_embed(s * s) @ R.transpose(1, 2)
    full = torch.stack([ic[:, 0], ic[:, 1], ic[:, 2], ic[:, 1], ic[:, 3], ic[:, 4], ic[:, 2], ic[:, 4], ic[:, 5]], -1).view(-1, 3, 3)
    assert torch.allclose(full @ cov, torch.eye(3).expand(50, 3, 3), atol=1e-4)

#!/usr/bin/env python3
"""Generates tests/golden/live_*.npz on a GPU from the UNMODIFIED reference CUDA code in oracle/_ref
(oracle/build_ref.sh: the reference kernels behind a raw-pointer shim; oracle/build_ref_ext.sh: the
reference's own pybind modules and Python wrappers):

    python tests/golden/make_golden_live.py <outdir>      # then copy <outdir>/live_*.npz into tests/golden/
    python tests/golden/make_golden_live.py --only edge <outdir>   # live_raster_edge.npz alone (needs only
                                                                   # oracle/_ref/libref_raster.so)

The inputs are not stored: every case is regenerated from its seed by relightable3dgaussian_b200.synth.
What the parity tests compared against the live reference is stored compactly:
  * integer outputs (radii, tile / sort lists, ranges, n_contrib, BVH topology): sha256 of the values,
    so the comparison stays bit-exact;
  * images: every channel at a fixed, seeded sample of pixels (the test checks max-abs there) and a
    random-sign sketch of the whole image (relative L2 over every pixel);
  * gradients: a 32-row random-sign sketch (tests/helpers.py:sketch) of every gradient tensor, which
    estimates the relative L2 error over all elements;
  * visibility and sampled directions: a fixed, seeded sample of rays.
The `edge` group (tests/helpers.py EDGE_CASES) also stores final_T bit-exact (sha256 of its int32 view), the bits
of depths / means2D / conic_opacity of the visible Gaussians, and noise_<grad>: the largest relative L2 gap between
the first of four backward runs of the reference and the others, i.e. its own atomic-order noise on these
ill-conditioned cases.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from helpers import EDGE_CASES, bvh_case, case_inputs, digest, edge_case, fixed_sample, npy, oracle_kwargs, raster_key, rel_l2, sketch  # noqa: E402
from oracle import ref_gpu  # noqa: E402

IMAGES = ("color", "opacity", "depth", "feature", "normal", "surface_xyz")
GRADS = ["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dfeatures", "dL_dcov3D", "dL_dsh",
         "dL_dscales", "dL_drotations"]
N_PIX = 64

# (P, W, H, S, view, center_shift, backward, sh_degree, M, scale_boost) of tests/test_raster_gpu.py
RASTER_CASES = [(200_000, 640, 480, 5, 5, True, True, 3, 16, 1.0),
                (300_000, 800, 800, 0, 1, False, False, 3, 16, 1.0),
                (300_000, 800, 800, 0, 2, False, True, 3, 16, 1.0),
                (1_000_000, 800, 800, 5, 0, False, True, 3, 16, 1.0),
                (1_500_000, 1600, 1200, 16, 3, True, True, 3, 16, 1.0),
                (2_000_000, 1920, 1080, 16, 6, False, True, 3, 16, 1.0)]
RASTER_CASES += [(6_000, 208, 144, S, S % 8, bool(S & 1), S <= 24, 3, 16, 2.0) for S in (1, 3, 7, 9, 12, 13, 17, 20, 21, 24, 28, 33)]
RASTER_CASES += [(9_000, 200, 136, 5, deg + 2, False, True, deg, M, 1.5) for deg, M in ((0, 1), (1, 4), (2, 9), (3, 16), (1, 16), (0, 16))]


def image_samples(out, H, W, seed, prefix, rec, names=IMAGES):
    pix = fixed_sample(H * W, N_PIX, seed)
    rec[prefix + "pix"] = pix
    for n in names:
        t = out[n]
        if t.numel():
            rec[prefix + "img_" + n] = npy(t.reshape(t.shape[0], -1)[:, torch.from_numpy(pix).to(t.device)])
            rec[prefix + "sk_img_" + n] = sketch(t)


def raster_live(rec):
    dev = lambda t: t if t is None else torch.as_tensor(t).cuda()
    for (P, W, H, S, view, shift, bwd, deg, M, boost) in RASTER_CASES:
        key = raster_key(P, W, H, S, view, shift, bwd, deg, M, boost) + "__"
        sc, cam = case_inputs(P, W, H, S, view=view, center_shift=shift, scale_boost=boost)
        kw = oracle_kwargs(sc, cam, torch.tensor([0.0, 0.5, 1.0]))
        extra = dict(shs=np.ascontiguousarray(npy(sc.shs)[:, :M]), scales=npy(sc.scales), rotations=npy(sc.rotations),
                     features=npy(sc.features) if S else None, sh_degree=deg)
        g = torch.Generator().manual_seed(2)
        cots = [torch.randn(c, H, W, generator=g) for c in (3, 1, 1, S)] if bwd else None
        ref = ref_gpu.RefRasterizer()
        tk = {k: (dev(v) if isinstance(v, np.ndarray) else v) for k, v in {**kw, **extra}.items() if v is not None}
        ro = ref.forward(**tk)
        rec[key + "num_rendered"] = ro["num_rendered"]
        rec[key + "dig_radii"] = digest(ro["radii"])
        for n in ("tiles_touched", "point_list", "point_list_keys", "ranges", "n_contrib"):
            rec[key + "dig_" + n] = digest(ref.intermediate(n))
        image_samples(ro, H, W, P + S, key, rec)
        gi = fixed_sample(P, N_PIX, P + 1)
        rec[key + "weights_idx"] = gi
        rec[key + "weights"] = npy(ro["weights"])[gi]
        rec[key + "weights_absmax"] = float(ro["weights"].abs().max())
        rec[key + "sk_weights"] = sketch(ro["weights"])
        if bwd:
            rg = ref.backward(ro, dL_dcolor=dev(cots[0]), dL_dopacity=dev(cots[1]), dL_ddepth=dev(cots[2]), dL_dfeature=dev(cots[3]),
                              **{k: v for k, v in tk.items() if k in ("means3D", "viewmatrix", "projmatrix", "campos", "bg",
                                                                      "tan_fovx", "tan_fovy", "shs", "scales", "rotations", "features", "sh_degree")})
            for n in GRADS:
                if rg[n].numel() and float(rg[n].abs().max()) > 0:
                    rec[key + "sk_" + n] = sketch(rg[n])
        print(f"[golden] raster {key[:-2]}: R={ro['num_rendered']}", flush=True)
        del ref
        torch.cuda.empty_cache()


def edge_live(rec):
    dev = lambda t: t if t is None else torch.as_tensor(t).cuda()
    for name in EDGE_CASES:
        key = name + "__"
        kw, cots = edge_case(name)
        P, W, H = kw["means3D"].shape[0], kw["W"], kw["H"]
        tk = {k: (dev(v) if isinstance(v, np.ndarray) else v) for k, v in kw.items() if v is not None}
        ref = ref_gpu.RefRasterizer()
        ro = ref.forward(**tk)
        rec[key + "num_rendered"] = ro["num_rendered"]
        rec[key + "dig_radii"] = digest(ro["radii"])
        for n in ("tiles_touched", "point_list", "point_list_keys", "ranges", "n_contrib"):
            rec[key + "dig_" + n] = digest(ref.intermediate(n))
        rec[key + "dig_final_T"] = digest(ref.intermediate("final_T").view(torch.int32))
        vis = ro["radii"] > 0
        for n in ("depths", "means2D", "conic_opacity"):
            rec[key + "dig_" + n] = digest(ref.intermediate(n)[vis].contiguous().view(torch.int32))
        image_samples(ro, H, W, P + 7, key, rec)
        gi = fixed_sample(P, N_PIX, P + 1)
        rec[key + "weights_idx"] = gi
        rec[key + "weights"] = npy(ro["weights"])[gi]
        rec[key + "weights_absmax"] = float(ro["weights"].abs().max())
        rec[key + "sk_weights"] = sketch(ro["weights"])
        bk = {k: v for k, v in tk.items() if k in ("means3D", "viewmatrix", "projmatrix", "campos", "bg", "tan_fovx", "tan_fovy",
                                                    "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp", "features",
                                                    "sh_degree", "scale_modifier")}
        cd = [dev(c) for c in cots]
        runs = [ref.backward(ro, dL_dcolor=cd[0], dL_dopacity=cd[1], dL_ddepth=cd[2], dL_dfeature=cd[3], **bk) for _ in range(4)]
        for n in GRADS:
            a = runs[0][n]
            if a.numel() and float(a.abs().max()) > 0:
                rec[key + "sk_" + n] = sketch(a)
                rec[key + "noise_" + n] = max(rel_l2(npy(r[n]), npy(a)) for r in runs[1:])
        print(f"[golden] edge {name}: R={ro['num_rendered']}", flush=True)
        del ref
        torch.cuda.empty_cache()


def dropin_live(rec):
    from test_dropin_gpu import BAKE_CASES, DROPIN_CASES, bvh_scene, render_through_wrapper, sampling_normals, sampling_pairs
    from oracle import oracle_sampling
    mod = ref_gpu.load_reference_wrapper("raster", "ref")
    for P, W, H, S in DROPIN_CASES:
        key = f"raster_P{P}_S{S}__"
        sc, cam = case_inputs(P, W, H, S, view=4, center_shift=True)
        g = torch.Generator().manual_seed(3)
        cots = [torch.randn(c, H, W, generator=g) for c in (3, 1, 1, S)]
        ro, rg = render_through_wrapper(mod, sc, cam, S, torch.tensor([0.3, 0.1, 0.7]), cots)
        rec[key + "num_rendered"] = ro["num_rendered"]
        for n in ("radii", "num_contrib", "visible"):
            rec[key + "dig_" + n] = digest(ro[n])
        image_samples(ro, H, W, P + S, key, rec)
        for n, t in rg.items():
            rec[key + "sk_" + n] = sketch(t)
        print(f"[golden] dropin raster P={P} S={S}", flush=True)
    # the reference RayTracer: topology / Morton codes and a ray sample of its visibility
    bvh = ref_gpu.load_reference_wrapper("bvh", "ref")
    xyz, s, r, op, nrm = bvh_scene(30_000)
    icov = oracle_sampling.inverse_covariance(s, r)
    rt = bvh.RayTracer(xyz, s, r)
    for n in ("tree", "morton"):
        if getattr(rt, n, None) is not None:
            rec["tracer__dig_" + n] = digest(getattr(rt, n))
    dirs, _ = oracle_sampling.sample_incident_rays(nrm, False, 24)
    vis = rt.trace_visibility(xyz[:, None].expand_as(dirs), dirs, xyz, icov, op, nrm)["visibility"].reshape(-1)
    idx = fixed_sample(vis.numel(), 4096, 24)
    rec["tracer__ray_idx"], rec["tracer__visibility"] = idx, npy(vis)[idx]
    # the reference's fibonacci_sphere_sampling (utils/graphics_utils.py), deterministic and randomly rotated
    sys.path.insert(0, os.path.join(os.path.dirname(ref_gpu.__file__), "_ref", "py"))
    from utils.graphics_utils import fibonacci_sphere_sampling as ref_fib
    nrm = sampling_normals()
    for N in (24, 32, 384):
        d, a = ref_fib(nrm, N, random_rotate=False)
        idx = sampling_pairs(nrm.shape[0], N)
        rec[f"sampling__idx_{N}"] = idx
        rec[f"sampling__dirs_{N}"] = npy(d).reshape(-1, 3)[idx]
        rec[f"sampling__dig_areas_{N}"] = digest(a.contiguous().view(torch.int32))
        rec[f"sampling__shape_{N}"] = np.array(d.shape)
    torch.manual_seed(5)
    d, _ = ref_fib(nrm, 32, random_rotate=True)
    rec["sampling__dirs_rot32"] = npy(d).reshape(-1, 3)[sampling_pairs(nrm.shape[0], 32)]
    # the reference's visibility bake (its tree, PyTorch sampling, its trace kernel, its chunk loop)
    for P, N in BAKE_CASES:
        xyz, s, r, op, nrm = bvh_scene(P)
        icov = oracle_sampling.inverse_covariance(s, r)
        rvis, rdirs, rareas, _ = ref_gpu.reference_update_visibility(xyz, s, r, icov, op, nrm, N)
        key = f"bake_P{P}_N{N}__"
        idx = fixed_sample(P * N, 4096, P + N)
        rec[key + "ray_idx"] = idx
        rec[key + "visibility"] = npy(rvis).reshape(-1)[idx]
        rec[key + "dirs"] = npy(rdirs).reshape(-1, 3)[idx]
        rec[key + "dig_areas"] = digest(rareas.contiguous().view(torch.int32))
        rec[key + "blocked"] = float((rvis == 0).float().mean())
        print(f"[golden] bake P={P} N={N}", flush=True)


def bvh_live(rec):
    c = bvh_case("cube-v1", 20_000, 600, 48, 2.0, seed=5)
    d = {k: v.cuda() for k, v in c.items()}
    rn, ra, rm = ref_gpu.ref_bvh_create(d["means3D"], d["scales"], d["rotations"])
    P = d["means3D"].shape[0]
    rec["cube20k__dig_nodes"] = digest(rn)
    rec["cube20k__dig_morton"] = digest(rm.contiguous().view(torch.int64))
    rec["cube20k__dig_leaf_aabbs"] = digest(ra[P - 1:].contiguous().view(torch.int32))
    # the reference's internal boxes where its racy refit left them short of the exact bottom-up boxes
    from oracle import oracle
    exact = torch.from_numpy(oracle.bvh_build(npy(c["means3D"]), npy(c["scales"]), npy(c["rotations"]))[1]).cuda()
    stale = torch.nonzero((ra[:P - 1] != exact[:P - 1]).any(dim=1)).reshape(-1)
    rec["cube20k__stale_idx"], rec["cube20k__stale_aabbs"] = npy(stale), npy(ra[stale])
    rc, rv = ref_gpu.ref_bvh_trace_opacity(rn, ra, d["rays_o"], d["rays_d"], d["means3D"], d["inv_cov"], d["opacity"], d["normals"])
    idx = fixed_sample(rv.numel(), 8192, 20)
    rec["cube20k__ray_idx"] = idx
    rec["cube20k__visibility"] = npy(rv).reshape(-1)[idx]
    rec["cube20k__contribute"] = npy(rc).reshape(-1)[idx]
    print("[golden] bvh cube20k", flush=True)


GROUPS = {"bvh": ("live_bvh", bvh_live), "dropin": ("live_dropin", dropin_live), "raster": ("live_raster", raster_live),
          "edge": ("live_raster_edge", edge_live)}


def main(outdir, only=None):
    os.makedirs(outdir, exist_ok=True)
    assert ref_gpu.available()
    if only is None:
        assert ref_gpu.bvh_available() and ref_gpu.ext_available("raster") and ref_gpu.ext_available("bvh")
    for name, fn in [GROUPS[g] for g in (only or GROUPS)]:
        rec = {}
        fn(rec)
        path = os.path.join(outdir, name + ".npz")
        rec = {k: np.asarray(v) for k, v in rec.items()}
        np.savez_compressed(path, **{k: v.astype(np.int32) if v.dtype == np.int64 else v for k, v in rec.items()})
        print(f"[golden] {path}: {os.path.getsize(path)} bytes", flush=True)


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir", nargs="?", default=HERE)
    ap.add_argument("--only", action="append", choices=sorted(GROUPS), help="generate only these groups (repeatable)")
    a = ap.parse_args()
    main(a.outdir, a.only)

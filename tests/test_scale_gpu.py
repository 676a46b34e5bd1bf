"""Real-scene sizes against exact truths: the paths that only millions of Gaussians, 4K images, large grids and many
parameter tensors reach (tests/test_scale_cpu.py restates the launchers' thresholds and pins the truths).

  * depth sort + binning with more 2048-pair sort tiles than sort CTAs (8 x SMs), so each CTA walks several tiles:
    tile lists bit-exact against the CPU oracle, images against its renderer, gradients at 3M / 1080p;
  * 4K binning, where bin_scatter reads the chunks' first slots from the count matrix, and 8K, which is refused;
  * the BVH and the kNN on the same multi-tile Morton sorts, and the kNN on degenerate clouds against fp64 cKDTree;
  * TSDF extraction over more than 1024 blocks (two rounds of the 64-bit block-sum scan);
  * a FusedAdam step over 40 tensors (three tables of 16).

Every case derives its threshold from the device (SMS = multiprocessor count, T1 = 8 * SMS * 2048) and asserts that it
reached the path it is named for.  Peak device memory stays below ~6 GB per case (the 4K case, 232M instances).

Measured on an H100 80GB HBM3 (SXM, 132 SMs, 700 W limit): the file takes about 3 minutes, most of it the CPU oracle
and the scene generation.  Per case: 4K 38 s, 3M / 1080p with the backward 30 s, the 6M raster 12 s, the 6M BVH 9 s,
the other raster and BVH sizes 3-9 s each, the 3M kNN 5 s, TSDF 4 s, every other case under 2 s.  The CPU oracle alone,
timed on an 8-thread host: 6M Gaussians at 800 x 800 about 8 s (48M instances), 3M at 3840 x 2160 about 33 s (232M
instances), the 6M BVH build 3 s."""
import numpy as np
import pytest
import torch

from helpers import bvh_case, case_inputs, edge_case, edge_coverage, npy, oracle_kwargs, rel_l2
from test_bvh_gpu import build_ours, check_tree, compare_vis
from test_raster_gpu import GRADS, _assert_close_up_to_flips, _our_edge_stats, run_ours
from test_scale_cpu import (EX_TILE, KNN_BOX, KNN_FEW, adam_launches, bin_plan, extract_plan, knn_truth, one_wave,
                            sort_grid)
from test_tsdf_gpu import _check_extract

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from relightable3dgaussian_b200 import _C_raster
    assert torch.cuda.is_available()
    return _C_raster


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


SIZES = {"T1": lambda t1: t1, "T1+1": lambda t1: t1 + 1, "T1+2049": lambda t1: t1 + 2049,
         "2T1+5": lambda t1: 2 * t1 + 5, "3M": lambda t1: 3_000_000, "6M": lambda t1: 6_000_000}


def _sort_path(P, sms, full_wave_ok=False):
    """Assert that a sort of P pairs walks more than one tile in some CTA (or, with full_wave_ok, exactly fills the
    wave); returns a line for the log."""
    ctas, ntiles = sort_grid(P, sms)
    if full_wave_ok and P == one_wave(sms):
        assert ntiles == ctas == 8 * sms
    else:
        assert ntiles > ctas == 8 * sms, (P, ntiles, ctas)
    return f"P={P}: {ntiles} sort tiles over {ctas} CTAs (up to {-(-ntiles // ctas)} per CTA)"


def _lists_match_oracle(o, f):
    """Tile lists bit-exact against the oracle, plus the GPU-only invariants: sorted keys, stable ties."""
    b = f["binned"]
    R = o["num_rendered"]
    assert R == b["num_rendered"] > 0
    keys, pl = o["mid"]("point_list_keys"), o["mid"]("point_list")
    assert bool((keys[1:] >= keys[:-1]).all())
    same = keys[1:] == keys[:-1]
    assert bool((pl[1:][same] > pl[:-1][same]).all())                   # equal keys: ascending Gaussian index
    assert np.array_equal(npy(keys).view(np.uint64), b["keys"])
    assert np.array_equal(npy(pl).view(np.uint32), b["point_list"])
    assert np.array_equal(npy(o["mid"]("ranges")).view(np.uint32), b["ranges"])
    return R


def _images_match_oracle(o, f, names=("color", "opacity", "depth")):
    err = {}
    for n in names:
        _assert_close_up_to_flips(npy(o[n]), f["img"][n], n)
        err[n] = float(np.abs(npy(o[n]) - f["img"][n]).max())
    return err


def _shell_forward(C, P, W, H, view, S=0):
    from oracle import oracle
    sc, cam = case_inputs(P, W, H, S, view=view)
    kw = oracle_kwargs(sc, cam, torch.tensor([0.1, 0.0, 0.3]))
    kw.update(shs=npy(sc.shs), scales=npy(sc.scales), rotations=npy(sc.rotations), features=npy(sc.features) if S else None)
    del sc
    return kw, oracle.rasterize_forward(computer_pseudo_normal=False, **kw)


@pytest.mark.parametrize("size", ["T1", "T1+1", "T1+2049", "2T1+5", "6M"])
def test_depth_sort_and_binning_beyond_one_wave(C, sms, size):
    P = SIZES[size](one_wave(sms))
    path = _sort_path(P, sms, full_wave_ok=True)
    kw, f = _shell_forward(C, P, 800, 800, view=1)
    o = run_ours(C, pseudo=False, **kw)
    R = _lists_match_oracle(o, f)
    err = _images_match_oracle(o, f)
    print(f"\n[scale] depth sort {size}: {path}; R={R} bit-exact; image max-abs {err}")
    del o
    torch.cuda.empty_cache()


def test_gradients_at_3M_1080p(C, sms):
    """3M Gaussians at 1920 x 1080: multi-tile sort, chunks longer than 2048, and the whole backward at the
    north-star tolerance (1e-3 relative L2 for every gradient), as the live-reference parity cases hold it."""
    from oracle import oracle
    P, W, H, S = 3_000_000, 1920, 1080, 5
    path = _sort_path(P, sms)
    plan = bin_plan(P, W, H)
    assert plan["chunk_len"] > 2048
    kw, f = _shell_forward(C, P, W, H, view=6, S=S)
    rng = np.random.default_rng(5)
    cots = [rng.standard_normal((c, H, W)).astype(np.float32) for c in (3, 1, 1, S)]
    o = run_ours(C, pseudo=False, cots=cots, **kw)
    R = _lists_match_oracle(o, f)
    err = _images_match_oracle(o, f, ("color", "opacity", "depth", "feature"))
    bk = {k: v for k, v in kw.items() if k not in ("opacities", "cx", "cy")}
    gr = oracle.rasterize_backward(f, dL_dcolor=cots[0], dL_dopacity=cots[1], dL_ddepth=cots[2], dL_dfeature=cots[3], **bk)
    rels = {}
    for n in GRADS:
        if gr[n].size:
            rels[n] = rel_l2(npy(o["grads"][n]), gr[n])
            assert rels[n] < 1e-3, (n, rels[n])
    print(f"\n[scale] 3M 1080p: {path}; chunk {plan['chunk_len']}, R={R}; image max-abs {err}; "
          f"max gradient rel-L2 {max(rels.values()):.2e}")
    del o
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", ["depth-equal", "depth-adjacent", "depth-narrow", "depth-3to5", "depth-wide"])
def test_every_sort_plan_beyond_one_wave(C, sms, name):
    """The depth family of tests/helpers.py (0, 1, 2, 3 and 4 radix passes; all depths equal is 0 passes and the
    identity order) at T1 + 1 Gaussians."""
    from oracle import oracle
    P = one_wave(sms) + 1
    path = _sort_path(P, sms)
    kw, _ = edge_case(name, P)
    o = run_ours(C, **kw)
    f = oracle.rasterize_forward(**kw)
    stats = _our_edge_stats(o, kw)
    edge_coverage(name, stats)                             # the plan it is named for
    R = _lists_match_oracle(o, f)
    err = _images_match_oracle(o, f)
    print(f"\n[scale] {name}: {path}; {stats['passes']} passes of {stats['w']} bits; R={R}; image max-abs {err}")


def test_4k_binning_reads_chunk_starts_from_the_count_matrix(C, sms):
    P, W, H = 3_000_000, 3840, 2160
    path = _sort_path(P, sms)
    plan = bin_plan(P, W, H)
    assert plan["supported"] and plan["starts_in_smem"] == 0, plan
    kw, f = _shell_forward(C, P, W, H, view=1)
    o = run_ours(C, pseudo=False, **kw)
    R = _lists_match_oracle(o, f)
    err = _images_match_oracle(o, f)
    print(f"\n[scale] 4K: {path}; {plan['tiles']} tiles, chunk {plan['chunk_len']}, starts_in_smem 0; R={R}; "
          f"image max-abs {err}")
    del o, f
    torch.cuda.empty_cache()


def test_8k_is_refused_before_any_launch(C):
    """7680 x 4320 is 129,600 tiles: more than the binning's 65,535, and a per-tile table larger than shared memory.
    The forward refuses it with R3DG_ERR_UNSUPPORTED from a host-side check that runs before anything is enqueued (the
    profiler sees no device activity), and the stream stays usable."""
    from torch.profiler import ProfilerActivity, profile
    P = 3_000_000
    assert not bin_plan(P, 7680, 4320)["supported"]
    sc, _ = case_inputs(P, 8, 8, 0)
    g = {k: getattr(sc, k).cuda() for k in ("means3D", "opacities", "scales", "rotations", "shs")}
    bg, feats = torch.zeros(3, device="cuda"), torch.empty((P, 0), device="cuda")
    cams = {(W, H): case_inputs(1, W, H, 0, view=1)[1] for W, H in ((7680, 4320), (1920, 1080))}
    mats = {k: [c.viewmatrix.cuda(), c.projmatrix.cuda(), c.campos.cuda()] for k, c in cams.items()}
    torch.cuda.synchronize()

    def forward(W, H):                                   # every input already on the device: only the call is profiled
        cam, (view, proj, campos) = cams[(W, H)], mats[(W, H)]
        return C.rasterize_gaussians(bg, g["means3D"], feats, torch.Tensor([]), g["opacities"], g["scales"],
                                     g["rotations"], 1.0, torch.Tensor([]), view, proj, cam.tanfovx, cam.tanfovy,
                                     cam.cx, cam.cy, H, W, g["shs"], 3, campos, False, False, False)

    def device_events(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

    def refused():
        with pytest.raises(RuntimeError, match="unsupported configuration"):
            forward(7680, 4320)
    events = device_events(refused)
    assert events == [], events
    seen = device_events(lambda: forward(1920, 1080))       # the same host path at 1080p: its kernels are seen
    assert len(seen) > 5, seen
    print(f"\n[scale] 8K refused before any launch; a 1080p forward shows {len(seen)} device events")


# ---- BVH -------------------------------------------------------------------------------------------------------------

def _trace_vs_oracle(rt, c, nodes, aabbs):
    from oracle import oracle
    from relightable3dgaussian_b200 import _C_bvh
    d = {k: v.cuda() for k, v in c.items()}
    cont, vis = _C_bvh.trace_bvh_opacity(rt.tree, rt.aabb, d["rays_o"], d["rays_d"], d["means3D"], d["inv_cov"],
                                         d["opacity"], d["normals"])
    oc, ov = oracle.bvh_trace_opacity(nodes, aabbs, npy(c["rays_o"]), npy(c["rays_d"]), npy(c["means3D"]), npy(c["inv_cov"]),
                                      npy(c["opacity"]), npy(c["normals"]))
    flips, err, cdiff = compare_vis(npy(vis).reshape(-1), npy(cont).reshape(-1), ov.reshape(-1), oc.reshape(-1))
    assert flips <= 2e-3 and err <= 1e-4 and cdiff <= 5e-3, (flips, err, cdiff)
    assert 0.02 < (ov == 0).mean() < 0.98                              # both outcomes
    return f"{ov.size} rays: blocked {(ov == 0).mean():.3f}, flip rate {flips:.1e}, max-abs {err:.1e}, contribute {cdiff:.1e}"


@pytest.mark.parametrize("size", ["T1+1", "2T1+5", "6M"])
def test_bvh_beyond_one_wave(sms, size):
    from oracle import oracle
    P = SIZES[size](one_wave(sms))
    path = _sort_path(P, sms)
    c = bvh_case("shell-v1", P, 512, 8, 2.0, seed=4)                 # 512 x 8 = 4096 rays: half into the shell,
    c["rays_d"][256:] = -c["rays_d"][256:]                             # half out of it
    c["rays_o"] = (c["means3D"][:512, None] + c["rays_d"] * 0.05).contiguous()
    rt = build_ours(c["means3D"], c["scales"], c["rotations"])
    nodes, aabbs, morton = oracle.bvh_build(npy(c["means3D"]), npy(c["scales"]), npy(c["rotations"]))
    check_tree(rt, nodes, aabbs, morton, aabbs)
    trace = _trace_vs_oracle(rt, c, nodes, aabbs)
    print(f"\n[scale] BVH {size}: {path}; nodes, Morton codes and boxes bit-exact; {trace}")
    del rt
    torch.cuda.empty_cache()


@pytest.mark.parametrize("scene", ["one-cell", "identical"])
def test_bvh_degenerate_scenes_beyond_one_wave(sms, scene):
    """90 % of the centres in one Morton cell (a shell of radius 1000 around it): inside the cell the order is the
    index order alone.  All Gaussians identical: every Morton code is equal (the bounds have zero width)."""
    from oracle import oracle
    P = one_wave(sms) + 4097
    path = _sort_path(P, sms)
    g = torch.Generator().manual_seed(21)
    if scene == "one-cell":
        n_cell = int(0.9 * P)
        # the bounds are [-1000, 1000] (+ the boxes' extent) on every axis: cell 512 spans [0, 1.953)
        cell = 0.9765625 + (torch.rand(n_cell, 3, generator=g) - 0.5) * 1e-4
        shell = torch.nn.functional.normalize(torch.randn(P - n_cell, 3, generator=g), dim=-1) * 1000.0
        shell[:6] = torch.tensor([[1e3, 0, 0], [-1e3, 0, 0], [0, 1e3, 0], [0, -1e3, 0], [0, 0, 1e3], [0, 0, -1e3]])
        perm = torch.randperm(P, generator=g)
        means = torch.cat([cell, shell])[perm].contiguous()
        in_cell = (perm < n_cell).numpy()
        scales = 1e-6 * (1.0 + torch.rand(P, 3, generator=g))
        rots = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1)
    else:
        means = torch.tensor([0.3, -0.2, 0.1]).expand(P, 3).contiguous()
        in_cell = np.ones(P, dtype=bool)
        scales = torch.tensor([0.01, 0.02, 0.03]).expand(P, 3).contiguous()
        rots = torch.tensor([0.9, 0.1, -0.3, 0.2]).expand(P, 4).contiguous()
    rt = build_ours(means, scales, rots)
    nodes, aabbs, morton = oracle.bvh_build(npy(means), npy(scales), npy(rots))
    check_tree(rt, nodes, aabbs, morton, aabbs)
    codes = npy(rt.morton).view(np.uint64) >> np.uint64(31)
    idx = (npy(rt.morton).view(np.uint64) & np.uint64(0x7fffffff)).astype(np.int64)
    assert np.unique(codes[in_cell[idx]]).size == 1                    # one Morton cell ...
    run = idx[in_cell[idx]]
    assert (np.diff(run) > 0).all()                                    # ... ordered by index alone
    print(f"\n[scale] BVH {scene}: {path}; {in_cell.sum()} Gaussians share one Morton code; tree bit-exact")
    del rt
    torch.cuda.empty_cache()


# ---- kNN -------------------------------------------------------------------------------------------------------------

def _knn_check(pts, label):
    from relightable3dgaussian_b200._C_knn import distCUDA2
    got = npy(distCUDA2(pts.cuda()))
    truth = knn_truth(npy(pts).astype(np.float64))
    assert got.shape == truth.shape and got.dtype == np.float32
    np.testing.assert_allclose(got, truth, rtol=2e-5, atol=1e-12, err_msg=label)
    assert (got[truth == 0] == 0).all(), label                        # >= 3 exact duplicates: exactly 0
    rel = np.abs(got - truth)[truth > 0] / truth[truth > 0]
    return f"max rel {rel.max() if rel.size else 0.0:.1e}, exact zeros {int((truth == 0).sum())}"


@pytest.mark.parametrize("size", ["1", "2", "3", "4", "1023", "1024", "1025", "2049", "T1+1", "3M"])
def test_knn_sizes(sms, size):
    """P <= 3 gives the reference's sentinel arithmetic (tests/test_scale_cpu.py knn_few_points); 1023 / 1024 /
    1025 / 2049 sit on either side of a 1024-point box; T1 + 1 and 3M sort their Morton codes in multi-tile CTAs."""
    from relightable3dgaussian_b200._C_knn import distCUDA2
    P = int(size) if size.isdigit() else SIZES[size](one_wave(sms))
    g = torch.Generator().manual_seed(P)
    pts = torch.randn(P, 3, generator=g)
    if P >= 1000:
        pts[: P // 4] *= 0.01                                          # a dense cluster inside the cloud
    if P <= 3:
        got = npy(distCUDA2(pts.cuda()))
        assert np.array_equal(got, np.full(P, KNN_FEW[P], np.float32)), got
        print(f"\n[scale] kNN P={P}: {got.tolist()}")
        return
    path = _sort_path(P, sms) if P > one_wave(sms) else f"P={P}: one wave"
    boxes = -(-P // KNN_BOX)
    print(f"\n[scale] kNN {size}: {path}; {boxes} boxes, last holds {P - (boxes - 1) * KNN_BOX}; "
          f"{_knn_check(pts, size)}")


def _duplicates(P, g):
    """P points, 25 % of them exact copies of another point, in groups of 2..5."""
    pts = torch.randn(P, 3, generator=g)
    perm = torch.randperm(P, generator=g).tolist()
    sizes = torch.randint(2, 6, (P,), generator=g).tolist()
    i = copies = 0
    for k in sizes:
        if copies >= P // 4:
            break
        grp = perm[i:i + k]
        pts[grp[1:]] = pts[grp[0]].clone()
        i += k
        copies += k - 1
    return pts


@pytest.mark.parametrize("case", ["duplicates", "duplicates-1025", "plane", "line", "lattice", "cluster", "far"])
def test_knn_degenerate_clouds(case):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    P = 50_000
    if case == "duplicates":
        pts = _duplicates(P, g)
    elif case == "duplicates-1025":
        pts = _duplicates(1025, g)
    elif case == "plane":                                              # z = 0: the z axis has zero width
        pts = torch.cat([torch.randn(P, 2, generator=g), torch.zeros(P, 1)], 1)
    elif case == "line":                                               # y = z = 0
        pts = torch.cat([torch.randn(P, 1, generator=g), torch.zeros(P, 2)], 1)
    elif case == "lattice":                                            # spacings 1, 2, 3: ties everywhere, shuffled
        ax = torch.arange(37, dtype=torch.float32)                    # (the 3rd neighbour: one of two at distance 2)
        pts = torch.stack(torch.meshgrid(ax, 2 * ax, 3 * ax, indexing="ij"), -1).reshape(-1, 3)
        pts = pts[torch.randperm(len(pts), generator=g)].contiguous()
    elif case == "cluster":                                            # 90 % within 1e-3, 10 % spread over 1e3
        pts = torch.rand(P, 3, generator=g) * 1e-3
        far = torch.rand(P, generator=g) < 0.1
        pts[far] = (torch.rand(int(far.sum()), 3, generator=g) - 0.5) * 1e3
    else:                                                              # extent 1 at 1e4: the bounds include the origin,
        pts = 1e4 + torch.rand(P, 3, generator=g) - 0.5                 # so a few Morton cells hold every point
    pts = pts.float().contiguous()
    msg = _knn_check(pts, case)
    if case.startswith("duplicates"):
        assert "exact zeros 0" not in msg
    print(f"\n[scale] kNN {case} ({len(pts)} points): {msg}")


# ---- TSDF extraction -------------------------------------------------------------------------------------------------

def test_tsdf_extract_beyond_one_scan_round():
    """131 x 97 x 103 = 1,308,821 grid points = 1279 blocks of 1024: the block sums are scanned in two rounds, the
    second starting from the first one's 64-bit carry.  The strides are odd, so cells straddle block boundaries.  A
    random field with zeros, -0.0 and unobserved boxes gives every block vertices, so every block moves the carry."""
    from relightable3dgaussian_b200 import tsdf
    g = torch.Generator().manual_seed(17)
    vol = tsdf.TSDFVolume((0.0, 0.0, 0.0), (1.30, 0.96, 1.02), 0.01, 0.04, device="cuda")
    assert vol.dims == (131, 97, 103)
    nblocks, rounds = extract_plan(vol.dims)
    assert nblocks > 1024 and rounds == 2
    field = torch.randn(vol.dims, generator=g)
    field[torch.rand(vol.dims, generator=g) < 0.1] = 0.0
    field[torch.rand(vol.dims, generator=g) < 0.05] = -0.0
    weight = torch.randint(1, 5, vol.dims, generator=g).float()
    for _ in range(12):                                                # unobserved boxes
        lo = [int(torch.randint(0, n - 4, (1,), generator=g)) for n in vol.dims]
        weight[lo[0]:lo[0] + 6, lo[1]:lo[1] + 9, lo[2]:lo[2] + 4] = 0.0
    vol.tsdf.copy_(field)
    vol.weight.copy_(weight)
    vol.color.copy_(torch.rand(vol.dims + (3,), generator=g))
    v, f = _check_extract(vol)
    # the grid point below each vertex (its owner, or the point across the edge when t > 0.999) -> its block
    ijk = np.floor((v - np.asarray(vol.origin)) / vol.voxel_size + 1e-3).astype(np.int64)
    ijk = np.clip(ijk, 0, np.asarray(vol.dims) - 1)
    per_block = np.bincount(np.ravel_multi_index(ijk.T, vol.dims) // EX_TILE, minlength=nblocks)
    assert per_block.min() > 0, int(per_block.argmin())
    print(f"\n[scale] TSDF {vol.dims}: {nblocks} blocks, {rounds} scan rounds; {len(v)} vertices, {len(f)} faces "
          f"bit-exact; fewest vertices in a block {per_block.min()}")


# ---- FusedAdam -------------------------------------------------------------------------------------------------------

def test_adam_splits_40_tensors_into_tables_of_16():
    """40 parameter tensors, 7 of them empty (they take no table slot) and 3 unaligned views: ceil(33 / 16) = 3
    launches per step, against torch.optim.Adam and the numpy oracle at tests/test_adam_gpu.py's tolerances.  A step
    without two of the gradients has 31 non-empty tensors among 38 entries: 2 launches."""
    from oracle import oracle_adam
    from relightable3dgaussian_b200 import _lib
    from relightable3dgaussian_b200.optim import FusedAdam
    cycle = [1, 4095, 4096, 4097, 70_000, 7, 300, 8193]
    sizes = [0 if i % 6 == 3 else cycle[i % len(cycle)] for i in range(40)]
    unaligned = {5, 17, 29}
    g = torch.Generator().manual_seed(9)
    pa, pb = [], []
    for i, n in enumerate(sizes):
        init = torch.randn(n, generator=g)
        if i in unaligned:
            base = torch.zeros(n + 1, device="cuda")
            base[1:] = init.cuda()
            p = base[1:].detach().requires_grad_(True)
            assert p.data_ptr() % 16 != 0
        else:
            p = init.cuda().requires_grad_(True)
        pa.append(p)
        pb.append(init.cuda().requires_grad_(True))
    lrs = [1e-3 * (1 + i % 5) for i in range(40)]
    oa = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(pa, lrs)], lr=0.0, eps=1e-15)
    ob = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(pb, lrs)], lr=0.0, eps=1e-15)
    p0 = [npy(p) for p in pa]
    orc = [(npy(p), np.zeros(p.shape, np.float32), np.zeros(p.shape, np.float32)) for p in pa]
    steps = [0] * 40
    lib = _lib.load()
    launches = []
    for step in range(1, 6):
        skip = {8, 20} if step == 4 else set()
        gg = torch.Generator().manual_seed(100 + step)
        for i, (p, q) in enumerate(zip(pa, pb)):
            t = torch.randn(sizes[i], generator=gg) * 1e-3
            t[1::3] = 0.0                                              # exact zeros (Gaussians out of view)
            if i in skip:
                p.grad = q.grad = None
                continue
            if i in unaligned:
                gb = torch.zeros(sizes[i] + 1, device="cuda")
                gb[1:] = t.cuda()
                p.grad = gb[1:]
            else:
                p.grad = t.cuda()
            q.grad = t.cuda()
            if sizes[i]:
                steps[i] += 1
                o = orc[i]
                orc[i] = oracle_adam.adam_step(o[0], t.numpy(), o[1], o[2], steps[i], lrs[i], eps=1e-15)
        n0 = lib.r3dg_launch_count()
        oa.step()
        torch.cuda.synchronize()
        launches.append(lib.r3dg_launch_count() - n0)
        ob.step()
        expect = adam_launches([n for i, n in enumerate(sizes) if i not in skip])
        assert launches[-1] == expect == (2 if skip else 3), (step, launches)
    for i, (p, q, o, q0) in enumerate(zip(pa, pb, orc, p0)):
        if sizes[i] == 0:
            assert p.numel() == 0
            continue
        sa, sb = oa.state[p], ob.state[q]
        assert float(sa["step"]) == float(sb["step"]) == steps[i]
        for ref_p, ref_m, ref_v, tol in ((npy(q), npy(sb["exp_avg"]), npy(sb["exp_avg_sq"]), 2e-6), (o[0], o[1], o[2], 1e-6)):
            np.testing.assert_allclose(npy(p), ref_p, rtol=1e-6, atol=2e-7, err_msg=str(i))
            assert np.linalg.norm(npy(p) - ref_p) <= 2e-5 * np.linalg.norm(ref_p - q0) + 1e-12, i
            np.testing.assert_allclose(npy(sa["exp_avg"]), ref_m, rtol=tol, atol=tol * float(np.abs(ref_m).max()), err_msg=str(i))
            np.testing.assert_allclose(npy(sa["exp_avg_sq"]), ref_v, rtol=tol, atol=1e-18, err_msg=str(i))
        assert np.array_equal(npy(sa["exp_avg_sq"]), o[2]), i
        assert not np.array_equal(npy(p), q0), i                          # every non-empty tensor moved
    print(f"\n[scale] FusedAdam, 40 tensors ({sum(n > 0 for n in sizes)} non-empty): launches per step {launches}")

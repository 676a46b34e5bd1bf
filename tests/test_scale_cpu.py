"""The truths and the path arithmetic behind tests/test_scale_gpu.py, without a GPU.

Several kernels change path only at real-scene sizes: the radix sort's CTAs walk more than one 2048-pair tile once n
exceeds 8 x SMs tiles, bin_scatter reads each chunk's first slots from the count matrix above ~1080p tile counts, the
TSDF extraction's block-sum scan carries across rounds of 1024 blocks, and a FusedAdam step splits into tables of 16
tensors.  The GPU tests decide whether a case reaches its path with the functions below, which restate the launchers'
formulas with constants read from the sources; the first test fails when a launcher's formula changes, so that the
restatement is updated with it.  The fp64 truths the GPU tests use (the kNN's cKDTree mean, the marching-cubes
oracle) are checked here against plain brute force."""
import math
import os
import re

import numpy as np
import pytest
from scipy.spatial import cKDTree

import tsdf_oracle as O
from helpers import ROOT

CSRC = os.path.join(ROOT, "relightable3dgaussian_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _define(name, path):
    return int(re.search(rf"#define {name} (\d+)", _src(path)).group(1))


def _constexpr(name, path):
    return int(re.search(rf"constexpr int {name} = (\d+);", _src(path)).group(1))


SORT_TILE = _define("R3DG_SORT_THREADS", "common.cuh") * _define("R3DG_SORT_ITEMS", "common.cuh")
BIN_MAX_CHUNKS = _define("R3DG_BIN_MAX_CHUNKS", "common.cuh")
BIN_SCATTER_THREADS = _define("BIN_SCATTER_THREADS", "binning.cu")
BIN_LONG_RUN = _define("BIN_LONG_RUN", "binning.cu")
BIN_MAX_LONG = _define("BIN_MAX_LONG", "binning.cu")
BIN_SMEM_MAX = 220 * 1024
KNN_BOX = _define("KNN_BOX", "knn.cu")
EX_TILE = _constexpr("kExThreads", "tsdf.cu") * _constexpr("kExItems", "tsdf.cu")
SCAN_ROUND = 1024                                    # block_sums_scan_kernel: one CTA of 1024 threads per round
ADAM_MAX_TENSORS = _define("ADAM_MAX_TENSORS", "adam.cu")

# The launcher lines the functions below restate, verbatim.
LAUNCHER_LINES = {
    "radix_sort.cu": ["const int grid = (int)std::min<long long>((long long)num_sms * 8, std::max<long long>(1, ntiles));",
                      "for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {"],
    "common.cuh": ["size_t c = ((size_t)1 << 26) / (T ? T : 1);",
                   "return (int)(c < 296 ? 296 : (c > R3DG_BIN_MAX_CHUNKS ? R3DG_BIN_MAX_CHUNKS : c));",
                   "int ch = ((P + 443) / 444 + 255) / 256 * 256;",
                   "ch = ch < 512 ? 512 : (ch > 2048 ? 2048 : ch);",
                   "const int need = ((P + max_chunks - 1) / max_chunks + 255) / 256 * 256;",
                   "return ch > need ? ch : need;"],
    "binning.cu": ["constexpr size_t kBinSmemMax = 220 * 1024;",
                   "return (((size_t)T + 3) & ~(size_t)3) * 4;",
                   "return bin_tile_bytes(T) + (size_t)(BIN_SCATTER_THREADS / 32) * 2 * ((CH + 31) / 32) * 4 + (size_t)CH * 12;",
                   "if (b.gx > 65535 || b.gy > 65535 || b.tiles > 65535 || CH > 65536 ||",
                   "bin_table_bytes(b.tiles, CH) + (size_t)CH * 4 > kBinSmemMax) return R3DG_ERR_UNSUPPORTED;",
                   "const size_t full_stage = std::min<size_t>((size_t)CH * 12, (size_t)BIN_MAX_LONG * BIN_LONG_RUN);",
                   "const int starts_in_smem = tbl_bytes + tile_bytes + full_stage * 4 <= smem_max ? 1 : 0;"],
    "api.cu": ["if ((rc = check_binning_limits(b)) != 0) return rc;"],
    "scan.cuh": ["for (long long base = 0; base < n; base += 1024) {"],
    "tsdf.cu": ["ExLayout(long long N) : nblocks((N + kExTile - 1) / kExTile) {",
                "block_sums_scan_kernel<2, unsigned long long><<<1, 1024, 0, stream>>>(L.nblocks, L.nblocks, sums, totals);"],
    "adam.cu": ["for (; i < num && tab.num < ADAM_MAX_TENSORS; ++i) {", "if (s.n == 0) continue;"],
    "knn.cu": ["for (int b = 0; b < nboxes; ++b) {", "const int e = min(P, (b + 1) * KNN_BOX);",
               "float best[3] = {FLT_MAX, FLT_MAX, FLT_MAX};",
               "out[__float_as_uint(me.w)] = (best[0] + best[1] + best[2]) / 3.0f;"],
}


def sort_grid(n, sms):
    """launch_sort (radix_sort.cu): (CTAs, 2048-pair tiles) of a sort of n pairs.  A CTA walks more than one tile
    exactly when tiles > CTAs, i.e. n > 8 * sms * 2048."""
    ntiles = -(-n // SORT_TILE)
    return min(8 * sms, max(1, ntiles)), ntiles


def one_wave(sms):
    """T1: the most pairs one wave of sort CTAs covers with one tile each."""
    return 8 * sms * SORT_TILE


def bin_plan(P, W, H):
    """launch_binning / raster_buffers (binning.cu, api.cu, common.cuh) for P Gaussians at W x H."""
    gx, gy = -(-W // 16), -(-H // 16)
    T = gx * gy
    max_chunks = min(max(2 ** 26 // max(T, 1), 296), BIN_MAX_CHUNKS)
    ch = min(max(((P + 443) // 444 + 255) // 256 * 256, 512), 2048)
    need = ((P + max_chunks - 1) // max_chunks + 255) // 256 * 256
    CH = max(ch, need)
    tile_bytes = (T + 3) // 4 * 4 * 4
    tbl = tile_bytes + (BIN_SCATTER_THREADS // 32) * 2 * ((CH + 31) // 32) * 4 + CH * 12
    supported = not (gx > 65535 or gy > 65535 or T > 65535 or CH > 65536 or tbl + CH * 4 > BIN_SMEM_MAX)
    full_stage = min(CH * 12, BIN_MAX_LONG * BIN_LONG_RUN)
    starts_in_smem = int(tbl + tile_bytes + full_stage * 4 <= BIN_SMEM_MAX)
    return dict(tiles=T, chunk_len=CH, chunks=-(-P // CH), supported=supported, starts_in_smem=starts_in_smem)


def extract_plan(dims):
    """TSDF extraction (tsdf.cu ExLayout, scan.cuh): (blocks of 1024 grid points, rounds of the block-sum scan)."""
    nblocks = -(-math.prod(dims) // EX_TILE)
    return nblocks, -(-nblocks // SCAN_ROUND)


def adam_launches(sizes):
    """launch_adam (adam.cu): one launch per table of 16 non-empty tensors; empty tensors take no slot."""
    return -(-sum(1 for n in sizes if n > 0) // ADAM_MAX_TENSORS)


def knn_truth(points):
    """fp64 mean squared distance to the 3 nearest other points: cKDTree's 4 nearest, minus one zero distance (the
    point itself, or an exact duplicate of it, which is the same value)."""
    p = np.asarray(points, np.float64)
    d, _ = cKDTree(p).query(p, k=4, workers=-1)
    return (d[:, 1:] ** 2).mean(axis=1)


def knn_few_points(P):
    """distCUDA2 for P <= 3 points, as simple_knn.cu's boxMeanDist computes it in fp32: best[] starts at FLT_MAX and
    the 3 - (P - 1) slots no neighbour fills keep it, so the result is (best[0] + best[1] + best[2]) / 3.0f with those
    sentinels.  P = 1: FLT_MAX + FLT_MAX overflows to inf.  P = 2: d + FLT_MAX rounds to FLT_MAX (d is far below half
    an ulp of FLT_MAX, 2^103), + FLT_MAX = inf.  P = 3: (d0 + d1) + FLT_MAX rounds to FLT_MAX, / 3 = 1.1342745e38."""
    flt_max = np.float32(np.finfo(np.float32).max)
    with np.errstate(over="ignore"):
        if P == 1:
            return np.float32(flt_max + flt_max + flt_max) / np.float32(3)
        if P == 2:
            return np.float32(np.float32(np.float32(1.0) + flt_max) + flt_max) / np.float32(3)
        return np.float32(np.float32(np.float32(1.0) + np.float32(2.0)) + flt_max) / np.float32(3)


# What tests/test_scale_gpu.py holds distCUDA2 of P <= 3 points to (derived in knn_few_points).
KNN_FEW = {1: np.inf, 2: np.inf, 3: np.float32(1.1342745e38)}


def test_launcher_formulas_are_the_ones_restated_here():
    for name, lines in LAUNCHER_LINES.items():
        src = _src(name)
        for line in lines:
            assert line in src, f"{name} no longer contains `{line}`: update the restatement in tests/test_scale_cpu.py"
    assert _src("radix_sort.cu").count(LAUNCHER_LINES["radix_sort.cu"][1]) == 2       # histogram and scatter
    assert (SORT_TILE, KNN_BOX, EX_TILE, ADAM_MAX_TENSORS, BIN_MAX_CHUNKS) == (2048, 1024, 1024, 16, 1024)


@pytest.mark.parametrize("sms", [114, 132])            # H100 PCIe, H100 SXM
def test_scale_cases_cross_their_paths_on_every_h100(sms):
    T1 = one_wave(sms)
    assert T1 == {114: 1_867_776, 132: 2_162_688}[sms]
    assert sort_grid(T1, sms) == (8 * sms, 8 * sms)                    # the full wave, one tile per CTA
    assert sort_grid(T1 + 1, sms) == (8 * sms, 8 * sms + 1)             # one CTA gets a second tile of one pair
    for n in (T1 + 2049, 2 * T1 + 5, 3_000_000, 6_000_000):
        ctas, ntiles = sort_grid(n, sms)
        assert ntiles > ctas == 8 * sms, n
    assert bin_plan(3_000_000, 3840, 2160)["supported"] and bin_plan(3_000_000, 3840, 2160)["starts_in_smem"] == 0
    assert bin_plan(2_000_000, 1920, 1080)["starts_in_smem"] == 1       # the largest raster case before this file
    assert bin_plan(3_000_000, 1920, 1080)["chunk_len"] > 2048          # > 1024 chunks' worth: chunks grow
    assert bin_plan(3_000_000, 1920, 1080)["starts_in_smem"] == 0
    assert not bin_plan(3_000_000, 7680, 4320)["supported"]             # 129,600 tiles: refused
    assert extract_plan((131, 97, 103)) == (1279, 2) and extract_plan((96, 96, 96)) == (864, 1)


def test_adam_launch_arithmetic():
    assert adam_launches([0] * 40) == 0
    assert adam_launches([1] * 16 + [0] * 30) == 1 and adam_launches([1] * 17) == 2
    assert adam_launches([5] * 33) == adam_launches([5] * 48) == 3


def _knn_bruteforce(p):
    d2 = ((p[:, None, :] - p[None, :, :]) ** 2).sum(-1)
    np.fill_diagonal(d2, np.inf)
    return np.sort(d2, axis=1)[:, :3].mean(axis=1)


@pytest.mark.parametrize("kind", ["random", "duplicates", "lattice", "plane"])
def test_knn_truth_matches_bruteforce(kind):
    rng = np.random.default_rng(3)
    if kind == "random":
        p = rng.standard_normal((700, 3))
    elif kind == "duplicates":                              # groups of 2..5 identical points
        p = rng.standard_normal((300, 3))
        p = np.repeat(p, rng.integers(1, 6, 300), axis=0)
    elif kind == "lattice":                                  # ties everywhere
        p = np.stack(np.meshgrid(*[np.arange(7.0)] * 3, indexing="ij"), -1).reshape(-1, 3)
    else:
        p = np.c_[rng.standard_normal((500, 2)), np.zeros(500)]
    p = p.astype(np.float32).astype(np.float64)
    np.testing.assert_allclose(knn_truth(p), _knn_bruteforce(p), rtol=1e-12, atol=0)
    if kind == "duplicates":
        _, inv, cnt = np.unique(p, axis=0, return_inverse=True, return_counts=True)
        assert (knn_truth(p)[cnt[inv.reshape(-1)] >= 4] == 0).all()


def test_knn_few_points_constants():
    for P in (1, 2, 3):
        assert np.array_equal(np.float32(KNN_FEW[P]), knn_few_points(P)), P
    assert np.isinf(KNN_FEW[2]) and np.isfinite(KNN_FEW[3])


def _marching_cubes_loops(tsdf, weight, origin, vs):
    """Loop-by-loop restatement of the extraction's definition (include/r3dg_b200.h): a cell is valid when its 8
    corners are observed; a point's +axis edge carries a vertex when it changes sign (inside = tsdf < 0) and some valid
    cell contains it; vertices in (point, axis) order; each valid cell's table triangles in cell order."""
    edges, count, tris = O.parse_table()
    NX, NY, NZ = tsdf.shape
    valid = lambda i, j, k: (0 <= i < NX - 1 and 0 <= j < NY - 1 and 0 <= k < NZ - 1 and
                             all(weight[i + (c & 1), j + (c >> 1 & 1), k + (c >> 2 & 1)] > 0 for c in range(8)))
    vid, verts = {}, []
    for i in range(NX):
        for j in range(NY):
            for k in range(NZ):
                for a in range(3):
                    q = (i + (a == 0), j + (a == 1), k + (a == 2))
                    if q[a] >= tsdf.shape[a] or (tsdf[i, j, k] < 0) == (tsdf[q] < 0):
                        continue
                    others = [b for b in range(3) if b != a]
                    cells = []
                    for s in (0, 1):
                        for t in (0, 1):
                            c = [i, j, k]
                            c[others[0]] -= s
                            c[others[1]] -= t
                            cells.append(valid(*c))
                    if any(cells):
                        v0, v1 = float(tsdf[i, j, k]), float(tsdf[q])
                        p = [origin[d] + vs * (i, j, k)[d] for d in range(3)]
                        p[a] += v0 / (v0 - v1) * vs
                        vid[(i, j, k, a)] = len(verts)
                        verts.append(p)
    faces = []
    for i in range(NX - 1):
        for j in range(NY - 1):
            for k in range(NZ - 1):
                if not valid(i, j, k):
                    continue
                cube = sum(int(tsdf[i + (c & 1), j + (c >> 1 & 1), k + (c >> 2 & 1)] < 0) << c for c in range(8))
                for t in range(count[cube]):
                    f = []
                    for e in tris[cube, t]:
                        c = edges[e][0]
                        f.append(vid[(i + (c & 1), j + (c >> 1 & 1), k + (c >> 2 & 1), e // 4)])
                    faces.append(f)
    return np.array(verts, np.float64).reshape(-1, 3), np.array(faces, np.int64).reshape(-1, 3)


def test_tsdf_oracle_on_an_odd_grid_matches_its_loops():
    """The vectorised oracle the TSDF scale case trusts, on a 7 x 5 x 9 grid with zeros, -0.0 and unobserved points."""
    rng = np.random.default_rng(8)
    t = rng.standard_normal((7, 5, 9)).astype(np.float32)
    t[rng.random(t.shape) < 0.15] = 0.0
    t[rng.random(t.shape) < 0.1] = -0.0
    w = (rng.random(t.shape) > 0.08).astype(np.float32)
    v, f, _ = O.marching_cubes(t, w, None, (0.5, -1.0, 2.0), 0.1)
    lv, lf = _marching_cubes_loops(t, w, (0.5, -1.0, 2.0), 0.1)
    assert len(f) > 50 and np.array_equal(f, lf)
    assert np.abs(v - lv).max() < 1e-12

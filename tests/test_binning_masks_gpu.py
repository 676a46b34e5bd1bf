"""The per-instance masks the binning scatter writes next to every list entry (csrc/binning.cu, bin_scatter):
`bmask` (which 8x4 pixel blocks of the entry's tile the Gaussian's block rectangle meets) and `cmask` (zeroed there,
then set by the forward compositor for the blocks that composited the entry).

The images and n_contrib parity tests already catch a missing bmask bit.  These tests also catch what they cannot:
a superfluous bmask bit (changes no image, only speed) and a cmask byte left over from the previous forward in a
reused binning buffer (only visible when the allocator happens to hand that buffer back)."""
import types

import numpy as np
import pytest
import torch

from helpers import EDGE_CASES, case_inputs, edge_case, npy, oracle_kwargs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from relightable3dgaussian_b200 import _C_raster
    assert torch.cuda.is_available()
    return _C_raster


def _dev(t):
    return torch.Tensor([]) if t is None else torch.as_tensor(t).cuda()


def _forward(C, kw, min_capacity=None):
    """One forward through the drop-in `_C` surface; returns the outputs and the binning intermediates."""
    k = dict(kw)
    P = k["means3D"].shape[0]
    feats = _dev(k.get("features")) if k.get("features") is not None else torch.empty((P, 0), device="cuda")
    out = C.rasterize_gaussians(_dev(k["bg"]), _dev(k["means3D"]), feats, _dev(k.get("colors_precomp")),
                                _dev(k["opacities"]), _dev(k.get("scales")), _dev(k.get("rotations")),
                                k.get("scale_modifier", 1.0), _dev(k.get("cov3D_precomp")), _dev(k["viewmatrix"]),
                                _dev(k["projmatrix"]), k["tan_fovx"], k["tan_fovy"], k["cx"], k["cy"], k["H"], k["W"],
                                _dev(k.get("shs")), k.get("sh_degree", 3), _dev(k["campos"]), False, True, False,
                                _min_capacity=min_capacity)
    R, geom, binning, img = out[0], out[10], out[11], out[12]
    S = feats.shape[1]
    mid = lambda n: npy(C.debug_intermediate(n, P, S, k["W"], k["H"], geom, img, binning, R))   # noqa: E731
    torch.cuda.synchronize()
    return dict(R=R, n_contrib=npy(out[1]), point_list=mid("point_list").view(np.uint32),
                ranges=mid("ranges").view(np.uint32), bmask=mid("bmask"), cmask=mid("cmask"),
                brects=mid("brects").view(np.uint32), binning=binning)


def _expected_bmask(point_list, ranges, brects, W):
    """numpy restatement of block_mask_of_rect (csrc/common.cuh) for every list entry: bit b = block b of the entry's
    tile (block row b >> 1, block column b & 1; blocks are 8 px wide and 4 px high) lies inside the Gaussian's
    inclusive block rectangle {bx0 | bx1 << 16, by0 | by1 << 16}."""
    gx = (W + 15) // 16
    lens = (ranges[:, 1] - ranges[:, 0]).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    nonempty = lens > 0
    assert np.array_equal(ranges[nonempty, 0].astype(np.int64), starts[nonempty])     # lists are contiguous, in tile order
    tile = np.repeat(np.arange(len(ranges), dtype=np.int64), lens)
    assert len(tile) == len(point_list)
    br = brects[point_list.astype(np.int64)].astype(np.int64)
    bx0, bx1, by0, by1 = br[:, 0] & 0xffff, br[:, 0] >> 16, br[:, 1] & 0xffff, br[:, 1] >> 16
    c0, r0 = 2 * (tile % gx), 4 * (tile // gx)
    mask = np.zeros(len(tile), np.uint8)
    for b in range(8):
        col, row = c0 + (b & 1), r0 + (b >> 1)
        hit = (bx0 <= col) & (col <= bx1) & (by0 <= row) & (row <= by1)
        mask |= hit.astype(np.uint8) << b
    return mask


def _check_masks(o, W):
    assert o["R"] > 0
    assert len(o["bmask"]) == len(o["cmask"]) == len(o["point_list"]) == o["R"]
    exp = _expected_bmask(o["point_list"], o["ranges"], o["brects"], W)
    bad = np.flatnonzero(o["bmask"] != exp)
    assert bad.size == 0, (int(bad.size), bad[:8], o["bmask"][bad[:8]], exp[bad[:8]])
    assert not (o["cmask"] & ~o["bmask"]).any()                         # only pre-filtered blocks composite an entry
    assert o["cmask"].any()


def _scene(P, W, H, S=0, view=1, boost=1.0):
    sc, cam = case_inputs(P, W, H, S, view=view, scale_boost=boost)
    kw = oracle_kwargs(sc, cam, torch.tensor([0.1, 0.0, 0.3]))
    kw.update(shs=npy(sc.shs), scales=npy(sc.scales), rotations=npy(sc.rotations),
              features=npy(sc.features) if S else None)
    return kw


@pytest.mark.parametrize("W,H,P", [(800, 800, 60_000), (1920, 1080, 20_000), (3840, 2160, 6_000)],
                         ids=["800x800", "1080p", "4k"])
def test_masks_match_block_rectangles(C, W, H, P):
    """The headline's 2500 tiles at reduced P, and the 8160 / 32400 tile tables of 1080p and 4K."""
    _check_masks(_forward(C, _scene(P, W, H, S=5 if W == 800 else 0)), W)


@pytest.mark.parametrize("name", EDGE_CASES)
def test_masks_edge_cases(C, name):
    kw, _ = edge_case(name)
    o = _forward(C, kw)
    if o["R"] == 0:
        pytest.skip("no instances")
    _check_masks(o, kw["W"])


def test_masks_multi_window(C, monkeypatch):
    """A staging area of one chunk: the scatter handles its chunks in several windows of tiles."""
    monkeypatch.setenv("R3DG_BIN_STAGE_CAP", "1")
    _check_masks(_forward(C, _scene(20_000, 320, 232, boost=1.5)), 320)


def test_masks_long_chunks(C, monkeypatch):
    """Chunks longer than 2048 Gaussians (a 3-row chunk x tile matrix)."""
    monkeypatch.setenv("R3DG_BIN_MAX_CHUNKS", "3")
    _check_masks(_forward(C, _scene(20_000, 320, 232, boost=1.5)), 320)


def test_masks_after_overflowing_first_attempt(C):
    """A binning buffer smaller than R: the forward is re-run with room to spare; the first attempt wrote only
    inside its buffer, the second attempt's masks are complete."""
    kw = _scene(30_000, 800, 800)
    R = _forward(C, kw)["R"]
    o = _forward(C, kw, min_capacity=R // 3)
    assert o["R"] == R
    _check_masks(o, 800)


def test_cmask_not_stale_in_reused_buffer(C, monkeypatch):
    """View A then view B in the same binning buffer: B's cmask equals B's cmask rendered into a zero-filled buffer."""
    kw_a, kw_b = _scene(40_000, 800, 800, view=1), _scene(40_000, 800, 800, view=2)
    cap = 2 * max(_forward(C, kw_a)["R"], _forward(C, kw_b)["R"]) + 4096
    nbytes = C._lib.load().r3dg_raster_binning_bytes(cap)
    shared = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")

    def run_into(buf, kw):
        def empty(shape, *args, **kwargs):
            if tuple(shape) == (nbytes,) and kwargs.get("dtype") is torch.uint8:
                return buf
            return torch.empty(shape, *args, **kwargs)
        shim = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith("__")})
        shim.empty = empty
        monkeypatch.setattr(C, "torch", shim)
        try:
            o = _forward(C, kw, min_capacity=cap)
        finally:
            monkeypatch.setattr(C, "torch", torch)
        assert o["binning"].data_ptr() == buf.data_ptr()
        return o

    run_into(shared, kw_a)
    b_reused = run_into(shared, kw_b)
    b_fresh = run_into(torch.zeros((nbytes,), dtype=torch.uint8, device="cuda"), kw_b)
    assert b_reused["R"] == b_fresh["R"] > 0
    for n in ("point_list", "bmask", "cmask", "n_contrib"):
        assert np.array_equal(b_reused[n], b_fresh[n]), n
    _check_masks(b_reused, 800)

"""The bilateral-grid slice (bilagrid.slice, csrc/bilagrid.cu) over grid shapes, image shapes and every backward
instantiation, against the fp64 truth of tests/bilagrid_oracle.py taken at the kernel's own fp32 coordinates.  Each
element is checked at the scale of its own terms (bilagrid_oracle.scales64), so a missing or doubled contribution to a
small gradient fails as surely as one to a large gradient:

  out         |o - o64| <= 16 eps32 m_out: three lerp levels and the affine row's fmas, a few roundings each;
  dL/drgb     |g - g64| <= 2e-5 m_drgb;
  dL/dgrids   |g - g64| <= 2e-5 m_dgrids, so exactly 0 where nothing contributes: staged nodes no pixel touches and
              grids no image id names.

No pixel is masked: at the kernel's coordinates the truth's cells, weights and border flags are the kernel's, so
dL/drgb has no jump between the two.  The cases cover: the four backward kernels <R, GRID> (R = 2 rows per lane from L = 9), each output alone; tiles that
stage exactly MAX_NODES = 1024 nodes with R = 1 and R = 2, and the shapes one node over, which are refused; grids
denser than the pixels and coarser than a tile; partial tiles, 1-pixel strips and GX != GY; many images over fewer
grids; luma below 0, inside and above 1 in every tile; unit and training-scale (L1 sign pattern) cotangents.  Last,
the C ABI with every output and the workspace inside canary padding.
"""
import numpy as np
import pytest
import torch

import bilagrid_oracle as bo
from relightable3dgaussian_b200 import _lib, bilagrid

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24
OUT_TOL = 16 * EPS32
GRAD_TOL = 2e-5
UNSUPPORTED = -10002


def make_case(G, N, H, W, L, GY, GX, cot, seed):
    """Grids at the identity plus N(0, 0.2) noise; rgb with luma spread over [-0.3, 1.3] (about one pixel in five below
    0 and one above 1, in every tile); dout unit N(0, 1) or the sign pattern of an L1 mean, +-1/(3NHW)."""
    rs = np.random.default_rng(seed)
    grids = bo.IDENTITY.reshape(1, 12, 1, 1, 1) + 0.2 * rs.standard_normal((G, 12, L, GY, GX))
    rgb = rs.uniform(-0.3, 1.3, (N, 1, H, W)) + rs.uniform(-0.05, 0.05, (N, 3, H, W))
    if cot == "unit":
        dout = rs.standard_normal((N, 3, H, W))
    else:
        dout = np.where(rs.random((N, 3, H, W)) < 0.5, -1.0, 1.0) / (3 * N * H * W)
    return grids.astype(np.float32), rgb.astype(np.float32), dout.astype(np.float32)


def run(grids, rgb, ids, dout, mode="both"):
    """out, dL/drgb, dL/dgrids from bilagrid.slice; mode "rgb" asks only for dL/drgb (the GRID = false kernel), "grids"
    only for dL/dgrids (dL_drgb NULL).  The output not asked for is None."""
    g = torch.from_numpy(grids).cuda().requires_grad_(mode != "rgb")
    x = torch.from_numpy(rgb).cuda().requires_grad_(mode != "grids")
    out = bilagrid.slice(g, x, ids)
    out.backward(torch.from_numpy(dout).cuda())
    return tuple(None if t is None else t.detach().cpu().numpy() for t in (out, x.grad, g.grad))


def truth(grids, rgb, ids, dout):
    out64 = bo.slice64(grids, rgb, ids, coords="fp32")
    drgb64, dgrids64, _ = bo.grads64(grids, rgb, ids, dout, coords="fp32")
    return (out64, drgb64, dgrids64), bo.scales64(grids, rgb, ids, dout, coords="fp32")


def assert_within(name, got, want, tol):
    err = np.abs(got.astype(np.float64) - want)
    bad = err > tol
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err - tol, -np.inf)), err.shape)
        raise AssertionError(f"{name}: {int(bad.sum())} of {err.size} elements off, worst at {i}: got {got[i]!r}, "
                             f"want {want[i]!r}, tolerance {tol[i]!r}")


def compare(got, want, scales):
    (out, drgb, dgrids), (out64, drgb64, dgrids64), (m_out, m_drgb, m_dgrids) = got, want, scales
    if out is not None:
        assert_within("out", out, out64, OUT_TOL * m_out)
    if drgb is not None:
        assert_within("dL/drgb", drgb, drgb64, GRAD_TOL * m_drgb)
    if dgrids is not None:
        assert_within("dL/dgrids", dgrids, dgrids64, GRAD_TOL * m_dgrids)
        assert np.all(dgrids[m_dgrids == 0] == 0)


# L on both sides of 4 L = 32 with one row per lane, and the first and last L with two
@pytest.mark.parametrize("cot", ["unit", "l1"])
@pytest.mark.parametrize("L", [2, 3, 8, 9, 16])
def test_every_backward_instantiation(L, cot):
    """2 images with partial tiles in x and y over 3 grids (grid 1 unused): both gradients, dL/drgb alone and dL/dgrids
    alone, each against the truth."""
    ids = [2, 0]
    grids, rgb, dout = make_case(3, 2, 70, 100, L, 5, 7, cot, seed=L)
    want, scales = truth(grids, rgb, ids, dout)
    assert np.all(scales[2][1] == 0)
    for mode in ("both", "rgb", "grids"):
        got = run(grids, rgb, ids, dout, mode)
        assert (got[1] is None) == (mode == "grids") and (got[2] is None) == (mode == "rgb")
        compare(got, want, scales)


# (name, G, ids, H, W, L, GY, GX, cotangent)
SHAPES = [
    # 64 x 8 x 2 and 8 x 8 x 16 = MAX_NODES staged nodes (R = 1, R = 2); the first is denser than its 20 x 20 pixels
    ("at_bound_r1_dense", 1, [0], 20, 20, 2, 8, 64, "unit"),
    ("at_bound_r2", 1, [0], 40, 40, 16, 8, 8, "unit"),
    ("tile_crosses_7_x_cells", 1, [0], 40, 64, 4, 4, 16, "unit"),
    ("coarse_grid_1080p", 1, [0], 1080, 1920, 8, 2, 2, "l1"),
    ("strip_1x37", 1, [0], 1, 37, 8, 2, 9, "unit"),
    ("strip_37x1", 1, [0], 37, 1, 8, 9, 2, "l1"),
    ("many_images_unused_grid", 4, [3, 0, 3, 1, 3, 3, 0, 1, 3], 48, 80, 8, 6, 10, "unit"),
    ("64_images_5_grids", 5, [(7 * k) % 5 for k in range(64)], 24, 40, 5, 4, 6, "l1"),
]
# partial tiles: every pair of H, W in {31, 32, 33, 65}, with (GY, GX) = (5, 3) and (7, 33)
SHAPES += [(f"partial_{H}x{W}_{GY}x{GX}", 2, [1], H, W, L, GY, GX, "unit" if (H + W) % 2 else "l1")
           for GY, GX, L in ((5, 3, 8), (7, 33, 4)) for H in (31, 32, 33, 65) for W in (31, 32, 33, 65)]


@pytest.mark.parametrize("case", SHAPES, ids=[c[0] for c in SHAPES])
def test_shape_matrix(case):
    _, G, ids, H, W, L, GY, GX, cot = case
    grids, rgb, dout = make_case(G, len(ids), H, W, L, GY, GX, cot, seed=H * 7 + W)
    want, scales = truth(grids, rgb, ids, dout)
    compare(run(grids, rgb, ids, dout), want, scales)
    for g in set(range(G)) - set(ids):
        assert np.all(scales[2][g] == 0)


def test_long_strip_needs_the_kernels_coordinates():
    """W = 100003 with GX = 1024: (px + 0.5)(GX - 1) is not exact in fp32, and the product's rounding and the
    quotient's put the kernel's ix about an ulp (6e-5 near 1023) from the fp64 one, at most 2 eps32 ix.  The kernel
    matches the truth at its own coordinates.  The fp64-coordinate truth is further from it than the output bound, and
    within (|dix| + |diz|) 2 max|grid| sum_j |x_j| of the fp32-coordinate truth: dA/dix and dA/diz are differences of
    two nodes."""
    ids, H, W, L, GX = [0], 1, 100003, 8, 1024
    grids, rgb, dout = make_case(1, 1, H, W, L, 2, GX, "unit", seed=11)
    want, scales = truth(grids, rgb, ids, dout)
    got = run(grids, rgb, ids, dout)
    compare(got, want, scales)
    out64 = bo.slice64(grids, rgb, ids, coords="fp64")
    i32, t32 = bo._axis(W, GX, coords="fp32")
    i64, t64 = bo._axis(W, GX, coords="fp64")
    dix = np.abs((i32 + t32) - (i64 + t64))
    assert 0 < dix.max() <= 2 * EPS32 * (GX - 1)
    diz = np.abs(bo.z_coord(rgb[0], L, coords="fp32")[2] - bo.z_coord(rgb[0], L, coords="fp64")[2])
    diff = np.abs(out64 - want[0])
    assert np.all(diff <= (dix + diz) * 2 * np.abs(grids).max() * (np.abs(rgb[0]).sum(0) + 1))
    assert (np.abs(got[0] - out64) > OUT_TOL * scales[0]).any()


@pytest.mark.parametrize("H,W,GY,GX,L", [(20, 20, 8, 65, 2), (40, 40, 8, 9, 16)])
def test_one_node_over_the_bound_is_refused_without_a_launch(H, W, GY, GX, L):
    """65 x 8 x 2 = 1040 and 9 x 8 x 16 = 1152 staged nodes: refused as unsupported, forward and backward, on real
    buffers, with nothing launched."""
    lib = _lib.load()
    grids, rgb, dout = make_case(1, 1, H, W, L, GY, GX, "unit", seed=1)
    g, x, d = (torch.from_numpy(a).cuda() for a in (grids, rgb, dout))
    ids = torch.zeros(1, dtype=torch.int32, device="cuda")
    o, dr, dg, tmp = torch.empty_like(x), torch.empty_like(x), torch.empty_like(g), _lib.scratch(1 << 24, "cuda")
    torch.cuda.synchronize()
    n0 = lib.r3dg_launch_count()
    shape = (1, 1, H, W, GX, GY, L)
    assert lib.r3dg_bilagrid_tmp_bytes(*shape) == 0
    stream = torch.cuda.current_stream().cuda_stream
    assert lib.r3dg_bilagrid_forward(*shape, g.data_ptr(), ids.data_ptr(), x.data_ptr(), o.data_ptr(),
                                     stream) == UNSUPPORTED
    assert lib.r3dg_bilagrid_backward(*shape, g.data_ptr(), ids.data_ptr(), x.data_ptr(), d.data_ptr(), dr.data_ptr(),
                                      dg.data_ptr(), tmp.data_ptr(), tmp.numel(), stream) == UNSUPPORTED
    with pytest.raises(RuntimeError, match="unsupported"):
        bilagrid.slice(g, x, [0])
    assert lib.r3dg_launch_count() == n0


@pytest.mark.parametrize("G,ids,H,W,L,GY,GX", [(1, [0], 20, 20, 2, 8, 64), (1, [0], 40, 40, 16, 8, 8),
                                                (4, [3, 0, 3, 1, 3, 3, 0, 1, 3], 48, 80, 8, 6, 10)])
def test_writes_stay_inside_their_buffers(G, ids, H, W, L, GY, GX):
    """out, dL/drgb, dL/dgrids and a workspace of exactly r3dg_bilagrid_tmp_bytes, each inside a larger allocation of
    canaries: after the forward and the backward the padding on both sides is unchanged, the outputs are written in
    full, and they equal bilagrid.slice's bit for bit.  A tile staging more nodes than the host sized its slab for
    would write past its slab here."""
    N, PAD, CAN = len(ids), 4096, -12345.5
    grids, rgb, dout = make_case(G, N, H, W, L, GY, GX, "unit", seed=3)
    g, x, d = (torch.from_numpy(a).cuda() for a in (grids, rgb, dout))
    idt = torch.tensor(ids, dtype=torch.int32, device="cuda")
    lib = _lib.load()
    tmp_bytes = lib.r3dg_bilagrid_tmp_bytes(G, N, H, W, GX, GY, L)
    assert tmp_bytes > 0 and tmp_bytes % 256 == 0

    def padded(numel):
        t = torch.full((numel + 2 * PAD,), CAN, device="cuda")
        return t, t[PAD:PAD + numel]

    (out, out_v), (drgb, drgb_v), (dgrids, dgrids_v) = padded(x.numel()), padded(x.numel()), padded(g.numel())
    tmp, tmp_v = padded(tmp_bytes // 4)
    shape = (G, N, H, W, GX, GY, L)
    _lib.call("r3dg_bilagrid_forward", x.device, *shape, g.data_ptr(), idt.data_ptr(), x.data_ptr(), out_v.data_ptr())
    _lib.call("r3dg_bilagrid_backward", x.device, *shape, g.data_ptr(), idt.data_ptr(), x.data_ptr(), d.data_ptr(),
              drgb_v.data_ptr(), dgrids_v.data_ptr(), tmp_v.data_ptr(), tmp_bytes)
    torch.cuda.synchronize()
    for t, v in ((out, out_v), (drgb, drgb_v), (dgrids, dgrids_v), (tmp, tmp_v)):
        assert bool((t[:PAD] == CAN).all()) and bool((t[PAD + v.numel():] == CAN).all())
    want = run(grids, rgb, ids, dout)
    for v, w in zip((out_v, drgb_v, dgrids_v), want):
        got = v.cpu().numpy().reshape(w.shape)
        assert not (got == CAN).any()
        assert np.array_equal(got.view(np.int32), w.view(np.int32))

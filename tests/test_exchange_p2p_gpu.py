"""The one-kernel peer-memory gradient exchange (r3dg_exchange_p2p, csrc/sh_exchange.cu) on ONE GPU.

Rank r's launch reads every rank's factor section and writes only its own dL_dsh (the SH rebuild), and reads and writes
only slice r of every rank's dense section (the dense mean); it never writes a factor section, which lies after
n_dense.  So launching ranks 0..W-1 one after another on one stream, with W local buffers standing in for the ranks'
symmetric buffers, gives what W concurrent ranks between the two barriers give.  Every buffer has NaN guards on both
sides.  The SH rebuild is checked against an fp64 truth (exchange64) and, bit for bit, against r3dg_sh_grad_from_factors
(the same kernel and summation order); the dense mean, bit for bit, against the numpy fp32 sum in rank order.

Not run here: the multicast path (multimem.ld_reduce / multimem.st needs an NVSwitch multicast mapping; two or more GPUs
run it in test_multigpu_gpu.py), and set_grad_exchange's rebuild inside each rank's backward, which needs ranks that
run concurrently."""
import ctypes

import numpy as np
import pytest
import torch

import exchange64
from helpers import case_inputs, npy, rel_l2
from test_exchange_gpu import _backward
from test_exchange_p2p_cpu import GUARD, bits, fake_symm, guarded, guards_intact  # noqa: F401 (fake_symm: fixture)
from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200.dist import LeafGradBucket, P2PGradExchange, view_for_rank

DENSE_CTAS, THREADS = 1184, 128          # csrc/sh_exchange.cu: CTAs of the dense job, threads per CTA

# (world, D, M, P, n_dense / 4).  3M % 4 != 0 (M = 1, 9) takes the scalar stores, the other M the float4 stores.
CASES = [
    (1, 0, 1, 1, 1),                         # one rank; one Gaussian; a one-float4 section
    (2, 0, 16, 127, 1),                      # n_dense / 4 < world: rank 1's slice is empty
    (3, 1, 4, 128, 0),                       # the SH job alone
    (3, 0, 1, 1000, 1),                      # M = 1 over several CTAs; ranks 1 and 2 have empty slices
    (8, 1, 16, 129, 1001),                   # one full 8-view chunk; 1001 % 8 != 0
    (9, 2, 9, 129, 10),                      # a full chunk and a 1-view chunk; 10 % 9 != 0
    (17, 2, 16, 1000, 5),                    # two full chunks and a 1-view chunk; 12 of 17 slices empty
    (64, 3, 16, 200, 130),                   # the most ranks; 130 % 64 != 0
    (3, 3, 16, 0, 778),                      # P = 0 with a dense job: every CTA is a dense CTA; 778 % 3 != 0
    (2, 3, 16, 1000, 2 * DENSE_CTAS * THREADS + 8199),   # slices of 155,652 float4 > 1184 x 128: the dense CTAs loop
    (3, 3, 16, 300_000, 3001),               # period 2, then SH CTAs after the last dense CTA
    (3, 3, 16, 1_000_000, 4099),             # period 7, then SH CTAs after the last dense CTA
]


def case_id(c):
    return "W{}-D{}-M{}-P{}-n{}".format(*c[:4], 4 * c[4])


def launch_layout(P, n_dense):
    """(period, SH CTAs after the last dense CTA) of the launch (csrc/sh_exchange.cu); (None, None) without a dense
    job.  The dense CTAs are blocks 0, period, 2 period, ... (DENSE_CTAS of them)."""
    if not n_dense:
        return None, None
    grid = (P + THREADS - 1) // THREADS + DENSE_CTAS
    period = max(1, grid // DENSE_CTAS)
    return period, grid - 1 - (DENSE_CTAS - 1) * period


def test_case_list_covers_every_edge():
    """The shapes where the launch's index arithmetic, the slicing and the stores go wrong are all in CASES."""
    assert {c[0] for c in CASES} >= {1, 2, 3, 8, 9, 17, 64}
    assert {(c[1], c[2]) for c in CASES} >= {(D, M) for D in range(4) for M in ((D + 1) ** 2, 16)}
    assert {c[2] for c in CASES} & {1, 9} and {c[2] for c in CASES} & {4, 16}
    assert {c[3] for c in CASES} >= {0, 1, 127, 128, 129}
    layouts = [launch_layout(c[3], 4 * c[4]) for c in CASES if c[3] > 0]
    assert any(p == 1 for p, _ in layouts)
    assert any(p == 2 and tail > 0 for p, tail in layouts) and any(p is not None and p >= 7 and tail > 0 for p, tail in layouts)
    assert {4 * c[4] for c in CASES} >= {0, 4}
    assert any(0 < c[4] < c[0] for c in CASES) and any(c[4] % c[0] for c in CASES)
    assert any(-(-c[4] // c[0]) > DENSE_CTAS * THREADS for c in CASES)
    assert any(c[3] == 0 and c[4] > 0 for c in CASES)


def _inputs(world, P, n_dense, seed):
    """Seeded fp32 inputs: means [P,3] within 2 of the origin, camera centres [world,3] at distance 4, factors
    [world,P,3] over 8 binades with rows zero in some views and in all views (as +0 and -0), and one Gaussian culled
    in view 0 whose camera centre sits on its mean; dense [world,n_dense] over 80 binades with zeros, -0 and
    subnormals, so that the rank-order sums round."""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((world, 3))
    campos = (4.0 * c / np.linalg.norm(c, axis=1, keepdims=True)).astype(np.float32)
    means = rng.uniform(-1.1, 1.1, (P, 3)).astype(np.float32)
    f = (rng.standard_normal((world, P, 3)) * np.exp(rng.uniform(-3, 3, (world, P, 1)))).astype(np.float32)
    g = np.arange(P)
    f[:, g % 7 == 3] = 0.0                                         # culled in every view
    f[:, g % 11 == 5] = -0.0
    for v in range(world):
        f[v, (g + v) % 5 == 1] = 0.0                               # culled in some views
    if P > 1 and world > 1:
        means[1] = campos[0]
        f[0, 1] = 0.0
    dense = (rng.standard_normal((world, n_dense)) * np.exp(rng.uniform(-27, 27, (world, n_dense)))).astype(np.float32)
    dense[:, 0::13] = 0.0
    dense[:, 5::17] = -0.0
    dense[:, 7::19] = np.float32(3e-41)
    dense[:, 8::23] = np.float32(-3e-41)
    return means, campos, f, dense


def _rank_order_mean(xs):
    """The numpy fp32 sum of xs in rank order, starting from +0, times fp32(1) / fp32(world)."""
    acc = np.zeros_like(xs[0], dtype=np.float32)
    for x in xs:
        acc = acc + np.asarray(x, np.float32)
    return acc * (np.float32(1) / np.float32(len(xs)))


def _args(P, D, M, world, rank, means, campos, out, sym, n_dense):
    a = _lib.ExchangeArgs()
    a.P, a.D, a.M, a.world, a.rank, a.n_dense = P, D, M, world, rank, n_dense
    a.means3D, a.campos, a.dL_dsh = means.data_ptr(), campos.data_ptr(), out.data_ptr()
    for v in range(world):
        a.dense[v] = sym[v].data_ptr()
        a.factors[v] = sym[v].data_ptr() + 4 * n_dense
    a.dense_multicast = None
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_exchange_p2p_simulated_ranks(case):
    world, D, M, P, n4 = case
    n_dense, dev = 4 * n4, torch.device("cuda")
    means_np, campos_np, f_np, dense_np = _inputs(world, P, n_dense, seed=CASES.index(case))
    # rank v's symmetric buffer: its dense section, then its factor section
    sym_full, sym = guarded(world, n_dense + 3 * P, dev)
    sym[:, :n_dense] = torch.from_numpy(dense_np).to(dev)
    sym[:, n_dense:] = torch.from_numpy(f_np.reshape(world, -1)).to(dev)
    out_full, out = guarded(world, P * M * 3, dev)
    m_full, m = guarded(1, 3 * P, dev)
    c_full, c = guarded(1, 3 * world, dev)
    m[0] = torch.from_numpy(means_np.reshape(-1)).to(dev)
    c[0] = torch.from_numpy(campos_np.reshape(-1)).to(dev)
    inputs_before = [bits(t).clone() for t in (m_full, c_full)]
    factors_before = bits(sym[:, n_dense:]).clone()

    mean = torch.from_numpy(_rank_order_mean(list(dense_np)).view(np.int32)).to(dev)
    per = -(-n4 // world)
    for r in range(world):
        before = bits(sym_full).clone()
        _lib.call("r3dg_exchange_p2p", dev, ctypes.byref(_args(P, D, M, world, r, m[0], c[0], out[r], sym, n_dense)))
        after = bits(sym_full)
        lo, hi = 4 * min(r * per, n4), 4 * min(r * per + per, n4)            # rank r's slice, in floats
        changed = (after != before).any(0).nonzero()[:, 0] - GUARD                 # columns of the data
        assert not ((changed < lo) | (changed >= hi)).any(), f"rank {r}'s launch wrote outside its slice [{lo}, {hi})"
        assert torch.equal(bits(sym[:, lo:hi]), mean[lo:hi].expand(world, -1)), f"rank {r}'s slice"
    assert torch.equal(bits(sym[:, :n_dense]), mean.expand(world, -1))
    assert torch.equal(bits(sym[:, n_dense:]), factors_before)
    assert guards_intact(sym_full, n_dense + 3 * P) and guards_intact(out_full, P * M * 3)
    assert all(torch.equal(bits(t), b) for t, b in zip((m_full, c_full), inputs_before))
    if P == 0:
        return

    assert not bool(torch.isnan(out).any()), "dL_dsh elements left unwritten"
    for r in range(1, world):
        assert torch.equal(bits(out[r]), bits(out[0])), f"rank {r}'s dL_dsh differs from rank 0's"
    fac_full, fac = guarded(1, world * P * 3, dev)
    fac[0] = torch.from_numpy(f_np.reshape(-1)).to(dev)
    ref_full, ref = guarded(1, P * M * 3, dev)
    _lib.call("r3dg_sh_grad_from_factors", dev, P, D, M, world, m.data_ptr(), c.data_ptr(), fac.data_ptr(),
              float(np.float32(1) / np.float32(world)), ref.data_ptr())
    assert guards_intact(ref_full, P * M * 3) and torch.equal(bits(ref[0]), bits(out[0]))
    g = out[0].view(P, M, 3)
    assert bool((g[:, (D + 1) ** 2:] == 0).all())
    assert bool((g[torch.from_numpy((f_np == 0).all(axis=(0, 2))).to(dev)] == 0).all())    # culled in every view
    exchange64.check(g, m[0].view(P, 3), c[0].view(world, 3), fac[0].view(world, P, 3), D, M)


@pytest.mark.gpu
@pytest.mark.parametrize("world,M,P", [(3, 1, 1000), (9, 16, 129), (17, 1, 5000), (64, 16, 300)])
def test_degree_0_rebuild_is_the_fp32_sum_in_view_order(world, M, P):
    """With D = 0 the basis is the constant C0, and with factors +-2^e every product C0 f is exact in fp32, so the
    kernel's result is known bit for bit whether or not it contracts the products into FMAs: the fp32 sum over the
    live views in view order, starting from +0, times fp32(1) / fp32(world).  This pins the summation order and the
    scale after the sum, which the fp64 bound cannot see."""
    dev = torch.device("cuda")
    means_np, campos_np, f_np, _ = _inputs(world, P, 0, seed=world)
    rng = np.random.default_rng(world)
    f_np = np.where(f_np == 0, f_np, np.ldexp(np.sign(f_np), rng.integers(-6, 7, f_np.shape))).astype(np.float32)
    live = (f_np != 0).any(axis=2, keepdims=True)
    c0 = np.float32(0.28209479177387814)
    acc = np.zeros((P, 3), np.float32)
    for v in range(world):
        acc = np.where(live[v], acc + c0 * f_np[v], acc)
    expect = np.zeros((P, M, 3), np.float32)
    expect[:, 0] = acc * (np.float32(1) / np.float32(world))
    sym_full, sym = guarded(world, 3 * P, dev)
    sym[:] = torch.from_numpy(f_np.reshape(world, -1)).to(dev)
    out_full, out = guarded(world, P * M * 3, dev)
    m, c = torch.from_numpy(means_np).to(dev), torch.from_numpy(campos_np).to(dev)
    for r in range(world):
        _lib.call("r3dg_exchange_p2p", dev, ctypes.byref(_args(P, 0, M, world, r, m, c, out[r], sym, 0)))
    assert guards_intact(out_full, P * M * 3)
    assert torch.equal(bits(out), torch.from_numpy(expect.reshape(1, -1).view(np.int32)).to(dev).expand(world, -1))


REFUSALS = {
    "n_dense_not_multiple_of_4": lambda a: setattr(a, "n_dense", 6),
    "negative_n_dense": lambda a: setattr(a, "n_dense", -4),
    "rank_equals_world": lambda a: setattr(a, "rank", 2),
    "negative_rank": lambda a: setattr(a, "rank", -1),
    "world_0": lambda a: setattr(a, "world", 0),
    "world_65": lambda a: setattr(a, "world", 65),
    "null_factor": lambda a: a.factors.__setitem__(1, None),
    "null_dense": lambda a: a.dense.__setitem__(1, None),
    "degree_needs_more_coefficients": lambda a: setattr(a, "D", 2),
    "null_means3D": lambda a: setattr(a, "means3D", None),
    "null_campos": lambda a: setattr(a, "campos", None),
    "null_dL_dsh": lambda a: setattr(a, "dL_dsh", None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(REFUSALS))
def test_exchange_p2p_refuses_before_any_launch(kind):
    """Each bad argument returns R3DG_ERR_BAD_ARG and changes nothing; the same call with the argument fixed does
    write (so an unrefused call would have been seen)."""
    world, D, M, P, n_dense, dev = 2, 1, 4, 129, 8, torch.device("cuda")
    means_np, campos_np, f_np, dense_np = _inputs(world, P, n_dense, seed=99)
    sym_full, sym = guarded(world, n_dense + 3 * P, dev)
    sym[:, :n_dense] = torch.from_numpy(dense_np).to(dev)
    sym[:, n_dense:] = torch.from_numpy(f_np.reshape(world, -1)).to(dev)
    out_full, out = guarded(world, P * M * 3, dev)
    m = torch.from_numpy(means_np).to(dev)
    c = torch.from_numpy(campos_np).to(dev)
    before = [bits(t).clone() for t in (sym_full, out_full)]
    a = _args(P, D, M, world, 0, m, c, out[0], sym, n_dense)
    REFUSALS[kind](a)
    lib = _lib.load()
    assert lib.r3dg_exchange_p2p(ctypes.byref(a), torch.cuda.current_stream(dev).cuda_stream) == -10001
    torch.cuda.synchronize(dev)
    assert all(torch.equal(bits(t), b) for t, b in zip((sym_full, out_full), before))
    _lib.call("r3dg_exchange_p2p", dev, ctypes.byref(_args(P, D, M, world, 0, m, c, out[0], sym, n_dense)))
    assert not torch.equal(bits(out_full), before[1]) and not torch.equal(bits(sym_full), before[0])


DENSE_NAMES = {"means3D": "dL_dmeans3D", "features": "dL_dfeatures", "opacity": "dL_dopacity", "scales": "dL_dscales",
               "rotations": "dL_drotations"}


@pytest.mark.gpu
def test_p2p_exchange_three_rank_step(fake_symm):
    """P2PGradExchange as bench.py's resident step uses it, for W = 3 simulated ranks: rank r renders view
    view_for_rank(step, r, W, views) and runs the deterministic backward into its exchange's views; then every rank
    exchanges, in rank order.  The dense gradients must be the rank-order mean of W deterministic one-view backwards
    bit for bit; dL_dsh must meet the fp64 bound and match the mean of the one-view dense dL_dsh."""
    from relightable3dgaussian_b200 import _C_raster as C
    from test_deterministic_gpu import deterministic
    W, P, Wi, Hi, S, deg, views, step = 3, 20_000, 160, 120, 5, 3, 8, 1
    fake = fake_symm(W, "cuda")
    exs = []
    for r in range(W):
        fake.rank = r
        exs.append(P2PGradExchange(P, S, 16, "cuda"))
    rng = np.random.default_rng(5)
    dense, cams = [], []
    with deterministic():
        for r, ex in enumerate(exs):
            sc, cam = case_inputs(P, Wi, Hi, S, view=view_for_rank(step, r, W, views))
            cots = [rng.standard_normal((c, Hi, Wi)).astype(np.float32) for c in (3, 1, 1, S)]
            gd, _ = _backward(C, sc, cam, S, deg, cots)                          # one-view dense backward
            again = torch.empty((P, 3), device="cuda")
            _backward(C, sc, cam, S, deg, cots, out={"sh_factor": again})
            _backward(C, sc, cam, S, deg, cots, out=ex.views)
            assert torch.equal(bits(again), bits(ex.factor)), "the deterministic backward's SH factor is not reproducible"
            for name, key in DENSE_NAMES.items():
                assert torch.equal(bits(ex.views[name]), bits(gd[key])), name
            dense.append(gd)
            cams.append(cam.campos)
    means3D = sc.means3D.cuda().contiguous()
    campos_all = torch.stack(cams).cuda().float().contiguous()
    for ex in exs:
        ex.exchange(means3D, campos_all, deg)
    assert fake.events == [("barrier", r, ch) for r in range(W) for ch in (0, 1)]
    for name, key in DENSE_NAMES.items():
        expect = _rank_order_mean([npy(g[key]) for g in dense])
        for r, ex in enumerate(exs):
            assert np.array_equal(npy(ex.grads[name]).view(np.int32), expect.view(np.int32)), (name, r)
    sh = exs[0].grads["sh"]
    for ex in exs[1:]:
        assert torch.equal(bits(ex.grads["sh"]), bits(sh))
    exchange64.check(sh, means3D, campos_all, torch.stack([ex.factor for ex in exs]), deg, 16)
    dense_sh = np.mean([npy(g["dL_dsh"]).astype(np.float64) for g in dense], axis=0)
    assert np.abs(dense_sh).max() > 0 and rel_l2(npy(sh), dense_sh) < 1e-6
    # the SH-only exchange leaves every rank's dense and factor sections alone
    sym_before, sh_before = bits(fake.full).clone(), bits(sh).clone()
    for ex in exs:
        ex.exchange(means3D, campos_all, deg, dense=False)
    assert torch.equal(bits(fake.full), sym_before) and torch.equal(bits(exs[0].grads["sh"]), sh_before)


@pytest.mark.gpu
def test_symmetric_leaf_grad_bucket_mean(fake_symm):
    """LeafGradBucket(symmetric=True).allreduce_mean for W = 3 simulated ranks leaves every parameter's .grad at the
    rank-order mean, bit for bit, including a .grad replaced after attach() (copied into the buffer first).  Rank 0
    replaces it: its copy-in precedes every launch, as barrier 0 makes every rank's copy-in do with concurrent ranks."""
    W = 3
    shapes = [(1000, 3), (333, 5), (7,), (1000, 16, 3)]
    fake = fake_symm(W, "cuda")
    buckets = []
    for r in range(W):
        fake.rank = r
        buckets.append(LeafGradBucket([torch.zeros(s, device="cuda", requires_grad=True) for s in shapes], symmetric=True))
    rng = np.random.default_rng(8)
    grads = [[(rng.standard_normal(s) * np.exp(rng.uniform(-20, 20, s))).astype(np.float32) for s in shapes]
             for _ in range(W)]
    for r, b in enumerate(buckets):
        b.zero()
        for i, (p, g) in enumerate(zip(b.params, grads[r])):
            if (r, i) == (0, 2):
                p.grad = torch.from_numpy(g).cuda()
            else:
                p.grad.copy_(torch.from_numpy(g))
    for b in buckets:
        b.allreduce_mean()
    assert fake.events == [("barrier", r, ch) for r in range(W) for ch in (0, 1)]
    for i in range(len(shapes)):
        expect = _rank_order_mean([grads[r][i] for r in range(W)])
        for r, b in enumerate(buckets):
            p = b.params[i]
            assert p.grad.data_ptr() == b.views[i].data_ptr(), (r, i)
            assert np.array_equal(npy(p.grad).view(np.int32), expect.view(np.int32)), (r, i)

"""Host side of the one-kernel peer-memory gradient exchange (dist.P2PGradExchange, dist.LeafGradBucket(symmetric=True),
dist._nvls_mean_inplace) on fake symmetric memory, with the kernel call replaced by a stand-in that records its
arguments: which buffers, offsets and sizes reach r3dg_exchange_p2p, and that the two barriers bracket the launch.

The `fake_symm` fixture is shared with tests/test_exchange_p2p_gpu.py, where the same fake lets W simulated ranks run
the real kernel one after another on one GPU."""
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist

import exchange64
from oracle import oracle
from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200.dist import LeafGradBucket, P2PGradExchange

GUARD = 64                          # floats of guard on each side of a buffer (a multiple of 4: rows stay 16-byte aligned)
NAN_BITS = 0x7FC0FFEE               # a quiet NaN with a payload no arithmetic produces


def guarded(rows, n, device):
    """`rows` buffers of n float32 each, with at least GUARD floats of NAN_BITS on both sides, as one tensor.
    Returns (full [rows, L], data [rows, n]); every data[r] is 16-byte aligned and every float of `full` starts as
    NAN_BITS."""
    L = GUARD + (n + 3) // 4 * 4 + GUARD
    full = torch.full((rows, L), NAN_BITS, dtype=torch.int32, device=device).view(torch.float32)
    return full, full[:, GUARD:GUARD + n]


def bits(t):
    return t.contiguous().view(torch.int32)


def guards_intact(full, n):
    """Every float of `full` (from guarded(rows, n, ...)) outside the data columns still holds NAN_BITS."""
    b = bits(full)
    return bool((b[:, :GUARD] == NAN_BITS).all()) and bool((b[:, GUARD + n:] == NAN_BITS).all())


class FakeSymmetricMemory:
    """torch.distributed._symmetric_memory for `world` simulated ranks in one process.  The first empty(n) allocates
    `world` guarded buffers; the k-th call returns buffer k, i.e. rank k's when the ranks are constructed in rank
    order.  rendezvous() returns a handle with every buffer's pointer, no multicast address, and a barrier that
    records its calls in `events` as ("barrier", rank, channel).  `rank` is what dist.get_rank() returns."""

    def __init__(self, world, device):
        self.world, self.device, self.rank = world, torch.device(device), 0
        self.full, self.data, self.calls, self.events = None, None, 0, []

    def empty(self, n, dtype=torch.float32, device=None):
        assert dtype == torch.float32 and torch.device(device).type == self.device.type
        if self.data is None:
            self.full, self.data = guarded(self.world, n, self.device)
        assert self.calls < self.world and self.data.shape[1] == n, "one empty() of the same size per rank"
        self.calls += 1
        return self.data[self.calls - 1]

    def rendezvous(self, t, group=None):
        ptrs = [self.data[r].data_ptr() for r in range(self.world)]
        k = ptrs.index(t.data_ptr())
        events = self.events

        class Handle:
            buffer_ptrs = ptrs
            multicast_ptr = 0

            @staticmethod
            def barrier(channel=0):
                events.append(("barrier", k, channel))
        return Handle()


@pytest.fixture
def fake_symm(monkeypatch):
    """install(world, device) -> FakeSymmetricMemory: replaces torch.distributed._symmetric_memory (the module in
    sys.modules and the attribute of torch.distributed, which `import a.b as c` reads first) and makes torch.distributed
    report an initialised group of `world` ranks, this process being rank `fake.rank`."""
    def install(world, device):
        fake = FakeSymmetricMemory(world, device)
        monkeypatch.setitem(sys.modules, "torch.distributed._symmetric_memory", fake)
        monkeypatch.setattr(dist, "_symmetric_memory", fake, raising=False)
        monkeypatch.setattr(dist, "is_initialized", lambda: True)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: world)
        monkeypatch.setattr(dist, "get_rank", lambda group=None: fake.rank)
        return fake
    return install


def _record_launches(monkeypatch, fake, on_launch=None):
    """Replaces _lib.call: each call appends ("launch", rank) to fake.events and its ExchangeArgs, as a dict, to the
    list returned, and calls on_launch()."""
    seen = []

    def call(name, device, args, what=None):
        assert name == "r3dg_exchange_p2p"
        a = args._obj
        rec = {f: getattr(a, f) for f in ("P", "D", "M", "world", "rank", "means3D", "campos", "dL_dsh", "n_dense",
                                          "dense_multicast")}
        rec["factors"], rec["dense"] = list(a.factors), list(a.dense)
        seen.append(rec)
        fake.events.append(("launch", a.rank))
        if on_launch:
            on_launch()
    monkeypatch.setattr(_lib, "call", call)
    return seen


def test_p2p_exchange_passes_its_symmetric_buffers(fake_symm, monkeypatch):
    W, P, S, M = 3, 301, 5, 16
    fake = fake_symm(W, "cpu")
    seen = _record_launches(monkeypatch, fake)
    exs = []
    for r in range(W):
        fake.rank = r
        exs.append(P2PGradExchange(P, S, M, "cpu"))
    ptrs = [fake.data[r].data_ptr() for r in range(W)]
    means3D, campos = torch.zeros(P, 3), torch.zeros(W, 3)
    for r, ex in enumerate(exs):
        assert (ex.world, ex.rank, ex.peer_ptrs, ex.multicast) == (W, r, ptrs, 0)
        assert ex.flat.data_ptr() == ptrs[r] and ex.factor.data_ptr() == ptrs[r] + 4 * ex.factor_off
        assert ex.n_dense == ex.factor_off and ex.factor_off % 4 == 0          # the factor section comes last
        for name, t in ex.views.items():                                         # every other section lies before it
            if name != "sh_factor":
                assert ptrs[r] <= t.data_ptr() and t.data_ptr() + 4 * t.numel() <= ptrs[r] + 4 * ex.n_dense, name
        for dense in (True, False):
            fake.events.clear()
            ex.exchange(means3D, campos, 2, dense=dense)
            assert fake.events == [("barrier", r, 0), ("launch", r), ("barrier", r, 1)]
            a = seen[-1]
            assert (a["P"], a["D"], a["M"], a["world"], a["rank"]) == (P, 2, M, W, r)
            assert (a["means3D"], a["campos"], a["dL_dsh"]) == (means3D.data_ptr(), campos.data_ptr(), ex.sh.data_ptr())
            assert a["n_dense"] == (ex.factor_off if dense else 0)
            assert a["factors"] == [p + 4 * ex.factor_off for p in ptrs] + [None] * (64 - W)
            assert a["dense"] == ptrs + [None] * (64 - W) and a["dense_multicast"] is None
        # the rank's own rebuild inside backward (rasterizer.set_grad_exchange) is the SH-only exchange
        fake.events.clear()
        ex.rebuild_sh(means3D, campos, 1)
        assert seen[-1]["n_dense"] == 0 and seen[-1]["D"] == 1 and fake.events[1] == ("launch", r)


def test_symmetric_leaf_bucket_mean_passes_the_whole_buffer(fake_symm, monkeypatch):
    W = 3
    fake = fake_symm(W, "cpu")
    at_launch = []
    seen = _record_launches(monkeypatch, fake, on_launch=lambda: at_launch.append(buckets[1].views[1].clone()))
    buckets = []
    for r in range(W):
        fake.rank = r
        buckets.append(LeafGradBucket([torch.zeros(5, 3, requires_grad=True), torch.zeros(130, requires_grad=True)],
                                      symmetric=True))
    ptrs = [fake.data[r].data_ptr() for r in range(W)]
    b = buckets[1]
    replaced = torch.full((130,), 7.0)
    b.params[1].grad = replaced                                 # a backward that replaced .grad: copied in before the mean
    b.allreduce_mean()
    assert fake.events == [("barrier", 1, 0), ("launch", 1), ("barrier", 1, 1)]
    assert torch.equal(at_launch[0], replaced) and b.params[1].grad.data_ptr() == b.views[1].data_ptr()
    a = seen[-1]
    assert (a["P"], a["M"], a["world"], a["rank"], a["n_dense"]) == (0, 1, W, 1, b.flat.numel())
    assert b.flat.numel() == 384 and a["dense"] == ptrs + [None] * (64 - W) and a["dense_multicast"] is None
    assert a["factors"] == [None] * 64 and a["dL_dsh"] is None


def test_fp64_truth_matches_the_fp32_oracle_and_zero_rows():
    """exchange64 against the fp32 restatement in oracle.py (a check of the truth itself), and its zero rows: a row
    whose factor is zero in a view adds exactly 0 from that view, even when the view's camera centre sits on the mean."""
    rng = np.random.default_rng(4)
    P, W = 500, 3
    means = rng.standard_normal((P, 3)).astype(np.float32)
    campos = (rng.standard_normal((W, 3)) * 5).astype(np.float32)
    f = rng.standard_normal((W, P, 3)).astype(np.float32)
    f[:, 7] = 0.0                                                    # culled in every view
    f[0, 8] = 0.0
    means[8] = campos[0]                                             # culled in view 0, whose camera sits on it
    for D, M in ((0, 1), (1, 4), (2, 16), (3, 16)):
        g64, mag = exchange64.sh_grad(torch.from_numpy(means), torch.from_numpy(campos), torch.from_numpy(f), D, M)
        assert g64.shape == (P, M, 3) and bool(torch.isfinite(g64).all()) and bool((g64[:, (D + 1) ** 2:] == 0).all())
        assert bool((g64[7] == 0).all()) and bool((mag[7] == 0).all())
        rest = [v for v in range(P) if v != 8]
        with np.errstate(invalid="ignore"):                         # the oracle has no skip: row 8 is NaN there
            ref = oracle.sh_grad_from_factors(means, list(campos), list(f), D, M, 1.0 / W)
        np.testing.assert_allclose(g64.numpy()[rest], ref[rest], rtol=0, atol=1e-5)
        one = exchange64.sh_grad(torch.from_numpy(means[8:9]), torch.from_numpy(campos[1:]), torch.from_numpy(f[1:, 8:9]),
                                 D, M)[0]
        assert torch.allclose(g64[8], one[0] * (W - 1) / W, rtol=1e-12, atol=0)
        assert bool((mag >= g64.abs() * (1 - 1e-12)).all())

"""MCMC densification without a GPU: the numerics of the source correction against mpmath, the growth count, argument
rejection before any launch, install / uninstall."""
import ctypes
import math

import pytest
import torch

import densify_oracle as do
import mcmc_oracle as mo
from relightable3dgaussian_b200 import _lib

OPACITIES = [0.005 + 1e-9, 0.0051, 0.01, 0.05, 0.1, 0.25, 0.5, 0.75, 0.9, 0.99, 0.999, 0.9999, 1.0 - 2.0 ** -23]


def test_correction_against_mpmath():
    """coef and the clamped opacity of the fp64 restatement (the kernel's formula) within 1e-11 of a 60-digit
    evaluation of the paper's double sum, for N = 2..51 over an opacity grid; 1 - (1 - x)^N = o before the clamp."""
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 60
    worst = 0.0
    for N in range(2, 52):
        o = torch.tensor(OPACITIES, dtype=torch.float64)
        x, coef, logit = mo.correction(o, torch.full(o.shape, N, dtype=torch.int64), 0.005)
        for k, ok in enumerate(OPACITIES):
            om = mp.mpf(ok)
            xm = 1 - (1 - om) ** (mp.mpf(1) / N)
            dbl = sum(mp.binomial(i - 1, kk) * (-1) ** kk * xm ** (kk + 1) / mp.sqrt(kk + 1)
                      for i in range(1, N + 1) for kk in range(i))
            cm = om / dbl
            on = min(max(xm, mp.mpf(0.005)), mp.mpf(mo.OMAX))
            lm = mp.log(on / (1 - on))
            rc = abs(float((mp.mpf(float(coef[k])) - cm) / cm))
            rl = abs(float((mp.mpf(float(logit[k])) - lm) / max(1, abs(lm))))         # logit(0.5) = 0
            rx = abs(float((mp.mpf(float(x[k])) - xm) / xm))
            worst = max(worst, rc, rl, rx)
            assert rc <= 1e-11 and rl <= 1e-11 and rx <= 1e-11, (N, ok, rc, rl, rx)
            back = 1 - (1 - mp.mpf(float(x[k]))) ** N
            assert abs(float((back - om) / om)) <= 1e-13, (N, ok)
    print(f"[mcmc] correction: worst relative error {worst:.2e}")


def test_single_sum_equals_double_sum():
    """sum_{j=1..N} (-1)^(j-1) C(N,j) x^j / sqrt(j) = sum_{i=1..N} sum_{k<i} C(i-1,k) (-1)^k x^(k+1) / sqrt(k+1)."""
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 60
    for N in (2, 3, 7, 20, 51, 64):
        for x in (mp.mpf("0.001"), mp.mpf("0.3"), mp.mpf("0.9")):
            single = sum((-1) ** (j - 1) * mp.binomial(N, j) * x ** j / mp.sqrt(j) for j in range(1, N + 1))
            double = sum(mp.binomial(i - 1, k) * (-1) ** k * x ** (k + 1) / mp.sqrt(k + 1)
                         for i in range(1, N + 1) for k in range(i))
            assert abs(single - double) <= mp.mpf(10) ** -30 * abs(double), (N, x)       # 60 digits less the cancellation


def test_binomial_table_is_exact_where_fp64_can_be():
    for n in range(57):
        for j in range(n + 1):
            assert int(mo.BINOM[n, j]) == math.comb(n, j)


def test_zero_opacity_source_has_the_limit_correction():
    x, coef, logit = mo.correction(torch.zeros(3, dtype=torch.float64), torch.tensor([2, 10, 51]), 0.005)
    assert torch.equal(x, torch.zeros(3, dtype=torch.float64)) and torch.equal(coef, torch.ones(3, dtype=torch.float64))
    assert torch.isfinite(logit).all()


def test_growth_count():
    from relightable3dgaussian_b200.mcmc import growth_count
    assert growth_count(1000, 10_000) == 50
    assert growth_count(1000, 1020) == 20
    assert growth_count(1000, 1000) == 0 and growth_count(1000, 10) == 0            # never prunes to the cap
    assert growth_count(19, 100) == 0                                               # int(19 * 1.05) = 19
    assert growth_count(20, 100) == 1
    assert growth_count(1 << 20, 3 << 20) == int((1 << 20) * 1.05) - (1 << 20)
    assert growth_count(100, 1000, 0.0) == 0 and growth_count(100, 1000, 1.0) == 100
    assert growth_count(0, 100) == 0


def test_entry_points_reject_bad_arguments_without_launching():
    lib = _lib.load()
    n0 = lib.r3dg_launch_count()
    F = ctypes.c_void_p(256)           # never dereferenced: every call below is refused first
    assert lib.r3dg_mcmc_tmp_bytes(1 << 20, 0) > 33 * (1 << 20)
    assert lib.r3dg_mcmc_tmp_bytes(1000, 100_000) > lib.r3dg_mcmc_tmp_bytes(1000, 0)
    assert lib.r3dg_mcmc_noise(-1, F, F, F, F, F, 1.0, 100.0, 0.005, None) == -10001
    assert lib.r3dg_mcmc_noise(10, None, F, F, F, F, 1.0, 100.0, 0.005, None) == -10001
    assert lib.r3dg_mcmc_noise(0, None, None, None, None, None, 1.0, 100.0, 0.005, None) == 0
    tb = lib.r3dg_mcmc_tmp_bytes(10, 0)
    assert lib.r3dg_mcmc_classify(0, F, 0.005, F, tb, None) == -10001
    assert lib.r3dg_mcmc_classify(10, None, 0.005, F, tb, None) == -10001
    assert lib.r3dg_mcmc_classify(10, F, 0.005, F, tb - 1, None) == -10001
    assert lib.r3dg_mcmc_classify(10, F, 0.005, ctypes.c_void_p(264), tb, None) == -10001        # tmp not 16-byte aligned
    d = (_lib.DensifyTensor * 1)()
    d[0].src = d[0].dst = 256
    d[0].row_bytes, d[0].kind = 12, 0

    def apply(P=10, n_new=0, n_max=51, num=1, descs=d, tmp_bytes=None):
        return lib.r3dg_mcmc_apply(P, n_new, F, F, F, 0.005, n_max, num, descs, F,
                                   lib.r3dg_mcmc_tmp_bytes(P, n_new) if tmp_bytes is None else tmp_bytes, None)
    assert apply(P=0) == -10001
    assert apply(n_max=1) == -10001 and apply(n_max=65) == -10001
    assert apply(num=0) == -10001 and apply(num=49) == -10001
    assert apply(tmp_bytes=lib.r3dg_mcmc_tmp_bytes(10, 0) - 1) == -10001
    assert apply(n_new=100, tmp_bytes=lib.r3dg_mcmc_tmp_bytes(10, 0)) == -10001     # too small for 100 draws
    assert apply(n_new=5) == -10001                                                # growth must not write in place
    assert lib.r3dg_mcmc_apply(10, 0, F, F, F, 0.005, 51, 1, d, ctypes.c_void_p(264), tb, None) == -10001
    for kind, row_bytes in ((4, 12), (2, 12), (3, 12), (7, 12), (5, 12), (6, 4), (0, 6), (0, 0)):
        d[0].kind, d[0].row_bytes = kind, row_bytes
        assert apply() == -10001, (kind, row_bytes)
    d[0].kind, d[0].row_bytes, d[0].dst = 0, 12, 512
    assert apply() == -10001                                                       # relocation writes in place
    assert lib.r3dg_launch_count() == n0


def _model(**over):
    case = mo.mcmc_case("s1_p7")
    m = do.build_model(case, mo.StandIn)
    for k, v in over.items():
        setattr(m, k, v)
    return m


def test_python_refusals_before_any_launch():
    from relightable3dgaussian_b200 import mcmc
    lib = _lib.load()
    n0 = lib.r3dg_launch_count()
    with pytest.raises(RuntimeError, match="baked visibility"):
        mcmc.relocate_and_grow(_model(_visibility_tracing=torch.zeros(7, 24)), 100)
    for bad in (1, 65, 2.5, True):
        with pytest.raises(ValueError, match="n_max"):
            mcmc.relocate_and_grow(_model(), 100, n_max=bad)
    for bad in (-1, 1.5, None):
        with pytest.raises(ValueError, match="cap_max"):
            mcmc.relocate_and_grow(_model(), bad)
    with pytest.raises(RuntimeError, match="CUDA"):
        mcmc.relocate_and_grow(_model(), 100)
    with pytest.raises(RuntimeError, match="CUDA"):
        mcmc.inject_noise(_model())
    m = _model()
    m.optimizer.param_groups[0]["name"] = "bogus"
    with pytest.raises(KeyError, match="relocate_and_grow"):
        mcmc.relocate_and_grow(m, 100)
    assert lib.r3dg_launch_count() == n0


def test_install_uninstall_and_the_densify_conflict():
    from relightable3dgaussian_b200 import densify, mcmc

    class M(mo.StandIn):
        pass
    names = ("densify_and_prune", "add_densification_stats", "reset_opacity", "step")
    orig = {n: getattr(M, n) for n in names}
    with pytest.raises(ValueError):
        mcmc.install(M, cap_max=-1)
    assert mcmc.install(M, cap_max=1000) is M
    try:
        assert mcmc.installed_on() is M
        assert all(getattr(M, n) is not orig[n] for n in names)
        with pytest.raises(RuntimeError, match="already installed"):
            mcmc.install(M, cap_max=1000)
        with pytest.raises(RuntimeError, match="mcmc.install"):
            densify.install(M)
        assert densify._saved is None
        m = _model()
        m.__class__ = M
        assert m.add_densification_stats(None, None, None) is None
        before = m._opacity.detach().clone()
        m.reset_opacity()
        assert torch.equal(m._opacity, before)
    finally:
        mcmc.uninstall()
    assert mcmc.installed_on() is None
    assert all(getattr(M, n) is orig[n] for n in names) and not any(n in M.__dict__ for n in names)
    densify.install(M)
    try:
        with pytest.raises(RuntimeError, match="densify.install"):
            mcmc.install(M, cap_max=1000)

        class Other(mo.StandIn):
            pass
        mcmc.install(Other, cap_max=10)                          # another class is fine
        mcmc.uninstall()
    finally:
        densify.uninstall()

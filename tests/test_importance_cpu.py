"""The importance sampler's fp64 oracle (importance64.py) against the header's definitions and the rendering equation,
and every host and C refusal.  No GPU."""
import math

import numpy as np
import pytest
import torch

import importance64 as I
from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200.shading import EnvSampler, importance_sample, rendering_equation_views


class FixedLight:
    def __init__(self, envmap, transform=None):
        self.envmap, self.transform = envmap, transform


def sphere_grid(nt, nphi):
    """midpoint (theta, phi) grid over the sphere: directions [nt,nphi,3] and solid angles [nt,1]"""
    th = (np.arange(nt) + 0.5) * (math.pi / nt)
    ph = (np.arange(nphi) + 0.5) * (2 * math.pi / nphi)
    d = np.stack([np.sin(th)[:, None] * np.cos(ph), np.sin(th)[:, None] * np.sin(ph), np.cos(th)[:, None] * np.ones_like(ph)], -1)
    return d, (np.sin(th) * (math.pi / nt) * (2 * math.pi / nphi))[:, None]


def random_env(He, We, seed):
    g = np.random.default_rng(seed)
    env = g.gamma(0.5, 1.0, (He, We, 3))
    env[He // 3, We // 4] = 500.0
    return env


# ---- table ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("He,We", [(2, 2), (2, 3), (5, 9), (64, 128), (33, 70)])
def test_table_pdf_integrates_to_one(He, We):
    tab = I.build_table(random_env(He, We, He * We))
    assert abs((tab["pdf"] * I.cell_solid_angle(He, We)[:, None]).sum() - 1) <= 1e-12
    assert np.all(np.diff(tab["row_cdf"]) >= 0) and np.all(np.diff(tab["col_cdf"], axis=1) >= 0)


def test_zero_env_is_uniform_on_the_sphere():
    for env in (np.zeros((16, 33, 3)), np.full((16, 33, 3), -1.0), np.full((16, 33, 3), np.nan)):
        tab = I.build_table(env)
        assert np.abs(tab["pdf"] * 4 * math.pi - 1).max() <= 1e-4         # the fp32 CDFs' rounding of small rows


def test_dark_cell_next_to_a_source_keeps_its_weight():
    env = np.zeros((9, 17, 3))
    env[4, 8] = 1.0
    tab = I.build_table(env)
    assert (tab["weight"] > 0).sum() == 9                # the source's 3 x 3 neighbourhood
    env = np.zeros((9, 17, 3))
    env[4, 16] = 1.0                                      # the seam column: azimuth 0
    tab = I.build_table(env)
    assert tab["weight"][4, 0] > 0 and tab["weight"][4, 1] > 0 and tab["weight"][4, 15] > 0


# ---- numbers --------------------------------------------------------------------------------------------------------
def test_lattice_numbers_follow_the_integer_formulas():
    def lb(x):
        x ^= x >> 16; x = (x * 0x7FEB352D) & 0xFFFFFFFF; x ^= x >> 15; x = (x * 0x846CA68B) & 0xFFFFFFFF; x ^= x >> 16
        return x
    for seed, q, s, n in ((0, 0, 0, 1), (7, 12345, 1, 13), (2 ** 32 - 1, 2 ** 31 + 5, 2, 64)):
        u1, u2 = I.lattice(seed, [q], s, n)
        h = lb(lb(lb(seed) ^ q) ^ s)
        h1, h2 = lb(h ^ 0), lb(h ^ 1)
        for k in range(n):
            a = ((k << 32) // n + h1) & 0xFFFFFFFF
            b = (k * 0x9E3779B9 + h2) & 0xFFFFFFFF
            assert u1[0, k] == (a >> 8) * 2.0 ** -24 and u2[0, k] == (b >> 8) * 2.0 ** -24
    u1, _ = I.lattice(3, [0], 0, 1000)
    assert np.ptp(np.sort(u1[0]) - np.arange(1000) / 1000) < 1.01e-3        # one point per stratum of u1


def test_counts_round_the_mix():
    assert I.counts(32) == (16, 8, 8) and I.counts(7) == (4, 1, 2) and I.counts(1, (0, 0, 1)) == (0, 0, 1)


# ---- strategy pdfs --------------------------------------------------------------------------------------------------
def test_each_strategy_pdf_integrates_to_one():
    d, w = sphere_grid(1200, 2400)
    env = random_env(16, 33, 1)
    tab = I.build_table(env)
    T = np.linalg.qr(np.random.default_rng(2).standard_normal((3, 3)))[0]
    assert abs((I.env_pdf(tab, T, d) * w).sum() - 1) < 2e-3
    n = I.normalize(np.array([0.3, -0.2, 0.9]))
    assert abs((I.cos_pdf(n, d) * w).sum() - 1) < 1e-5
    v = I.normalize(n + np.array([0.4, 0.1, 0.0]))
    for r in (0.3, 0.6, 0.9):
        V, Ns, a2 = I.ggx_frame(n[None], v[None], np.array([r]))
        # in l: the NDF's mass over the half-vectors with V.h > 0 (the others are not samples), computed in h
        nh, vh = (d * Ns[0]).sum(-1), (d * V[0]).sum(-1)
        mass = (np.where((nh > 0) & (vh > 0), a2[0] / (math.pi * (nh * nh * (a2[0] - 1) + 1) ** 2) * nh, 0) * w).sum()
        assert 0.95 < mass <= 1 + 1e-3
        assert abs((I.ggx_pdf(V[0], Ns[0], a2[0], d) * w).sum() - mass) < 2e-3, r


def _chi2(dirs, pdf, nt=12, nphi=24, sub=24):
    """chi^2 of the direction counts over an (theta, phi) grid against n times the pdf's integral over each bin"""
    th = np.arccos(np.clip(dirs[:, 2], -1, 1))
    ph = np.mod(np.arctan2(dirs[:, 1], dirs[:, 0]), 2 * math.pi)
    cnt = np.zeros((nt, nphi))
    np.add.at(cnt, (np.minimum((th / math.pi * nt).astype(int), nt - 1), np.minimum((ph / (2 * math.pi) * nphi).astype(int), nphi - 1)), 1)
    d, w = sphere_grid(nt * sub, nphi * sub)
    exp = (pdf(d) * w).reshape(nt, sub, nphi, sub).sum((1, 3)) * len(dirs)
    keep = exp >= 5
    return float((((cnt - exp) ** 2)[keep] / exp[keep]).sum()), int(keep.sum()) - 1, float(cnt[~keep].sum())


@pytest.mark.parametrize("strategy", ["env", "ggx", "cos"])
def test_directions_follow_their_pdf(strategy):
    n_s = 20000
    tab = I.build_table(random_env(16, 33, 3))
    T = np.linalg.qr(np.random.default_rng(4).standard_normal((3, 3)))[0]
    n = I.normalize(np.array([[0.2, 0.5, 0.8]]))
    v = I.normalize(n + np.array([[0.5, -0.2, 0.1]]))
    r = np.array([0.5])
    if strategy == "env":
        d, a, _ = I.sample(tab, T, n, n_s + 1, n_s, 0, 5)
        dirs, pdf = d[0, :n_s], lambda x: I.env_pdf(tab, T, x)
    elif strategy == "ggx":
        d, a, _ = I.sample(tab, T, n, n_s + 1, 0, n_s, 5, viewdirs=v, roughness=r)
        V, Ns, a2 = I.ggx_frame(n, v, r)
        ok = a[0, :n_s] > 0
        dirs, pdf = d[0, :n_s][ok], lambda x: I.ggx_pdf(V[0], Ns[0], a2[0], x)
    else:
        d, a, _ = I.sample(tab, T, n, n_s, 0, 0, 5)
        dirs, pdf = d[0], lambda x: I.cos_pdf(n[0], x)
    chi2, dof, outside = _chi2(dirs, pdf)
    assert dof > 30
    assert chi2 <= dof + 5 * math.sqrt(2 * dof), (chi2, dof)
    assert outside <= 0.05 * len(dirs)                  # counts in bins too small for the test


# ---- the estimator against the rendering equation ---------------------------------------------------------------------
@pytest.mark.parametrize("rough", [0.12, 0.5, 0.9])
def test_quality_against_the_quadrature_truth(rough, record_property):
    """The plane of the per-pixel quality test under its 1200:1 source, one pixel, N = 32 over 64 seeds: the mixture
    converges to the integral, the Fibonacci sampler does not.  Oracle numbers (CPU): RMS 0.033 / 0.056 / 0.034,
    mean within 1 standard error, Fibonacci N = 32 error 0.84 - 0.86."""
    env = I.plane_env()
    tab = I.build_table(env)
    p, n, cam = I.plane_pixel()
    tr = I.truth(env, p, n, cam, 0.5, rough, 600, 1200)
    N = 32
    ne, ng, _ = I.counts(N)
    ests = []
    for seed in range(64):
        d, a, _ = I.sample(tab, None, n[None], N, ne, ng, seed, q=[24 * 64 + 32], viewdirs=(cam - p)[None],
                           roughness=np.array([rough]))
        ests.append(I.estimate(env, p, n, cam, 0.5, rough, d[0], a[0]))
    ests = np.array(ests)
    rms = math.sqrt(np.mean([np.sum((e - tr) ** 2) / np.sum(tr ** 2) for e in ests]))
    se = ests.std(0, ddof=1) / math.sqrt(len(ests))
    fib = I.estimate(env, p, n, cam, 0.5, rough, I.fibonacci_dirs(n, N), np.full(N, 2 * math.pi))
    fib_err = float(np.linalg.norm(fib - tr) / np.linalg.norm(tr))
    record_property("rms_importance_n32", rms)
    record_property("err_fibonacci_n32", fib_err)
    assert rms <= 0.1
    assert np.all(np.abs(ests.mean(0) - tr) <= 3 * se)
    assert fib_err >= 0.8


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_host_refusals():
    env = torch.ones(8, 16, 3)
    for mix in ((0.5, 0.6, -0.1), (0.5, 0.25, 0.5), (0.5, 0.5)):
        with pytest.raises(ValueError, match="mix"):
            EnvSampler(FixedLight(env), mix=mix)
    for bad in (torch.ones(1, 16, 3), torch.ones(8, 1, 3)):
        with pytest.raises(ValueError, match="He, We >= 2"):
            EnvSampler(FixedLight(bad))
    with pytest.raises(ValueError, match="orthonormal"):
        EnvSampler(FixedLight(env, torch.eye(3) * 1.01))
    with pytest.raises(ValueError, match="one \\[3,3\\]"):
        EnvSampler(FixedLight(env, torch.eye(3).expand(2, 3, 3)))
    with pytest.raises(ValueError, match="seed"):
        EnvSampler(FixedLight(env), seed=2 ** 32)
    s = EnvSampler.__new__(EnvSampler)
    s.mix = (0.5, 0.5, 0.0)
    with pytest.raises(ValueError, match="cosine"):
        s.counts(8)
    s.mix = (0.5, 0.25, 0.25)
    with pytest.raises(ValueError, match="GGX samples need viewdirs"):
        importance_sample(torch.ones(4, 3), s, 8)
    P, N = 4, 8
    z = torch.zeros
    with pytest.raises(ValueError, match="GGX"):
        rendering_equation_views(z(P, 3), z(P, 1), z(P, 3), z(2, P, 3), z(P, 16, 3), FixedLight(env), z(P, N, 1),
                                 z(P, N, 3), z(P, N, 1), sampler=s)
    s.mix = (0.5, 0.0, 0.5)
    with pytest.raises(ValueError, match="per-view"):
        rendering_equation_views(z(P, 3), z(P, 1), z(P, 3), z(2, P, 3), z(P, 16, 3), FixedLight(env, torch.eye(3).expand(2, 3, 3)),
                                 z(P, N, 1), z(P, N, 3), z(P, N, 1), sampler=s)


def test_c_refusals_before_any_launch():
    lib = _lib.load()
    F = 0x10000
    assert lib.r3dg_env_sampler_floats(1, 8) == 0 and lib.r3dg_env_sampler_floats(8, 1) == 0
    assert lib.r3dg_env_sampler_floats(64, 128) == 4 + 2 * 64 + 3 * 65 + 64 * 128 + 64 * 127
    assert lib.r3dg_env_sampler_build(F, 1, 8, F, None) == -10001
    assert lib.r3dg_env_sampler_build(None, 8, 8, F, None) == -10001
    call = lambda P, N, n_env, n_ggx, view=F, rough=F, seed=0: lib.r3dg_sample_importance_dirs(
        P, N, F, view, rough, F, None, n_env, n_ggx, seed, F, F, None)
    assert call(4, 8, 4, 4) == -10001                   # n_cos = 0
    assert call(4, 8, 4, 2, view=None) == -10001        # GGX samples without viewdirs
    assert call(4, 8, 4, 2, rough=None) == -10001
    assert call(4, 8, -1, 2) == -10001 and call(4, 0, 0, 0) == -10001 and call(-1, 8, 4, 2) == -10001
    assert call(4, 8, 4, 2, seed=2 ** 32) == -10001
    assert call(0, 8, 4, 2) == 0                        # nothing to sample: nothing launched
    assert lib.r3dg_sample_importance_dirs(4, 8, None, F, F, F, None, 4, 2, 0, F, F, None) == -10001

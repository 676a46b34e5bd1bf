"""Deterministic mode without a GPU: the order-independent fixed-point accumulation (csrc/detacc.cuh) through its host
build r3dg_det_sum_host, checked against exact rational sums, and the C ABI fields and sizing functions of the mode."""
import ctypes
import itertools
import math
from fractions import Fraction

import numpy as np
import pytest

from relightable3dgaussian_b200 import _lib

UNIT = Fraction(1, 2 ** 48)          # resolution: every term is rounded to a multiple of 2^-48
RANGE = 2.0 ** 47                    # |term| < 2^47, larger finite terms saturate to +-Inf


def det_sum(terms):
    a = np.ascontiguousarray(np.asarray(terms, dtype=np.float32))
    out = ctypes.c_float(0.0)
    assert _lib.load().r3dg_det_sum_host(a.size, a.ctypes.data if a.size else None, ctypes.byref(out)) == 0
    return np.float32(out.value)


def f32(x):
    """Fraction -> nearest float32 (ties to even), exactly."""
    if x == 0:
        return np.float32(0.0)
    s, a = (-1 if x < 0 else 1), abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    q = a / ulp
    n = math.floor(q)
    r = q - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return np.float32(s * float(n * ulp))


def quantized(x):
    """The term as the accumulator holds it: nearest multiple of 2^-48, ties to even."""
    q = Fraction(float(np.float32(x))) / UNIT
    n = math.floor(q)
    r = q - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return n * UNIT


def check_exact(terms):
    """The result is the exact sum of the quantised terms rounded to fp32 once, and within the documented resolution
    (n * 2^-49 plus that one rounding) of the exact sum of the terms themselves."""
    got = det_sum(terms)
    exact_q = sum((quantized(x) for x in terms), Fraction(0))
    assert got.view(np.uint32) == f32(exact_q).view(np.uint32), (got, f32(exact_q))
    exact = sum((Fraction(float(np.float32(x))) for x in terms), Fraction(0))
    half_ulp = abs(Fraction(float(f32(exact))) - Fraction(float(np.nextafter(f32(exact), np.float32(np.inf))))) / 2
    assert abs(Fraction(float(got)) - exact) <= len(terms) * UNIT / 2 + half_ulp + UNIT
    return got


def check_permutations(terms, rng, k=200):
    ref = det_sum(terms).view(np.uint32)
    n = len(terms)
    perms = itertools.permutations(range(n)) if n <= 6 else (rng.permutation(n) for _ in range(k))
    for p in perms:
        assert det_sum([terms[i] for i in p]).view(np.uint32) == ref


def test_cancelling_terms_sum_to_exactly_positive_zero():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(500) * 10.0 ** rng.uniform(-12, 12, 500)).astype(np.float32)
    terms = np.concatenate([x, -x])
    rng.shuffle(terms)
    got = check_exact(terms)
    assert got.view(np.uint32) == 0                    # +0, not -0
    assert det_sum([-0.0, -0.0]).view(np.uint32) == 0
    check_permutations(terms, rng)


def test_magnitudes_spanning_the_range_and_its_edges():
    rng = np.random.default_rng(1)
    top = np.nextafter(np.float32(RANGE), np.float32(0))            # largest float below 2^47
    edges = [top, -top, np.float32(2.0 ** -48), np.float32(2.0 ** -49), np.float32(3 * 2.0 ** -50),
             np.float32(-3 * 2.0 ** -50), np.float32(2.0 ** -49 * 3), np.float32(1.0), np.float32(-1.0 - 2.0 ** -23)]
    assert det_sum([2.0 ** -49]) == 0.0                             # a tie rounds to even (0)
    assert det_sum([3 * 2.0 ** -49]) == np.float32(2 * 2.0 ** -48)  # 1.5 units -> 2
    assert det_sum([top]) == top
    for seed in range(6):
        r = np.random.default_rng(seed)
        mags = 10.0 ** r.uniform(-16, 14, 300)
        terms = list((r.choice([-1.0, 1.0], 300) * mags).astype(np.float32)) + edges
        check_exact(terms)
        check_permutations(terms, rng, 50)
    big = [top] * 100_000                                           # a total far beyond a single term's range
    assert det_sum(big) == f32(Fraction(float(top)) * 100_000)


def test_subnormal_terms():
    rng = np.random.default_rng(2)
    sub = (rng.uniform(-1, 1, 200) * 2.0 ** -130).astype(np.float32)
    assert (np.abs(sub) < np.finfo(np.float32).tiny).all() and (sub != 0).any()
    assert det_sum(sub) == 0.0                                      # far below the resolution
    terms = list(sub) + list((rng.standard_normal(50) * 1e-3).astype(np.float32))
    check_exact(terms)
    check_permutations(terms, rng, 50)


@pytest.mark.parametrize("terms,want", [
    ([1.0, np.inf], np.inf), ([-np.inf, 5.0], -np.inf), ([np.inf, np.inf, 1.0], np.inf),
    ([np.inf, -np.inf], np.nan), ([np.nan, 1.0], np.nan), ([np.nan, np.inf], np.nan), ([-np.inf, np.nan, -np.inf], np.nan),
    ([2.0 ** 47, 1.0], np.inf), ([-2.0 ** 47], -np.inf), ([1e30, -3.0], np.inf), ([2.0 ** 47, -2.0 ** 47], np.nan),
    ([np.float32(np.finfo(np.float32).max), -1.0], np.inf),
])
def test_non_finite_and_out_of_range_terms(terms, want):
    """NaN wins, +Inf with -Inf gives NaN, and a finite term outside the range saturates to +-Inf instead of wrapping."""
    rng = np.random.default_rng(3)
    got = det_sum(terms)
    if np.isnan(want):
        assert np.isnan(got)
    else:
        assert got == want
    pad = list((rng.standard_normal(5)).astype(np.float32)) + list(terms)
    check_permutations(pad, rng, 100)
    assert (np.isnan(det_sum(pad)) and np.isnan(want)) or det_sum(pad) == want


def test_bad_arguments():
    lib = _lib.load()
    out = ctypes.c_float(0)
    assert lib.r3dg_det_sum_host(-1, None, ctypes.byref(out)) == -10001
    assert lib.r3dg_det_sum_host(3, None, ctypes.byref(out)) == -10001
    assert lib.r3dg_det_sum_host(0, None, None) == -10001
    assert lib.r3dg_det_sum_host(0, None, ctypes.byref(out)) == 0 and out.value == 0.0


def test_workspace_sizes():
    lib = _lib.load()
    assert lib.r3dg_raster_fwd_det_bytes(1000) >= 8 * 1000
    rec = lambda S: 8 + 4 * ((3 + S + 3) // 4)
    for P, S in ((1, 0), (1000, 5), (1_000_000, 5), (1_500_000, 16), (6000, 24)):
        n = lib.r3dg_raster_bwd_det_bytes(P, S)
        assert 24 * P * rec(S) <= n <= 24 * P * rec(S) + P * rec(S) // 4 + 1024 and n % 256 == 0
    assert 350e6 < lib.r3dg_raster_bwd_det_bytes(1_000_000, 5) < 420e6          # "a few hundred MB" at the headline
    assert lib.r3dg_shade_det_bytes(16, 32) >= 24 * 16 * 32 * 3
    assert lib.r3dg_shade_det_bytes(0, 32) == 0


def test_zero_filled_structs_mean_the_default_mode():
    for cls in (_lib.RasterFwdArgs, _lib.RasterBwdArgs, _lib.ShadeArgs):
        a = cls()
        assert a.deterministic == 0 and not a.det_work and a.det_work_bytes == 0


FAKE = 0x10000      # never dereferenced: every call below is refused before anything is launched


def test_missing_or_short_workspace_is_refused_without_touching_the_gpu():
    lib = _lib.load()
    P, S, W, H = 100, 5, 64, 48
    a = _lib.RasterFwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.colors_precomp = a.cov3D_precomp = FAKE
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(W, H)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.deterministic = 1
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001
    a.det_work, a.det_work_bytes = FAKE, lib.r3dg_raster_fwd_det_bytes(P) - 1
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001
    b = _lib.RasterBwdArgs()
    b.P, b.S, b.W, b.H = P, S, W, H
    b.deterministic = 1
    assert lib.r3dg_raster_backward(ctypes.byref(b), None) == -10001
    b.det_work, b.det_work_bytes = FAKE, lib.r3dg_raster_bwd_det_bytes(P, S) - 1
    assert lib.r3dg_raster_backward(ctypes.byref(b), None) == -10001
    s = _lib.ShadeArgs()
    s.P, s.N, s.sh_coeffs, s.env_h, s.env_w = 10, 8, 16, 16, 32
    (s.dL_dpbr, s.dL_dbase_color, s.dL_droughness, s.dL_dviewdirs, s.dL_dincidents, s.dL_denv) = [FAKE] * 6
    s.deterministic = 1
    assert lib.r3dg_render_equation_backward(ctypes.byref(s), None) == -10001
    s.det_work, s.det_work_bytes = FAKE, lib.r3dg_shade_det_bytes(16, 32) - 1
    assert lib.r3dg_render_equation_backward(ctypes.byref(s), None) == -10001

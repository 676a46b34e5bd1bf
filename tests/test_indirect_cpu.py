"""The fp64 truth of the radiance bake and the incident-SH fit (tests/indirect64.py) on cases with a closed-form
answer: one head-on Gaussian, two overlapping ones in both index orders, a t tie, and the ridge fit against an
augmented least-squares system."""
import numpy as np
import pytest

import indirect64 as ind


def _scene(centres, opacities, colours, sigma=0.2):
    """Isotropic Gaussians facing -z, degree-0 payload of the given colours, boxes of +-3 sigma."""
    mu = np.asarray(centres, np.float64)
    P = mu.shape[0]
    inv = np.tile([1 / sigma ** 2, 0, 0, 1 / sigma ** 2, 0, 1 / sigma ** 2], (P, 1))
    nr = np.tile([0.0, 0.0, -1.0], (P, 1))
    shs = ((np.asarray(colours, np.float64) - 0.5) / ind.C0)[:, None, :]
    boxes = np.concatenate([mu - 3 * sigma, mu + 3 * sigma], axis=1)
    return mu, inv, np.asarray(opacities, np.float32), nr, shs, boxes


def _ray(z0=0.0):
    return np.array([[0.0, 0.0, z0]]), np.array([[0.0, 0.0, 1.0]])


def test_one_head_on_gaussian_gives_alpha_times_colour():
    mu, inv, op, nr, shs, boxes = _scene([[0, 0, 1.0]], [0.7], [[0.2, 0.5, 0.9]])
    L, T, h, fr = ind.bake_radiance(mu, inv, op, nr, shs, 0, boxes, *_ray())
    a = float(np.float32(0.7))
    np.testing.assert_allclose(L[0], a * np.array([0.2, 0.5, 0.9]), rtol=1e-12, atol=1e-15)
    assert T[0] == pytest.approx(1 - a, abs=1e-15) and h[0] == 1 and not fr[0]


@pytest.mark.parametrize("swap", [False, True])
def test_two_overlapping_gaussians_composite_front_to_back(swap):
    """Near red (t = 1, alpha a) in front of far green (t = 1.2, alpha b): L = a red + (1 - a) b green, whichever
    index either Gaussian has."""
    cs, ops, cols = [[0, 0, 1.0], [0, 0, 1.2]], [0.6, 0.8], [[1.0, 0, 0], [0, 1.0, 0]]
    if swap:
        cs, ops, cols = cs[::-1], ops[::-1], cols[::-1]
    mu, inv, op, nr, shs, boxes = _scene(cs, ops, cols)
    L, T, h, _ = ind.bake_radiance(mu, inv, op, nr, shs, 0, boxes, *_ray())
    a, b = float(np.float32(0.6)), float(np.float32(0.8))
    np.testing.assert_allclose(L[0], [a, (1 - a) * b, 0.0], rtol=1e-12, atol=1e-15)
    assert T[0] == pytest.approx((1 - a) * (1 - b), abs=1e-15) and h[0] == 2
    # the other order would give a different answer: the test above pins the order
    assert abs(L[0][1] - b) > 0.1


def test_equal_t_is_broken_by_gaussian_index_and_flagged():
    mu, inv, op, nr, shs, boxes = _scene([[0, 0, 1.0], [0, 0, 1.0]], [0.5, 0.5], [[1.0, 0, 0], [0, 0, 1.0]])
    L, _, h, fr = ind.bake_radiance(mu, inv, op, nr, shs, 0, boxes, *_ray())
    np.testing.assert_allclose(L[0], [0.5, 0.0, 0.25], rtol=1e-12)
    assert h[0] == 2 and fr[0]


def test_hit_rule_and_stop():
    """Back-facing, too transparent, behind t = 0.01 and outside the box: no hit.  An opaque stack stops at
    T < 1e-4 without compositing what lies behind."""
    mu, inv, op, nr, shs, boxes = _scene([[0, 0, 1.0], [0, 0, 1.5], [0, 0, 0.005], [0, 0, 2.0]],
                                         [0.9, 1.0 / 300, 0.9, 0.9], [[1, 1, 1]] * 4)
    nr[0] = [0, 0, 1.0]                                   # back-facing
    boxes[3] = [5, 5, 5, 6, 6, 6]                         # the ray misses its box
    L, T, h, _ = ind.bake_radiance(mu, inv, op, nr, shs, 0, boxes, *_ray())
    assert h[0] == 0 and T[0] == 1.0 and not L[0].any()
    mu, inv, op, nr, shs, boxes = _scene([[0, 0, 1.0 + 0.1 * k] for k in range(8)], [0.99] * 8, [[1, 1, 1]] * 8)
    L, T, h, _ = ind.bake_radiance(mu, inv, op, nr, shs, 0, boxes, *_ray())
    assert h[0] == 2 and T[0] < ind.T_MIN


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("N", [4, 64])
def test_fit_equals_augmented_lstsq(deg, N):
    rng = np.random.default_rng(deg * 10 + N)
    P, ridge = 5, 1e-3
    d = rng.normal(size=(P, N, 3))
    d[..., 2] = np.abs(d[..., 2])                         # one hemisphere, as the bake samples
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    L = rng.uniform(0, 1, size=(P, N, 3))
    got = ind.fit_incident_sh(L, d, deg, ridge)
    Y = ind.sh_basis(deg, d)
    n = (deg + 1) ** 2
    for p in range(P):
        A = np.concatenate([Y[p] / np.sqrt(N), np.sqrt(ridge) * np.eye(n)])
        rhs = np.concatenate([L[p] / np.sqrt(N), np.zeros((n, 3))])
        want = np.linalg.lstsq(A, rhs, rcond=None)[0]
        np.testing.assert_allclose(got[p], want, rtol=1e-9, atol=1e-11)

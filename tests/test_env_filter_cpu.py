"""The filtered environment lookup's definition, on its fp64 oracle (tests/envfilter64.py): level sizes, the four
pyramid properties, the exact fallback to grid_sample at footprints below a texel, and the error against a brute-force
cone mean on an HDR map with small bright sources.  No GPU; every environment is generated from a seed."""
import math

import pytest
import torch
import torch.nn.functional as F

import envfilter64 as ef
from oracle.oracle_sampling import fibonacci_sphere_sampling


@pytest.mark.parametrize("He,We,sizes", [
    (1000, 2000, [(1000, 2000), (500, 1000), (250, 500), (125, 250), (63, 125), (32, 63), (16, 32), (8, 16), (4, 8), (2, 4)]),
    (512, 1024, [(512, 1024), (256, 512), (128, 256), (64, 128), (32, 64), (16, 32), (8, 16), (4, 8), (2, 4)]),
    (250, 500, [(250, 500), (125, 250), (63, 125), (32, 63), (16, 32), (8, 16), (4, 8), (2, 4)]),
    (16, 32, [(16, 32), (8, 16), (4, 8), (2, 4)]),
    (2, 2, [(2, 2)]),
    (1, 8, [(1, 8)]),
])
def test_level_sizes(He, We, sizes):
    assert ef.level_sizes(He, We) == sizes


def hdr_env(He, We, seed, sources=12, peak=200.0):
    """A seeded HDR lat-long map: a smooth sky, texel noise and `sources` small sources up to `peak` times brighter."""
    g = torch.Generator().manual_seed(seed)
    v = torch.linspace(0, 1, He, dtype=torch.float64)[:, None, None]
    u = torch.linspace(0, 1, We, dtype=torch.float64)[None, :, None]
    sky = 0.6 + 0.4 * torch.cos(math.pi * v) * torch.tensor([0.6, 0.8, 1.0], dtype=torch.float64) + 0.1 * torch.sin(2 * math.pi * u)
    env = sky * (1 + 0.2 * torch.rand(He, We, 3, generator=g, dtype=torch.float64))
    yy, xx = torch.meshgrid(torch.arange(He, dtype=torch.float64), torch.arange(We, dtype=torch.float64), indexing="ij")
    for _ in range(sources):
        cy, cx = 0.1 * He + 0.8 * He * torch.rand(1, generator=g).item(), We * torch.rand(1, generator=g).item()
        r = 1.0 + 2.0 * torch.rand(1, generator=g).item()
        amp = peak * (0.3 + 0.7 * torch.rand(1, generator=g).item())
        dx = torch.remainder(xx - cx + We / 2, We - 1) - We / 2
        env = env + amp * torch.exp(-((yy - cy) ** 2 + dx ** 2) / (2 * r * r))[..., None]
    env[:, -1] = env[:, 0]
    return env


@pytest.mark.parametrize("He,We", [(1000, 2000), (512, 1024), (250, 500), (16, 32), (5, 9), (3, 3)])
def test_pyramid_properties(He, We):
    g = torch.Generator().manual_seed(He)
    env = torch.rand(He, We, 3, generator=g, dtype=torch.float64) * 3 + 0.1
    levels = ef.pyramid(env)
    m0 = ef.sphere_mean(levels[0])
    for l, lv in enumerate(levels):
        assert tuple(lv.shape[:2]) == ef.level_sizes(He, We)[l]
        torch.testing.assert_close(ef.sphere_mean(lv), m0, rtol=1e-12, atol=0)
        if l == 0:
            continue
        assert torch.equal(lv[:, 0], lv[:, -1]), l                         # the seam
        assert torch.equal(lv[0], lv[0, :1].expand_as(lv[0])), l           # the poles
        assert torch.equal(lv[-1], lv[-1, :1].expand_as(lv[-1])), l
    const = torch.full((He, We, 3), 0.7315, dtype=torch.float64)
    for lv in ef.pyramid(const)[1:]:
        torch.testing.assert_close(lv, const[: lv.shape[0], : lv.shape[1]], rtol=1e-14, atol=0)


def test_constant_env_is_exact_in_fp32():
    """fp64 weights normalised by their own sum, then one rounding: a constant fp32 env stays exactly that constant."""
    for c in (0.7315, 1e-3, 123.456, 2.0 ** -20):
        c32 = torch.tensor(c, dtype=torch.float32).double()
        for lv in ef.pyramid(torch.full((250, 500, 3), c32.item(), dtype=torch.float64))[1:]:
            assert torch.equal(lv.float(), torch.full_like(lv, c32.item()).float())


def test_point_lookup_below_one_texel():
    """lambda <= 0 everywhere (16x32 env, N = 4096): the filtered lookup is fp64 grid_sample(align_corners=True)."""
    g = torch.Generator().manual_seed(4)
    n = F.normalize(torch.randn(64, 3, generator=g, dtype=torch.float64), dim=-1)
    dirs, areas = fibonacci_sphere_sampling(n.float(), 4096, random_rotate=False)
    env = torch.rand(16, 32, 3, generator=g, dtype=torch.float64)
    d = dirs.reshape(-1, 3).double()
    lam = ef.lod(d, areas.reshape(-1).double() / 4096, 16, 32, 4)
    assert lam.max().item() == 0.0
    got = ef.direct_light_filtered(env, dirs.double(), areas.double())
    ref = F.grid_sample(env.permute(2, 0, 1)[None], torch.stack((-torch.atan2(d[:, 1], d[:, 0]) / math.pi,
                                                                  (torch.arccos(d[:, 2]) - 1e-6) / math.pi * 2 - 1), -1)[None, None],
                        align_corners=True)[0, :, 0].T
    assert torch.equal(got.reshape(-1, 3), ref)


def cone_means(env, d, omega, chunk=32):
    """Brute force: the solid-angle-weighted mean of the level-0 texels inside each sample's cone (solid angle omega)."""
    He, We = env.shape[0], env.shape[1]
    wt = ef.texel_weights(He, We).reshape(-1)
    pol = torch.arange(He, dtype=torch.float64) * math.pi / (He - 1)
    azi = -(2 * torch.arange(We, dtype=torch.float64) / (We - 1) - 1) * math.pi
    P, A = torch.meshgrid(pol, azi, indexing="ij")
    tex = torch.stack((torch.sin(P) * torch.cos(A), torch.sin(P) * torch.sin(A), torch.cos(P)), -1).reshape(-1, 3)
    vals = env.reshape(-1, 3)
    cos_a = 1 - omega / (2 * math.pi)
    out = []
    for s in range(0, d.shape[0], chunk):
        inside = ((d[s:s + chunk] @ tex.T) >= cos_a).double() * wt
        out.append((inside @ vals) / inside.sum(1, keepdim=True))
    return torch.cat(out)


# The filtered lookup's error against the cone mean must be at most this share of the point lookup's.  The oracle
# measures 0.137 (N = 32) and 0.048 (N = 64) on this map; the bound leaves room for other maps and seeds.
QUALITY_RATIO = 0.25


@pytest.mark.parametrize("N", [32, 64])
def test_filtered_lookup_tracks_the_cone_mean(N):
    He, We = 512, 1024
    env = hdr_env(He, We, seed=7)
    g = torch.Generator().manual_seed(N)
    n = F.normalize(torch.randn(16, 3, generator=g), dim=-1)
    dirs, areas = fibonacci_sphere_sampling(n, N, random_rotate=False)
    d = dirs.reshape(-1, 3).double()
    omega = 2 * math.pi / N
    target = cone_means(env, d, omega)
    point = ef.bilinear(env, d)
    filt = ef.direct_light_filtered(env, dirs.double(), areas.double()).reshape(-1, 3)
    rms = lambda x: torch.sqrt(((x - target) ** 2).mean()) / torch.sqrt((target ** 2).mean())
    e_point, e_filt = rms(point).item(), rms(filt).item()
    print(f"\n[env filter] N={N}: point {e_point:.3f} filtered {e_filt:.3f} ratio {e_filt / e_point:.3f}")
    assert e_filt <= QUALITY_RATIO * e_point, (e_point, e_filt)

"""The PyTorch restatement of the shading step (oracle/oracle_shading.py) pinned, in fp32 AND in fp64, to outputs and
autograd gradients of the reference's own function bodies on the adversarial cases of tests/golden/shade_edge.npz
(make_golden_shading_edge.py): zero and non-positive SH light, the GGX nom clamp, V perpendicular to N, back-facing
and n.d == 0 samples, L == -V, the env seam and poles, random-rotate sampling, EnvLight with a permutation and a
general rotation, env maps of 16x32, 24x48 and 64x128.  The fp64 restatement is the truth of the GPU tests."""
import numpy as np
import pytest
import torch

import shading_edge as se
from helpers import rel_l2

CASES = se.load_cases()
NAMES = sorted(CASES)


def test_fixture_has_every_case():
    assert set(NAMES) == {"zero_incidents", "zero_incidents_dc", "nom_clamp", "v_perp_n", "back_facing", "l_eq_minus_v",
                          "seam_poles", "seam_poles_64", "random_rotate", "envlight_perm", "envlight_rot"}
    sizes = {tuple(CASES[n]["in_env"].shape[-3:-1]) for n in NAMES}
    assert {(16, 32), (24, 48), (64, 128)} <= sizes                 # the three env-gradient modes of the backward


@pytest.mark.parametrize("name", NAMES)
def test_case_reaches_its_path(name):
    se.assert_reaches(name, se.path_stats(se.inputs(CASES[name])))


@pytest.mark.parametrize("tag", ["32", "64"])
@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_function_golden(name, tag):
    c = CASES[name]
    dtype = torch.float32 if tag == "32" else torch.float64
    rec = se.oracle_run(se.inputs(c), dtype)
    for k, v in rec.items():
        assert v.dtype == dtype, (k, v.dtype)
    # fp32: the same torch ops on the same device as the reference bodies; fp64: equal up to a few fp64 roundings
    rtol, atol, gtol = (1e-5, 1e-6, 1e-5) if tag == "32" else (1e-12, 1e-14, 1e-12)
    for k in ("pbr",) + se.EXTRAS:
        np.testing.assert_allclose(rec[k].numpy(), c[f"{tag}/{k}"], rtol=rtol, atol=atol, err_msg=k)
    for k in se.LEAVES:
        got, want = rec["grad_" + k].numpy(), c[f"{tag}/grad_{k}"]
        assert got.shape == want.shape and rel_l2(got, want) < gtol, (k, rel_l2(got, want))


@pytest.mark.parametrize("name", NAMES)
def test_env_scatter_is_grid_sample_adjoint(name):
    """The explicit fp64 scatter of the four bilinear taps (the GPU tests' per-texel truth) equals autograd's env
    gradient through grid_sample, texel by texel, relative to the texel's sum of |contribution|."""
    t = se.inputs(CASES[name])
    rec = se.oracle_run(t, torch.float64)
    He, We = rec["grad_tex"].shape[-3:-1]
    T = t.get("transform")
    e = se.env_frame(t["incident_dirs"].double(), None if T is None else T.double())
    grad, mag = se.env_scatter64(e, rec["g_light"], He, We)
    auto = rec["grad_tex"].reshape(He, We, 3)
    assert (mag > 0).sum() > 0
    assert ((grad - auto).abs() <= 1e-12 * mag).all(), float(((grad - auto).abs() - 1e-12 * mag).max())
    assert (auto[mag == 0] == 0).all()

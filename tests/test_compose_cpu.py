"""The fp64 truth of the similarity transform (tests/compose64.py): its SH basis against the reference's, the
properties of its D^l, the kernel's construction table against it, pose_from_matrix, the refusals of the C and Python
layers, and the reference's set_transform rebinding.  No GPU."""
import ctypes
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

import compose64 as C64
from helpers import ROOT, sh_case
from relightable3dgaussian_b200 import _lib, compose

FAKE = 0x10000      # never dereferenced: every call below is refused (or does nothing) before anything is enqueued
D = torch.float64


def _rot(axis, angle):
    axis = torch.as_tensor(axis, dtype=D)
    axis = axis / axis.norm()
    q = torch.cat([torch.tensor([math.cos(angle / 2)], dtype=D), math.sin(angle / 2) * axis])
    return C64.build_rotation(q)


def _random_rotations(n, seed):
    g = torch.Generator().manual_seed(seed)
    return C64.build_rotation(torch.randn(n, 4, generator=g, dtype=D))


def test_basis_matches_the_reference():
    gold = np.load(os.path.join(ROOT, "tests", "golden", "sh_eval.npz"))
    for deg in (0, 1, 2, 3):
        sh, dirs = sh_case(10_000 if deg == 3 else 1_000, seed=deg)
        got = C64.eval_sh(deg, sh.double(), dirs.double()).numpy()
        np.testing.assert_allclose(got, gold[f"deg{deg}"], rtol=1e-5, atol=2e-6)
    sh4 = torch.randn(256, 3, 25, generator=torch.Generator().manual_seed(9))
    d4 = torch.nn.functional.normalize(torch.randn(256, 3, generator=torch.Generator().manual_seed(10)), dim=-1)
    np.testing.assert_allclose(C64.eval_sh(4, sh4.double(), d4.double()).numpy(), gold["deg4_small"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("l", [1, 2, 3, 4])
def test_rotation_defines_the_rotated_function(l):
    """sum_m Y_lm(d) (D c)_m = sum_m Y_lm(R^T d) c_m at directions the fit never saw."""
    R = _random_rotations(4, l)
    g = torch.Generator().manual_seed(7)
    d = torch.nn.functional.normalize(torch.randn(100, 3, generator=g, dtype=D), dim=-1)
    c = torch.randn(2 * l + 1, generator=g, dtype=D)
    sl = slice(l * l, (l + 1) ** 2)
    for k in range(4):
        Dl = C64.sh_rotation(R[k], l)
        lhs = C64.sh_basis(d)[:, sl] @ (Dl @ c)
        rhs = C64.sh_basis(d @ R[k])[:, sl] @ c
        torch.testing.assert_close(lhs, rhs, rtol=0, atol=1e-12)


@pytest.mark.parametrize("l", [1, 2, 3, 4])
def test_rotation_properties(l):
    R = _random_rotations(8, 10 + l)
    I = torch.eye(2 * l + 1, dtype=D)
    torch.testing.assert_close(C64.sh_rotation(torch.eye(3, dtype=D), l), I, rtol=0, atol=1e-12)
    for k in range(0, 8, 2):
        D1, D2 = C64.sh_rotation(R[k], l), C64.sh_rotation(R[k + 1], l)
        torch.testing.assert_close(D1.T @ D1, I, rtol=0, atol=1e-12)
        torch.testing.assert_close(C64.sh_rotation(R[k] @ R[k + 1], l), D1 @ D2, rtol=0, atol=1e-12)
    for angle in (math.pi, 1e-6):
        for axis in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0)):
            Dl = C64.sh_rotation(_rot(axis, angle), l)
            torch.testing.assert_close(Dl.T @ Dl, I, rtol=0, atol=1e-12)


def test_band_one_is_a_signed_permutation_of_R():
    """Y_1(d) = C1 (-y, z, -x) = C1 P d, so D^1 = P R P^T."""
    P = torch.tensor([[0, -1, 0], [0, 0, 1], [-1, 0, 0]], dtype=D)
    for R in _random_rotations(5, 3):
        torch.testing.assert_close(C64.sh_rotation(R, 1), P @ R @ P.T, rtol=0, atol=1e-12)


def _generator():
    spec = importlib.util.spec_from_file_location("gen_sh_rotation_table", os.path.join(ROOT, "tools", "gen_sh_rotation_table.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_kernel_table_is_generated_and_builds_the_oracle_rotation():
    """The committed table is what the generator writes, and its construction D^l = A_l^-1 Y_l(R^T U_l) (evaluated
    here in fp64 from the header's numbers) equals the oracle's least-squares D^l."""
    gen = _generator()
    text = gen.render()
    assert open(gen.OUT).read() == text
    body = text.split("SHROT_DIRS[24][3] = {")[1]
    dirs_txt, ainv_txt = body.split("SHROT_AINV[164] = {")
    nums = lambda s: [float(v) for v in s.split("};")[0].replace("{", " ").replace("}", " ").replace(",", " ").split()]
    U = torch.tensor(nums(dirs_txt), dtype=D).reshape(24, 3)
    Ainv = torch.tensor(nums(ainv_txt), dtype=D)
    off = 0
    for l in range(1, 5):
        n = 2 * l + 1
        Al_inv = Ainv[off:off + n * n].reshape(n, n)
        Ul = U[l * l - 1:(l + 1) ** 2 - 1]
        torch.testing.assert_close(Ul.norm(dim=-1), torch.ones(n, dtype=D), rtol=0, atol=1e-15)
        for R in list(_random_rotations(3, 20 + l)) + [_rot((1, 1, 0), math.pi), _rot((0, 0, 1), 1e-6)]:
            Dl = Al_inv @ C64.sh_basis(Ul @ R)[:, l * l:(l + 1) ** 2]
            torch.testing.assert_close(Dl, C64.sh_rotation(R, l), rtol=0, atol=1e-12)
        off += n * n


# ---- pose_from_matrix ------------------------------------------------------------------------------------------------
def _similarity(R, t, s):
    M = torch.eye(4, dtype=D)
    M[:3, :3] = s * R
    M[:3, 3] = torch.as_tensor(t, dtype=D)
    return M


@pytest.mark.parametrize("axis,angle", [((1, 0, 0), 0.0), ((0, 1, 1), 1e-6), ((1, 0, 0), math.pi), ((0, 1, 0), math.pi),
                                        ((0, 0, 1), math.pi), ((1, 1, 0), math.pi), ((1, -2, 3), 2.0)])
def test_pose_from_matrix(axis, angle):
    R = _rot(axis, angle)
    for s in (1e-3, 1.0, 1e3):
        q, t, sc = compose.pose_from_matrix(_similarity(R, (0.5, -2.0, 3.0), s))
        assert q.shape == (1, 4) and t.shape == (1, 3) and sc.shape == (1,)
        torch.testing.assert_close(C64.build_rotation(q.double())[0], R, rtol=0, atol=3e-7)
        torch.testing.assert_close(t[0].double(), torch.tensor([0.5, -2.0, 3.0], dtype=D))
        assert abs(float(sc[0]) / s - 1) < 1e-6
    if angle == 1e-6:       # the rotation is not lost to rounding: the vector part carries it
        q, _, _ = compose.pose_from_matrix(_similarity(R, (0, 0, 0), 1.0))
        assert abs(2 * float(q[0, 1:].double().norm()) - 1e-6) < 1e-12


def test_pose_from_matrix_batches():
    Ms = torch.stack([_similarity(_rot((1, 1, 0), math.pi), (1, 2, 3), 2.0), _similarity(_rot((0, 0, 1), 0.3), (0, 0, 0), 1.0)])
    q, t, s = compose.pose_from_matrix(Ms)
    assert q.shape == (2, 4) and t.shape == (2, 3) and s.tolist() == pytest.approx([2.0, 1.0])


def test_pose_from_matrix_refusals():
    good = _similarity(_rot((1, 2, 3), 0.7), (1, 2, 3), 2.0)
    bad_bottom = good.clone()
    bad_bottom[3, 0] = 0.1
    shear = good.clone()
    shear[0, 1] += 0.05
    nonuniform = good @ torch.diag(torch.tensor([1.0, 1.0, 1.01, 1.0], dtype=D))
    reflection = good @ torch.diag(torch.tensor([1.0, 1.0, -1.0, 1.0], dtype=D))
    for M in (bad_bottom, shear, nonuniform, reflection, torch.zeros(4, 4, dtype=D)):
        with pytest.raises(ValueError):
            compose.pose_from_matrix(M)
    with pytest.raises(ValueError):
        compose.pose_from_matrix(torch.eye(3))
    tiny = good @ torch.diag(torch.tensor([1.0, 1.0, 1.0 + 2e-5, 1.0], dtype=D))      # inside the 1e-4 tolerance
    compose.pose_from_matrix(tiny)


# ---- refusals --------------------------------------------------------------------------------------------------------
def _args(P=300, K=2, offsets=None, n_sh=2, degrees=(3, 4), channels=(3, 1)):
    a = _lib.ComposeArgs()
    a.P, a.K = P, K
    o = offsets if offsets is not None else [0] + [P * (k + 1) // K for k in range(K)]
    a.offsets_buf = (ctypes.c_int32 * max(len(o), 1))(*o)              # alive as long as the struct
    a.offsets = ctypes.cast(a.offsets_buf, ctypes.c_void_p)
    for f in ("quat", "translation", "scale", "xyz", "normal", "rotation", "scaling", "xyz_out", "normal_out",
              "rotation_out", "scaling_out", "dL_dxyz_out", "dL_dnormal_out", "dL_drotation_out", "dL_dscaling_out",
              "dL_dxyz", "dL_dnormal", "dL_drotation", "dL_dscaling", "dL_dR", "dL_dquat", "dL_dtranslation", "dL_dscale",
              "work"):
        setattr(a, f, FAKE)
    a.n_sh = n_sh
    for i in range(3):
        a.sh_degree[i], a.sh_channels[i] = (degrees + (1, 1, 1))[i], (channels + (3, 3, 3))[i]
        a.sh[i] = a.sh_out[i] = a.dL_dsh_out[i] = a.dL_dsh[i] = FAKE
    a.work_bytes = _lib.load().r3dg_compose_work_bytes(P, K)
    return a


def test_c_layer_refuses_bad_arguments():
    lib = _lib.load()
    fwd, bwd = lib.r3dg_compose_forward, lib.r3dg_compose_backward
    keep = []

    def run(call, a):
        keep.append(a)
        return call(ctypes.byref(a), None)
    for call in (fwd, bwd):
        assert call(None, None) == -10001
        assert run(call, _args(P=-1, offsets=[0, 0, -1])) == -10001
        for K in (0, 65):
            assert run(call, _args(K=K, offsets=list(range(K + 1)))) == -10001, K
        for o in ([1, 100, 300], [0, 100, 299], [0, 200, 100, 300][:3], [0, 301, 300]):
            assert run(call, _args(offsets=o)) == -10001, o
        a = _args()
        a.offsets = None
        assert run(call, a) == -10001
        assert run(call, _args(n_sh=4)) == -10001 and run(call, _args(n_sh=-1)) == -10001
        assert run(call, _args(degrees=(5, 1))) == -10001 and run(call, _args(degrees=(-1, 1))) == -10001
        assert run(call, _args(channels=(2, 1))) == -10001 and run(call, _args(channels=(3, 4))) == -10001
        for field in ("quat", "translation", "scale", "xyz", "normal", "rotation", "scaling"):
            a = _args()
            setattr(a, field, None)
            assert run(call, a) == -10001, field
        a = _args()
        a.sh[1] = None
        assert run(call, a) == -10001
    for field in ("xyz_out", "normal_out", "rotation_out", "scaling_out"):
        a = _args()
        setattr(a, field, None)
        assert run(fwd, a) == -10001, field
    a = _args()
    a.sh_out[0] = None
    assert run(fwd, a) == -10001
    for field in ("dL_dxyz_out", "dL_dnormal_out", "dL_drotation_out", "dL_dscaling_out", "dL_dxyz", "dL_dnormal",
                  "dL_drotation", "dL_dscaling", "dL_dR", "dL_dquat", "dL_dtranslation", "dL_dscale", "work"):
        a = _args()
        setattr(a, field, None)
        assert run(bwd, a) == -10001, field
    for field in ("dL_dsh_out", "dL_dsh"):
        a = _args()
        getattr(a, field)[1] = None
        assert run(bwd, a) == -10001, field
    a = _args()
    a.work_bytes -= 1
    assert run(bwd, a) == -10001
    # a tensor of degree 0 has no coefficients: its pointers are not needed; P = 0 launches nothing
    a = _args(degrees=(0, 4))
    a.sh[0] = a.sh_out[0] = None
    a.P, a.offsets_buf[1], a.offsets_buf[2] = 0, 0, 0
    assert run(fwd, a) == 0
    assert run(fwd, _args(P=0, offsets=[0, 0, 0])) == 0
    assert lib.r3dg_compose_work_bytes(0, 1) == 0 and lib.r3dg_compose_work_bytes(10, 0) == 0
    assert lib.r3dg_compose_work_bytes(1000, 3) >= (1000 // 128 + 3) * 182 * 4


def test_python_layer_checks_before_launching():
    P = 4
    z3, z4 = torch.zeros(P, 3), torch.zeros(P, 4)
    q, t, s = torch.tensor([[1.0, 0, 0, 0]]), torch.zeros(1, 3), torch.ones(1)
    with pytest.raises(RuntimeError):
        compose.transform_gaussians(z3, z3, z4, z3, [torch.zeros(P, 15, 3)], q, t, s)       # CPU tensors: no fallback
    with pytest.raises(ValueError):
        compose.transform_gaussians(z3, z3, z4, z3, [torch.zeros(P, 14, 3)], q, t, s)       # not (L+1)^2 - 1 coefficients
    with pytest.raises(ValueError):
        compose.transform_gaussians(z3, z3, z4, z3, [torch.zeros(P, 35, 3)], q, t, s)       # L = 5
    with pytest.raises(ValueError):
        compose.transform_gaussians(z3, z3, z4, z3, [torch.zeros(P, 15, 2)], q, t, s)       # C = 2
    with pytest.raises(ValueError):
        compose.transform_gaussians(z3, z3, z4, z3, [torch.zeros(P, 15)], q, t, s)          # not [P,K,C]
    assert [compose._sh_degree(torch.zeros(P, n, c)) for n, c in ((0, 3), (3, 1), (8, 3), (15, 3), (24, 1))] == [0, 1, 2, 3, 4]
    with pytest.raises(ValueError):
        compose.transform_gaussians(z3, z3, z4, z3, [torch.zeros(P, 3, 1)] * 4, q, t, s)    # four SH tensors
    with pytest.raises(ValueError):
        compose.transform_gaussians(z3, z3, z3, z3, [], q, t, s)                            # rotation not [P,4]
    q2, t2, s2 = q.repeat(2, 1), t.repeat(2, 1), s.repeat(2)
    with pytest.raises(ValueError):
        compose.transform_gaussians(z3, z3, z4, z3, [], q2, t2, s2)                         # K = 2 needs offsets
    for o in ([0, 2], [0, 3, 2], [1, 2, 4], [0, 2, 5]):
        with pytest.raises(ValueError):
            compose.transform_gaussians(z3, z3, z4, z3, [], q2, t2, s2, offsets=o)
    with pytest.raises(ValueError):
        compose.transform_gaussians(z3, z3, z4, z3, [], q.repeat(65, 1), t.repeat(65, 1), s.repeat(65),
                                    offsets=[0] * 61 + [1, 2, 3, 4, 4])


# ---- the reference's set_transform -----------------------------------------------------------------------------------
class StandIn:
    """The attributes of the reference's GaussianModel that set_transform reads and writes."""

    def __init__(self, P, seed):
        g = torch.Generator().manual_seed(seed)
        self.use_pbr = True
        self._xyz = torch.nn.Parameter(torch.randn(P, 3, generator=g))
        self._normal = torch.nn.Parameter(torch.randn(P, 3, generator=g))
        self._rotation = torch.nn.Parameter(torch.randn(P, 4, generator=g))
        self._scaling = torch.nn.Parameter(torch.randn(P, 3, generator=g))
        self._shs_rest = torch.nn.Parameter(torch.randn(P, 15, 3, generator=g))
        self._incidents_rest = torch.nn.Parameter(torch.randn(P, 15, 3, generator=g))
        self._visibility_rest = torch.nn.Parameter(torch.randn(P, 15, 1, generator=g))
        self._opacity = torch.nn.Parameter(torch.randn(P, 1, generator=g))

    def set_transform(self, rotation=None, center=None, scale=None, offset=None, transform=None):
        return "original"

    def model(self):
        return {k: getattr(self, a).detach().clone() for k, a in compose.ATTRS.items()}


def _oracle_transform(xyz, normal, rotation, scaling, sh_rests, quat, translation, scale, offsets=None):
    """compose.transform_gaussians computed by the fp64 oracle, so the host logic runs without a GPU."""
    P = xyz.shape[0]
    o = offsets if offsets is not None else [0, P]
    out = C64.transform(*[t.double() for t in (xyz, normal, rotation, scaling)], [t.double() for t in sh_rests],
                        quat.reshape(-1, 4).double(), translation.reshape(-1, 3).double(),
                        torch.as_tensor(scale).reshape(-1).double(), o)
    out = [t.float() for t in out]
    return out[0], out[1], out[2], out[3], out[4:]


def test_install_rebinds_set_transform(monkeypatch):
    monkeypatch.setattr(compose, "transform_gaussians", _oracle_transform)
    R = _rot((1, 2, -1), 2.5)
    center, offset, scale = torch.tensor([0.1, -0.2, 0.3]), torch.tensor([1.0, 2.0, -3.0]), 1.7
    M = _similarity(R, (1.0, 2.0, -3.0), 1.7)
    compose.install(StandIn)
    try:
        with pytest.raises(RuntimeError):
            compose.install(StandIn)
        for kwargs, (q, t, s) in (
                (dict(transform=M.float()), compose.pose_from_matrix(M)),
                (dict(rotation=R.float(), center=center, scale=scale, offset=offset),
                 compose.pose_from_matrix(_similarity(R, offset.double() - scale * R @ center.double(), scale))),
                (dict(rotation=R.float()), compose.pose_from_matrix(_similarity(R, (0, 0, 0), 1.0))),
                (dict(offset=offset), (torch.tensor([[1.0, 0, 0, 0]]), offset[None], torch.ones(1)))):
            m = StandIn(50, 3)
            want = compose.transform(m.model(), q, t, s)
            xyz_param = m._xyz
            assert m.set_transform(**kwargs) is None
            assert m._xyz is xyz_param                      # parameters are updated in place, as the reference does
            for k, a in compose.ATTRS.items():
                torch.testing.assert_close(getattr(m, a).data, want[k], rtol=1e-5, atol=1e-5, msg=lambda s: f"{k}: {s}")
        with pytest.raises(ValueError):
            StandIn(5, 1).set_transform(scale=torch.tensor([1.0, 2.0, 1.0]))
    finally:
        compose.uninstall()
    assert StandIn(1, 0).set_transform() == "original"

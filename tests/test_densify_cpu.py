"""CPU checks of the densification test oracle and C ABI: the restatement in tests/densify_oracle.py reproduces the
reference's own densify_and_prune (tests/golden/densify.npz, make_golden_densify.py) bit for bit, the reference's
torch.normal draw equals randn * std under one seed, and the new entry points refuse bad arguments before any launch."""
import contextlib
import ctypes
import io
import os
import re

import numpy as np
import pytest
import torch

import densify_oracle as do
from helpers import GOLDEN, ROOT
from relightable3dgaussian_b200 import _lib

G = np.load(os.path.join(GOLDEN, "densify.npz"))


@pytest.mark.parametrize("name", do.FIXTURE_CASES)
def test_restatement_reproduces_reference_fixture(name):
    case = do.densify_case(name)
    m = do.build_model(case, do.StandIn)
    z = torch.as_tensor(G[f"{name}/z"])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        r = do.restate_densify_and_prune(m, z=z, **case["args"])
    a, P1, b, P2 = (int(v) for v in G[f"{name}/counts"])
    assert buf.getvalue() == f"densify_and_split_normal: {a} / {P1}\nweights_accum: {b} / {P2}\n"
    assert r["code"].numpy().tolist() == G[f"{name}/code"].tolist()
    splitrow = r["code"].numpy() % 4 >= 2
    assert np.array_equal(m._xyz.detach().numpy()[splitrow], G[f"{name}/split_xyz"])
    assert np.array_equal(m._scaling.detach().numpy()[splitrow], G[f"{name}/split_scaling"])
    for k, t in do.output_tensors(m).items():
        assert do.digest(t) == str(G[f"{name}/digest/{k}"]), k
    # the fixture's implied outputs (row code + split values) are the outputs themselves
    exp = do.expected_from_code(case, G[f"{name}/code"], G[f"{name}/split_xyz"], G[f"{name}/split_scaling"])
    for k, t in do.output_tensors(m).items():
        assert torch.equal(exp[k], t), k


def test_restatement_draws_with_torch_normal():
    """The reference's torch.normal(mean=0, std) is normal_(0, 1) then mul_(std).add_(mean): randn((n, 3)) * std."""
    std = torch.rand(37, 3) + 0.01
    torch.manual_seed(1234)
    a = torch.normal(mean=torch.zeros(37, 3), std=std)
    torch.manual_seed(1234)
    z = torch.randn((37, 3))
    assert torch.equal(a, z * std + 0)
    torch.manual_seed(1234)
    torch.normal(mean=torch.zeros(0, 3), std=torch.zeros(0, 3))
    b = torch.randn(5)
    torch.manual_seed(1234)
    assert torch.equal(b, torch.randn(5))          # an empty draw consumes nothing


def test_restatement_default_sampler_matches_injected():
    case = do.densify_case("s1_p2049")
    m1, m2 = do.build_model(case, do.StandIn), do.build_model(case, do.StandIn)
    torch.manual_seed(7)
    r1 = do.restate_densify_and_prune(m1, verbose=False, **case["args"])
    r2 = do.restate_densify_and_prune(m2, z=r1["z"], verbose=False, **case["args"])
    for k, t in do.output_tensors(m1).items():
        assert torch.equal(t, do.output_tensors(m2)[k]), k


def test_abi_structs_match_header():
    hdr = open(os.path.join(ROOT, "include", "r3dg_b200.h")).read()
    for cname, cls in (("r3dg_densify_tensor", _lib.DensifyTensor), ("r3dg_densify_thresholds", _lib.DensifyThresholds)):
        body = re.search(r"typedef struct " + cname + r" \{(.*?)\} " + cname + ";", hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if decl:
                names = re.sub(r"^(const\s+)?(float|int|void|long long)\s*\**", "", decl)
                fields += [n.replace("*", "").strip() for n in names.split(",")]
        assert fields == [f[0] for f in cls._fields_], cname


def test_densify_entry_points_reject_bad_arguments_without_launching():
    lib = _lib.load()
    th = _lib.DensifyThresholds()
    assert lib.r3dg_densify_tmp_bytes(0) > 0 and lib.r3dg_densify_tmp_bytes(1 << 20) > 17 * (1 << 20)
    assert lib.r3dg_densify_stats(-1, None, 3, None, None, None, None, None, None, None, None, None, None) == -10001
    assert lib.r3dg_densify_stats(10, None, 3, None, None, None, None, None, None, None, None, None, None) == -10001
    assert lib.r3dg_densify_stats(0, None, 3, None, None, None, None, None, None, None, None, None, None) == 0
    assert lib.r3dg_densify_classify(10, None, None, None, None, None, None, None, None, 0, None, None) == -10001
    assert lib.r3dg_densify_classify(10, None, None, None, None, None, None, ctypes.byref(th), None, 0, None, None) == -10001
    tot = (ctypes.c_int * 7)(5, 0, 0, 0, 0, 0, 0)
    assert lib.r3dg_densify_apply(10, tot, 1, None, None, None, None, 0.625, None, 0, None) == -10001
    d = (_lib.DensifyTensor * 1)()
    d[0].row_bytes, d[0].kind = 6, 0                        # not a multiple of 4
    assert lib.r3dg_densify_apply(10, tot, 1, d, None, None, None, 0.625, ctypes.c_void_p(256), 1 << 20, None) == -10001
    d[0].row_bytes, d[0].kind = 16, 2                       # an xyz row must be 12 bytes
    assert lib.r3dg_densify_apply(10, tot, 1, d, None, None, None, 0.625, ctypes.c_void_p(256), 1 << 20, None) == -10001
    bad = (ctypes.c_int * 7)(11, 0, 0, 0, 0, 0, 0)          # more kept rows than rows
    assert lib.r3dg_densify_apply(10, bad, 0, None, None, None, None, 0.625, ctypes.c_void_p(256), 1 << 20, None) == -10001
    big = (_lib.DensifyTensor * 49)()
    assert lib.r3dg_densify_apply(10, tot, 49, big, None, None, None, 0.625, ctypes.c_void_p(256), 1 << 20, None) == -10001


def test_install_requires_uninstall_and_restores(monkeypatch):
    from relightable3dgaussian_b200 import densify

    class M(do.StandIn):
        pass
    orig_s, orig_d = M.add_densification_stats, M.densify_and_prune
    assert densify.install(M) is M
    try:
        assert M.densify_and_prune is not orig_d and M.add_densification_stats is not orig_s
        with pytest.raises(RuntimeError):
            densify.install(M)
    finally:
        densify.uninstall()
    assert M.densify_and_prune is orig_d and M.add_densification_stats is orig_s
    assert "densify_and_prune" not in M.__dict__       # inherited methods are not copied onto the subclass


def test_cpu_tensors_are_rejected():
    from relightable3dgaussian_b200 import densify
    case = do.densify_case("s1_p7")
    m = do.build_model(case, do.StandIn)
    with pytest.raises(RuntimeError, match="CUDA"):
        densify.densify_and_prune(m, **case["args"])

#!/usr/bin/env python3
"""Generates tests/golden/densify.npz by EXECUTING the reference's own densification code on the CPU.

`densify_and_prune`, `densify_and_clone`, `densify_and_split`, `densification_postfix`, `cat_tensors_to_optimizer`,
`_prune_optimizer`, `prune_points` and `add_densification_stats` are cut out of GaussianModel
(scene/gaussian_model.py) with `ast`, and `build_rotation` out of utils/general_utils.py; they are compiled unmodified
onto a minimal model class carrying the reference's activations (exp, sigmoid, log).  The module's `torch` is a proxy
that drops device="cuda" and records the standard normals inside `torch.normal` (normal_(0, 1), then mul_(std) and
add_(mean), as torch computes it).  Inputs come from the seeded `densify_case` of tests/densify_oracle.py with a
torch.optim.Adam state after two steps (`build_model`).  Stored per case: the row code (source row * 4 + kind: 0
original, 1 clone, 2 / 3 split copy 1 / 2), the new xyz and scaling of the split copies, z, the two printed counts
and a sha256 digest of every output tensor.  The reference tree is absent on the GPU machine: only outputs are
committed.

    python tests/golden/make_golden_densify.py [reference root]
"""
import ast
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import densify_oracle as do  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
METHODS = ["densify_and_prune", "densify_and_clone", "densify_and_split", "densification_postfix",
           "cat_tensors_to_optimizer", "_prune_optimizer", "prune_points", "add_densification_stats"]
RECORD = []


class _TorchCPU(types.ModuleType):
    """`torch` whose factory functions ignore device="cuda" and whose `normal` records its standard normals."""

    def __getattr__(self, name):
        attr = getattr(torch, name)
        if name in ("zeros", "ones", "empty", "tensor", "zeros_like"):
            def f(*a, **k):
                if k.get("device") == "cuda":
                    k["device"] = "cpu"
                return attr(*a, **k)
            return f
        if name == "normal":
            def normal(mean, std):
                z = torch.empty_like(std).normal_(0, 1)
                RECORD.append(z.clone())
                return z.mul_(std).add_(mean)
            return normal
        return attr


def cut(path, names, cls=None):
    src = open(path).read()
    body = ast.parse(src).body
    if cls is not None:
        body = next(n for n in body if isinstance(n, ast.ClassDef) and n.name == cls).body
    out = {n.name: ast.get_source_segment(src, n) for n in body if isinstance(n, ast.FunctionDef) and n.name in names}
    assert sorted(out) == sorted(names), (path, names, sorted(out))
    return out


def reference_class():
    import textwrap
    ns = dict(torch=_TorchCPU("torch"), nn=torch.nn)
    for s in cut(os.path.join(REF, "utils", "general_utils.py"), ["build_rotation"]).values():
        exec(compile(s, "general_utils.py", "exec"), ns)
    for s in cut(os.path.join(REF, "scene", "gaussian_model.py"), METHODS, "GaussianModel").values():
        exec(compile(textwrap.dedent(s), "gaussian_model.py", "exec"), ns)

    class RefModel(do.StandIn):
        scaling_inverse_activation = staticmethod(torch.log)
    for n in METHODS:
        setattr(RefModel, n, ns[n])
    return RefModel


def main():
    RefModel = reference_class()
    rec = {}
    for name in do.FIXTURE_CASES:
        case = do.densify_case(name)
        m = do.build_model(case, RefModel)
        P = case["P"]
        torch.manual_seed(case["seed"])
        RECORD.clear()
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            m.densify_and_prune(**case["args"])
        lines = buf.getvalue().split("\n")
        a = [int(x) for x in lines[0].split(":")[1].split("/")]
        b = [int(x) for x in lines[1].split(":")[1].split("/")]
        assert len(RECORD) == 1
        z = RECORD[0]
        # row code: every row's rotation identifies its source (rotations are unique random rows and copied raw);
        # split copies have a new scaling, clones zero xyz moments (xyz always has state), copies come in two halves
        rot_in = {bytes(r): i for i, r in enumerate(case["params"]["rotation"].numpy())}
        out = do.output_tensors(m)
        rot = out["param/rotation"].numpy()
        src = np.array([rot_in[bytes(r)] for r in rot], dtype=np.int64)
        sc_in = case["params"]["scaling"].numpy()
        is_split = np.any(out["param/scaling"].numpy() != sc_in[src], axis=1)
        m_xyz = out["exp_avg/xyz"].numpy()
        is_clone = ~is_split & ~np.any(m_xyz != 0, axis=1)
        kind = np.where(is_clone, 1, 0)
        sp = np.flatnonzero(is_split)
        kind[sp[len(sp) // 2:]] = 3
        kind[sp[: len(sp) // 2]] = 2
        code = (src * 4 + kind).astype(np.int32)
        rec[f"{name}/code"] = code
        rec[f"{name}/split_xyz"] = out["param/xyz"].numpy()[is_split]
        rec[f"{name}/split_scaling"] = out["param/scaling"].numpy()[is_split]
        rec[f"{name}/z"] = z.numpy()
        rec[f"{name}/counts"] = np.array(a + b, dtype=np.int64)
        for k, t in out.items():
            rec[f"{name}/digest/{k}"] = np.array(do.digest(t))
        print(f"{name:18s} P {P:6d} -> {len(code):6d}  |S| {z.shape[0] // 2:5d}  prints {a} {b}")
    path = os.path.join(HERE, "densify.npz")
    np.savez_compressed(path, **rec)
    print(f"wrote {path}: {os.path.getsize(path) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()

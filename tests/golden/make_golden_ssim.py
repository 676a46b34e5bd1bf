#!/usr/bin/env python3
"""Generates tests/golden/ssim.npz by EXECUTING the reference's own SSIM (CPU): `gaussian`,
`create_window`, `ssim` and `_ssim` (/root/reference/utils/loss_utils.py:20-63) are cut out of the
file with `ast` and compiled unmodified (the module itself imports kornia, which is absent here).
Every case of tests/ssim_oracle.py:GOLDEN_CASES runs in fp32 and in fp64; autograd supplies the
gradients with respect to both images.  Only outputs are stored: the inputs are regenerated from the
seeded `ssim_case`.  /root/reference is absent on the GPU machine: only the outputs are committed."""
import ast
import os
import sys
from math import exp

import numpy as np
import torch
import torch.nn.functional as F
from torch.autograd import Variable

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from ssim_oracle import GOLDEN_CASES, ssim_case, value_and_grads  # noqa: E402

REF = "/root/reference"
NAMES = ["gaussian", "create_window", "ssim", "_ssim"]


def cut(path, names):
    src = open(path).read()
    out = [ast.get_source_segment(src, n) for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(out) == len(names), (path, names)
    return out


ns = dict(torch=torch, F=F, Variable=Variable, exp=exp)
for s in cut(os.path.join(REF, "utils/loss_utils.py"), NAMES):
    exec(compile(s, "loss_utils.py", "exec"), ns)


def ref(a, b, size_average):
    return ns["ssim"](a, b, size_average=size_average)


rec = {"window1d": ns["gaussian"](11, 1.5).numpy()}
for name, kind, shape, size_average, seed in GOLDEN_CASES:
    a, b, cot = ssim_case(kind, shape, seed)
    for tag, dt in (("32", torch.float32), ("64", torch.float64)):
        v, ga, gb = value_and_grads(ref, a, b, cot, size_average, dt)
        rec[f"{name}/value{tag}"] = v.numpy()
        rec[f"{name}/grad1_{tag}"] = ga.numpy()
        rec[f"{name}/grad2_{tag}"] = gb.numpy()
    print(f"{name:16s} {tuple(shape)} ssim {np.asarray(rec[f'{name}/value64']).ravel()[:2]}")
path = os.path.join(HERE, "ssim.npz")
np.savez_compressed(path, **rec)
print(f"wrote {path}: {os.path.getsize(path) / 1e3:.0f} kB")

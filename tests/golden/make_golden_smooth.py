#!/usr/bin/env python3
"""Generates tests/golden/smooth.npz by EXECUTING the reference's own smoothness regularisers (CPU):
`first_order_edge_aware_loss` and `tv_loss` (/root/reference/utils/loss_utils.py:104-105,113-117) are
cut out of the file with `ast` and compiled unmodified (the module itself imports kornia, which is absent
here).  The one piece not executed from upstream code is kornia's `spatial_gradient`, which the bodies
call: it is bound to the restatement in tests/smooth_oracle.py (Sobel / 8, replicate padding, as in
kornia 0.6.12, the version the reference's readme pins).  Every case of smooth_oracle.EDGE_CASES and
TV_CASES runs in fp32 and in fp64; autograd supplies the gradients with respect to every input.  Only
outputs are stored: the inputs are regenerated from the seeded `smooth_case` / `tv_case`.
/root/reference is absent on the GPU machine: only the outputs are committed."""
import ast
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import smooth_oracle as so  # noqa: E402

REF = "/root/reference"
NAMES = ["first_order_edge_aware_loss", "tv_loss"]


def cut(path, names):
    src = open(path).read()
    out = [ast.get_source_segment(src, n) for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(out) == len(names), (path, names)
    return out


ns = dict(torch=torch, spatial_gradient=so.spatial_gradient)
for s in cut(os.path.join(REF, "utils/loss_utils.py"), NAMES):
    exec(compile(s, "loss_utils.py", "exec"), ns)

rec = {}
for name, kind, Cd, Ci, H, W, seed in so.EDGE_CASES:
    d, i, cot = so.smooth_case(kind, Cd, Ci, H, W, seed)
    for tag, dt in (("32", torch.float32), ("64", torch.float64)):
        v, (gd, gi) = so.value_and_grads(ns["first_order_edge_aware_loss"], [d, i], cot, dt)
        rec[f"edge/{name}/value{tag}"] = v.numpy()
        rec[f"edge/{name}/grad_data{tag}"] = gd.numpy()
        rec[f"edge/{name}/grad_img{tag}"] = gi.numpy()
    print(f"edge {name:16s} {Cd}x{Ci} {H}x{W} L {float(rec[f'edge/{name}/value64']):.6e}")
for name, shape, permuted, seed in so.TV_CASES:
    x, cot = so.tv_case(shape, permuted, seed)
    for tag, dt in (("32", torch.float32), ("64", torch.float64)):
        v, (gx,) = so.value_and_grads(ns["tv_loss"], [x], cot, dt)
        rec[f"tv/{name}/value{tag}"] = v.numpy()
        rec[f"tv/{name}/grad{tag}"] = gx.numpy()
    print(f"tv   {name:16s} {shape} L {float(rec[f'tv/{name}/value64']):.6e}")
path = os.path.join(HERE, "smooth.npz")
np.savez_compressed(path, **rec)
print(f"wrote {path}: {os.path.getsize(path) / 1e3:.0f} kB")

"""Sweep the compositors' resident-CTAs-per-SM knobs (r3dg_tune composite_fwd_ctas / composite_bwd_ctas): per
setting, mean stage times of the raster fwd+bwd over a few views.  TAG labels the output lines.
usage: python tools/residency_sweep.py TAG P W H S "f,b f,b ..." """
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
STAGES = ["project", "depth_sort", "bin_count", "bin_offsets", "bin_scatter", "composite_fwd", "surface_normal", "composite_bwd", "project_bwd"]


def main():
    from relightable3dgaussian_b200 import _C_raster, _lib
    from helpers import case_inputs
    tag = sys.argv[1]
    P, W, H, S = (int(x) for x in sys.argv[2:6])
    settings = [tuple(int(v) for v in s.split(",")) for s in sys.argv[6].split()]
    lib = _lib.load()
    d = lambda t: t.cuda().contiguous()
    e = torch.Tensor([])
    views = []
    for v in range(4):
        sc, cam = case_inputs(P, W, H, S, view=v)
        views.append(cam)
    g = torch.Generator().manual_seed(1)
    cots = [d(torch.randn(c, H, W, generator=g)) for c in (3, 1, 1, S)]
    base = (d(torch.zeros(3)), d(sc.means3D), d(sc.features) if S else torch.empty(P, 0, device="cuda"), e, d(sc.opacities), d(sc.scales), d(sc.rotations))
    shs = d(sc.shs)

    def step(cam):
        a = base + (1.0, e, d(cam.viewmatrix), d(cam.projmatrix), cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, H, W, shs, 3, d(cam.campos), False, True, False)
        out = _C_raster.rasterize_gaussians(*a)
        _C_raster.rasterize_gaussians_backward(a[0], a[1], a[2], out[9], e, a[5], a[6], 1.0, e, a[9], a[10], cam.tanfovx, cam.tanfovy, *cots, shs, 3,
                                               a[19], out[10], out[0], out[11], out[12], True, False)

    for f, b in settings:
        _lib.tune("composite_fwd_ctas", f)
        _lib.tune("composite_bwd_ctas", b)
        for i in range(4):
            step(views[i % 4])
        torch.cuda.synchronize()
        n = 16
        lib.r3dg_prof_begin(n)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            step(views[i % 4])
        e1.record()
        torch.cuda.synchronize()
        arr = (ctypes.c_float * 9)()
        nf, nb = ctypes.c_int(0), ctypes.c_int(0)
        lib.r3dg_prof_end(arr, ctypes.byref(nf), ctypes.byref(nb))
        st = {k: arr[i] / max(nf.value if i < 7 else nb.value, 1) for i, k in enumerate(STAGES)}
        print(json.dumps(dict(tag=tag, P=P, W=W, H=H, S=S, fwd_ctas=f, bwd_ctas=b, step_ms=round(e0.elapsed_time(e1) / n, 4),
                              composite_fwd=round(st["composite_fwd"], 4), composite_bwd=round(st["composite_bwd"], 4))), flush=True)


if __name__ == "__main__":
    main()

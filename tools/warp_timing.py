"""Load-balance study of the two compositors (diagnostic build only).

Build the library with  R3DG_NVCC_DEFS=-DR3DG_WARP_TIMING python -m relightable3dgaussian_b200.build --force , run this
on an H100: one fwd+bwd of the headline view with every compositor warp recording (start, end, entries composited, SM);
prints the makespan against the per-SM busy time and the heaviest warps, and stores the raw table in gpurun_out/."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    from relightable3dgaussian_b200 import _C_raster, _lib
    from helpers import case_inputs
    P, W, H, S = (int(x) for x in (sys.argv[1:5] or (1_000_000, 800, 800, 5)))
    lib = _lib.load()
    sc, cam = case_inputs(P, W, H, S, view=0)
    d = lambda t: t.cuda().contiguous()
    e = torch.Tensor([])
    args = (d(torch.zeros(3)), d(sc.means3D), d(sc.features) if S else torch.empty(P, 0, device="cuda"), e, d(sc.opacities), d(sc.scales),
            d(sc.rotations), 1.0, e, d(cam.viewmatrix), d(cam.projmatrix), cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, H, W, d(sc.shs), 3,
            d(cam.campos), False, True, False)
    g = torch.Generator().manual_seed(1)
    cots = [d(torch.randn(c, H, W, generator=g)) for c in (3, 1, 1, S)]
    for _ in range(3):
        out = _C_raster.rasterize_gaussians(*args)
        _C_raster.rasterize_gaussians_backward(args[0], args[1], args[2], out[9], e, args[5], args[6], 1.0, e, args[9], args[10], cam.tanfovx,
                                               cam.tanfovy, *cots, args[17], 3, args[19], out[10], out[0], out[11], out[12], True, False)
    torch.cuda.synchronize()
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    n = tiles * 2 * 4
    dt = np.dtype([("t0", "<u8"), ("t1", "<u8"), ("iters", "<u4"), ("smid", "<u4")])
    res = {}
    for name in ("fwd", "bwd"):
        buf = np.zeros(n, dtype=dt)
        fn = getattr(lib, f"r3dg_debug_wt_{name}")
        fn.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
        rc = fn(buf.ctypes.data, buf.nbytes)
        assert rc == 0, rc
        t0, t1 = buf["t0"].astype(np.int64), buf["t1"].astype(np.int64)
        start = t0.min()
        span = (t1.max() - start) / 1e3
        dur = (t1 - t0) / 1e3
        order = np.argsort(-dur)
        sm_busy = {}
        for s in np.unique(buf["smid"]):
            m = buf["smid"] == s
            sm_busy[int(s)] = ((t1[m].max() - start) / 1e3)
        last = np.array(sorted(sm_busy.values()))
        res[name] = dict(makespan_us=float(span), warps=int(n), warp_us_sum=float(dur.sum()), warp_us_max=float(dur.max()),
                         warp_us_p99=float(np.percentile(dur, 99)), warp_us_median=float(np.median(dur)),
                         iters_total=int(buf["iters"].sum()), iters_max=int(buf["iters"].max()),
                         sm_finish_us=dict(min=float(last.min()), median=float(np.median(last)), max=float(last.max())),
                         top=[dict(warp=int(i), cta=int(i // 4), start_us=float((t0[i] - start) / 1e3), dur_us=float(dur[i]), iters=int(buf["iters"][i]))
                              for i in order[:12]],
                         ns_per_iter_top=float(dur[order[:50]].sum() * 1e3 / max(1, buf["iters"][order[:50]].sum())))
        np.save(os.path.join(ROOT, "gpurun_out", f"warp_timing_{name}.npy"), buf)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    main()

"""Selective against dense optimiser step, on one GPU.

Adam alone: the stage-1 group layout (7 groups, 62 floats per Gaussian) at 1M Gaussians and the stage-2 layout (the 11
groups that get gradients, 114 floats) at 1.5M, each stepped densely and with a row mask.  The masks are the real
`weights > 0` of the benchmark scenes (shell-v1, camera 0: 1M at 800x800 and 1.5M at 1600x1200, rendered here) and
random masks of fixed density.  The Gaussians of the scene are in random index order, so a random mask of the same
density is a fair stand-in.  Each arm is the library call on a prebuilt descriptor table (the kernel, without
FusedAdam's per-step Python), timed with CUDA events over `iters` calls; the arms alternate and the median of `rounds`
is reported.  Beside each time: the bytes a 32-byte-sector model of the mask says the step must move (every touched
sector of p, g, m, v read and of p, m, v written, plus one mask byte per row and tensor) and the rate over them.

A stage-1 training step at the headline: GaussianRasterizer forward, L1 loss, backward, FusedAdam.step over the 7
groups, densely and with `visibility=weights[:, 0] > 0`, in steps/s.  The parameters enter the rasterizer as they are
(no activations), and every group's lr is 0 so that both arms render the same scene at every step (the optimiser's
work does not depend on lr).  Prints one JSON line that starts with the device name and power limit read in the same run.

    python tools/bench_selective_adam.py [--rounds 3] [--iters 200] [--train-steps 50]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_views import device_info, timed  # noqa: E402
from relightable3dgaussian_b200 import _lib, synth  # noqa: E402
from relightable3dgaussian_b200.optim import FusedAdam  # noqa: E402
from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer  # noqa: E402

# the reference's per-Gaussian groups (scene/gaussian_model.py): name, floats per row, lr
STAGE1 = [("xyz", 3, 1.6e-4), ("normal", 3, 1e-3), ("rotation", 4, 1e-3), ("scaling", 3, 5e-3), ("opacity", 1, 5e-2),
          ("f_dc", 3, 2.5e-3), ("f_rest", 45, 2.5e-3 / 20)]
STAGE2 = STAGE1 + [("base_color", 3, 1e-2), ("roughness", 1, 1e-2), ("incidents_dc", 3, 2e-3),
                   ("incidents_rest", 45, 1e-4)]
SCENES = {"1M_800x800": (1_000_000, 800, 800, 5), "1.5M_1600x1200": (1_500_000, 1600, 1200, 16)}
LAYOUTS = {"stage1_1M": (STAGE1, "1M_800x800"), "stage2_1.5M": (STAGE2, "1.5M_1600x1200")}
DENSITIES = (0.0, 0.14, 0.17, 0.31, 0.78, 1.0)


def settings(W, H, cam):
    return GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, torch.zeros(3, device="cuda"),
                                         1.0, cam.viewmatrix.cuda(), cam.projmatrix.cuda(), 3, cam.campos.cuda(),
                                         False, True, True, False)


def scene_mask(P, W, H, S):
    """`weights > 0` of camera 0 of the benchmark scene."""
    sc = synth.make_scene(P, "shell-v1", 0, S)
    d = lambda t: t.cuda().contiguous()
    with torch.no_grad():
        out = GaussianRasterizer(settings(W, H, synth.make_camera(0, W, H)))(
            d(sc.means3D), torch.zeros(P, 3, device="cuda"), d(sc.opacities), shs=d(sc.shs), scales=d(sc.scales),
            rotations=d(sc.rotations), features=d(sc.features))
    return out[8][:, 0] > 0


def sector_bytes(mask, widths):
    """Bytes of a masked step over tensors of `widths` floats per row under the sector model."""
    P = mask.shape[0]
    total, cache = 0, {}
    for w in widths:
        if w not in cache:
            n = P * w
            on = mask[torch.arange(n, device="cuda") // w]
            on = torch.nn.functional.pad(on, (0, (-n) % 8))
            cache[w] = int(on.view(-1, 8).any(1).sum()) * 32 * 7 + P
        total += cache[w]
    return total


def adam_table(layout, P, mask):
    gen = torch.Generator(device="cuda").manual_seed(0)
    keep, entries = [], []
    for _, w, lr in layout:
        p, g = (torch.randn(P, w, device="cuda", generator=gen) for _ in range(2))
        g *= 1e-3
        m, v = torch.zeros_like(p), torch.zeros_like(p)
        keep += [p, g, m, v]
        e = _lib.AdamTensor()
        e.param, e.grad, e.exp_avg, e.exp_avg_sq = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()
        e.n, e.step, e.lr, e.beta1, e.beta2, e.eps = p.numel(), 1, lr, 0.9, 0.999, 1e-15
        if mask is not None:
            e.row_mask, e.row_elems = mask.data_ptr(), w
        entries.append(e)
    arr = (_lib.AdamTensor * len(entries))(*entries)

    def run():
        _lib.call("r3dg_adam_step", torch.device("cuda"), len(entries), arr, what="bench")
    run.keep = keep
    return run


def bench_adam(args, masks):
    res = {}
    for lname, (layout, sname) in LAYOUTS.items():
        P = SCENES[sname][0]
        widths = [w for _, w, _ in layout]
        dense_bytes = 28 * P * sum(widths)
        cases = {"weights>0": masks[sname]}
        gen = torch.Generator(device="cuda").manual_seed(1)
        cases.update({f"random_{round(d * 100)}%": torch.rand(P, device="cuda", generator=gen) < d for d in DENSITIES})
        dense = adam_table(layout, P, None)
        for cname, mask in cases.items():
            mask = mask.contiguous().view(torch.uint8)
            sel = adam_table(layout, P, mask)
            ms = {"dense": [], "selective": []}
            for _ in range(args.rounds):
                ms["dense"].append(timed(dense, args.iters))
                ms["selective"].append(timed(sel, args.iters))
            d, s = statistics.median(ms["dense"]), statistics.median(ms["selective"])
            b = sector_bytes(mask.bool(), widths)
            res[f"{lname}_{cname}"] = {
                "rows_on": round(float(mask.float().mean()), 4), "dense_ms": round(d, 4), "selective_ms": round(s, 4),
                "speedup": round(d / s, 3), "dense_GBps": round(dense_bytes / d / 1e6, 1),
                "model_bytes_fraction": round(b / dense_bytes, 4), "selective_GBps_over_model": round(b / s / 1e6, 1),
                "dense_ms_rounds": [round(x, 4) for x in ms["dense"]],
                "selective_ms_rounds": [round(x, 4) for x in ms["selective"]]}
            del sel
        del dense
        torch.cuda.empty_cache()
    return res


def train_arm(P, W, H, S, selective):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    d = lambda t: t.cuda().contiguous().requires_grad_(True)
    prm = {"xyz": d(sc.means3D), "normal": d(sc.normals), "rotation": d(sc.rotations), "scaling": d(sc.scales),
           "opacity": d(sc.opacities), "f_dc": d(sc.shs[:, :1]), "f_rest": d(sc.shs[:, 1:])}
    aux = sc.features[:, 3:].cuda().contiguous()
    opt = FusedAdam([{"params": [prm[n]], "lr": 0.0, "name": n} for n, _, _ in STAGE1], lr=0.0, eps=1e-15)
    rs = settings(W, H, synth.make_camera(0, W, H))
    target = torch.rand(3, H, W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))

    def step():
        means2D = torch.zeros(P, 3, device="cuda", requires_grad=True)
        out = GaussianRasterizer(rs)(means3D=prm["xyz"], means2D=means2D, opacities=prm["opacity"],
                                     shs=torch.cat([prm["f_dc"], prm["f_rest"]], 1), scales=prm["scaling"],
                                     rotations=prm["rotation"], features=torch.cat([prm["normal"], aux], 1))
        (out[2] - target).abs().mean().backward()
        opt.step(visibility=out[8][:, 0] > 0) if selective else opt.step()
        opt.zero_grad()
    return step


def bench_train(args):
    P, W, H, S = SCENES["1M_800x800"]
    arms = {"dense": train_arm(P, W, H, S, False), "selective": train_arm(P, W, H, S, True)}
    ms = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, run in arms.items():
            ms[k].append(timed(run, args.train_steps))
    d, s = statistics.median(ms["dense"]), statistics.median(ms["selective"])
    return {"train_step_1M_800x800": {"dense_steps_per_s": round(1e3 / d, 1), "selective_steps_per_s": round(1e3 / s, 1),
                                      "dense_ms": round(d, 4), "selective_ms": round(s, 4),
                                      "dense_ms_rounds": [round(x, 4) for x in ms["dense"]],
                                      "selective_ms_rounds": [round(x, 4) for x in ms["selective"]]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--train-steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_selective_adam.py needs a CUDA GPU")
    res = device_info()
    masks = {name: scene_mask(*cfg) for name, cfg in SCENES.items()}
    res["weights>0_fraction"] = {name: round(float(m.float().mean()), 4) for name, m in masks.items()}
    torch.cuda.empty_cache()
    res.update(bench_adam(args, masks))
    res.update(bench_train(args))
    print(json.dumps(res))


if __name__ == "__main__":
    main()

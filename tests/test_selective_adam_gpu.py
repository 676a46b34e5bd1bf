"""Selective optimiser step: `FusedAdam.step(visibility=mask)` updates only the rows of per-Gaussian parameters whose
mask byte is nonzero.  Set rows are bitwise equal to the dense step from the same state, the other rows keep p,
exp_avg and exp_avg_sq bitwise (whatever their gradient holds), parameters that are not per-Gaussian take the dense
step and every step counter advances."""
import copy

import pytest
import torch

from test_adam_gpu import GROUPS
from relightable3dgaussian_b200 import _lib, synth
from relightable3dgaussian_b200.optim import FusedAdam, prune_optimizer
from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_views

pytestmark = pytest.mark.gpu

# the reference's 13 groups, a row of 15 floats, and an environment map that is not per-Gaussian
LAYOUT = [(n, shp, lr) for n, shp, lr in GROUPS] + [("extra15", (15,), 1e-3)]
ENV_SHAPE, ENV_LR = (1, 16, 32, 3), 1e-2


def make(P, seed, unaligned=False):
    g = torch.Generator().manual_seed(seed)
    params = []
    for _, shp, _ in LAYOUT:
        t = torch.randn((P,) + shp, generator=g)
        if unaligned:                               # a view one element into its buffer: the kernel's scalar path
            buf = torch.empty(t.numel() + 1, device="cuda")
            buf[1:].copy_(t.reshape(-1).cuda())
            params.append(buf[1:].view(t.shape).detach().requires_grad_(True))
        else:
            params.append(t.cuda().requires_grad_(True))
    env = torch.randn(ENV_SHAPE, generator=g).cuda().requires_grad_(True)
    groups = [{"params": [p], "lr": lr, "name": n} for p, (n, _, lr) in zip(params, LAYOUT)]
    opt = FusedAdam(groups + [{"params": [env], "lr": ENV_LR, "name": "env"}], lr=0.0, eps=1e-15)
    return params + [env], opt


def set_grads(params, P, step, seed, bad_rows=None):
    g = torch.Generator().manual_seed(1000 * seed + step)
    for p in params:
        t = torch.randn(p.shape, generator=g) * 1e-3
        if p.shape[0] == P and p.dim() > 0:
            t[::3] = 0.0
            if bad_rows is not None:                    # NaN and Inf in rows the mask leaves out
                bad = bad_rows.cpu()
                t[bad] = torch.tensor([float("nan"), float("inf"), -float("inf")])[torch.arange(int(bad.sum())) % 3].reshape(
                    (-1,) + (1,) * (t.dim() - 1))
        p.grad = t.cuda()


def dense_clone(opt):
    """A FusedAdam over clones of `opt`'s parameters, state and gradients."""
    groups, params = [], []
    for g in opt.param_groups:
        p = g["params"][0]
        q = p.detach().clone().requires_grad_(True)
        q.grad = p.grad.clone()
        params.append(q)
        groups.append({k: v for k, v in g.items() if k != "params"} | {"params": [q]})
    o = FusedAdam(groups, lr=0.0, eps=1e-15)
    for g, q in zip(opt.param_groups, params):
        st = opt.state.get(g["params"][0])
        if st:
            o.state[q] = {k: v.clone() for k, v in st.items()}
    return params, o


def snapshot(params, opt):
    return [(p.detach().clone(), *((opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone())
                                   if p in opt.state else (None, None))) for p in params]


def check_step(params, opt, P, mask, step):
    """Run opt.step(visibility=mask) and check it row by row against a dense step from the same state."""
    on = mask.reshape(-1).bool()
    before = snapshot(params, opt)
    ref_params, ref = dense_clone(opt)
    ref.step()
    opt.step(visibility=mask)
    for p, q, (p0, m0, v0), grp in zip(params, ref_params, before, opt.param_groups):
        st, rst = opt.state[p], ref.state[q]
        assert float(st["step"]) == float(rst["step"]) == step, grp["name"]
        got = (p.detach(), st["exp_avg"], st["exp_avg_sq"])
        want = (q.detach(), rst["exp_avg"], rst["exp_avg_sq"])
        if p.shape[0] != P:                                     # not per-Gaussian: the dense step
            for a, b in zip(got, want):
                assert torch.equal(a, b), grp["name"]
            continue
        for a, b in zip(got, want):
            assert torch.equal(a[on], b[on]), grp["name"]
        if m0 is None:                                          # first step: moments start at zero
            m0, v0 = torch.zeros_like(p0), torch.zeros_like(p0)
        for a, b in zip(got, (p0, m0, v0)):
            assert torch.equal(a[~on], b[~on]), grp["name"]


def random_mask(P, density, gen):
    return torch.rand(P, generator=gen, device="cuda") < density


def test_all_ones_mask_is_the_dense_step():
    P = 70_001
    pa, oa = make(P, 0)
    pb, ob = make(P, 0)
    ones = torch.ones(P, dtype=torch.bool, device="cuda")
    lib = _lib.load()
    for step in range(1, 7):
        if step == 4:
            oa.param_groups[0]["lr"] = ob.param_groups[0]["lr"] = 0.9e-4
        set_grads(pa, P, step, 0)
        set_grads(pb, P, step, 0)
        n0 = lib.r3dg_launch_count()
        oa.step(visibility=ones)
        n1 = lib.r3dg_launch_count()
        ob.step()
        assert n1 - n0 == lib.r3dg_launch_count() - n1 == 1      # 15 tensors: one launch either way
    for p, q in zip(pa, pb):
        assert torch.equal(p, q)
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(oa.state[p][k], ob.state[q][k])
        assert float(oa.state[p]["step"]) == float(ob.state[q]["step"]) == 6.0


@pytest.mark.parametrize("unaligned", [False, True])
@pytest.mark.parametrize("P", [1, 1365, 4097, 70_001])
def test_random_masks_every_step(P, unaligned):
    params, opt = make(P, 1, unaligned)
    if unaligned:
        assert all(p.data_ptr() % 16 for p in params[:-1])
    gen = torch.Generator(device="cuda").manual_seed(P)
    step = 0
    for density in (0.0, 0.17, 0.5, 1.0):
        for _ in range(2):
            step += 1
            set_grads(params, P, step, 1)
            check_step(params, opt, P, random_mask(P, density, gen), step)


@pytest.mark.parametrize("unaligned", [False, True])
def test_nan_and_inf_gradients_in_rows_left_out(unaligned):
    P = 4097
    params, opt = make(P, 2, unaligned)
    gen = torch.Generator(device="cuda").manual_seed(7)
    for step in (1, 2, 3):
        mask = random_mask(P, 0.3, gen)
        set_grads(params, P, step, 2, bad_rows=~mask)
        check_step(params, opt, P, mask, step)
        for p in params[:-1]:
            assert torch.isfinite(p).all() and torch.isfinite(opt.state[p]["exp_avg_sq"]).all()


def test_mask_forms_agree():
    P = 1365
    gen = torch.Generator(device="cuda").manual_seed(3)
    on = random_mask(P, 0.4, gen)
    u8 = on.to(torch.uint8) * torch.randint(1, 256, (P,), generator=gen, device="cuda", dtype=torch.uint8)
    forms = [on, on[:, None], on.to(torch.uint8), u8, u8[:, None]]
    results = []
    for form in forms:
        params, opt = make(P, 3)
        for step in (1, 2):
            set_grads(params, P, step, 3)
            opt.step(visibility=form)
        results.append([t.clone() for p in params for t in (p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])])
    for r in results[1:]:
        assert all(torch.equal(a, b) for a, b in zip(results[0], r))


def _scene(P, S=5):
    sc = synth.make_scene(P, "shell-v1", 0, S)
    leaves = dict(means3D=sc.means3D, opacities=sc.opacities, scales=sc.scales, rotations=sc.rotations,
                  shs=sc.shs, features=sc.features)
    params = {k: v.cuda().contiguous().requires_grad_(True) for k, v in leaves.items()}
    opt = FusedAdam([{"params": [p], "lr": 1e-3, "name": k} for k, p in params.items()], lr=0.0, eps=1e-15)
    return params, opt


def _settings(k, W, H):
    cam = synth.make_camera(k, W, H)
    return GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                         torch.tensor([0.1, 0.2, 0.3], device="cuda"), 1.0, cam.viewmatrix.cuda(),
                                         cam.projmatrix.cuda(), 3, cam.campos.cuda(), False, True, True, False)


@pytest.mark.parametrize("views", [1, 3])
def test_through_the_renderer(views):
    P, W, H = 300_000, 400, 400                        # a shell that saturates: many rows are never composited
    params, opt = _scene(P)
    plist = list(params.values())
    kw = {k: v for k, v in params.items() if k not in ("means3D", "opacities")}
    target = torch.rand(3, H, W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    for step in (1, 2):
        if views == 1:
            m2d = torch.zeros(P, 3, device="cuda", requires_grad=True)
            out = GaussianRasterizer(_settings(0, W, H))(params["means3D"], m2d, params["opacities"], **kw)
            mask = out[8][:, 0] > 0
        else:
            m2d = torch.zeros(views, P, 3, device="cuda", requires_grad=True)
            out = rasterize_views(params["means3D"], m2d, params["opacities"],
                                  settings=[_settings(k, W, H) for k in (0, 3, 5)], **kw)
            mask = (out[8] > 0).any(0)
        assert mask.any() and not mask.all()
        (out[2] - target).abs().mean().backward()
        check_step(plist, opt, P, mask, step)
        opt.zero_grad()


def test_after_densification_and_state_dict_interchange():
    P = 5000
    params, opt = make(P, 4)
    gen = torch.Generator(device="cuda").manual_seed(4)
    for step in (1, 2):
        set_grads(params, P, step, 4)
        opt.step(visibility=random_mask(P, 0.3, gen))
    keep = random_mask(P, 0.6, gen)
    new, _ = prune_optimizer(opt, keep)
    Pn = int(keep.sum())
    params = [g["params"][0] for g in opt.param_groups]
    assert all(new[g["name"]] is g["params"][0] for g in opt.param_groups[:-1])
    set_grads(params, Pn, 3, 4)
    check_step(params, opt, Pn, random_mask(Pn, 0.3, gen), 3)
    # checkpoints: a selective optimiser's state loads into torch.optim.Adam and back
    pt = [p.detach().clone().requires_grad_(True) for p in params]
    ot = torch.optim.Adam([{"params": [q], "lr": g["lr"], "name": g["name"]} for q, g in zip(pt, opt.param_groups)],
                          lr=0.0, eps=1e-15)
    ot.load_state_dict(copy.deepcopy(opt.state_dict()))
    set_grads(pt, Pn, 4, 4)
    ot.step()
    pf = [p.detach().clone().requires_grad_(True) for p in pt]
    of = FusedAdam([{"params": [q], "lr": g["lr"], "name": g["name"]} for q, g in zip(pf, opt.param_groups)],
                   lr=0.0, eps=1e-15)
    of.load_state_dict(copy.deepcopy(ot.state_dict()))
    set_grads(pf, Pn, 5, 4)
    check_step(pf, of, Pn, random_mask(Pn, 0.5, gen), 5)


def test_refusals_leave_everything_untouched():
    P = 1365
    params, opt = make(P, 5)
    set_grads(params, P, 1, 5)
    opt.step()
    set_grads(params, P, 2, 5)
    before = snapshot(params, opt)
    for bad in (torch.ones(P, dtype=torch.bool),                                   # CPU
                torch.ones(P, device="cuda"),                                       # float
                torch.ones(P + 1, dtype=torch.bool, device="cuda"),                 # no parameter has P + 1 rows
                torch.ones(P, 2, dtype=torch.bool, device="cuda")):                 # not [P] or [P, 1]
        with pytest.raises((ValueError, RuntimeError)):
            opt.step(visibility=bad)
    for p, (p0, m0, v0) in zip(params, before):
        assert torch.equal(p, p0) and torch.equal(opt.state[p]["exp_avg"], m0)
        assert torch.equal(opt.state[p]["exp_avg_sq"], v0) and float(opt.state[p]["step"]) == 1.0
    # a gradient on the environment map alone: P rows match nothing with a gradient
    for p in params[:-1]:
        p.grad = None
    with pytest.raises(ValueError):
        opt.step(visibility=torch.ones(P, dtype=torch.bool, device="cuda"))
    # no gradient at all: a no-op, as without a mask
    params[-1].grad = None
    opt.step(visibility=torch.ones(P + 7, dtype=torch.bool, device="cuda"))
    assert float(opt.state[params[0]]["step"]) == 1.0

"""GPU tests of the MCMC densification (relightable3dgaussian_b200/mcmc.py, csrc/mcmc.cu), against the restatement in
tests/mcmc_oracle.py on the same device with the same injected samples.

* relocate_and_grow: the same sources (no draw may fall within 1e-12 total of a CDF boundary, where the two fp64
  prefix sums may round apart; the count is reported), every copied column, zeroed moment and statistic bitwise equal,
  the corrected opacity and scale within 1 ulp; shapes, row order, state["step"], state_dict; torch.optim.Adam and
  FusedAdam; stage-1 and PBR groups, 1M rows.
* inject_noise: within 4 eps32 (|x| + sum |noise terms|) of the fp64 restatement; zero learning rate; generator use.
* No host sync, fixed launch counts, bitwise determinism, the sampling law, the edge cases, a 1000-step training loop.
"""
import contextlib

import numpy as np
import pytest
import torch

import densify_oracle as do
import mcmc_oracle as mo

pytestmark = pytest.mark.gpu


def mc():
    from relightable3dgaussian_b200 import mcmc
    return mcmc


@contextlib.contextmanager
def injected(**samples):
    """Serve mcmc's draws from `samples`: randn -> samples["z"], rand -> samples["rand"] (a list, consumed in order)."""
    m = mc()
    prev = m._sampler
    queue = list(samples.get("rand", []))

    def sampler(kind, shape, device):
        t = samples["z"] if kind == "randn" else queue.pop(0)
        assert tuple(t.shape) == tuple(shape), (kind, shape, t.shape)
        return t.to(device).contiguous()
    m._sampler = sampler
    try:
        yield
    finally:
        m._sampler = prev


def ulp_close(a, b, ulps=1):
    return bool(((a - b).abs() <= ulps * torch.as_tensor(np.spacing(np.abs(b.cpu().numpy())), device=b.device)).all())


def compare(fm, rm, out):
    """fm fused, rm restated: bitwise except the corrected opacity / scale (1 ulp)."""
    P = out["reloc_rewritten"].shape[0]
    rew = out["reloc_rewritten"].clone()
    if out["n_new"]:
        rew |= out["grow_src"]
    Pn = P + out["n_new"]
    mask = torch.cat((rew, torch.ones(out["n_new"], dtype=torch.bool, device=rew.device)))
    a, b = do.output_tensors(fm), do.output_tensors(rm)
    assert set(a) == set(b)
    for k in a:
        x, y = a[k], b[k]
        assert x.shape == y.shape and x.shape[0] == Pn, (k, x.shape, y.shape)
        if k in ("param/opacity", "param/scaling"):
            assert torch.equal(x[~mask], y[~mask]), k
            assert ulp_close(x[mask], y[mask]), (k, float((x[mask] - y[mask]).abs().max()))
        else:
            assert torch.equal(x, y), (k, int((x != y).sum()))


def boundary_draws(out):
    n = mo.near_boundary(*out["reloc"]) + (mo.near_boundary(*out["grow"]) if out["n_new"] else 0)
    return n


def run_pair(case, cap_max, optim_cls=torch.optim.Adam, seed=0, **kw):
    fm = do.build_model(case, mo.StandIn, optim_cls, device="cuda")
    rm = do.build_model(case, mo.StandIn, optim_cls, device="cuda")
    P = case["P"]
    n_new = mc().growth_count(P, cap_max, kw.get("growth_rate", 0.05))
    g = torch.Generator(device="cuda").manual_seed(seed)
    ur, ug = torch.rand(P, generator=g, device="cuda"), torch.rand(n_new, generator=g, device="cuda")
    with injected(rand=[ur] + ([ug] if n_new else [])):
        assert mc().relocate_and_grow(fm, cap_max, **kw) == n_new
    out = mo.restate_relocate_and_grow(rm, cap_max, u_reloc=ur, u_grow=ug, **kw)
    nb = boundary_draws(out)
    print(f"[mcmc] {case['name']}: P {P} dead {int((out['reloc'][0] >= 0).sum())} new {n_new} "
          f"draws near a CDF boundary {nb}")
    assert nb == 0, f"{nb} draws within 1e-12 total of a CDF boundary: pick another seed"
    compare(fm, rm, out)
    return fm, rm, out


CASES = ["s1_p2049", "pbr_p2049", "s1_p20k", "no_state"]


@pytest.mark.parametrize("fused_adam", [False, True])
@pytest.mark.parametrize("name", CASES + ["s1_p1m", "pbr_p1m"])
def test_matches_restatement(name, fused_adam):
    from relightable3dgaussian_b200.optim import FusedAdam
    cls = FusedAdam if fused_adam else torch.optim.Adam
    case = mo.mcmc_case(name, device="cuda" if name in do.LARGE else "cpu")
    P = case["P"]
    fm0 = do.build_model(case, mo.StandIn, cls, device="cuda")
    steps = {g["name"]: fm0.optimizer.state[g["params"][0]]["step"].clone()
             for g in fm0.optimizer.param_groups if g["params"][0] in fm0.optimizer.state}
    fm, rm, out = run_pair(case, 2 * P, cls)
    assert out["n_new"] == int(P * 1.05) - P and int((out["reloc"][0] >= 0).sum()) > 0
    for g in fm.optimizer.param_groups:
        p = g["params"][0]
        assert p is getattr(fm, do.ATTRS[g["name"]]) and p.requires_grad and p.is_leaf
        if g["name"] in steps:
            assert torch.equal(fm.optimizer.state[p]["step"], steps[g["name"]])
        else:
            assert p not in fm.optimizer.state
    sd = fm.optimizer.state_dict()
    opt2 = cls([{"params": [g["params"][0]], "lr": g["lr"], "name": g["name"]} for g in fm.optimizer.param_groups],
               lr=0.0, eps=1e-15)
    opt2.load_state_dict(sd)
    for g in opt2.param_groups:
        p = g["params"][0]
        if p in opt2.state:
            assert torch.equal(opt2.state[p]["exp_avg"], fm.optimizer.state[p]["exp_avg"])
    for g in fm.optimizer.param_groups:
        g["params"][0].grad = torch.full_like(g["params"][0], 1e-3)
    fm.optimizer.step()
    assert all(torch.isfinite(g["params"][0]).all() for g in fm.optimizer.param_groups)


@pytest.mark.parametrize("name", ["s1_p20k", "s1_p1m"])
def test_noise_matches_fp64_restatement(name):
    case = mo.mcmc_case(name, device="cuda" if name in do.LARGE else "cpu")
    m = do.build_model(case, mo.StandIn, device="cuda")
    P = case["P"]
    g = torch.Generator(device="cuda").manual_seed(3)
    for lr, noise_lr in ((1.6e-4, 5e5), (1e-2, 5e6)):             # the second: noise far above |x|
        m.optimizer.param_groups[0]["lr"] = lr
        z = torch.randn((P, 3), generator=g, device="cuda")
        exp, bound = mo.restate_inject_noise(m, z, noise_lr=noise_lr)
        with injected(z=z):
            mc().inject_noise(m, noise_lr=noise_lr)
        err = (m._xyz.detach().double() - exp).abs()
        print(f"[mcmc] noise {name} lr {lr} x noise_lr {noise_lr}: max err / bound {float((err / bound).max()):.3f}")
        assert (err <= bound).all(), float((err / bound).max())


def test_noise_zero_lr_and_generator_use():
    lib = mc()._lib.load()
    case = mo.mcmc_case("s1_p20k")
    m = do.build_model(case, mo.StandIn, device="cuda")
    P = case["P"]
    mom = {k: v.clone() for k, v in do.output_tensors(m).items() if not k.startswith("param/")}
    x0 = m._xyz.detach().clone()
    torch.cuda.manual_seed(5)
    st = torch.cuda.get_rng_state()
    n0 = lib.r3dg_launch_count()
    mc().inject_noise(m, noise_lr=0.0)
    m.optimizer.param_groups[0]["lr"] = 0.0
    mc().inject_noise(m)
    assert lib.r3dg_launch_count() == n0 and torch.equal(m._xyz, x0)
    assert torch.equal(torch.cuda.get_rng_state(), st)             # nothing drawn
    m.optimizer.param_groups[0]["lr"] = 1.6e-4
    torch.cuda.manual_seed(5)
    mc().inject_noise(m)
    assert lib.r3dg_launch_count() == n0 + 1 and not torch.equal(m._xyz, x0)
    after = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(5)
    z = torch.randn((P, 3), device="cuda")
    assert torch.equal(torch.cuda.get_rng_state(), after)          # the generator moved as torch.randn((P, 3)) moves it
    m2 = do.build_model(case, mo.StandIn, device="cuda")
    with injected(z=z):
        mc().inject_noise(m2)
    assert torch.equal(m2._xyz, m._xyz)                             # and the draw is that one
    for k, v in do.output_tensors(m).items():
        if not k.startswith("param/"):
            assert torch.equal(v, mom[k]), k                        # moments and statistics untouched


def test_sync_free_with_fixed_launch_counts():
    lib = mc()._lib.load()
    case = mo.mcmc_case("s1_p20k")
    P = case["P"]
    for cap, launches in ((2 * P, 12), (P, 6), (0, 6)):
        m = do.build_model(case, mo.StandIn, device="cuda")
        n0 = lib.r3dg_launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            mc().relocate_and_grow(m, cap)
            mc().inject_noise(m)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert lib.r3dg_launch_count() - n0 == launches + 1, cap
        assert m._xyz.shape[0] == max(P, min(cap, int(P * 1.05)))


def test_bitwise_deterministic():
    case = mo.mcmc_case("s1_p1m", device="cuda")
    P = case["P"]
    g = torch.Generator(device="cuda").manual_seed(8)
    ur, ug = torch.rand(P, generator=g, device="cuda"), torch.rand(int(P * 1.05) - P, generator=g, device="cuda")
    outs = []
    for _ in range(2):
        m = do.build_model(case, mo.StandIn, device="cuda")
        with injected(rand=[ur, ug]):
            mc().relocate_and_grow(m, 2 * P)
        outs.append(do.output_tensors(m))
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


def test_growth_sampling_law():
    """One fixed-seed chi-square test of the growth draws against the opacity proportions (all rows alive and with
    distinct positions, so each new row's source is the row with its xyz)."""
    from scipy.stats import chisquare
    case = mo.mcmc_case("s1_p2049", dead=0.0)
    case["params"]["opacity"] = case["params"]["opacity"].clamp_min(float(np.log(0.01 / 0.99)))
    P = case["P"]
    m = do.build_model(case, mo.StandIn, device="cuda")
    torch.cuda.manual_seed(1234)
    n_new = mc().relocate_and_grow(m, 100 * P, growth_rate=20.0)
    xyz = m._xyz.detach()
    assert torch.equal(xyz[:P], case["params"]["xyz"].cuda())
    key = {tuple(r): i for i, r in enumerate(xyz[:P].cpu().numpy().tolist())}
    src = torch.tensor([key[tuple(r)] for r in xyz[P:].cpu().numpy().tolist()])
    counts = torch.bincount(src, minlength=P).double().numpy()
    w = torch.sigmoid(case["params"]["opacity"][:, 0]).double().numpy()
    p = chisquare(counts, w / w.sum() * n_new).pvalue
    print(f"[mcmc] sampling law: {n_new} draws over {P} sources, chi-square p = {p:.3f}")
    assert p > 1e-3


def test_edge_no_row_alive():
    case = mo.mcmc_case("s1_p2049", dead=1.0)
    case["params"]["opacity"][:7] = -200.0                          # sigma32 underflows to 0: coef is its limit 1
    fm, rm, out = run_pair(case, 2 * case["P"])
    assert not bool((out["reloc"][0] >= 0).any()) and out["reloc"][2] == 0
    assert all(torch.isfinite(t).all() for t in do.output_tensors(fm).values())


def test_edge_no_dead_row_is_identity():
    case = mo.mcmc_case("s1_p2049", dead=0.0)
    case["params"]["opacity"] = case["params"]["opacity"].clamp_min(float(np.log(0.01 / 0.99)))
    m = do.build_model(case, mo.StandIn, device="cuda")
    before = {k: v.clone() for k, v in do.output_tensors(m).items()}
    mc().relocate_and_grow(m, case["P"])
    for k, v in do.output_tensors(m).items():
        assert torch.equal(v, before[k]), k


def test_edge_cap_at_or_below_p_never_prunes():
    case = mo.mcmc_case("s1_p2049")
    for cap in (case["P"], case["P"] // 2, 0):
        fm, rm, out = run_pair(case, cap)
        assert fm._xyz.shape[0] == case["P"] and out["n_new"] == 0


def test_edge_oversampled_source():
    """One live row, 2048 dead ones: every dead row draws it, c = 2048 > n_max - 1, so N = n_max for all copies."""
    case = mo.mcmc_case("s1_p2049", dead=1.0)
    case["params"]["opacity"][5] = 2.0
    fm, rm, out = run_pair(case, case["P"], n_max=51)
    assert int(out["reloc_count"][5]) == case["P"] - 1
    op, sc = fm._opacity.detach(), fm._scaling.detach()
    assert (op == op[5]).all() and (sc == sc[5]).all()
    o = torch.sigmoid(torch.tensor([2.0], device="cuda")).double().cpu()
    _, _, lg = mo.correction(o, torch.tensor([51]), 0.005)
    assert ulp_close(op[5].cpu(), lg.float())


def test_rejections_on_device():
    case = mo.mcmc_case("s1_p2049")
    lib = mc()._lib.load()
    n0 = lib.r3dg_launch_count()
    m = do.build_model(case, mo.StandIn, device="cuda")
    m.optimizer.param_groups.pop()
    with pytest.raises(ValueError, match="relocate_and_grow"):
        mc().relocate_and_grow(m, 10**6)
    m = do.build_model(case, mo.StandIn, device="cuda")
    m.denom = torch.zeros((case["P"], 2), device="cuda")[:, :1]
    with pytest.raises(RuntimeError, match="contiguous"):
        mc().relocate_and_grow(m, 10**6)
    m = do.build_model(case, mo.StandIn, device="cuda")
    m._visibility_tracing = torch.zeros((case["P"], 24), device="cuda")
    with pytest.raises(RuntimeError, match="baked visibility"):
        mc().relocate_and_grow(m, 10**6)
    assert lib.r3dg_launch_count() == n0


@pytest.mark.parametrize("fused_adam", [False, True])
def test_install_at_cap_drops_stale_gradients(fused_adam):
    """train.py calls densify_and_prune after the backward pass and before step().  At the cap relocation rewrites rows
    in place; the gradients they hold belong to the rows before relocation, and with the rewritten rows' zero moments
    any of them would move the row by ~3 lr per component.  So relocate_and_grow leaves no gradient, the step skips
    every parameter, and after step() the model is exactly the relocation output."""
    from relightable3dgaussian_b200.optim import FusedAdam
    m_ = mc()

    class Fused(mo.StandIn):
        pass
    case = mo.mcmc_case("s1_p20k")
    P = case["P"]
    m_.install(Fused, cap_max=P, noise_lr=0.0)
    try:
        m = do.build_model(case, Fused, FusedAdam if fused_adam else torch.optim.Adam, device="cuda")
        g = torch.Generator(device="cuda").manual_seed(21)
        for grp in m.optimizer.param_groups:
            grp["params"][0].grad = torch.randn(grp["params"][0].shape, generator=g, device="cuda") * 1e-3
        steps = {id(p): st["step"].clone() for p, st in m.optimizer.state.items()}
        m.densify_and_prune(0.0002, 0.005, 4.0, 20, 0.0004)
        assert m._xyz.shape[0] == P
        assert all(grp["params"][0].grad is None for grp in m.optimizer.param_groups)
        relocated = {k: v.clone() for k, v in do.output_tensors(m).items()}
        rew = relocated["exp_avg/opacity"][:, 0] == 0
        assert int(rew.sum()) > 0
        m.step()
        for k, v in do.output_tensors(m).items():
            assert torch.equal(v, relocated[k]), k
        assert all(torch.equal(st["step"], steps[id(p)]) for p, st in m.optimizer.state.items())
    finally:
        m_.uninstall()


def relocation_exclusions(opacity, out, tol=1e-12):
    """Rows a near-boundary relocation draw may change: the drawing row, the restated source and its live neighbours
    (either may be the fused pick) and every row copied from one of them.  Returns (mask [P], number of such draws)."""
    pick, cdf, total, v = out["reloc"]
    P = pick.shape[0]
    alive = torch.sigmoid(opacity[:, 0]) > 0.005
    ok = pick >= 0
    p = pick.clamp_min(0)
    hi = cdf[p]
    lo = torch.where(p > 0, cdf[(p - 1).clamp_min(0)], torch.zeros_like(hi))
    amb = ok & (((hi - v).abs() <= tol * total) | ((v - lo).abs() <= tol * total))
    live = torch.nonzero(alive).squeeze(-1)
    k = torch.searchsorted(live, pick[amb])
    cand = torch.cat((pick[amb], live[(k - 1).clamp_min(0)], live[(k + 1).clamp_max(len(live) - 1)]))
    excl = amb | torch.isin(torch.arange(P, device=pick.device), cand) | (ok & torch.isin(pick, cand))
    return excl, int(amb.sum())


def test_relocation_above_two_scan_chunks():
    """3M rows = 1536 blocks of 2048: the block-sum scan carries between its 1024-element chunks.  Relocation only
    (cap = P), against the restatement; rows a near-boundary draw may change are counted, reported and left out."""
    case = mo.mcmc_case("s1_p3m", device="cuda")
    P = case["P"]
    fm = do.build_model(case, mo.StandIn, device="cuda")
    rm = do.build_model(case, mo.StandIn, device="cuda")
    ur = torch.rand(P, generator=torch.Generator(device="cuda").manual_seed(4), device="cuda")
    with injected(rand=[ur]):
        assert mc().relocate_and_grow(fm, P) == 0
    out = mo.restate_relocate_and_grow(rm, P, u_reloc=ur)
    excl, nb = relocation_exclusions(case["params"]["opacity"], out)
    print(f"[mcmc] s1_p3m relocation: dead {int((out['reloc'][0] >= 0).sum())}, draws near a CDF boundary {nb}, "
          f"rows left out {int(excl.sum())}")
    assert int(excl.sum()) <= 64 * max(nb, 1)
    a, b = do.output_tensors(fm), do.output_tensors(rm)
    rew = out["reloc_rewritten"] & ~excl
    for k in a:
        x, y = a[k][~excl], b[k][~excl]
        if k in ("param/opacity", "param/scaling"):
            keep = ~out["reloc_rewritten"][~excl]
            assert torch.equal(x[keep], y[keep]), k
            assert ulp_close(a[k][rew], b[k][rew]), k
        else:
            assert torch.equal(x, y), (k, int((x != y).sum()))


def test_training_loop_1000_steps():
    """A stand-in model trained through install() with seeded synthetic gradients and FusedAdam: noise after every
    step, relocation and growth every 100 steps after step 500 (the reference's schedule).  Every noise step and
    every relocate_and_grow call is checked against the restatement with the same samples, and the fused tensors are
    then copied over so that each call is checked on its own."""
    from relightable3dgaussian_b200 import optim
    m_ = mc()

    class Fused(mo.StandIn):
        pass
    case = mo.mcmc_case("s1_p20k")
    cap = case["P"] + 2500
    optim.install()
    m_.install(Fused, cap_max=cap)
    rec = []
    prev = m_._sampler

    def recording(kind, shape, device):
        t = prev(kind, shape, device)
        rec.append(t)
        return t
    m_._sampler = recording
    try:
        fm = do.build_model(case, Fused, torch.optim.Adam, device="cuda")
        rm = do.build_model(case, mo.StandIn, torch.optim.Adam, device="cuda")
        assert isinstance(fm.optimizer, optim.FusedAdam)
        g = torch.Generator(device="cuda").manual_seed(11)
        calls = 0
        for it in range(1, 1001):
            P = fm._xyz.shape[0]
            assert rm._xyz.shape[0] == P and P <= cap
            grads = {grp["name"]: torch.randn(grp["params"][0].shape, generator=g, device="cuda") * 1e-3
                     for grp in fm.optimizer.param_groups}
            for mdl in (fm, rm):
                for grp in mdl.optimizer.param_groups:
                    grp["params"][0].grad = grads[grp["name"]].clone()
            fm.add_densification_stats(None, None, None)
            if it > 500 and it % 100 == 0:
                rec.clear()
                fm.densify_and_prune(0.0002, 0.005, 4.0, 20, 0.0004)
                n_new = mc().growth_count(P, cap)
                out = mo.restate_relocate_and_grow(rm, cap, u_reloc=rec[0], u_grow=rec[1] if n_new else None)
                assert boundary_draws(out) == 0
                compare(fm, rm, out)
                with torch.no_grad():
                    rm._opacity.copy_(fm._opacity)
                    rm._scaling.copy_(fm._scaling)
                for mdl in (fm, rm):                              # this iteration's step skips every parameter
                    assert all(grp["params"][0].grad is None for grp in mdl.optimizer.param_groups)
                calls += 1
            rec.clear()
            fm.step()
            rm.step()
            exp, bound = mo.restate_inject_noise(rm, rec[0])
            assert ((fm._xyz.detach().double() - exp).abs() <= bound).all(), it
            with torch.no_grad():
                rm._xyz.copy_(fm._xyz)
            for k, v in do.output_tensors(fm).items():
                assert torch.isfinite(v).all(), (it, k)
        assert calls == 5 and fm._xyz.shape[0] == cap
        print(f"[mcmc] training loop: {case['P']} -> {fm._xyz.shape[0]} rows (cap {cap})")
    finally:
        m_._sampler = prev
        m_.uninstall()
        optim.uninstall()

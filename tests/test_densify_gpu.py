"""GPU parity of the fused densification (relightable3dgaussian_b200/densify.py, csrc/densify.cu).

* Against the restatement in tests/densify_oracle.py on the same device (fixture cases and 1M / 3M rows at about
  2 % clone, 1 % split, 3 % prune): row order, counts, every copied row, the moments, the new scaling and all
  statistics bit-exact; the split copies' xyz within 4 eps32 (|x| + sum_j |R_ij s_j|) per component (torch.bmm's
  summation order is cuBLAS's).
* Against the reference's own outputs (tests/golden/densify.npz) with the fixture's z injected: the same, with the
  split copies' scaling within 2 ulp plus 4 eps32 absolute (the fixture's exp, division and log ran on the CPU, and
  log turns the argument's relative rounding into an absolute error).
* With the default sampler and one CUDA seed: equal to the restatement calling torch.normal.
* Statistics, launch counts, optimizer continuation, state_dict, install / uninstall, rejections, and a 1000-step
  stand-in training loop.
"""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

import densify_oracle as do
from helpers import GOLDEN

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(GOLDEN, "densify.npz"))
EPS = float(np.finfo(np.float32).eps)


def dz():
    from relightable3dgaussian_b200 import densify
    return densify


@contextlib.contextmanager
def injected(z):
    d = dz()
    prev = d._sampler

    def sampler(shape, device):
        assert tuple(shape) == tuple(z.shape), (shape, z.shape)
        return z.to(device).contiguous()
    d._sampler = sampler
    try:
        yield
    finally:
        d._sampler = prev


def run_fused(m, args, z=None):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        if z is None:
            dz().densify_and_prune(m, **args)
        else:
            with injected(z):
                dz().densify_and_prune(m, **args)
    return buf.getvalue()


def run_restated(m, args, z=None):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        r = do.restate_densify_and_prune(m, z=z, **args)
    return r, buf.getvalue()


def xyz_bound(case, code, z):
    """4 eps32 (|x| + sum_j |R_ij s_j|) for every output row (0 where the row is not a split copy)."""
    code = torch.as_tensor(code).long().cpu()
    src, kind = code // 4, code % 4
    P = case["P"]
    nS = z.shape[0] // 2
    dev = "cpu"
    # rank of each split source among the split rows: the split rows are exactly the sources of kind 2 / 3 copies,
    # but pruned copies are absent, so rebuild S from the input (the split set depends on no random value)
    bound = torch.zeros((len(code), 3))
    rows = torch.nonzero(kind >= 2).squeeze(-1)
    if len(rows) == 0:
        return bound
    split_src = SPLIT_SETS[case["name"]].cpu()
    rank = torch.full((P,), -1, dtype=torch.long)
    rank[split_src] = torch.arange(len(split_src))
    k = rank[src[rows]] + (kind[rows] == 3).long() * nS
    rot = case["params"]["rotation"].to(dev)[src[rows]]
    v = z.cpu()[k] * torch.exp(case["params"]["scaling"].to(dev)[src[rows]].double()).float()
    R = do.rotation_matrices(rot.double()).float()
    mag = case["params"]["xyz"].to(dev)[src[rows]].abs() + torch.bmm(R.abs(), v.abs().unsqueeze(-1)).squeeze(-1)
    bound[rows] = 4 * EPS * mag
    return bound


SPLIT_SETS = {}


def compare(fused, expected, code, case, z, transcendental_ulps=0):
    """fused / expected: {name: tensor}.  Everything bit-exact except the split copies' xyz (bounded) and, with
    transcendental_ulps > 0, their scaling."""
    code_t = torch.as_tensor(code).long()
    splitrow = (code_t % 4 >= 2).cpu()
    bound = xyz_bound(case, code, z)
    assert set(fused) == set(expected), (sorted(fused), sorted(expected))
    for k in fused:
        a, b = fused[k].detach().cpu(), expected[k].detach().cpu()
        assert a.shape == b.shape and a.dtype == b.dtype, (k, a.shape, b.shape)
        if k == "param/xyz":
            assert torch.equal(a[~splitrow], b[~splitrow]), k
            err = (a[splitrow] - b[splitrow]).abs()
            assert (err <= bound[splitrow]).all(), (k, float((err / bound[splitrow].clamp_min(1e-30)).max()))
        elif k == "param/scaling" and transcendental_ulps:
            assert torch.equal(a[~splitrow], b[~splitrow]), k
            # log(exp(s) / 1.6): `transcendental_ulps` ulp of the result, plus the argument's relative error (exp and the
            # division each round on both sides), which log turns into an absolute one
            ulp = torch.as_tensor(np.spacing(np.abs(b[splitrow].numpy())))
            tol = transcendental_ulps * ulp + 2 * transcendental_ulps * EPS
            assert ((a[splitrow] - b[splitrow]).abs() <= tol).all(), k
        else:
            assert torch.equal(a, b), (k, (a != b).sum().item() if a.shape == b.shape else None)


def check_same_device(case, optim_cls=torch.optim.Adam, z_seed=0):
    fm = do.build_model(case, do.StandIn, optim_cls, device="cuda")
    rm = do.build_model(case, do.StandIn, optim_cls, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(z_seed)
    # |S| is known only after classification: draw z for the largest possible split set and cut it
    zfull = torch.randn((2 * case["P"], 3), generator=g, device="cuda")
    holder = {}

    def sampler(shape, device):
        holder["z"] = zfull[: shape[0]].contiguous()
        return holder["z"]
    d = dz()
    prev = d._sampler
    d._sampler = sampler
    try:
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            d.densify_and_prune(fm, **case["args"])
    finally:
        d._sampler = prev
    r, out_r = run_restated(rm, case["args"], z=holder["z"])
    assert buf.getvalue() == out_r
    SPLIT_SETS[case["name"]] = torch.nonzero(r["split"]).squeeze(-1)
    compare(do.output_tensors(fm), do.output_tensors(rm), r["code"].cpu().numpy(), case_cpu(case), holder["z"])
    return fm, rm, r


def case_cpu(case):
    return dict(case, params={k: v.cpu() for k, v in case["params"].items()})


@pytest.mark.parametrize("name", do.FIXTURE_CASES)
def test_fused_matches_restatement_on_device(name):
    case = do.densify_case(name)
    case = dict(case, params={k: v.cuda() for k, v in case["params"].items()})
    check_same_device(case)


@pytest.mark.parametrize("name", list(do.LARGE))
def test_fused_matches_restatement_large(name):
    case = do.densify_case(name, device="cuda")
    fm, rm, r = check_same_device(case)
    P = case["P"]
    nC, nS, Pn = int(r["clone"].sum()), int(r["split"].sum()), fm._xyz.shape[0]
    print(f"[densify] {name}: P {P} clone {nC / P:.3%} split {nS / P:.3%} -> {Pn}")
    assert 0.01 < nC / P < 0.03 and 0.005 < nS / P < 0.02


@pytest.mark.parametrize("name", do.FIXTURE_CASES)
def test_fused_matches_reference_fixture(name, capsys):
    case = do.densify_case(name)
    m = do.build_model(case, do.StandIn, device="cuda")
    z = torch.as_tensor(G[f"{name}/z"])
    with injected(z):
        dz().densify_and_prune(m, **case["args"])
    a, P1, b, P2 = (int(v) for v in G[f"{name}/counts"])
    assert capsys.readouterr().out == f"densify_and_split_normal: {a} / {P1}\nweights_accum: {b} / {P2}\n"
    code = G[f"{name}/code"]
    # split set of the reference run: restated on the CPU inputs (the CPU test pins the restatement to the fixture)
    rm = do.build_model(case, do.StandIn)
    with contextlib.redirect_stdout(io.StringIO()):
        r = do.restate_densify_and_prune(rm, z=z, **case["args"])
    SPLIT_SETS[name] = torch.nonzero(r["split"]).squeeze(-1)
    exp = do.expected_from_code(case, code, G[f"{name}/split_xyz"], G[f"{name}/split_scaling"])
    compare(do.output_tensors(m), exp, code, case, z, transcendental_ulps=2)


def test_default_sampler_matches_torch_normal():
    case = do.densify_case("s1_p20k")
    fm = do.build_model(case, do.StandIn, device="cuda")
    rm = do.build_model(case, do.StandIn, device="cuda")
    torch.cuda.manual_seed(99)
    run_fused(fm, case["args"])
    torch.cuda.manual_seed(99)
    r, _ = run_restated(rm, case["args"])
    SPLIT_SETS[case["name"]] = torch.nonzero(r["split"]).squeeze(-1)
    compare(do.output_tensors(fm), do.output_tensors(rm), r["code"].cpu().numpy(), case, r["z"])


def test_torch_cuda_arithmetic_the_kernels_mirror():
    """torch's CUDA x / 1.6 multiplies by the fp32 reciprocal; sigmoid is 1 / (1 + exp(-x)); comparisons with a Python
    float round it to fp32.  The kernel assumes all three; the bit-exact tests above depend on them."""
    x = torch.randn(1 << 20, device="cuda") * 4
    r = float(np.float32(1.0) / np.float32(1.6))
    assert torch.equal(x / (0.8 * 2), x * torch.tensor(r, device="cuda"))
    assert not torch.equal(x / (0.8 * 2), x / torch.tensor(1.6, device="cuda"))
    assert torch.equal(torch.sigmoid(x), 1.0 / (1.0 + torch.exp(-x)))
    t = torch.tensor([0.5], device="cuda")
    assert bool(t < 0.5 + 2.0 ** -30) is False and bool(t <= 0.5 + 2.0 ** -30) is True


def test_stats_bit_exact_and_sync_free():
    case = do.densify_case("s1_p20k")
    fm = do.build_model(case, do.StandIn, device="cuda")
    rm = do.build_model(case, do.StandIn, device="cuda")
    P = case["P"]
    g = torch.Generator(device="cuda").manual_seed(5)
    lib = dz()._lib.load()
    for step in range(50):
        vg = torch.randn((P, 3), generator=g, device="cuda") * 1e-3
        ng = torch.randn((P, 3), generator=g, device="cuda") * 1e-2
        filt = torch.rand(P, generator=g, device="cuda") < 0.7
        w = torch.rand((P, 1), generator=g, device="cuda") * 0.01
        radii = torch.randint(0, 40, (P,), generator=g, device="cuda", dtype=torch.int32)
        vpt = torch.zeros((P, 3), device="cuda", requires_grad=True)
        vpt.grad = vg
        fm._normal.grad, rm._normal.grad = ng, ng
        n0 = lib.r3dg_launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            dz().add_densification_stats(fm, vpt, filt, w, radii=radii)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert lib.r3dg_launch_count() - n0 == 1
        do.restate_add_densification_stats(rm, vpt, filt, w, radii=radii)
    for n in ("weights_accum", "denom", "max_radii2D"):
        assert torch.equal(getattr(fm, n), getattr(rm, n)), n
    for n in ("xyz_gradient_accum", "normal_gradient_accum"):
        a, b = getattr(fm, n), getattr(rm, n)
        assert ((a - b).abs() <= 1e-6 * b.abs()).all(), n
    torch.cuda.set_sync_debug_mode("error")
    try:
        with pytest.raises(RuntimeError):
            do.restate_add_densification_stats(rm, vpt, filt, w)       # boolean indexing syncs
    finally:
        torch.cuda.set_sync_debug_mode(0)


@pytest.mark.parametrize("name", ["s1_p2049", "pbr_p2049"])
def test_launch_count_is_fixed(name):
    lib = dz()._lib.load()
    case = do.densify_case(name)
    m = do.build_model(case, do.StandIn, device="cuda")
    n0 = lib.r3dg_launch_count()
    run_fused(m, case["args"])
    assert lib.r3dg_launch_count() - n0 == 4


@pytest.mark.parametrize("fused_adam", [False, True])
def test_optimizer_continues_and_state_dict_round_trips(fused_adam):
    from relightable3dgaussian_b200.optim import FusedAdam
    cls = FusedAdam if fused_adam else torch.optim.Adam
    case = do.densify_case("no_state")
    m = do.build_model(case, do.StandIn, cls, device="cuda")
    steps_before = {g["name"]: m.optimizer.state[g["params"][0]]["step"].clone()
                    for g in m.optimizer.param_groups if g["params"][0] in m.optimizer.state}
    run_fused(m, case["args"])
    Pn = m._xyz.shape[0]
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        assert p is getattr(m, do.ATTRS[g["name"]]) and p.shape[0] == Pn and p.requires_grad
        if g["name"] in steps_before:
            assert torch.equal(m.optimizer.state[p]["step"], steps_before[g["name"]])
        else:
            assert p not in m.optimizer.state
    sd = m.optimizer.state_dict()
    for g in m.optimizer.param_groups:
        g["params"][0].grad = torch.full_like(g["params"][0], 1e-3)
    m.optimizer.step()
    assert all(torch.isfinite(g["params"][0]).all() for g in m.optimizer.param_groups)
    opt2 = cls([{"params": [g["params"][0]], "lr": g["lr"], "name": g["name"]} for g in m.optimizer.param_groups],
               lr=0.0, eps=1e-15)
    opt2.load_state_dict(sd)
    assert len(opt2.state) == len(sd["state"]) == len(steps_before)
    for g2 in opt2.param_groups:
        p2 = g2["params"][0]
        if p2 in opt2.state:
            assert opt2.state[p2]["exp_avg"].shape == p2.shape


def test_rejections():
    d = dz()
    case = do.densify_case("s1_p2049")
    m = do.build_model(case, do.StandIn, device="cuda")
    P = case["P"]
    vpt = torch.zeros((P, 3), device="cuda", requires_grad=True)
    vpt.grad = torch.zeros((P, 3), device="cuda")
    filt = torch.ones(P, dtype=torch.bool, device="cuda")
    w = torch.zeros((P, 1), device="cuda")
    lib = d._lib.load()
    n0 = lib.r3dg_launch_count()
    with pytest.raises(RuntimeError, match="_normal has no .grad"):
        d.add_densification_stats(m, vpt, filt, w)
    m._normal.grad = torch.zeros((P, 3), device="cuda")
    with pytest.raises(RuntimeError):
        d.add_densification_stats(m, vpt, filt.to(torch.uint8), w)
    with pytest.raises(RuntimeError):
        d.add_densification_stats(m, vpt, filt, w.double())
    m.denom = torch.zeros((P, 2), device="cuda")[:, :1]                      # non-contiguous
    with pytest.raises(RuntimeError, match="contiguous"):
        d.densify_and_prune(m, **case["args"])
    m.denom = torch.zeros((P, 1), device="cuda")
    m.optimizer.param_groups[0]["name"] = "bogus"
    with pytest.raises(KeyError):
        d.densify_and_prune(m, **case["args"])
    assert lib.r3dg_launch_count() == n0


def test_install_on_stand_in_class():
    d = dz()

    class Model(do.StandIn):
        pass
    case = do.densify_case("s1_p2049")
    d.install(Model)
    try:
        with pytest.raises(RuntimeError):
            d.install(Model)
        m = do.build_model(case, Model, device="cuda")
        lib = d._lib.load()
        n0 = lib.r3dg_launch_count()
        with contextlib.redirect_stdout(io.StringIO()):
            m.densify_and_prune(**case["args"])
        assert lib.r3dg_launch_count() - n0 == 4 and not hasattr(m, "last")
    finally:
        d.uninstall()
    assert Model.densify_and_prune is do.StandIn.densify_and_prune


def test_training_loop_1000_steps():
    """A stand-in model trained with seeded synthetic gradients (independent of the parameters): stats every step,
    densify_and_prune every 100 steps, FusedAdam.  After every densify call the fused model and the restatement have
    the same rows and masks, parameters agree (xyz of the new split copies within the per-call bound), and the
    fused xyz is then copied over so that each call is checked on its own."""
    from relightable3dgaussian_b200 import optim
    d = dz()

    class Fused(do.StandIn):
        pass
    case = do.densify_case("s1_p20k")
    optim.install()
    d.install(Fused)
    try:
        fm = do.build_model(case, Fused, torch.optim.Adam, device="cuda")
        rm = do.build_model(case, do.StandIn, torch.optim.Adam, device="cuda")
        assert isinstance(fm.optimizer, optim.FusedAdam)
        g = torch.Generator(device="cuda").manual_seed(11)
        checked = 0
        for it in range(1, 1001):
            P = fm._xyz.shape[0]
            assert rm._xyz.shape[0] == P
            vpt = torch.zeros((P, 3), device="cuda", requires_grad=True)
            vpt.grad = torch.randn((P, 3), generator=g, device="cuda") * 2e-4
            filt = torch.rand(P, generator=g, device="cuda") < 0.8
            w = torch.rand((P, 1), generator=g, device="cuda") * 0.02
            for mdl in (fm, rm):
                for grp in mdl.optimizer.param_groups:
                    grp["params"][0].grad = None
            grads = {grp["name"]: torch.randn(grp["params"][0].shape, generator=g, device="cuda") * 1e-3
                     for grp in fm.optimizer.param_groups}
            for mdl in (fm, rm):
                for grp in mdl.optimizer.param_groups:
                    grp["params"][0].grad = grads[grp["name"]].clone()
            fm.add_densification_stats(vpt, filt, w)
            rm.add_densification_stats(vpt, filt, w)
            fm.optimizer.step()
            rm.optimizer.step()
            if it % 100 == 0:
                state = torch.cuda.get_rng_state()
                with contextlib.redirect_stdout(io.StringIO()):
                    fm.densify_and_prune(0.0002, 0.005, 4.0, 20 if it > 500 else None, 0.0004)
                torch.cuda.set_rng_state(state)
                rm.densify_and_prune(0.0002, 0.005, 4.0, 20 if it > 500 else None, 0.0004)
                r = rm.last
                code = r["code"].cpu().numpy()
                splitrow = torch.as_tensor(code % 4 >= 2)
                a, b = do.output_tensors(fm), do.output_tensors(rm)
                for k in a:
                    if k == "param/xyz":
                        assert torch.equal(a[k][~splitrow.cuda()], b[k][~splitrow.cuda()])
                        err = (a[k] - b[k]).abs()[splitrow.cuda()]
                        assert (err <= 1e-5 * (1 + b[k].abs()[splitrow.cuda()])).all()
                    else:
                        assert torch.equal(a[k], b[k]), (it, k)
                with torch.no_grad():
                    rm._xyz.copy_(fm._xyz)
                checked += 1
        assert checked == 10
        print(f"[densify] training loop: {case['P']} -> {fm._xyz.shape[0]} rows")
    finally:
        d.uninstall()
        optim.uninstall()

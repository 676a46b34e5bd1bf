"""GPU tests of the similarity transform (csrc/compose.cu, compose.py): the forward against the fp64 truth
(tests/compose64.py) over sizes, object counts, SH shapes, rotations and scales; the backward against fp64 autograd;
bitwise reproducibility; invariance of the rasterizer's image and of the shading step under a rigid motion of scene
and camera; and the recovery of an object's pose by fitting renders."""
import math

import pytest
import torch

import compose64 as C64
from relightable3dgaussian_b200 import compose, synth
from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
D = torch.float64
EPS = 2.0 ** -24


def _quat(axis, angle):
    axis = torch.as_tensor(axis, dtype=D)
    axis = axis / axis.norm()
    return torch.cat([torch.tensor([math.cos(angle / 2)], dtype=D), math.sin(angle / 2) * axis])


ROTATIONS = {"identity": lambda g: _quat((1, 0, 0), 0.0), "x180": lambda g: _quat((1, 0, 0), math.pi),
             "y180": lambda g: _quat((0, 1, 0), math.pi), "z180": lambda g: _quat((0, 0, 1), math.pi),
             "tiny": lambda g: _quat(torch.randn(3, generator=g, dtype=D), 1e-6),
             "random": lambda g: torch.randn(4, generator=g, dtype=D)}
SH_SETS = ([(3, 3), (3, 3), (4, 1)], [(0, 3), (1, 1), (2, 3)], [(4, 3)], [(3, 3), (4, 1)], [])


def _offsets(P, K, g):
    """K ranges over P rows, some of them empty."""
    if K == 1:
        return [0, P]
    cuts = sorted(torch.randint(0, P + 1, (K - 1,), generator=g).tolist())
    o = [0] + cuts + [P]
    if K > 2:
        o[2] = o[1]                                           # object 1 is empty
    return o


def _case(P, K, sh_set, rot, scale, seed):
    g = torch.Generator().manual_seed(seed)
    rows = [torch.randn(P, w, generator=g) for w in (3, 3, 4, 3)]
    shs = [torch.randn(P, (L + 1) ** 2 - 1, C, generator=g) for L, C in sh_set]
    quat = torch.stack([ROTATIONS[rot](g) if k % 2 == 0 else torch.randn(4, generator=g, dtype=D) for k in range(K)]).float()
    t = torch.randn(K, 3, generator=g) * 2
    s = torch.full((K,), float(scale))
    return rows, shs, quat, t, s, _offsets(P, K, g)


def _to(ts):
    return [t.to(DEV) for t in ts]


FWD_CASES = []
for i, (P, rot) in enumerate([(P, r) for P in (0, 1, 257, 1_000_000) for r in ROTATIONS]):
    FWD_CASES.append((P, (1, 3, 64)[i % 3], SH_SETS[i % len(SH_SETS)], rot, (1e-3, 1.0, 1e3)[(i // 3) % 3], i))


@pytest.mark.parametrize("P,K,sh_set,rot,scale,seed", FWD_CASES,
                         ids=[f"P{c[0]}-K{c[1]}-{c[3]}-s{c[4]:g}-sh{len(c[2])}" for c in FWD_CASES])
def test_forward_against_fp64(P, K, sh_set, rot, scale, seed):
    rows, shs, quat, t, s, offsets = _case(P, K, sh_set, rot, scale, seed)
    rows, shs, quat, t, s = _to(rows), _to(shs), quat.to(DEV), t.to(DEV), s.to(DEV)
    xyz, normal, rotation, scaling, out_sh = compose.transform_gaussians(*rows, shs, quat, t, s, offsets)
    ref = C64.transform(*[r.double() for r in rows], [x.double() for x in shs], quat.double(), t.double(), s.double(), offsets)
    # per row: xyz within a few roundings of s |x| + |t|, normals of |n|, quaternions of |r|, log-scales of |scaling| + |log s|
    obj = torch.repeat_interleave(torch.arange(K, device=DEV), torch.tensor([b - a for a, b in zip(offsets, offsets[1:])], device=DEV))
    tol_x = 8 * EPS * (s[obj, None].double() * rows[0].double().norm(dim=-1, keepdim=True) + t[obj].double().norm(dim=-1, keepdim=True))
    assert bool(((xyz.double() - ref[0]).abs() <= tol_x).all())
    assert bool(((normal.double() - ref[1]).abs() <= 8 * EPS * rows[1].double().norm(dim=-1, keepdim=True)).all())
    assert bool(((rotation.double() - ref[2]).abs() <= 8 * EPS * rows[2].double().norm(dim=-1, keepdim=True)).all())
    tol_s = 4 * EPS * (rows[3].double().abs() + s[obj, None].double().log().abs())
    assert bool(((scaling.double() - ref[3]).abs() <= tol_s).all())
    for (L, C), x, got, want in zip(sh_set, shs, out_sh, ref[4:]):
        assert got.shape == x.shape
        for l in range(1, L + 1):
            sl = slice(l * l - 1, (l + 1) ** 2 - 1)
            err = (got[:, sl].double() - want[:, sl]).norm(dim=1)
            bound = 2e-6 * (x[:, sl].double().norm(dim=1) + 1)
            assert bool((err <= bound).all()), (l, float((err / bound).max()))


@pytest.mark.parametrize("P", [1000, 100_000])
def test_backward_against_fp64_autograd(P):
    K = 3
    sh_set = [(3, 3), (3, 3), (4, 1)]
    rows, shs, quat, t, s, offsets = _case(P, K, sh_set, "random", 1.0, P)
    s = torch.tensor([0.7, 1.0, 2.5])
    leaves = [x.to(DEV).requires_grad_(True) for x in rows + [quat, t, s] + shs]
    outs = compose.transform_gaussians(*leaves[:4], leaves[7:], *leaves[4:7], offsets)
    outs = list(outs[:4]) + outs[4]
    g = torch.Generator().manual_seed(5)
    cots = [torch.randn(o.shape, generator=g).to(DEV) for o in outs]
    got = torch.autograd.grad(sum((o * c).sum() for o, c in zip(outs, cots)), leaves)
    leaves64 = [x.detach().double().requires_grad_(True) for x in leaves]
    ref_outs = C64.transform(*leaves64[:4], leaves64[7:], *leaves64[4:7], offsets)
    want = torch.autograd.grad(sum((o * c.double()).sum() for o, c in zip(ref_outs, cots)), leaves64)
    names = ["xyz", "normal", "rotation", "scaling", "quat", "translation", "scale", "f_rest", "incidents_rest", "visibility_rest"]
    for name, a, b in zip(names, got, want):
        rel = float((a.double() - b).norm() / b.norm())
        assert rel <= (1e-4 if name in ("quat", "translation", "scale") else 1e-5), (name, rel)


@pytest.mark.parametrize("deterministic", [False, True])
def test_bitwise_reproducible(deterministic):
    P, K = 300_000, 16
    rows, shs, quat, t, s, offsets = _case(P, K, [(3, 3), (3, 3), (4, 1)], "random", 1.0, 7)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        runs = []
        for _ in range(2):
            leaves = [x.to(DEV).requires_grad_(True) for x in rows + [quat, t, s] + shs]
            outs = compose.transform_gaussians(*leaves[:4], leaves[7:], *leaves[4:7], offsets)
            outs = list(outs[:4]) + outs[4]
            g = torch.Generator().manual_seed(3)
            loss = sum((o * torch.randn(o.shape, generator=g).to(DEV)).sum() for o in outs)
            grads = torch.autograd.grad(loss, leaves)
            runs.append([o.detach() for o in outs] + list(grads))
        for a, b in zip(*runs):
            assert torch.equal(a, b)
    finally:
        torch.use_deterministic_algorithms(prev)


# ---- invariance ------------------------------------------------------------------------------------------------------
def _rigid(seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.nn.functional.normalize(torch.randn(4, generator=g, dtype=D), dim=0)
    return q.float(), (torch.randn(3, generator=g) * 0.5)


def _render(means, scales, rots, opac, shs, feats, cam, V, Pm, campos):
    rs = GaussianRasterizationSettings(cam.image_height, cam.image_width, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                       torch.zeros(3, device=DEV), 1.0, V.to(DEV), Pm.to(DEV), 3, campos.to(DEV),
                                       False, True, False, False)
    means2D = torch.zeros_like(means)
    out = GaussianRasterizer(rs)(means3D=means, means2D=means2D, opacities=opac, shs=shs, scales=scales, rotations=rots,
                                 features=feats)
    return out[2], out[3], out[4]


def _moved_camera(cam, q, t):
    """viewmatrix and projmatrix (row-vector convention) and campos of the camera moved with the scene by T = [R, t]."""
    R = C64.build_rotation(q.double())
    Tinv = torch.eye(4, dtype=D)
    Tinv[:3, :3] = R.T
    Tinv[:3, 3] = -R.T @ t.double()
    V = (Tinv.T @ cam.viewmatrix.double()).float()
    Pm = (Tinv.T @ cam.projmatrix.double()).float()
    return V, Pm, (R @ cam.campos.double() + t.double()).float()


def test_rasterizer_image_is_invariant_under_a_rigid_motion():
    P = 20_000
    sc = synth.make_scene(P, "shell-v1", 4, 3)
    g = torch.Generator().manual_seed(11)
    shs = sc.shs.clone()
    shs[:, 1:] = torch.randn(P, 15, 3, generator=g) * 0.6                   # strongly view dependent
    cam = synth.make_camera(1, 160, 120)
    q, t = _rigid(2)
    m = {k: v.to(DEV) for k, v in dict(xyz=sc.means3D, normal=sc.normals, rotation=sc.rotations,
                                       scaling=sc.scales.log(), f_rest=shs[:, 1:].contiguous()).items()}
    moved = compose.transform(m, q.to(DEV), t.to(DEV), 1.0)
    base = [x.to(DEV) for x in (sc.opacities, sc.features)]
    ref = _render(m["xyz"], m["scaling"].exp(), m["rotation"], base[0], shs.to(DEV), base[1], cam, cam.viewmatrix,
                  cam.projmatrix, cam.campos)
    V, Pm, campos = _moved_camera(cam, q, t)
    shs_moved = torch.cat([shs[:, :1].to(DEV), moved["f_rest"]], 1)
    got = _render(moved["xyz"], moved["scaling"].exp(), moved["rotation"], base[0], shs_moved, base[1], cam, V, Pm, campos)
    for name, a, b in zip(("image", "opacity", "depth"), got, ref):
        d = (a - b).abs().flatten()
        # a pair whose alpha sits within rounding of the 1/255 cut-off may flip: allow a handful of such pixels
        assert float(torch.quantile(d, 0.999)) <= 1e-4 and float(d.mean()) <= 1e-6, (name, float(d.max()))
    stale = _render(moved["xyz"], moved["scaling"].exp(), moved["rotation"], base[0], shs.to(DEV), base[1], cam, V, Pm, campos)
    assert float((stale[0] - ref[0]).abs().max()) > 1e-2             # the unrotated SH is told apart


class _Env:                 # duck-types scene/envmap.py:EnvLight (envmap + transform)
    def __init__(self, envmap, transform):
        self.envmap, self.transform = envmap, transform


def test_shading_is_invariant_under_a_rotation():
    from relightable3dgaussian_b200.shading import rendering_equation
    P, N = 4000, 24
    g = torch.Generator().manual_seed(21)
    unit = lambda *s: torch.nn.functional.normalize(torch.randn(*s, 3, generator=g), dim=-1)
    base, rough = torch.rand(P, 3, generator=g), torch.rand(P, 1, generator=g) * 0.8 + 0.1
    normals, viewdirs, dirs = unit(P), unit(P), unit(P, N)
    vis, areas = torch.rand(P, N, 1, generator=g), torch.full((P, N, 1), 2 * math.pi / N)
    incidents = torch.randn(P, 16, 3, generator=g) * 0.3
    env = torch.rand(32, 64, 3, generator=g) + 0.1
    T = C64.build_rotation(torch.randn(4, generator=g, dtype=D)).float()
    q, _ = _rigid(5)
    R = C64.build_rotation(q.double()).float()
    cuda = lambda *ts: [x.to(DEV) for x in ts]
    pbr0, ex0 = rendering_equation(*cuda(base, rough, normals, viewdirs, incidents), _Env(env.to(DEV), T.to(DEV)),
                                   *cuda(vis, dirs, areas))
    m = dict(xyz=torch.zeros(P, 3), normal=normals, rotation=torch.zeros(P, 4), scaling=torch.zeros(P, 3),
             incidents_rest=incidents[:, 1:].contiguous())
    moved = compose.transform({k: v.to(DEV) for k, v in m.items()}, q.to(DEV), torch.zeros(3, device=DEV), 1.0)
    inc = torch.cat([incidents[:, :1].to(DEV), moved["incidents_rest"]], 1)
    pbr1, ex1 = rendering_equation(base.to(DEV), rough.to(DEV), moved["normal"], viewdirs.to(DEV) @ R.T.to(DEV), inc,
                                   _Env(env.to(DEV), (T @ R.T).to(DEV)), vis.to(DEV), dirs.to(DEV) @ R.T.to(DEV),
                                   areas.to(DEV))
    for a, b in ((pbr1, pbr0), (ex1["diffuse_light"], ex0["diffuse_light"]), (ex1["specular"], ex0["specular"])):
        assert float((a - b).abs().max()) <= 1e-4


# ---- pose recovery ---------------------------------------------------------------------------------------------------
def _blob(P, seed):
    """An elongated object of large Gaussians whose colour varies with position, so its pose is visible at every scale."""
    g = torch.Generator().manual_seed(seed)
    xyz = (torch.rand(P, 3, generator=g) * 2 - 1) * torch.tensor([0.8, 0.45, 0.25])
    shs = torch.randn(P, 16, 3, generator=g) * 0.05
    shs[:, 0] = (0.6 * xyz / torch.tensor([0.8, 0.45, 0.25])) / synth.SH_C0
    return dict(xyz=xyz, normal=torch.nn.functional.normalize(xyz, dim=-1), rotation=torch.tensor([[1.0, 0, 0, 0]]).repeat(P, 1),
                scaling=torch.full((P, 3), math.log(0.08)), f_rest=shs[:, 1:].contiguous()), shs[:, :1], torch.full((P, 1), 0.7)


def test_pose_recovery_by_fitting_renders():
    torch.manual_seed(0)
    model, dc, opac = _blob(1500, 1)
    model = {k: v.to(DEV) for k, v in model.items()}
    dc, opac = dc.to(DEV), opac.to(DEV)
    cams = [synth.make_camera(k, 96, 96, radius=3.0) for k in (0, 2, 5)]
    q_true = _quat((1, 2, 0.5), 0.6)
    t_true = torch.tensor([0.25, -0.15, 0.1])

    def render_all(q, t):
        m = compose.transform(model, q, t, torch.ones((), device=DEV))
        shs = torch.cat([dc, m["f_rest"]], 1)
        return [_render(m["xyz"], m["scaling"].exp(), m["rotation"], opac, shs, None, c, c.viewmatrix, c.projmatrix,
                        c.campos)[0] for c in cams]

    with torch.no_grad():
        target = render_all(q_true.float().to(DEV), t_true.to(DEV))
    q = C64.quat_mul(q_true, _quat((0.3, -1, 0.7), math.radians(10.0))).float().to(DEV).requires_grad_(True)
    t = (t_true * 1.05).to(DEV).requires_grad_(True)
    steps = 400
    opt = torch.optim.Adam([q, t], lr=1e-2)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 0.02 ** (i / steps))
    for _ in range(steps):
        opt.zero_grad()
        loss = sum(((a - b) ** 2).mean() for a, b in zip(render_all(q, t), target))
        loss.backward()
        opt.step()
        sched.step()
    R, R_true = C64.build_rotation(q.detach().double().cpu()), C64.build_rotation(q_true)
    angle = math.degrees(math.acos(min(1.0, (float(torch.trace(R.T @ R_true)) - 1) / 2)))
    t_err = float((t.detach().cpu().double() - t_true.double()).norm() / t_true.double().norm())
    assert angle <= 0.5 and t_err <= 0.01, (angle, t_err)

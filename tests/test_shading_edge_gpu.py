"""The fused shading step (csrc/shading.cu through relightable3dgaussian_b200.shading) against an fp64 truth on
adversarial inputs, under every kernel variant r3dg_tune selects.

truth  the reference's function bodies in fp64 (tests/golden/shade_edge.npz), or oracle/oracle_shading.py run in fp64
       on the GPU on the same fp32 inputs (a CPU test pins the two together);
ref32  the same computation in fp32: the reference's own arithmetic, whose error e_ref = |ref32 - truth| sets the scale.

Per Gaussian row (outputs, per-sample extras, leaf gradients):  max|ours - truth| <= K * (max|ref32 - truth| +
eps32 * max|truth|), i.e. A = B = K in  A * e_ref + B * eps32 * scale  with scale the row's fp64 magnitude.  Whole
tensor:  ||ours - truth|| <= C * max(||ref32 - truth||, eps32 ||truth||).  Environment-map gradient, per texel:
|ours - truth| <= K_TEXEL * (|ref32 - truth| + eps32 * sum|contribution|), the truth being the explicit fp64 scatter of
the four bilinear taps (shading_edge.env_scatter64); a texel no sample reaches must be exactly 0.
Run with -s to see the observed ratios (`[shade-edge]` lines) and the seam-ambiguity count."""
import contextlib
import ctypes
import functools
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import shading_edge as se
from helpers import SHADE_KNOBS

pytestmark = pytest.mark.gpu
CASES = se.load_cases()
NAMES = sorted(CASES)
KNOBS = [{}] + SHADE_KNOBS
EPS = se.EPS32

# Calibrated on the unmodified kernels (H100 80GB HBM3, 400 W power limit) at under 4x the worst ratio observed over
# every case, knob combination and cotangent set of this file.  Worst observed: 53.5 (training-scale specular),
# 157.9 (d_roughness, general-rotation case), 4.2 (whole-tensor specular, zero_incidents_dc), 126.1 (env texel,
# random_rotate).
K_OUT = 200.0       # pbr / diffuse_light / specular / per-sample lights / means, per row
K_GRAD = 600.0      # base_color / roughness / viewdirs / incidents gradients, per row
C_TENSOR = 16.0     # whole tensors
K_TEXEL = 400.0     # env-map gradient, per texel
SEAM_AMBIGUOUS_MAX = 1e-4   # fraction of samples whose env column depends on the rounding of `dirs @ T.T`

WORST = {}


def _note(kind, tag, r):
    WORST[kind] = max(WORST.get(kind, 0.0), r)
    print(f"[shade-edge] {kind:7s} {tag:60s} ratio {r:8.3f}  (worst {WORST[kind]:.3f})")


@contextlib.contextmanager
def tuned(knobs):
    from relightable3dgaussian_b200 import _lib
    old = {k: _lib.tune(k, v) for k, v in knobs.items()}
    try:
        yield
    finally:
        for k, v in old.items():
            _lib.tune(k, v)


def _dd(x):
    return (torch.from_numpy(x) if isinstance(x, np.ndarray) else x).cuda().double()


def check_rows(kind, tag, ours, truth, ref32, mag=None, keep=None):
    """Per Gaussian row and whole-tensor bounds (module docstring); `mag` (se.oracle_magnitudes) is the row's fp64
    magnitude, |truth| where it is None.  A truth of None (no path from the loss) requires exact zeros."""
    if truth is None:
        assert not ours.any(), (tag, "must be exactly 0")
        return
    P = ours.shape[0]
    o, t, r = (_dd(x).reshape(P, -1) for x in (ours, truth, ref32))
    m = t.abs() if mag is None else _dd(mag).reshape(P, -1)
    if keep is not None:
        o, t, r, m = o[keep], t[keep], r[keep], m[keep]
    assert torch.isfinite(o).all(), (tag, "non-finite")
    ek, er, sc = (o - t).abs().amax(1), (r - t).abs().amax(1), m.amax(1)
    den = er + EPS * sc
    zero = den == 0
    assert (ek[zero] == 0).all(), (tag, "must be exact where the truth and ref32 agree exactly", float(ek[zero].max()))
    ratio = float((ek[~zero] / den[~zero]).max()) if (~zero).any() else 0.0
    k = K_GRAD if kind == "grad" else K_OUT
    worst = int(torch.argmax(torch.where(zero, 0.0, ek / den.clamp_min(1e-300))))
    assert ratio <= k, (tag, ratio, "row", worst, o[worst].tolist()[:6], t[worst].tolist()[:6], r[worst].tolist()[:6])
    _note(kind, tag, ratio)
    nk, nr, nt = float(torch.linalg.norm(o - t)), float(torch.linalg.norm(r - t)), float(torch.linalg.norm(t))
    floor = max(nr, EPS * nt)
    assert (nk == 0) if floor == 0 else nk <= C_TENSOR * floor, (tag, "whole tensor", nk, nr, nt)
    _note("tensor", tag, nk / floor if floor > 0 else 0.0)


def check_texels(tag, ours, truth, ref32, mag, slack=None):
    """Per-texel env-gradient bound; `slack` (>= 0) widens it where samples of ambiguous column were excluded."""
    o, t, r, m = (_dd(x).reshape(-1) for x in (ours, truth, ref32, mag))
    assert torch.isfinite(o).all(), tag
    ek = (o - t).abs()
    if slack is not None:
        ek = (ek - _dd(slack).reshape(-1)).clamp_min(0)
    den = (r - t).abs() + EPS * m
    zero = den == 0
    assert (ek[zero] == 0).all(), (tag, "texel no sample reaches is not 0", float(ek[zero].max()))
    ratio = float((ek[~zero] / den[~zero]).max()) if (~zero).any() else 0.0
    assert ratio <= K_TEXEL, (tag, "texel", ratio)
    _note("texel", tag, ratio)


# ---- running the fused path -------------------------------------------------------------------------------------------
class SoftplusLight:            # duck-types DirectLightMap; keeps the texture so the test can read its gradient
    def __init__(self, env_raw):
        self.env = env_raw

    @property
    def get_env(self):
        self.tex = F.softplus(self.env)
        self.tex.retain_grad()
        return self.tex


class FixedLight:               # duck-types EnvLight (envmap + transform)
    def __init__(self, envmap, transform):
        self.envmap, self.transform = envmap, transform


def run_ours(t, cots=se.COTS):
    """rendering_equation on inputs t (fp32, cuda), L = sum <output, cot_output> over `cots`; outputs, the three lazy
    per-sample extras, gradients of the leaves (grad_env as in se.oracle_run) and of the texture (grad_tex)."""
    from relightable3dgaussian_b200.shading import rendering_equation
    leaves = {k: t[k].clone().requires_grad_(True) for k in se.LEAVES}
    T = t.get("transform")
    light = FixedLight(leaves["env"], T) if T is not None else SoftplusLight(leaves["env"])
    pbr, ex = rendering_equation(leaves["base_color"], leaves["roughness"], t["normals"], leaves["viewdirs"],
                                 leaves["incidents"], light, visibility_precompute=t["visibility"],
                                 incident_dirs_precompute=t["incident_dirs"], incident_areas_precompute=t["incident_areas"])
    assert ex["incident_dirs"] is t["incident_dirs"] and ex["incident_visibility"] is t["visibility"]
    outs = dict(pbr=pbr, diffuse=ex["diffuse_light"], specular=ex["specular"])
    sum((outs[k] * t["cot_" + k]).sum() for k in cots).backward()
    rec = {"pbr": pbr.detach(), "diffuse_light": ex["diffuse_light"].detach(), "specular": ex["specular"].detach()}
    rec.update({k: ex[k] for k in se.EXTRAS[:3]})               # materialised through _LazyExtras here
    rec.update({"grad_" + k: v.grad for k, v in leaves.items()})
    rec["grad_tex"] = leaves["env"].grad if T is not None else light.tex.grad[0]
    return rec


def run_means(t):
    """_RenderEquation with want_means=True (the only caller of the mean_* outputs of the C ABI)."""
    from relightable3dgaussian_b200.shading import _RenderEquation
    T = t.get("transform")
    tex = t["env"] if T is not None else F.softplus(t["env"])[0]
    with torch.no_grad():
        return _RenderEquation.apply(t["base_color"], t["roughness"], t["viewdirs"], t["incidents"], tex, t["normals"],
                                     t["visibility"], t["incident_dirs"], t["incident_areas"], T, True)


def check_means(tag, means, truth, ref32, vis):
    ml, mloc, mg, mv = means[3:]
    for got, k in ((ml, "incident_lights"), (mloc, "local_incident_lights"), (mg, "global_incident_lights")):
        check_rows("out", f"{tag} mean_{k}", got, _dd(truth[k]).mean(1), torch.as_tensor(ref32[k]).cuda().mean(1))
    check_rows("out", f"{tag} mean_visibility", mv, vis.double().mean(1), vis.mean(1))


def is_permutation(T):
    return T is None or bool(((T == 0) | (T.abs() == 1)).all())


def seam_ambiguous(dirs, T):
    """Samples whose env column flips between 0 and We-1 with the rounding of `dirs @ T.T`: x < 0 in the env frame
    and |y| within a few fp32 roundings of its terms (fp64).  None for a signed permutation, which is exact."""
    if is_permutation(T):
        return torch.zeros(dirs.shape[:2], dtype=torch.bool, device=dirs.device)
    d, Td = dirs.reshape(-1, 3).double(), T.double()
    e = d @ Td.T
    tol = 4 * EPS * (d.abs() @ Td.abs().T)[:, 1]
    return ((e[:, 0] < 0) & (e[:, 1].abs() <= tol)).reshape(dirs.shape[:2])


@functools.lru_cache(maxsize=None)
def gpu_truth(name, cots=se.COTS):
    """fp64 and fp32 oracle runs of a fixture case on the GPU, and the fp64 scatter of the env gradient."""
    t = se.inputs(CASES[name], "cuda")
    r64, r32 = se.oracle_run(t, torch.float64, cots), se.oracle_run(t, torch.float32, cots)
    He, We = r64["grad_tex"].shape[-3:-1]
    T = t.get("transform")
    e = se.env_frame(t["incident_dirs"].double(), None if T is None else T.double())
    grad, mag = se.env_scatter64(e, r64["g_light"], He, We)
    assert ((grad - r64["grad_tex"].reshape(He, We, 3)).abs() <= 1e-12 * mag).all(), name      # grid_sample's adjoint
    return r64, r32, grad, se.oracle_magnitudes(t, cots)


# ---- every fixture case, every kernel variant ---------------------------------------------------------------------------
@pytest.mark.parametrize("knobs", KNOBS, ids=lambda k: ",".join(f"{a[6:]}={b}" for a, b in k.items()) or "default")
@pytest.mark.parametrize("name", NAMES)
def test_fixture_case_against_fp64(name, knobs):
    c = CASES[name]
    t = se.inputs(c, "cuda")
    with tuned(knobs):
        ours = run_ours(t)
        means = run_means(t)
    tag = f"{name} {','.join(f'{a[6:]}={b}' for a, b in knobs.items()) or 'default'}"
    T = t.get("transform")
    amb = seam_ambiguous(t["incident_dirs"], T)
    assert not amb.any(), (name, int(amb.sum()))            # the fixture's rotation keeps clear of the seam
    truth = {k[3:]: v for k, v in c.items() if k.startswith("64/")}
    ref32 = {k[3:]: v for k, v in c.items() if k.startswith("32/")}
    _, r32, grad, mags = gpu_truth(name)
    for k in ("pbr",) + se.EXTRAS:
        check_rows("out", f"{tag} {k}", ours[k], truth[k], ref32[k], mags.get(k))
    for k in ("base_color", "roughness", "viewdirs", "incidents"):
        check_rows("grad", f"{tag} d_{k}", ours["grad_" + k], truth["grad_" + k], ref32["grad_" + k], mags["grad_" + k])
    # whole env gradient against the reference's (through softplus for a DirectLightMap)
    o, tr, r = (_dd(x).reshape(1, -1) for x in (ours["grad_env"], truth["grad_env"], ref32["grad_env"]))
    nk, floor = float(torch.linalg.norm(o - tr)), max(float(torch.linalg.norm(r - tr)), EPS * float(torch.linalg.norm(tr)))
    assert nk <= C_TENSOR * floor, (tag, "d_env", nk, floor)
    _note("tensor", f"{tag} d_env", nk / floor)
    check_texels(f"{tag} d_env texel", ours["grad_tex"], grad, r32["grad_tex"], mags["tex"])
    check_means(tag, means, truth, ref32, t["visibility"])


# ---- the cotangent sets training produces ---------------------------------------------------------------------------------
COT_SETS = [("pbr", "diffuse"), ("diffuse",), se.COTS]


@pytest.mark.parametrize("cots", COT_SETS, ids=["+".join(c) for c in COT_SETS])
@pytest.mark.parametrize("name", NAMES)
def test_cotangent_sets_against_fp64(name, cots):
    """Training reads pbr and diffuse_light only (specular's cotangent is None); some losses read diffuse_light only."""
    t = se.inputs(CASES[name], "cuda")
    ours = run_ours(t, cots)
    r64, r32, grad, mags = gpu_truth(name, cots)
    tag = f"{name} cots={'+'.join(cots)}"
    for k in ("base_color", "roughness", "viewdirs", "incidents"):
        check_rows("grad", f"{tag} d_{k}", ours["grad_" + k], r64["grad_" + k], r32["grad_" + k], mags["grad_" + k])
    check_texels(f"{tag} d_env texel", ours["grad_tex"], grad, r32["grad_tex"], mags["tex"])


# ---- training scale ----------------------------------------------------------------------------------------------------------
def training_inputs(P, N, He, seed, zero_frac=0.3):
    """Stage-2 shaped inputs on the GPU: random-rotate sampling (sample_incident_rays(is_training=True)) around normals
    that have drifted since, SH incidents exactly 0 on a fraction of rows (their initial value)."""
    from oracle.oracle_sampling import fibonacci_sphere_sampling
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, device="cuda")
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")
    n = F.normalize(rn(P, 3), dim=-1)
    dirs, areas = fibonacci_sphere_sampling(n, N, random_rotate=True, phase=r(P))
    inc = rn(P, 16, 3) * 0.3
    inc[r(P) < zero_frac] = 0.0
    vis = torch.where(r(P, N, 1) < 0.4, torch.zeros(P, N, 1, device="cuda"), 0.9 + 0.1 * r(P, N, 1))
    return dict(base_color=torch.sigmoid(rn(P, 3)) * 0.77 + 0.03, roughness=torch.sigmoid(rn(P, 1)) * 0.9 + 0.09,
                normals=(n + 0.3 * rn(P, 3)).contiguous(), viewdirs=F.normalize(rn(P, 3), dim=-1), incidents=inc.contiguous(),
                env=rn(1, He, 2 * He, 3), visibility=vis.contiguous(), incident_dirs=dirs.contiguous(),
                incident_areas=areas.contiguous(), cot_pbr=rn(P, 3), cot_diffuse=rn(P, 3), cot_specular=rn(P, 3))


SHARED = ("env", "transform")


def rows_of(t, idx):
    return {k: (v if k in SHARED else v[idx]) for k, v in t.items()}


def test_training_scale_against_fp64():
    """P = 1.5M, N = 32, env 16x32 (env_resolution = 16): the persistent grid-stride loop and the shared-memory
    env-gradient flush.  Per-Gaussian rows on a seeded 20k sample; the full env gradient in fp64, 100k rows at a time."""
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    P, N, He = 1_500_000, 32, 16
    cots = ("pbr", "diffuse")
    t = training_inputs(P, N, He, seed=77)
    zero_rows = int((t["incidents"].reshape(P, -1) == 0).all(1).sum())
    back = int(((t["normals"][:, None] * t["incident_dirs"]).sum(-1) < 0).sum())
    assert zero_rows > P // 5 and back > P, (zero_rows, back)
    ours = run_ours(t, cots)
    for k in ("pbr", "diffuse_light", "specular", "grad_base_color", "grad_roughness", "grad_viewdirs", "grad_incidents"):
        assert torch.isfinite(ours[k]).all(), k
    idx = torch.from_numpy(np.sort(np.random.default_rng(5).choice(P, 20_000, replace=False))).cuda()
    sub = rows_of(t, idx)
    r64, r32 = se.oracle_run(sub, torch.float64, cots), se.oracle_run(sub, torch.float32, cots)
    mags = se.oracle_magnitudes(sub, cots)
    for k in ("pbr", "diffuse_light", "specular"):
        check_rows("out", f"train1.5M {k}", ours[k][idx], r64[k], r32[k], mags[k])
    for k in ("base_color", "roughness", "viewdirs", "incidents"):
        check_rows("grad", f"train1.5M d_{k}", ours["grad_" + k][idx], r64["grad_" + k], r32["grad_" + k], mags["grad_" + k])
    del r64, r32, sub, mags
    g64 = torch.zeros(He, 2 * He, 3, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(g64)
    g32 = torch.zeros(He, 2 * He, 3, device="cuda")
    for s in range(0, P, 100_000):
        ch = rows_of(t, slice(s, s + 100_000))
        r = se.oracle_run(ch, torch.float64, cots)
        gs, m = se.env_scatter64(ch["incident_dirs"], r["g_light"], He, 2 * He)
        assert ((gs - r["grad_tex"].reshape(He, 2 * He, 3)).abs() <= 1e-12 * m).all()
        g64 += gs
        absc = {k: (v.abs() if k.startswith("cot_") else v) for k, v in ch.items()}
        mag += se.env_scatter64(ch["incident_dirs"], se.oracle_run(absc, torch.float64, cots)["g_light"], He, 2 * He)[1]
        del r
        g32 += se.oracle_run(ch, torch.float32, cots)["grad_tex"].reshape(He, 2 * He, 3)
    check_texels("train1.5M d_env texel", ours["grad_tex"], g64, g32, mag)
    dt = time.time() - t0
    print(f"[shade-edge] training-scale case: {dt:.1f} s, {zero_rows} zero-incident rows, peak memory "
          f"{torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert dt < 60, dt


# ---- bit-level invariants --------------------------------------------------------------------------------------------------
def _bits(x):
    return x.contiguous().view(torch.int32)


def test_forward_variants_bit_identical_and_reruns_reproducible():
    """Forward variants 0 and 1 at 8 lanes per Gaussian sum k = 0..15 in the same order (-fmad=false): bit-identical
    outputs.  Every variant: forward outputs and per-Gaussian gradients are bit-identical across two runs (only the env
    gradient uses float atomics)."""
    t = training_inputs(20_001, 32, 16, seed=9)
    outs = []
    for v in (0, 1):
        with tuned(dict(shade_group=8, shade_fwd_variant=v)):
            m = run_means(t)
            o = run_ours(t)
        outs.append(list(m) + [o[k] for k in se.EXTRAS[:3]])
    for a, b in zip(*outs):
        assert torch.equal(_bits(a), _bits(b))
    keys = ("pbr", "diffuse_light", "specular") + se.EXTRAS[:3] + tuple("grad_" + k for k in se.LEAVES[:4])
    for knobs in KNOBS:
        with tuned(knobs):
            a, b = run_ours(t), run_ours(t)
        for k in keys:
            assert torch.equal(_bits(a[k]), _bits(b[k])), (knobs, k)


# ---- no writes outside the outputs -----------------------------------------------------------------------------------------
SLACK = 256


@pytest.mark.parametrize("G", [8, 16, 32])
@pytest.mark.parametrize("P", [37, 4_097])
def test_no_writes_outside_outputs(G, P):
    """The C ABI with NaN-filled output buffers that run SLACK floats past row P: every output element is written,
    nothing after it.  P is not a multiple of 4, so the last warp has idle groups; at 32 lanes the `sub*RQ + q < 48`
    guard decides which lanes write d_incidents."""
    from relightable3dgaussian_b200 import _lib
    from relightable3dgaussian_b200.shading import _args
    lib = _lib.load()
    N, He = 24, 16
    t = training_inputs(P, N, He, seed=P)
    tex = F.softplus(t["env"])[0].contiguous()
    buf = lambda n: torch.full((n + SLACK,), float("nan"), device="cuda")
    sizes = dict(pbr=3 * P, diffuse_light=3 * P, specular=3 * P, mean_incident_lights=3 * P, mean_local_lights=3 * P,
                 mean_global_lights=3 * P, mean_visibility=P, incident_lights=3 * P * N, local_incident_lights=3 * P * N,
                 global_incident_lights=3 * P * N, dL_dbase_color=3 * P, dL_droughness=P, dL_dviewdirs=3 * P,
                 dL_dincidents=48 * P, dL_denv=tex.numel())
    out = {k: buf(n) for k, n in sizes.items()}
    a = _args(P, N, He, 2 * He)
    (a.base_color, a.roughness, a.normals, a.viewdirs, a.incidents, a.env, a.visibility, a.incident_dirs,
     a.incident_areas) = [x.data_ptr() for x in (t["base_color"], t["roughness"], t["normals"], t["viewdirs"],
                                                 t["incidents"], tex, t["visibility"], t["incident_dirs"], t["incident_areas"])]
    a.dL_dpbr, a.dL_ddiffuse_light, a.dL_dspecular = (t[k].data_ptr() for k in ("cot_pbr", "cot_diffuse", "cot_specular"))
    for k, v in out.items():
        setattr(a, k, v.data_ptr())
    stream = torch.cuda.current_stream().cuda_stream
    with tuned(dict(shade_group=G)):
        _lib.check(lib.r3dg_render_equation_forward(ctypes.byref(a), stream), "forward")
        _lib.check(lib.r3dg_render_equation_backward(ctypes.byref(a), stream), "backward")
        ref = run_ours(dict(t, env=t["env"]))
    torch.cuda.synchronize()
    for k, n in sizes.items():
        assert torch.isfinite(out[k][:n]).all(), (k, "not fully written")
        assert torch.isnan(out[k][n:]).all(), (k, "written past the end", int((~torch.isnan(out[k][n:])).sum()))
    for k, r in (("pbr", ref["pbr"]), ("dL_dincidents", ref["grad_incidents"]), ("dL_dviewdirs", ref["grad_viewdirs"]),
                 ("incident_lights", ref["incident_lights"])):
        assert torch.equal(_bits(out[k][:sizes[k]]), _bits(r.reshape(-1))), k


# ---- EnvLight with a general rotation: the seam ----------------------------------------------------------------------------
def test_general_rotation_seam_ambiguity_bounded():
    """`dirs @ T.T` in torch and the kernel's left-to-right dot products may round differently, so where the env-frame
    y is a few ulp of 0 with x < 0 the lookup can land in column 0 or We-1 on either side.  Those samples are found
    from the fp64 truth, counted, kept below SEAM_AMBIGUOUS_MAX of all samples and left out of the elementwise checks
    (their rows, and their taps on both sides of the seam in the per-texel bound); everything else is checked."""
    P, N, He = 50_000, 32, 16
    t = training_inputs(P, N, He, seed=31)
    g = torch.Generator().manual_seed(31)
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r))
    T = (q if torch.det(q) > 0 else -q).float().cuda()
    dirs = t["incident_dirs"]
    for _ in range(3):                           # |e_z| > 1 after rounding is NaN in the reference too: stay off the poles
        bad = (dirs @ T.T)[..., 2].abs() > 0.99
        dirs[bad] = F.normalize(dirs[bad] + torch.tensor([0.3, 0.3, 0.3], device="cuda") @ T, dim=-1)
    assert not ((dirs @ T.T)[..., 2].abs() > 0.99).any()
    # 64 samples planted on the seam (env-frame y = 0 before rounding to fp32), each lit by its row's normal
    a = torch.rand(64, generator=g, dtype=torch.float64) * 2 - 1
    e = torch.stack([-torch.cos(a), torch.zeros_like(a), torch.sin(a)], -1)
    planted = (e @ q.double() if torch.det(q) > 0 else e @ -q.double()).float().cuda()
    rows = torch.arange(64, device="cuda") * (P // 64)
    dirs[rows, 5] = planted
    t["normals"][rows] = planted
    t["visibility"][rows, 5] = 1.0
    t.update(transform=T, env=torch.rand(He, 2 * He, 3, generator=g).cuda() * 2)
    amb = seam_ambiguous(dirs, T)
    count = int(amb.sum())
    print(f"[shade-edge] general rotation: {count} of {P * N} samples ({count / (P * N):.2e}) have a rounding-dependent "
          f"env column; bound {SEAM_AMBIGUOUS_MAX:.0e}")
    assert 0 < count <= SEAM_AMBIGUOUS_MAX * P * N
    keep = ~amb.any(1)
    ours = run_ours(t)
    r64, r32 = se.oracle_run(t, torch.float64), se.oracle_run(t, torch.float32)
    mags = se.oracle_magnitudes(t)
    for k in ("pbr",) + se.EXTRAS:
        check_rows("out", f"rot seam {k}", ours[k], r64[k], r32[k], mags.get(k), keep=keep)
    for k in ("base_color", "roughness", "viewdirs", "incidents"):
        check_rows("grad", f"rot seam d_{k}", ours["grad_" + k], r64["grad_" + k], r32["grad_" + k], mags["grad_" + k], keep=keep)
    ef = se.env_frame(dirs.double(), T.double())
    grad, _ = se.env_scatter64(ef, r64["g_light"], He, 2 * He)
    a_idx = amb.reshape(-1)
    flip = ef[a_idx].clone()
    flip[:, 1] = -flip[:, 1]
    _, m_here = se.env_scatter64(ef[a_idx], r64["g_light"].reshape(-1, 3)[a_idx], He, 2 * He)
    _, m_there = se.env_scatter64(flip, r64["g_light"].reshape(-1, 3)[a_idx], He, 2 * He)
    check_texels("rot seam d_env texel", ours["grad_tex"], grad, r32["grad_tex"], mags["tex"], slack=(m_here + m_there) * (1 + 1e-6))

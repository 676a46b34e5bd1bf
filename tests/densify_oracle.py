"""Test-side code for the fused densification (relightable3dgaussian_b200/densify.py).

* `densify_case(name, device)`: seeded inputs of one case (parameters, Adam moments, statistics, thresholds).  The
  fixture generator (tests/golden/make_golden_densify.py) and the tests regenerate the same inputs from the name.
* `build_model(case, cls, optim_cls)`: a model object carrying the reference's attributes and an Adam optimizer whose
  state is that of two real steps, with the case's moments written over it.
* `restate_densify_and_prune` / `restate_add_densification_stats`: a PyTorch restatement of the reference's
  semantics (scene/gaussian_model.py:890-937) with the same tensor operations, so it is bit-exact to the reference
  on one device.  It also returns the masks and a per-output-row code `source_row * 4 + kind` (kind 0 original,
  1 clone, 2 split copy 1, 3 split copy 2).
* `StandIn`: a GaussianModel stand-in whose methods are the restatement, for install() and training-loop tests.
"""
import hashlib
import math

import numpy as np
import torch

STAGE1 = {"xyz": (3,), "normal": (3,), "rotation": (4,), "scaling": (3,), "opacity": (1,), "f_dc": (1, 3), "f_rest": (15, 3)}
PBR = {"base_color": (3,), "roughness": (1,), "incidents_dc": (1, 3), "incidents_rest": (15, 3), "visibility_dc": (1, 1),
       "visibility_rest": (15, 1)}
ATTRS = dict({"xyz": "_xyz", "normal": "_normal", "rotation": "_rotation", "scaling": "_scaling", "opacity": "_opacity",
              "f_dc": "_shs_dc", "f_rest": "_shs_rest"}, **{n: "_" + n for n in PBR})
STATS = ("weights_accum", "xyz_gradient_accum", "normal_gradient_accum", "denom")
LRS = {"xyz": 1.6e-4, "normal": 0.01, "rotation": 1e-3, "scaling": 5e-3, "opacity": 0.05, "f_dc": 2.5e-3, "f_rest": 1.25e-4,
       "base_color": 0.01, "roughness": 0.01, "incidents_dc": 2.5e-3, "incidents_rest": 1.25e-4, "visibility_dc": 2.5e-3,
       "visibility_rest": 1.25e-4}


def f32(x):
    return float(np.float32(x))


def up(x):
    return float(np.nextafter(np.float32(x), np.float32(np.inf)))


def down(x):
    return float(np.nextafter(np.float32(x), np.float32(-np.inf)))


BASE = dict(max_grad=0.0002, min_opacity=0.005, extent=4.0, max_screen_size=None, max_grad_normal=0.0004,
            weights_threshold=1e-4, percent_dense=0.01)
# name: (P, pbr, kind, overrides of BASE)
CASES = {
    "s1_p1": (1, False, "real", {}),
    "s1_p7": (7, False, "real", {}),
    "s1_p2049": (2049, False, "real", {}),
    "s1_p20k": (20011, False, "real", {}),
    "pbr_p7": (7, True, "real", {}),
    "pbr_p2049": (2049, True, "real", {}),
    "none": (513, False, "none", {}),
    "all_clone": (300, False, "all_clone", {}),
    "all_split": (2049, True, "all_split", {}),
    "all_pruned": (257, False, "real", {"min_opacity": 1.5}),
    "denom0": (300, False, "denom0", {}),
    "denom0_zero_thr": (300, False, "denom0", {"max_grad": 0.0, "max_grad_normal": 0.0}),   # NaN -> 0 passes 0 >= 0
    "normal_only": (600, False, "normal_only", {}),
    "mss_none": (1500, False, "big", {}),
    "mss_20": (1500, False, "big", {"max_screen_size": 20}),
    "no_state": (700, True, "real", {"no_state": "incidents_rest"}),
    "thr_nonpos": (300, False, "real", {"max_grad": 0.0, "max_grad_normal": -1.0}),
    "thr_grad": (64, False, "thr_grad", {}),
    "thr_weights": (64, False, "thr_weights", {}),
    "thr_scale_at": (64, False, "unit_scale", {"percent_dense": 0.25}),
    "thr_scale_up": (64, False, "unit_scale", {"percent_dense": up(1.0) / 4.0}),
    "thr_scale_down": (64, False, "unit_scale", {"percent_dense": down(1.0) / 4.0}),
    "thr_scale_py": (64, False, "unit_scale", {"percent_dense": (1.0 + 2.0 ** -30) / 4.0}),
    "thr_opacity_at": (64, False, "half_opacity", {"min_opacity": 0.5}),
    "thr_opacity_up": (64, False, "half_opacity", {"min_opacity": up(0.5)}),
    "thr_opacity_down": (64, False, "half_opacity", {"min_opacity": down(0.5)}),
    "thr_opacity_py": (64, False, "half_opacity", {"min_opacity": 0.5 + 2.0 ** -30}),
    "thr_big_at": (64, False, "unit_big", {"extent": 10.0, "max_screen_size": 20}),
    "thr_big_up": (64, False, "unit_big", {"extent": up(1.0) / 0.1, "max_screen_size": 20}),
    "thr_big_down": (64, False, "unit_big", {"extent": down(1.0) / 0.1, "max_screen_size": 20}),
}
FIXTURE_CASES = list(CASES)
# GPU-only sizes (generated on the device; the restatement runs on the same device)
LARGE = {"s1_p1m": (1 << 20, False, "real", {}), "s1_p3m": (3 * (1 << 20), False, "real", {}),
         "pbr_p1m": (1 << 20, True, "real", {})}


def case_params(name):
    P, pbr, kind, over = (CASES.get(name) or LARGE[name])
    prm = dict(BASE, **over)
    return P, pbr, kind, prm


def _u(g, shape, lo, hi, device):
    return torch.rand(shape, generator=g, device=device) * (hi - lo) + lo


def densify_case(name, device="cpu"):
    """Seeded inputs of case `name`: dict(P, pbr, params {group: tensor}, moments {group: (m, v) or None},
    stats {name: tensor}, max_radii2D, args (the reference's call arguments), percent_dense)."""
    P, pbr, kind, prm = case_params(name)
    seed = int(hashlib.sha256(name.encode()).hexdigest()[:8], 16)
    g = torch.Generator(device=device).manual_seed(seed)
    shapes = dict(STAGE1, **(PBR if pbr else {}))
    params = {n: torch.randn((P,) + s, generator=g, device=device) for n, s in shapes.items()}
    params["xyz"] *= 2.0
    u = torch.rand(P, generator=g, device=device)
    cls = torch.zeros(P, dtype=torch.int64, device=device)          # 0 plain, 1 clone, 2 split, 3 prune
    if kind in ("real", "big", "denom0"):
        cls[u < 0.02] = 1
        cls[(u >= 0.02) & (u < 0.03)] = 2
        cls[(u >= 0.03) & (u < 0.06)] = 3
    elif kind == "all_clone":
        cls[:] = 1
    elif kind == "all_split":
        cls[:] = 2
    elif kind == "normal_only":
        cls[u < 0.1] = 1
        cls[(u >= 0.1) & (u < 0.2)] = 2
    denom = torch.randint(1, 50, (P, 1), generator=g, device=device).float()
    sel = (cls == 1) | (cls == 2)
    ratio = torch.where(sel[:, None], _u(g, (P, 1), 3e-4, 1e-2, device), _u(g, (P, 1), 0.0, 1.5e-4, device))
    nratio = _u(g, (P, 1), 0.0, 3e-4, device)
    if kind == "normal_only":
        nratio = torch.where(sel[:, None], _u(g, (P, 1), 5e-4, 1e-2, device), nratio)
        ratio = _u(g, (P, 1), 0.0, 1.5e-4, device)
    xacc, nacc = ratio * denom, nratio * denom
    # scales: clone rows below percent_dense * extent, split rows above, the rest anywhere
    dense = prm["percent_dense"] * prm["extent"]
    sc = _u(g, (P, 3), 0.2 * dense, 8 * dense, device)
    sc = torch.where((cls == 1)[:, None], _u(g, (P, 3), 0.05 * dense, 0.9 * dense, device), sc)
    big = torch.where((cls == 2)[:, None], _u(g, (P, 3), 1.2 * dense, 6 * dense, device), sc)
    sc = big
    opac = _u(g, (P, 1), 0.05, 0.99, device)
    w = _u(g, (P, 1), 1e-3, 1.0, device)
    pr = cls == 3
    half = torch.rand(P, generator=g, device=device) < 0.5
    opac = torch.where((pr & half)[:, None], _u(g, (P, 1), 1e-4, 4e-3, device), opac)
    w = torch.where((pr & ~half)[:, None], _u(g, (P, 1), 0.0, 5e-5, device), w)
    if kind == "big":                       # world-space giants: pruned only when max_screen_size is given
        gi = torch.rand(P, generator=g, device=device) < 0.05
        sc = torch.where(gi[:, None], _u(g, (P, 3), 0.11 * prm["extent"], 0.3 * prm["extent"], device), sc)
    params["scaling"] = torch.log(sc)
    params["opacity"] = torch.log(opac / (1 - opac))
    mr = _u(g, (P,), 0.0, 10.0, device).floor()
    if kind == "big":
        mr = mr + 1000.0                    # far above 20: must not prune (the reference zeroed max_radii2D first)
    if kind == "none":
        xacc, nacc = xacc * 0, nacc * 0
    if kind == "denom0":
        z0 = torch.rand(P, generator=g, device=device) < 0.3
        denom = torch.where(z0[:, None], torch.zeros_like(denom), denom)
        zz = torch.rand(P, generator=g, device=device) < 0.5                 # 0/0 = NaN -> 0, x/0 = inf stays
        xacc = torch.where((z0 & zz)[:, None], torch.zeros_like(xacc), xacc)
        nacc = torch.where((z0 & ~zz)[:, None], torch.zeros_like(nacc), nacc)
    if kind == "thr_grad":                  # g and gn at the fp32 thresholds and one ulp either side (denom = 1)
        denom = torch.ones_like(denom)
        vals = [f32(prm["max_grad"]), up(prm["max_grad"]), down(prm["max_grad"])]
        nvals = [f32(prm["max_grad_normal"]), up(prm["max_grad_normal"]), down(prm["max_grad_normal"])]
        xacc = torch.tensor([vals[i % 3] if i % 2 == 0 else 0.0 for i in range(P)], device=device)[:, None]
        nacc = torch.tensor([nvals[i % 3] if i % 2 == 1 else 0.0 for i in range(P)], device=device)[:, None]
        params["scaling"][: P // 2] = math.log(0.5 * dense)                  # first half clone candidates, rest split
    if kind == "thr_weights":
        wt = prm["weights_threshold"]
        w = torch.tensor([[f32(wt), up(wt), down(wt)][i % 3] for i in range(P)], device=device)[:, None]
    if kind in ("unit_scale", "unit_big"):  # exp(0) = 1 exactly on every device: the thresholds move instead
        params["scaling"] = torch.where((torch.arange(P, device=device) % 2 == 0)[:, None],
                                        torch.zeros_like(params["scaling"]), params["scaling"])
        xacc = torch.where((torch.arange(P, device=device) % 4 < 2)[:, None], 1e-2 * denom, xacc)
    if kind == "half_opacity":              # sigmoid(0) = 0.5 exactly
        params["opacity"] = torch.where((torch.arange(P, device=device) % 2 == 0)[:, None],
                                        torch.zeros_like(params["opacity"]), params["opacity"])
        xacc = torch.where((torch.arange(P, device=device) % 3 == 0)[:, None], 1e-2 * denom, xacc)
    stats = {"weights_accum": w, "xyz_gradient_accum": xacc.contiguous(), "normal_gradient_accum": nacc.contiguous(),
             "denom": denom}
    moments = {}
    for n, t in params.items():
        m = torch.randn(t.shape, generator=g, device=device) * 1e-3
        v = torch.rand(t.shape, generator=g, device=device) * 1e-6
        moments[n] = None if prm.get("no_state") == n else (m, v)
    args = dict(max_grad=prm["max_grad"], min_opacity=prm["min_opacity"], extent=prm["extent"],
                max_screen_size=prm["max_screen_size"], max_grad_normal=prm["max_grad_normal"],
                weights_threshold=prm["weights_threshold"])
    return dict(name=name, P=P, pbr=pbr, params={n: t.contiguous() for n, t in params.items()}, moments=moments,
                stats=stats, max_radii2D=mr, args=args, percent_dense=prm["percent_dense"], seed=seed)


def build_model(case, cls, optim_cls=torch.optim.Adam, device=None):
    """An instance of `cls` (its __init__ is not called) with the case's tensors and an optimizer in the reference's
    layout.  Groups with state went through two real steps; their parameters and moments are then overwritten with the
    case's values.  A group named in the case's `no_state` has no state at all."""
    dev = device or next(iter(case["params"].values())).device
    m = cls.__new__(cls)
    m.use_pbr = case["pbr"]
    m.percent_dense = case["percent_dense"]
    groups = []
    for n, t in case["params"].items():
        p = torch.nn.Parameter(t.to(dev).clone().requires_grad_(True))
        setattr(m, ATTRS[n], p)
        groups.append({"params": [p], "lr": LRS[n], "name": n})
    m.optimizer = optim_cls(groups, lr=0.0, eps=1e-15)
    stepped = [g["params"][0] for g in groups if case["moments"][g["name"]] is not None]
    for _ in range(2):
        for p in stepped:
            p.grad = torch.full_like(p, 1e-3)
        m.optimizer.step()
    with torch.no_grad():
        for g in groups:
            p = g["params"][0]
            p.grad = None
            p.copy_(case["params"][g["name"]].to(dev))
            mv = case["moments"][g["name"]]
            if mv is not None:
                m.optimizer.state[p]["exp_avg"].copy_(mv[0].to(dev))
                m.optimizer.state[p]["exp_avg_sq"].copy_(mv[1].to(dev))
    for n, t in case["stats"].items():
        setattr(m, n, t.to(dev).clone())
    m.max_radii2D = case["max_radii2D"].to(dev).clone()
    return m


def rotation_matrices(q):
    """The reference's build_rotation restated: normalise, then the usual quaternion matrix, op by op in the same order."""
    n = torch.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3])
    r, x, y, z = (q / n[:, None]).unbind(1)
    rows = [1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
            2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
            2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]
    return torch.stack(rows, 1).reshape(-1, 3, 3)


def restate_densify_and_prune(m, max_grad, min_opacity, extent, max_screen_size, max_grad_normal, weights_threshold=1e-4,
                              z=None, verbose=True):
    """The reference's densify_and_prune on model `m`, in place.  z: injected [2|S|,3] standard normals, or None to
    call torch.normal(mean=0, std) as the reference does.  Returns dict(clone, split, prune, code, z, counts)."""
    dev = m._xyz.device
    opt = m.optimizer
    groups = [(g, g["name"]) for g in opt.param_groups]
    P = m._xyz.shape[0]
    code = torch.arange(P, device=dev) * 4
    grads = m.xyz_gradient_accum / m.denom
    grads_n = m.normal_gradient_accum / m.denom
    grads = torch.where(grads.isnan(), torch.zeros_like(grads), grads)
    grads_n = torch.where(grads_n.isnan(), torch.zeros_like(grads_n), grads_n)
    smax = torch.exp(m._scaling).max(dim=1).values
    dense = m.percent_dense * extent
    clone = ((torch.norm(grads, dim=-1) >= max_grad) | (torch.norm(grads_n, dim=-1) >= max_grad_normal)) & (smax <= dense)

    def grow(new_rows, weights_new):
        for g, n in groups:
            old = g["params"][0]
            st = opt.state.get(old, None)
            ext = new_rows[n]
            newp = torch.nn.Parameter(torch.cat((old, ext), dim=0).requires_grad_(True))
            if st is not None:
                st["exp_avg"] = torch.cat((st["exp_avg"], torch.zeros_like(ext)), dim=0)
                st["exp_avg_sq"] = torch.cat((st["exp_avg_sq"], torch.zeros_like(ext)), dim=0)
                del opt.state[old]
                opt.state[newp] = st
            g["params"][0] = newp
            setattr(m, ATTRS[n], newp)
        m.weights_accum = torch.cat([m.weights_accum, weights_new], dim=0)

    def keep_rows(keep):
        for g, n in groups:
            old = g["params"][0]
            st = opt.state.get(old, None)
            newp = torch.nn.Parameter(old[keep].requires_grad_(True))
            if st is not None:
                st["exp_avg"], st["exp_avg_sq"] = st["exp_avg"][keep], st["exp_avg_sq"][keep]
                del opt.state[old]
                opt.state[newp] = st
            g["params"][0] = newp
            setattr(m, ATTRS[n], newp)
        m.weights_accum = m.weights_accum[keep]

    nC = int(clone.sum())
    grow({n: g["params"][0][clone] for g, n in groups}, torch.ones((nC, 1), device=dev))
    code = torch.cat((code, code[clone] + 1))
    P1 = P + nC
    pad = torch.zeros(P1, device=dev)
    pad[:P] = grads.squeeze()
    pad_n = torch.zeros(P1, device=dev)
    pad_n[:P] = grads_n.squeeze()
    sel_n = pad_n >= max_grad_normal
    n_normal = int(sel_n.sum())
    split = ((pad >= max_grad) | sel_n) & (torch.exp(m._scaling).max(dim=1).values > dense)
    nS = int(split.sum())
    stds = torch.exp(m._scaling)[split].repeat(2, 1)
    means = torch.zeros((stds.size(0), 3), device=dev)
    if z is None:
        gen_state = torch.cuda.get_rng_state(dev) if dev.type == "cuda" else torch.get_rng_state()
        samples = torch.normal(mean=means, std=stds)
        if dev.type == "cuda":                                     # recover z from the same generator state
            torch.cuda.set_rng_state(gen_state, dev)
        else:
            torch.set_rng_state(gen_state)
        z_used = torch.empty_like(stds).normal_(0, 1)
    else:
        z_used = z.to(dev)
        samples = z_used.clone().mul_(stds).add_(means)
    rots = rotation_matrices(m._rotation[split]).repeat(2, 1, 1)
    new = {}
    for g, n in groups:
        src = g["params"][0][split]
        new[n] = src.repeat(2, *([1] * (src.dim() - 1)))
    new["xyz"] = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + m._xyz[split].repeat(2, 1)
    new["scaling"] = torch.log(torch.exp(m._scaling)[split].repeat(2, 1) / (0.8 * 2))
    grow(new, torch.ones((2 * nS, 1), device=dev))
    code = torch.cat((code, code[split] + 2, code[split] + 3))
    keep = ~torch.cat((split, torch.zeros(2 * nS, device=dev, dtype=torch.bool)))
    keep_rows(keep)
    code = code[keep]
    P2 = m._xyz.shape[0]
    prune = (torch.sigmoid(m._opacity) < min_opacity).squeeze(-1)
    light = m.weights_accum[:, 0] < weights_threshold
    prune = prune | light
    if verbose:
        print("densify_and_split_normal:", n_normal, "/", P1)
        print("weights_accum:", int(light.sum()), "/", P2)
    if max_screen_size:
        prune = prune | (torch.zeros(P2, device=dev) > max_screen_size) | (torch.exp(m._scaling).max(dim=1).values > 0.1 * extent)
    keep_rows(~prune)
    code = code[~prune]
    Pn = m._xyz.shape[0]
    for n in STATS:
        setattr(m, n, torch.zeros((Pn, 1), device=dev))
    m.max_radii2D = torch.zeros((Pn,), device=dev)
    return dict(clone=clone, split=split[:P], prune=prune, code=code, z=z_used,
                counts=(n_normal, P1, int(light.sum()), P2))


def restate_add_densification_stats(m, viewspace_point_tensor, update_filter, weights, radii=None):
    m.weights_accum += weights
    gxy = viewspace_point_tensor.grad[update_filter, :2]
    m.xyz_gradient_accum[update_filter] += torch.norm(gxy, dim=-1, keepdim=True)
    m.normal_gradient_accum[update_filter] += torch.norm(m._normal.grad[update_filter], dim=-1, keepdim=True)
    m.denom[update_filter] += 1
    if radii is not None:
        m.max_radii2D[update_filter] = torch.max(m.max_radii2D[update_filter], radii[update_filter])


class StandIn:
    """GaussianModel stand-in: the reference's attribute layout, activations, and the restatement as its methods."""

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_scaling(self):
        return torch.exp(self._scaling)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    def add_densification_stats(self, viewspace_point_tensor, update_filter, weights):
        restate_add_densification_stats(self, viewspace_point_tensor, update_filter, weights)

    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, max_grad_normal, weights_threshold=1e-4):
        self.last = restate_densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, max_grad_normal,
                                              weights_threshold)


def output_tensors(m):
    """{name: tensor} of everything densify_and_prune replaces: parameters, moments (when present) and statistics."""
    out = {}
    for g in m.optimizer.param_groups:
        n, p = g["name"], g["params"][0]
        out[f"param/{n}"] = p.detach()
        st = m.optimizer.state.get(p, None)
        if st is not None:
            out[f"exp_avg/{n}"], out[f"exp_avg_sq/{n}"] = st["exp_avg"], st["exp_avg_sq"]
    for n in STATS + ("max_radii2D",):
        out[f"stat/{n}"] = getattr(m, n)
    return out


def digest(t):
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy()).tobytes()).hexdigest()


def expected_from_code(case, code, split_xyz, split_scaling):
    """The outputs implied by a row code and the split copies' new xyz / scaling: copies of the inputs' rows, zero
    moments and statistics for new rows.  Used to compare the GPU result with the fixture."""
    src = torch.as_tensor(code // 4).long()
    kind = torch.as_tensor(code % 4)
    new_row = kind > 0
    splitrow = kind >= 2
    out = {}
    for n, t in case["params"].items():
        e = t[src].clone()
        if n == "xyz":
            e[splitrow] = torch.as_tensor(split_xyz)
        if n == "scaling":
            e[splitrow] = torch.as_tensor(split_scaling)
        out[f"param/{n}"] = e
        mv = case["moments"][n]
        if mv is not None:
            for k, mt in zip(("exp_avg", "exp_avg_sq"), mv):
                e = mt[src].clone()
                e[new_row] = 0
                out[f"{k}/{n}"] = e
    Pn = len(src)
    for n in STATS:
        out[f"stat/{n}"] = torch.zeros((Pn, 1))
    out["stat/max_radii2D"] = torch.zeros((Pn,))
    return out

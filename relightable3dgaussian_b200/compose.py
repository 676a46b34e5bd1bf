"""Similarity transforms of Gaussian models, for composing objects into one scene (include/r3dg_b200.h, COMPOSE).

The reference composes relighting scenes with `GaussianModel.set_transform` (scene/gaussian_model.py:89-112), which
moves xyz, normals, quaternions and log-scales but leaves every SH tensor as it was: after a rotation the object's
stage-1 radiance (`f_rest`), learned incident light (`incidents_rest`) and visibility (`visibility_rest`) still point
the way they did before.  Here every SH "rest" tensor is rotated with the object, band by band, by the matrix D^l(R)
defined by  sum_m Y_lm(d) c'_m = sum_m Y_lm(R^T d) c_m  for every direction d, so an object renders and lights the
same from every view after it is moved.

    quat, t, s = pose_from_matrix(M)                # [4,4] or [K,4,4] similarity -> (quat [K,4], t [K,3], s [K])
    scene = compose([model_a, model_b], [M_a, M_b])  # the concatenation, transformed in one launch
    xyz, normal, rotation, scaling, shs = transform_gaussians(...)   # one autograd node, gradients to the pose too

Models are the dicts of formats.py.  `install()` rebinds the reference's `GaussianModel.set_transform` to this
kernel, so the reference's relighting.py gets rotated SH unchanged.

There is no PyTorch fallback: CUDA float32 tensors only, anything else raises before a launch.
"""
import ctypes

import torch

from . import _lib

MAX_OBJECTS = 64          # R3DG_MAX_OBJECTS (include/r3dg_b200.h)
MAX_SH = 3                # R3DG_COMPOSE_MAX_SH
SH_KEYS = ("f_rest", "incidents_rest", "visibility_rest")
SIMILARITY_RTOL = 1e-4    # relative tolerance of M^T M = s^2 I in pose_from_matrix


def build_rotation(q):
    """R(q / |q|) [K,3,3] of quaternions (w,x,y,z) [K,4]: the reference's build_rotation convention."""
    q = q / q.norm(dim=-1, keepdim=True)
    r, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(q.shape[:-1] + (3, 3))


def _sh_degree(t):
    n = t.shape[1] + 1 if t.dim() == 3 else 0
    L = int(round(n ** 0.5)) - 1
    if t.dim() != 3 or (L + 1) ** 2 != n or L > 4 or t.shape[2] not in (1, 3):
        raise ValueError(f"an SH rest tensor must be [P,(L+1)^2-1,C] with L <= 4 and C in (1, 3) (got {tuple(t.shape)})")
    return L


def _offsets(offsets, P, K):
    if offsets is None:
        if K != 1:
            raise ValueError(f"offsets are required for K = {K} objects")
        offsets = [0, P]
    o = [int(v) for v in (offsets.tolist() if torch.is_tensor(offsets) else offsets)]
    if len(o) != K + 1 or o[0] != 0 or o[-1] != P or any(b < a for a, b in zip(o, o[1:])):
        raise ValueError(f"offsets must rise from 0 to P = {P} in K + 1 = {K + 1} steps (got {o})")
    return o


def _args(P, K, offsets_c, pose, rows, shs):
    a = _lib.ComposeArgs()
    a.P, a.K = P, K
    a.offsets = ctypes.cast(offsets_c, ctypes.c_void_p)
    a.quat, a.translation, a.scale = [_lib.ptr(t) for t in pose]
    a.xyz, a.normal, a.rotation, a.scaling = [_lib.ptr(t) for t in rows]
    a.n_sh = len(shs)
    for i, t in enumerate(shs):
        a.sh_degree[i], a.sh_channels[i], a.sh[i] = _sh_degree(t), t.shape[2], _lib.ptr(t)
    return a


class _Transform(torch.autograd.Function):
    """transform_gaussians as one node: inputs (xyz, normal, rotation, scaling, quat, translation, scale, *shs)."""

    @staticmethod
    def forward(ctx, offsets, xyz, normal, rotation, scaling, quat, translation, scale, *shs):
        P, K = xyz.shape[0], quat.shape[0]
        pose = [_lib.f32(t) for t in (quat, translation, scale)]
        rows = [_lib.f32(t) for t in (xyz, normal, rotation, scaling)]
        shs_c = [_lib.f32(t) for t in shs]
        outs = [torch.empty_like(t) for t in rows]
        sh_outs = [torch.empty_like(t) for t in shs_c]
        offsets_c = (ctypes.c_int32 * (K + 1))(*offsets)
        a = _args(P, K, offsets_c, pose, rows, shs_c)
        a.xyz_out, a.normal_out, a.rotation_out, a.scaling_out = [_lib.ptr(t) for t in outs]
        for i, t in enumerate(sh_outs):
            a.sh_out[i] = _lib.ptr(t)
        if P > 0:
            _lib.call("r3dg_compose_forward", xyz.device, ctypes.byref(a), what="compose")
        ctx.save_for_backward(*pose, *rows, *shs_c)
        ctx.offsets, ctx.n_sh = offsets, len(shs)
        return (*outs, *sh_outs)

    @staticmethod
    def backward(ctx, *grads):
        saved = ctx.saved_tensors
        pose, rows, shs = saved[:3], saved[3:7], saved[7:]
        quat, scale = pose[0], pose[2]
        P, K = rows[0].shape[0], quat.shape[0]
        dev = rows[0].device
        gz = [torch.zeros_like(t) if g is None else _lib.f32(g) for g, t in zip(grads, list(rows) + list(shs))]
        d_rows = [torch.empty_like(t) for t in rows]
        d_shs = [torch.empty_like(t) for t in shs]
        f = dict(dtype=torch.float32, device=dev)
        dR, dq, dt, ds = (torch.empty((K, 9), **f), torch.empty((K, 4), **f), torch.empty((K, 3), **f),
                          torch.empty((K,), **f))
        offsets_c = (ctypes.c_int32 * (K + 1))(*ctx.offsets)
        a = _args(P, K, offsets_c, pose, rows, shs)
        a.dL_dxyz_out, a.dL_dnormal_out, a.dL_drotation_out, a.dL_dscaling_out = [_lib.ptr(t) for t in gz[:4]]
        a.dL_dxyz, a.dL_dnormal, a.dL_drotation, a.dL_dscaling = [_lib.ptr(t) for t in d_rows]
        for i in range(len(shs)):
            a.dL_dsh_out[i], a.dL_dsh[i] = _lib.ptr(gz[4 + i]), _lib.ptr(d_shs[i])
        a.dL_dR, a.dL_dquat, a.dL_dtranslation, a.dL_dscale = [_lib.ptr(t) for t in (dR, dq, dt, ds)]
        work = _lib.scratch(_lib.load().r3dg_compose_work_bytes(P, K), dev)
        a.work, a.work_bytes = _lib.ptr(work), work.numel()
        _lib.call("r3dg_compose_backward", dev, ctypes.byref(a), what="compose backward")
        # the K-row chain through q^ = q / |q| and R(q^)
        with torch.enable_grad():
            q = quat.detach().double().requires_grad_(True)
            qn = q / q.norm(dim=-1, keepdim=True)
            surrogate = (build_rotation(qn).reshape(K, 9) * dR.double()).sum() + (qn * dq.double()).sum()
            d_quat, = torch.autograd.grad(surrogate, q)
        return (None, *d_rows, d_quat.float(), dt, ds, *d_shs)


def transform_gaussians(xyz, normal, rotation, scaling, sh_rests, quat, translation, scale, offsets=None):
    """Apply K similarities to K contiguous row ranges of a model, as one autograd node.

    xyz, normal, scaling [P,3] (log-scales), rotation [P,4] (w,x,y,z), sh_rests: up to MAX_SH tensors
    [P,(L+1)^2-1,C] (L <= 4, C in (1, 3)); quat [K,4] (normalised here, as build_rotation does), translation [K,3],
    scale [K] (> 0); offsets: K + 1 host ints from 0 to P (None for K = 1).  Object k's rows get
    xyz' = s R xyz + t, normal' = R normal, rotation' = q^ (x) rotation, scaling' = scaling + log s and every SH band
    rotated by D^l(R).  Returns (xyz', normal', rotation', scaling', [sh' ...]).  Gradients reach every input,
    the pose included."""
    sh_rests = list(sh_rests)
    quat, translation = quat.reshape(-1, 4), translation.reshape(-1, 3)
    scale = torch.as_tensor(scale, dtype=torch.float32, device=quat.device).reshape(-1)
    K, P = quat.shape[0], xyz.shape[0]
    if not 1 <= K <= MAX_OBJECTS:
        raise ValueError(f"transform_gaussians takes 1 to {MAX_OBJECTS} objects (got {K})")
    if translation.shape != (K, 3) or scale.shape != (K,):
        raise ValueError(f"translation must be [K,3] and scale [K] with K = {K}")
    if len(sh_rests) > MAX_SH:
        raise ValueError(f"at most {MAX_SH} SH tensors per call (got {len(sh_rests)})")
    for name, t, w in (("xyz", xyz, 3), ("normal", normal, 3), ("rotation", rotation, 4), ("scaling", scaling, 3)):
        if t.shape != (P, w):
            raise ValueError(f"{name} must be [P,{w}] with P = {P} (got {tuple(t.shape)})")
    for t in sh_rests:
        _sh_degree(t)
        if t.shape[0] != P:
            raise ValueError(f"SH tensors must have P = {P} rows (got {tuple(t.shape)})")
    o = _offsets(offsets, P, K)
    tensors = [xyz, normal, rotation, scaling, quat, translation, scale] + sh_rests
    if not all(t.is_cuda for t in tensors):
        raise RuntimeError("transform_gaussians runs on the GPU only (no CPU path)")
    if len({t.device for t in tensors}) != 1:
        raise ValueError("every input of transform_gaussians must be on one device")
    if not bool((scale > 0).all()):
        raise ValueError("scale must be positive")
    out = _Transform.apply(o, xyz, normal, rotation, scaling, quat, translation, scale, *sh_rests)
    return out[0], out[1], out[2], out[3], list(out[4:])


def _quat_from_rotation(R):
    """Unit quaternions (w,x,y,z) [K,4] of rotation matrices [K,3,3] by the largest of the diagonal terms (Shepperd),
    so no branch divides by a small number; w >= 0."""
    r00, r11, r22 = R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]
    cand = torch.stack([r00 + r11 + r22, r00, r11, r22], -1)
    pick = cand.argmax(-1)
    out = torch.empty(R.shape[0], 4, dtype=R.dtype, device=R.device)
    for k in range(R.shape[0]):
        m = R[k]
        if pick[k] == 0:
            w = 0.5 * torch.sqrt(1 + cand[k, 0])
            q = [w, (m[2, 1] - m[1, 2]) / (4 * w), (m[0, 2] - m[2, 0]) / (4 * w), (m[1, 0] - m[0, 1]) / (4 * w)]
        elif pick[k] == 1:
            x = 0.5 * torch.sqrt(1 + m[0, 0] - m[1, 1] - m[2, 2])
            q = [(m[2, 1] - m[1, 2]) / (4 * x), x, (m[0, 1] + m[1, 0]) / (4 * x), (m[0, 2] + m[2, 0]) / (4 * x)]
        elif pick[k] == 2:
            y = 0.5 * torch.sqrt(1 - m[0, 0] + m[1, 1] - m[2, 2])
            q = [(m[0, 2] - m[2, 0]) / (4 * y), (m[0, 1] + m[1, 0]) / (4 * y), y, (m[1, 2] + m[2, 1]) / (4 * y)]
        else:
            z = 0.5 * torch.sqrt(1 - m[0, 0] - m[1, 1] + m[2, 2])
            q = [(m[1, 0] - m[0, 1]) / (4 * z), (m[0, 2] + m[2, 0]) / (4 * z), (m[1, 2] + m[2, 1]) / (4 * z), z]
        q = torch.stack(q)
        q = q / q.norm()
        out[k] = q if q[0] >= 0 else -q
    return out


def pose_from_matrix(M):
    """(quat [K,4], t [K,3], s [K]) of similarities M [4,4] or [K,4,4] = [[s R, t], [0, 0, 0, 1]], in float32 on M's
    device.  Refuses, with ValueError, a bottom row other than [0, 0, 0, 1], a reflection or a singular matrix
    (det <= 0), and shear or non-uniform scale (M^T M = s^2 I off by more than SIMILARITY_RTOL relative): none of
    them is a similarity."""
    M = torch.as_tensor(M)
    if M.shape[-2:] != (4, 4) or M.dim() not in (2, 3):
        raise ValueError(f"pose_from_matrix takes [4,4] or [K,4,4] (got {tuple(M.shape)})")
    dev = M.device
    M = M.detach().double().cpu().reshape(-1, 4, 4)
    bottom = torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64)
    if not bool((M[:, 3] == bottom).all()):
        raise ValueError("pose_from_matrix: the bottom row must be [0, 0, 0, 1] (not an affine transform)")
    A = M[:, :3, :3]
    det = torch.linalg.det(A)
    if not bool((det > 0).all()):
        raise ValueError("pose_from_matrix: det <= 0: a reflection or a singular matrix is not a similarity")
    s = det.pow(1.0 / 3.0)
    gram = A.transpose(1, 2) @ A
    err = (gram - s[:, None, None] ** 2 * torch.eye(3, dtype=torch.float64)).abs().amax(dim=(1, 2))
    if not bool((err <= SIMILARITY_RTOL * s ** 2).all()):
        raise ValueError("pose_from_matrix: M^T M is not s^2 I: shear or non-uniform scale is not a similarity")
    quat = _quat_from_rotation(A / s[:, None, None])
    return quat.float().to(dev), M[:, :3, 3].float().to(dev), s.float().to(dev)


def _pose(p):
    if torch.is_tensor(p) and p.shape[-2:] == (4, 4):
        return pose_from_matrix(p)
    q, t, s = p
    return q.reshape(-1, 4), t.reshape(-1, 3), torch.as_tensor(s, dtype=torch.float32, device=q.device).reshape(-1)


def _apply(model, quat, t, s, offsets):
    keys = [k for k in SH_KEYS if k in model]
    xyz, normal, rotation, scaling, shs = transform_gaussians(model["xyz"], model["normal"], model["rotation"],
                                                              model["scaling"], [model[k] for k in keys], quat, t, s,
                                                              offsets)
    out = dict(model)
    out.update(xyz=xyz, normal=normal, rotation=rotation, scaling=scaling)
    out.update(zip(keys, shs))
    return out


def transform(model, quat, t, s):
    """A new model dict (formats.py keys): `model` moved by one similarity (quat [4] or [1,4], t [3], s).  xyz, normal,
    rotation, scaling and every SH rest tensor present are new; the other entries are the same tensors."""
    return _apply(model, quat.reshape(1, 4), t.reshape(1, 3), torch.as_tensor(s).reshape(1), None)


def compose(models, poses):
    """The concatenation of `models` (formats.py dicts with the same keys and trailing shapes), each moved by its pose
    (a [4,4] similarity or a (quat, t, s) triple), transformed in one launch.  Returns a new model dict."""
    if len(models) != len(poses) or not 1 <= len(models) <= MAX_OBJECTS:
        raise ValueError(f"compose takes 1 to {MAX_OBJECTS} models with one pose each")
    keys = list(models[0])
    for m in models[1:]:
        if list(m) != keys or any(m[k].shape[1:] != models[0][k].shape[1:] for k in keys):
            raise ValueError("compose: every model must have the same keys and trailing shapes")
    merged = {k: torch.cat([m[k] for m in models]) for k in keys}
    ps = [_pose(p) for p in poses]
    quat, t, s = (torch.cat([p[i] for p in ps]).to(merged["xyz"].device) for i in range(3))
    offsets = [0]
    for m in models:
        offsets.append(offsets[-1] + m["xyz"].shape[0])
    return _apply(merged, quat, t, s, offsets)


# ---- the reference's GaussianModel.set_transform -------------------------------------------------------------------
ATTRS = dict(xyz="_xyz", normal="_normal", rotation="_rotation", scaling="_scaling", f_rest="_shs_rest",
             incidents_rest="_incidents_rest", visibility_rest="_visibility_rest")


def set_transform(model, rotation=None, center=None, scale=None, offset=None, transform=None):
    """`GaussianModel.set_transform` (scene/gaussian_model.py:89-112) on the kernel, with the SH rotated.  `transform`
    is a [4,4] similarity; otherwise center, rotation [3,3], a uniform scale and offset compose into one similarity
    xyz' = s R (xyz - center) + offset, i.e. t = offset - s R center.  Parameters are replaced in place (`.data`)."""
    dev = model._xyz.device
    if transform is not None:
        quat, t, s = pose_from_matrix(torch.as_tensor(transform).to(dev))
    else:
        R = torch.eye(3, dtype=torch.float64) if rotation is None else torch.as_tensor(rotation).detach().double().cpu()
        sc = 1.0 if scale is None else torch.as_tensor(scale).detach().double().cpu().reshape(-1)
        if torch.is_tensor(sc):
            if not bool((sc == sc[0]).all()):
                raise ValueError("set_transform: a non-uniform scale is not a similarity")
            sc = float(sc[0])
        c = torch.zeros(3, dtype=torch.float64) if center is None else torch.as_tensor(center).detach().double().cpu().reshape(3)
        o = torch.zeros(3, dtype=torch.float64) if offset is None else torch.as_tensor(offset).detach().double().cpu().reshape(3)
        M = torch.eye(4, dtype=torch.float64)
        M[:3, :3] = sc * R
        M[:3, 3] = o - sc * (R @ c)
        quat, t, s = pose_from_matrix(M)
        quat, t, s = quat.to(dev), t.to(dev), s.to(dev)
    m = {k: getattr(model, a) for k, a in ATTRS.items() if torch.is_tensor(getattr(model, a, None))
         and getattr(model, a).numel() > 0}
    with torch.no_grad():
        out = _apply({k: v.detach() for k, v in m.items()}, quat, t, s, None)
    for k, a in ATTRS.items():
        if k in m:
            getattr(model, a).data = out[k]


_saved = None


def install(cls=None):
    """Rebind `cls.set_transform` (default: the reference's scene.gaussian_model.GaussianModel) to set_transform
    above.  Raises if already installed."""
    global _saved
    if _saved is not None:
        raise RuntimeError("compose.install(): already installed; call uninstall() first")
    if cls is None:
        from scene.gaussian_model import GaussianModel as cls
    _saved = (cls, cls.__dict__.get("set_transform"))

    def _st(self, rotation=None, center=None, scale=None, offset=None, transform=None):
        return set_transform(self, rotation=rotation, center=center, scale=scale, offset=offset, transform=transform)

    cls.set_transform = _st
    return cls


def uninstall():
    """Restore what install() replaced."""
    global _saved
    if _saved is None:
        return
    cls, fn = _saved
    if fn is None:
        delattr(cls, "set_transform")
    else:
        cls.set_transform = fn
    _saved = None

"""fp64 restatement of the per-pixel shading (include/r3dg_b200.h, PIXEL SHADING): the shading step's rendering
equation at every valid pixel of planar material images, with the sampler's N directions around the pixel's unit
normal (area 2 pi), viewdir = campos - point and the point env lookup.  Written from the formulas, independently of
oracle/oracle_shading.py (which it is checked against on rows) and of the kernels."""
import math

import torch

C0, C1 = 0.28209479177387814, 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)
D = torch.float64


def sample_dirs(n, N):
    """n [M,3] unit normals -> [M,N,3]: the Fibonacci samples z_i = max(1 - 2i/(2N-1), sin 10 deg), azimuth
    i pi (3 - sqrt 5), rotated from +z to n (the rotation about (-n.y, n.x, 0); -I when n.z = -1) and normalised."""
    i = torch.arange(N, dtype=D)
    z = (1 - 2 * i / (2 * N - 1)).clamp_min(math.sin(math.radians(10)))
    r = torch.sqrt(1 - z * z)
    th = i * math.pi * (3 - math.sqrt(5))
    s = torch.stack([torch.sin(th) * r, torch.cos(th) * r, z], -1)                # [N,3]
    ax, ay, nz = -n[:, 1], n[:, 0], n[:, 2]
    c = (nz + 1).clamp_min(1e-7)
    R = torch.stack([torch.stack([1 - ay * ay / c, ax * ay / c, ay], -1),
                     torch.stack([ax * ay / c, 1 - ax * ax / c, -ax], -1),
                     torch.stack([-ay, ax, 1 - (ay * ay + ax * ax) / c], -1)], -2)
    R = torch.where((nz + 1 > 0)[:, None, None], R, -torch.eye(3, dtype=D).expand_as(R))
    d = torch.einsum("mij,nj->mni", R, s)
    return d / d.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def sh_basis(d):
    """The 16 real SH of degree <= 3 at d [...,3] in eval_sh's order and signs -> [...,16]."""
    x, y, z = d.unbind(-1)
    xx, yy, zz = x * x, y * y, z * z
    return torch.stack([torch.full_like(x, C0), -C1 * y, C1 * z, -C1 * x,
                        C2[0] * x * y, C2[1] * y * z, C2[2] * (2 * zz - xx - yy), C2[3] * x * z, C2[4] * (xx - yy),
                        C3[0] * y * (3 * xx - yy), C3[1] * x * y * z, C3[2] * y * (4 * zz - xx - yy),
                        C3[3] * z * (2 * zz - 3 * xx - 3 * yy), C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy),
                        C3[6] * x * (xx - 3 * yy)], -1)


def env_lookup(env, d):
    """Bilinear lat-long lookup of env [He,We,3] at d [...,3] (grid_sample align_corners=True, zero padding): column
    u (We-1) with u = (1 - atan2(y, x) / pi) / 2, row v (He-1) with v = (acos(z) - 1e-6) / pi."""
    He, We = env.shape[0], env.shape[1]
    ix = (1 - torch.atan2(d[..., 1], d[..., 0]) / math.pi) / 2 * (We - 1)
    iy = (torch.acos(d[..., 2].clamp(-1, 1)) - 1e-6) / math.pi * (He - 1)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    out = torch.zeros(d.shape[:-1] + (3,), dtype=D)
    for dx in (0, 1):
        for dy in (0, 1):
            xs, ys = x0 + dx, y0 + dy
            w = (1 - (ix - xs).abs()) * (1 - (iy - ys).abs())
            ok = (xs >= 0) & (xs < We) & (ys >= 0) & (ys < He)
            tex = env[ys.clamp(0, He - 1).long(), xs.clamp(0, We - 1).long()]
            out = out + torch.where(ok[..., None], tex * w[..., None], torch.zeros_like(tex))
    return out


def ggx(n, v, l, rough):
    """GGX_specular of neilf.py for rows: n [M,3] raw normals, v [M,3] view directions, l [M,N,3], rough [M,1]."""
    L = l / l.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    V = v / v.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    H = (L + V[:, None]) / 2
    H = H / H.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    Nn = n / n.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    Nn = Nn * torch.sign((V * Nn).sum(-1, keepdim=True))
    NoL = (Nn[:, None] * L).sum(-1, keepdim=True).clamp(1e-6, 1)
    NoV = (Nn * V).sum(-1, keepdim=True).clamp(1e-6, 1)[:, None]
    NoH = (Nn[:, None] * H).sum(-1, keepdim=True).clamp(1e-6, 1)
    VoH = (V[:, None] * H).sum(-1, keepdim=True).clamp(1e-6, 1)
    a2 = (rough * rough) ** 2
    k = ((rough * rough + 2 * rough + 1) / 8)[:, None]
    frac = (0.04 + 0.96 * torch.pow(2.0, (-5.55473 * VoH - 6.98316) * VoH)) * a2[:, None]
    nom = (4 * math.pi * (NoH * NoH * (a2[:, None] - 1) + 1) ** 2 * (NoV * (1 - k) + k) * (NoL * (1 - k) + k)).clamp(1e-6, 4 * math.pi)
    return frac / nom


def shade_pixels(base_color, roughness, normal, points, campos, T, env, transform=None, incidents=None, mask=None):
    """One view of planar images ([3,H,W], [1,H,W], [3,H,W], [3,H,W], campos [3], T [N,H,W], incidents [48,H,W] or
    None, mask [H,W] or None; env [He,We,3] activated, transform [3,3] or None), everything promoted to fp64.
    Returns dict(pbr, diffuse_light, specular [3,H,W], visibility [1,H,W]), masked pixels 0."""
    H, W = base_color.shape[-2:]
    N = T.shape[0]
    rows = lambda t: t.to(D).reshape(t.shape[0], H * W).T                        # [HW,C]
    b, r, n, p, vis = rows(base_color), rows(roughness), rows(normal), rows(points), rows(T)
    v = campos.to(D)[None] - p
    nh = n / n.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    d = sample_dirs(nh, N)                                                         # [HW,N,3]
    de = d if transform is None else d @ transform.to(D).T
    glob = env_lookup(env.to(D), de) * vis[..., None]
    loc = torch.zeros_like(glob)
    if incidents is not None:
        inc = rows(incidents).reshape(-1, 16, 3)
        loc = torch.einsum("mnk,mkc->mnc", sh_basis(d), inc).clamp_min(0)
    ndi = (n[:, None] * d).sum(-1, keepdim=True).clamp_min(0)
    transport = (loc + glob) * (2 * math.pi) * ndi
    fs = ggx(n, v, d, r)
    out = {"pbr": ((b[:, None] / math.pi + fs) * transport).mean(1), "diffuse_light": transport.mean(1),
           "specular": (fs * transport).mean(1), "visibility": vis.mean(1, keepdim=True)}
    keep = torch.ones(H * W, dtype=torch.bool) if mask is None else mask.reshape(-1).bool()
    return {k: torch.where(keep[:, None], x, torch.zeros_like(x)).T.reshape(-1, H, W) for k, x in out.items()}

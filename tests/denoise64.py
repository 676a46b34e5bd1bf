"""fp64 restatement of the DENOISE block of include/r3dg_b200.h: the a-trous filter by pad, shift and sum (with autograd
to x), and its transpose written separately from the header's backward formula.  Runs on the device of its inputs."""
import torch

D = torch.float64
H5 = (1 / 16, 4 / 16, 6 / 16, 4 / 16, 1 / 16)


def tap(t, dy, dx):
    """out[..., y, x] = t[..., y + dy, x + dx], zero outside the image"""
    H, W = t.shape[-2], t.shape[-1]
    out = torch.zeros_like(t)
    ys, yd = slice(max(dy, 0), H + min(dy, 0)), slice(max(-dy, 0), H + min(-dy, 0))
    xs, xd = slice(max(dx, 0), W + min(dx, 0)), slice(max(-dx, 0), W + min(-dx, 0))
    if ys.start < ys.stop and xs.start < xs.stop:
        out[..., yd, xd] = t[..., ys, xs]
    return out


def guides(normal, points, mask=None, features=None):
    """[V,..,H,W] fp64 guides: unit normal (F.normalize), points, validity (1 / 0) and features (None for F = 0)"""
    n = normal.to(D)
    nh = n / n.norm(dim=1, keepdim=True).clamp_min(1e-12)
    valid = torch.ones_like(n[:, 0]) if mask is None else (mask != 0).to(D)
    f = None if features is None or features.shape[1] == 0 else features.to(D)
    return nh, points.to(D), valid, f


def weights(g, step, sigma_normal, sigma_plane, sigma_features):
    """{(oy, ox): w(p, p + step o) [V,H,W]} of one pass, with the taps outside the image or on invalid pixels at 0"""
    nh, x, valid, f = g
    out = {}
    for oy in range(-2, 3):
        for ox in range(-2, 3):
            dy, dx = oy * step, ox * step
            inside = tap(torch.ones_like(valid), dy, dx) * tap(valid, dy, dx)
            if oy == 0 and ox == 0:
                out[(oy, ox)] = H5[2] * H5[2] * valid
                continue
            wn = (nh * tap(nh, dy, dx)).sum(1).clamp(0, 1) ** sigma_normal
            d = tap(x, dy, dx) - x
            dn = d.norm(dim=1)
            t = torch.where(dn > 0, (nh * d).sum(1).abs() / torch.where(dn > 0, dn, torch.ones_like(dn)), torch.zeros_like(dn))
            w = H5[oy + 2] * H5[ox + 2] * wn * torch.exp(-t / sigma_plane)
            if f is not None:
                w = w * torch.exp(-((tap(f, dy, dx) - f) ** 2).sum(1) / sigma_features ** 2)
            out[(oy, ox)] = w * inside * valid
    return out


def atrous(x, normal, points, mask=None, features=None, passes=4, sigma_normal=128.0, sigma_plane=0.1,
           sigma_features=0.1):
    """y [V,C,H,W] (fp64, differentiable in x) of x [V,C,H,W]; per pass y_{k+1} = sum_o w y_k(p + s o) / W"""
    g = guides(normal, points, mask, features)
    valid = g[2][:, None]
    y = torch.where(valid > 0, x.to(D), torch.zeros((), dtype=D, device=x.device))
    for k in range(passes):
        w = weights(g, 2 ** k, sigma_normal, sigma_plane, sigma_features)
        acc = sum(wo[:, None] * tap(y, oy * 2 ** k, ox * 2 ** k) for (oy, ox), wo in w.items())
        W = sum(w.values())[:, None]
        y = torch.where(valid > 0, acc / torch.where(valid > 0, W, torch.ones_like(W)), torch.zeros_like(acc))
    return y


def transpose(g_out, normal, points, mask=None, features=None, passes=4, sigma_normal=128.0, sigma_plane=0.1,
              sigma_features=0.1):
    """A^T g by the header's backward: g^ = g_{k+1} / W_k, g_k(q) = sum_o w(q - s o, q) g^(q - s o)"""
    g = guides(normal, points, mask, features)
    valid = g[2][:, None]
    gk = torch.where(valid > 0, g_out.to(D), torch.zeros((), dtype=D, device=g_out.device))
    for k in reversed(range(passes)):
        s = 2 ** k
        w = weights(g, s, sigma_normal, sigma_plane, sigma_features)
        W = sum(w.values())[:, None]
        gh = torch.where(valid > 0, gk / torch.where(valid > 0, W, torch.ones_like(W)), torch.zeros_like(gk))
        gk = sum(tap(wo[:, None] * gh, -oy * s, -ox * s) for (oy, ox), wo in w.items()) * valid
    return gk


def gbuffer(V, H, W, F=0, seed=0, masked=True, device="cpu"):
    """Guides of V views with a 90 degree crease (x > 0.6: the plane x = 0.6, normal +x) and a depth step (y < 0.3: the
    ground 0.5 closer, normal +z), small seeded normal and point noise, normals of random length, smooth features with
    noise and (masked) a random 15 % of pixels plus a block invalid.  fp32 tensors: normal, points [V,3,H,W], mask
    [V,H,W] bool or None, features [V,F,H,W] or None."""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid((torch.arange(H) + 0.5) / H, (torch.arange(W) + 0.5) / W, indexing="ij")
    crease, step = (xs > 0.6), (ys < 0.3)
    pts = torch.stack([xs.clone(), ys.clone(), torch.zeros_like(xs)])
    pts[2] = torch.where(step, 0.5, 0.0)
    pts[0] = torch.where(crease, 0.6, pts[0])
    pts[2] = torch.where(crease, xs - 0.6, pts[2])
    nrm = torch.stack([crease.double(), torch.zeros_like(xs).double(), (~crease).double()]).float()
    normal = (nrm[None] + 0.04 * torch.randn(V, 3, H, W, generator=g)) * (0.5 + torch.rand(V, 1, H, W, generator=g))
    points = pts[None] + (0.1 / max(H, W)) * torch.randn(V, 3, H, W, generator=g)
    mask = None
    if masked:
        mask = torch.rand(V, H, W, generator=g) > 0.15
        mask[:, H // 3:H // 3 + max(H // 5, 1), W // 4:W // 4 + max(W // 6, 1)] = False
    feats = None
    if F:
        feats = 0.2 * torch.sin(3 * xs + 2 * ys)[None, None] + 0.05 * torch.randn(V, F, H, W, generator=g)
    to = lambda t: None if t is None else t.to(device)
    return to(normal), to(points), to(mask), to(feats)

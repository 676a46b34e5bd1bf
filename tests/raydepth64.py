"""fp64 truth of the ray-depth mode (csrc/projection.cu, composite.cu, composite_bwd.cu, projection_bwd.cu).

Under the projection's local affine (EWA) approximation a Gaussian with mean m and covariance Sigma maps the screen
position u and the camera z jointly to a Gaussian: u = mean2D + T (x - m), z = tz + w_z . (x - m), T = J W the
projection's 2x3 Jacobian (proj64.cov2d: the reference's J with its frustum clamp), w_z the view matrix's camera-z
column.  With the screen filter's 0.3 px^2 on u only,

    Cov(u) = T Sigma T^T + 0.3 I,   c = Cov(u, z) = T Sigma w_z,   p = Cov(u)^-1 c = conic c,

and the depth at which the filtered Gaussian peaks along the pixel's line {u = pixel} is the conditional mean
d(pixel) = tz + p . (pixel - mean2D).  plane() is that closed form (conic with proj64's linearised inverse, so that its
derivative follows the kernel's chain), brute_peak() maximises the joint density along the line numerically, and
perspective_peak() is the exact peak of the 3D Gaussian along the true (perspective) ray, the limit the affine plane
approaches as the Gaussian shrinks relative to its depth.  record() is proj64.record with the plane appended, and
composite() an fp64 front-to-back compositor of the depth image on given per-pixel lists."""
import torch

import aa_oracle
import proj64


def _T(m, cam):
    """(T [2,3], tz) of the projection at mean m: the reference's J (frustum clamp as proj64) times W."""
    t = m @ cam.V[:3, :3] + cam.V[3, :3]
    tx, ty, tz = t[0], t[1], t[2]
    hx, hy = cam.W / (2.0 * cam.tanfovx), cam.H / (2.0 * cam.tanfovy)
    t0x = proj64._clamp_t(tx, tz, 1.3 * cam.tanfovx)
    t0y = proj64._clamp_t(ty, tz, 1.3 * cam.tanfovy)
    zero = torch.zeros_like(tz)
    J = torch.stack([hx / tz, zero, -hx * t0x / (tz * tz), zero, hy / tz, -hy * t0y / (tz * tz)]).view(2, 3)
    return J @ cam.V[:3, :3].T, tz


def plane(m, sigma, cam, dilation=aa_oracle.DILATION, linearised=True):
    """The depth plane p [2] of one Gaussian (m [3], sigma [3,3]) in camera `cam` (proj64.Camera)."""
    T, _ = _T(m, cam)
    wz = cam.V[:3, 2]
    C = T @ sigma @ T.T
    a, b, c = C[0, 0] + dilation, C[0, 1], C[1, 1] + dilation
    det = a * c - b * b
    if linearised:
        conic = torch.stack([proj64._lin_div(c, det), proj64._lin_div(-b, det), proj64._lin_div(a, det)])
    else:
        conic = torch.stack([c / det, -b / det, a / det])
    cv = T @ (sigma @ wz)
    return torch.stack([conic[0] * cv[0] + conic[1] * cv[1], conic[1] * cv[0] + conic[2] * cv[1]])


def joint(m, sigma, cam, dilation=aa_oracle.DILATION):
    """(K [3,3], tz): the affine frame's joint covariance of (u.x, u.y, z) and the mean's camera z."""
    T, tz = _T(m, cam)
    wz = cam.V[:3, 2]
    A = torch.cat([T, wz[None]], 0)
    K = A @ sigma @ A.T
    K = K + torch.diag(torch.tensor([dilation, dilation, 0.0], dtype=K.dtype))
    return K, tz


def brute_peak(m, sigma, cam, offset, n=20001, span=6.0):
    """argmax over z of the joint density at u = mean2D + offset, by a grid over tz +- span sd(z) and a parabola
    through the best grid point and its neighbours."""
    K, tz = joint(m, sigma, cam)
    Ki = torch.linalg.inv(K)
    sd = torch.sqrt(K[2, 2])
    z = tz + torch.linspace(-span, span, n, dtype=K.dtype) * sd
    v = torch.stack([torch.full_like(z, float(offset[0])), torch.full_like(z, float(offset[1])), z - tz], -1)
    q = ((v @ Ki) * v).sum(-1)                     # -2 log density + const
    i = int(torch.argmin(q[1:-1])) + 1
    h = z[1] - z[0]
    den = q[i - 1] - 2 * q[i] + q[i + 1]
    return z[i] + 0.5 * h * (q[i - 1] - q[i + 1]) / den


def perspective_peak(mc, sigma_c, ray):
    """Camera z of the maximum of the 3D Gaussian (camera-frame mean mc, covariance sigma_c) along the ray s * ray
    (ray.z = 1): s = (r^T S^-1 m) / (r^T S^-1 r)."""
    Si = torch.linalg.inv(sigma_c)
    return (ray @ Si @ mc) / (ray @ Si @ ray) * ray[2]


def record(leaves, const, cam, D, aa=False, f3d=False):
    """proj64.record of one Gaussian with its depth plane appended: ([12], terms)."""
    rec, terms = proj64.record(leaves, const, cam, D, aa=aa, f3d=f3d)
    m = leaves["means3D"]
    if "cov3D" in leaves:
        sigma = aa_oracle.cov3d_from_six(leaves["cov3D"][None])[0]
    else:
        s = leaves["scales"]
        if f3d:
            import filter3d_oracle
            s = filter3d_oracle.dilate(s[None], leaves["opacities"].reshape(1), const["filter_3d"].reshape(1))[0][0]
        sigma = aa_oracle.cov3d_of(proj64._modified(s, cam.mod)[None], leaves["rotations"][None])[0]
    return torch.cat([rec, plane(m, sigma, cam)]), terms


def composite_depth(mean2D, conic, opacity, tz, p, order, n_contrib, W, H, ray_depth=True):
    """fp64 depth image [H,W] of the Gaussians listed per pixel: order[pix] the depth-sorted ids of the pixel's tile
    (a list of LongTensors), n_contrib[pix] the kernel's count of list entries walked.  Each entry adds
    alpha T d with d the plane depth (ray_depth) or tz; alpha, the skip and stop tests are the forward's."""
    out = torch.zeros(H * W, dtype=torch.float64)
    for pix in range(H * W):
        ids = order[pix][:int(n_contrib[pix])]
        if ids.numel() == 0:
            continue
        x, y = float(pix % W), float(pix // W)
        dx, dy = mean2D[ids, 0] - x, mean2D[ids, 1] - y
        power = -0.5 * (conic[ids, 0] * dx * dx + conic[ids, 2] * dy * dy) - conic[ids, 1] * dx * dy
        alpha = torch.clamp(opacity[ids] * torch.exp(power), max=0.99)
        d = tz[ids] - p[ids, 0] * dx - p[ids, 1] * dy if ray_depth else tz[ids]
        T, acc = 1.0, 0.0
        for k in range(ids.numel()):
            if power[k] > 0 or alpha[k] < 1.0 / 255.0:
                continue
            if T * (1 - alpha[k]) < 1e-4:
                break
            acc += float(alpha[k] * T * d[k])
            T *= float(1 - alpha[k])
        out[pix] = acc
    return out.view(H, W)

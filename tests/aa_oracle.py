"""fp64 closed form of the antialiased mode's opacity factor (csrc/projection.cu, projection_bwd.cu) for the tests.

With a0, b, c0 the 2D covariance of a Gaussian before the fixed 0.3 px^2 dilation, a1 = a0 + 0.3, c1 = c0 + 0.3,
det0 = a0 c0 - b^2 and det1 = a1 c1 - b^2, the mode multiplies the opacity by rho = sqrt(max(r, 2.5e-5)) with
r = det0 / det1, and r = 0 where det0 <= 0.  rho() is a differentiable torch function of means3D, the view matrix and
scales / rotations or cov3D_precomp, following the projection's closed form: t = [m,1] viewmatrix, x/z and y/z clamped
to 1.3 tan(fov), J the perspective Jacobian at the clamped point, T = J W, cov2D = T Sigma T^T."""
import torch

DILATION = 0.3
FLOOR = 2.5e-5


def cov3d_of(scales, rotations, scale_modifier=1.0):
    """Sigma = R diag(s)^2 R^T of the projection (the quaternion (r, x, y, z) is used as given, not normalised)."""
    r, x, y, z = rotations.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).view(-1, 3, 3)
    s = scales * scale_modifier
    return R @ torch.diag_embed(s * s) @ R.transpose(1, 2)


def cov3d_from_six(c6):
    """[P,6] (xx, xy, xz, yy, yz, zz) -> [P,3,3]."""
    xx, xy, xz, yy, yz, zz = c6.unbind(-1)
    return torch.stack([xx, xy, xz, xy, yy, yz, xz, yz, zz], -1).view(-1, 3, 3)


def cov2d(means3D, sigma, viewmatrix, W, H, tanfovx, tanfovy):
    """(a0, b, c0) of every Gaussian: the 2D covariance before the dilation.  viewmatrix is [4,4] in torch's
    world_view_transform layout (t = [m,1] viewmatrix)."""
    t = means3D @ viewmatrix[:3, :3] + viewmatrix[3, :3]
    tx, ty, tz = t.unbind(-1)
    limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
    cx, cy = (tx / tz).clamp(-limx, limx), (ty / tz).clamp(-limy, limy)
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz, zero, -fx * cx / tz, zero, fy / tz, -fy * cy / tz], -1).view(-1, 2, 3)
    T = J @ viewmatrix[:3, :3].T
    C = T @ sigma @ T.transpose(1, 2)
    return C[:, 0, 0], C[:, 0, 1], C[:, 1, 1]


def ratio(a0, b, c0):
    """r = det0 / det1, 0 where det0 <= 0."""
    det0 = a0 * c0 - b * b
    det1 = (a0 + DILATION) * (c0 + DILATION) - b * b
    return torch.where(det0 > 0, det0 / det1, torch.zeros_like(det0))


def ratio_grad(a0, b, c0):
    """(dr/da, dr/db, dr/dc) in the cancellation-free forms the projection backward uses (valid where det0 > 0)."""
    h = DILATION
    a1, c1 = a0 + h, c0 + h
    det1 = a1 * c1 - b * b
    return h * (c0 * c1 + b * b) / det1 ** 2, -2 * b * (h * (a0 + c0) + h * h) / det1 ** 2, h * (a0 * a1 + b * b) / det1 ** 2


def rho_of_cov2d(a0, b, c0):
    return ratio(a0, b, c0).clamp_min(FLOOR).sqrt()


def rho(means3D, viewmatrix, W, H, tanfovx, tanfovy, scales=None, rotations=None, cov3D=None, scale_modifier=1.0):
    """rho of every Gaussian (fp64 when the inputs are), differentiable in every tensor argument."""
    sigma = cov3d_from_six(cov3D) if cov3D is not None else cov3d_of(scales, rotations, scale_modifier)
    return rho_of_cov2d(*cov2d(means3D, sigma, viewmatrix, W, H, tanfovx, tanfovy))

"""fp64 truth of the similarity transform of Gaussian models (relightable3dgaussian_b200/compose.py, csrc/compose.cu).

The SH rotation D^l(R) is built independently of the kernel's table: a least-squares fit over N_DIRS random directions,
D^l = pinv(Y_l(U)) Y_l(R^T U), which satisfies  sum_m Y_lm(d) c'_m = sum_m Y_lm(R^T d) c_m  for every d because band l
of the basis is closed under rotation.  Everything is torch float64 on the inputs' device, differentiable end to end.
"""
import torch

N_DIRS = 256
C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)
C4 = (2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892, 0.10578554691520431,
      -0.6690465435572892, 0.47308734787878004, -1.7701307697799304, 0.6258357354491761)


def sh_basis(d):
    """Y_k(d) for k < 25, d [...,3] -> [...,25]: the reference's eval_sh basis through degree 4."""
    x, y, z = d.unbind(-1)
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    return torch.stack([
        torch.full_like(x, C0),
        -C1 * y, C1 * z, -C1 * x,
        C2[0] * xy, C2[1] * yz, C2[2] * (2 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy),
        C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy),
        C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy),
        C4[0] * xy * (xx - yy), C4[1] * yz * (3 * xx - yy), C4[2] * xy * (7 * zz - 1), C4[3] * yz * (7 * zz - 3),
        C4[4] * (zz * (35 * zz - 30) + 3), C4[5] * xz * (7 * zz - 3), C4[6] * (xx - yy) * (7 * zz - 1),
        C4[7] * xz * (xx - 3 * yy), C4[8] * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))], -1)


def eval_sh(deg, sh, d):
    """The reference's eval_sh: sh [...,C,(deg+1)^2] at unit d [...,3] -> [...,C]."""
    n = (deg + 1) ** 2
    return (sh[..., :n] * sh_basis(d)[..., None, :n]).sum(-1)


def _dirs(device):
    g = torch.Generator().manual_seed(12345)
    u = torch.randn(N_DIRS, 3, generator=g, dtype=torch.float64)
    return (u / u.norm(dim=-1, keepdim=True)).to(device)


def sh_rotation(R, l):
    """D^l(R) [...,2l+1,2l+1] for rotations R [...,3,3] (fp64, least squares over N_DIRS directions)."""
    U = _dirs(R.device)
    sl = slice(l * l, (l + 1) ** 2)
    A = sh_basis(U)[:, sl]                                     # [N,2l+1]
    B = sh_basis(torch.einsum("...ba,nb->...na", R, U))[..., sl]   # Y_l(R^T u_n)
    return torch.linalg.pinv(A) @ B


def build_rotation(q):
    q = q / q.norm(dim=-1, keepdim=True)
    r, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(q.shape[:-1] + (3, 3))


def quat_mul(q1, q2):
    """The reference's quaternion_multiply (Hamilton product, (w,x,y,z))."""
    w1, x1, y1, z1 = q1.unbind(-1)
    w2, x2, y2, z2 = q2.unbind(-1)
    return torch.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                        w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1)


def rotate_sh(sh, R):
    """sh [P,(L+1)^2-1,C] rotated band by band by D^l(R) (R [3,3] or [P,3,3])."""
    L = int(round((sh.shape[1] + 1) ** 0.5)) - 1
    out = []
    for l in range(1, L + 1):
        D = sh_rotation(R, l)
        c = sh[:, l * l - 1:(l + 1) ** 2 - 1]
        out.append(torch.matmul(D, c) if D.dim() == 3 else torch.einsum("ij,pjc->pic", D, c))
    return torch.cat(out, 1) if out else sh.clone()


def transform(xyz, normal, rotation, scaling, shs, quat, t, s, offsets):
    """The similarity transform in fp64: object k = rows offsets[k]:offsets[k+1] of every tensor."""
    outs = [[] for _ in range(4 + len(shs))]
    for k in range(quat.shape[0]):
        a, b = offsets[k], offsets[k + 1]
        qn = quat[k] / quat[k].norm()
        R = build_rotation(qn)
        outs[0].append(s[k] * xyz[a:b] @ R.T + t[k])
        outs[1].append(normal[a:b] @ R.T)
        outs[2].append(quat_mul(qn.expand(b - a, 4), rotation[a:b]))
        outs[3].append(scaling[a:b] + torch.log(s[k]))
        for i, sh in enumerate(shs):
            outs[4 + i].append(rotate_sh(sh[a:b], R))
    return [torch.cat(o) for o in outs]

"""Drop-in replacement for the reference's pybind module `bvh_tracing._C`
(bvh/src/bindings.cpp:8-13): `create_bvh`, `trace_bvh_opacity`, `trace_bvh`, same positional
arguments and return tuples as bvh/src/bvh.cu:8-27 / :88-116 / :29-86, on top of the C ABI of
libr3dg_b200.so (include/r3dg_b200.h)."""
import torch

from . import _lib


def create_bvh(means3D, scales, rotations, nodes, aabbs):
    """== create_bvh (bvh/src/bvh.cu:8-27).  `nodes` i32[2P-1,5] / `aabbs` f32[2P-1,6] are pre-filled
    by the caller (bvh/__init__.py:32-57) and completed IN PLACE; returns (nodes, aabbs, morton i64[P]).
    means3D / scales / rotations are unused by the reference's construct_bvh too."""
    P = means3D.size(0)
    assert nodes.is_cuda and nodes.dtype == torch.int32 and nodes.is_contiguous() and nodes.shape == (2 * P - 1, 5)
    assert aabbs.is_cuda and aabbs.dtype == torch.float32 and aabbs.is_contiguous() and aabbs.shape == (2 * P - 1, 6)
    morton = torch.zeros((P,), dtype=torch.int64, device=means3D.device)
    tmp = _lib.scratch(_lib.load().r3dg_bvh_build_tmp_bytes(P), means3D.device)
    _lib.call("r3dg_bvh_build", means3D.device, P, nodes.data_ptr(), aabbs.data_ptr(), morton.data_ptr(), tmp.data_ptr(),
              tmp.numel(), what="create_bvh")
    return nodes, aabbs, morton


def _trace(nodes, aabbs, rays_o, rays_per_origin, origin_offset, rays_d, means3D, covs3D, opacities, normals):
    P = means3D.size(0)
    dev = rays_d.device
    out_shape = rays_d.shape[:-1]
    num_rays = rays_d.numel() // 3
    num_contributes = torch.empty(out_shape, dtype=torch.int32, device=dev)
    rendered_opacity = torch.empty(out_shape, dtype=torch.float32, device=dev)
    if num_rays == 0:
        return num_contributes, rendered_opacity
    nodes = nodes.to(torch.int32).contiguous()
    aabbs, rays_o, rays_d = _lib.f32(aabbs), _lib.f32(rays_o), _lib.f32(rays_d)
    means3D, covs3D, opacities, normals = _lib.f32(means3D), _lib.f32(covs3D), _lib.f32(opacities), _lib.f32(normals)
    tmp = _lib.scratch(_lib.load().r3dg_bvh_trace_tmp_bytes(P), dev)
    _lib.call("r3dg_bvh_trace_opacity", dev, P, num_rays, nodes.data_ptr(), aabbs.data_ptr(), rays_o.data_ptr(),
              int(rays_per_origin), float(origin_offset), rays_d.data_ptr(), means3D.data_ptr(), covs3D.data_ptr(),
              opacities.data_ptr(), normals.data_ptr(), num_contributes.data_ptr(), rendered_opacity.data_ptr(),
              tmp.data_ptr(), tmp.numel(), what="trace_bvh_opacity")
    return num_contributes, rendered_opacity


def trace_bvh_opacity(nodes, aabbs, rays_o, rays_d, means3D, covs3D, opacities, normals):
    """== trace_bvh_opacity (bvh/src/bvh.cu:88-116): returns (num_contributes i32[...],
    rendered_opacity f32[...]) shaped like rays_o.shape[:-1]."""
    return _trace(nodes, aabbs, rays_o, 1, 0.0, rays_d, means3D, covs3D, opacities, normals)


def trace_bvh(nodes, aabbs, rays_o, rays_d, means3D, covs3D, opacities):
    """`trace_bvh` (bvh/src/bvh.cu:29-86, trace.cu:8-192) has no Python caller anywhere in the
    reference (SURVEY.md §2.3 K23) and is out of the hot-path scope."""
    raise NotImplementedError("bvh_tracing._C.trace_bvh is unused by the reference and not provided")

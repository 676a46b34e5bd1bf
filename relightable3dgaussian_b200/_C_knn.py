"""Drop-in replacement for `simple_knn._C` (submodules/simple-knn/ext.cpp:15-17): `distCUDA2`."""
import torch

from . import _lib


def distCUDA2(points):
    """== distCUDA2 (spatial.cu:15-26): f32[P] mean squared distance to the 3 nearest neighbours."""
    P = points.size(0)
    pts = _lib.f32(points)
    out = torch.full((P,), 0.0, dtype=torch.float32, device=points.device)
    if P > 0:
        tmp = _lib.scratch(_lib.load().r3dg_knn_tmp_bytes(P), points.device)
        _lib.call("r3dg_knn_dist2", points.device, P, pts.data_ptr(), out.data_ptr(), tmp.data_ptr(), tmp.numel(),
                  what="distCUDA2")
    return out

"""Multi-GPU view parallelism (SURVEY.md §8e): the model is replicated, rank r renders view r of
the step's batch, and ONE all-reduce over a flat per-Gaussian gradient buffer follows backward.

The reference has no multi-GPU code (single process, `cuda:0` pinned, utils/general_utils.py:167;
one view per iteration, train.py:115-127), so an N-view step is defined here as the mean of N
single-view losses: grad = (1/N) * sum_r grad_r.  The path shards over independent views with no
data-path collective other than this gradient sum.

`GradBucket` is pure torch (works on CPU tensors with the gloo backend — that is how the host
logic is tested without a GPU); on the GPU box it is backed by NCCL over NVLink and the backward
kernels write directly into its views (`_C_raster.rasterize_gaussians_backward(_out=...)`), so
no packing copy precedes the collective.
"""
import ctypes
from collections import OrderedDict

import torch
import torch.distributed as dist

from . import _lib

# per-Gaussian parameter gradients that are summed across views (means2D / colors / cov3D are
# per-view by-products: means2D feeds per-view densification statistics, SURVEY.md §8e)
REDUCED = ("means3D", "features", "sh", "opacity", "scales", "rotations")


class GradBucket:
    def __init__(self, P, S, M, device, names=REDUCED):
        shapes = OrderedDict(means3D=(P, 3), features=(P, S), sh=(P, M, 3), opacity=(P, 1),
                             scales=(P, 3), rotations=(P, 4))
        self.names = tuple(n for n in names if n in shapes)
        self.shapes = OrderedDict((n, shapes[n]) for n in self.names)
        sizes = [int(torch.Size(s).numel()) for s in self.shapes.values()]
        # 128-float (512 B) aligned sections so every view starts on a cache-line boundary
        self.offsets, off = [], 0
        for n in sizes:
            self.offsets.append(off)
            off += (n + 127) // 128 * 128
        self.flat = torch.zeros(max(off, 1), dtype=torch.float32, device=device)
        self.views = OrderedDict()
        for (name, shape), o, n in zip(self.shapes.items(), self.offsets, sizes):
            self.views[name] = self.flat[o:o + n].view(shape)

    def bytes(self):
        return self.flat.numel() * 4

    def allreduce_mean(self, group=None, async_op=False):
        """One collective for the whole step.  Returns the work handle when async_op."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return None
        world = dist.get_world_size(group)
        if dist.get_backend(group) == "nccl":          # averaging is fused into the collective (no 2 x 256 MB pre-scale pass)
            return dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=group, async_op=async_op)
        self.flat.mul_(1.0 / world)                    # gloo (CPU tests) has no AVG
        return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)


class FactoredGradExchange:
    """The exchange step with the SH gradient factorised (csrc/sh_exchange.cu).

    For one view dL_dsh[g,k,:] = basis_k(dir(g, campos)) * f[g,:]: 192 of the 248 gradient bytes of a
    Gaussian are an outer product of 16 numbers every rank can recompute with 3 numbers only the
    rendering rank has.  So per step: ONE all-reduce (mean) of the small dense rest (means3D,
    features, opacity, scales, rotations: 64 B per Gaussian at S=5), ONE all-gather of the factors
    (12 B per Gaussian and view) and a local kernel that rebuilds mean_v(dL_dsh) — identical on all
    ranks (fixed summation order), equal to the dense all-reduce up to fp32 summation order.

    Two ways to use it.  Operator level (the caller owns the per-Gaussian tensors as leaves, e.g.
    bench.py's resident path): `rasterize_gaussians_backward(..., _out=ex.views)`, then
    `ex.exchange(means3D, campos_of_all_ranks, degree)`; gradients are `ex.grads[name]`.  Autograd
    level (`rasterizer.set_grad_exchange`): only the SH factor goes through this object — the dense
    rest is averaged at the leaf parameters (`LeafGradBucket`), because the maps from the leaves to
    `features` / `means3D` are view dependent in the reference's render functions.
    `gather_factors()` is pure torch.distributed (runs under gloo in the CPU tests); the rebuild is
    the CUDA kernel (no CPU path)."""

    def __init__(self, P, S, M, device, world=None):
        self.P, self.S, self.M = P, S, M
        self.world = world if world is not None else (dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1)
        self.dense = GradBucket(P, S, M, device, names=tuple(n for n in REDUCED if n != "sh"))
        self.factor = torch.zeros((P, 3), dtype=torch.float32, device=device)
        self.gathered = torch.zeros((self.world, P, 3), dtype=torch.float32, device=device) if self.world > 1 else self.factor.view(1, P, 3)
        self.sh = torch.zeros((P, M, 3), dtype=torch.float32, device=device)
        self.views = OrderedDict(self.dense.views)
        self.views["sh_factor"] = self.factor
        self.grads = OrderedDict(self.dense.views)
        self.grads["sh"] = self.sh

    def bytes(self):
        """Bytes a rank contributes to the collectives of one step (dense all-reduce + its factor)."""
        return self.dense.bytes() + self.factor.numel() * 4

    def gather_factors(self, group=None):
        if self.world > 1:
            # output viewed as the dim-0 concatenation [world*P, 3] (the layout gloo insists on; NCCL accepts both)
            gather = getattr(dist, "all_gather_into_tensor", None) or dist._all_gather_base      # torch 1.12 (readme.md:26) has only the latter
            gather(self.gathered.view(self.world * self.P, 3), self.factor, group=group)
        return self.gathered

    def rebuild_sh(self, means3D, campos_all, degree):
        """dL_dsh = (1/world) * sum_v basis(dir(means3D, campos_all[v])) x gathered[v]  (CUDA kernel)."""
        assert campos_all.shape == (self.world, 3) and campos_all.is_contiguous() and campos_all.dtype == torch.float32
        assert means3D.is_contiguous() and means3D.dtype == torch.float32 and means3D.shape == (self.P, 3)
        if not means3D.is_cuda:
            raise RuntimeError("FactoredGradExchange.rebuild_sh runs on the GPU only (no CPU path)")
        _lib.call("r3dg_sh_grad_from_factors", means3D.device, self.P, int(degree), self.M, self.world, means3D.data_ptr(),
                  campos_all.data_ptr(), self.gathered.data_ptr(), 1.0 / self.world, self.sh.data_ptr(), what="sh_grad_from_factors")
        return self.sh

    def exchange(self, means3D, campos_all, degree, group=None):
        self.dense.allreduce_mean(group=group)
        self.gather_factors(group=group)
        return self.rebuild_sh(means3D, campos_all, degree)


class P2PGradExchange:
    """The exchange step as ONE kernel over NVLink peer memory — no NCCL collective on the data path
    (csrc/sh_exchange.cu: r3dg_exchange_p2p).  The per-view SH-gradient factors [P,3] and the dense per-Gaussian
    gradient section (means3D, features, opacity, scales, rotations) live in ONE symmetric buffer that
    `torch.distributed._symmetric_memory` maps into every rank (allocation / rendezvous / barriers only — the
    arithmetic and the transfers are ours).  Per step, after this rank's backward wrote into `views`:

        barrier -> [ one launch: rebuild mean_v(dL_dsh_v) with view v's factors loaded straight from rank v's
                     buffer (P2P loads overlapping the outer-product math)  +  in-switch NVLS all-reduce
                     (multimem.ld_reduce / multimem.st) of the dense section, slice r by rank r ] -> barrier

    Same interface as FactoredGradExchange (`views`, `grads`, `exchange()`); equal results up to fp32 summation
    order.  Raises at construction when symmetric memory cannot be set up (callers fall back to the NCCL classes)."""

    def __init__(self, P, S, M, device, group=None):
        import torch.distributed._symmetric_memory as symm_mem
        self.P, self.S, self.M = P, S, M
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        shapes = OrderedDict(means3D=(P, 3), features=(P, S), opacity=(P, 1), scales=(P, 3), rotations=(P, 4), sh_factor=(P, 3))
        sizes = [int(torch.Size(s).numel()) for s in shapes.values()]
        offs, off = [], 0
        for n in sizes:
            offs.append(off)
            off += (n + 127) // 128 * 128
        self.n_dense = offs[-1]                                   # the factor section comes last: everything before it is averaged
        self.flat = symm_mem.empty(max(off, 128), dtype=torch.float32, device=device)
        self.flat.zero_()
        self.hdl = symm_mem.rendezvous(self.flat, self.group)
        self.views = OrderedDict((name, self.flat[o:o + n].view(shape)) for (name, shape), o, n in zip(shapes.items(), offs, sizes))
        self.factor = self.views["sh_factor"]
        self.factor_off = offs[-1]
        self.sh = torch.zeros((P, M, 3), dtype=torch.float32, device=device)
        self.grads = OrderedDict((k, v) for k, v in self.views.items() if k != "sh_factor")
        self.grads["sh"] = self.sh
        self.multicast = int(self.hdl.multicast_ptr) if getattr(self.hdl, "multicast_ptr", 0) else 0
        self.peer_ptrs = [int(x) for x in self.hdl.buffer_ptrs]

    def bytes(self):
        """Bytes of this rank's buffer that other ranks read in one step."""
        return (self.n_dense + self.P * 3) * 4

    def exchange(self, means3D, campos_all, degree, dense=True):
        assert campos_all.shape == (self.world, 3) and campos_all.is_contiguous() and campos_all.dtype == torch.float32
        assert means3D.is_contiguous() and means3D.dtype == torch.float32 and means3D.shape == (self.P, 3)
        a = _exchange_args(self.world, self.rank, self.peer_ptrs, self.n_dense if dense else 0, self.multicast)
        a.P, a.D, a.M = self.P, int(degree), self.M
        a.means3D, a.campos, a.dL_dsh = means3D.data_ptr(), campos_all.data_ptr(), self.sh.data_ptr()
        for v in range(self.world):
            a.factors[v] = self.peer_ptrs[v] + 4 * self.factor_off
        self.hdl.barrier(channel=0)                    # every rank's backward has written its factors / dense rows
        _lib.call("r3dg_exchange_p2p", means3D.device, ctypes.byref(a), what="exchange_p2p")
        self.hdl.barrier(channel=1)                    # every rank is done reading / writing everyone's buffers
        return self.sh

    # the two calls rasterizer.set_grad_exchange makes inside backward (SH only; the leaves are averaged separately)
    def gather_factors(self, group=None):
        return None                                    # nothing to gather: the rebuild reads the peers' buffers directly

    def rebuild_sh(self, means3D, campos_all, degree):
        return self.exchange(means3D, campos_all, degree, dense=False)


def _exchange_args(world, rank, peer_ptrs, n_dense, multicast):
    """ExchangeArgs of the dense job: the first n_dense floats of every rank's symmetric buffer (peer_ptrs[v]) are
    replaced by their mean over the ranks, through the multicast address when there is one (0: none)."""
    a = _lib.ExchangeArgs()
    a.world, a.rank, a.n_dense = world, rank, n_dense
    for v in range(world):
        a.dense[v] = peer_ptrs[v]
    a.dense_multicast = multicast if multicast else None
    return a


def _nvls_mean_inplace(flat, hdl, world, rank, multicast, peer_ptrs):
    """In-place mean over the ranks of a symmetric flat fp32 buffer: barrier, one r3dg_exchange_p2p launch (dense job
    only), barrier."""
    a = _exchange_args(world, rank, peer_ptrs, flat.numel() // 4 * 4, multicast)
    a.M = 1
    hdl.barrier(channel=0)
    _lib.call("r3dg_exchange_p2p", flat.device, ctypes.byref(a), what="nvls mean")
    hdl.barrier(channel=1)


class LeafGradBucket:
    """Flat fp32 buffer holding the `.grad` of a list of LEAF parameters as views, so that one
    collective averages a whole N-view step at the place where averaging is always valid: the leaf
    parameters, after `loss.backward()` (every view-dependent map between the leaves and the
    rasterizer inputs — depth channels, brdf_color(viewdirs), viewdirs(means3D) — has been
    back-propagated by then; gradient paths that bypass the rasterizer, e.g. the environment map or
    regularisers, are covered too).  Autograd accumulates into the views in place, so no packing copy
    precedes the collective.  Usage per step: `zero()`, `loss.backward()`, `allreduce_mean()`.
    Parameters whose gradient is exchanged elsewhere (the SH leaves under `rasterizer.set_grad_exchange`)
    are simply left out of `params`."""

    def __init__(self, params, device=None, symmetric=False, group=None):
        self.params = [p for p in params]
        device = device if device is not None else self.params[0].device
        sizes = [p.numel() for p in self.params]
        self.offsets, off = [], 0
        for n in sizes:
            self.offsets.append(off)
            off += (n + 127) // 128 * 128
        self.hdl = None
        if symmetric:                       # NVLink path: the buffer is mapped into every rank, the mean is one NVLS kernel
            import torch.distributed._symmetric_memory as symm_mem
            group = group if group is not None else dist.group.WORLD
            self.flat = symm_mem.empty(max(off, 128), dtype=torch.float32, device=device)
            self.flat.zero_()
            self.hdl = symm_mem.rendezvous(self.flat, group)
            self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
            self.multicast = int(self.hdl.multicast_ptr) if getattr(self.hdl, "multicast_ptr", 0) else 0
            self.peer_ptrs = [int(x) for x in self.hdl.buffer_ptrs]
        else:
            self.flat = torch.zeros(max(off, 1), dtype=torch.float32, device=device)
        self.views = [self.flat[o:o + n].view(p.shape) for p, o, n in zip(self.params, self.offsets, sizes)]
        self.attach()

    def attach(self):
        """(Re-)bind every parameter's `.grad` to its view (call again after `p.grad = None`)."""
        for p, v in zip(self.params, self.views):
            p.grad = v

    def zero(self):
        self.flat.zero_()
        self.attach()

    def bytes(self):
        return self.flat.numel() * 4

    def allreduce_mean(self, group=None, async_op=False):
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return None
        for p, v in zip(self.params, self.views):          # a backward that replaced .grad (e.g. set_to_none) is copied in
            if p.grad is not None and p.grad.data_ptr() != v.data_ptr():
                v.copy_(p.grad)
                p.grad = v
        if self.hdl is not None:
            return _nvls_mean_inplace(self.flat, self.hdl, self.world, self.rank, self.multicast, self.peer_ptrs)
        if dist.get_backend(group) == "nccl":
            return dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=group, async_op=async_op)
        self.flat.mul_(1.0 / dist.get_world_size(group))
        return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)


def average_leaf_grads(params, group=None, skip=()):
    """One-off form of LeafGradBucket for callers that keep their own `.grad` tensors: averages
    `p.grad` of every parameter not in `skip` over the ranks (one all-reduce per tensor, in place)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return
    world = dist.get_world_size(group)
    skip_ids = {id(p) for p in skip}
    nccl = dist.get_backend(group) == "nccl"
    for p in params:
        if id(p) in skip_ids or p.grad is None:
            continue
        if nccl:
            dist.all_reduce(p.grad, op=dist.ReduceOp.AVG, group=group)
        else:
            p.grad.mul_(1.0 / world)
            dist.all_reduce(p.grad, op=dist.ReduceOp.SUM, group=group)


def allreduce_densification_stats(weights, xyz_grad_norm, normal_grad_norm, update_filter, radii, group=None):
    """Per-step densification statistics of an N-view step (SURVEY.md §8e).  The reference accumulates,
    per rendered view (scene/gaussian_model.py:931-937, train.py:161-165):
        weights_accum += weights;  xyz_gradient_accum[f] += ||viewspace_grad[f,:2]||;
        normal_gradient_accum[f] += ||normal_grad[f]||;  denom[f] += 1;  max_radii2D[f] = max(., radii[f])
    The norms are taken per view BEFORE accumulation, so the ranks exchange their per-view terms, not a
    summed gradient: ONE sum all-reduce of a packed [P,4] tensor (weights, masked xyz norm, masked normal
    norm, filter as 0/1) and ONE max all-reduce of the masked radii.  Inputs are this rank's view:
    weights [P,1], xyz_grad_norm [P,1], normal_grad_norm [P,1], update_filter bool [P], radii int [P].
    Returns (weights_sum [P,1], xyz_norm_sum [P,1], normal_norm_sum [P,1], denom_inc [P,1], radii_max [P])
    — the increments to add to / max into the five accumulators; identical on all ranks."""
    f = update_filter.reshape(-1, 1).to(weights.dtype)
    packed = torch.cat([weights.reshape(-1, 1), xyz_grad_norm.reshape(-1, 1) * f, normal_grad_norm.reshape(-1, 1) * f, f], dim=1).contiguous()
    rmax = torch.where(update_filter.reshape(-1), radii.reshape(-1), torch.zeros_like(radii.reshape(-1))).contiguous()
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(rmax, op=dist.ReduceOp.MAX, group=group)
    return packed[:, 0:1], packed[:, 1:2], packed[:, 2:3], packed[:, 3:4], rmax


def view_for_rank(step, rank, world, num_views):
    """Views of a step are dealt round-robin: rank r of step s renders view (s*world + r) % V."""
    return (step * world + rank) % num_views


def init_from_env(backend=None):
    """torchrun-style initialisation (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_* from the env).
    Returns (rank, local_rank, world)."""
    import os
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, local, world

"""Host-side mirror of the optimiser the reference trains with: `torch.optim.Adam(l, lr=0.0,
eps=1e-15)` over 7-13 per-Gaussian parameter groups (scene/gaussian_model.py:465-497), backed by
ONE fused sm_90a launch for all groups (r3dg_adam_step, csrc/adam.cu) instead of ~8 elementwise
kernels per group.

`FusedAdam` keeps torch.optim.Adam's observable behaviour for the configuration the reference
uses: same constructor arguments, `param_groups` (the reference edits `group['lr']` per step,
gaussian_model.py:499-505), and the same per-parameter state layout {step, exp_avg, exp_avg_sq} —
the densification surgery reads and replaces those entries (`_prune_optimizer`,
`cat_tensors_to_optimizer`, `replace_tensor_to_optimizer`, gaussian_model.py:667-750) and
checkpoints store `optimizer.state_dict()` (:129), so state dicts are interchangeable with
torch.optim.Adam in both directions.  weight_decay / amsgrad / maximize are not used by the
reference and are rejected.  There is no CPU path: parameters must be CUDA float32.
"""
import torch

from . import _lib


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *,
                 maximize=False, **unsupported):
        if weight_decay != 0 or amsgrad or maximize:
            raise ValueError("FusedAdam implements the reference's configuration only: weight_decay=0, amsgrad=False, maximize=False")
        for k in ("foreach", "capturable", "differentiable", "fused"):      # accepted and ignored (torch >= 2 keyword noise)
            unsupported.pop(k, None)
        if unsupported:
            raise TypeError(f"unexpected arguments {sorted(unsupported)}")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f"Invalid beta parameters: {betas}")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=0, amsgrad=False, maximize=False))

    @torch.no_grad()
    def step(self, closure=None, *, visibility=None):
        """One Adam step over every parameter that has a gradient.

        `visibility` (optional): a CUDA bool or uint8 tensor of P elements, shaped [P] or [P, 1], for a selective
        step.  Parameters with P rows (`param.shape[0] == P`, the rule of `prune_optimizer`) update only the rows
        whose byte is nonzero, with exactly the dense step's arithmetic; the other rows keep param, exp_avg and
        exp_avg_sq bit for bit and their gradient is not read.  Other parameters take the dense step, and
        `state["step"]` counts every step, so an all-ones mask is the dense step.  This is not Adam: a row left
        out keeps its moments instead of decaying them and moving on them.  No host synchronisation."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        todo = []
        device = None
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                if not p.is_cuda or p.dtype != torch.float32 or p.grad.dtype != torch.float32 or p.grad.is_sparse:
                    raise RuntimeError("FusedAdam: parameters and gradients must be dense CUDA float32 tensors (no CPU path)")
                if not p.is_contiguous():
                    raise RuntimeError("FusedAdam: parameters must be contiguous")
                device = device or p.device
                if p.device != device:
                    raise RuntimeError("FusedAdam: all parameters must live on one device")
                todo.append((group, p))
        mask = None if visibility is None else _row_mask(visibility, device, [p for _, p in todo])
        entries, keep = [], [mask]
        for group, p in todo:
            beta1, beta2 = group["betas"]
            st = self.state[p]
            if len(st) == 0:
                st["step"] = torch.tensor(0.0, dtype=torch.float32)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            step = st["step"]
            if torch.is_tensor(step):
                step += 1
                t = int(step.item())
            else:                                   # state dicts written by torch < 1.12 hold a Python int
                t = st["step"] = step + 1
            g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
            m, v = st["exp_avg"], st["exp_avg_sq"]
            if not (m.is_contiguous() and v.is_contiguous()):
                m = st["exp_avg"] = m.contiguous()
                v = st["exp_avg_sq"] = v.contiguous()
            keep.append(g)
            e = _lib.AdamTensor()
            e.param, e.grad, e.exp_avg, e.exp_avg_sq = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()
            e.n, e.step = p.numel(), t
            e.lr, e.beta1, e.beta2, e.eps = float(group["lr"]), float(beta1), float(beta2), float(group["eps"])
            if mask is not None and is_per_gaussian(p, mask.shape[0]) and mask.shape[0] > 0:
                e.row_mask, e.row_elems = mask.data_ptr(), p.numel() // mask.shape[0]
            entries.append(e)
        if entries:
            arr = (_lib.AdamTensor * len(entries))(*entries)
            _lib.call("r3dg_adam_step", device, len(entries), arr, what="FusedAdam.step")
        return loss


def is_per_gaussian(p, P):
    """A tensor holds one row per Gaussian of a model of P Gaussians when its first dimension is P."""
    return p.dim() > 0 and p.shape[0] == P


def _row_mask(visibility, device, params):
    """`visibility` as a contiguous uint8 tensor [P] for FusedAdam.step, checked against the parameters that have a
    gradient (none: the step is a no-op and any length is accepted)."""
    if not torch.is_tensor(visibility) or visibility.dtype not in (torch.bool, torch.uint8):
        raise ValueError("FusedAdam.step: visibility must be a bool or uint8 tensor")
    if not visibility.is_cuda or (device is not None and visibility.device != device):
        raise ValueError("FusedAdam.step: visibility must be on the parameters' CUDA device")
    if not (visibility.dim() == 1 or (visibility.dim() == 2 and visibility.shape[1] == 1)):
        raise ValueError(f"FusedAdam.step: visibility must be shaped [P] or [P, 1], got {tuple(visibility.shape)}")
    P = visibility.shape[0]
    if params and not any(is_per_gaussian(p, P) for p in params):
        raise ValueError(f"FusedAdam.step: no parameter with a gradient has {P} rows to match visibility")
    mask = visibility.reshape(P).contiguous()
    return mask.view(torch.uint8) if mask.dtype == torch.bool else mask


_torch_adam = None


def install():
    """Make the unmodified reference pick up the fused step: rebinds `torch.optim.Adam` (the name
    scene/gaussian_model.py:489 resolves at call time) to FusedAdam.  `uninstall()` restores it."""
    global _torch_adam
    if _torch_adam is None:
        _torch_adam = torch.optim.Adam
        torch.optim.Adam = FusedAdam
    return FusedAdam


def uninstall():
    global _torch_adam
    if _torch_adam is not None:
        torch.optim.Adam = _torch_adam
        _torch_adam = None


# ---------------------------------------------------------------------------------------------
# Densification surgery (SURVEY.md §8(f)3): the reference's `_prune_optimizer` / `prune_points`
# (scene/gaussian_model.py:682-729) apply one boolean mask to every per-Gaussian tensor, one
# `tensor[mask]` launch chain each.  `compact_rows` does the whole set with one scan of the mask and
# one gather launch (r3dg_compact_scan / r3dg_compact_rows).
# ---------------------------------------------------------------------------------------------
_compact_pinned = None


def compact_rows(tensors, keep):
    """[t[keep] for t in tensors] for tensors that share dim 0 (fp32 / int32 / any dtype whose row is a
    multiple of 4 bytes; other rows fall back to boolean indexing).  One host read-back of the kept
    count — boolean indexing has the same one."""
    global _compact_pinned
    keep = keep.reshape(-1)
    P = keep.shape[0]
    dev = keep.device
    if not keep.is_cuda:
        raise RuntimeError("compact_rows runs on the GPU only (no CPU path)")
    k8 = keep.to(torch.uint8).contiguous() if keep.dtype != torch.uint8 else keep.contiguous()
    if keep.dtype == torch.bool:
        k8 = keep.contiguous().view(torch.uint8)
    tmp = _lib.scratch(_lib.load().r3dg_compact_tmp_bytes(P), dev)
    if _compact_pinned is None:
        _compact_pinned = torch.zeros(1, dtype=torch.int32).pin_memory()
    _lib.call("r3dg_compact_scan", dev, P, k8.data_ptr(), tmp.data_ptr(), tmp.numel(), _compact_pinned.data_ptr(),
              what="compact_scan")
    torch.cuda.current_stream(dev).synchronize()
    count = int(_compact_pinned.item())
    outs, descs, hold = [], [], []
    for t in tensors:
        assert t.shape[0] == P, "all tensors must share dim 0 with the mask"
        row_bytes = (t.numel() // max(P, 1)) * t.element_size() if P > 0 else 0
        if P == 0 or row_bytes % 4 != 0 or not t.is_cuda:
            outs.append(t[keep.bool()])
            continue
        src = t.detach().contiguous()
        dst = torch.empty((count,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
        hold.append(src)
        d = _lib.CompactTensor()
        d.src, d.dst, d.row_bytes = src.data_ptr(), dst.data_ptr(), row_bytes
        descs.append(d)
        outs.append(dst)
    if descs and count > 0:
        arr = (_lib.CompactTensor * len(descs))(*descs)
        _lib.call("r3dg_compact_rows", dev, P, len(descs), arr, k8.data_ptr(), tmp.data_ptr(), what="compact_rows")
    return outs


def prune_optimizer(optimizer, keep, extra=()):
    """`GaussianModel._prune_optimizer(mask)` (scene/gaussian_model.py:682-700) for every per-Gaussian group at
    once: parameters and both Adam moments of all groups whose parameter has `keep.shape[0]` rows (+ any `extra`
    per-Gaussian tensors, e.g. xyz_gradient_accum / denom / max_radii2D of prune_points :702-729) are compacted by ONE
    launch.  Returns ({group name: new nn.Parameter}, [compacted extras]); optimizer state is re-keyed like the reference."""
    P = keep.reshape(-1).shape[0]
    groups = [g for g in optimizer.param_groups if len(g["params"]) == 1 and is_per_gaussian(g["params"][0], P)]
    work, slots = [], []
    for g in groups:
        p = g["params"][0]
        st = optimizer.state.get(p, None)
        work.append(p.data); slots.append((g, "param"))
        if st is not None and "exp_avg" in st:
            work.append(st["exp_avg"]); slots.append((g, "exp_avg"))
            work.append(st["exp_avg_sq"]); slots.append((g, "exp_avg_sq"))
    n_model = len(work)
    work += list(extra)
    outs = compact_rows(work, keep)
    new = {}
    per_group = {}
    for (g, kind), t in zip(slots, outs[:n_model]):
        per_group.setdefault(id(g), {"g": g})[kind] = t
    for rec in per_group.values():
        g = rec["g"]
        old = g["params"][0]
        st = optimizer.state.pop(old, None)
        newp = torch.nn.Parameter(rec["param"].requires_grad_(True))
        g["params"][0] = newp
        if st is not None:
            if "exp_avg" in rec:
                st["exp_avg"], st["exp_avg_sq"] = rec["exp_avg"], rec["exp_avg_sq"]
            optimizer.state[newp] = st
        new[g.get("name", str(len(new)))] = newp
    return new, outs[n_model:]

"""fp64 truth of the rasterizer's depth statistics (csrc/composite.cu, composite_bwd.cu with depth statistics on).

Per pixel, with the composited entries' weights w = alpha T and depths d (tz, or the ray-depth plane of
raydepth64.plane) in list order:

    depth2  = sum w d^2,
    median  = d of the last composited entry whose transmittance before it, T, is > 0.5 (2DGS's rule), 0 for none.

stats() forms both, and the median's 1-based position among the pixel's list entries, from [n, L] tensors of w, d, T
and a composited mask; it is differentiable in w and d (the median is a selection: its gradient reaches the selected
entry's d only).  distortion() is the pairwise form  sum_i sum_j w_i w_j (d_i - d_j)^2 / 2, which equals
A depth2 - depth^2 with A = sum w.  walk_stats() takes the pairs of a raster64.Walk (the kernel's own lists and
n_contrib) with d = the records' tz or the plane depth of raydepth64, and `ambiguous` marks pixels whose T before some
composited entry lies within AMBIGUOUS of 0.5: there fp32 and fp64 may select different entries."""
import torch

AMBIGUOUS = 1e-5


def stats(w, d, T, valid):
    """(depth2 [n], median [n], median position [n], 1-based, 0 for none) of the pixels' lists: w, d, T [n, L] with T
    the transmittance before each entry, valid [n, L] the composited entries."""
    zero = torch.zeros_like(w)
    w = torch.where(valid, w, zero)
    d = torch.where(valid, d, zero)
    depth2 = (w * d * d).sum(1)
    sel = valid & (T > 0.5)
    L = w.shape[1]
    j = torch.arange(1, L + 1, device=w.device)
    pos = torch.where(sel, j[None, :], torch.zeros_like(j)[None, :]).amax(1) if L else torch.zeros(w.shape[0],
                                                                                                     dtype=torch.long)
    k = (pos - 1).clamp_min(0)
    median = torch.where(pos > 0, d.gather(1, k[:, None])[:, 0] if L else zero.sum(1), zero.sum(1))
    return depth2, median, pos


def distortion(w, d, valid):
    """sum_i sum_j w_i w_j (d_i - d_j)^2 / 2 per pixel [n], by the pairwise sum."""
    zero = torch.zeros_like(w)
    w = torch.where(valid, w, zero)
    d = torch.where(valid, d, zero)
    return 0.5 * (w[:, :, None] * w[:, None, :] * (d[:, :, None] - d[:, None, :]) ** 2).sum((1, 2))


def lists(alphas, t_cut=1e-4):
    """(w, T, valid) of hand-built lists: alphas [n, L] (<= 0 marks an entry that is skipped, as alpha < 1/255 is), the
    forward's early stop (T (1 - alpha) < t_cut: that entry and everything after it is not composited)."""
    n, L = alphas.shape
    w = torch.zeros(n, L, dtype=torch.float64)
    Tb = torch.zeros(n, L, dtype=torch.float64)
    valid = torch.zeros(n, L, dtype=torch.bool)
    for i in range(n):
        T = 1.0
        for k in range(L):
            a = float(alphas[i, k])
            Tb[i, k] = T
            if a <= 0.0:
                continue
            if T * (1.0 - a) < t_cut:
                break
            valid[i, k] = True
            w[i, k] = a * T
            T *= 1.0 - a
    return w, Tb, valid


def walk_stats(wk, depth):
    """(depth2, median, position, ambiguous) of the pixels of a raster64.Walk, d = depth [n, L] per pair."""
    w = wk.alpha * wk.T
    d2, med, pos = stats(w, depth, wk.T, wk.valid)
    amb = (wk.valid & ((wk.T - 0.5).abs() <= AMBIGUOUS)).any(1)
    return d2, med, pos, amb

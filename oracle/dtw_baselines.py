"""ORACLE (test infrastructure only; see oracle/__init__.py): the baseline pitch alignments of the paper's comparison, a vectorised
numpy / torch restatement of LoNDTW (modules/voice_conversion/dtw/local_norm_dtw.py), NaiveDTW / ZMNaiveDTW / NNaiveDTW
(naive_dtw.py) and NInterpo (naive_interpo.py), with time_warp / align_from_distances from oracle/sadtw.py.
tests/golden/dtw_baselines.npz pins it to the unmodified reference.

The costs are the reference's own torch CPU operations on the same tensors (torch.cdist, Tensor.mean / std), so they reproduce the
reference bit for bit; only get_local_context's double loop becomes an unfold of the zero-padded contour.  The CUDA path
(csrc/sadtw.cu) computes the same formulas in a fixed summation order, so it is compared with these costs within a rounding bound.
"""
import numpy as np
import torch

from oracle import sadtw as O

METHODS = ('LoNDTW', 'NaiveDTW', 'ZMNaiveDTW', 'NNaiveDTW', 'NInterpo')
CONTEXT = 32


def _t(x):
    return x.detach().cpu() if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))


def local_context(f0):
    """get_local_context(f0) as a tensor [S, 64] in f0's type: row t = f0[t - 32 .. t + 31], zeros outside [0, S)."""
    f = _t(f0).reshape(-1)
    z = torch.zeros(CONTEXT, dtype=f.dtype)
    return torch.cat([z, f, z]).unfold(0, 2 * CONTEXT, 1)[:f.shape[0]].contiguous()


def cdist_cost(method, src, tgt):
    """The reference's dists.squeeze(0) [S, T] in the input's type."""
    a, b = _t(src), _t(tgt)
    if method == 'LoNDTW':
        a, b = local_context(a), local_context(b)
        a = a - a.mean(-1).unsqueeze(-1)
        b = b - b.mean(-1).unsqueeze(-1)
        return torch.cdist(a[None], b[None])[0]
    if method == 'NaiveDTW':
        if a.dim() != 2 or b.dim() != 2:
            raise ValueError('NaiveDTW takes [S, H] features')
        return torch.cdist(a[None], b[None])[0]
    a, b = a.reshape(-1), b.reshape(-1)
    if method == 'ZMNaiveDTW':
        a, b = a - a.mean(), b - b.mean()
    elif method == 'NNaiveDTW':
        a, b = (a - a.mean()) / (a.std() + 0.00000001), (b - b.mean()) / (b.std() + 0.00000001)
    else:
        raise ValueError(f'no cost for {method!r}')
    return torch.cdist(a[None, :, None], b[None, :, None])[0]


def cost(method, src, tgt):
    """numpy [T, S]: the matrix time_warp sees (costs.T)."""
    return cdist_cost(method, src, tgt).T.contiguous().numpy()


def nearest_index(S, T):
    """F.interpolate(size=T, mode='nearest')'s source frame of each output frame: int64 [T]."""
    i = np.arange(T)
    if T == S:
        return i.astype(np.int64)
    if T == 2 * S:
        return (i >> 1).astype(np.int64)
    scale = np.float32(S) / np.float32(T)
    return np.minimum(np.floor(i.astype(np.float32) * scale).astype(np.int64), S - 1)


def align(method, src, tgt, full=False):
    """(alignment int64 [T], DTW value at the last cell) of method(src, tgt, .); NInterpo: (index map, None).  full=True adds the
    [T, S] cost and the DTW matrix."""
    if method == 'NInterpo':
        return nearest_index(_t(src).shape[0], _t(tgt).shape[0]), None
    c = cost(method, src, tgt)
    dtw = O.time_warp(c)
    al = np.asarray(O.align_from_dtw(dtw), np.int64)
    if full:
        return al, dtw[-1, -1], dict(cost=c, dtw=dtw)
    return al, dtw[-1, -1]


def path_cost(costs, dirs_dtw):
    """Sum of costs [T, S] over the cells of the path align_from_distances walks on the DTW matrix dirs_dtw (cells with i, j >= 1:
    time_warp's value at the last cell when dirs_dtw = time_warp(costs))."""
    i, j = costs.shape[0] - 1, costs.shape[1] - 1
    s = costs.dtype.type(0)
    while i > 0 and j > 0:
        s = s + costs[i, j]
        best, bv = (i - 1, j), dirs_dtw[i - 1, j]
        for cand in ((i, j - 1), (i - 1, j - 1)):
            if dirs_dtw[cand] < bv:
                best, bv = cand, dirs_dtw[cand]
        i, j = best
    return s


def alignment_accuracy(alignment, amateur_mel2ph, prof_mel2ph):
    """job()'s (prof_mel2ph == amateur_mel2ph[alignment]).sum() / (prof_mel2ph != 0).sum()."""
    a, m, p = np.asarray(alignment), np.asarray(amateur_mel2ph), np.asarray(prof_mel2ph)
    return (p == m[a]).sum() / (p != 0).sum()


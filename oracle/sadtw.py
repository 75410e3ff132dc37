"""ORACLE (test infrastructure only; see oracle/__init__.py): shape-aware DTW pitch alignment, a vectorised numpy restatement of
SADTW (modules/voice_conversion/dtw/shape_aware_dtw.py) and EHSADTW (enhance_sadtw.py) over time_warp / align_from_distances
(align.py).  tests/golden/sadtw.npz pins it to the unmodified reference; the CUDA path (csrc/sadtw.cu) is compared with it bit for
bit.

1. histogram (cal_hist_of_f0, max_window=64, normalize_hist=True): 48 bins per frame = 8 slope windows x 6 regions.  Window w of
   frame t covers the frames [clamp(t + int(lo * s)), clamp(t + int(hi * s))) (int truncates toward zero, a left boundary of 0
   becomes 1, clamp to [0, T]).  slope = (f[i] - f[t]) / (i - t) in the input's type (float32 stays float32: numpy 2 / torch
   promotion with Python scalars), times 0.5 / 0.75 / 0.9 in EHSADTW's windows 0 and 7 / 1 and 6 / 2 and 5.  |slope| < 0.57735,
   < 1.73205, else: regions 2 / 1 / 0 when f[i] - f[t] >= 0, else 3 / 4 / 5.  A bin is k / total in double (Python), then float32
   (torch.tensor).
2. cost (cal_hist_dist): float32 sum over the 48 bins of 0.5 (b - a)^2 / (b + a + 1e-8), here summed sequentially over the bins
   (the reference sums in torch's CPU reduction order, which may differ in the last bits), as [T, S] = the matrix time_warp sees.
3. time_warp: dtw[0, 0] = 0, the rest of row 0 and column 0 = inf, dtw[i, j] = cost[i, j] + min(up, left, diag) in the cost's type,
   min() keeping the first operand unless a later one is strictly smaller (Python's min).
4. align_from_distances: from the last cell while i > 0 and j > 0: results[i] = j, then the first minimum of dtw at (i-1, j),
   (i, j-1), (i-1, j-1).  results[0] = 0; rows never reached stay 0.
"""
import numpy as np

WINDOWS = {
    'SADTW': [(-64, -32), (-32, -16), (-16, -8), (-8, 0), (0, 8), (8, 16), (16, 32), (32, 64)],
    'EHSADTW': [(-64, -48), (-48, -32), (-32, -16), (-16, 0), (0, 16), (16, 32), (32, 48), (48, 64)],
}
EH_WEIGHTS = (0.5, 0.75, 0.9, None, None, 0.9, 0.75, 0.5)
BINS = 48


def f0_numpy(f):
    """numpy view of a 1-D (or [S, 1]) f0 given as numpy or torch, keeping float32 / float64."""
    if hasattr(f, 'detach'):
        f = f.detach().cpu().numpy()
    f = np.asarray(f)
    if f.ndim == 2 and f.shape[1] == 1:
        f = f[:, 0]
    if f.ndim != 1:
        raise ValueError(f'f0 must be [S] or [S, 1], got {f.shape}')
    if f.dtype not in (np.float32, np.float64):
        raise TypeError(f'f0 must be float32 or float64, got {f.dtype}')
    return f


def scaled_windows(method, scale=1.0):
    out = []
    for lo, hi in WINDOWS[method]:
        lo, hi = int(lo * scale), int(hi * scale)
        out.append((1 if lo == 0 else lo, hi))
    return out


def counts(f0, method='SADTW', scale=1.0):
    """int64 [T, 48] region counts of cal_hist_of_f0."""
    f = f0_numpy(f0)
    dt = f.dtype.type
    T = len(f)
    c = np.zeros((T, BINS), np.int64)
    t = np.arange(T)
    for w, (lo, hi) in enumerate(scaled_windows(method, scale)):
        for off in range(lo, hi):
            tv = t[(t + off >= 0) & (t + off < T)]
            if len(tv) == 0:
                continue
            d = f[tv + off] - f[tv]
            tan = d / dt(off)
            if method == 'EHSADTW' and EH_WEIGHTS[w] is not None:
                tan = tan * dt(EH_WEIGHTS[w])
            a, up = np.abs(tan), d >= 0
            region = np.where(a < dt(0.57735), np.where(up, 2, 3), np.where(a < dt(1.73205), np.where(up, 1, 4), np.where(up, 0, 5)))
            np.add.at(c, (tv, w * 6 + region), 1)
    return c


def histogram(f0, method='SADTW', scale=1.0):
    """float32 [T, 48]: torch.tensor(cal_hist_of_f0(f0, normalize_hist=True, scale_factor=scale))."""
    c = counts(f0, method, scale)
    total = c.sum(1)
    if len(total) < 2 or (total == 0).any():
        raise ValueError('every frame needs a non-empty slope window (the reference divides by zero)')
    return (c.astype(np.float64) / total[:, None].astype(np.float64)).astype(np.float32)


def cost(hist_src, hist_tgt, chunk=256):
    """float32 [T, S]: costs.T of cal_hist_dist(hist_src, hist_tgt), summed sequentially over the bins, chunked over rows."""
    a, b = np.asarray(hist_src, np.float32), np.asarray(hist_tgt, np.float32)
    out = np.empty((len(b), len(a)), np.float32)
    half, eps = np.float32(0.5), np.float32(1e-8)
    for r0 in range(0, len(b), chunk):
        bb = b[r0:r0 + chunk, None, :]
        acc = np.zeros((bb.shape[0], len(a)), np.float32)
        for m in range(BINS):
            x, y = a[None, :, m], bb[:, :, m]
            d = y - x
            acc = acc + (half * (d * d)) / ((y + x) + eps)
        out[r0:r0 + chunk] = acc
    return out


def time_warp(costs):
    """align.time_warp, the recurrence vectorised along the anti-diagonals, in the cost's type."""
    c = np.asarray(costs)
    R, C = c.shape
    dtw = np.zeros_like(c)
    dtw[0, 1:] = np.inf
    dtw[1:, 0] = np.inf
    for d in range(2, R + C - 1):
        i = np.arange(max(1, d - C + 1), min(d - 1, R - 1) + 1)
        if len(i) == 0:
            continue
        j = d - i
        m = dtw[i - 1, j].copy()
        left, dg = dtw[i, j - 1], dtw[i - 1, j - 1]
        sel = left < m
        m[sel] = left[sel]
        sel = dg < m
        m[sel] = dg[sel]
        dtw[i, j] = c[i, j] + m
    return dtw


def align_from_dtw(dtw):
    """align.align_from_distances given time_warp's matrix: a Python list of length rows."""
    i, j = dtw.shape[0] - 1, dtw.shape[1] - 1
    results = [0] * dtw.shape[0]
    while i > 0 and j > 0:
        results[i] = j
        best, bv = (i - 1, j), dtw[i - 1, j]
        for cand in ((i, j - 1), (i - 1, j - 1)):
            if dtw[cand] < bv:
                best, bv = cand, dtw[cand]
        i, j = best
    return results


def align_from_distances(distance_matrix):
    return align_from_dtw(time_warp(distance_matrix))


def shape_aware_align(src_f0, tgt_f0, method='EHSADTW', scale=None, full=False):
    """SADTW / EHSADTW(src, tgt, .)'s alignment as int64 [T] and the DTW value at the last cell.  full=True also returns the two
    histograms, the [T, S] cost and the DTW matrix."""
    src, tgt = f0_numpy(src_f0), f0_numpy(tgt_f0)
    if len(src) < 2 or len(tgt) < 2:
        raise ValueError('both contours need at least 2 frames')
    hs = histogram(src, method, 1.0)
    ht = histogram(tgt, method, len(tgt) / len(src) if scale is None else scale)
    cst = cost(hs, ht)
    dtw = time_warp(cst)
    align = np.asarray(align_from_dtw(dtw), np.int64)
    if full:
        return align, dtw[-1, -1], dict(hist_src=hs, hist_tgt=ht, cost=cst, dtw=dtw)
    return align, dtw[-1, -1]

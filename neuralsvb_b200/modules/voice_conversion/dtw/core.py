"""Pitch alignment on the GPU (csrc/sadtw.cu): the batched entry points behind the drop-in ``align``, ``shape_aware_dtw``,
``enhance_sadtw``, ``local_norm_dtw``, ``naive_dtw`` and ``naive_interpo`` modules, plus ``align_pitch`` for a binarizer,
``a2p_alignment_batch`` for ``MleSVBVAE``'s ``a2p`` way and ``alignment_accuracy`` for the paper's comparison of the six methods.

f0 contours may be numpy arrays or torch tensors, on the host or on a CUDA device, shaped [S] or [S, 1], float32 or float64; the
arithmetic runs in that type, like the reference's.  Host inputs are copied to the current CUDA device.  There is no CPU path.
"""
import ctypes

import numpy as np
import torch

from neuralsvb_b200 import _native

VARIANTS = {'SADTW': 0, 'EHSADTW': 1}
BASELINES = {'LoNDTW': 0, 'NaiveDTW': 1, 'ZMNaiveDTW': 2, 'NNaiveDTW': 3, 'NInterpo': 4}
METHODS = tuple(VARIANTS) + tuple(BASELINES)
DTYPES = {torch.float32: 0, torch.float64: 1}
BINS = 48


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _i32(v):
    a = np.ascontiguousarray(v, dtype=np.int32)
    return a, ctypes.c_void_p(a.ctypes.data)


def _check(rc, what):
    if rc is not None and rc < 0:
        msg = _native.lib().svb_last_error().decode('utf-8', 'replace')
        if rc == -1:                   # SVB_ERR_INVALID: rejected before any launch
            raise ValueError(f'{what}: {msg}')
        raise RuntimeError(f'libsvb_vocoder {what} failed ({rc}): {msg}')
    return rc


def device_of(*xs):
    """The CUDA device of the first device tensor among xs, else the current CUDA device."""
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise RuntimeError('shape-aware DTW runs on CUDA: neuralsvb_b200 has no CPU fallback')
    return torch.device('cuda', torch.cuda.current_device())


def as_tensor(x):
    if torch.is_tensor(x):
        return x.detach()
    return torch.from_numpy(np.ascontiguousarray(x))


def f0_tensor(f, device):
    """1-D contiguous device tensor of an f0 contour ([S] or [S, 1], float32 or float64)."""
    t = as_tensor(f)
    if t.dim() == 2 and t.shape[1] == 1:
        t = t[:, 0]
    if t.dim() != 1:
        raise ValueError(f'an f0 contour must be [S] or [S, 1], got {tuple(t.shape)}')
    if t.dtype not in DTYPES:
        raise TypeError(f'an f0 contour must be float32 or float64, got {t.dtype}')
    return t.to(device).contiguous()


def _check_finite(t):
    if not bool(torch.isfinite(t).all()):
        raise ValueError('f0 contains NaN or inf (the reference exits on it)')


def _batch_f0(fs, device, what):
    ts = [f0_tensor(f, device) for f in fs]
    dts = {t.dtype for t in ts}
    if len(dts) > 1:
        raise TypeError(f'{what} f0 contours mix float32 and float64; a batch runs in one type')
    lens = [int(t.shape[0]) for t in ts]
    if min(lens) < 2:
        raise ValueError(f'{what} contour of {min(lens)} frames: at least 2 are needed (the reference divides by zero)')
    cat = torch.cat(ts) if len(ts) > 1 else ts[0]
    _check_finite(cat)
    return cat, lens, ts[0].dtype


class AlignResult:
    """alignment: int64 device tensor [sum T] (pair p's rows after the pairs before it), offsets: its row offsets [n + 1] (host),
    path_cost: float32 [n] DTW value at each pair's last cell, stage_ms: (histogram, cost, dtw, backtrack) CUDA-event times or None,
    workspace / sections: the workspace and its section byte offsets when keep_workspace=True."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def split(self):
        """One host int64 numpy array per pair."""
        a = self.alignment.cpu().numpy()
        return [a[self.offsets[p]:self.offsets[p + 1]] for p in range(len(self.offsets) - 1)]


def align_batch(srcs, tgts, method='EHSADTW', scales=None, stage_ms=False, keep_workspace=False):
    """Shape-aware DTW of n pairs in one launch sequence: srcs = amateur contours (S_p frames), tgts = professional ones (T_p
    frames); scales: the professional histogram's scale factor per pair (default T_p / S_p, cal_shape_dist's).  The baseline
    methods (BASELINES) go to baseline_batch."""
    if method in BASELINES:
        return baseline_batch(srcs, tgts, method, stage_ms)
    return _sadtw(srcs, tgts, method, scales, stage_ms, keep_workspace, 'sadtw')


LONG_MAX_FRAMES = 65536


def align_long(srcs, tgts, method='EHSADTW', scales=None, stage_ms=False, keep_workspace=False):
    """align_batch for whole songs: each take of a pair up to LONG_MAX_FRAMES frames (6.3 min at 22.05 kHz / hop 128).  A pair
    whose shorter take exceeds 8192 frames runs its DTW on a thread-block cluster; the others on the one-CTA kernel of
    align_batch, in the same call.  Same results as align_batch on any pair both accept.  The workspace holds every pair's cost
    matrix (5 bytes per cell: 8.5 GB for a 4-minute pair), long_workspace_bytes."""
    if method not in VARIANTS:
        raise ValueError(f'align_long runs {sorted(VARIANTS)}, got {method!r}')
    return _sadtw(srcs, tgts, method, scales, stage_ms, keep_workspace, 'sadtw_long')


def long_workspace_bytes(src_len, tgt_len):
    """Bytes of align_long's device workspace for pairs of these amateur / professional frame counts (ValueError past its
    limits)."""
    s_arr, s_p = _i32(src_len)
    t_arr, t_p = _i32(tgt_len)
    if s_arr.shape != t_arr.shape or s_arr.ndim != 1:
        raise ValueError(f'{s_arr.shape} amateur and {t_arr.shape} professional lengths')
    return _check(_native.lib().svb_sadtw_long_workspace_bytes(len(s_arr), s_p, t_p, None), 'sadtw_long_workspace_bytes')


SONGS_WORKSPACE_BYTES = 24 << 30
STRIPE_MODES = ('single_pass', 'checkpointed')


class StripePlan(ctypes.Structure):
    """svb_sadtw_stripe_plan: the mode (index into STRIPE_MODES), the stripe width K in anti-diagonals, the stripe count, the byte
    offsets of the workspace sections, the workspace size and the smallest budget the planner accepts."""
    _fields_ = [('mode', ctypes.c_int32), ('stripe_diags', ctypes.c_int32), ('stripes', ctypes.c_int32),
                ('reserved', ctypes.c_int32), ('offsets', ctypes.c_int64 * 8), ('total_bytes', ctypes.c_int64),
                ('min_budget_bytes', ctypes.c_int64)]


def striped_plan(src_len, tgt_len, budget):
    """The plan of align_songs for pairs of these amateur / professional frame counts within ``budget`` bytes of workspace
    (host only; ValueError past align_long's limits or below the smallest workable budget, which the message names)."""
    s_arr, s_p = _i32(src_len)
    t_arr, t_p = _i32(tgt_len)
    if s_arr.shape != t_arr.shape or s_arr.ndim != 1:
        raise ValueError(f'{s_arr.shape} amateur and {t_arr.shape} professional lengths')
    plan = StripePlan()
    _check(_native.lib().svb_sadtw_striped_plan(len(s_arr), s_p, t_p, int(budget), ctypes.byref(plan)), 'sadtw_striped_plan')
    return plan


def striped_workspace_bytes(src_len, tgt_len, budget):
    """Bytes of align_songs' device workspace for these frame counts within ``budget`` (<= budget; ValueError as striped_plan)."""
    return striped_plan(src_len, tgt_len, budget).total_bytes


def _frames(f):
    t = as_tensor(f)
    if t.dim() == 1 or (t.dim() == 2 and t.shape[1] == 1):
        return int(t.shape[0])
    raise ValueError(f'an f0 contour must be [S] or [S, 1], got {tuple(t.shape)}')


def align_songs(srcs, tgts, method='EHSADTW', workspace_bytes=SONGS_WORKSPACE_BYTES, stage_ms=False):
    """align_long's results, bit for bit, in at most ``workspace_bytes`` of device workspace: a budget, not a choice of
    algorithm.  The planner (striped_plan) runs a single pass that keeps every direction byte (1 byte per cell instead of
    align_long's 5) when that fits, else a checkpointed forward and backward pass over stripes of K anti-diagonals whose memory
    is linear in the takes' lengths.  The result also carries ``mode`` (one of STRIPE_MODES), ``stripe_diags`` (K),
    ``stripes`` and ``workspace_bytes``; stage_ms: (histogram, forward, backward, backtrack) CUDA-event times.  Lengths,
    method and budget are checked before any device work."""
    if method not in VARIANTS:
        raise ValueError(f'align_songs runs {sorted(VARIANTS)}, got {method!r}')
    if len(srcs) != len(tgts) or len(srcs) == 0:
        raise ValueError(f'{len(srcs)} amateur and {len(tgts)} professional contours')
    plan = striped_plan([_frames(f) for f in srcs], [_frames(f) for f in tgts], workspace_bytes)
    device = device_of(*srcs, *tgts)
    src, S, dt = _batch_f0(srcs, device, 'amateur')
    tgt, T, dt2 = _batch_f0(tgts, device, 'professional')
    if dt != dt2:
        raise TypeError('amateur and professional f0 must have the same type')
    n, lib = len(S), _native.lib()
    s_arr, s_p = _i32(S)
    t_arr, t_p = _i32(T)
    ws = torch.empty(plan.total_bytes, dtype=torch.uint8, device=device)
    out = torch.empty(int(t_arr.sum()), dtype=torch.int64, device=device)
    pc = torch.empty(n, dtype=torch.float32, device=device)
    ms = (ctypes.c_float * 4)() if stage_ms else None
    with torch.cuda.device(device):
        _check(lib.svb_sadtw_align_striped(_vp(src), _vp(tgt), DTYPES[dt], VARIANTS[method], n, s_p, t_p, None, _vp(ws),
                                           plan.total_bytes, int(workspace_bytes), _vp(out), _vp(pc), ms,
                                           _native.current_stream_ptr(device)), 'sadtw_align_striped')
    return AlignResult(alignment=out, offsets=np.concatenate([[0], np.cumsum(T)]).astype(np.int64), path_cost=pc,
                       stage_ms=tuple(ms) if stage_ms else None, src_len=S, tgt_len=T, workspace=None, sections=None,
                       mode=STRIPE_MODES[plan.mode], stripe_diags=plan.stripe_diags, stripes=plan.stripes,
                       workspace_bytes=plan.total_bytes)


def _sadtw(srcs, tgts, method, scales, stage_ms, keep_workspace, entry):
    if method not in VARIANTS:
        raise ValueError(f'method must be one of {sorted(METHODS)}, got {method!r}')
    if len(srcs) != len(tgts) or len(srcs) == 0:
        raise ValueError(f'{len(srcs)} amateur and {len(tgts)} professional contours')
    device = device_of(*srcs, *tgts)
    src, S, dt = _batch_f0(srcs, device, 'amateur')
    tgt, T, dt2 = _batch_f0(tgts, device, 'professional')
    if dt != dt2:
        raise TypeError('amateur and professional f0 must have the same type')
    n, lib = len(S), _native.lib()
    s_arr, s_p = _i32(S)
    t_arr, t_p = _i32(T)
    sec = (ctypes.c_int64 * 5)()
    size_fn = lib.svb_sadtw_workspace_bytes if entry == 'sadtw' else lib.svb_sadtw_long_workspace_bytes
    align_fn = lib.svb_sadtw_align if entry == 'sadtw' else lib.svb_sadtw_align_long
    ws_bytes = _check(size_fn(n, s_p, t_p, sec), f'{entry}_workspace_bytes')
    sc = None
    if scales is not None:
        sc = np.ascontiguousarray(scales, dtype=np.float64)
        if sc.shape != (n,):
            raise ValueError(f'{n} pairs but {sc.shape} scale factors')
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    out = torch.empty(int(t_arr.sum()), dtype=torch.int64, device=device)
    pc = torch.empty(n, dtype=torch.float32, device=device)
    ms = (ctypes.c_float * 4)() if stage_ms else None
    with torch.cuda.device(device):
        _check(align_fn(_vp(src), _vp(tgt), DTYPES[dt], VARIANTS[method], n, s_p, t_p,
                        None if sc is None else ctypes.c_void_p(sc.ctypes.data), _vp(ws), ws_bytes, _vp(out), _vp(pc), ms,
                        _native.current_stream_ptr(device)), f'{entry.replace("sadtw", "sadtw_align")}')
    return AlignResult(alignment=out, offsets=np.concatenate([[0], np.cumsum(T)]).astype(np.int64), path_cost=pc,
                       stage_ms=tuple(ms) if stage_ms else None, src_len=S, tgt_len=T,
                       workspace=ws if keep_workspace else None, sections=list(sec) if keep_workspace else None)


def histogram(f0s, method='SADTW', scales=None, counts=False):
    """The histogram kernel alone on n contours: float32 device [sum len, 48] (k / total) and, with counts=True, int32 k."""
    device = device_of(*f0s)
    f, lens, dt = _batch_f0(f0s, device, 'the')
    n, lib = len(lens), _native.lib()
    l_arr, l_p = _i32(lens)
    sc = np.ascontiguousarray(np.ones(n) if scales is None else scales, dtype=np.float64)
    ws_bytes = _check(lib.svb_sadtw_histogram_workspace_bytes(n), 'sadtw_histogram_workspace_bytes')
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    rows = int(l_arr.sum())
    hist = torch.empty(rows, BINS, dtype=torch.float32, device=device)
    cnt = torch.empty(rows, BINS, dtype=torch.int32, device=device) if counts else None
    with torch.cuda.device(device):
        _check(lib.svb_sadtw_histogram(_vp(f), DTYPES[dt], VARIANTS[method], n, l_p, ctypes.c_void_p(sc.ctypes.data), _vp(ws),
                                       ws_bytes, _vp(hist), _vp(cnt), _native.current_stream_ptr(device)), 'sadtw_histogram')
    return (hist, cnt) if counts else hist


def hist_of_f0(input_f, method, max_window=64, normalize_hist=False, scale_factor=1.):
    """cal_hist_of_f0: a list of T lists of 48 numbers (ints, or k / total floats with normalize_hist)."""
    if max_window != 64:
        raise NotImplementedError(f'max_window={max_window}: only the 64-frame windows the pitch alignment uses are implemented')
    _, c = histogram([input_f], method, [float(scale_factor)], counts=True)
    c = c.cpu().numpy().astype(np.int64)
    if normalize_hist:
        return (c.astype(np.float64) / c.sum(1, keepdims=True).astype(np.float64)).tolist()
    return c.tolist()


def hist_dist(hist_a, hist_b):
    """cal_hist_dist: float32 [T1, T2] on hist_a's device."""
    device = device_of(hist_a, hist_b)
    a = as_tensor(hist_a).to(device=device, dtype=torch.float32).contiguous()
    b = as_tensor(hist_b).to(device=device, dtype=torch.float32).contiguous()
    if a.dim() != 2 or b.dim() != 2 or a.shape[1] != BINS or b.shape[1] != BINS:
        raise ValueError(f'histograms must be [T, {BINS}], got {tuple(a.shape)} and {tuple(b.shape)}')
    dist = torch.empty(a.shape[0], b.shape[0], dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        _check(_native.lib().svb_sadtw_cost(_vp(a), a.shape[0], _vp(b), b.shape[0], _vp(dist), _native.current_stream_ptr(device)),
               'sadtw_cost')
    home = hist_a.device if torch.is_tensor(hist_a) else torch.device('cpu')
    return dist.to(home)


def shape_dist(src, tgt, src_len, tgt_len, method):
    """cal_shape_dist: [1, S, T] float32 (the amateur histogram at scale 1, the professional one at tgt_len / src_len)."""
    hs = histogram([src], method)
    ht = histogram([tgt], method, [tgt_len / src_len])
    d = hist_dist(hs, ht)
    return d.unsqueeze(0).to(src.device if torch.is_tensor(src) else torch.device('cpu'))


def dtw(costs, alignment=True, matrix=False):
    """time_warp / align_from_distances on a [rows, cols] float32 or float64 cost: (alignment int64 [rows] or None, DTW value at
    the last cell, DTW matrix or None), device tensors."""
    device = device_of(costs)
    c = as_tensor(costs)
    if c.dim() != 2:
        raise ValueError(f'a cost matrix is [rows, cols], got {tuple(c.shape)}')
    if c.dtype not in DTYPES:
        raise TypeError(f'a cost matrix must be float32 or float64, got {c.dtype}')
    c = c.to(device).contiguous()
    R, C = c.shape
    lib = _native.lib()
    ws_bytes = lib.svb_dtw_workspace_bytes(DTYPES[c.dtype], R, C)
    if ws_bytes < 0:
        raise ValueError(f'time_warp: unsupported cost shape {tuple(c.shape)} (min(rows, cols) <= 8192)')
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    al = torch.empty(R, dtype=torch.int64, device=device) if alignment else None
    pc = torch.empty(1, dtype=c.dtype, device=device)
    full = torch.empty_like(c) if matrix else None
    with torch.cuda.device(device):
        _check(lib.svb_dtw_align(_vp(c), DTYPES[c.dtype], R, C, _vp(ws), ws_bytes, _vp(al), _vp(pc), _vp(full),
                                 _native.current_stream_ptr(device)), 'dtw_align')
    return al, pc, full


def align_one(src, tgt, input, method):
    """SADTW / EHSADTW(src, tgt, input) -> (input[alignment], alignment as a list)."""
    alignment = align_batch([src], [tgt], method).alignment.cpu().tolist()
    return input[alignment], alignment


def dtw_align_batch(srcs, tgts, inputs, srcs_lens, tgt_lens, method):
    """DTW_align: every pair of the padded batch in one launch sequence, the histograms over the whole padded rows and the
    professional scale factor tgt_len / src_len, as the reference does."""
    B = len(srcs)
    sl = [int(x) for x in (srcs_lens if srcs_lens is not None else [srcs[b].shape[0] for b in range(B)])]
    tl = [int(x) for x in (tgt_lens if tgt_lens is not None else [tgts[b].shape[0] for b in range(B)])]
    r = align_batch([srcs[b] for b in range(B)], [tgts[b] for b in range(B)], method, scales=[t / s for s, t in zip(sl, tl)])
    return torch.stack([inputs[b][a.tolist()] for b, a in enumerate(r.split())], dim=0)


def align_pitch(src_f0s, tgt_f0s, method='EHSADTW'):
    """Batched pitch alignment for a binarizer: the a2p alignment of every (amateur, professional) pair, as host int64 arrays of
    the professional lengths (what binarize_para.get_pitch_align stores per item)."""
    return align_batch(list(src_f0s), list(tgt_f0s), method).split()


def a2p_alignment_batch(amateur_f0, prof_f0, amateur_len, prof_len, method='EHSADTW'):
    """The [B, T_prof] int64 device tensor MleSVBVAE.forward takes as a2p_alignment, from padded f0 batches [B, T_ama] / [B, T_prof]
    and the true lengths: pair b aligns amateur_f0[b, :amateur_len[b]] with prof_f0[b, :prof_len[b]], then MultiSpkEmbDataset's rule
    (alignment[:prof_len].clip(max=amateur_len - 1)) and collate_1d's zero padding up to T_prof = prof_f0.shape[1]."""
    a, p = as_tensor(amateur_f0), as_tensor(prof_f0)
    if a.dim() != 2 or p.dim() != 2 or a.shape[0] != p.shape[0]:
        raise ValueError(f'amateur_f0 / prof_f0 must be [B, T], got {tuple(a.shape)} and {tuple(p.shape)}')
    B, Tp = p.shape
    la = [int(x) for x in as_tensor(amateur_len).reshape(-1).tolist()]
    lp = [int(x) for x in as_tensor(prof_len).reshape(-1).tolist()]
    if len(la) != B or len(lp) != B:
        raise ValueError(f'{B} pairs but {len(la)} / {len(lp)} lengths')
    if max(lp) > Tp or max(la) > a.shape[1]:
        raise ValueError('a length exceeds the padded f0 batch')
    device = device_of(amateur_f0, prof_f0)
    r = align_batch([a[b, :la[b]] for b in range(B)], [p[b, :lp[b]] for b in range(B)], method)
    lp_t = torch.tensor(lp, device=device)
    cap = torch.repeat_interleave(torch.tensor(la, device=device) - 1, lp_t)
    out = torch.zeros(B, Tp, dtype=torch.int64, device=device)
    out[torch.arange(Tp, device=device)[None, :] < lp_t[:, None]] = torch.minimum(r.alignment, cap)
    return out


# ---- baseline alignments (LoNDTW, NaiveDTW, ZMNaiveDTW, NNaiveDTW, NInterpo) ---------------------------------------------------

def _baseline_inputs(xs, what, method):
    """Host-side checks of one side of a batch, before any device is looked for: 1-D f0 ([S] or [S, 1]) for every method but
    NaiveDTW, which takes [S, H] features ([S] is [S, 1]); float32 or float64, one type, at least 2 frames."""
    ts = []
    for x in xs:
        t = as_tensor(x)
        if method == 'NaiveDTW':
            t = t[:, None] if t.dim() == 1 else t
            if t.dim() != 2:
                raise ValueError(f'NaiveDTW features must be [S, H], got {tuple(t.shape)}')
        else:
            t = t[:, 0] if t.dim() == 2 and t.shape[1] == 1 else t
            if t.dim() != 1:
                raise ValueError(f'an f0 contour must be [S] or [S, 1], got {tuple(t.shape)}')
        if t.dtype not in DTYPES:
            raise TypeError(f'{what} input must be float32 or float64, got {t.dtype}')
        ts.append(t)
    if len({t.dtype for t in ts}) > 1:
        raise TypeError(f'{what} inputs mix float32 and float64; a batch runs in one type')
    if len({tuple(t.shape[1:]) for t in ts}) > 1:
        raise ValueError(f'{what} features of different widths in one batch')
    if min(t.shape[0] for t in ts) < 2:
        raise ValueError(f'{what} sequence of {min(t.shape[0] for t in ts)} frames: at least 2 are needed')
    return ts


def _baseline_prepare(srcs, tgts, method):
    if method not in BASELINES:
        raise ValueError(f'method must be one of {sorted(BASELINES)}, got {method!r}')
    if len(srcs) != len(tgts) or len(srcs) == 0:
        raise ValueError(f'{len(srcs)} amateur and {len(tgts)} professional sequences')
    a = _baseline_inputs(srcs, 'amateur', method)
    b = _baseline_inputs(tgts, 'professional', method)
    if a[0].dtype != b[0].dtype:
        raise TypeError('amateur and professional inputs must have the same type')
    if a[0].shape[1:] != b[0].shape[1:]:
        raise ValueError(f'amateur features {tuple(a[0].shape[1:])} but professional ones {tuple(b[0].shape[1:])}')
    device = device_of(*srcs, *tgts)
    src = torch.cat([t.to(device) for t in a]).contiguous()
    tgt = torch.cat([t.to(device) for t in b]).contiguous()
    if method != 'NInterpo':
        _check_finite(src)
        _check_finite(tgt)
    S, T = [int(t.shape[0]) for t in a], [int(t.shape[0]) for t in b]
    H = int(a[0].shape[1]) if method == 'NaiveDTW' else 1
    return src, tgt, S, T, H, device


def baseline_batch(srcs, tgts, method, stage_ms=False):
    """A baseline alignment of n pairs in one launch sequence: the method's cost kernel writes the skewed cost, then the DTW and
    backtrack kernels of the shape-aware path run unchanged (NInterpo: the nearest-neighbour index map alone).  path_cost is in
    the input's type (None for NInterpo); stage_ms: (features, cost, dtw, backtrack) CUDA-event times."""
    src, tgt, S, T, H, device = _baseline_prepare(srcs, tgts, method)
    n, lib, dt = len(S), _native.lib(), src.dtype
    s_arr, s_p = _i32(S)
    t_arr, t_p = _i32(T)
    ws_bytes = _check(lib.svb_dtw_baselines_workspace_bytes(BASELINES[method], DTYPES[dt], n, s_p, t_p), 'dtw_baselines_workspace_bytes')
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    out = torch.empty(int(t_arr.sum()), dtype=torch.int64, device=device)
    pc = torch.empty(n, dtype=dt, device=device) if method != 'NInterpo' else None
    ms = (ctypes.c_float * 4)() if stage_ms else None
    with torch.cuda.device(device):
        _check(lib.svb_dtw_baselines_align(_vp(src), _vp(tgt), DTYPES[dt], BASELINES[method], n, s_p, t_p, H, _vp(ws), ws_bytes,
                                           _vp(out), _vp(pc), ms, _native.current_stream_ptr(device)), 'dtw_baselines_align')
    return AlignResult(alignment=out, offsets=np.concatenate([[0], np.cumsum(T)]).astype(np.int64), path_cost=pc,
                       stage_ms=tuple(ms) if stage_ms else None, src_len=S, tgt_len=T, workspace=None, sections=None)


def baseline_costs(srcs, tgts, method):
    """The cost kernel alone: per pair the cdist matrix [S_p, T_p] in the input's type, device tensors (views of one buffer)."""
    if method == 'NInterpo':
        raise ValueError('NInterpo has no cost matrix')
    src, tgt, S, T, H, device = _baseline_prepare(srcs, tgts, method)
    n, lib, dt = len(S), _native.lib(), src.dtype
    s_arr, s_p = _i32(S)
    t_arr, t_p = _i32(T)
    ws_bytes = _check(lib.svb_dtw_baselines_workspace_bytes(BASELINES[method], DTYPES[dt], n, s_p, t_p), 'dtw_baselines_workspace_bytes')
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    cells = [s * t for s, t in zip(S, T)]
    out = torch.empty(sum(cells), dtype=dt, device=device)
    with torch.cuda.device(device):
        _check(lib.svb_dtw_baselines_cost(_vp(src), _vp(tgt), DTYPES[dt], BASELINES[method], n, s_p, t_p, H, _vp(ws), ws_bytes,
                                          _vp(out), _native.current_stream_ptr(device)), 'dtw_baselines_cost')
    return [c.view(s, t) for c, s, t in zip(torch.split(out, cells), S, T)]


def alignment_accuracy(alignments, amateur_mel2ph, prof_mel2ph):
    """The paper's alignment accuracy per pair, job()'s (prof_mel2ph == amateur_mel2ph[alignment]).sum() / (prof_mel2ph != 0).sum(),
    for n pairs at once on the device: alignments (an AlignResult, or n int sequences of the professional lengths), the amateur
    and professional mel2ph tracks (n each).  Returns a float64 numpy array [n]."""
    if isinstance(alignments, AlignResult):
        alignments = [alignments.alignment[alignments.offsets[p]:alignments.offsets[p + 1]] for p in range(len(alignments.offsets) - 1)]
    n = len(alignments)
    if n == 0 or len(amateur_mel2ph) != n or len(prof_mel2ph) != n:
        raise ValueError(f'{n} alignments, {len(amateur_mel2ph)} amateur and {len(prof_mel2ph)} professional mel2ph tracks')
    al = [as_tensor(a).reshape(-1) for a in alignments]
    am = [as_tensor(m).reshape(-1) for m in amateur_mel2ph]
    pm = [as_tensor(m).reshape(-1) for m in prof_mel2ph]
    for p in range(n):
        if al[p].shape[0] != pm[p].shape[0]:
            raise ValueError(f'pair {p}: an alignment of {al[p].shape[0]} frames for {pm[p].shape[0]} professional frames')
        if al[p].dtype.is_floating_point or al[p].dtype == torch.bool:
            raise TypeError(f'pair {p}: alignment indices must be integers, got {al[p].dtype}')
    device = device_of(*alignments, *amateur_mel2ph, *prof_mel2ph)
    S = torch.tensor([m.shape[0] for m in am], device=device)
    T = torch.tensor([m.shape[0] for m in pm], device=device)
    pair = torch.repeat_interleave(torch.arange(n, device=device), T)
    idx = torch.cat([a.to(device, torch.int64) for a in al])
    if bool(((idx < 0) | (idx >= S[pair])).any()):
        raise ValueError('an alignment index is outside its amateur track')
    first = torch.cumsum(S, 0) - S
    ama = torch.cat([m.to(device) for m in am])[idx + first[pair]]
    prof = torch.cat([m.to(device) for m in pm])
    hit = torch.zeros(n, dtype=torch.float64, device=device).index_add_(0, pair, (prof == ama).double())
    voiced = torch.zeros(n, dtype=torch.float64, device=device).index_add_(0, pair, (prof != 0).double())
    return (hit / voiced).cpu().numpy()

"""Whole songs in segments the acoustic model takes: ``plan_song`` cuts a professional take into overlapping segments of at most
``segment_frames`` frames, each with the amateur slice its a2p alignment reads, and ``stitch_mels`` joins the segments' a2p mels
into one mel of the whole take with a linear cross-fade over each overlap.  Host logic on per-frame arrays, no model."""
import numpy as np
import torch

MIN_FRAMES = 60                 # the shortest clip the acoustic model takes (check_frames at frames_multiple 4)


def _fail(name, frame, why):
    raise ValueError(f'{name}: cannot plan the segments at professional frame {frame}: {why}')


def segment_sizes(hp, segment_frames=None, overlap_frames=64, name='song'):
    """(segment_frames, overlap_frames) checked: segments a multiple of frames_multiple in [60, max_frames] (default
    max_frames), overlaps a multiple of frames_multiple in [0, segment_frames / 2].  ValueError naming ``name`` otherwise."""
    fm, mx = int(hp['frames_multiple']), int(hp['max_frames'])
    seg = mx if segment_frames is None else int(segment_frames)
    ov = int(overlap_frames)
    lmin = -(-MIN_FRAMES // fm) * fm
    if seg % fm or not lmin <= seg <= mx:
        raise ValueError(f'{name}: segment_frames = {seg} must be a multiple of frames_multiple = {fm} in [{lmin}, max_frames = {mx}]')
    if ov % fm or not 0 <= ov <= seg // 2:
        raise ValueError(f'{name}: overlap_frames = {ov} must be a multiple of frames_multiple = {fm} in [0, segment_frames / 2]')
    return seg, ov


def plan_song(Tp, Ta, a2p, prof_uv, hp, segment_frames=None, overlap_frames=64, name='song'):
    """Segments (s, e, a_lo, a_hi) of a song whose cropped takes have Tp professional and Ta amateur frames (multiples of
    frames_multiple).  ``a2p``: the amateur frame of each professional frame (clip_alignment's rule: values in [0, Ta));
    ``prof_uv``: the professional unvoiced flags.

    - The professional ranges [s, e) cover [0, Tp) in order and consecutive ones overlap by exactly ``overlap_frames``; every
      bound is a multiple of frames_multiple and every length is in [60, segment_frames] (default max_frames).
    - The amateur range [a_lo, a_hi) is the smallest frames_multiple-aligned slice holding a2p[s:e], widened to 60 frames when
      shorter; it is at most max_frames long, and a segment ends earlier when its amateur span would be longer.
    - A cut prefers the unvoiced: the window is [s, latest allowed end]; among the allowed ends in its last quarter, the one whose
      overlap [e - overlap, e) holds the most unvoiced professional frames, the latest on a tie.
    - A song with Tp <= segment_frames and Ta <= max_frames is one segment, the whole cropped pair: (0, Tp, 0, Ta).

    A pair that cannot be planned raises ValueError naming ``name`` and the professional frame where planning failed."""
    fm, mx = int(hp['frames_multiple']), int(hp['max_frames'])
    seg, ov = segment_sizes(hp, segment_frames, overlap_frames, name)
    lmin = -(-MIN_FRAMES // fm) * fm
    Tp, Ta = int(Tp), int(Ta)
    if Tp % fm or Ta % fm:
        raise ValueError(f'{name}: {Tp} professional and {Ta} amateur frames are not cropped to a multiple of {fm}')
    if Tp < lmin or Ta < lmin:
        _fail(name, 0, f'the cropped takes have {Tp} professional and {Ta} amateur frames, fewer than {lmin}')
    a2p = np.asarray(a2p, dtype=np.int64).reshape(-1)
    uv = np.asarray(prof_uv).reshape(-1)
    if len(a2p) < Tp or len(uv) < Tp:
        raise ValueError(f'{name}: {len(a2p)} alignment entries and {len(uv)} unvoiced flags for {Tp} professional frames')
    a2p, uv = a2p[:Tp], uv[:Tp] > 0
    if a2p.min() < 0 or a2p.max() >= Ta:
        raise ValueError(f'{name}: an alignment entry lies outside the {Ta} amateur frames')
    if Tp <= seg and Ta <= mx:
        return [(0, Tp, 0, Ta)]
    least = max(lmin, 2 * ov)         # a segment also holds its overlaps with both neighbours whole
    unv = np.concatenate([[0], np.cumsum(uv)])
    plan, s = [], 0
    while True:
        top = min(s + seg, Tp)
        lo_run = np.minimum.accumulate(a2p[s:top])
        hi_run = np.maximum.accumulate(a2p[s:top])

        def span(e):
            lo = int(lo_run[e - s - 1]) // fm * fm
            hi = -(-(int(hi_run[e - s - 1]) + 1) // fm) * fm
            hi = min(Ta, max(hi, lo + lmin))
            return min(lo, hi - lmin), hi

        def fits(e):
            lo, hi = span(e)
            return hi - lo <= mx

        if top == Tp and fits(Tp):
            plan.append((s, Tp) + span(Tp))
            return plan
        first, last = s + least, min(top, Tp - least + ov, Tp - fm) // fm * fm
        ends = [e for e in range(first, last + 1, fm) if fits(e)]
        if not ends:
            _fail(name, s, f'every segment end in [{first}, {last}] gives an amateur span over max_frames = {mx}' if first <= last
                  else f'{Tp - s} frames remain, too few for a segment and the one after it')
        e_max = ends[-1]
        quarter = [e for e in ends if e >= e_max - (e_max - s) // 4]
        score = [unv[e] - unv[e - ov] for e in quarter]
        best = max(range(len(quarter)), key=lambda q: (score[q], quarter[q]))
        e = quarter[best]
        plan.append((s, e) + span(e))
        s = e - ov


def stitch_weights(overlap_frames):
    """The cross-fade weight of the next segment at overlap frame t: (t + 0.5) / overlap_frames, float32 (host)."""
    return (np.arange(overlap_frames, dtype=np.float32) + np.float32(0.5)) / np.float32(overlap_frames)


def stitch_mels(mels, plan, overlap_frames=64):
    """One [Tp, n_mel] float32 mel from the segments' mels (mels[k]: at least e_k - s_k rows, the segment's frames first), on
    their device: a segment's frames outside the overlaps as they are, and in the overlap [s_{k+1}, e_k) the float32
    (1 - w) * m_k + w * m_{k+1} with w = stitch_weights(overlap_frames)[t - s_{k+1}]."""
    Tp, ov = plan[-1][1], int(overlap_frames)
    out = mels[0].new_empty(Tp, mels[0].shape[1])
    n = len(plan)
    for k, (s, e, _, _) in enumerate(plan):
        a, b = s + (ov if k > 0 else 0), e - (ov if k + 1 < n else 0)
        out[a:b] = mels[k][a - s:b - s]
    if n > 1 and ov > 0:
        w = torch.from_numpy(stitch_weights(ov)).to(out.device)[:, None]
        u = torch.from_numpy(np.float32(1) - stitch_weights(ov)).to(out.device)[:, None]
        for k in range(n - 1):
            s0, s1 = plan[k][0], plan[k + 1][0]
            out[s1:s1 + ov] = torch.add(torch.mul(u, mels[k][s1 - s0:s1 - s0 + ov]), torch.mul(w, mels[k + 1][:ov]))
    return out

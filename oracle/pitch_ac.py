"""ORACLE (test infrastructure only; see oracle/__init__.py): the autocorrelation pitch tracker behind ``get_pitch``, in float64
numpy.  The CUDA path (csrc/pitch_ac.cu) implements the same text and is compared with this file.

This is Boersma's (1993) autocorrelation method as Praat's ``To Pitch (ac)`` describes it, with the settings of the reference's
``get_pitch`` call (data_gen/tts/data_gen_utils.py:150-184): time step hop / sr, pitch floor 80 Hz, ceiling 750 Hz, voicing threshold
0.6, and Praat's documented defaults for the rest: 15 candidates, a Hann window, silence threshold 0.03, octave cost 0.01, octave-jump
cost 0.35, voiced / unvoiced cost 0.14.  Neither Praat nor its source is used here, so every choice is fixed below; agreement with
parselmouth has not been measured.

Grid.  The clip is x[0..N), sample k at time (k + 0.5) / sr, D = N / sr.
  W = 3 / floor seconds, L = 2 * floor(W * sr / 2) + 1 samples (827 at 22050 Hz), h = (L - 1) / 2.
  n = floor((D - W) / dt) + 1 frames (all in float64); n < 1 raises ValueError naming the clip.
  Frame j is centred at t_j = D / 2 - (n - 1) dt / 2 + j dt, on sample round(t_j sr - 0.5) with ties rounded up, which is exactly
  c_j = floor((N - (n - 1) hop) / 2) + j hop (dt sr = hop).  Its window is samples c_j - h .. c_j + h, zero outside the clip.
Per frame.
  Subtract the window's plain mean (over all L values); localPeak = max |x - mean|; multiply by w[k] = 0.5 - 0.5 cos(2 pi (k + 1) /
  (L + 1)); r_a(tau) = sum_k x'[k] x'[k + tau] for tau = 0 .. tau_max + 1, tau_max = ceil(sr / floor);
  r(tau) = (r_a(tau) / r_a(0)) / (r_w(tau) / r_w(0)) with r_w the window's own autocorrelation.
Voiced candidates.
  Every integer tau in 1 .. tau_max with r(tau - 1) < r(tau) >= r(tau + 1) is a peak, refined by the parabola through its three
  points: d = 0.5 (r[-1] - r[+1]) / (r[-1] - 2 r[0] + r[+1]), lag = tau + d, height = r[0] - 0.25 (r[-1] - r[+1]) d.  A peak is kept
  if sr / ceiling <= lag <= sr / floor and height > 0.5 voicing_threshold; its strength is height - octave_cost log2(floor lag / sr)
  and its frequency sr / lag.  At most 14 are kept, strongest first, ties to the smaller lag.  r_a(0) == 0: no voiced candidates.
Unvoiced candidate (index 0): strength VT + max(0, 2 - (localPeak / globalPeak) / (ST / (1 + VT))), globalPeak = max |x - mean(x)|
  over the clip.  globalPeak == 0: every frame has only this candidate.
Path.  Maximise the summed strengths minus transition costs, both costs scaled by c = 0.01 / dt: unvoiced -> unvoiced 0, voiced <->
  unvoiced voiced_unvoiced_cost c, voiced -> voiced octave_jump_cost c |log2(f_prev / f_cur)|.  Ties go to the lower candidate index,
  in the recursion and at the last frame.  The output is the path's frequency, 0 where it is unvoiced.
Placement (``place``), the reference's get_pitch rule taken literally.  The clip is the wav ``wav2spec`` returns (len(mel) hop samples).
  lpad = 2 pad_size zero frames go in front (pad_size 4 at hop 128, 2 at hop 256; other hops raise), then the result is cut to
  len(mel) or extended with its last value.  With this grid the reference's ``np.pad`` would get rpad = -2 at hop 128 and raise
  (its comment says "new versions" of the libraries do this); the cut replaces it.  So f0[i] describes the audio about 4.5 frames
  (hop 128) before mel frame i, as the reference's padding intends.
"""
import math

import numpy as np

DEFAULTS = dict(floor=80.0, ceiling=750.0, voicing_threshold=0.6, silence_threshold=0.03, octave_cost=0.01,
                octave_jump_cost=0.35, voiced_unvoiced_cost=0.14)
MAX_CAND = 15          # the unvoiced candidate + 14 voiced ones


def pad_size(hop):
    if hop == 128:
        return 4
    if hop == 256:
        return 2
    raise ValueError(f'get_pitch places f0 for hop 128 or 256 only, not hop {hop} (the reference asserts the same)')


def grid(N, sr, dt, floor=80.0, name='clip'):
    """(n frames, L window samples, c_0 first centre sample, tau_max)."""
    D, W = N / sr, 3.0 / floor
    L = 2 * int(math.floor(W * sr / 2.0)) + 1
    n = int(math.floor((D - W) / dt)) + 1
    if n < 1:
        raise ValueError(f'{name}: {N} samples ({D:.4f} s) is shorter than one pitch window ({W:.4f} s at floor {floor} Hz)')
    hop = int(round(dt * sr))
    c0 = (N - (n - 1) * hop) // 2
    return n, L, c0, int(math.ceil(sr / floor))


def window(L):
    k = np.arange(L, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * (k + 1) / (L + 1))


def lag_autocorr(x, nlags):
    """r[..., tau] = sum_k x[..., k] x[..., k + tau], tau = 0 .. nlags - 1 (float64, via a zero-padded FFT)."""
    L = x.shape[-1]
    nfft = 1 << int(math.ceil(math.log2(L + nlags)))
    X = np.fft.rfft(x, nfft)
    return np.fft.irfft(X * np.conj(X), nfft)[..., :nlags]


def normalised_autocorr(x, sr, dt, floor=80.0, name='clip'):
    """(r [n, tau_max + 2], localPeak [n], r_a(0) [n], globalPeak) of clip x."""
    x = np.asarray(x, np.float64)
    N = len(x)
    n, L, c0, tau_max = grid(N, sr, dt, floor, name)
    h, hop = (L - 1) // 2, int(round(dt * sr))
    idx = c0 - h + np.arange(n)[:, None] * hop + np.arange(L)[None, :]
    fr = np.where((idx >= 0) & (idx < N), x[np.clip(idx, 0, max(N - 1, 0))], 0.0)
    fr = fr - fr.mean(axis=1, keepdims=True)
    local_peak = np.abs(fr).max(axis=1)
    w = window(L)
    ra = lag_autocorr(fr * w, tau_max + 2)
    rw = lag_autocorr(w, tau_max + 2)
    with np.errstate(invalid='ignore', divide='ignore'):
        r = (ra / ra[:, :1]) / (rw / rw[0])
    r[ra[:, 0] == 0] = 0.0
    global_peak = float(np.abs(x - x.mean()).max()) if N else 0.0
    return r, local_peak, ra[:, 0], global_peak


def peaks(r_row, sr, p):
    """All refined peaks of one frame that pass the lag and height tests: list of (strength, lag, height), unsorted."""
    tau_max = len(r_row) - 2
    t = np.arange(1, tau_max + 1)
    a, b, c = r_row[t - 1], r_row[t], r_row[t + 1]
    m = (a < b) & (b >= c)
    t, a, b, c = t[m], a[m], b[m], c[m]
    d = 0.5 * (a - c) / (a - 2 * b + c)
    lag = t + d
    height = b - 0.25 * (a - c) * d
    keep = (lag >= sr / p['ceiling']) & (lag <= sr / p['floor']) & (height > 0.5 * p['voicing_threshold'])
    lag, height = lag[keep], height[keep]
    strength = height - p['octave_cost'] * np.log2(p['floor'] * lag / sr)
    return strength, lag, height


def candidates_from_r(r, local_peak, ra0, global_peak, sr, **kw):
    """freq [n, 15], strength [n, 15], count [n] (index 0 = unvoiced, freq 0; unused slots freq 0, strength -inf)."""
    p = dict(DEFAULTS, **kw)
    n = r.shape[0]
    freq = np.zeros((n, MAX_CAND))
    strength = np.full((n, MAX_CAND), -np.inf)
    count = np.ones(n, np.int64)
    VT, ST = p['voicing_threshold'], p['silence_threshold']
    for j in range(n):
        if global_peak == 0:
            strength[j, 0] = VT + 2.0
            continue
        strength[j, 0] = VT + max(0.0, 2.0 - (local_peak[j] / global_peak) / (ST / (1.0 + VT)))
        if ra0[j] == 0:
            continue
        s, lag, _ = peaks(r[j], sr, p)
        order = np.lexsort((lag, -s))[:MAX_CAND - 1]
        k = len(order)
        freq[j, 1:1 + k] = sr / lag[order]
        strength[j, 1:1 + k] = s[order]
        count[j] = 1 + k
    return freq, strength, count


def candidates(x, sr, hop, name='clip', **kw):
    p = dict(DEFAULTS, **kw)
    dt = hop / sr
    r, lp, ra0, gp = normalised_autocorr(x, sr, dt, p['floor'], name)
    return candidates_from_r(r, lp, ra0, gp, sr, **kw)


def _trans(f_prev, f_cur, c, p):
    """cost [K_prev, K_cur] of every transition."""
    vp, vc = f_prev[:, None] > 0, f_cur[None, :] > 0
    with np.errstate(divide='ignore', invalid='ignore'):
        oj = p['octave_jump_cost'] * c * np.abs(np.log2(f_prev[:, None] / f_cur[None, :]))
    return np.where(vp & vc, oj, np.where(vp ^ vc, p['voiced_unvoiced_cost'] * c, 0.0))


def viterbi(freq, strength, count, dt, margins=False, **kw):
    """Path frequencies [n] (0 = unvoiced); with ``margins`` also, per frame, the gap between the best path score and the best
    score of a path through another candidate of that frame (a tie at a frame shows as a margin near 0)."""
    p = dict(DEFAULTS, **kw)
    c = 0.01 / dt
    n = freq.shape[0]
    delta = np.full((n, MAX_CAND), -np.inf)
    back = np.zeros((n, MAX_CAND), np.int64)
    delta[0, :count[0]] = strength[0, :count[0]]
    for j in range(1, n):
        kp, kc = count[j - 1], count[j]
        sc = delta[j - 1, :kp, None] - _trans(freq[j - 1, :kp], freq[j, :kc], c, p)
        back[j, :kc] = np.argmax(sc, axis=0)                     # first maximum: the lower index wins a tie
        delta[j, :kc] = sc[back[j, :kc], np.arange(kc)] + strength[j, :kc]
    path = np.zeros(n, np.int64)
    path[-1] = int(np.argmax(delta[-1, :count[-1]]))
    for j in range(n - 1, 0, -1):
        path[j - 1] = back[j, path[j]]
    f0 = freq[np.arange(n), path]
    if not margins:
        return f0
    beta = np.zeros((n, MAX_CAND))
    for j in range(n - 2, -1, -1):
        kc, kn = count[j], count[j + 1]
        sc = -_trans(freq[j, :kc], freq[j + 1, :kn], c, p) + (strength[j + 1, :kn] + beta[j + 1, :kn])[None, :]
        beta[j, :kc] = sc.max(axis=1)
    through = delta + beta
    best = through.max(axis=1)
    marg = np.full(n, np.inf)
    for j in range(n):
        others = np.delete(through[j, :count[j]], path[j])
        if len(others):
            marg[j] = best[j] - others.max()
    return f0, marg


def track(x, sr, hop, name='clip', margins=False, **kw):
    """f0 [n] in Hz on the analysis grid (no placement)."""
    p = dict(DEFAULTS, **kw)
    dt = hop / sr
    freq, strength, count = candidates(x, sr, hop, name, **kw)
    return viterbi(freq, strength, count, dt, margins, **p)


def place(f0, n_mel, hop):
    """The reference's get_pitch placement: lpad zero frames in front, then cut to n_mel or extend with the last value."""
    lpad = 2 * pad_size(hop)
    f = np.concatenate([np.zeros(lpad), np.asarray(f0, np.float64)])
    if len(f) < n_mel:
        f = np.concatenate([f, np.full(n_mel - len(f), f[-1])])
    return f[:n_mel]


def get_pitch(wav, n_mel, sr, hop, name='clip', **kw):
    """(placed f0 [n_mel], pitch ids [n_mel]) of the wav wav2spec returned."""
    from neuralsvb_b200.utils.pitch_utils import f0_to_coarse
    pad_size(hop)
    f0 = place(track(wav, sr, hop, name, **kw), n_mel, hop)
    return f0, f0_to_coarse(f0)

"""The float64 pitch-tracker oracle (oracle/pitch_ac.py) on signals with known f0: accuracy on write_svb_raw-style takes, silence and
noise, the placement rule, tie breaking and the refused inputs.  CPU only."""
import numpy as np
import pytest

from neuralsvb_b200.utils import synthetic as S
from oracle import pitch_ac as P

SR, HOP = 22050, 128
FPS = SR / HOP


def frame_truth(n_samples, true_f0):
    """True f0 at every analysis frame's centre sample, and the frames at least 4 frames from a voicing boundary."""
    n, L, c0, _ = P.grid(n_samples, SR, HOP / SR)
    tv = true_f0[c0 + np.arange(n) * HOP]
    v = tv > 0
    ok = np.ones(n, bool)
    for e in np.nonzero(np.diff(v.astype(int)))[0]:
        ok[max(0, e - 3):e + 5] = False
    return tv, ok


def score(pairs):
    """(gross error fraction, median |cents|, voicing error fraction) over (estimate, truth, mask) triples."""
    gross = voiced = verr = total = 0
    cents = []
    for est, tv, ok in pairs:
        both = ok & (tv > 0) & (est > 0)
        rel = np.abs(est[both] / tv[both] - 1)
        gross += int((rel > 0.2).sum())
        voiced += int((ok & (tv > 0)).sum())
        verr += int((ok & ((tv > 0) != (est > 0))).sum())
        total += int(ok.sum())
        cents += list(np.abs(1200 * np.log2(est[both] / tv[both])))
    return gross / voiced, float(np.median(cents)), verr / total


def test_accuracy_on_sung_takes():
    pairs = []
    for seed in range(4):
        fa, fp = S.make_f0_pair(seed, int(2.5 * FPS), int(2.8 * FPS), FPS)
        for f, shift in ((fa, 5), (fp, -4)):
            wav, truth = S.make_sung_take(f * 2 ** (shift / 12), seed, SR, HOP)
            tv, ok = frame_truth(len(wav), truth)
            pairs.append((P.track(wav, SR, HOP), tv, ok))
    gross, cents, verr = score(pairs)
    assert gross < 0.01, gross
    assert cents < 10.0, cents
    assert verr < 0.05, verr


def test_silence_and_noise_are_unvoiced():
    assert (P.track(np.zeros(SR), SR, HOP) == 0).all()
    rs = np.random.RandomState(3)
    assert (P.track(0.01 * rs.standard_normal(SR), SR, HOP) == 0).all()
    assert (P.track(1e-4 * rs.standard_normal(SR), SR, HOP) == 0).all()


def test_placement_of_a_tone_onset():
    """A 220 Hz tone starting at sample s: the first voiced frame of the placed f0 sits where the grid puts the first window that
    is mostly tone, within one frame."""
    T = 400
    N = T * HOP
    for s in (20000, 20000 + 37, 31111):
        x = np.zeros(N)
        k = np.arange(N - s)
        x[s:] = 0.4 * np.sin(2 * np.pi * 220 * k / SR) + 0.1 * np.sin(2 * np.pi * 440 * k / SR)
        f0, pitch = P.get_pitch(x, T, SR, HOP)
        assert f0.shape == (T,) and pitch.shape == (T,)
        n, L, c0, _ = P.grid(N, SR, HOP / SR)
        # the first frame whose centre is past the onset: half its window is tone
        j = int(np.ceil((s - c0) / HOP))
        first = int(np.nonzero(f0)[0][0])
        assert abs(first - (8 + j)) <= 1, (first, 8 + j)
        assert abs(f0[first + 10] - 220) < 2


def test_grid_and_placement_rule():
    n, L, c0, tau_max = P.grid(400 * HOP, SR, HOP / SR)
    assert (L, tau_max, n) == (827, 276, 394)          # 400 mel frames -> 394 analysis frames, 8 in front, cut by 2
    assert c0 == (400 * HOP - 393 * HOP) // 2
    f = P.place(np.arange(1, n + 1, dtype=float), 400, HOP)
    assert (f[:8] == 0).all() and f[8] == 1 and f[-1] == 392 and len(f) == 400
    g = P.place(np.array([5.0, 6.0]), 14, HOP)
    assert g.tolist() == [0] * 8 + [5, 6, 6, 6, 6, 6]   # extended with the last value
    assert P.place(np.array([5.0]), 4, HOP).tolist() == [0] * 4
    assert len(P.place(np.ones(3), 10, 256)) == 10 and (P.place(np.ones(3), 10, 256)[:4] == 0).all()


def test_short_clip_and_hop_are_refused():
    short = 826                                        # less than one 0.0375 s window
    with pytest.raises(ValueError, match='my_clip'):
        P.track(np.zeros(short), SR, HOP, name='my_clip')
    one = 827 + HOP                                    # one window plus one hop: frames exist
    assert len(P.track(np.zeros(one), SR, HOP)) >= 1
    with pytest.raises(ValueError, match='hop'):
        P.get_pitch(np.zeros(SR), 100, SR, 200)
    with pytest.raises(ValueError, match='hop'):
        P.pad_size(64)


def test_candidate_ties_prefer_the_smaller_lag():
    """Two peaks of equal strength: the smaller lag comes first.  And the path takes the lower index on a tie."""
    r = np.zeros(278)
    r[0] = 1
    # two identical symmetric peaks (d = 0): heights 0.8, strengths differ only by the octave cost term unless equal lags
    for t in (100, 200):
        r[t - 1], r[t], r[t + 1] = 0.7, 0.8, 0.7
    s, lag, h = P.peaks(r, SR, P.DEFAULTS)
    assert np.allclose(lag, [100, 200]) and np.allclose(h, 0.8)
    # octave cost favours the smaller lag, so it is first
    freq, strength, count = P.candidates_from_r(r[None], np.array([1.0]), np.array([1.0]), 1.0, SR)
    assert count[0] == 3 and freq[0, 1] > freq[0, 2]
    # exact tie: zero octave cost makes the strengths equal; the smaller lag still comes first
    freq, strength, count = P.candidates_from_r(r[None], np.array([1.0]), np.array([1.0]), 1.0, SR, octave_cost=0.0)
    assert strength[0, 1] == strength[0, 2] and freq[0, 1] > freq[0, 2]
    # path: two frames, two candidates of equal total score -> the lower index
    fr = np.zeros((2, P.MAX_CAND))
    st = np.full((2, P.MAX_CAND), -np.inf)
    fr[:, 1], fr[:, 2] = 200.0, 200.0
    st[:, 0], st[:, 1], st[:, 2] = 0.0, 1.0, 1.0
    f0, marg = P.viterbi(fr, st, np.array([3, 3]), HOP / SR, margins=True)
    assert f0.tolist() == [200.0, 200.0] and marg[0] == 0.0

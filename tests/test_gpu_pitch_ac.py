"""-m gpu: the autocorrelation pitch tracker (csrc/pitch_ac.cu) against the float64 oracle (oracle/pitch_ac.py), and the paired
binarizer end to end.

  * every (sample rate, hop, lpad) of CONFIGS, which between them run both instantiations of the candidate kernel (R = 9 lags per
    lane up to 288 lags, R = 18 above) at their full width, both reference hops and a hop that is not a multiple of 32;
  * ragged batches of clips built at the configuration's rate: sung takes, one with a DC offset and exactly constant stretches,
    the shortest and longest clips with one analysis frame, frame counts 8k and 8k + 1, digital silence, noise, f0 near the floor
    and the ceiling, a tone above the ceiling (more than 14 qualifying peaks) and a full-scale clipped square wave: r(tau) within
    2e-5, candidates within 1e-5 relative (frequency, plus what the r bar moves a flat parabola by) and 2e-5 (strength) at R = 9,
    the bars of BARS at R = 18; an exactly constant window with only the unvoiced candidate and r = 0; the path kernel equal to the
    float64 Viterbi on its own candidates, and its f0 the oracle's candidate on every frame where the oracle's best path is more
    than 1e-4 ahead of the best path through another candidate;
  * every clip bit-identical alone and in the batch, with or without the optional outputs; a clip scaled by 2^20 or 2^-20 gives the
    same candidates and f0 bit for bit; get_pitch equal to get_pitch_batch and to pitch_ac_device;
  * placement for lpad 0 .. beyond len(mel), a 300-clip batch with a 60 s clip, a short workspace refused on the device, and the
    comparison helpers catching corrupted outputs;
  * write_svb_raw -> the binarize CLI -> the dataset on disk (keys, mel / f0 / alignment against the single-clip calls, the stats
    files, the skipped items, the f0 accuracy against the ground truth) -> tasks/run.py trains, resumes and infers on it."""
import collections
import ctypes
import glob
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.data_gen.tts import data_gen_utils as DG
from neuralsvb_b200.utils import synthetic as S
from oracle import pitch_ac as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR, HOP = 22050, 128
FPS = SR / HOP
HP = {'audio_sample_rate': SR, 'hop_size': HOP}

Cfg = collections.namedtuple('Cfg', 'sr hop lpad R')
# R: lags per lane of the candidate kernel this configuration runs (9 while tau_max + 2 <= 288, else 18)
CONFIGS = [
    Cfg(22050, 128, 8, 9),       # the product configuration
    Cfg(22050, 256, 4, 9),       # the other reference hop
    Cfg(22880, 128, 8, 9),       # R = 9 at full width: 288 lags, lane 31's last lag reads the last float of the zero tail
    Cfg(22881, 128, 8, 18),      # the smallest R = 18 case (289 lags)
    Cfg(24000, 128, 8, 18),
    Cfg(44100, 256, 4, 18),      # L = 1653
    Cfg(45920, 256, 4, 18),      # R = 18 at full width (576 lags)
    Cfg(16000, 110, 0, 9),       # a hop that is not a multiple of 32 (or 4), explicit lpad; W * sr is exactly 600 samples
]
CFG_IDS = [f'{c.sr}-{c.hop}-{c.lpad}' for c in CONFIGS]
# (r, candidate frequency relative, candidate strength) per lags-per-lane instantiation.  R = 18 sums up to twice as many fp32 terms
# per lag (L = 1723 at 45920 Hz).  Worst measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, R = 18: r 1.83e-5 (44100 Hz),
# strength 1.25e-5 (45920 Hz); R = 9: r 3.1e-6, strength 2.7e-6.  The R = 18 bars are about 5x the R = 18 worst.
BARS = {9: (2e-5, 1e-5, 2e-5), 18: (1e-4, 1e-5, 6e-5)}


def nlag_of(sr):
    return int(math.ceil(sr / 80.0)) + 2


def hp_of(cfg):
    return {'audio_sample_rate': cfg.sr, 'hop_size': cfg.hop}


def frames_of(N, sr, hop):
    try:
        return P.grid(N, sr, hop / sr)[0]
    except ValueError:
        return 0


def one_frame_bounds(sr, hop):
    """(shortest, longest) clip with exactly one analysis frame, from the oracle's grid."""
    lo = int(3.0 / 80.0 * sr) - 2
    assert frames_of(lo, sr, hop) == 0
    while frames_of(lo, sr, hop) == 0:
        lo += 1
    hi = lo + hop - 4
    while frames_of(hi + 1, sr, hop) == 1:
        hi += 1
    assert frames_of(lo, sr, hop) == 1 == frames_of(hi, sr, hop) and frames_of(hi + 1, sr, hop) == 2
    return lo, hi


def length_with_frames(n, sr, hop):
    N = one_frame_bounds(sr, hop)[0] + (n - 1) * hop + hop // 2
    assert frames_of(N, sr, hop) == n
    return N


def tone(f, seconds, seed, sr=SR):
    rs = np.random.RandomState(seed)
    t = np.arange(int(seconds * sr)) / sr
    f = f * (1 + 0.01 * np.sin(2 * np.pi * 5 * t))
    ph = 2 * np.pi * np.cumsum(f) / sr
    return (0.4 * np.sin(ph) + 0.15 * np.sin(2 * ph) + 0.002 * rs.standard_normal(len(t))).astype(np.float32)


def sung(i, sec, sr, hop):
    fps = sr / hop
    fa, _ = S.make_f0_pair(i, int(sec * fps), int(sec * fps), fps)
    return S.make_sung_take(fa * 2 ** ((3 * i - 4) / 12), i, sr, hop)[0]


def clips(cfg):
    """[(name, float32 wav)] at cfg.sr: about 40 s of audio."""
    sr, hop = cfg.sr, cfg.hop
    out = [(f'sung{i}', sung(i, sec, sr, hop)) for i, sec in enumerate((2.0, 5.3, 12.0, 3.1))]
    L = P.grid(sr, sr, hop / sr)[1]
    lo, hi = one_frame_bounds(sr, hop)
    out.append(('window_plus_hop', tone(220.0, 1.0, 5, sr)[:L + hop]))
    out.append(('one_frame_shortest', tone(180.0, 1.0, 6, sr)[:lo]))
    out.append(('one_frame_longest', tone(310.0, 1.0, 7, sr)[:hi]))
    take = sung(4, 1.0, sr, hop)
    for n in (16, 17, 57):                                                 # 8k and 8k + 1 frames: the last CTA has 8 or 1 warps
        out.append((f'frames{n}', take[:length_with_frames(n, sr, hop)]))
    out.append(('silence', np.zeros(int(2.5 * sr), np.float32)))          # digital silence
    out.append(('noise', (0.05 * np.random.RandomState(9).standard_normal(int(2.2 * sr))).astype(np.float32)))
    out.append(('near_floor', tone(84.0, 3.0, 11, sr)))
    out.append(('near_ceiling', tone(720.0, 2.4, 12, sr)))
    out.append(('above_ceiling', tone(1500.0, 1.0, 13, sr)))               # more than 14 peaks pass: the top-14 selection truncates
    t = np.arange(int(1.0 * sr)) / sr
    out.append(('square', np.clip(4.0 * np.sin(2 * np.pi * 196.0 * t), -1.0, 1.0).astype(np.float32)))
    # DC offset, with gated stretches held at a constant value (longer than a window: some windows are exactly constant)
    dc = sung(5, 3.0, sr, hop) + np.float32(0.1)
    for a, b, v in ((0.4, 0.9, 0.1234567), (1.6, 2.2, -0.6543210), (2.5, 2.56, 0.3)):
        dc[int(a * sr):int(b * sr)] = np.float32(v)
    out.append(('dc_constant', dc.astype(np.float32)))
    return out


@pytest.fixture(scope='module')
def batch(request):
    """One tracker call over clips() at a configuration of CONFIGS: the product one unless a test is parametrised over others."""
    cfg = getattr(request, 'param', CONFIGS[0])
    torch.cuda.set_device(0)
    named = clips(cfg)
    names, ws = [n for n, _ in named], [w for _, w in named]
    lens = np.array([len(w) for w in ws])
    n_mel = lens // cfg.hop + 1
    cat = torch.from_numpy(np.concatenate(ws)).cuda()
    tr = DG.pitch_ac_device(cat, lens, n_mel, hp_of(cfg), want_cand=True, want_r=True, lpad=cfg.lpad)
    torch.cuda.synchronize()
    # the instantiation this configuration runs, so the sweep cannot lose a branch of run()
    assert tr.r.shape[1] == nlag_of(cfg.sr) and (nlag_of(cfg.sr) <= 32 * 9) == (cfg.R == 9), (cfg, tr.r.shape)
    return cfg, names, ws, lens, n_mel, tr


EVERY_CONFIG = pytest.mark.parametrize('batch', CONFIGS, ids=CFG_IDS, indirect=True)


def at_the_other_configurations(test):
    """``test`` (written for the product configuration, which it runs as it stands) at every other configuration of CONFIGS."""
    @pytest.mark.parametrize('batch', CONFIGS[1:], ids=CFG_IDS[1:], indirect=True)
    def run(batch):
        test(batch)
    run.__name__, run.__doc__ = test.__name__ + '_at_the_other_configurations', test.__doc__
    return run


def test_the_sweep_covers_both_candidate_kernels_at_full_width():
    widths = {c.R: [] for c in CONFIGS}
    for c in CONFIGS:
        assert (nlag_of(c.sr) <= 288) == (c.R == 9), c
        widths[c.R].append(nlag_of(c.sr))
    assert max(widths[9]) == 32 * 9 and min(widths[18]) == 32 * 9 + 1 and max(widths[18]) == 32 * 18
    assert {c.hop for c in CONFIGS} >= {128, 256} and any(c.hop % 32 for c in CONFIGS)


def split(tr, lens, n_mel):
    fo = np.concatenate([[0], np.cumsum(tr.frames)])
    oo = np.concatenate([[0], np.cumsum(n_mel)])
    r, cand, cnt, f0 = tr.r.cpu().numpy(), tr.cand.cpu().numpy(), tr.count.cpu().numpy(), tr.f0.cpu().numpy()
    return [(r[fo[c]:fo[c + 1]], cand[fo[c]:fo[c + 1]], cnt[fo[c]:fo[c + 1]], f0[oo[c]:oo[c + 1]]) for c in range(len(lens))]


def oracle_r(w, cfg):
    return P.normalised_autocorr(w, cfg.sr, cfg.hop / cfg.sr)


def r_errors(r, ro, ra0, bar):
    """[(frame, reason)] where the kernel's r(tau) is off: beyond bar on a frame with r_a(0) > 0, not exactly 0 on one without."""
    assert r.shape == ro.shape, (r.shape, ro.shape)
    bad = []
    for j in range(len(r)):
        if ra0[j] > 0:
            e = float(np.abs(r[j] - ro[j]).max())
            if not e < bar:
                bad.append((j, f'r error {e:.3g}'))
        elif (r[j] != 0).any():
            bad.append((j, 'r != 0 on a constant window'))
    return bad


def candidate_errors(cand, cnt, ro, lp, ra0, gp, cfg, bars):
    """(compared frames, total frames, [(frame, reason)], worst frequency error (relative), worst strength error, compared frames
    that no comparison closer than the bars could change) of the kernel's
    candidate lists against the oracle's.  The kernel's list must be in its own strength order (ties to the smaller lag); its voiced
    candidates are matched to the oracle's by frequency, so two candidates whose strengths are closer than the bars may trade
    places.  A peak's frequency may differ by the bar plus what an r error of the r bar moves its parabolic refinement by (much
    more than the bar where the parabola is flat).  A frame whose list hangs on a comparison closer than the r bar is skipped when
    it differs; a frame with r_a(0) = 0 is always compared."""
    rbar, fbar, sbar = bars
    k_near = rbar / 2e-5
    fo, so, co = P.candidates_from_r(ro, lp, ra0, gp, cfg.sr)
    compared, firm, bad = [], [], []
    worst_f = worst_s = 0.0
    for j in range(len(cand)):
        if ra0[j] == 0:
            near = False
        else:
            d = np.abs(np.diff(ro[j]))
            s_all, lag, h = P.peaks(ro[j], cfg.sr, P.DEFAULTS)
            near = (d.min() < 4e-5 * k_near or (np.abs(h - 0.3) < 1e-4 * k_near).any()
                    or (np.abs(lag - cfg.sr / 750) < 1e-3).any() or (np.abs(lag - cfg.sr / 80) < 1e-3).any()
                    or (len(s_all) > 14 and np.sort(s_all)[-14] - np.sort(s_all)[-15] < 1e-4 * k_near))
        if cnt[j] != co[j]:
            if not near:
                bad.append((j, f'count {cnt[j]} != {co[j]}'))
            continue
        k = cnt[j]
        f, s = cand[j, 1:k, 0].astype(np.float64), cand[j, 1:k, 1].astype(np.float64)
        order = (s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (f[:-1] > f[1:]))
        if not order.all() or cand[j, 0, 0] != 0 or (cand[j, k:, 1] != -np.inf).any():
            bad.append((j, f'list out of order {cand[j, :k]}'))
            continue
        ik, io = np.argsort(f), np.argsort(fo[j, 1:k])
        lag = cfg.sr / fo[j, 1:k][io]
        t = np.rint(lag).astype(np.int64)
        a, b, c = ro[j, t - 1], ro[j, t], ro[j, t + 1]
        den = np.abs(a - 2 * b + c)
        ftol = fbar + rbar * (1 / den + 2 * np.abs(a - c) / den ** 2) / lag
        fe = np.abs(f[ik] - fo[j, 1:k][io]) / fo[j, 1:k][io]
        if not (fe <= ftol).all():
            if not near:
                bad.append((j, f'frequencies {f[ik]} != {fo[j, 1:k][io]}'))
            continue
        compared.append(j)
        if not near:
            firm.append(j)
        se = np.abs(np.concatenate([[cand[j, 0, 1] - so[j, 0]], s[ik] - so[j, 1:k][io]]))
        worst_f, worst_s = max(worst_f, float(fe.max(initial=0))), max(worst_s, float(se.max()))
        if not se.max() < sbar:
            bad.append((j, f'strength error {se.max():.3g}'))
    return compared, len(cand), bad, worst_f, worst_s, firm


def place(f0, n_mel, lpad):
    """P.place for any lpad: lpad zero frames in front, then cut to n_mel or extend with the last value."""
    f = np.concatenate([np.zeros(lpad), np.asarray(f0, np.float64)])
    if len(f) < n_mel:
        f = np.concatenate([f, np.full(n_mel - len(f), f[-1])])
    return f[:n_mel]


def same_f0(f0, ref, rtol):
    return ((ref > 0) == (f0 > 0)) & (np.abs(f0 - ref) <= rtol * ref)


def path_errors(f0, fo, marg, n_mel, lpad, margin=1e-4, rtol=5e-4):
    """(frames that differ, [placed frames that differ where the reference path is at least ``margin`` ahead]).  Two refined peaks
    of one frame are at least one lag apart (1.8e-3 relative at the floor), so ``rtol`` 5e-4 asks for the same candidate and
    leaves its frequency to the candidate comparison."""
    placed = place(fo, n_mel, lpad)
    pm = place(marg, n_mel, lpad)
    pm[:lpad] = np.inf
    bad = ~same_f0(f0, placed, rtol)
    return int(bad.sum()), np.nonzero(bad & (pm >= margin))[0]


def test_autocorrelation_and_candidates_match_the_oracle(batch):
    cfg, names, ws, lens, n_mel, tr = batch
    bars = BARS[cfg.R]
    compared = total = 0
    truncated = constant = 0
    worst_r = worst_s = worst_f = 0.0
    for c, (r, cand, cnt, _) in enumerate(split(tr, lens, n_mel)):
        ro, lp, ra0, gp = oracle_r(ws[c], cfg)
        bad = r_errors(r, ro, ra0, bars[0])
        assert not bad, (cfg, names[c], bad[:5])
        done, n, bad, wf, ws_, _ = candidate_errors(cand, cnt, ro, lp, ra0, gp, cfg, bars)
        assert not bad, (cfg, names[c], bad[:5])
        compared += len(done)
        total += n
        live = ra0 > 0
        worst_r = max(worst_r, float(np.abs(r[live] - ro[live]).max(initial=0)))
        worst_f, worst_s = max(worst_f, wf), max(worst_s, ws_)
        if names[c] == 'above_ceiling':
            truncated = sum(len(P.peaks(ro[j], cfg.sr, P.DEFAULTS)[0]) > 14 for j in range(len(ro)))
            assert truncated > len(ro) // 2, (cfg, truncated, len(ro))
            assert (cnt == 15).sum() > len(ro) // 2
        if names[c] == 'dc_constant':
            constant = int((ra0 == 0).sum())
            assert constant >= 10 and (cnt[ra0 == 0] == 1).all()
    print(f'{cfg}: worst r error {worst_r:.3g}, candidate frequency {worst_f:.3g} relative, strength {worst_s:.3g}; '
          f'{compared} / {total} frames compared, {truncated} truncated, {constant} constant')
    assert compared > 0.97 * total, (cfg, compared, total)


test_autocorrelation_and_candidates_match_the_oracle_at_the_other_configurations = at_the_other_configurations(test_autocorrelation_and_candidates_match_the_oracle)


def test_path_matches_the_oracle(batch):
    """The path kernel equals the float64 Viterbi on the kernel's own candidates wherever that path is more than 1e-9 ahead, and
    the placed f0 is the oracle's candidate on every frame where the oracle's path is more than 1e-4 ahead."""
    cfg, names, ws, lens, n_mel, tr = batch
    differ, worst = 0, 0.0
    parts = split(tr, lens, n_mel)
    for c, (_, cand, cnt, f0) in enumerate(parts):
        fk, mk = P.viterbi(cand[:, :, 0].astype(np.float64), cand[:, :, 1].astype(np.float64), cnt.astype(np.int64), cfg.hop / cfg.sr,
                           margins=True)
        n, bad = path_errors(f0, fk, mk, n_mel[c], cfg.lpad, 1e-9, 0.0)
        assert len(bad) == 0, (cfg, names[c], 'path kernel', bad[:10])
        fo, marg = P.track(ws[c], cfg.sr, cfg.hop, margins=True)
        n, bad = path_errors(f0, fo, marg, n_mel[c], cfg.lpad)
        differ += n
        pm = place(marg, n_mel[c], cfg.lpad)
        worst = max([worst] + [float(pm[i]) for i in np.nonzero(~same_f0(f0, place(fo, n_mel[c], cfg.lpad), 5e-4))[0] if i >= cfg.lpad])
        assert len(bad) == 0, (cfg, names[c], bad[:10], pm[bad[:10]])
    print(f'{cfg}: {differ} placed frames differ from the oracle, the largest oracle margin among them {worst:.3g}')
    assert differ < 10, (cfg, differ)
    for name in ('silence', 'noise'):
        assert (parts[names.index(name)][3] == 0).all(), name


test_path_matches_the_oracle_at_the_other_configurations = at_the_other_configurations(test_path_matches_the_oracle)


def test_each_clip_is_bit_identical_alone_and_in_the_batch(batch):
    cfg, names, ws, lens, n_mel, tr = batch
    hp = hp_of(cfg)
    parts = split(tr, lens, n_mel)
    for c, w in enumerate(ws):
        one = DG.pitch_ac_device(torch.from_numpy(w).cuda(), lens[c:c + 1], n_mel[c:c + 1], hp, want_cand=True, want_r=True,
                                 lpad=cfg.lpad)
        r, cand, cnt, f0 = parts[c]
        assert np.array_equal(one.r.cpu().numpy(), r) and np.array_equal(one.cand.cpu().numpy(), cand), names[c]
        assert np.array_equal(one.count.cpu().numpy(), cnt) and np.array_equal(one.f0.cpu().numpy(), f0), names[c]
    # the same batch reversed
    rev = ws[::-1]
    tr2 = DG.pitch_ac_device(torch.from_numpy(np.concatenate(rev)).cuda(), lens[::-1], n_mel[::-1], hp, lpad=cfg.lpad)
    oo = np.concatenate([[0], np.cumsum(n_mel[::-1])])
    for i, c in enumerate(range(len(ws) - 1, -1, -1)):
        assert np.array_equal(tr2.f0.cpu().numpy()[oo[i]:oo[i + 1]], parts[c][3])
    # f0 does not depend on which optional outputs are requested
    cat = torch.from_numpy(np.concatenate(ws)).cuda()
    f0 = tr.f0.cpu().numpy()
    for kw in ({}, {'want_cand': True}, {'want_r': True}, {'stage_ms': True}):
        other = DG.pitch_ac_device(cat, lens, n_mel, hp, lpad=cfg.lpad, **kw)
        assert np.array_equal(other.f0.cpu().numpy(), f0), kw
        if kw.get('stage_ms'):
            assert other.stage_ms.shape == (3,) and (other.stage_ms > 0).all()


test_each_clip_is_bit_identical_alone_and_in_the_batch_at_the_other_configurations = at_the_other_configurations(test_each_clip_is_bit_identical_alone_and_in_the_batch)


@EVERY_CONFIG
def test_scaling_by_a_power_of_two_changes_nothing(batch):
    """Power-of-two scaling is exact in every fp32 operation of the kernels while nothing underflows or overflows: an absolute
    threshold hidden anywhere would show as a difference."""
    cfg, names, ws, lens, n_mel, tr = batch
    parts = split(tr, lens, n_mel)
    for name in ('sung0', 'noise', 'dc_constant', 'square'):
        c = names.index(name)
        w = ws[c]
        scaled = [w * np.float32(2.0 ** 20), w * np.float32(2.0 ** -20)]
        assert all(np.array_equal(s / np.float32(2.0 ** e), w) for s, e in zip(scaled, (20, -20)))
        L = np.array([len(w)] * 2)
        M = np.array([n_mel[c]] * 2)
        t = DG.pitch_ac_device(torch.from_numpy(np.concatenate(scaled)).cuda(), L, M, hp_of(cfg), want_cand=True, want_r=True,
                               lpad=cfg.lpad)
        r, cand, cnt, f0 = parts[c]
        n = len(cnt)
        for k in range(2):
            assert np.array_equal(t.r.cpu().numpy()[k * n:(k + 1) * n], r), (name, k)
            assert np.array_equal(t.cand.cpu().numpy()[k * n:(k + 1) * n], cand), (name, k)
            assert np.array_equal(t.count.cpu().numpy()[k * n:(k + 1) * n], cnt), (name, k)
            assert np.array_equal(t.f0.cpu().numpy()[k * M[0]:(k + 1) * M[0]], f0), (name, k)


def test_get_pitch_equals_get_pitch_batch(batch):
    cfg, names, ws, lens, n_mel, tr = batch
    hp = hp_of(cfg)
    mels = [np.zeros((int(t), 80), np.float32) for t in n_mel]
    if cfg.hop not in (128, 256):
        with pytest.raises(ValueError, match='hop_size 128 or 256'):
            DG.get_pitch_batch(ws[:2], mels[:2], hp)
        return
    assert cfg.lpad == 2 * DG.pad_size(cfg.hop)
    many = DG.get_pitch_batch(ws, mels, hp)
    parts = split(tr, lens, n_mel)
    for c in range(len(ws)):
        assert np.array_equal(many[c][0], parts[c][3].astype(np.float64)), names[c]
    for name in ('sung0', 'sung3', 'silence', 'near_floor', 'dc_constant'):
        c = names.index(name)
        f0, pitch = DG.get_pitch(ws[c], mels[c], hp)
        assert np.array_equal(f0, many[c][0]) and np.array_equal(pitch, many[c][1])
    short = one_frame_bounds(cfg.sr, cfg.hop)[0] - 1
    with pytest.raises(ValueError, match='clip 0'):
        DG.get_pitch(np.zeros(short, np.float32), np.zeros((7, 80)), hp)


test_get_pitch_equals_get_pitch_batch_at_the_other_configurations = at_the_other_configurations(test_get_pitch_equals_get_pitch_batch)


@EVERY_CONFIG
def test_the_comparisons_catch_corrupted_outputs(batch):
    """The helpers above report each deliberate corruption of a real output, so their bars are not vacuous."""
    cfg, names, ws, lens, n_mel, tr = batch
    bars = BARS[cfg.R]
    parts = split(tr, lens, n_mel)
    # r: the last R lags of one voiced frame (the lags of the last live lane) zeroed
    c = names.index('sung0')
    r, cand, cnt, f0 = parts[c]
    ro, lp, ra0, gp = oracle_r(ws[c], cfg)
    j = int(np.argmax(np.where(ra0 > 0, np.abs(ro[:, -cfg.R:]).min(axis=1), 0)))
    assert np.abs(ro[j, -cfg.R:]).min() > 10 * bars[0]
    bad_r = r.copy()
    bad_r[j, -cfg.R:] = 0
    assert not r_errors(r, ro, ra0, bars[0]) and [b[0] for b in r_errors(bad_r, ro, ra0, bars[0])] == [j]
    # a candidate list with its 14th voiced entry dropped
    c = names.index('above_ceiling')
    r, cand, cnt, f0 = parts[c]
    ro, lp, ra0, gp = oracle_r(ws[c], cfg)
    _, _, bad, _, _, firm = candidate_errors(cand, cnt, ro, lp, ra0, gp, cfg, bars)
    assert not bad
    full = [j for j in firm if cnt[j] == 15]
    assert full
    j = full[len(full) // 2]
    cand2, cnt2 = cand.copy(), cnt.copy()
    cand2[j, 14] = (0.0, -np.inf)
    cnt2[j] = 14
    assert [b[0] for b in candidate_errors(cand2, cnt2, ro, lp, ra0, gp, cfg, bars)[2]] == [j]
    # one f0 frame moved to another candidate of that frame
    c = names.index('sung1')
    r, cand, cnt, f0 = parts[c]
    fo, marg = P.track(ws[c], cfg.sr, cfg.hop, margins=True)
    assert len(path_errors(f0, fo, marg, n_mel[c], cfg.lpad)[1]) == 0
    voiced = [j for j in range(len(fo)) if fo[j] > 0 and marg[j] > 1e-3 and cnt[j] > 2 and cfg.lpad + j < n_mel[c]]
    j = voiced[len(voiced) // 2]
    other = next(cand[j, k, 0] for k in range(1, cnt[j]) if abs(cand[j, k, 0] - f0[cfg.lpad + j]) > 1e-3 * fo[j])
    bad_f0 = f0.copy()
    bad_f0[cfg.lpad + j] = other
    assert path_errors(bad_f0, fo, marg, n_mel[c], cfg.lpad)[1].tolist() == [cfg.lpad + j]


def test_placement_for_any_lpad_and_track_length():
    """lpad 0, 4, 8 and more than len(mel); len(mel) 0, below lpad, inside the track, exactly lpad + n and beyond (extended with
    the last frame, which is voiced in the first clip), against the oracle track placed by the generalised rule."""
    torch.cuda.set_device(0)
    take = sung(2, 3.0, SR, HOP)
    end = int(np.nonzero(np.abs(take) > 0.05)[0][-1])             # end inside a voiced stretch
    base = [take[:end - 2000], sung(3, 1.5, SR, HOP), tone(300.0, 0.6, 3)]
    tracks = [P.track(w, SR, HOP, margins=True) for w in base]
    assert tracks[0][0][-1] > 0
    for lpad in (0, 4, 8, 200):
        ws, T, owner = [], [], []
        for b, (w, (fo, _)) in enumerate(zip(base, tracks)):
            n = len(fo)
            for t in sorted({0, min(3, lpad), max(lpad - 1, 0), lpad + n // 2, lpad + n, lpad + n + 37}):
                ws.append(w)
                T.append(t)
                owner.append(b)
        lens = np.array([len(w) for w in ws])
        tr = DG.pitch_ac_device(torch.from_numpy(np.concatenate(ws)).cuda(), lens, np.array(T), HP, lpad=lpad)
        f0 = tr.f0.cpu().numpy()
        assert f0.shape == (sum(T),)
        oo = np.concatenate([[0], np.cumsum(T)])
        for i, (w, b) in enumerate(zip(ws, owner)):
            fo, marg = tracks[b]
            out = f0[oo[i]:oo[i + 1]]
            assert (out[:lpad] == 0).all()
            _, bad = path_errors(out, fo, marg, T[i], lpad)
            assert len(bad) == 0, (lpad, T[i], bad[:10])
            if T[i] > lpad + len(fo):
                assert (out[lpad + len(fo):] == out[lpad + len(fo) - 1]).all()


def test_a_large_ragged_batch_with_a_long_clip():
    """300 clips of 1-2 s and one of 60 s in one call: the candidate kernel's clip search spans them all, and a sample of clips is
    bit-identical alone."""
    torch.cuda.set_device(0)
    rs = np.random.RandomState(3)
    takes = [sung(i, 2.6, SR, HOP) for i in range(8)]
    ws = []
    for i in range(300):
        t = takes[i % 8]
        n = int(rs.uniform(1.0, 2.0) * SR)
        o = rs.randint(0, len(t) - n)
        ws.append(t[o:o + n])
    ws.insert(137, np.concatenate(takes * 3)[:60 * SR])
    lens = np.array([len(w) for w in ws])
    n_mel = lens // HOP + 1
    tr = DG.pitch_ac_device(torch.from_numpy(np.concatenate(ws)).cuda(), lens, n_mel, HP, want_cand=True, want_r=True)
    parts = split(tr, lens, n_mel)
    assert int(tr.frames.sum()) == sum(P.grid(int(N), SR, HOP / SR)[0] for N in lens)
    for c in (0, 1, 136, 137, 138, 211, 299, 300):
        one = DG.pitch_ac_device(torch.from_numpy(ws[c]).cuda(), lens[c:c + 1], n_mel[c:c + 1], HP, want_cand=True, want_r=True)
        r, cand, cnt, f0 = parts[c]
        assert np.array_equal(one.r.cpu().numpy(), r) and np.array_equal(one.cand.cpu().numpy(), cand), c
        assert np.array_equal(one.count.cpu().numpy(), cnt) and np.array_equal(one.f0.cpu().numpy(), f0), c
    # the long clip against the oracle's path
    fo, marg = P.track(ws[137], SR, HOP, margins=True)
    n, bad = path_errors(parts[137][3], fo, marg, n_mel[137], 8)
    assert len(bad) == 0 and n < 10, (n, bad[:10])


def test_a_short_workspace_is_refused_on_the_device():
    torch.cuda.set_device(0)
    w = sung(0, 2.0, SR, HOP)
    lens, n_mel = np.array([len(w)], np.int64), np.array([len(w) // HOP + 1], np.int64)
    cfg = DG.pitch_config(HP)
    l = _native.lib()
    need = l.svb_pitch_ac_workspace_bytes(ctypes.byref(cfg), lens.ctypes.data, 1, None)
    assert need > 0
    wav = torch.from_numpy(w).cuda()
    ws = torch.empty(need - 1, dtype=torch.uint8, device='cuda')
    f0 = torch.full((int(n_mel[0]),), float('nan'), device='cuda')
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    with pytest.raises(ValueError, match=f'workspace of {need - 1} bytes, {need} needed'):
        DG._check(l.svb_pitch_ac_batch(ctypes.byref(cfg), vp(wav), lens.ctypes.data, 1, n_mel.ctypes.data, vp(f0), vp(ws), need - 1,
                                       None, None, None, None, _native.current_stream_ptr(wav.device)), 'pitch_ac')
    torch.cuda.synchronize()
    assert torch.isnan(f0).all()
    # the same call with the full workspace writes every frame
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')
    DG._check(l.svb_pitch_ac_batch(ctypes.byref(cfg), vp(wav), lens.ctypes.data, 1, n_mel.ctypes.data, vp(f0), vp(ws), need,
                                   None, None, None, None, _native.current_stream_ptr(wav.device)), 'pitch_ac')
    torch.cuda.synchronize()
    assert not torch.isnan(f0).any()


# ------------------------------------------------------------------------------------------------- binarizer end to end
def _cli(module, args, cwd, timeout=1200):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, '-m', module] + args, cwd=cwd, env=env, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_binarize_cli_then_train_and_infer(tmp_path):
    from scipy.io import wavfile

    from neuralsvb_b200.modules.voice_conversion.dtw.core import align_pitch
    from neuralsvb_b200.tasks.singing.dataset_utils import MultiSpkEmbDataset
    from neuralsvb_b200.utils import hparams as H
    from neuralsvb_b200.utils.indexed_datasets import IndexedDataset
    from neuralsvb_b200.vocoders.hifigan import HifiGAN
    raw, binary = str(tmp_path / 'raw'), str(tmp_path / 'bin')
    truth = S.write_svb_raw(raw, binary)
    ov = f'processed_data_dir={raw},binary_data_dir={binary},spk_emb_data_dir={raw}/spk_emb'
    out = _cli('neuralsvb_b200.data_gen.tts.bin.binarize', ['--config', os.path.join(ROOT, 'egs', 'svb_binarize_synthetic.yaml'),
                                                            '--hparams', ov], tmp_path)
    assert '| Skip item (Empty f0). item_name: Male1#singing#Song_A_Amateur_1' in out
    with open(os.path.join(binary, 'bad_case.txt')) as f:
        assert f.read().startswith('Gap is too large: Female2#singing#Song_B_Amateur_1')
    hp = H.set_hparams(os.path.join(ROOT, 'egs', 'svb_binarize_synthetic.yaml'), '', ov, print_hparams=False, global_hparams=False)
    keys = {'item_name', 'mel', 'prof_mel', 'f0', 'prof_f0', 'pitch', 'prof_pitch', 'a2p_f0_alignment', 'multi_spk_emb'}
    expect = {'train': ['Female1#singing#Song_A_Amateur_0', 'Female1#singing#Song_A_Amateur_1', 'Female1#singing#Song_B_Amateur_0',
                        'Female1#singing#Song_B_Amateur_1', 'Female2#singing#Song_A_Amateur_0', 'Female2#singing#Song_A_Amateur_1',
                        'Female2#singing#Song_B_Amateur_0'],
              'test': ['Male1#singing#Song_A_Amateur_0', 'Male1#singing#Song_B_Amateur_0', 'Male1#singing#Song_B_Amateur_1']}
    pairs = []
    for prefix in ('train', 'valid', 'test'):
        ds = IndexedDataset(os.path.join(binary, prefix))
        items = [ds[i] for i in range(len(ds))]
        assert [it['item_name'] for it in items] == expect['train' if prefix == 'train' else 'test']
        f0s = []
        for it in items:
            assert set(it) == keys
            name = it['item_name']
            wav_fn = glob.glob(os.path.join(raw, 'data', '*', name + '.wav'))[0]
            prof_fn = wav_fn.replace('Amateur', 'Professional')
            for fn, mk, fk in ((wav_fn, 'mel', 'f0'), (prof_fn, 'prof_mel', 'prof_f0')):
                wav, mel = HifiGAN.wav2spec(fn, hp=hp)
                assert np.array_equal(it[mk], mel), name
                f0, pitch = DG.get_pitch(wav, mel, hp)
                assert np.array_equal(it[fk], f0) and np.array_equal(it[fk.replace('f0', 'pitch')], pitch), name
                tv = truth[os.path.splitext(os.path.basename(fn))[0]]
                # placed frame i >= 8 is analysis frame i - 8 centred on sample c0 + (i - 8) hop
                n, L, c0, _ = P.grid(len(wav), SR, HOP / SR)
                idx = np.arange(8, len(f0))
                centre = np.minimum(c0 + (idx - 8) * HOP, len(tv) - 1)
                t = np.zeros(len(f0))
                t[idx] = tv[centre]
                ok = np.zeros(len(f0), bool)
                ok[idx] = True
                v = t > 0
                for e in np.nonzero(np.diff(v.astype(int)))[0]:
                    ok[max(0, e - 3):e + 5] = False
                pairs.append((f0, t, ok))
            assert np.array_equal(it['a2p_f0_alignment'], align_pitch([it['f0']], [it['prof_f0']], 'EHSADTW')[0])
            f0s += [it['f0'], it['prof_f0']]
        lengths = np.load(os.path.join(binary, f'{prefix}_lengths.npy'))
        assert lengths.tolist() == [max(len(it['mel']), len(it['prof_mel'])) for it in items]
        f = np.concatenate(f0s)
        assert np.allclose(np.load(os.path.join(binary, f'{prefix}_f0s_mean_std.npy')), [f[f > 0].mean(), f[f > 0].std()])
    gross = voiced = verr = total = 0
    cents = []
    for est, t, ok in pairs:
        both = ok & (t > 0) & (est > 0)
        gross += int((np.abs(est[both] / t[both] - 1) > 0.2).sum())
        voiced += int((ok & (t > 0)).sum())
        verr += int((ok & ((t > 0) != (est > 0))).sum())
        total += int(ok.sum())
        cents += list(np.abs(1200 * np.log2(est[both] / t[both])))
    assert gross < 0.01 * voiced and np.median(cents) < 10 and verr < 0.05 * total, (gross, voiced, np.median(cents), verr, total)
    # the dataset reads it
    hp_train = H.set_hparams(os.path.join(ROOT, 'egs', 'svb_vae_train_synthetic.yaml'), '', f'binary_data_dir={binary}',
                             print_hparams=False, global_hparams=False)
    ds = MultiSpkEmbDataset('train', hp_train)
    assert len(ds) == 7 and ds[0]['multi_spk_emb'].shape == (5, 256)
    # tasks/run.py: train, resume, infer
    cfg = os.path.join(ROOT, 'egs', 'svb_vae_train_synthetic.yaml')
    tov = (f'binary_data_dir={binary},pretrain_asr_ckpt={binary}/asr,vocoder_ckpt={binary}/hifigan,max_updates=6,phase_2_steps=4,'
           'val_check_interval=3,valid_infer_interval=3,tb_log_interval=1')
    out = _cli('neuralsvb_b200.tasks.run', ['--config', cfg, '--exp_name', 'svb_raw', '--reset', '--hparams', tov], tmp_path)
    assert 'Training end' in out
    out = _cli('neuralsvb_b200.tasks.run', ['--config', cfg, '--exp_name', 'svb_raw', '--hparams', 'max_updates=8'], tmp_path)
    assert '| step 6:' in out and '| step 5:' not in out and 'Training end' in out
    _cli('neuralsvb_b200.tasks.run', ['--config', cfg, '--exp_name', 'svb_raw', '--infer'], tmp_path)
    wavs = sorted(glob.glob(str(tmp_path / 'checkpoints' / 'svb_raw' / 'generated_*_' / 'wavs' / 'a2p_wavout' / '*.wav')))
    assert len(wavs) == 3, wavs
    assert wavfile.read(wavs[0])[0] == SR

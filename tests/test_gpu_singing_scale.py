"""-m gpu: the singing vocoder chain at the sizes the beautifier (neuralsvb_b200/inference/beautify.py) accepts, against float64
and the float32 oracle: takes of up to max_frames = 5000 frames (640 000 samples at hop 128), ragged batches of many pairs and
the NSF draws of the in-kernel Philox generator.

  1. the singing front end (n_fft 512, hop 128, win 512, fmin 50, fmax 11025, log10 mel, zero centre padding) on a ragged batch
     from 1 sample to beyond max_frames, against float64 torch.stft and each clip's single-clip call;
  2. the NSF source at 5000 frames (hop 128 and 256), with f0 that changes every frame across 80-750 Hz, against the oracle, and
     the number of mantissa bits its exact phase sums need;
  3. the Philox draws (noise and initial phases) read back through the public model: standard normal, independent, uniform;
  4. the hop-128 generator launch by launch at the beautifier's shapes, including a batch whose activations pass 2^31 bytes;
  5. the denoise post-filter at the singing STFT configuration;
  6. spec2wav of a 70 000-frame mel (a 6.8-minute song at hop 128) in every precision: its frames pass the 65 535-block limit
     of gridDim.y, and on tensor cores its convs overflow one launch's work-item table and run in slices of rows.

Timings and peak device memory of this file are printed per test (MEASURED lines)."""
import contextlib
import ctypes
import io
import math
import os
import time

import numpy as np
import pytest
import scipy.stats
import torch
import yaml

from neuralsvb_b200 import _native
from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
from neuralsvb_b200.utils import audio
from neuralsvb_b200.utils import synthetic as S
from neuralsvb_b200.vocoders.hifigan import HifiGAN
from oracle import frontend as FE
from oracle import hifigan as O
from tests import gpu_util as U
from tests.test_gpu_generator_forward import (BARS, MARGIN, compare, describe, group_errors, judge, make_model, ref_weights,
                                              say, schedules)
from tests.test_gpu_generator_ragged import alone, bits_equal, clip_errors, run
from tests.test_gpu_stft_kernels import (FWD_TOL, LOG10_MEL, ZERO, assert_clear_of_eps, errors, make_wave, run_wav2spec,
                                         stft_reference)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, 'egs', 'svb_vae_train_synthetic.yaml')) as _f:
    _CFG = yaml.safe_load(_f)
HP = {k: _CFG[k] for k in ('audio_sample_rate', 'hop_size', 'fft_size', 'win_size', 'fmin', 'fmax', 'audio_num_mel_bins')}
MAX_FRAMES = int(_CFG['max_frames'])
SR, HOP = HP['audio_sample_rate'], HP['hop_size']
assert (HOP, HP['fft_size'], HP['win_size'], HP['fmin'], HP['fmax'], MAX_FRAMES) == (128, 512, 512, 50, 11025, 5000)
EPS = 1e-10                                                  # wav2spec_eps default (HifiGAN.wav2spec_device)


@pytest.fixture(autouse=True)
def device_memory(request, capfd):
    """Wall time and peak device memory of each test: torch's allocator and the whole device (the generator's workspace is the
    native library's own cudaMalloc, which torch does not see)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    free0, total = torch.cuda.mem_get_info()
    yield
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    say(capfd, f'MEASURED {request.node.name}: {time.time() - t0:.1f} s, torch peak {torch.cuda.max_memory_allocated() / 2**30:.2f} '
               f'GiB, device in use at the end {(total - free1) / 2**30:.2f} GiB (at the start {(total - free0) / 2**30:.2f})')
    torch.cuda.empty_cache()


def hop_of(h):
    return int(np.prod(h['upsample_rates']))


# ------------------------------------------------------------------ 1. the singing front end
def test_singing_front_end_on_a_long_ragged_batch_matches_float64_and_single_clip_device_calls(capfd):
    cfg = (HP['fft_size'], HOP, HP['win_size'], ZERO, LOG10_MEL, 0, HP['audio_num_mel_bins'], 1, EPS)
    c = _native.StftConfig(*cfg)
    # 1 sample; 127 / 128 / 129 samples (around one hop); a 60-frame take; 8 s; exactly max_frames frames; one clip beyond
    # (the front end has no cap; max_frames is checked by the beautifier after it); exact silence
    lengths = [1, 127, 128, 129, 60 * HOP - 1, 8 * SR, MAX_FRAMES * HOP - 1, 1_000_003, 3000]
    clips = [make_wave(1, L, ('singing', i))[0] for i, L in enumerate(lengths)]
    clips[-1] = torch.zeros(lengths[-1])
    basis = torch.from_numpy(np.asarray(audio.build_mel_basis(HP), np.float32))
    # At n_fft 512 (43 Hz bins) the lowest slaney filters above fmin 50 Hz are one or two bins wide, yet every row holds filter
    # weight, so no mel row is pinned to log10(eps).  Silent frames are: the last clip is exact silence.
    empty = [i for i in range(basis.shape[0]) if not bool((basis[i] != 0).any())]
    widths = (basis != 0).sum(1)
    say(capfd, f'MEASURED singing mel basis: empty rows {empty}, fewest non-zero bins in a row {int(widths.min())} '
               f'(row {int(widths.argmin())})')
    assert empty == [], empty
    mel, wav, frames = HifiGAN.wav2spec_device(torch.cat(clips).cuda(), lengths, HP, basis.cuda())
    torch.cuda.synchronize()
    assert frames.tolist() == [L // HOP + 1 for L in lengths]
    assert frames[6] == MAX_FRAMES and frames[7] > MAX_FRAMES
    mel, wav = mel.cpu(), wav.cpu()
    # the clamp's fp32 log10f of fp32 eps, as the device computes it, and within one fp32 ulp of the float64 value
    log10_eps = torch.log10(torch.tensor(np.float32(EPS), device='cuda')).cpu()
    assert abs(float(log10_eps) - math.log10(float(np.float32(EPS)))) <= float(np.spacing(np.float32(10.0)))
    off, worst = 0, (0.0, 0.0, -1)
    for i, (L, x) in enumerate(zip(lengths, clips)):
        fr = int(frames[i])
        m, w = mel[off:off + fr], wav[off * HOP:(off + fr) * HOP]
        off += fr
        single = torch.full((fr, cfg[6]), float('nan'), device='cuda')
        single_wav = torch.full((fr * HOP,), float('nan'), device='cuda')
        assert run_wav2spec(c, x.cuda(), [L], basis.cuda(), single, single_wav) == fr
        single, single_wav = single.cpu(), single_wav.cpu()
        assert torch.equal(m, single), f'clip {i} (length {L}): the batch differs from its single-clip call'
        lpad, rpad = FE.librosa_pad_lr(x.numpy(), HP['fft_size'], HOP)
        want = np.pad(x.numpy(), (lpad, rpad))[:fr * HOP]
        assert np.array_equal(w.numpy(), want) and np.array_equal(single_wav.numpy(), want), f'clip {i}: padded waveform'
        ref, ratio = stft_reference(x[None].cuda(), cfg, basis.cuda())
        assert_clear_of_eps(ratio, f'clip {i}')
        e = errors(m.cuda(), ref[0])
        if e[1] > worst[1]:
            worst = (e[0], e[1], i)
        assert e[0] <= FWD_TOL[0] and e[1] <= FWD_TOL[1], (i, L, e)
        if L == lengths[-1]:
            assert torch.equal(m, log10_eps.expand_as(m)), (float(m.min()), float(m.max()), float(log10_eps))
    say(capfd, f'MEASURED singing front end: worst clip {worst[2]} (length {lengths[worst[2]]}) relative L2 {worst[0]:.2e}, '
               f'L-inf {worst[1]:.2e} (bars {FWD_TOL})')


# ------------------------------------------------------------------ 2. the NSF source at max_frames
def f0_vibrato(T, rs):
    """f0 moving every frame across 80-750 Hz: a 5.3-frame-period vibrato on a slow glide, plus jitter, so every frame's rad has
    its own mantissa."""
    t = np.arange(T)
    f = 415 + 300 * np.sin(2 * np.pi * t / 911.3) + 35 * np.sin(2 * np.pi * t / 5.3) + rs.uniform(-1, 1, T)
    return np.clip(f, 80, 750)


def f0_floor_after_stretch(T, rs):
    """A long 750 Hz stretch, then the 80 Hz floor beside it: the finest rad ulp arrives on the largest partial sum."""
    f = np.full(T, 750.0)
    f[T - T // 5:] = 80.0
    f[T - T // 5 - 7:T - T // 5:2] = 80.0                   # and a few floor frames between the 750 Hz ones
    return f


def f0_flips(T, rs):
    """Voicing that flips every frame, a long unvoiced run, then a new random f0 in [80, 750] every frame."""
    f = rs.uniform(80, 750, T)
    f[:T // 3:2] = 0.0
    f[T // 3:2 * T // 3] = 0.0
    return f


def f0_random(T, rs):
    return rs.uniform(80, 750, T)


F0_KINDS = {'vibrato': f0_vibrato, 'floor_after_stretch': f0_floor_after_stretch, 'flips': f0_flips, 'random': f0_random}


def rad32(f0, k):
    """rad of harmonic k per frame as nsf_source.cu computes it: fp32 f0 * (k + 1) / sr, fmod 1."""
    f = np.asarray(f0, np.float32)
    return np.fmod((f * np.float32(k + 1)) / np.float32(SR), np.float32(1.0)).astype(np.float32)


def phase_sum_bits(f0, hop, ri):
    """log2(largest partial phase sum / smallest ulp of its terms) over the 9 harmonics of one clip.  The kernel's double
    partial sums S1 are exact (hence order-free and equal to the reference's sequential sum) while this stays below 53: every
    term -- hop x rad, (j + 1) x rad, fl32(rad_0 + rand_ini) -- is a multiple of the smallest ulp, and no partial sum exceeds
    the largest."""
    worst = 0.0
    for k in range(9):
        r = rad32(f0, k)
        r0p = np.float32(r[0] + np.float32(ri[k]))
        terms = np.concatenate([r[r > 0], [r0p] if r0p > 0 else []])
        if terms.size == 0:
            continue
        ulp = float(np.spacing(terms.astype(np.float32)).min())
        top = float(r0p) + float(np.cumsum(r.astype(np.float64) * hop).max())
        worst = max(worst, math.log2(top / ulp))
    return worst


def nsf_case(arch, kinds, T):
    h = S.hifigan_config(True, hop=128 if arch == 'hop128' else 256)
    hop = hop_of(h)
    rs = np.random.RandomState(4321)
    B = len(kinds)
    mel, _ = S.make_mel_f0(B, T, U.SEED)
    f0 = torch.from_numpy(np.stack([F0_KINDS[k](T, rs) for k in kinds]).astype(np.float32))
    ri, nz = S.make_nsf_noise(B, T * hop, U.SEED)
    return h, hop, mel, f0, ri, nz


def har_errors(m, h, f0, ri, nz, lengths):
    """(L-inf, clip, sample) of the har_source tap against the float32 oracle run on each clip alone."""
    hop = hop_of(h)
    har = m.get_tap('har_source')[:, 0].cpu()
    w = m.folded_state()
    worst = (-1.0, 0, 0)
    for b, L in enumerate(lengths):
        f0_up = torch.repeat_interleave(f0[b:b + 1, :L], hop, dim=1)[:, :, None]
        ref, _ = O.source_module(f0_up, w, ri[b:b + 1], nz[b:b + 1, :L * hop], sr=h['audio_sample_rate'])
        d = (har[b, :L * hop] - ref[0, :, 0]).abs()
        assert (har[b, L * hop:] == 0).all()
        if float(d.max()) > worst[0]:
            worst = (float(d.max()), b, int(d.argmax()))
    return worst


NSF_CASES = [
    pytest.param('hop128', ['vibrato', 'floor_after_stretch', 'flips', 'random'], None, id='hop128_B4_max_frames'),
    pytest.param('hop256', ['vibrato', 'floor_after_stretch'], None, id='hop256_B2_max_frames'),
    pytest.param('hop128', ['vibrato', 'random', 'flips', 'floor_after_stretch'], [MAX_FRAMES, 60, 1, 333],
                 id='hop128_ragged_long_beside_short'),
]


@pytest.mark.parametrize('arch,kinds,lengths', NSF_CASES)
def test_nsf_source_at_max_frames_matches_oracle(arch, kinds, lengths, monkeypatch, capfd):
    T = MAX_FRAMES
    m, _ = make_model(arch, 'bf16x3', monkeypatch)
    h, hop, mel, f0, ri, nz = nsf_case(arch, kinds, T)
    bits = max(phase_sum_bits(f0[b, :L].numpy(), hop, ri[b].numpy()) for b, L in enumerate(lengths or [T] * len(kinds)))
    run(m, mel, f0, ri, nz, lengths)
    e, b, t = har_errors(m, h, f0, ri, nz, lengths or [T] * len(kinds))
    say(capfd, f'MEASURED har_source {arch} {kinds} lengths {lengths or T}: L-inf {e:.2e} at clip {b} ({kinds[b]}) sample {t} '
               f'(frame {t // hop}); exact phase sums need {bits:.1f} of 53 bits')
    assert bits < 53, bits
    assert e < 5e-6, (e, b, t)                          # test_gpu_parity.py::test_nsf_source_matches_oracle


# ------------------------------------------------------------------ 3. the Philox draws
# nsf_source.cu draws, when no rand_ini / noise are injected:
#   noise of harmonic k = 3 g + i at sample t of clip b: Box-Muller of Philox4x32-10(counter (t, b, g, 'NSF'), key seed), t the
#     sample within the clip and b the clip's index within the call (so a clip draws other noise alone than in a batch);
#   initial phase of harmonic k >= 1 of clip b: u01 of Philox4x32-10(counter (b, k, 0x1234, 0), key seed ^ 0x5eed << 32);
#     harmonic 0 starts at phase 0.
# They are read back through the model: with m_source.l_linear = e_k (bias 0), har = tanh(l_linear(x)) = tanh(x_k) where
# x_k = 0.1 / 3 n_k on unvoiced samples and 0.1 sin(2 pi (phase_k + t rad_k)) + 0.003 n_k on voiced ones.
NOISE_AMP_UV = float(np.float32(np.float32(0.1) / np.float32(3.0)))
Z5 = 5.0                                                     # every bound below is about 5 sigma for its sample count
KS5 = 2.75                                                   # P(sqrt(N) D > 2.75) ~ 2 exp(-2 2.75^2) = 5.4e-7, as 5 sigma


def one_hot_model(monkeypatch):
    m, h = make_model('hop128', 'bf16x3', monkeypatch)
    return m, h


def set_one_hot(m, k):
    with torch.no_grad():
        w = m.get_parameter('m_source.l_linear.weight')
        w.zero_()
        w[0, k] = 1.0
        m.get_parameter('m_source.l_linear.bias').zero_()


def draws(m, mel, f0, lengths, seed, k):
    set_one_hot(m, k)
    run(m, mel, f0, None, None, lengths, seed=seed)
    har = m.get_tap('har_source')[:, 0].double().cpu()
    return [har[b, :L * HOP] for b, L in enumerate(lengths)]


def corr(a, b):
    a, b = a - a.mean(), b - b.mean()
    return float((a * b).sum() / math.sqrt(float((a * a).sum() * (b * b).sum())))


def test_philox_noise_is_standard_normal_and_independent(monkeypatch, capfd):
    m, h = one_hot_model(monkeypatch)
    lengths = [1000, 990, 1000, 985, 1000, 995, 1000, 1000]            # 1.02M samples per harmonic
    B, T = len(lengths), max(lengths)
    mel, _ = S.make_mel_f0(B, T, U.SEED)
    f0 = torch.zeros(B, T)
    seed = 20261017
    n = {}
    for s in (seed, seed + 1):
        for k in range(9):
            n[s, k] = [torch.atanh(x) / NOISE_AMP_UV for x in draws(m, mel, f0, lengths, s, k)]
    N = sum(L * HOP for L in lengths)
    bad, rec = [], {}

    def check(name, value, bound):
        rec[name] = max(rec.get(name, 0.0), abs(value) / bound)
        if not abs(value) <= bound:
            bad.append(f'{name}: {value:.3e} beyond {bound:.3e}')
    for k in range(9):
        x = torch.cat(n[seed, k])
        check('mean', float(x.mean()), Z5 / math.sqrt(N))
        check('variance - 1', float(x.var()) - 1.0, Z5 * math.sqrt(2.0 / N))
        check('KS distance to N(0, 1)', scipy.stats.kstest(x.numpy(), 'norm').statistic, KS5 / math.sqrt(N))
        for j in range(k):
            check('harmonics at one sample', corr(x, torch.cat(n[seed, j])), Z5 / math.sqrt(N))
        check('seed s and s + 1', corr(x, torch.cat(n[seed + 1, k])), Z5 / math.sqrt(N))
        for lag in range(1, HOP + 1):
            a = torch.cat([v[:-lag] for v in n[seed, k]])
            b = torch.cat([v[lag:] for v in n[seed, k]])
            check(f'lags 1..{HOP}', corr(a, b), Z5 / math.sqrt(a.numel()))
        for b1 in range(B):
            for b2 in range(b1):
                L = min(lengths[b1], lengths[b2]) * HOP
                check('clips at one sample', corr(n[seed, k][b1][:L], n[seed, k][b2][:L]), Z5 / math.sqrt(L))
    say(capfd, f'MEASURED Philox noise over {N} samples x 9 harmonics, largest statistic / its bound: ' +
               ', '.join(f'{k} {v:.2f}' for k, v in rec.items()))
    assert not bad, '\n'.join(bad[:20])


def test_philox_initial_phases_are_uniform_and_harmonic_0_starts_at_0(monkeypatch, capfd):
    m, h = one_hot_model(monkeypatch)
    B, T = 64, 32                                                        # 4096 samples a clip, 64 x 8 phases
    mel, _ = S.make_mel_f0(B, T, U.SEED)
    f0c = (110.0 + 2.9 * np.arange(B)).astype(np.float32)               # 9 x f0 < 2.7 kHz: rad in (0.005, 0.12)
    f0 = torch.from_numpy(np.repeat(f0c[:, None], T, 1))
    t = np.arange(T * HOP, dtype=np.float64)
    phases = np.zeros((B, 9))
    amp_err = 0.0
    for k in range(9):
        for b, x in enumerate(draws(m, mel, f0, [T] * B, 777, k)):
            # S2[t] = fl32(rad + phase) + t rad, less whole cycles: the ramp t rad with an unknown phase, by least squares
            r = float(rad32(f0c[b:b + 1], k)[0])
            A = np.stack([np.sin(2 * np.pi * t * r), np.cos(2 * np.pi * t * r)], 1)
            (c1, c2), *_ = np.linalg.lstsq(A, np.arctanh(x.numpy()), rcond=None)
            amp_err = max(amp_err, abs(math.hypot(c1, c2) - 0.1) / 0.1)
            phases[b, k] = (math.atan2(c2, c1) / (2 * np.pi) - r) % 1.0   # less the first sample's own rad
    d0 = np.abs((phases[:, 0] + 0.5) % 1.0 - 0.5)
    ks = scipy.stats.kstest(phases[:, 1:].ravel(), 'uniform')
    say(capfd, f'MEASURED Philox initial phases: harmonic 0 within {d0.max():.2e} cycles of 0, KS distance of the {B * 8} '
               f'others to U[0, 1) {ks.statistic:.3f} (bound {KS5 / math.sqrt(B * 8):.3f}), sine amplitude within {amp_err:.1e}')
    assert amp_err < 0.02, amp_err                       # the fit sees the 0.1 sine: the model of har above holds
    assert d0.max() < 2e-3, d0.max()
    assert ks.statistic < KS5 / math.sqrt(B * 8), ks


# ------------------------------------------------------------------ 4. the hop-128 generator at beautifier shapes
BENCH_FRAMES = 1378                                          # 8 s at hop 128: tools/beautify_bench.py's takes


def ragged_lengths(shape):
    rs = np.random.RandomState(1378)
    if shape == 'bench64':                                   # 64 clips of 1378 +- 15 % frames
        return rs.randint(int(BENCH_FRAMES * 0.85), int(BENCH_FRAMES * 1.15) + 1, 64).tolist()
    if shape == 'max_frames_among_short':
        return [60, 61, MAX_FRAMES, 127, 128, 129, 1377, 1378, 1379, 1, 17, 333, 4096]
    if shape == 'past_2gib':                                 # clips padded to max_frames; the last one a whole take
        return rs.randint(60, 400, 27).tolist() + [MAX_FRAMES]
    raise ValueError(shape)


def float64_clips(shape, lengths):
    """The clips of a ragged shape checked against float64 one by one (a float64 pass over every clip of bench64 or past_2gib
    is the slowest part of this file, and the bit-identity with each clip alone covers them all)."""
    if shape == 'bench64':
        order = np.argsort(lengths, kind='stable')
        picks = np.random.RandomState(64).choice(np.arange(1, 63), 4, replace=False).tolist()
        return sorted({int(order[-1]), int(order[0]), 0, 63, *picks})
    if shape == 'max_frames_among_short':
        return [lengths.index(MAX_FRAMES), lengths.index(60), lengths.index(129)]
    return [len(lengths) - 1]


def subset_errors(m, h, w, mel, y, lengths, clips):
    """test_gpu_generator_ragged.clip_errors for the clips listed only, each tap read once and cut to those clips; the worst
    clip of each tap is named by its index in the batch."""
    taps = {}
    names = ['har_source', 'conv_pre'] + [f'{p}{i}' for i in range(len(h['upsample_rates'])) for p in ('ups', 'stage')]
    for k in names:
        t = m.get_tap(k)
        taps[k] = t[clips].clone()
        del t
    torch.cuda.empty_cache()

    class Taps:                                              # what clip_errors reads from the model: clip j of the list
        def __init__(self, j):
            self.j = j

        def get_tap(self, k):
            return taps[k][self.j:self.j + 1]
    worst = {}
    for j, b in enumerate(clips):
        for tap, (e, l2, (_, c, t)) in clip_errors(Taps(j), h, w, mel[b:b + 1], y[b:b + 1], [lengths[b]]).items():
            if tap not in worst or e > worst[tap][0]:
                worst[tap] = (e, l2, (b, c, t))
    return worst


def ragged_inputs(h, lengths, seed=U.SEED):
    B, T = len(lengths), max(lengths)
    mel, f0 = S.make_mel_f0(B, T, seed)
    ri, nz = S.make_nsf_noise(B, T * hop_of(h), seed)
    return mel, f0, ri, nz


def verbose_run(m, mel, f0, ri, nz, lengths, monkeypatch, capfd):
    capfd.readouterr()
    monkeypatch.setenv('SVB_TC_VERBOSE', '1')
    y = run(m, mel, f0, ri, nz, lengths)
    monkeypatch.delenv('SVB_TC_VERBOSE')
    return y, capfd.readouterr().err.splitlines()


# The schedule every stage of the hop-128 generator runs at these shapes, as observed on an H100 80GB HBM3 (132 SMs, 700 W
# power limit), pinned so that a planner change that moves them shows up here.  The 64 bench clips overflow the per-CTA item
# table of every merged or fused launch, so each conv runs as a launch of its own; stage 2 (64 channels at 64 x T rows) never
# fuses at these lengths.  (The relative L2 printed for the ragged shapes is that of the worst clip alone.)
SCHEDULE = {
    ('uniform8x1378', 'bf16x3'): ['merged-staged', 'merged-staged', 'single', 'fused2'],
    ('uniform8x1378', 'tf32x3'): ['merged', 'merged', 'single', 'single'],
    ('bench64', 'bf16x3'): ['single'] * 4,
    ('bench64', 'tf32x3'): ['single'] * 4,
    ('max_frames_among_short', 'bf16x3'): ['merged-staged', 'merged-staged', 'single', 'single'],
    ('max_frames_among_short', 'tf32x3'): ['merged', 'merged', 'single', 'single'],
    ('past_2gib', 'bf16x3'): ['merged-staged', 'merged-staged', 'single', 'fused2'],
    ('past_2gib', 'tf32x3'): ['merged', 'merged', 'single', 'single'],
}
SHAPES4 = ['uniform8x1378', 'bench64', 'max_frames_among_short', 'past_2gib']


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3'])
@pytest.mark.parametrize('shape', SHAPES4)
def test_hop128_generator_at_beautifier_shapes_matches_float64(shape, precision, monkeypatch, capfd):
    m, h = make_model('hop128', precision, monkeypatch)
    w = ref_weights(m)
    hop = hop_of(h)
    tag = f'hop128 {shape} {precision}'
    bad = []
    if shape == 'uniform8x1378':
        B, T = 8, BENCH_FRAMES
        mel, f0, ri, nz = ragged_inputs(h, [T] * B)
        y, plan = verbose_run(m, mel, f0, ri, nz, None, monkeypatch, capfd)
        judge(tag, precision, group_errors(m, h, w, mel, y[:, None].cuda()), capfd, bad)
    else:
        lengths = ragged_lengths(shape)
        T = max(lengths)
        mel, f0, ri, nz = ragged_inputs(h, lengths)
        y, plan = verbose_run(m, mel, f0, ri, nz, lengths, monkeypatch, capfd)
        if shape == 'past_2gib':
            st3 = m.get_tap('stage3')
            nbytes, last = st3.numel() * 4, (st3.shape[0] - 1) * st3[0].numel() * 4
            del st3
            say(capfd, f'MEASURED {tag}: stage-3 activations {nbytes / 2**30:.2f} GiB, the last clip from byte {last} '
                       f'(2^31 = {2**31})')
            assert last > 2**31
        clips = float64_clips(shape, lengths)
        judge(f'{tag} clips {clips}', precision, subset_errors(m, h, w, mel, y, lengths, clips), capfd, bad)
        differ = []
        for b, L in enumerate(lengths):
            one = alone(m, h, mel, f0, ri, nz, b, L, True)
            if not bits_equal(y[b, :L * hop], one):
                d = (y[b, :L * hop] - one).abs()
                differ.append(f'clip {b} (L {L}): {int((d > 0).sum())} samples differ, max {float(d.max()):.3e} at frame '
                              f'{int(d.argmax()) // hop}')
            assert (y[b, L * hop:] == 0).all()
        assert not differ, '\n'.join(differ)
    sched = schedules(h, T, plan)
    say(capfd, f'SCHEDULE {tag}: {sched}')
    assert not bad, '\n'.join(bad)
    assert sched == SCHEDULE[shape, precision], sched


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3'])
def test_per_clip_linf_sees_a_fault_past_row_2_17_of_a_max_frames_take(precision, monkeypatch, capfd):
    """2e-3 x max |ref| added to one 16-row x 32-channel piece of the stage-3 tap of the 5000-frame clip, at row 140 848 (tile
    1100, past 2^17): the per-clip L-inf check fails it by MARGIN, among 640 000 rows."""
    m, h = make_model('hop128', precision, monkeypatch)
    w = ref_weights(m)
    lengths = ragged_lengths('max_frames_among_short')
    mel, f0, ri, nz = ragged_inputs(h, lengths)
    run(m, mel, f0, ri, nz, lengths)
    b = lengths.index(MAX_FRAMES)
    L = MAX_FRAMES * hop_of(h)
    ups, got = m.get_tap('ups3')[b:b + 1, :, :L].clone(), m.get_tap('stage3')[b:b + 1, :, :L].clone()
    ref = O.stage_forward(w, h, 3, ups.double())
    li = BARS[precision]['stage3'][0]
    clean = compare(got, lambda _: ref)
    assert clean[0] <= li, describe('clean', 'stage3', clean)
    r0 = 1100 * 128 + 3 * 16
    assert r0 > 2**17
    faulty = got.clone()
    faulty[0, :32, r0:r0 + 16] += 2e-3 * float(ref.abs().max())
    res = compare(faulty, lambda _: ref)
    say(capfd, f'MEASURED {describe(f"hop128 5000-frame take {precision} one faulty piece", "stage3", res)}: '
               f'{res[0] / li:.1f} x its bar')
    assert r0 <= res[2][2] < r0 + 16, res
    assert res[0] >= MARGIN * li, res


# ------------------------------------------------------------------ 5. denoise at the singing configuration
# Worst |got - oracle| over the cases below, measured on an H100 80GB HBM3 at a 700 W power limit: 3.0e-7 (v 0.1 and 0.5, clip 2
# of the B = 3 call; 2.1e-7 for the max_frames take); exact silence gives exactly 0.  The bar is about 4x that.
DENOISE_BAR = 1.2e-6


def denoise_batch(x, v):
    """svb_denoise of the rows of x [B, n] in ONE call, at the singing STFT.  (A row need not equal its own B = 1 call bit for
    bit: the overlap-add sums each sample's n_fft / hop frames with atomics, in no fixed order.)"""
    c = _native.StftConfig(HP['fft_size'], HOP, HP['win_size'], ZERO, _native.OUT_MAG_RAW, 0, 0, 1, 0.0)
    x = x.cuda().contiguous()
    out = torch.full((x.shape[0], HOP * (x.shape[1] // HOP)), float('nan'), device='cuda')
    _native.check(_native.lib().svb_denoise(ctypes.byref(c), _native.ptr(x), x.shape[0], x.shape[1], ctypes.c_float(v),
                                            _native.ptr(out), None), 'denoise')
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize('v', [0.1, 0.5])
def test_denoise_at_the_singing_stft_matches_oracle(v, capfd):
    from neuralsvb_b200.vocoders.vocoder_utils import denoise_device
    cases = {'max_frames take': S.make_clip(MAX_FRAMES * HOP, seed=1),
             'length off the hop': S.make_clip(100_001, seed=2),
             'one hop + 1': S.make_clip(HOP + 1, seed=3),
             'silence': np.zeros(20_000, np.float32)}
    worst = {}
    for name, x in cases.items():
        got = denoise_device(torch.from_numpy(x).cuda(), v, HP).cpu().numpy()
        ref = FE.denoise(x, v, HP['fft_size'], HOP, HP['win_size'])
        assert got.shape == ref.shape == (HOP * (len(x) // HOP),)
        worst[name] = float(np.abs(got - ref).max())
        if name == 'silence':
            assert not got.any()
    three = np.stack([S.make_clip(30_000, seed=s) * a for s, a in ((4, 1.0), (5, 0.3), (6, 2.0))])
    got = denoise_batch(torch.from_numpy(three), v)
    for b in range(3):
        ref = FE.denoise(three[b], v, HP['fft_size'], HOP, HP['win_size'])
        worst[f'B = 3, clip {b}'] = float(np.abs(got[b] - ref).max())
    say(capfd, f'MEASURED denoise v {v}: ' + ', '.join(f'{k} {e:.2e}' for k, e in worst.items()))
    assert max(worst.values()) < DENOISE_BAR, worst


# ------------------------------------------------------------------ 6. the longest mel spec2wav takes
SONG_FRAMES = 70_000                                         # 6.8 minutes at hop 128, past gridDim.y's 65 535


def song_vocoder(precision):
    h = S.hifigan_config(False, hop=128)
    gm = HifiGanGenerator(h, precision=precision)
    gm.load_state_dict(S.make_generator_state_dict(h, U.SEED), strict=True)
    with contextlib.redirect_stdout(io.StringIO()):
        gm.remove_weight_norm()
    return HifiGAN.from_model(gm.eval().cuda(), h), h


def receptive_frames(h):
    """Frames of mel on each side that reach one output sample of the generator without NSF, from its kernel sizes and
    dilations: conv_pre, then per stage the transposed conv (input rows within ceil(k / u) + 1 of an output row) and the
    widest ResBlock (sum over its steps of the c1 and c2 halos), then conv_post, each in rows of its own rate."""
    halo = 3.0                                                   # conv_pre, k 7
    R = 1
    for u, k in zip(h['upsample_rates'], h['upsample_kernel_sizes']):
        halo += (math.ceil(k / u) + 1) / R
        R *= u
        rb = max((kk - 1) // 2 * sum(d + 1 for d in dil) for kk, dil in zip(h['resblock_kernel_sizes'],
                                                                           h['resblock_dilation_sizes']))
        halo += rb / R
    halo += 3 / R                                                # conv_post, k 7
    return math.ceil(halo)


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3', 'fp32'])
def test_spec2wav_of_a_70000_frame_mel_matches_excerpts(precision, capfd):
    """The frame-major mel is converted by a kernel that strides over the frames (a grid of one block row per frame stopped
    at 65 535 frames).  On the tensor-core precisions one clip of 70 000 frames has more work items in a conv than one launch
    lists (the 32-channel stage has 70 000 128-row tiles), so those convs run in slices of rows.  Rows are independent of
    the call they are computed in beyond the receptive field: samples of inner windows of the song (across each slice
    boundary, and past frame 65 535) equal spec2wav of a mel excerpt around them with margins wider
    than that field (excerpts start on 16-frame boundaries, so every stage's tiles line up as in the song, and are short
    enough to run each conv in one launch); the ragged host entry gives the song beside a short clip bit for bit."""
    voc, h = song_vocoder(precision)
    hop = hop_of(h)
    mel = S.make_mel_f0(1, SONG_FRAMES, U.SEED)[0][0].T.contiguous().numpy()       # frame-major [T, 80]
    t0 = time.time()
    y = voc.spec2wav(mel)
    say(capfd, f'MEASURED spec2wav of {SONG_FRAMES} frames ({precision}): {time.time() - t0:.2f} s')
    assert y.shape == (SONG_FRAMES * hop,) and np.isfinite(y).all()
    rf = receptive_frames(h)
    margin = rf + 16
    # On a 132-SM H100 a slice is 120 x 132 tiles of 128 rows = 2 027 520 rows: the first slice of stage 3 (128 rows a frame)
    # ends at frame 15 840, of stage 2 and its upsampler (64) at 31 680, of stage 1 (32) at 63 360; windows straddle each
    # (other SM counts move the boundaries; the windows still hold)
    bad = []
    for w0, w1 in ((0, 200), (15_800, 15_900), (31_650, 31_750), (63_300, 63_400), (65_500, 65_600), (69_800, SONG_FRAMES)):
        s = max(0, (w0 - margin) // 16 * 16)
        e = min(SONG_FRAMES, w1 + margin)
        assert w0 - s >= rf or s == 0
        assert e - w1 >= rf or e == SONG_FRAMES
        part = voc.spec2wav(mel[s:e])
        if not bits_equal(torch.from_numpy(y[w0 * hop:w1 * hop]), torch.from_numpy(part[(w0 - s) * hop:(w1 - s) * hop])):
            d = np.abs(y[w0 * hop:w1 * hop] - part[(w0 - s) * hop:(w1 - s) * hop])
            bad.append(f'frames [{w0}, {w1}) from excerpt [{s}, {e}): max {d.max():.3e} at frame {w0 + int(d.argmax()) // hop}')
    short = mel[:77]
    got = voc.spec2wav_batch([short, mel])
    assert bits_equal(torch.from_numpy(got[1]), torch.from_numpy(y)), 'ragged spec2wav of the song differs from spec2wav'
    assert bits_equal(torch.from_numpy(got[0]), torch.from_numpy(voc.spec2wav(short)))
    say(capfd, f'MEASURED spec2wav excerpts {precision}: receptive field {rf} frames a side, margins {margin}: {len(bad)} '
               f'windows differ')
    assert not bad, '\n'.join(bad)

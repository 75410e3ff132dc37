"""-m gpu: the fused STFT front end (svb_stft_forward = stft_mel_v2_kernel, svb_stft_backward = stft_mel_bwd_kernel,
svb_wav2spec_batch) against float64 torch.stft on the same fp32 waveform, per output kind and padding mode as
include/svb_vocoder.h documents them, at the product configurations and at the edges of the kernels: n_fft 64 / 4096,
mel filters read from global memory, hops that do not divide n_fft, partial last CTAs, the shortest legal reflect clips,
input clamping, empty mel rows, silence (magnitude floor and log clamps) and ragged batches.  The backward is compared
with float64 autograd of the same function for a random cotangent."""
import ctypes
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200 import _native
from neuralsvb_b200.utils import audio

pytestmark = pytest.mark.gpu

ZERO, REFLECT, HALF = _native.PAD_CENTER_ZERO, _native.PAD_CENTER_REFLECT, _native.PAD_HALF_REFLECT
LOG10_MEL, LN_MEL, MAG, MAG_RAW, MEL_MAG = (_native.OUT_LOG10_MEL, _native.OUT_LN_MEL, _native.OUT_MAG, _native.OUT_MAG_RAW,
                                            _native.OUT_MEL_MAG)
MEL_KINDS = (LOG10_MEL, LN_MEL, MEL_MAG)
# Every value a clamp compares with eps lies outside [eps / 1.15, 1.15 eps] (or is exactly 0, a fully silent frame, which is
# exactly 0 in fp32 too).  The fp32 error of a bin's power is relative to its frame's energy: ~1e-2 of the power of a bin
# near the 1e-7 floor in a loud 2048-point frame, far less in the quiet frames at the edges of silence.
EPS_MARGIN = 1.15


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


# ------------------------------------------------------------------ float64 reference
def stft_reference(wav, cfg, basis):
    """float64 output of svb_stft_forward for cfg = (n_fft, hop, win, pad_mode, out_kind, clamp_input, n_mels, frames_major,
    eps) on wav [B, n] (any dtype: computed in float64, on wav's device), and the tensor each eps clamp compares (or None).
    basis [n_mels, n_fft/2+1] (fp32 values, upcast) or None."""
    n_fft, hop, win, mode, kind, clamp, n_mels, frames_major, eps = cfg
    eps = float(np.float32(eps))                           # the kernel sees the fp32 value
    x = wav.double()
    if clamp:
        x = x.clamp(-1.0, 1.0)
    window = torch.hann_window(win, periodic=True, dtype=torch.float64, device=wav.device)
    if mode == HALF:
        p = (n_fft - hop) // 2
        x = F.pad(x[:, None], (p, p), mode='reflect')[:, 0]
        X = torch.stft(x, n_fft, hop, win, window, center=False, return_complex=True)
    else:
        X = torch.stft(x, n_fft, hop, win, window, center=True, pad_mode='constant' if mode == ZERO else 'reflect',
                       return_complex=True)
    pw = X.real ** 2 + X.imag ** 2                         # [B, bins, frames]
    bd = None if basis is None else basis.double().to(wav.device)
    if kind == LOG10_MEL:
        arg = bd @ pw.sqrt()
        out = torch.log10(torch.clamp(arg, min=eps))
    elif kind == LN_MEL:
        arg = bd @ torch.sqrt(pw + 1e-9)
        out = torch.log(torch.clamp(arg, min=eps))
    elif kind == MAG:
        arg = pw
        out = torch.sqrt(torch.clamp(pw, min=eps))
    elif kind == MEL_MAG:
        arg = pw
        out = bd @ torch.sqrt(torch.clamp(pw, min=eps))
    else:
        arg, out = None, pw.sqrt()
    if frames_major:
        out = out.transpose(1, 2)
    return out.contiguous(), (None if arg is None else arg.detach() / eps)


def assert_clear_of_eps(ratio, what):
    """fp32 and float64 may only disagree about a clamp when the clamped value is within rounding of eps."""
    if ratio is None:
        return
    near = (ratio != 0) & (ratio > 1 / EPS_MARGIN) & (ratio < EPS_MARGIN)
    assert not bool(near.any()), f'{what}: {int(near.sum())} reference values within a factor {EPS_MARGIN} of eps'


def packed_filter_values(basis):
    """Values mel_pack_kernel keeps: every row from its first to its last non-zero bin."""
    nz = basis != 0
    idx = torch.arange(basis.shape[1])
    first = torch.where(nz, idx, basis.shape[1]).min(1).values
    last = torch.where(nz, idx, -1).max(1).values
    return int(torch.clamp(last - first + 1, min=0).sum())


# ------------------------------------------------------------------ inputs
def make_wave(B, n, key, kind='wave'):
    """B different clips: a few harmonics at a random pitch + noise, peak near 0.6; 'loud' scales them beyond +-1 and
    sets samples to exactly +-1; 'silence' zeroes two segments (one at the start)."""
    g = _gen('wave', B, n, key)
    t = torch.arange(n, dtype=torch.float64) / 22050
    f0 = 80 + 400 * torch.rand(B, 1, generator=g, dtype=torch.float64)
    ph = 2 * np.pi * torch.rand(B, 5, generator=g, dtype=torch.float64)
    y = sum(0.25 / h * torch.sin(2 * np.pi * h * f0 * t + ph[:, h - 1:h]) for h in range(1, 6))
    y = y + 0.05 * torch.randn(B, n, generator=g, dtype=torch.float64)
    if kind == 'loud':
        y = 2.5 * y
        y[:, 5::97], y[:, 11::89] = 1.0, -1.0
    elif kind == 'silence':
        y[:, :1100] = 0
        y[:, n // 2 - 700:n // 2 + 1300] = 0
    return y.float()


def make_basis(kind, n_fft, n_mels):
    n_bins = n_fft // 2 + 1
    if kind is None:
        return None
    if kind == 'loss80':                                   # the vocoder's mel-loss basis (fmin 80, fmax 7600)
        b = audio.mel_filterbank(22050, n_fft, 80, 80, 7600)
    elif kind == 'full80':                                 # the use_mel_loss basis, librosa.filters.mel(22050, n_fft, 80)
        b = audio.mel_filterbank(22050, n_fft, 80, 0, 11025)
    elif kind == 'zero_rows':
        b = audio.mel_filterbank(22050, n_fft, 80, 0, 11025).copy()
        b[0], b[41] = 0, 0
    else:                                                  # 'dense': every bin non-zero
        b = np.abs(torch.randn(n_mels, n_bins, generator=_gen('basis', n_fft, n_mels)).numpy()) * (2.0 / n_bins)
    return torch.from_numpy(np.array(b, dtype=np.float32))


# (tag, cfg, n, B, basis, signal, backward); cfg = (n_fft, hop, win, pad_mode, out_kind, clamp_input, n_mels, frames_major, eps)
CASES = [
    # product configurations
    ('mel_loss_ln_half_clamp', (1024, 256, 1024, HALF, LN_MEL, 1, 80, 0, 1e-5), 8192, 2, 'loss80', 'wave', True),
    ('mr_mag_1024', (1024, 120, 600, REFLECT, MAG, 0, 0, 1, 1e-7), 8192, 2, None, 'wave', True),
    ('mr_mag_2048', (2048, 240, 1200, REFLECT, MAG, 0, 0, 1, 1e-7), 8192, 2, None, 'wave', True),
    ('mr_mag_512', (512, 50, 240, REFLECT, MAG, 0, 0, 1, 1e-7), 8192, 2, None, 'wave', True),
    ('mr_melmag_1024', (1024, 120, 600, REFLECT, MEL_MAG, 0, 80, 1, 1e-7), 8192, 2, 'full80', 'wave', True),
    ('mr_melmag_2048', (2048, 240, 1200, REFLECT, MEL_MAG, 0, 80, 1, 1e-7), 8192, 2, 'full80', 'wave', True),
    ('mr_melmag_512', (512, 50, 240, REFLECT, MEL_MAG, 0, 80, 1, 1e-7), 8192, 2, 'full80', 'wave', True),
    ('wav2spec_log10_zero', (1024, 256, 512, ZERO, LOG10_MEL, 0, 80, 0, 1e-10), 8192, 2, 'loss80', 'wave', False),
    ('mag_raw_zero', (1024, 256, 512, ZERO, MAG_RAW, 0, 0, 1, 0.0), 8192, 2, None, 'wave', False),
    # n_fft 64 and 4096 (the backward's full 9 bins per thread; 80 triangular filters pack 4003 values <= the 4096 cap)
    ('nfft64_mag', (64, 16, 64, REFLECT, MAG, 0, 0, 1, 1e-7), 1000, 2, None, 'wave', True),
    ('nfft64_melmag_dense', (64, 16, 48, ZERO, MEL_MAG, 0, 7, 0, 1e-7), 1000, 2, 'dense', 'wave', True),
    ('nfft4096_mag', (4096, 1024, 4096, REFLECT, MAG, 0, 0, 1, 1e-7), 16384, 2, None, 'wave', True),
    ('nfft4096_ln_mel_shared_filters', (4096, 1024, 4096, HALF, LN_MEL, 0, 80, 0, 1e-5), 16384, 2, 'full80', 'wave', True),
    # filters beyond the shared-memory cap: read from global memory
    ('global_filters_2048', (2048, 512, 2048, REFLECT, MEL_MAG, 0, 5, 1, 1e-7), 8192, 2, 'dense', 'wave', True),
    ('global_filters_4096_ln', (4096, 1024, 3000, HALF, LN_MEL, 0, 3, 0, 1e-5), 16384, 2, 'dense', 'wave', True),
    # hop not dividing n_fft, odd n_fft - win
    ('hop300_win1001', (1024, 300, 1001, REFLECT, MAG, 0, 0, 1, 1e-7), 7000, 2, None, 'wave', True),
    ('hop300_win1001_half_ln', (1024, 300, 1001, HALF, LN_MEL, 1, 80, 0, 1e-5), 7000, 2, 'loss80', 'wave', True),
    # frame counts 1, 2, 3 (mod 4): a partial last CTA
    ('frames9', (1024, 256, 1024, ZERO, MEL_MAG, 0, 80, 0, 1e-7), 2048, 2, 'full80', 'wave', True),
    ('frames10', (1024, 256, 1024, REFLECT, MAG, 0, 0, 0, 1e-7), 2304, 2, None, 'wave', True),
    ('frames11', (1024, 256, 1024, HALF, LN_MEL, 1, 80, 1, 1e-5), 2816, 2, 'loss80', 'wave', True),
    # the shortest legal clips of the reflect modes: n = reach + 1
    ('shortest_center_reflect', (1024, 256, 1024, REFLECT, MAG, 0, 0, 1, 1e-7), 513, 2, None, 'wave', True),
    ('shortest_half_reflect', (1024, 256, 1024, HALF, LN_MEL, 1, 80, 0, 1e-5), 385, 2, 'loss80', 'wave', True),
    # input clamp with samples beyond and exactly at +-1
    ('clamp_loud', (1024, 256, 1024, HALF, LN_MEL, 1, 80, 0, 1e-5), 8192, 2, 'loss80', 'loud', True),
    ('clamp_loud_mag', (512, 128, 512, REFLECT, MAG, 1, 0, 1, 1e-7), 4096, 2, None, 'loud', True),
    # mel rows that are all zero
    ('zero_mel_rows', (1024, 256, 1024, REFLECT, MEL_MAG, 0, 80, 1, 1e-7), 4096, 2, 'zero_rows', 'wave', True),
    ('zero_mel_rows_ln', (1024, 256, 1024, HALF, LN_MEL, 0, 80, 0, 1e-5), 4096, 2, 'zero_rows', 'wave', True),
    # B > 1, different content per clip
    ('batch5', (1024, 256, 1024, HALF, LN_MEL, 1, 80, 0, 1e-5), 4096, 5, 'loss80', 'wave', True),
    # exact silence: magnitude floor and log clamps
    ('silence_ln_mel', (1024, 256, 1024, HALF, LN_MEL, 1, 80, 0, 1e-5), 8192, 2, 'loss80', 'silence', True),
    ('silence_mag', (1024, 120, 600, REFLECT, MAG, 0, 0, 1, 1e-7), 8192, 2, None, 'silence', True),
    ('silence_melmag', (512, 50, 240, REFLECT, MEL_MAG, 0, 80, 1, 1e-7), 8192, 2, 'full80', 'silence', True),
    ('silence_log10', (1024, 256, 1024, ZERO, LOG10_MEL, 0, 80, 0, 1e-10), 8192, 2, 'loss80', 'silence', False),
]

# Bars (rel L2, rel L-inf), about 5x the worst error measured over CASES on an H100 80GB HBM3 (400 W power limit):
#   out  5.4e-7 / 1.2e-6 (mel filters from global memory; 1e-7 / 4e-7 elsewhere, the ragged batch included)
#   dwav 1.6e-6 / 3.1e-6, except the three cases below: 2.7e-6 / 6.4e-6, 8.0e-6 / 1.3e-5 and 1.1e-5 / 6.7e-6.  Those are
#        the conditioning of the function in float32, not the kernel: the same float32 function through torch.stft on the CPU
#        lands at 1.6e-6 / 4.0e-6, 9.2e-6 / 1.3e-5 and 2.6e-5 / 1.8e-5 against the float64 reference (the ln-mel gradient is
#        scaled by 1 / mel, large in the quiet frames at the edges of silence).
FWD_TOL = (3e-6, 6e-6)
BWD_TOL = (8e-6, 1.6e-5)
BWD_TOL_ILL = {'hop300_win1001': (1.4e-5, 3.2e-5), 'hop300_win1001_half_ln': (4e-5, 7e-5), 'silence_ln_mel': (6e-5, 3.5e-5)}


def case_inputs(case):
    tag, cfg, n, B, basis_kind, signal, _ = case
    wav = make_wave(B, n, tag, signal)
    basis = make_basis(basis_kind, cfg[0], cfg[6])
    return wav, basis


def frames_of(cfg, n):
    return int(_native.lib().svb_stft_num_frames(ctypes.byref(_native.StftConfig(*cfg)), n))


def run_forward(cfg, wav, basis):
    B, n = wav.shape
    n_out = cfg[6] if cfg[4] in MEL_KINDS else cfg[0] // 2 + 1
    fr = frames_of(cfg, n)
    out = torch.full((B, fr, n_out) if cfg[7] else (B, n_out, fr), float('nan'), device='cuda')
    _native.check(_native.lib().svb_stft_forward(ctypes.byref(_native.StftConfig(*cfg)), _native.ptr(wav), B, n, _native.ptr(basis),
                                                 _native.ptr(out), None), 'stft_forward')
    return out


def run_wav2spec(c, wav, lengths, basis, mel, wav_out=None, frames=None):
    """svb_wav2spec_batch (StftConfig c) of the clips back to back in the CUDA tensor wav, into the CUDA tensors mel / wav_out and
    the host int64 array frames (both may be None), with a workspace of the size svb_wav2spec_workspace_bytes gives -> its return
    value."""
    lib = _native.lib()
    lens = np.ascontiguousarray(lengths, np.int64)
    ws = lib.svb_wav2spec_workspace_bytes(ctypes.byref(c), lens.ctypes.data_as(ctypes.c_void_p), len(lens), None)
    buf = torch.empty(int(ws), dtype=torch.uint8, device='cuda')
    return lib.svb_wav2spec_batch(ctypes.byref(c), _native.ptr(wav), lens.ctypes.data_as(ctypes.c_void_p), len(lens), _native.ptr(basis),
                                  _native.ptr(mel), _native.ptr(wav_out), None if frames is None else frames.ctypes.data_as(ctypes.c_void_p),
                                  ctypes.c_void_p(buf.data_ptr()), int(ws), None)


def run_backward(cfg, wav, basis, dout):
    B, n = wav.shape
    dwav = torch.zeros_like(wav)
    _native.check(_native.lib().svb_stft_backward(ctypes.byref(_native.StftConfig(*cfg)), _native.ptr(wav), B, n, _native.ptr(basis),
                                                  _native.ptr(dout), _native.ptr(dwav), None), 'stft_backward')
    return dwav


def errors(got, ref):
    d = got.double() - ref
    return float(d.norm() / ref.norm()), float(d.abs().max() / ref.abs().max())


def _within(e, tol):
    return e[0] <= tol[0] and e[1] <= tol[1]


@pytest.mark.parametrize('case', CASES, ids=lambda c: c[0])
def test_stft_forward_and_backward_match_float64_torch(case):
    tag, cfg, n, B, basis_kind, signal, backward = case
    wav, basis = case_inputs(case)
    if tag.startswith('global_filters'):
        assert packed_filter_values(basis) > 4096                               # filters from global memory
    if cfg[0] == 4096 and basis_kind == 'full80':
        assert packed_filter_values(basis) <= 4096                              # filters from shared memory
    wav_d = wav.cuda()
    basis_d = None if basis is None else basis.cuda()
    ref, ratio = stft_reference(wav_d, cfg, basis_d)
    assert_clear_of_eps(ratio, tag)
    out = run_forward(cfg, wav_d, basis_d)
    assert out.shape == ref.shape
    e = {'out': errors(out, ref)}
    if backward:
        dout = torch.randn(out.shape, generator=_gen('dout', tag)).cuda()
        dwav = run_backward(cfg, wav_d, basis_d, dout)
        w64 = wav_d.double().requires_grad_(True)
        stft_reference(w64, cfg, basis_d)[0].backward(dout.double())
        e['dwav'] = errors(dwav, w64.grad)
    print('MEASURED', tag, {k: f'{a:.2e}/{b:.2e}' for k, (a, b) in e.items()})
    assert _within(e['out'], FWD_TOL), (tag, e)
    assert not backward or _within(e['dwav'], BWD_TOL_ILL.get(tag, BWD_TOL)), (tag, e)


def test_wav2spec_ragged_batch_matches_single_clip_device_calls_and_float64_torch():
    """Clips of 1-5 frames between long ones in ONE launch: every clip's block range is found by the binary search over the
    clip table; each clip must equal its own single-clip call (bit for bit) and the float64 reference."""
    cfg = (1024, 256, 1024, ZERO, LOG10_MEL, 0, 80, 1, 1e-10)
    c = _native.StftConfig(*cfg)
    lengths = [8192, 1, 300, 5000, 600, 773, 1024, 7001, 17, 1280, 4096]
    clips = [make_wave(1, L, ('ragged', i))[0] for i, L in enumerate(lengths)]
    basis = make_basis('loss80', 1024, 80).cuda()
    wav_cat = torch.cat(clips).cuda()
    fr = np.zeros(len(lengths), np.int64)
    total = sum(1 + L // 256 for L in lengths)
    mel = torch.full((total, 80), float('nan'), device='cuda')
    got = run_wav2spec(c, wav_cat, lengths, basis, mel, frames=fr)
    assert _native.check(got, 'wav2spec_batch') == total
    assert fr.tolist() == [1 + L // 256 for L in lengths] and {1, 2, 3, 4, 5} <= set(fr.tolist())
    off = 0
    worst = (0.0, 0.0)
    for i, (L, x) in enumerate(zip(lengths, clips)):
        m = mel[off:off + fr[i]]
        off += fr[i]
        single = torch.full((fr[i], 80), float('nan'), device='cuda')
        assert run_wav2spec(c, x.cuda(), [L], basis, single) == fr[i]
        assert torch.equal(m, single), f'clip {i} (length {L}) differs from its single-clip call'
        ref, ratio = stft_reference(x[None].cuda(), cfg, basis)
        assert_clear_of_eps(ratio, f'clip {i}')
        e = errors(m, ref[0])
        worst = max(worst, e)
        assert _within(e, FWD_TOL), (i, L, e)
    print('MEASURED ragged', f'{worst[0]:.2e}/{worst[1]:.2e}')

"""The resampling oracle (oracle/resample.py) against a literal transcription of resampy 0.2.2's loop, its lengths, filter and
signal properties, WAV decoding, the C ABI's host-side plan, and the binarizer's header-based grouping.  No GPU."""
import ctypes
import math

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import resample as R

RATES = [(48000, 22050), (44100, 22050), (32000, 22050), (16000, 22050), (8000, 22050), (44100, 24000)]


def scalar_resample(x, sr_orig, sr_new):
    """resampy.resample + interpn.resample_f + librosa's fix_length, transcribed line by line (one channel)."""
    win, num_table = R.sinc_window(**R.KAISER_BEST)
    sample_ratio = float(sr_new) / sr_orig
    n_res = int(len(x) * sample_ratio)
    if n_res < 1:
        raise ValueError('too short')
    y = np.zeros(n_res, np.float32)
    interp_win = np.array(win)
    if sample_ratio < 1:
        interp_win *= sample_ratio
    interp_delta = np.zeros_like(interp_win)
    interp_delta[:-1] = np.diff(interp_win)
    scale = min(1.0, sample_ratio)
    time_increment = 1. / sample_ratio
    index_step = int(scale * num_table)
    time_register = 0.0
    nwin = interp_win.shape[0]
    n_orig = x.shape[0]
    for t in range(n_res):
        n = int(time_register)
        frac = scale * (time_register - n)
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        i_max = min(n + 1, (nwin - offset) // index_step)
        for i in range(i_max):
            weight = (interp_win[offset + i * index_step] + eta * interp_delta[offset + i * index_step])
            y[t] = np.float32(float(y[t]) + weight * float(x[n - i]))
        frac = scale - frac
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        k_max = min(n_orig - n - 1, (nwin - offset) // index_step)
        for k in range(k_max):
            weight = (interp_win[offset + k * index_step] + eta * interp_delta[offset + k * index_step])
            y[t] = np.float32(float(y[t]) + weight * float(x[n + k + 1]))
        time_register += time_increment
    out = np.zeros(int(np.ceil(len(x) * sample_ratio)), np.float32)
    out[:n_res] = y
    return out


def _clip(n, seed):
    rs = np.random.RandomState(seed)
    t = np.arange(n)
    return (0.4 * np.sin(0.05 * t + rs.uniform(0, 6)) + 0.1 * rs.standard_normal(n)).astype(np.float32)


@pytest.mark.parametrize('sr,target', RATES)
def test_vectorised_oracle_is_the_scalar_loop_bit_for_bit(sr, target):
    # 601 samples reach past both wings in the middle; 97 is shorter than one wing (64 .. 139 input samples), so both min() clamps bind
    for n, seed in ((601, 1), (97, 2)):
        x = _clip(n, seed)
        got, want = R.resample(x, sr, target), scalar_resample(x, sr, target)
        assert got.dtype == np.float32 and got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (sr, target, n)


def test_time_register_is_the_sequential_sum():
    inc = 1.0 / (22050.0 / 48000)
    tr, acc = R.time_register(5000, inc), 0.0
    for t in range(5000):
        assert tr[t] == acc
        acc += inc
    # and it is not t * increment
    assert not np.array_equal(tr, np.arange(5000) * inc)


@pytest.mark.parametrize('sr,target', RATES + [(96000, 22050)])
def test_output_lengths(sr, target):
    ratio = float(target) / sr
    for n in (1001, 44101, 48001):
        n_res, n_out = R.lengths(n, sr, target)
        assert n_res == int(n * ratio) and n_out == int(math.ceil(n * ratio))
        y = R.resample(_clip(n, 3), sr, target) if n == 1001 else None
        if y is not None:
            assert len(y) == n_out and np.all(y[n_res:] == 0)


def test_equal_rates_return_the_input():
    x = _clip(1001, 4)
    assert R.resample(x, 22050, 22050) is x
    assert R.lengths(1001, 22050, 22050) == (1001, 1001)


def test_a_clip_that_yields_no_sample_raises():
    n = R.min_length(96000, 22050)
    assert n == 5
    R.resample(_clip(n, 5), 96000, 22050)
    with pytest.raises(ValueError):
        R.resample(_clip(n - 1, 5), 96000, 22050)


def test_filter_table():
    win, num_table = R.sinc_window(**R.KAISER_BEST)
    rolloff = R.KAISER_BEST['rolloff']
    assert win.dtype == np.float64 and len(win) == 32769 and num_table == 512
    assert win[0] == rolloff
    # the zero crossings of sinc(rolloff x) sit at x = m / rolloff, i.e. index 512 m / rolloff
    sign = np.nonzero(np.diff(np.sign(win)) != 0)[0]
    expect = [512 * m / rolloff for m in range(1, 61)]
    assert len(sign) >= 60
    for s, e in zip(sign, expect):
        assert abs(s + 0.5 - e) < 1.0, (s, e)


def test_package_window_is_the_oracle_window():
    from neuralsvb_b200.utils import audio
    win, num_table = audio.kaiser_best_window()
    ow, ont = R.sinc_window(**R.KAISER_BEST)
    assert num_table == ont and np.array_equal(win.view(np.uint64), ow.view(np.uint64))


def _sine(f, sr, seconds=1.0, amp=0.5):
    return (amp * np.sin(2 * np.pi * f * np.arange(int(sr * seconds)) / sr)).astype(np.float32)


@pytest.mark.parametrize('sr,target,bar', [(44100, 22050, 2e-6), (48000, 22050, 5e-4)])
def test_passband_sine_matches_the_analytic_sine(sr, target, bar):
    # measured max |error| over samples 500 .. n - 500 of a 0.5-amplitude 1 kHz sine: 4.9e-7 at 44.1 kHz (every output at the
    # table's zero phase) and 2.5e-4 at 48 kHz (the table's linear interpolation between phases); the bars are 4x and 2x that
    y = R.resample(_sine(1000.0, sr), sr, target)
    ref = 0.5 * np.sin(2 * np.pi * 1000.0 * np.arange(len(y)) / target)
    assert np.abs(y[500:-500] - ref[500:-500]).max() < bar


@pytest.mark.parametrize('f', [12000.0, 15000.0])
def test_a_tone_above_the_rolloff_is_attenuated(f):
    # 44.1 -> 22.05 kHz: rolloff x Nyquist = 10447 Hz.  Measured output / input RMS: 9.4e-8 at 12 kHz, 2.7e-8 at 15 kHz (below
    # -140 dB); the bar is 1e-6 (-120 dB)
    x = _sine(f, 44100)
    y = R.resample(x, 44100, 22050)
    assert np.sqrt((y[500:-500] ** 2).mean()) / np.sqrt((x ** 2).mean()) < 1e-6


# ---- decoding ---------------------------------------------------------------------------------------------------------------
def _write_24bit(path, sr, ints):
    """A 24-bit PCM WAV (scipy cannot write one)."""
    import struct
    b = b''.join(int(v).to_bytes(3, 'little', signed=True) for v in ints)
    fmt = struct.pack('<HHIIHH', 1, 1, sr, sr * 3, 3, 24)
    with open(path, 'wb') as f:
        f.write(b'RIFF' + struct.pack('<I', 4 + 8 + len(fmt) + 8 + len(b)) + b'WAVE')
        f.write(b'fmt ' + struct.pack('<I', len(fmt)) + fmt + b'data' + struct.pack('<I', len(b)) + b)


def test_decoding_follows_librosa(tmp_path):
    from neuralsvb_b200.utils import audio
    rs = np.random.RandomState(6)
    cases = {}
    i16 = rs.randint(-32768, 32768, 300).astype(np.int16)
    cases['i16'] = (i16, i16.astype(np.float64) / 2 ** 15)
    i32 = rs.randint(-2 ** 31, 2 ** 31, 300, dtype=np.int64).astype(np.int32)
    cases['i32'] = (i32, i32.astype(np.float64) / 2 ** 31)
    u8 = rs.randint(0, 256, 300).astype(np.uint8)
    cases['u8'] = (u8, (u8.astype(np.float64) - 128) / 128)
    f32 = rs.uniform(-1, 1, 300).astype(np.float32)
    cases['f32'] = (f32, f32.astype(np.float64))
    st = rs.randint(-32768, 32768, (300, 2)).astype(np.int16)
    cases['stereo'] = (st, (st[:, 0].astype(np.float64) + st[:, 1]) / 2 / 2 ** 15)
    for name, (data, want) in cases.items():
        p = str(tmp_path / f'{name}.wav')
        wavfile.write(p, 44100, data)
        for decode in (audio.read_wav, R.decode):
            got, sr = decode(p)
            assert sr == 44100 and got.dtype == np.float32 and got.ndim == 1
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-7 if name != 'i32' else 1e-7, err_msg=name)
        assert audio.wav_info(p) == (44100, 300, data.shape[1] if data.ndim > 1 else 1)
    i24 = rs.randint(-2 ** 23, 2 ** 23, 300)
    p = str(tmp_path / 'i24.wav')
    _write_24bit(p, 48000, i24)
    for decode in (audio.read_wav, R.decode):
        got, sr = decode(p)
        assert sr == 48000 and np.array_equal(got, (i24 / 2 ** 23).astype(np.float32))
    assert audio.wav_info(p) == (48000, 300, 1)


def test_load_wav_at_the_file_rate_needs_no_device(tmp_path):
    from neuralsvb_b200.utils import audio
    x = np.random.RandomState(7).randint(-32768, 32768, 500).astype(np.int16)
    p = str(tmp_path / 'a.wav')
    wavfile.write(p, 22050, x)
    for sr in (22050, None):
        y, got_sr = audio.load_wav(p, sr)
        assert got_sr == 22050 and np.array_equal(y, x.astype(np.float32) / 32768)


# ---- the C ABI's plan (host only) ---------------------------------------------------------------------------------------------
def _plan(target, srs, lens, nwin=32769, num_table=512):
    from neuralsvb_b200 import _native
    srs = np.ascontiguousarray(srs, np.int32)
    lens = np.ascontiguousarray(lens, np.int64)
    res, out = np.zeros(len(lens), np.int64), np.zeros(len(lens), np.int64)
    ws = _native.lib().svb_resample_plan(target, srs.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                                         len(lens), nwin, num_table, res.ctypes.data_as(ctypes.c_void_p),
                                         out.ctypes.data_as(ctypes.c_void_p))
    return ws, res, out


def test_plan_lengths_match_the_oracle():
    srs = [48000, 44100, 32000, 16000, 8000, 96000, 22050, 44100]
    lens = [48001, 1001, 32001, 16001, 801, 5, 777, 3]
    ws, res, out = _plan(22050, srs, lens[:-1] + [7])
    assert ws > 0
    for s, n, a, b in zip(srs, lens[:-1] + [7], res, out):
        assert (a, b) == R.lengths(n, s, 22050)
    # one table (32769 x 16 bytes) per distinct source rate other than the target
    assert ws >= 6 * 32769 * 16
    from neuralsvb_b200.utils import audio
    r2, o2 = audio.resample_lengths(lens[:-1], srs[:-1], 22050)
    assert list(o2) == [R.lengths(n, s, 22050)[1] for s, n in zip(srs[:-1], lens[:-1])]


@pytest.mark.parametrize('target,srs,lens,nwin,num_table', [
    (22050, [96000], [4], 32769, 512),          # yields no sample
    (22050, [44100], [1], 32769, 512),
    (0, [44100], [100], 32769, 512),            # bad target
    (22050, [0], [100], 32769, 512),            # bad source rate
    (22050, [-44100], [100], 32769, 512),
    (22050, [44100], [-1], 32769, 512),         # bad length
    (22050, [44100], [100], 1, 512),            # bad filter
    (22050, [44100], [100], 32769, 0),
    (100, [1000000], [10 ** 6], 32769, 512),    # ratio below 1 / num_table
])
def test_plan_refuses_bad_input(target, srs, lens, nwin, num_table):
    assert _plan(target, srs, lens, nwin, num_table)[0] == -1
    if nwin == 32769 and num_table == 512:
        from neuralsvb_b200.utils import audio
        with pytest.raises(ValueError):
            audio.resample_lengths(lens, srs, target)


# ---- the binarizer's grouping ---------------------------------------------------------------------------------------------------
def test_batches_read_seconds_from_the_wav_header(tmp_path, monkeypatch):
    from neuralsvb_b200.data_gen.tts.base_binarizer import VocoderBinarizer
    from neuralsvb_b200.utils.hparams import hparams
    monkeypatch.setitem(hparams, 'audio_sample_rate', 22050)
    paths = []
    for k in range(3):                         # 1 s each, at 44.1 kHz stereo: 4 s by the old file-size estimate
        p = str(tmp_path / f'{k}.wav')
        wavfile.write(p, 44100, np.zeros((44100, 2), np.int16))
        paths.append(p)
    b = VocoderBinarizer({}, binary_data_dir=str(tmp_path), batch_seconds=2.5)
    metas = [(f'i{k}', p, 0) for k, p in enumerate(paths)]
    assert [len(g) for g in b._batches(metas)] == [2, 1]
    arr = np.zeros(22050 * 2, np.float32)       # arrays are at audio_sample_rate: 2 s
    assert [len(g) for g in b._batches([('a', arr, 0), ('b', arr, 0)])] == [1, 1]

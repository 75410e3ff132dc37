"""ORACLE (test infrastructure only; see oracle/__init__.py): how the reference loads audio at the model's rate, in numpy.  The
CUDA path (csrc/resample.cu) implements the same text and is compared with this file bit for bit.

The reference reads every waveform with ``librosa.core.load(wav_path, sr=sample_rate)`` (data_gen/tts/data_gen_utils.py:111).  With
its pinned librosa 0.8.0 and resampy 0.2.2 that call folds the file to mono and resamples it with resampy's ``kaiser_best`` filter.
This file restates that call for WAV input.

Decode (``decode``).  WAV through ``scipy.io.wavfile``.  Integer PCM becomes float32 divided by 2^(bits - 1) (24-bit arrives from scipy
  as int32, left-justified, so it is divided by 2^31); uint8 becomes (x - 128) / 128; float WAV is cast to float32.  Several channels
  become their float32 mean, taken before resampling (``librosa.to_mono``).
Filter (``sinc_window``).  resampy's construction: num_bits = 2^precision, n = num_bits num_zeros,
  win = rolloff sinc(rolloff linspace(0, num_zeros, n + 1)) * kaiser(2 n + 1, beta)[n:], all float64.  ``kaiser_best`` is num_zeros 64,
  precision 9, beta 14.769656459379492, rolloff 0.9475937167399596: 32769 taps and num_table = 512.  resampy 0.2.2 loads this table
  from a precomputed ``kaiser_best.npz``; here it is regenerated from the construction with scipy's ``kaiser``.  Whether the two
  tables agree to the last bit has NOT been checked (resampy was not available where this was written); whoever has resampy 0.2.2
  can compare ``sinc_window()`` with its ``get_filter('kaiser_best')`` and ``resample`` with its output.
Resample (``resample``; resampy.resample + interpn.resample_f).
  sr == target: the input is returned unchanged.
  ratio = float(target) / sr; n_res = int(n_in ratio); n_res < 1 raises ValueError.
  ratio < 1: the table is multiplied by ratio.  delta[:-1] = diff(win), delta[-1] = 0.
  scale = min(1, ratio), index_step = int(scale num_table), time_increment = 1 / ratio.
  time_register starts at 0.0 and grows by ``+= time_increment`` once per output: a sequential float64 sum, not t * increment (the
  two differ once the increment is inexact).  Per output t:
    n = int(time_register), frac = scale (time_register - n), offset = int(frac num_table), eta = frac num_table - offset;
    left wing  i < min(n + 1, (nwin - offset) // index_step) over x[n - i], tap j = offset + i index_step;
    frac = scale - frac, with its own offset / eta;
    right wing k < min(n_in - n - 1, (nwin - offset) // index_step) over x[n + k + 1].
  Each tap: weight = win[j] + eta delta[j] in float64, then y = float32(float64(y) + weight float64(x)): the float32 output is
  rounded after every tap, with no fused multiply-add (numba's ``y[t] += weight * x`` into a float32 array).  Order: the left wing
  from i = 0, then the right wing from k = 0.
  Finally ``librosa.util.fix_length``: zero-pad to int(ceil(n_in ratio)).

The code below vectorises over t and loops over taps, which keeps the per-tap float32 rounding.
"""
import numpy as np

KAISER_BEST = dict(num_zeros=64, precision=9, beta=14.769656459379492, rolloff=0.9475937167399596)


def sinc_window(num_zeros=64, precision=9, beta=14.769656459379492, rolloff=0.9475937167399596):
    """(win float64 [num_table num_zeros + 1], num_table): the right wing of the windowed sinc."""
    from scipy.signal.windows import kaiser
    num_bits = 2 ** precision
    n = num_bits * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = kaiser(2 * n + 1, beta)[n:]
    return taper * sinc_win, num_bits


def decode(path):
    """(float32 mono samples, file rate) of a WAV file."""
    from scipy.io import wavfile
    sr, data = wavfile.read(path)
    if data.dtype.kind == 'i':
        data = data.astype(np.float32) / float(np.iinfo(data.dtype).max + 1)
    elif data.dtype.kind == 'u':
        data = (data.astype(np.float32) - 128.0) / 128.0
    data = data.astype(np.float32)
    if data.ndim > 1:
        data = data.mean(axis=1)
    return data, int(sr)


def lengths(n_in, sr, target):
    """(n_res, n_out): samples before and after fix_length."""
    if sr == target:
        return n_in, n_in
    ratio = float(target) / sr
    n_res = int(n_in * ratio)
    if n_res < 1:
        raise ValueError(f'Input signal length={n_in} is too small to resample from {sr}->{target}')
    return n_res, int(np.ceil(n_in * ratio))


def time_register(n_out, increment):
    """The sequential float64 sum: [0, inc, inc + inc, ...] (np.add.accumulate adds in order)."""
    tr = np.empty(n_out, np.float64)
    tr[0] = 0.0
    if n_out > 1:
        tr[1:] = np.add.accumulate(np.full(n_out - 1, increment, np.float64))
    return tr


def tables(ratio, win=None, num_table=512):
    """(scaled win, delta) of one ratio."""
    if win is None:
        win, num_table = sinc_window(**KAISER_BEST)
    win = np.array(win, np.float64)
    if ratio < 1:
        win *= ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    return win, delta


def _phase(frac, num_table):
    index_frac = frac * num_table
    offset = index_frac.astype(np.int64)
    return offset, index_frac - offset


def resample(x, sr, target):
    """float32 [n_in] at sr -> float32 [ceil(n_in target / sr)] at target (the input itself when sr == target)."""
    x = np.asarray(x, np.float32)
    if sr == target:
        return x
    n_in = len(x)
    n_res, n_out = lengths(n_in, sr, target)
    base, num_table = sinc_window(**KAISER_BEST)
    ratio = float(target) / sr
    win, delta = tables(ratio, base, num_table)
    nwin = len(win)
    scale = min(1.0, ratio)
    index_step = int(scale * num_table)
    tr = time_register(n_res, 1.0 / ratio)
    n = tr.astype(np.int64)
    xd = x.astype(np.float64)
    y = np.zeros(n_res, np.float32)

    def wing(offset, eta, count, src):
        for i in range(int(count.max(initial=0))):
            m = np.nonzero(i < count)[0]
            j = offset[m] + i * index_step
            w = win[j] + eta[m] * delta[j]
            y[m] = (y[m].astype(np.float64) + w * xd[src(m, i)]).astype(np.float32)

    frac = scale * (tr - n)
    offset, eta = _phase(frac, num_table)
    wing(offset, eta, np.minimum(n + 1, (nwin - offset) // index_step), lambda m, i: n[m] - i)
    frac = scale - frac
    offset, eta = _phase(frac, num_table)
    wing(offset, eta, np.minimum(n_in - n - 1, (nwin - offset) // index_step), lambda m, i: n[m] + i + 1)
    out = np.zeros(n_out, np.float32)
    out[:n_res] = y
    return out


def load(path, sr):
    """``librosa.core.load(path, sr=sr, mono=True)`` for a WAV file: (float32 samples at sr, sr)."""
    x, file_sr = decode(path)
    return resample(x, file_sr, sr), sr


def min_length(sr, target):
    """The shortest clip that yields at least one sample."""
    ratio = float(target) / sr
    return next(n for n in range(1, 1 << 20) if int(n * ratio) >= 1)


"""The resampler (csrc/resample.cu) against oracle/resample.py bit for bit, and the load paths built on it: HifiGAN.wav2spec /
wav2spec_batch on files at other rates and the paired binarizer on a 44.1 kHz stereo set."""
import os

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import resample as R

pytestmark = pytest.mark.gpu

TARGET = 22050


def _clip(n, seed):
    rs = np.random.RandomState(seed)
    t = np.arange(n) / 44100.0
    f = rs.uniform(110, 880)
    x = 0.3 * np.sin(2 * np.pi * f * t) + 0.1 * np.sin(2 * np.pi * 3.1 * f * t) + 0.05 * rs.standard_normal(n)
    return x.astype(np.float32)


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope='module')
def ragged():
    """Every source rate, lengths from the shortest legal clip to 30 s, in a shuffled order."""
    rates = [48000, 44100, 32000, 16000, 8000, 96000, 22050]
    clips = []
    for k, sr in enumerate(rates):
        for n in (R.min_length(sr, TARGET), 97, 1001, int(sr * 1.37) + 1):
            clips.append((sr, n))
    clips += [(96000, 96000 * 30), (44100, 44100 * 30 + 1), (48000, int(48000 * 8.3))]
    rs = np.random.RandomState(0)
    rs.shuffle(clips)
    wavs = [_clip(n, 100 + i) for i, (_, n) in enumerate(clips)]
    srs = [sr for sr, _ in clips]
    want = [R.resample(w, sr, TARGET) for w, sr in zip(wavs, srs)]
    return wavs, srs, want


def test_ragged_batch_is_bit_identical_to_the_oracle(ragged):
    from neuralsvb_b200.utils import audio
    wavs, srs, want = ragged
    got = audio.resample_batch(wavs, srs, TARGET)
    assert len(got) == len(want)
    for g, w, sr, x in zip(got, want, srs, wavs):
        assert g.shape == w.shape, (sr, len(x))
        bad = np.nonzero(_bits(g) != _bits(w))[0]
        assert len(bad) == 0, f'{sr} Hz, {len(x)} samples: {len(bad)} samples differ, first at {bad[:5]}'


def test_each_clip_alone_equals_the_clip_in_the_batch(ragged):
    from neuralsvb_b200.utils import audio
    wavs, srs, _ = ragged
    batch = audio.resample_batch(wavs, srs, TARGET)
    for i in range(0, len(wavs), 3):
        alone = audio.resample_batch([wavs[i]], [srs[i]], TARGET)[0]
        assert np.array_equal(_bits(alone), _bits(batch[i])), (srs[i], len(wavs[i]))


def test_44100_to_24000_is_bit_identical_to_the_oracle():
    from neuralsvb_b200.utils import audio
    wavs = [_clip(n, 7 + n) for n in (R.min_length(44100, 24000), 139, 44101, 441000)]
    got = audio.resample_batch(wavs, [44100] * len(wavs), 24000)
    for g, x in zip(got, wavs):
        assert np.array_equal(_bits(g), _bits(R.resample(x, 44100, 24000))), len(x)


def test_device_entry_point_and_stage_times():
    import ctypes

    import torch

    from neuralsvb_b200 import _native
    from neuralsvb_b200.utils import audio
    wavs = [_clip(48000 * 2 + 3, 11), _clip(44100 + 7, 12)]
    srs = np.array([48000, 44100], np.int32)
    lens = np.array([len(w) for w in wavs], np.int64)
    _, out_lens = audio.resample_lengths(lens, srs, TARGET)
    win, num_table = audio.kaiser_best_window()
    lib = _native.lib()
    ws_bytes = lib.svb_resample_plan(TARGET, srs.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p), 2, len(win),
                                     num_table, None, None)
    x = torch.from_numpy(np.concatenate(wavs)).cuda()
    y = torch.empty(int(out_lens.sum()), device='cuda')
    ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device='cuda')
    ms = np.zeros(2, np.float32)
    args = lambda n_ws: (TARGET, srs.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p), 2,
                         win.ctypes.data_as(ctypes.c_void_p), len(win), num_table, ctypes.c_void_p(x.data_ptr()),
                         ctypes.c_void_p(y.data_ptr()), ctypes.c_void_p(ws.data_ptr()), n_ws, ms.ctypes.data_as(ctypes.c_void_p),
                         _native.current_stream_ptr())
    assert lib.svb_resample_batch(*args(int(ws_bytes) - 1)) == -1          # a short workspace is refused before any launch
    _native.check(lib.svb_resample_batch(*args(int(ws_bytes))), 'resample')
    y = y.cpu().numpy()
    assert np.all(ms > 0)
    o = 0
    for w, sr, n in zip(wavs, srs, out_lens):
        assert np.array_equal(_bits(y[o:o + n]), _bits(R.resample(w, int(sr), TARGET)))
        o += n


def _write(path, sr, mono, channels, fmt='int16'):
    data = mono if channels == 1 else np.stack([mono * np.float32(1 - 0.2 * c) for c in range(channels)], axis=1)
    if fmt == 'int16':
        data = np.round(np.clip(data, -1, 1) * 32767).astype(np.int16)
    wavfile.write(path, sr, data)


def test_wav2spec_on_files_at_other_rates(tmp_path):
    from neuralsvb_b200.utils import synthetic as S
    from neuralsvb_b200.vocoders.hifigan import HifiGAN
    hp = S.hifigan_config()
    hp = dict(hp, audio_sample_rate=TARGET)
    paths = []
    for k, (sr, ch) in enumerate([(44100, 1), (44100, 2), (48000, 1), (48000, 2)]):
        p = str(tmp_path / f'{k}.wav')
        _write(p, sr, _clip(int(sr * 1.3) + k, 20 + k), ch)
        paths.append(p)
    p = str(tmp_path / 'native.wav')
    _write(p, TARGET, _clip(TARGET + 5, 30), 1)
    paths.append(p)
    arrays = [R.load(p, TARGET)[0] for p in paths]
    got_b = HifiGAN.wav2spec_batch(paths, hp=hp)
    want_b = HifiGAN.wav2spec_batch(arrays, hp=hp)
    for p, a, (gw, gm), (ww, wm) in zip(paths, arrays, got_b, want_b):
        assert np.array_equal(_bits(gw), _bits(ww)) and np.array_equal(_bits(gm), _bits(wm)), p
        sw, sm = HifiGAN.wav2spec(p, hp=hp)
        ow, om = HifiGAN.wav2spec(a, hp=hp)
        assert np.array_equal(_bits(sw), _bits(ow)) and np.array_equal(_bits(sm), _bits(om)), p


def _binarize(raw, out):
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, 'phone_set.json'), 'w') as f:
        json.dump([f'ph{i}' for i in range(60)], f)
    r = subprocess.run([sys.executable, '-m', 'neuralsvb_b200.data_gen.tts.bin.binarize', '--config',
                        os.path.join(root, 'egs', 'svb_binarize_synthetic.yaml'), '--hparams',
                        f'processed_data_dir={raw},binary_data_dir={out},spk_emb_data_dir={raw}/spk_emb'],
                       cwd=out, env=dict(os.environ, PYTHONPATH=root), capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def test_paired_binarizer_on_a_44100_stereo_set(tmp_path):
    from neuralsvb_b200.utils import synthetic as S
    from neuralsvb_b200.utils.indexed_datasets import IndexedDataset
    hi, lo = str(tmp_path / 'raw44'), str(tmp_path / 'raw22')
    S.write_svb_raw(hi, file_sr=44100, channels=2)
    # the same recordings, resampled by the oracle and written as float32 WAV at the model's rate (decoded exactly)
    for d, _, files in os.walk(hi):
        rel = os.path.relpath(d, hi)
        os.makedirs(os.path.join(lo, rel), exist_ok=True)
        for f in files:
            src, dst = os.path.join(d, f), os.path.join(lo, rel, f)
            if f.endswith('.wav'):
                wavfile.write(dst, TARGET, R.load(src, TARGET)[0])
            else:
                with open(src, 'rb') as a, open(dst, 'wb') as b:
                    b.write(a.read())
    _binarize(hi, str(tmp_path / 'bin44'))
    _binarize(lo, str(tmp_path / 'bin22'))
    for prefix in ('train', 'valid', 'test'):
        a, b = str(tmp_path / 'bin44' / prefix), str(tmp_path / 'bin22' / prefix)
        if not os.path.exists(a + '.idx'):
            assert not os.path.exists(b + '.idx')
            continue
        da, db = IndexedDataset(a), IndexedDataset(b)
        assert len(da) == len(db) > 0
        for i in range(len(da)):
            ia, ib = da[i], db[i]
            assert sorted(ia) == sorted(ib)
            for k in ia:
                if isinstance(ia[k], np.ndarray):
                    assert ia[k].dtype == ib[k].dtype and np.array_equal(ia[k], ib[k]), (prefix, i, k)
                else:
                    assert ia[k] == ib[k], (prefix, i, k)
        sa = np.load(str(tmp_path / 'bin44' / f'{prefix}_f0s_mean_std.npy'))
        sb = np.load(str(tmp_path / 'bin22' / f'{prefix}_f0s_mean_std.npy'))
        assert np.array_equal(sa, sb)
        assert np.array_equal(np.load(a + '_lengths.npy'), np.load(b + '_lengths.npy'))

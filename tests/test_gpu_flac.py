"""csrc/flac.cu on the GPU: the FFmpeg-made fixtures and test-encoder streams covering each coding branch decode bit-identically to
the oracle, and to read_wav of a WAV holding the same PCM; a ragged batch equals each stream decoded alone; damaged streams end in a
ValueError naming the file and byte offset; wav2spec_batch on FLAC takes equals the same call on WAV takes."""
import glob
import os

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import flac as F

pytestmark = pytest.mark.gpu
GOLDEN_FLAC = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'flac')


def signal(n, chans, bits, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n)[:, None]
    x = 0.6 * np.sin(t * 0.013 * (1 + np.arange(chans))) + 0.05 * rng.standard_normal((n, chans))
    q = 1 << (bits - 1)
    return np.clip(np.round(x * q), -q, q - 1).astype(np.int64)


def gpu_decode(blobs, names=None):
    from neuralsvb_b200.utils import audio
    y, lens, rates = audio.flac_decode_device(blobs, names)
    y = y.cpu().numpy()
    return np.split(y, np.cumsum(lens)[:-1]), rates


BRANCHES = [
    dict(),
    dict(subframe=dict(type='verbatim')),
    dict(subframe=dict(type='fixed', order=0)),
    dict(subframe=dict(type='fixed', order=1, partition_order=3)),
    dict(subframe=dict(type='fixed', order=3, rice2=True)),
    dict(subframe=dict(type='fixed', order=4, escape={0, 2}, partition_order=2)),
    dict(subframe=dict(type='lpc', order=1, precision=4, shift=2)),
    dict(subframe=dict(type='lpc', order=12, partition_order=4, rice2=True)),
    dict(subframe=dict(type='lpc', order=32, precision=15, shift=14, escape=True)),
    dict(subframe=dict(type='fixed', order=2, wasted=0)),
    dict(block_tail=True, rate_code='streaminfo', bits_code='streaminfo'),
    dict(channel_mode=F.LEFT_SIDE, subframe=dict(type='lpc', order=6)),
    dict(channel_mode=F.SIDE_RIGHT, subframe=dict(type='fixed', order=2)),
    dict(channel_mode=F.MID_SIDE, subframe=dict(type='lpc', order=6)),
]


def branch_streams():
    out = []
    for bits in (8, 12, 16, 20, 24):
        for chans in (1, 2, 6, 8):
            x = signal(700, chans, bits, seed=bits + chans)
            for k, opt in enumerate(BRANCHES):
                if 'channel_mode' in opt and chans != 2:
                    continue
                out.append((f'b{bits}c{chans}o{k}', x, bits, F.encode(x, 44100, bits, block_size=256, **opt)))
    x = signal(1000, 2, 16)
    out.append(('variable', x, 16, F.encode(x, 22050, 16, block_size=[100, 7, 893], variable=True, metadata=(1, 2, 3, 4, 5, 6))))
    c = np.full((700, 2), -1234, np.int64) << 3
    out.append(('constant', c, 20, F.encode(c, 8000, 20, block_size=200, subframe=dict(type='constant'), block_tail=True)))
    return out


def test_fixtures_decode_bit_identically():
    paths = sorted(glob.glob(os.path.join(GOLDEN_FLAC, '*.flac')))
    blobs = [open(p, 'rb').read() for p in paths]
    ys, rates = gpu_decode(blobs, paths)
    for p, y, r in zip(paths, ys, rates):
        ref = np.load(p[:-5] + '.npz')
        assert r == int(ref['sr'])
        np.testing.assert_array_equal(y, F.to_float(ref['pcm'], int(ref['bits'])), err_msg=p)


def test_every_branch_matches_the_oracle_and_batch_independence():
    streams = branch_streams()
    ys, _ = gpu_decode([s[3] for s in streams], [s[0] for s in streams])
    for (name, x, bits, data), y in zip(streams, ys):
        pcm, _ = F.decode(data, name, check_md5=True)
        np.testing.assert_array_equal(y, F.to_float(pcm, bits), err_msg=name)
    # a ragged batch of about 20 streams equals each stream decoded alone
    pick = streams[::max(1, len(streams) // 20)][:20]
    batch, _ = gpu_decode([s[3] for s in pick])
    for s, y in zip(pick, batch):
        alone, _ = gpu_decode([s[3]])
        np.testing.assert_array_equal(y, alone[0], err_msg=s[0])


@pytest.mark.parametrize('bits', [8, 16, 24])
@pytest.mark.parametrize('chans', [1, 2, 6, 8])
def test_read_wav_of_flac_equals_read_wav_of_wav(tmp_path, bits, chans):
    from neuralsvb_b200.utils import audio
    x = signal(5000, chans, bits, seed=bits * chans)
    w = tmp_path / 'a.wav'
    stored = (x + 128).astype(np.uint8) if bits == 8 else x.astype(np.int16) if bits == 16 else (x << 8).astype(np.int32)
    wavfile.write(str(w), 32000, stored)
    f = tmp_path / 'a.flac'
    f.write_bytes(F.encode(x, 32000, bits, block_size=1152, subframe=dict(type='lpc', order=8)))
    yw, rw = audio.read_wav(str(w))
    yf, rf = audio.read_wav(str(f))
    assert rw == rf == 32000 and yf.dtype == np.float32
    np.testing.assert_array_equal(yf, yw)


def test_damaged_streams_raise_with_file_and_offset(tmp_path):
    from neuralsvb_b200.utils import audio
    x = signal(4000, 2, 16)
    data = F.encode(x, 44100, 16, block_size=1024, subframe=dict(type='fixed', order=2))
    _, _, first = F.parse_metadata(data)
    h = F.parse_frame_header(data, first)
    # a flipped bit inside the first frame's residual fails that frame's CRC-16
    bad = bytearray(data)
    bad[first + h['header_bytes'] + 200] ^= 0x04
    p = tmp_path / 'flip.flac'
    p.write_bytes(bytes(bad))
    with pytest.raises(ValueError, match=rf'flip\.flac: frame fails its CRC-16 at byte {first}'):
        audio.read_wav(str(p))
    # a truncated file
    p = tmp_path / 'cut.flac'
    p.write_bytes(data[:len(data) - 300])
    with pytest.raises(ValueError, match=r'cut\.flac: .* at byte \d+'):
        audio.read_wav(str(p))
    # frames that stop short of STREAMINFO's total
    y = signal(3000, 2, 16)
    short = bytearray(F.encode(y, 44100, 16, block_size=1024))
    v = int.from_bytes(short[8 + 10:8 + 18], 'big') + 500
    short[8 + 10:8 + 18] = v.to_bytes(8, 'big')
    p = tmp_path / 'short.flac'
    p.write_bytes(bytes(short))
    with pytest.raises(ValueError, match=r'short\.flac: the frames stop short of STREAMINFO.s total sample count at byte \d+'):
        audio.read_wav(str(p))
    # bytes after the last frame: a copied frame (a valid header) appended to a whole stream
    p = tmp_path / 'trail.flac'
    p.write_bytes(data + data[first:first + 64])
    with pytest.raises(ValueError, match=rf'trail\.flac: data after the last frame at byte {len(data)}'):
        audio.read_wav(str(p))


def test_wav2spec_batch_on_flac_equals_wav(tmp_path):
    """decode_wavs' one-call FLAC path through the resampler and the front end: 44.1 kHz stereo 24-bit and 22.05 kHz mono 16-bit
    takes give the arrays of the same takes as WAV."""
    from neuralsvb_b200.utils import synthetic as S
    from neuralsvb_b200.vocoders.hifigan import HifiGAN
    hp = S.hifigan_config()
    takes = [(44100, 24, signal(44100, 2, 24, seed=1)), (22050, 16, signal(30000, 1, 16, seed=2))]
    wavs, flacs = [], []
    for k, (sr, bits, x) in enumerate(takes):
        w, f = tmp_path / f'{k}.wav', tmp_path / f'{k}.flac'
        wavfile.write(str(w), sr, x.astype(np.int16) if bits == 16 else (x << 8).astype(np.int32))
        f.write_bytes(F.encode(x, sr, bits, block_size=4096, subframe=dict(type='lpc', order=12)))
        wavs.append(str(w)), flacs.append(str(f))
    a, b = HifiGAN.wav2spec_batch(wavs, hp=hp), HifiGAN.wav2spec_batch(flacs, hp=hp)
    for (wa, ma), (wb, mb) in zip(a, b):
        np.testing.assert_array_equal(wa, wb)
        np.testing.assert_array_equal(ma, mb)


def _flac_twin(wav_path, dst_dir, bits=None):
    """(WAV path, FLAC path) holding the same integer PCM: a float32 WAV is quantised to ``bits`` and rewritten as an integer WAV."""
    sr, data = wavfile.read(wav_path)
    name = os.path.splitext(os.path.basename(wav_path))[0]
    if data.dtype.kind == 'f':
        q = 1 << (bits - 1)
        pcm = np.clip(np.round(data.astype(np.float64) * q), -q, q - 1).astype(np.int64)
        wav_path = os.path.join(dst_dir, name + '.wav')
        wavfile.write(wav_path, sr, (pcm << (32 - bits)).astype(np.int32) if bits > 16 else pcm.astype(np.int16))
    else:
        pcm, bits = data.astype(np.int64), 8 * data.dtype.itemsize
    flac_path = os.path.join(dst_dir, name + '.flac')
    with open(flac_path, 'wb') as f:
        f.write(F.encode(pcm, sr, bits, block_size=4096, subframe=dict(type='fixed', order=2)))
    return wav_path, flac_path


def test_beautify_on_flac_takes_equals_wav_takes(tmp_path):
    """beautify_batch and beautify_songs: a 44.1 kHz stereo 24-bit pair and a 22.05 kHz mono 16-bit pair as FLAC give the arrays of
    the same takes as WAV, with the same seed and eps."""
    import torch

    from neuralsvb_b200.inference import beautify as BF
    from tests.test_gpu_beautify import make_experiment, regular
    work, pairs22 = make_experiment(str(tmp_path / 'e22'))
    _, pairs44 = make_experiment(str(tmp_path / 'e44'), file_sr=44100, channels=2, sample_format='float32')
    p44, p22 = regular(pairs44)[0], regular(pairs22)[1]
    twins = tmp_path / 'twins'
    twins.mkdir()
    takes = [_flac_twin(p44[1], str(twins), 24), _flac_twin(p22[1], str(twins)), _flac_twin(p44[2], str(twins), 24),
             _flac_twin(p22[2], str(twins))]
    assert wavfile.read(takes[0][0])[1].shape[1] == 2 and F.parse_metadata(open(takes[0][1], 'rb').read())[0]['bits'] == 24
    emb = [p44[3], p22[3]]
    b = BF.SVBBeautifier(work)
    eps = torch.randn(2, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(3))
    for call in (b.beautify_batch, b.beautify_songs):
        ww = call([takes[0][0], takes[1][0]], [takes[2][0], takes[3][0]], emb, seed=11, eps=eps)
        ff = call([takes[0][1], takes[1][1]], [takes[2][1], takes[3][1]], emb, seed=11, eps=eps)
        for i in range(2):
            assert np.array_equal(ww[i], ff[i]), (call.__name__, i)


def test_binarizer_on_flac_copy_writes_the_wav_copys_data(tmp_path):
    import shutil

    from neuralsvb_b200.utils import synthetic as S
    from neuralsvb_b200.utils.indexed_datasets import IndexedDataset
    from tests.test_gpu_resample import _binarize
    wav_raw, flac_raw = str(tmp_path / 'raw_wav'), str(tmp_path / 'raw_flac')
    S.write_svb_raw(wav_raw)
    for d, _, files in os.walk(wav_raw):
        out = os.path.join(flac_raw, os.path.relpath(d, wav_raw))
        os.makedirs(out, exist_ok=True)
        for f in files:
            if f.endswith('.wav'):
                _flac_twin(os.path.join(d, f), out)               # int16 WAV: only the FLAC is written to out
            else:
                shutil.copy(os.path.join(d, f), os.path.join(out, f))
    assert not glob.glob(os.path.join(flac_raw, 'data', '*', '*.wav'))
    _binarize(wav_raw, str(tmp_path / 'bin_wav'))
    _binarize(flac_raw, str(tmp_path / 'bin_flac'))

    def norm(v):
        return v.replace(flac_raw, wav_raw).replace('.flac', '.wav') if isinstance(v, str) else v
    n = 0
    for prefix in ('train', 'valid', 'test'):
        a, b = str(tmp_path / 'bin_wav' / prefix), str(tmp_path / 'bin_flac' / prefix)
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
                    assert ia[k] == norm(ib[k]), (prefix, i, k)
            n += 1
        for stats in (f'{prefix}_f0s_mean_std.npy',):
            if os.path.exists(str(tmp_path / 'bin_wav' / stats)):
                assert np.array_equal(np.load(str(tmp_path / 'bin_wav' / stats)), np.load(str(tmp_path / 'bin_flac' / stats)))
    assert n > 0

"""FLAC without a GPU: the oracle's encoder/decoder round trip over every coding option, the STREAMINFO MD5, the oracle on the
FFmpeg-made fixtures, metadata parsing and wav_info of FLAC, svb_flac_plan's refusals, and the binarizer's listing of WAV and FLAC
items."""
import ctypes
import glob
import os

import numpy as np
import pytest

from oracle import flac as F

GOLDEN_FLAC = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'flac')


def signal(n, chans, bits, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n)[:, None]
    x = 0.6 * np.sin(t * 0.013 * (1 + np.arange(chans))) + 0.05 * rng.standard_normal((n, chans))
    q = 1 << (bits - 1)
    return np.clip(np.round(x * q), -q, q - 1).astype(np.int64)


OPTIONS = [
    dict(),
    dict(subframe=dict(type='verbatim')),
    dict(subframe=dict(type='fixed', order=0)),
    dict(subframe=dict(type='fixed', order=1, partition_order=2)),
    dict(subframe=dict(type='fixed', order=3, rice2=True)),
    dict(subframe=dict(type='fixed', order=4, escape={0, 2}, partition_order=2)),
    dict(subframe=dict(type='lpc', order=1, precision=4, shift=2)),
    dict(subframe=dict(type='lpc', order=8, partition_order=4, rice2=True)),
    dict(subframe=dict(type='lpc', order=32, precision=15, shift=14, escape=True)),
    dict(subframe=dict(type='fixed', order=2, wasted=0)),
    dict(block_tail=True, rate_code='streaminfo', bits_code='streaminfo'),
]
STEREO = [dict(channel_mode=m, subframe=dict(type='lpc', order=6)) for m in (F.LEFT_SIDE, F.SIDE_RIGHT, F.MID_SIDE)]


@pytest.mark.parametrize('bits', [8, 12, 16, 20, 24])
@pytest.mark.parametrize('chans', [1, 2, 3, 8])
def test_oracle_round_trip_every_option(bits, chans):
    x = signal(512, chans, bits, seed=bits * 10 + chans)
    for opt in OPTIONS + (STEREO if chans == 2 else []):
        data = F.encode(x, 44100, bits, block_size=256, **opt)
        y, si = F.decode(data, check_md5=True)
        assert np.array_equal(x, y), opt
        assert (si['bits'], si['channels'], si['total_samples']) == (bits, chans, len(x))


def test_oracle_channel_counts_rates_and_blocking():
    for chans in range(1, 9):
        x = signal(300, chans, 16, seed=chans)
        assert np.array_equal(F.decode(F.encode(x, 22050, 16, block_size=192))[0], x)
    x = signal(1000, 2, 16)
    for sr, code in [(22050, 'table'), (48000, 'khz'), (11025, 'hz'), (96010, 'tens'), (44100, 'streaminfo')]:
        data = F.encode(x, sr, 16, block_size=[100, 7, 893], variable=True, rate_code=code, metadata=(1, 2, 3, 4, 5, 6))
        y, si = F.decode(data, check_md5=True)
        assert np.array_equal(x, y) and si['sample_rate'] == sr
    q = np.arange(-40, 40)[:, None] * np.ones((1, 2), np.int64)     # Rice parameter 0: one unary run per residual
    assert np.array_equal(F.decode(F.encode(q, 8000, 8, block_size=80, subframe=dict(type='fixed', order=0, rice_param=0)))[0], q)
    # constant channels, wasted bits, 8- and 16-bit block-size tails
    c = np.full((700, 2), -1234, np.int64) << 3
    for bs in (200, 700):
        y, _ = F.decode(F.encode(c, 8000, 20, block_size=bs, subframe=dict(type='constant'), block_tail=True), check_md5=True)
        assert np.array_equal(y, c)


def test_oracle_checks_md5_and_crc():
    x = signal(600, 2, 16)
    data = bytearray(F.encode(x, 44100, 16, block_size=300))
    si, _, first = F.parse_metadata(data)
    md5_at = 4 + 4 + 18
    bad = bytearray(data)
    bad[md5_at] ^= 1
    F.decode(bytes(bad))                                   # MD5 is off by default
    with pytest.raises(F.FlacError, match='MD5'):
        F.decode(bytes(bad), check_md5=True)
    bad = bytearray(data)
    bad[first + 40] ^= 0x10
    with pytest.raises(F.FlacError):
        F.decode(bytes(bad))
    with pytest.raises(F.FlacError, match='Ogg'):
        F.parse_metadata(b'OggS' + bytes(40))


def fixtures():
    return sorted(glob.glob(os.path.join(GOLDEN_FLAC, '*.flac')))


def test_fixtures_cover_the_issue():
    names = [os.path.basename(f) for f in fixtures()]
    assert any(n.startswith('l0_') for n in names) and any(n.startswith('l5_') for n in names) \
        and any(n.startswith('l12_') for n in names)
    assert {'l5_s16_stereo.flac', 'l5_s24_mono.flac', 'l5_u8_mono.flac', 'l5_s16_6ch.flac', 'l8_s16_odd.flac'} <= set(names)


@pytest.mark.parametrize('path', fixtures(), ids=os.path.basename)
def test_oracle_decodes_ffmpeg_fixtures(path):
    ref = np.load(path[:-5] + '.npz')
    with open(path, 'rb') as f:
        pcm, si = F.decode(f.read(), path, check_md5=True)
    assert np.array_equal(pcm, ref['pcm']) and si['sample_rate'] == int(ref['sr']) and si['bits'] == int(ref['bits'])


def test_flac_info_and_wav_info(tmp_path):
    from neuralsvb_b200.utils import audio
    x = signal(1234, 3, 24)
    data = F.encode(x, 48000, 24, block_size=512, metadata=(4, 1))
    p = tmp_path / 'a.flac'
    p.write_bytes(data)
    info = audio.flac_info(data)
    assert info == dict(sample_rate=48000, channels=3, bits=24, total_samples=1234, first_frame=F.parse_metadata(data)[2])
    assert audio.wav_info(str(p)) == (48000, 1234, 3)
    assert audio.wav_seconds(str(p)) == 1234 / 48000
    assert audio.is_flac(str(p))
    o = tmp_path / 'o.flac'
    o.write_bytes(b'OggS' + bytes(60))
    with pytest.raises(ValueError, match='Ogg'):
        audio.flac_info(o.read_bytes(), str(o))
    junk = tmp_path / 'j.wav'
    junk.write_bytes(b'JUNK' + bytes(60))
    with pytest.raises(ValueError, match='not a RIFF/WAVE file.*FLAC'):
        audio.wav_info(str(junk))
    with pytest.raises(ValueError, match='cut: bad FLAC metadata block'):
        audio.flac_info(data[:20], 'cut')


def _plan(nbytes, first, sr, ch, bits, total):
    from neuralsvb_b200 import _native
    arrs = [np.array(nbytes, np.int64), np.array(first, np.int64), np.array(sr, np.int32), np.array(ch, np.int32),
            np.array(bits, np.int32), np.array(total, np.int64)]
    out = np.zeros(len(nbytes), np.int64)
    lib = _native.lib()
    r = lib.svb_flac_plan(len(nbytes), *[a.ctypes.data_as(ctypes.c_void_p) for a in arrs], out.ctypes.data_as(ctypes.c_void_p))
    return r, out, lib.svb_last_error().decode()


def test_flac_plan_refusals_before_any_cuda_call():
    pytest.importorskip('neuralsvb_b200._native')
    from neuralsvb_b200 import _native
    try:
        _native.build()
    except RuntimeError:
        pass
    if not os.path.exists(_native.LIB_PATH):
        pytest.skip('library not built')
    r, out, _ = _plan([1000, 500], [42, 42], [44100, 22050], [2, 1], [16, 24], [5000, 300])
    assert r > 0 and list(out) == [5000, 300]
    for args, msg in [(([100, 100], [42, 42], [44100, 44100], [2, 2], [16, 32], [10, 10]), 'stream 1: 32 bits'),
                      (([100], [42], [44100], [2], [3], [10]), 'stream 0: 3 bits'),
                      (([100, 100], [42, 42], [44100, 44100], [1, 1], [16, 16], [10, 0]), 'stream 1: STREAMINFO gives no total'),
                      (([100], [42], [44100], [9], [16], [10]), 'stream 0: 9 channels')]:
        r, _, err = _plan(*args)
        assert r == -1 and msg in err, err


def _touch(root, rel):
    p = os.path.join(root, 'data', rel)
    os.makedirs(os.path.dirname(p), exist_ok=True)
    open(p, 'wb').close()


def _listing(root):
    from neuralsvb_b200.data_gen.singing.binarize import SingingBinarizer
    from neuralsvb_b200.utils.hparams import hparams
    hparams.update(dict(datasets=['x'], test_prefixes=['zz'], binarization_args={}, audio_sample_rate=22050))
    b = SingingBinarizer(str(root))
    b.load_meta_data()
    return b.item2wavfn


def test_binarizer_lists_wav_and_flac(tmp_path):
    from neuralsvb_b200.utils.hparams import hparams
    saved = dict(hparams)
    try:
        wav = tmp_path / 'wav'
        for n in ('x#a#1', 'x#b#2'):
            _touch(str(wav), f'd/{n}.wav')
        assert _listing(wav) == {n: str(wav / 'data' / 'd' / f'{n}.wav') for n in ('x#a#1', 'x#b#2')}
        mixed = tmp_path / 'mixed'
        _touch(str(mixed), 'd/x#a#1.wav')
        _touch(str(mixed), 'e/x#b#2.flac')
        assert _listing(mixed) == {'x#a#1': str(mixed / 'data' / 'd' / 'x#a#1.wav'), 'x#b#2': str(mixed / 'data' / 'e' / 'x#b#2.flac')}
        clash = tmp_path / 'clash'
        _touch(str(clash), 'd/x#a#1.wav')
        _touch(str(clash), 'd/x#a#1.flac')
        with pytest.raises(ValueError, match="'x#a#1'"):
            _listing(clash)
        mp3 = tmp_path / 'mp3'
        _touch(str(mp3), 'd/x#a#1.mp3')
        with pytest.raises(ValueError, match='mp3 files only.*FLAC is also accepted'):
            _listing(mp3)
    finally:
        hparams.clear()
        hparams.update(saved)


@pytest.mark.parametrize('chans', [1, 2, 3, 6, 7, 8])
def test_to_float_is_read_wav_of_the_same_pcm(tmp_path, chans):
    from scipy.io import wavfile

    from neuralsvb_b200.utils import audio
    x = signal(20000, chans, 24, seed=chans)
    p = tmp_path / 'a.wav'
    wavfile.write(str(p), 16000, (x << 8).astype(np.int32))
    assert np.array_equal(F.to_float(x, 24), audio.read_wav(str(p))[0])


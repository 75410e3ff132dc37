"""Host helpers of the wav -> mel front end (reference: utils/audio.py:57-117 and the call
sites of librosa.filters.mel in data_gen/tts/data_gen_utils.py:130, modules/hifigan/mel_utils.py:62).
The STFT / magnitude / mel projection / log themselves run in the fused CUDA kernel
(csrc/frontend.cu); what stays on the host is the constant mel filterbank and index arithmetic.

Loading audio (``load_takes``, ``load_wav``): the reference's ``librosa.core.load(path, sr=sr)`` for WAV and FLAC files -- decode
(WAV on the host, FLAC on the GPU, csrc/flac.cu), fold to mono, resample with resampy's ``kaiser_best`` filter -- with the
resampling in csrc/resample.cu (oracle/resample.py states the algorithm).  ``load_takes`` is the one route to the device: one
host-to-device copy of the samples decoded on the host, FLAC samples left where they were decoded, and one resampler call over the
off-rate takes.  ``load_wav``, ``read_wav``'s FLAC branch and ``resample_batch`` are that route with a copy back to the host."""
import ctypes
import functools
import struct

import numpy as np


def _slaney_hz_to_mel(hz):
    hz = np.atleast_1d(np.asarray(hz, dtype=np.float64))
    lin = hz * (3.0 / 200.0)
    log = 15.0 + np.log(np.maximum(hz, 1e-30) / 1000.0) * (27.0 / np.log(6.4))
    return np.where(hz >= 1000.0, log, lin)


def _slaney_mel_to_hz(mel):
    mel = np.atleast_1d(np.asarray(mel, dtype=np.float64))
    lin = mel * (200.0 / 3.0)
    log = 1000.0 * np.exp((np.log(6.4) / 27.0) * (mel - 15.0))
    return np.where(mel >= 15.0, log, lin)


@functools.lru_cache(maxsize=32)
def _mel_filterbank_cached(sr, n_fft, n_mels, fmin, fmax):
    bins = np.linspace(0.0, sr / 2.0, n_fft // 2 + 1)
    edges = _slaney_mel_to_hz(np.linspace(_slaney_hz_to_mel(fmin)[0], _slaney_hz_to_mel(fmax)[0], n_mels + 2))
    lo, ce, hi = edges[:-2, None], edges[1:-1, None], edges[2:, None]
    up = (bins[None, :] - lo) / (ce - lo)
    down = (hi - bins[None, :]) / (hi - ce)
    tri = np.clip(np.minimum(up, down), 0.0, None).astype(np.float32)
    area = (2.0 / (hi - lo)).astype(np.float64)
    fb = (tri * area).astype(np.float32)            # float32 storage then Slaney area norm, like librosa
    fb.setflags(write=False)
    return fb


def mel_filterbank(sr, n_fft, n_mels=80, fmin=0.0, fmax=None):
    """Slaney-scale, area-normalised triangular filterbank [n_mels, n_fft//2+1] float32 -- the
    matrix ``librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)`` (0.8 defaults) returns."""
    fmax = sr / 2.0 if fmax is None else fmax
    return _mel_filterbank_cached(int(sr), int(n_fft), int(n_mels), float(fmin), float(fmax))


def build_mel_basis(hparams):
    """utils/audio.py:98-101."""
    assert hparams['fmax'] <= hparams['audio_sample_rate'] // 2
    return mel_filterbank(hparams['audio_sample_rate'], hparams['fft_size'], hparams['audio_num_mel_bins'],
                          hparams['fmin'], hparams['fmax'])


def librosa_pad_lr(x, fsize, fshift, pad_sides=1):
    """Right (or both-sides) padding that makes len(x) = (len(x)//hop + 1) * hop (utils/audio.py:67-76)."""
    assert pad_sides in (1, 2)
    pad = (x.shape[0] // fshift + 1) * fshift - x.shape[0]
    return (0, pad) if pad_sides == 1 else (pad // 2, pad - pad // 2)


def amp_to_db(x):
    return 20 * np.log10(np.maximum(1e-5, x))


def normalize(S, hparams):
    return (S - hparams['min_level_db']) / -hparams['min_level_db']


def save_wav(wav, path, sr, norm=False):
    """float waveform -> int16 wav file (utils/audio.py:11-16).  An int16 array (the device-side conversion of
    ``HifiGAN.spec2wav_batch(int16=True)``) is written as is."""
    from scipy.io import wavfile
    wav = np.asarray(wav)
    if wav.dtype == np.int16:
        wavfile.write(path, sr, wav)
        return
    wav = wav.astype(np.float32)
    if norm:
        wav = wav / np.abs(wav).max()
    wavfile.write(path, sr, (wav * np.float32(32767)).astype(np.int16))


KAISER_BEST = dict(num_zeros=64, precision=9, beta=14.769656459379492, rolloff=0.9475937167399596)


@functools.lru_cache(maxsize=1)
def kaiser_best_window():
    """(win float64 [32769], num_table 512): resampy's ``sinc_window`` right wing for ``kaiser_best``, rebuilt from its
    construction (resampy 0.2.2 ships it precomputed; bit agreement with that file has not been checked)."""
    from scipy.signal.windows import kaiser
    p = KAISER_BEST
    num_bits = 2 ** p['precision']
    n = num_bits * p['num_zeros']
    sinc_win = p['rolloff'] * np.sinc(p['rolloff'] * np.linspace(0, p['num_zeros'], num=n + 1, endpoint=True))
    win = np.ascontiguousarray(kaiser(2 * n + 1, p['beta'])[n:] * sinc_win)
    win.setflags(write=False)
    return win, num_bits


def is_flac(path):
    """True when the file starts with the native FLAC marker ``fLaC`` (a path, or a WAV path: False)."""
    with open(path, 'rb') as f:
        return f.read(4) == b'fLaC'


def flac_info(data, name='stream'):
    """STREAMINFO of FLAC bytes (a whole file, or at least its metadata): dict(sample_rate, channels, bits, total_samples,
    first_frame), first_frame being the byte where the metadata blocks end.  Raises ValueError naming ``name`` for a stream that is
    not native FLAC (Ogg-encapsulated FLAC is refused) or whose metadata is cut short."""
    data = memoryview(data)
    if bytes(data[:4]) == b'OggS':
        raise ValueError(f'{name}: Ogg-encapsulated FLAC is not supported; store it as native FLAC (.flac)')
    if bytes(data[:4]) != b'fLaC':
        raise ValueError(f'{name}: not a FLAC stream (no fLaC marker)')
    off, info = 4, None
    while True:
        if off + 4 > len(data):
            raise ValueError(f'{name}: FLAC metadata runs past the end of the file at byte {off}')
        head = bytes(data[off:off + 4])
        last, btype, n = head[0] >> 7, head[0] & 0x7F, int.from_bytes(head[1:], 'big')
        if btype == 127 or off + 4 + n > len(data) or (btype == 0) != (info is None) or (btype == 0 and n != 34):
            raise ValueError(f'{name}: bad FLAC metadata block (type {btype}, {n} bytes) at byte {off}')
        if btype == 0:
            v = int.from_bytes(bytes(data[off + 14:off + 22]), 'big')
            info = dict(sample_rate=v >> 44, channels=((v >> 41) & 7) + 1, bits=((v >> 36) & 31) + 1, total_samples=v & ((1 << 36) - 1))
        off += 4 + n
        if last:
            info['first_frame'] = off
            return info


def wav_info(path):
    """(sample rate, frames, channels) from a WAV file's header or a FLAC file's STREAMINFO, without reading its samples."""
    with open(path, 'rb') as f:
        riff = f.read(12)
        if riff[:4] == b'fLaC':
            head, off, last = bytearray(riff), 4, False      # read the metadata blocks only, header by header
            while not last:
                head += f.read(max(0, off + 4 - len(head)))
                if len(head) < off + 4:
                    break
                last = head[off] >> 7
                off += 4 + int.from_bytes(head[off + 1:off + 4], 'big')
                head += f.read(max(0, off - len(head)))
            i = flac_info(bytes(head), path)
            return i['sample_rate'], i['total_samples'], i['channels']
        if len(riff) < 12 or riff[:4] != b'RIFF' or riff[8:12] != b'WAVE':
            raise ValueError(f'{path}: not a RIFF/WAVE file (FLAC files are also accepted)')
        fmt = None
        while True:
            head = f.read(8)
            if len(head) < 8:
                raise ValueError(f'{path}: no data chunk')
            cid, size = head[:4], struct.unpack('<I', head[4:])[0]
            if cid == b'fmt ':
                body = f.read(size + (size & 1))
                channels, sr = struct.unpack('<HI', body[2:8])
                block_align = struct.unpack('<H', body[12:14])[0]
                fmt = (sr, channels, block_align)
            elif cid == b'data':
                if fmt is None:
                    raise ValueError(f'{path}: data chunk before fmt chunk')
                return fmt[0], size // fmt[2], fmt[1]
            else:
                f.seek(size + (size & 1), 1)


def wav_seconds(path):
    """Duration of a WAV file in seconds, from its header."""
    sr, frames, _ = wav_info(path)
    return frames / sr


def flac_decode_device(blobs, names=None, device=None, stage_ms=None):
    """Decode FLAC files held in memory (``blobs``: bytes of whole files) in ONE device call (svb_flac_decode_batch): the bytes go to
    the device in one copy -> (float32 CUDA tensor of every stream's mono samples back to back, int64 numpy lengths, rates).  The
    samples are bit-identical to ``read_wav`` of a WAV file holding the same PCM.  Raises ValueError naming the file (``names``) and
    byte offset for a stream that does not decode.  ``stage_ms`` (a list): the CUDA-event time of the decode launches is appended."""
    import torch

    from neuralsvb_b200 import _native
    names = [f'stream {i}' for i in range(len(blobs))] if names is None else list(names)
    infos = [flac_info(b, n) for b, n in zip(blobs, names)]
    nbytes = np.array([len(b) for b in blobs], np.int64)
    first = np.array([i['first_frame'] for i in infos], np.int64)
    srs = np.array([i['sample_rate'] for i in infos], np.int32)
    chans = np.array([i['channels'] for i in infos], np.int32)
    bits = np.array([i['bits'] for i in infos], np.int32)
    total = np.array([i['total_samples'] for i in infos], np.int64)
    lib = _native.lib()
    args = [len(blobs)] + [a.ctypes.data_as(ctypes.c_void_p) for a in (nbytes, first, srs, chans, bits, total)]
    lens = np.zeros(len(blobs), np.int64)
    ws_bytes = lib.svb_flac_plan(*args, lens.ctypes.data_as(ctypes.c_void_p))
    if ws_bytes < 0:
        raise ValueError(_flac_error(lib.svb_last_error().decode('utf-8', 'replace'), names))
    if not torch.cuda.is_available():
        raise RuntimeError('FLAC decoding runs on CUDA: neuralsvb_b200 has no CPU fallback')
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    host = torch.from_numpy(np.frombuffer(b''.join(bytes(b) for b in blobs), np.uint8).copy())
    data = host.to(device)
    out = torch.empty(max(int(lens.sum()), 1), device=device)
    ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device=device)
    ms = ctypes.c_float(0.0)
    with torch.cuda.device(device):
        rc = lib.svb_flac_decode_batch(*args, ctypes.c_void_p(data.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                       ctypes.c_void_p(ws.data_ptr()), int(ws_bytes), None if stage_ms is None else ctypes.byref(ms),
                                       _native.current_stream_ptr(device))
    if stage_ms is not None and rc == 0:
        stage_ms.append(ms.value)
    if rc == -1:
        raise ValueError(_flac_error(lib.svb_last_error().decode('utf-8', 'replace'), names))
    _native.check(rc, 'flac_decode_batch')
    return out[:int(lens.sum())], lens, [int(r) for r in srs]


def _flac_error(msg, names):
    """'flac: stream 3: ...' -> the same message naming the file."""
    import re
    m = re.match(r'flac: stream (\d+): (.*)', msg)
    return f'{names[int(m.group(1))]}: {m.group(2)}' if m else msg


def read_wav(path):
    """(float32 mono samples, file rate) of a WAV or FLAC file (recognised by its magic bytes), decoded as ``librosa.load``
    documents: integer PCM / 2^(bits - 1) (scipy returns 24-bit WAV as left-justified int32; FLAC 8-bit is signed), uint8 WAV as
    (x - 128) / 128, float as is; channels averaged in float32.  A FLAC file is decoded on the GPU (``load_wav`` at its own rate);
    a WAV file needs no device."""
    if is_flac(path):
        return load_wav(path, None)
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


def _resample_args(orig_srs, lengths):
    srs = np.ascontiguousarray(orig_srs, dtype=np.int32)
    lens = np.ascontiguousarray(lengths, dtype=np.int64)
    if srs.shape != lens.shape:
        raise ValueError(f'{len(srs)} sample rates for {len(lens)} clips')
    return srs, lens


def resample_lengths(lengths, orig_srs, target_sr):
    """(before, after) padding: int(n ratio) and ceil(n ratio) samples per clip (n itself at the target rate).  Raises ValueError for a
    clip that yields no sample or a bad rate.  No CUDA call."""
    from neuralsvb_b200 import _native
    srs, lens = _resample_args(orig_srs, lengths)
    win, num_table = kaiser_best_window()
    res, out = np.zeros(len(lens), np.int64), np.zeros(len(lens), np.int64)
    if _native.lib().svb_resample_plan(int(target_sr), srs.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                                       len(lens), len(win), num_table, res.ctypes.data_as(ctypes.c_void_p),
                                       out.ctypes.data_as(ctypes.c_void_p)) < 0:
        raise ValueError(_native.lib().svb_last_error().decode('utf-8', 'replace'))
    return res, out


def resample_batch(wavs, orig_srs, target_sr):
    """Resample each float32 clip from its own rate to ``target_sr`` with resampy's kaiser_best filter, zero-padded to
    ceil(n target_sr / sr) samples like ``librosa.resample(..., fix=True)``: the clips go to the device in one copy, through
    ``resample_device`` and back.  A clip already at target_sr comes back unchanged.  Raises ValueError for a clip too short to
    yield a sample or a bad rate."""
    import torch
    wavs = [np.ascontiguousarray(w, dtype=np.float32) for w in wavs]
    if not wavs:
        return []
    if any(w.ndim != 1 for w in wavs):
        raise ValueError('resample_batch takes 1-D (mono) clips')
    srs, lens = _resample_args(orig_srs, [len(w) for w in wavs])
    _, out_lens = resample_lengths(lens, srs, target_sr)
    if not torch.cuda.is_available():
        raise RuntimeError('resample_batch runs on CUDA: neuralsvb_b200 has no CPU fallback')
    x = torch.from_numpy(np.concatenate(wavs)).to(torch.device('cuda', torch.cuda.current_device()))
    out = resample_device(x, lens, srs, target_sr).cpu().numpy()
    res, o = [], 0
    for w, sr, n in zip(wavs, srs, out_lens):
        res.append(w if int(sr) == int(target_sr) else out[o:o + int(n)])
        o += int(n)
    return res


def resample_device(wav_concat, lengths, orig_srs, target_sr):
    """``resample_batch`` on device memory (svb_resample_batch): a float32 CUDA tensor of the clips back to back, their host
    ``lengths`` and rates -> a CUDA tensor of the resampled clips back to back (``resample_lengths``' second array gives their
    lengths)."""
    import torch

    from neuralsvb_b200 import _native
    if not (torch.is_tensor(wav_concat) and wav_concat.is_cuda and wav_concat.dtype == torch.float32):
        raise TypeError('resample_device takes a float32 CUDA tensor')
    srs, lens = _resample_args(orig_srs, lengths)
    if int(lens.sum()) != wav_concat.numel():
        raise ValueError(f'lengths sum to {int(lens.sum())}, the waveform tensor has {wav_concat.numel()} samples')
    win, num_table = kaiser_best_window()
    lib = _native.lib()
    out_lens = np.zeros(len(lens), np.int64)
    ws_bytes = lib.svb_resample_plan(int(target_sr), srs.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                                     len(lens), len(win), num_table, None, out_lens.ctypes.data_as(ctypes.c_void_p))
    if ws_bytes < 0:
        raise ValueError(lib.svb_last_error().decode('utf-8', 'replace'))
    x = wav_concat.contiguous()
    out = torch.empty(max(int(out_lens.sum()), 1), device=x.device)
    ws = torch.empty(max(int(ws_bytes), 1), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        _native.check(lib.svb_resample_batch(int(target_sr), srs.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                                             len(lens), win.ctypes.data_as(ctypes.c_void_p), len(win), num_table,
                                             ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                             ctypes.c_void_p(ws.data_ptr()), int(ws_bytes), None,
                                             _native.current_stream_ptr(x.device)), 'resample')
    return out[:int(out_lens.sum())]


def decode_wavs(takes, sr, device=None):
    """[(float32 mono samples, rate)] of each take, decoded as ``read_wav`` does; a float32 array is taken to be at sr already, and a
    (samples, rate) pair, as this function returns it, is passed through.  WAV files and arrays stay numpy arrays and make no CUDA
    call.  The FLAC files of a call are read into one host buffer and decoded together (``flac_decode_device``: one copy of the
    compressed bytes to ``device``, one svb_flac_decode_batch); their samples stay there as CUDA tensors."""
    import torch
    out = [None] * len(takes)
    flac = [i for i, w in enumerate(takes) if isinstance(w, str) and is_flac(w)]
    for i, w in enumerate(takes):
        if isinstance(w, tuple):
            out[i] = w
        elif isinstance(w, str):
            if i not in flac:
                out[i] = read_wav(w)
        else:
            out[i] = (np.ascontiguousarray(w, dtype=np.float32), sr)
    if flac:
        blobs = []
        for i in flac:
            with open(takes[i], 'rb') as f:
                blobs.append(f.read())
        y, lens, rates = flac_decode_device(blobs, [takes[i] for i in flac], device)
        for i, piece, r in zip(flac, torch.split(y, [int(n) for n in lens]), rates):
            out[i] = (piece, r)
    return out


def load_takes(takes, sr, device=None):
    """The takes -- WAV or FLAC paths at any rate, float32 arrays at ``sr``, or ``decode_wavs``' (samples, rate) pairs -- as
    ``librosa.core.load(path, sr=sr)`` reads them, on the device: (float32 CUDA tensor of the takes back to back at ``sr``, int64
    numpy lengths).  One host-to-device copy of all samples decoded on the host; FLAC takes are decoded on the device and stay
    there; the off-rate takes go through one ``resample_device`` call."""
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError('load_takes runs on CUDA: neuralsvb_b200 has no CPU fallback')
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    dec = decode_wavs(takes, sr, device)
    pieces = [w for w, _ in dec]
    host = [k for k, w in enumerate(pieces) if not torch.is_tensor(w)]
    if host:
        up = torch.from_numpy(np.concatenate([pieces[k] for k in host])).to(device)
        for k, p in zip(host, torch.split(up, [len(pieces[k]) for k in host])):
            pieces[k] = p
    off = [k for k, (_, r) in enumerate(dec) if r != sr]
    if off:
        n_in, rates = [len(pieces[k]) for k in off], [dec[k][1] for k in off]
        y = resample_device(torch.cat([pieces[k] for k in off]), n_in, rates, sr)
        for k, p in zip(off, torch.split(y, [int(n) for n in resample_lengths(n_in, rates, sr)[1]])):
            pieces[k] = p
    lens = np.array([len(p) for p in pieces], np.int64)
    if len(host) == len(dec) and not off:
        return up, lens                             # already back to back
    return torch.cat(pieces), lens


def load_wav(path, sr=22050):
    """``librosa.core.load(path, sr=sr)`` for a WAV or FLAC file: (float32 mono samples at ``sr``, sr); ``sr=None`` keeps the file's
    rate.  A WAV file at ``sr`` needs no device; a file at another rate goes through ``load_takes`` and back."""
    dec = decode_wavs([path], sr)
    y, file_sr = dec[0]
    if sr is None or file_sr == sr:
        return (y if isinstance(y, np.ndarray) else y.cpu().numpy()), file_sr
    return load_takes(dec, sr)[0].cpu().numpy(), sr

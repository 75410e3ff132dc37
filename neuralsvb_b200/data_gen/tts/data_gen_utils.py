"""f0 extraction for the binarizers: the reference's ``get_pitch`` (data_gen/tts/data_gen_utils.py:150-184) on the GPU.

The reference runs Praat's autocorrelation tracker through parselmouth, once per file in a CPU worker pool.  Here the tracker is
this package's own CUDA implementation (csrc/pitch_ac.cu) of the algorithm oracle/pitch_ac.py states: the reference's settings
(time step hop / sr, floor 80 Hz, ceiling 750 Hz, voicing threshold 0.6) and Praat's documented defaults for the rest.  It is not
Praat, and agreement with parselmouth has not been measured; a user who has parselmouth can pass the reference extractor as a
binarizer's ``pitch_fn`` instead.  ``pitch_ac_device`` is the entry point; ``get_pitch_batch`` / ``get_pitch`` copy host waveforms
to the device, call it and copy the f0 back.

Placement follows the reference: ``2 * pad_size`` zero frames in front (pad_size 4 at hop 128, 2 at hop 256), then the track is cut
to ``len(mel)`` or extended with its last value.  The reference's ``np.pad`` would receive a negative right pad on this grid (its
comment notes that newer library versions do this); the cut replaces it.  ``f0[i]`` therefore describes the audio about 4.5 frames
(hop 128) before mel frame ``i``, as in the reference.
"""
import ctypes
import math

import numpy as np
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.utils.pitch_utils import f0_to_coarse

F0_MIN, F0_MAX = 80.0, 750.0
MAX_CAND = 15


def pad_size(hop):
    if hop == 128:
        return 4
    if hop == 256:
        return 2
    raise ValueError(f'get_pitch places f0 for hop_size 128 or 256 only, not {hop} (the reference asserts the same)')


def pitch_config(hparams, lpad=None):
    """The tracker's settings for ``hparams`` (audio_sample_rate, hop_size)."""
    sr, hop = int(hparams['audio_sample_rate']), int(hparams['hop_size'])
    c = _native.PitchConfig()
    c.sr, c.hop, c.floor, c.ceiling, c.time_step = sr, hop, F0_MIN, F0_MAX, hop / sr
    c.voicing_threshold, c.silence_threshold, c.octave_cost = 0.6, 0.03, 0.01
    c.octave_jump_cost, c.voiced_unvoiced_cost = 0.35, 0.14
    c.lpad = 2 * pad_size(hop) if lpad is None else int(lpad)
    return c


def _check(rc, what):
    if rc is not None and rc < 0:
        msg = _native.lib().svb_last_error().decode('utf-8', 'replace')
        if rc == -1:                   # SVB_ERR_INVALID: rejected before any launch
            raise ValueError(f'{what}: {msg}')
        raise RuntimeError(f'libsvb_vocoder {what} failed ({rc}): {msg}')
    return rc


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError('get_pitch runs on CUDA: neuralsvb_b200 has no CPU fallback')
    return torch.device('cuda', torch.cuda.current_device())


def pitch_frames(n_samples, hparams, floor=F0_MIN):
    """Analysis frames of a clip of ``n_samples`` (floor((N / sr - 3 / floor) / (hop / sr)) + 1; below 1: too short to track)."""
    sr, hop = int(hparams['audio_sample_rate']), int(hparams['hop_size'])
    return int(math.floor((n_samples / sr - 3.0 / floor) / (hop / sr))) + 1


def analysis_frames(lengths, hparams):
    """Analysis frame count of each clip (raises ValueError for a clip shorter than one window)."""
    cfg = pitch_config(hparams)
    lens = np.ascontiguousarray(lengths, dtype=np.int64)
    out = np.zeros(len(lens), np.int32)
    if _native.lib().svb_pitch_ac_workspace_bytes(ctypes.byref(cfg), lens.ctypes.data_as(ctypes.c_void_p), len(lens),
                                                  out.ctypes.data_as(ctypes.c_void_p)) < 0:
        _check(-1, 'pitch_ac')
    return out


def get_pitch_batch(wavs, mels, hparams):
    """[(f0 [len(mel)] float64 Hz, pitch ids [len(mel)] int64)] for each (wav, mel) pair: ONE device call over the ragged batch
    (one H2D copy of the waveforms, ``pitch_ac_device``, one D2H copy of the f0).  ``mels`` may also be frame counts."""
    wavs = [np.ascontiguousarray(w, dtype=np.float32) for w in wavs]
    if not wavs:
        return []
    n_mel = np.array([m if np.isscalar(m) else len(m) for m in mels], np.int64)
    assert len(n_mel) == len(wavs), (len(n_mel), len(wavs))
    x = torch.from_numpy(np.concatenate(wavs)).to(_device())
    out = pitch_ac_device(x, [len(w) for w in wavs], n_mel, hparams).f0.cpu().numpy()
    res, o = [], 0
    for T in n_mel:
        f0 = out[o:o + int(T)].astype(np.float64)
        res.append((f0, f0_to_coarse(f0)))
        o += int(T)
    return res


def get_pitch(wav_data, mel, hparams):
    """The reference's drop-in: wav [T * hop] (as wav2spec returns it), mel [T, 80] -> (f0 [T] Hz, pitch_coarse [T])."""
    return get_pitch_batch([wav_data], [mel], hparams)[0]


class PitchTrack:
    """Device tensors of one svb_pitch_ac_batch call: ``f0`` (placed, [sum mel frames]), ``cand`` [frames, 15, 2],
    ``count`` [frames], ``r`` [frames, tau_max + 2], ``frames`` (analysis frames per clip), ``stage_ms`` (3 stage times or None)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def pitch_ac_device(wav_concat, lengths, mel_frames, hparams, want_cand=False, want_r=False, stage_ms=False, lpad=None):
    """The tracker on a float32 CUDA tensor of concatenated clips (svb_pitch_ac_batch); ``lengths`` / ``mel_frames`` on the host."""
    if not (torch.is_tensor(wav_concat) and wav_concat.is_cuda and wav_concat.dtype == torch.float32):
        raise TypeError('pitch_ac_device takes a float32 CUDA tensor')
    wav_concat = wav_concat.contiguous()
    device = wav_concat.device
    cfg = pitch_config(hparams, lpad)
    lib = _native.lib()
    lens = np.ascontiguousarray(lengths, dtype=np.int64)
    n_mel = np.ascontiguousarray(mel_frames, dtype=np.int64)
    if int(lens.sum()) != wav_concat.numel():
        raise ValueError(f'lengths sum to {int(lens.sum())}, the waveform tensor has {wav_concat.numel()} samples')
    frames = np.zeros(len(lens), np.int32)
    ws_bytes = lib.svb_pitch_ac_workspace_bytes(ctypes.byref(cfg), lens.ctypes.data_as(ctypes.c_void_p), len(lens),
                                                frames.ctypes.data_as(ctypes.c_void_p))
    if ws_bytes < 0:
        _check(-1, 'pitch_ac')
    F = int(frames.sum())
    nlag = int(np.ceil(cfg.sr / cfg.floor)) + 2
    ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device=device)
    f0 = torch.empty(max(int(n_mel.sum()), 1), dtype=torch.float32, device=device)
    cand = torch.empty(F, MAX_CAND, 2, dtype=torch.float32, device=device) if want_cand else None
    count = torch.empty(F, dtype=torch.int32, device=device) if want_cand else None
    r = torch.empty(F, nlag, dtype=torch.float32, device=device) if want_r else None
    ms = np.zeros(3, np.float32) if stage_ms else None
    vp = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    with torch.cuda.device(device):
        _check(lib.svb_pitch_ac_batch(ctypes.byref(cfg), vp(wav_concat), lens.ctypes.data_as(ctypes.c_void_p), len(lens),
                                      n_mel.ctypes.data_as(ctypes.c_void_p), vp(f0), vp(ws), int(ws_bytes), vp(cand), vp(count), vp(r),
                                      None if ms is None else ms.ctypes.data_as(ctypes.c_void_p),
                                      _native.current_stream_ptr(device)), 'pitch_ac')
    return PitchTrack(f0=f0[:int(n_mel.sum())], cand=cand, count=count, r=r, frames=frames, stage_ms=ms)

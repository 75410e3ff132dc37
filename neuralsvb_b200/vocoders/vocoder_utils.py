"""Post-processing of the vocoder output (reference: vocoders/vocoder_utils.py:7-15)."""
import ctypes

import numpy as np
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.utils.hparams import hparams


def denoise(wav, v=0.1, hp=None):
    """Spectral subtraction: STFT(fft_size, hop_size, win_size, pad 'constant') -> max(|X| - v, 0), phase kept -> iSTFT.
    ``wav``: 1-D float array (host) -> float32 array of length hop * (len // hop), like the reference
    (librosa.stft / istft); computed by ``svb_denoise`` on the current CUDA device."""
    if not torch.cuda.is_available():
        raise RuntimeError('denoise needs a CUDA device: there is no CPU fallback')
    return denoise_device(torch.from_numpy(np.ascontiguousarray(wav, np.float32)).cuda(), v, hp).cpu().numpy()


def denoise_device(wav, v=0.1, hp=None):
    """``denoise`` of a 1-D float32 CUDA tensor, left on its device."""
    hp = hparams if hp is None else hp
    lib = _native.lib()
    x = wav.contiguous()[None]
    n = x.shape[1]
    hop = int(hp['hop_size'])
    c = _native.StftConfig(int(hp['fft_size']), hop, int(hp['win_size']), _native.PAD_CENTER_ZERO, _native.OUT_MAG_RAW, 0, 0, 1, 0.0)
    out = torch.empty(1, hop * (n // hop), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _native.check(lib.svb_denoise(ctypes.byref(c), _native.ptr(x), 1, n, ctypes.c_float(float(v)), _native.ptr(out),
                                      _native.current_stream_ptr(x.device)), 'denoise')
    return out[0]


def wav_to_int16(wav, norm=False):
    """save_wav's sample conversion (utils/audio.py:11-16: [wav / max|wav| per clip,] wav * 32767, truncation toward
    zero) on the device: CUDA float tensor [B, n] or [n] -> int16 tensor of the same shape (svb_wav_to_int16)."""
    if not wav.is_cuda:
        raise RuntimeError('wav_to_int16 needs a CUDA tensor: there is no CPU fallback')
    x = wav.contiguous().float()
    x2 = x.view(1, -1) if x.dim() == 1 else x.view(x.shape[0], -1)
    out = torch.empty(x2.shape, device=x.device, dtype=torch.int16)
    with torch.cuda.device(x.device):
        _native.check(_native.lib().svb_wav_to_int16(_native.ptr(x2), x2.shape[0], x2.shape[1], int(bool(norm)),
                                                     ctypes.c_void_p(out.data_ptr()), _native.current_stream_ptr(x.device)),
                      'wav_to_int16')
    return out.view(wav.shape)

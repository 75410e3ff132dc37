"""HiFi-GAN(-NSF) vocoder plugin backed by libsvb_vocoder.so.

Same surface as the reference class (vocoders/hifigan.py:39-69 + PWG.wav2spec,
vocoders/pwg.py:105-122): no-arg constructor reading ``hparams['vocoder_ckpt']``,
``spec2wav(mel[T,80], f0=[T]) -> np.float32[T*hop]``, static ``wav2spec(wav_fn)``,
registered under the names ``HifiGAN`` / ``hifigan``.  ``wav2spec`` / ``wav2spec_batch`` load their takes with
``utils.audio.load_takes`` and run ``wav2spec_device`` (svb_wav2spec_batch) on them.
"""
import ctypes
import glob
import json
import os
import re

import numpy as np
import torch

from neuralsvb_b200 import _native, utils
from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
from neuralsvb_b200.utils import audio
from neuralsvb_b200.utils.hparams import hparams, set_hparams
from neuralsvb_b200.vocoders.base_vocoder import BaseVocoder, register_vocoder


def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError('neuralsvb_b200.vocoders.hifigan needs a CUDA device: the native path has no CPU fallback')
    return torch.device('cuda', torch.cuda.current_device())


def load_model(config_path, checkpoint_path):
    """reference: vocoders/hifigan.py:17-33 (yaml -> ckpt['state_dict']['model_gen'],
    json -> ckpt['generator']; strict load; fold weight norm; eval on the GPU)."""
    device = _require_cuda()
    ckpt_dict = torch.load(checkpoint_path, map_location='cpu', weights_only=False)
    if '.yaml' in config_path:
        config = set_hparams(config_path, global_hparams=False)
        state = ckpt_dict['state_dict']['model_gen']
    elif '.json' in config_path:
        with open(config_path) as f:
            config = json.load(f)
        state = ckpt_dict['generator']
    else:
        raise ValueError(f'unknown vocoder config type: {config_path}')
    model = HifiGanGenerator(config)
    model.load_state_dict(state, strict=True)
    model.remove_weight_norm()
    model = model.eval().to(device)
    model.native_handle(device)                     # pack + upload once, like .to(device)
    print(f'| Loaded model parameters from {checkpoint_path}.')
    print(f'| HifiGAN device: {device}.')
    return model, config, device


def stft_config(hp, pad_mode, out_kind, eps, frames_major=1, clamp=0):
    c = _native.StftConfig()
    c.n_fft, c.hop, c.win = int(hp['fft_size']), int(hp['hop_size']), int(hp['win_size'])
    c.pad_mode, c.out_kind, c.clamp_input = pad_mode, out_kind, clamp
    c.n_mels, c.frames_major, c.eps = int(hp['audio_num_mel_bins']), frames_major, float(eps)
    return c


@register_vocoder
class HifiGAN(BaseVocoder):
    def __init__(self):
        base_dir = hparams['vocoder_ckpt']
        config_path = f'{base_dir}/config.yaml'
        if os.path.exists(config_path):
            ckpts = glob.glob(f'{base_dir}/model_ckpt_steps_*.ckpt')
            ckpt = sorted(ckpts, key=lambda x: int(re.findall(r'model_ckpt_steps_(\d+)\.ckpt', x)[0]))[-1]
            print('| load HifiGAN: ', ckpt)
            self.model, self.config, self.device = load_model(config_path=config_path, checkpoint_path=ckpt)
        else:
            config_path = f'{base_dir}/config.json'
            ckpt = f'{base_dir}/generator_v1'
            if os.path.exists(config_path):
                self.model, self.config, self.device = load_model(config_path=config_path, checkpoint_path=ckpt)
            else:
                raise FileNotFoundError(f'no config.yaml / config.json under vocoder_ckpt={base_dir!r}')

    @classmethod
    def from_model(cls, model, config, device=None):
        """Build the plugin around an in-memory generator (no checkpoint directory)."""
        self = cls.__new__(cls)
        self.device = device or _require_cuda()
        self.model, self.config = model.eval().to(self.device), config
        self.model.native_handle(self.device)
        return self

    def spec2wav(self, mel, **kwargs):
        """mel [T, n_mel] (numpy or CPU tensor, log10-mel), f0=[T] Hz or None -> np.float32 [T*hop]."""
        return self.spec2wav_batch(np.asarray(mel, dtype=np.float32)[None],
                                   None if kwargs.get('f0') is None
                                   else np.asarray(kwargs['f0'], dtype=np.float32)[None],
                                   seed=kwargs.get('seed'))[0]

    def spec2wav_batch(self, mels, f0s=None, seed=None, int16=False, norm=False):
        """mels [B, T, n_mel], f0s [B, T] or None (host arrays) -> np.float32 [B, T*hop].
        One call = pinned staging + H2D + generator + D2H + stream sync (svb_gen_spec2wav_host).
        ``int16=True``: save_wav's sample conversion (utils/audio.py:11-16; ``norm`` = its peak normalisation) runs on
        the device and np.int16 [B, T*hop] comes back -- half the D2H bytes, nothing left for the CPU writer pool to do
        but ``wavfile.write`` (svb_gen_spec2wav_host_i16; the denoise post-filter needs the float path).

        A list of [T_b, n_mel] mels (f0s: a list of [T_b] or None) is a ragged batch: one call vocodes every clip as
        ``spec2wav`` would vocode it alone (svb_gen_spec2wav_ragged_host), and a list of 1-D arrays of T_b*hop samples comes
        back; ``int16`` / ``norm`` / ``vocoder_denoise_c`` act per clip."""
        if isinstance(mels, (list, tuple)):
            return self._spec2wav_ragged(mels, f0s, seed, int16, norm)
        mels = np.ascontiguousarray(mels, dtype=np.float32)
        B, T, C = mels.shape
        if f0s is not None:
            f0s = np.ascontiguousarray(f0s, dtype=np.float32)
            assert f0s.shape == (B, T), (f0s.shape, (B, T))
        lib = _native.lib()
        g = self.model.native_handle(self.device)
        hop = int(lib.svb_gen_hop(g))
        if int16 and hparams.get('vocoder_denoise_c', 0.0) > 0:
            raise ValueError('int16 output and vocoder_denoise_c > 0 are exclusive (the post-filter works on floats)')
        out = np.empty((B, T * hop), np.int16 if int16 else np.float32)
        if seed is None:
            self.model.seed += 1
            seed = self.model.seed
        if int16:
            with torch.no_grad(), torch.cuda.device(self.device):
                with utils.Timer('hifigan', enable=hparams.get('profile_infer', False)):
                    _native.check(lib.svb_gen_spec2wav_host_i16(
                        g, mels.ctypes.data_as(ctypes.c_void_p),
                        None if f0s is None else f0s.ctypes.data_as(ctypes.c_void_p),
                        ctypes.c_uint64(seed), B, T, int(bool(norm)), out.ctypes.data_as(ctypes.c_void_p),
                        _native.current_stream_ptr(self.device)), 'spec2wav_i16')
            return out
        with torch.no_grad(), torch.cuda.device(self.device):
            with utils.Timer('hifigan', enable=hparams.get('profile_infer', False)):
                st = _native.current_stream_ptr(self.device)
                _native.check(lib.svb_gen_spec2wav_host(
                    g, mels.ctypes.data_as(ctypes.c_void_p),
                    None if f0s is None else f0s.ctypes.data_as(ctypes.c_void_p),
                    ctypes.c_uint64(seed), B, T, out.ctypes.data_as(ctypes.c_void_p), st), 'spec2wav')
        if hparams.get('vocoder_denoise_c', 0.0) > 0:                  # vocoders/hifigan.py:66-69
            from neuralsvb_b200.vocoders.vocoder_utils import denoise
            out = np.stack([denoise(o, v=hparams['vocoder_denoise_c']) for o in out])
        return out

    def _spec2wav_ragged(self, mels, f0s, seed, int16, norm):
        mels = [np.asarray(m, dtype=np.float32) for m in mels]
        if not mels:
            return []
        C = mels[0].shape[1] if mels[0].ndim == 2 else -1
        if any(m.ndim != 2 or m.shape[1] != C or m.shape[0] < 1 for m in mels):
            raise ValueError(f'spec2wav_batch: every mel must be [T_b >= 1, {C}], got {[m.shape for m in mels]}')
        lengths = np.array([m.shape[0] for m in mels], np.int32)
        mel_cat = np.ascontiguousarray(np.concatenate(mels))
        f0_cat = None
        if f0s is not None:
            f0s = [np.asarray(f, dtype=np.float32).reshape(-1) for f in f0s]
            if len(f0s) != len(mels) or any(len(f) != n for f, n in zip(f0s, lengths)):
                raise ValueError('spec2wav_batch: one f0 of T_b frames per mel')
            f0_cat = np.ascontiguousarray(np.concatenate(f0s))
        lib = _native.lib()
        g = self.model.native_handle(self.device)
        hop = int(lib.svb_gen_hop(g))
        if int16 and hparams.get('vocoder_denoise_c', 0.0) > 0:
            raise ValueError('int16 output and vocoder_denoise_c > 0 are exclusive (the post-filter works on floats)')
        out = np.empty(int(lengths.sum()) * hop, np.int16 if int16 else np.float32)
        if seed is None:
            self.model.seed += 1
            seed = self.model.seed
        f0p = None if f0_cat is None else f0_cat.ctypes.data_as(ctypes.c_void_p)
        with torch.no_grad(), torch.cuda.device(self.device):
            with utils.Timer('hifigan', enable=hparams.get('profile_infer', False)):
                st = _native.current_stream_ptr(self.device)
                if int16:
                    _native.check(lib.svb_gen_spec2wav_ragged_host_i16(
                        g, mel_cat.ctypes.data_as(ctypes.c_void_p), f0p, ctypes.c_uint64(seed), len(mels),
                        lengths.ctypes.data_as(ctypes.c_void_p), int(bool(norm)), out.ctypes.data_as(ctypes.c_void_p), st),
                        'spec2wav_ragged_i16')
                else:
                    _native.check(lib.svb_gen_spec2wav_ragged_host(
                        g, mel_cat.ctypes.data_as(ctypes.c_void_p), f0p, ctypes.c_uint64(seed), len(mels),
                        lengths.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), st), 'spec2wav_ragged')
        outs = np.split(out, np.cumsum(lengths.astype(np.int64) * hop)[:-1])
        if not int16 and hparams.get('vocoder_denoise_c', 0.0) > 0:      # vocoders/hifigan.py:66-69, clip by clip
            from neuralsvb_b200.vocoders.vocoder_utils import denoise
            outs = [denoise(o, v=hparams['vocoder_denoise_c']) for o in outs]
        return outs

    @staticmethod
    def wav2spec_batch(wav_fns, hp=None):
        """The binarizer's per-file ``wav2spec`` loop (data_gen/tts/base_binarizer.py:168-178,
        data_gen/singing/binarize_para.py:116-217) as ONE device call over a ragged batch: list of paths / float arrays
        -> list of host (wav [T*hop], mel [T, n_mel] log10), identical to ``wav2spec`` clip by clip.  The takes reach the device
        through ``audio.load_takes`` (files at another rate than audio_sample_rate resampled together there), then
        ``wav2spec_device``; the mels and the padded waveforms come back in one copy each."""
        hp = hparams if hp is None else hp
        device = _require_cuda()
        if hp.get('loud_norm', False):
            raise NotImplementedError('loud_norm (pyloudnorm BS.1770) is data preparation, outside this path')
        if not wav_fns:
            return []
        x, lengths = audio.load_takes(wav_fns, hp['audio_sample_rate'], device)
        mel, wav, frames = HifiGAN.wav2spec_device(x, lengths, hp)
        mel, wav = mel.cpu().numpy(), wav.cpu().numpy()
        offs, hop = np.concatenate([[0], np.cumsum(frames)]), int(hp['hop_size'])
        return [(wav[a * hop:b * hop], mel[a:b]) for a, b in zip(offs[:-1], offs[1:])]

    @staticmethod
    def wav2spec_device(wav_concat, lengths, hp=None, mel_basis=None):
        """``wav2spec_batch`` on device memory (svb_wav2spec_batch: one launch, no copy of the samples): float32 CUDA tensor of the
        clips back to back at audio_sample_rate, their host ``lengths`` -> (mels [sum T_c, n_mel] log10, waveforms [sum T_c * hop]
        zero-padded per clip, frame counts T_c as an int64 numpy array), device tensors back to back as wav2spec_batch returns
        them clip by clip.  ``mel_basis``: the [n_mel, n_fft / 2 + 1] filters already on the device (default: uploaded here)."""
        hp = hparams if hp is None else hp
        if not (torch.is_tensor(wav_concat) and wav_concat.is_cuda and wav_concat.dtype == torch.float32):
            raise TypeError('wav2spec_device takes a float32 CUDA tensor')
        wav_concat = wav_concat.contiguous()
        device = wav_concat.device
        lib = _native.lib()
        cfg = stft_config(hp, _native.PAD_CENTER_ZERO, _native.OUT_LOG10_MEL, float(hp.get('wav2spec_eps', 1e-10)))
        lens = np.ascontiguousarray(lengths, dtype=np.int64)
        if int(lens.sum()) != wav_concat.numel():
            raise ValueError(f'lengths sum to {int(lens.sum())}, the waveform tensor has {wav_concat.numel()} samples')
        frames = np.zeros(len(lens), np.int64)
        ws_bytes = lib.svb_wav2spec_workspace_bytes(ctypes.byref(cfg), lens.ctypes.data_as(ctypes.c_void_p), len(lens),
                                                    frames.ctypes.data_as(ctypes.c_void_p))
        if ws_bytes < 0:
            raise ValueError(f'wav2spec: {lib.svb_last_error().decode("utf-8", "replace")}')
        if mel_basis is None:
            mel_basis = torch.tensor(audio.build_mel_basis(hp), dtype=torch.float32, device=device)
        n = int(frames.sum())
        mel = torch.empty(n, cfg.n_mels, device=device)
        wav = torch.empty(n * cfg.hop, device=device)
        ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            _native.check(lib.svb_wav2spec_batch(ctypes.byref(cfg), _native.ptr(wav_concat), lens.ctypes.data_as(ctypes.c_void_p),
                                                 len(lens), _native.ptr(mel_basis.contiguous()), _native.ptr(mel), _native.ptr(wav),
                                                 None, ctypes.c_void_p(ws.data_ptr()), int(ws_bytes),
                                                 _native.current_stream_ptr(device)), 'wav2spec_batch')
        return mel, wav, frames

    @staticmethod
    def wav2spec(wav_fn, return_linear=False, hp=None):
        """wav file path (any sample rate: resampled like librosa.core.load) or float array at audio_sample_rate ->
        (wav [T*hop], mel [T, n_mel] log10)
        [+ normalised dB linear spectrogram [T, n_fft/2+1]]   (vocoders/pwg.py:105-122): ``wav2spec_batch`` of one take."""
        hp = hparams if hp is None else hp
        wav, mel = HifiGAN.wav2spec_batch([wav_fn], hp)[0]
        if not return_linear:
            return wav, mel
        x, n = audio.load_takes([wav_fn], hp['audio_sample_rate'])     # the linear spectrogram is of the unpadded samples
        cfg = stft_config(hp, _native.PAD_CENTER_ZERO, _native.OUT_MAG_RAW, 0.0)
        lin = torch.empty(len(mel), cfg.n_fft // 2 + 1, device=x.device)
        with torch.cuda.device(x.device):
            _native.check(_native.lib().svb_stft_forward(ctypes.byref(cfg), _native.ptr(x), 1, int(n[0]), None, _native.ptr(lin),
                                                         _native.current_stream_ptr(x.device)), 'stft_forward')
        return wav, mel, audio.normalize(audio.amp_to_db(lin.cpu().numpy()), hp)

"""Drop-in for modules/voice_conversion/dtw/naive_interpo.py (NInterpo) on the GPU: the nearest-neighbour index map of
F.interpolate(mode='nearest') (float32 scale S / T, floor, clamp to S - 1) comes from csrc/sadtw.cu, the gathers run where the
inputs are.  Name, signature and return types are the reference's; the inputs are torch tensors."""
import torch

from neuralsvb_b200.modules.voice_conversion.dtw import core as _core


def NInterpo(src, tgt, input, amateur_mel2ph, amateur_mel=None):
    """src [S] f0, tgt [..., T] (only its length is used), amateur_mel2ph [S], amateur_mel [S, H] or None ->
    (src resampled to T frames [T, 1], amateur_mel2ph resampled [T, 1] int64, amateur_mel resampled [T, H] or None).  input is
    not used, as in the reference."""
    if not (torch.is_tensor(src) and torch.is_tensor(tgt) and torch.is_tensor(amateur_mel2ph)):
        raise TypeError('NInterpo takes torch tensors, as the reference does')
    if src.dim() != 1 or amateur_mel2ph.shape != src.shape:
        raise ValueError(f'NInterpo takes src [S] and amateur_mel2ph [S], got {tuple(src.shape)} and {tuple(amateur_mel2ph.shape)}')
    if amateur_mel is not None and (amateur_mel.dim() != 2 or amateur_mel.shape[0] != src.shape[0]):
        raise ValueError(f'amateur_mel must be [S, H], got {tuple(amateur_mel.shape)}')
    T = int(tgt.shape[-1])
    idx = _core.baseline_batch([src], [torch.zeros(T, dtype=src.dtype, device=src.device)], 'NInterpo').alignment
    idx = idx.to(src.device)
    output = src[idx][:, None]
    aligned_mel2ph = amateur_mel2ph.to(idx.device).float()[idx][:, None].long()
    aligned_mel = amateur_mel[idx.to(amateur_mel.device)] if amateur_mel is not None else None
    return output, aligned_mel2ph, aligned_mel


def spec_to_figure(spec, vmin=None, vmax=None, name=''):
    raise NotImplementedError('plotting is not part of neuralsvb_b200')


def f0_to_figure(f0_src, f0_aligned=None, f0_prof=None, name='f0.png'):
    raise NotImplementedError('plotting is not part of neuralsvb_b200')

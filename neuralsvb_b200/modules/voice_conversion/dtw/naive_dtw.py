"""Drop-in for modules/voice_conversion/dtw/naive_dtw.py (NaiveDTW, ZMNaiveDTW, NNaiveDTW) on the GPU: the normalisation, the cdist
cost, the DTW and the backtrack run in csrc/sadtw.cu.  Names, signatures and return types are the reference's.  As in the
reference the inputs are torch tensors (host or device, float32 or float64): NaiveDTW takes [S, H] features (f0 as [S, 1], or a
mel as [S, 80] for the clean-mel upper bound), ZMNaiveDTW / NNaiveDTW take 1-D f0 [S]."""
import torch

from neuralsvb_b200.modules.voice_conversion.dtw import core as _core


def _torch_inputs(name, src, tgt, dim):
    if not (torch.is_tensor(src) and torch.is_tensor(tgt)):
        raise TypeError(f'{name} takes torch tensors, as the reference does')
    if src.dim() != dim or tgt.dim() != dim:
        raise ValueError(f'{name} takes {"[S, H] features" if dim == 2 else "1-D f0 [S]"}, got {tuple(src.shape)} and '
                         f'{tuple(tgt.shape)}')


def NaiveDTW(src, tgt, input):
    """One pair: (input[alignment], alignment) with the cost cdist(src [S, H], tgt [T, H])."""
    _torch_inputs('NaiveDTW', src, tgt, 2)
    return _core.align_one(src, tgt, input, 'NaiveDTW')


def ZMNaiveDTW(src, tgt, input):
    """One pair: (input[alignment], alignment) with the cost |(src - mean) - (tgt - mean)| (cdist's arithmetic)."""
    _torch_inputs('ZMNaiveDTW', src, tgt, 1)
    return _core.align_one(src, tgt, input, 'ZMNaiveDTW')


def NNaiveDTW(src, tgt, input):
    """One pair: (input[alignment], alignment) on (f0 - mean) / (std + 1e-8), std unbiased."""
    _torch_inputs('NNaiveDTW', src, tgt, 1)
    return _core.align_one(src, tgt, input, 'NNaiveDTW')


def spec_to_figure(spec, vmin=None, vmax=None, name=''):
    raise NotImplementedError('plotting is not part of neuralsvb_b200')


def f0_to_figure(f0_src, f0_aligned=None, f0_prof=None, name='f0.png'):
    raise NotImplementedError('plotting is not part of neuralsvb_b200')

"""Mel reconstruction loss of the SVB acoustic step on one CUDA kernel pair (csrc/mel_loss.cu): the masked L1 and the SSIM loss
that ``mel_loss: "ssim:0.5|l1:0.5"`` asks for (``FastSpeech2Task.l1_loss`` / ``ssim_loss(bias=6.0)``, tasks/tts/fs2.py:158-175 of the
reference, with ``ssim(..., size_average=False)``, modules/commons/ssim.py:319-351).  Both losses come from one forward launch pair
and one backward launch; the caller applies the lambdas::

    l1, ssim = mel_l1_ssim_loss(mel_out, target)
    losses['l1' + way], losses['ssim' + way] = 0.5 * l1, 0.5 * ssim
"""
import ctypes

import torch

from neuralsvb_b200 import _native


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class _MelLossFn(torch.autograd.Function):
    """(l1, ssim) as one autograd node; the backward reads both upstream gradients on the device (svb_mel_loss_backward)."""

    @staticmethod
    def forward(ctx, mel_out, target, bias):
        B, T, M = mel_out.shape
        lib = _native.lib()
        ws = torch.empty(max(1, int(_native.check(lib.svb_mel_loss_workspace_bytes(B, T, M), 'mel_loss_workspace_bytes')) // 8),
                         device=mel_out.device, dtype=torch.float64)
        stats = torch.empty(3, device=mel_out.device, dtype=torch.float64)
        with torch.cuda.device(mel_out.device):
            _native.check(lib.svb_mel_loss_forward(_vp(mel_out), _vp(target), B, T, M, ctypes.c_float(bias), _vp(ws), _vp(stats),
                                                   _native.current_stream_ptr(mel_out.device)), 'mel_loss_forward')
        ctx.bias = bias
        ctx.save_for_backward(mel_out, target, stats)
        return stats[0].float(), stats[1].float()

    @staticmethod
    def backward(ctx, g_l1, g_ssim):
        mel_out, target, stats = ctx.saved_tensors
        B, T, M = mel_out.shape
        g_l1 = None if g_l1 is None else g_l1.detach().float().contiguous()
        g_ssim = None if g_ssim is None else g_ssim.detach().float().contiguous()
        d = torch.empty_like(mel_out)
        with torch.cuda.device(mel_out.device):
            _native.check(_native.lib().svb_mel_loss_backward(_vp(mel_out), _vp(target), B, T, M, ctypes.c_float(ctx.bias), _vp(stats),
                                                              _vp(g_l1), _vp(g_ssim), _vp(d), _native.current_stream_ptr(mel_out.device)),
                          'mel_loss_backward')
        return d, None, None


def mel_l1_ssim_loss(mel_out, target, bias=6.0):
    """mel_out, target [B, T, M] (M <= 128; all-zero target frames are padding) -> (l1, ssim): float32 device scalars,
    differentiable with respect to ``mel_out``.  Both are NaN when every target frame is padding, as in the reference."""
    if not (mel_out.is_cuda and target.is_cuda):
        raise RuntimeError('neuralsvb_b200 has no CPU path: move the mel tensors to a CUDA device')
    if mel_out.shape != target.shape or mel_out.dim() != 3:
        raise ValueError(f'mel_l1_ssim_loss: mel_out {tuple(mel_out.shape)} and target {tuple(target.shape)} must both be [B, T, M]')
    return _MelLossFn.apply(mel_out.float().contiguous(), target.detach().float().contiguous(), float(bias))

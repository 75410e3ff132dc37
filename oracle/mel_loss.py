"""ORACLE (test infrastructure only; see oracle/__init__.py): restatement of the mel reconstruction losses of the SVB acoustic step,
``FastSpeech2Task.l1_loss`` / ``ssim_loss(bias=6.0)`` (tasks/tts/fs2.py:158-175 of the reference) with ``ssim(..., size_average=False)``
(modules/commons/ssim.py:319-351) and ``weights_nonzero_speech`` (tasks/tts/tts.py:127-131).  Runs in the dtype of its inputs (float64
for the GPU tests' references).  Pinned by tests/golden/mel_loss.npz, which oracle/gen_golden_train.py writes from the UNMODIFIED reference."""
import math

import torch
import torch.nn.functional as F


def window(dtype=torch.float64, size=11, sigma=1.5):
    g = torch.tensor([math.exp(-(x - size // 2) ** 2 / (2 * sigma ** 2)) for x in range(size)], dtype=dtype)
    g = g / g.sum()
    return (g[:, None] @ g[None, :])[None, None]


def weights(target):
    """[B, T, M]: 1 on frames whose target row has a non-zero element."""
    return target.abs().sum(-1, keepdim=True).ne(0).to(target.dtype).repeat(1, 1, target.shape[-1])


def ssim_map(img1, img2):
    """_ssim(..., size_average=False) on [B, 1, T, M] images."""
    w = window(img1.dtype).to(img1.device)
    mu1, mu2 = F.conv2d(img1, w, padding=5), F.conv2d(img2, w, padding=5)
    s11 = F.conv2d(img1 * img1, w, padding=5) - mu1 * mu1
    s22 = F.conv2d(img2 * img2, w, padding=5) - mu2 * mu2
    s12 = F.conv2d(img1 * img2, w, padding=5) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))).mean(1)


def l1_loss(mel_out, target):
    w = weights(target)
    return ((mel_out - target).abs() * w).sum() / w.sum()


def ssim_loss(mel_out, target, bias=6.0):
    w = weights(target)
    s = 1 - ssim_map(mel_out[:, None] + bias, target[:, None] + bias)
    return (s * w).sum() / w.sum()


def mel_l1_ssim_loss(mel_out, target, bias=6.0):
    return l1_loss(mel_out, target), ssim_loss(mel_out, target, bias)

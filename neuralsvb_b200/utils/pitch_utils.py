"""The paired singing dataset's f0 round trip (utils/pitch_utils.py of the reference): the binarized f0 in Hz goes through
norm_interp_f0 when an item is loaded (numpy, then a float32 tensor), and denorm_f0 turns it back into Hz with unvoiced and padding
frames zeroed, which is the contour the pitch alignments see.  Host code: it runs once per item."""
import numpy as np
import torch

F0_MAX = 1100.0
F0_BIN, F0_MIN = 256, 50.0
F0_MEL_MIN, F0_MEL_MAX = 1127 * np.log(1 + F0_MIN / 700), 1127 * np.log(1 + F0_MAX / 700)


def f0_to_coarse(f0):
    """Coarse pitch ids in [1, 255] from f0 in Hz (numpy): the mel-scaled f0 quantised into F0_BIN - 2 bins, unvoiced -> 1."""
    f0_mel = 1127 * np.log(1 + np.asarray(f0) / 700)
    f0_mel[f0_mel > 0] = (f0_mel[f0_mel > 0] - F0_MEL_MIN) * (F0_BIN - 2) / (F0_MEL_MAX - F0_MEL_MIN) + 1
    f0_mel[f0_mel <= 1] = 1
    f0_mel[f0_mel > F0_BIN - 1] = F0_BIN - 1
    return np.rint(f0_mel).astype(np.int64)


def norm_interp_f0(f0, hparams):
    """(float32 tensor of the normalised f0 with unvoiced frames linearly interpolated, float32 uv) from a numpy f0 in Hz."""
    f0 = np.array(f0, copy=True)
    uv = f0 == 0
    if hparams['pitch_norm'] == 'standard':
        f0 = (f0 - hparams['f0_mean']) / hparams['f0_std']
    if hparams['pitch_norm'] == 'log':
        f0 = np.log2(f0 + 1e-8)
    if hparams['use_uv']:
        f0[uv > 0] = 0
    if sum(uv) == len(f0):
        f0[uv] = 0
    elif sum(uv) > 0:
        f0[uv] = np.interp(np.where(uv)[0], np.where(~uv)[0], f0[~uv])
    return torch.FloatTensor(f0), torch.FloatTensor(uv)


def denorm_f0(f0, uv, hparams, pitch_padding=None):
    """f0 in Hz from norm_interp_f0's tensors, clamped to [0, 1100], zero where uv > 0 (use_uv) and where pitch_padding is set."""
    if hparams['pitch_norm'] == 'standard':
        f0 = f0 * hparams['f0_std'] + hparams['f0_mean']
    if hparams['pitch_norm'] == 'log':
        f0 = 2 ** f0
    f0 = f0.clamp(min=0).clamp(max=F0_MAX)
    if uv is not None and hparams['use_uv']:
        f0[uv > 0] = 0
    if pitch_padding is not None:
        f0[pitch_padding] = 0
    return f0

"""The mel discriminator of the SVB model's GAN (reference: modules/fastspeech/multi_window_disc.py, built by
tasks/tts/fs2_adv.py:22-34) on the CUDA operators of csrc/mel_disc.cu and the 2-D wgmma layer of csrc/tc_layer.cu.

Same classes, constructors, ``state_dict`` names and ``forward(x, cond=None, start_frames_wins=None)`` ->
``{'y', 'y_c', 'h', 'start_frames_wins'}`` as the reference, so a task's ``build_disc_model`` binds by changing its import.
Per window (32, 64, 128 frames of the mel, viewed as [B, 1, win, 80]) three blocks of Conv2d(3x3, stride 2, pad 1) +
LeakyReLU(0.2) + Dropout2d(0.25) [+ InstanceNorm2d(affine) on blocks 2 and 3], then ``adv_layer``.  Each operator is a
``torch.autograd.Function`` whose backward is a CUDA kernel; input and weight gradients follow ``needs_input_grad`` (the G step
wants only d mel, the D step only the parameter gradients).

  * Block 1 (Cin = 1) runs on the fp32 CUDA-core conv with the Dropout2d scale fused into its output.
  * Blocks 2 and 3 run on the wgmma layer handle (``svb_tc_layer_create_2d``, precision ``discriminators.TC_PRECISION``) when
    ``USE_TC`` is True, else on the fp32 conv; Dropout2d + InstanceNorm2d is one fused kernel pair.
  * ``adv_layer`` is a per-clip dot product kernel.

Randomness as the reference draws it: one ``np.random.randint`` start frame per window (shared by every clip), Dropout2d masks as
``torch.empty(B, C, 1, 1).bernoulli_(1 - p)`` in the reference's layer order.  ``x_len.max()`` is read once per forward (one host
synchronisation).  ``dropout_scales=`` (per window, per block: [B, C] tensors of 0 or 1/(1-p)) replaces the drawn masks.

Not supported (raise NotImplementedError at construction): ``norm_type`` other than 'in', ``reduction='none'`` and the
conditional discriminator (``cond_size > 0``); the shipped config uses none of them.  There is no CPU path.
"""
import ctypes

import numpy as np
import torch
from torch import nn

from neuralsvb_b200 import _native
from neuralsvb_b200.modules.hifigan import discriminators as D

USE_TC = True            # blocks 2 and 3 on the wgmma kernel (svb_tc_layer_create_2d); False: fp32 CUDA cores
LRELU_SLOPE = 0.2
DROPOUT_P = 0.25
IN_EPS = 1e-5


def _cuda(t):
    if not t.is_cuda:
        raise RuntimeError('the mel discriminator needs CUDA tensors: there is no CPU path')
    return t.contiguous().float()


def _mel_input(x):
    """The kernels are float32 only: a half / bfloat16 mel (autocast) is refused rather than silently run and returned as float32."""
    if x.dtype != torch.float32:
        raise TypeError(f'the mel discriminator takes a float32 mel, got {x.dtype}')
    return _cuda(x)


def _opt(t):
    return None if t is None else _cuda(t)


def _geom(conv):
    (kh, kw), (sh, sw), (ph, pw) = conv.kernel_size, conv.stride, conv.padding
    return kh, kw, sh, sw, ph, pw


def _out_hw(h, w, g):
    kh, kw, sh, sw, ph, pw = g
    return (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1


class _Conv2dFn(torch.autograd.Function):
    """y = scale[b, c] * leaky_relu(conv2d(x, w) + b) on the fp32 CUDA cores (svb_conv2d_forward / _backward)."""

    @staticmethod
    def forward(ctx, x, w, b, scale, g):
        x, w, b, scale = _cuda(x), _cuda(w), _cuda(b), _opt(scale)
        B, Cin, H, W = x.shape
        Ho, Wo = _out_hw(H, W, g)
        y = torch.empty(B, w.shape[0], Ho, Wo, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _native.check(_native.lib().svb_conv2d_forward(_native.ptr(x), _native.ptr(w), _native.ptr(b), _native.ptr(scale),
                                                           _native.ptr(y), B, Cin, w.shape[0], H, W, *g, ctypes.c_float(LRELU_SLOPE),
                                                           _native.current_stream_ptr(x.device)), 'conv2d_forward')
        ctx.save_for_backward(x, w, y, scale)
        ctx.g = g
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y, scale = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        dy = _cuda(dy)
        dz = torch.empty_like(y)
        dx = torch.empty_like(x) if need_x else None
        dw = torch.zeros_like(w) if need_w else None
        db = torch.zeros(w.shape[0], device=x.device, dtype=torch.float32) if need_b else None
        B, Cin, H, W = x.shape
        with torch.cuda.device(x.device):
            _native.check(_native.lib().svb_conv2d_backward(_native.ptr(x), _native.ptr(w), _native.ptr(y), _native.ptr(scale),
                                                            _native.ptr(dy), B, Cin, w.shape[0], H, W, *ctx.g,
                                                            ctypes.c_float(LRELU_SLOPE), _native.ptr(dz), _native.ptr(dx),
                                                            _native.ptr(dw), _native.ptr(db), _native.current_stream_ptr(x.device)),
                          'conv2d_backward')
        return dx, dw, db, None, None


class _TcLayer2d:
    """Owner of one 2-D svb_tc_layer handle (created on the first CUDA call; weights re-packed by discriminators._tc_sync_weight
    when their version changes, which reads and writes ``wkey`` / ``wref``)."""

    def __init__(self):
        self.h, self.key, self.wkey = None, None, None

    def close(self):
        if self.h is not None:
            _native.lib().svb_tc_layer_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get(self, cin, cout, g, device):
        key = (cin, cout, g, device.index, D.TC_PRECISION)
        if self.h is None or self.key != key:
            self.close()
            h = ctypes.c_void_p()
            dev = device.index if device.index is not None else torch.cuda.current_device()
            _native.check(_native.lib().svb_tc_layer_create_2d(cin, cout, *g, _native.PREC[D.TC_PRECISION], dev, ctypes.byref(h)),
                          'tc_layer_create_2d')
            self.h, self.key, self.wkey = h, key, None
        return self.h


class _Conv2dTcFn(torch.autograd.Function):
    """y = leaky_relu(conv2d(x, w) + b) on the wgmma kernel through a 2-D layer handle."""

    @staticmethod
    def forward(ctx, x, w, b, layer, g):
        x, w, b = _cuda(x), _cuda(w), _cuda(b)
        B, Cin, H, W = x.shape
        Ho, Wo = _out_hw(H, W, g)
        y = torch.empty(B, w.shape[0], Ho, Wo, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            st = _native.current_stream_ptr(x.device)
            h = layer.get(Cin, w.shape[0], g, x.device)
            D._tc_sync_weight(layer, h, w, b, st)
            _native.check(_native.lib().svb_tc_layer_forward(h, _native.ptr(x), B, H, W, ctypes.c_float(LRELU_SLOPE), _native.ptr(y), st),
                          'tc_layer_forward')
        ctx.save_for_backward(x, w, b, y)
        ctx.layer, ctx.g = layer, g
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, b, y = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        dy = _cuda(dy)
        dx = torch.empty_like(x) if need_x else None
        dw = torch.zeros_like(w) if need_w else None
        db = torch.zeros_like(b) if need_b else None
        B, Cin, H, W = x.shape
        with torch.cuda.device(x.device):
            st = _native.current_stream_ptr(x.device)
            h = ctx.layer.get(Cin, w.shape[0], ctx.g, x.device)
            D._tc_sync_weight(ctx.layer, h, w, b, st)        # no-op unless the handle took other weights since the forward
            _native.check(_native.lib().svb_tc_layer_backward(h, _native.ptr(x), _native.ptr(y), _native.ptr(dy), B, H, W,
                                                              ctypes.c_float(LRELU_SLOPE), _native.ptr(dx), _native.ptr(dw),
                                                              _native.ptr(db), st), 'tc_layer_backward')
        return dx, dw, db, None, None


class _DropINormFn(torch.autograd.Function):
    """InstanceNorm2d(affine)(scale[b, c] * v): svb_drop_inorm_forward / _backward."""

    @staticmethod
    def forward(ctx, v, scale, gamma, beta):
        v, scale, gamma, beta = _cuda(v), _opt(scale), _cuda(gamma), _cuda(beta)
        B, C = v.shape[:2]
        N = v[0, 0].numel()
        y = torch.empty_like(v)
        mean = torch.empty(B, C, device=v.device, dtype=torch.float32)
        rstd = torch.empty_like(mean)
        with torch.cuda.device(v.device):
            _native.check(_native.lib().svb_drop_inorm_forward(_native.ptr(v), _native.ptr(scale), _native.ptr(gamma), _native.ptr(beta),
                                                               B, C, N, ctypes.c_float(IN_EPS), _native.ptr(y), _native.ptr(mean),
                                                               _native.ptr(rstd), _native.current_stream_ptr(v.device)),
                          'drop_inorm_forward')
        ctx.save_for_backward(v, scale, gamma, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        v, scale, gamma, mean, rstd = ctx.saved_tensors
        need_v, _, need_g, need_b = ctx.needs_input_grad
        dy = _cuda(dy)
        B, C = v.shape[:2]
        dv = torch.empty_like(v) if need_v else None
        dg = torch.zeros_like(gamma) if need_g else None
        db = torch.zeros_like(gamma) if need_b else None
        with torch.cuda.device(v.device):
            _native.check(_native.lib().svb_drop_inorm_backward(_native.ptr(v), _native.ptr(scale), _native.ptr(gamma), _native.ptr(mean),
                                                                _native.ptr(rstd), _native.ptr(dy), B, C, v[0, 0].numel(), _native.ptr(dv),
                                                                _native.ptr(dg), _native.ptr(db), _native.current_stream_ptr(v.device)),
                          'drop_inorm_backward')
        return dv, None, dg, db


class _Linear1Fn(torch.autograd.Function):
    """adv_layer = Linear(N, 1) on x [B, N]: svb_linear1_forward / _backward."""

    @staticmethod
    def forward(ctx, x, w, b):
        x, w, b = _cuda(x), _cuda(w), _cuda(b)
        y = torch.empty(x.shape[0], 1, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _native.check(_native.lib().svb_linear1_forward(_native.ptr(x), _native.ptr(w), _native.ptr(b), x.shape[0], x.shape[1],
                                                            _native.ptr(y), _native.current_stream_ptr(x.device)), 'linear1_forward')
        ctx.save_for_backward(x, w)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad
        dy = _cuda(dy)
        dx = torch.empty_like(x) if need_x else None
        dw = torch.zeros_like(w) if need_w else None
        db = torch.zeros(1, device=x.device, dtype=torch.float32) if need_b else None
        with torch.cuda.device(x.device):
            _native.check(_native.lib().svb_linear1_backward(_native.ptr(x), _native.ptr(w), _native.ptr(dy), x.shape[0], x.shape[1],
                                                             _native.ptr(dx), _native.ptr(dw), _native.ptr(db),
                                                             _native.current_stream_ptr(x.device)), 'linear1_backward')
        return dx, dw, db


def mel_x_len(x):
    """Frames of x [B, c_in, T, F] whose bins do not all sum to 0 (a count of frames, not the index of the last one)."""
    return x.sum([1, -1]).ne(0).int().sum([-1])


def clip_starts(len_max, win_lengths, start_frames_wins, batch):
    """MultiWindowDiscriminator.clip for every window: a window longer than ``len_max`` (= x_len.max()) is skipped and its entry of
    ``start_frames_wins`` left as it is; otherwise a missing entry gets ``[np.random.randint(0, len_max - win + 1)] * batch``
    and a given one is kept.  Updates ``start_frames_wins`` in place; returns which windows fit."""
    fits = []
    for i, win in enumerate(win_lengths):
        t_end = len_max - win
        fits.append(t_end >= 0)
        if t_end >= 0 and start_frames_wins[i] is None:
            start_frames_wins[i] = [np.random.randint(low=0, high=t_end + 1)] * batch
    return fits


def _tc_eligible(cin, cout, g):
    kh, kw = g[0], g[1]
    return USE_TC and cout % 32 == 0 and cout <= 1024 and (cin * kh * kw) % 32 == 0 and cin * kh * kw <= 3072


def _check_config(norm_type, reduction, cond_size):
    if norm_type != 'in':
        raise NotImplementedError(f"mel discriminator: norm_type {norm_type!r} is not implemented natively (only 'in')")
    if reduction not in ('sum', 'stack'):
        raise NotImplementedError(f"mel discriminator: reduction {reduction!r} is not implemented natively (only 'sum' and 'stack')")
    if cond_size > 0:
        raise NotImplementedError('mel discriminator: the conditional discriminator (cond_size > 0) is not implemented natively')


class Discriminator2DFactory(nn.Module):
    """One window's discriminator.  The blocks are the reference's nn.Sequential(Conv2d, LeakyReLU, Dropout2d[, InstanceNorm2d])
    so parameter names, shapes and initialisation are the reference's; ``forward`` runs them on the native operators."""

    def __init__(self, time_length, freq_length=80, kernel=(3, 3), c_in=1, hidden_size=128, norm_type='bn', reduction='sum'):
        super().__init__()
        _check_config(norm_type, reduction, 0)
        padding = (kernel[0] // 2, kernel[1] // 2)

        def block(cin, cout, first=False):
            layers = [nn.Conv2d(cin, cout, kernel, (2, 2), padding), nn.LeakyReLU(LRELU_SLOPE, inplace=True), nn.Dropout2d(DROPOUT_P)]
            if not first:
                layers.append(nn.InstanceNorm2d(cout, affine=True))
            return nn.Sequential(*layers)

        self.model = nn.ModuleList([block(c_in, hidden_size, True), block(hidden_size, hidden_size), block(hidden_size, hidden_size)])
        self.reduction = reduction
        ds_size = (time_length // 2 ** 3, (freq_length + 7) // 2 ** 3)
        self.adv_layer = nn.Linear(hidden_size * ds_size[0] * ds_size[1], 1)
        self._tc = [None, _TcLayer2d(), _TcLayer2d()]

    def draw_dropout_scales(self, B, device):
        """The per-(b, c) Dropout2d factors of the three blocks, drawn like F.dropout2d in training mode (None in eval mode)."""
        if not self.training:
            return [None] * len(self.model)
        out = []
        for blk in self.model:
            p = blk[2].p
            out.append(torch.empty(B, blk[0].out_channels, 1, 1, device=device).bernoulli_(1 - p).div_(1 - p))
        return out

    def forward(self, x, dropout_scales=None):
        """x [B, c_in, win, F] float32 -> (validity [B, 1], h = the three block outputs)."""
        x = _mel_input(x)
        B = x.shape[0]
        if dropout_scales is None:
            dropout_scales = self.draw_dropout_scales(B, x.device)
        h = []
        for i, blk in enumerate(self.model):
            conv = blk[0]
            g = _geom(conv)
            scale = dropout_scales[i]
            scale = None if scale is None else scale.reshape(B, conv.out_channels)
            if i == 0 or not _tc_eligible(conv.in_channels, conv.out_channels, g):
                x = _Conv2dFn.apply(x, conv.weight, conv.bias, scale if i == 0 else None, g)
            else:
                x = _Conv2dTcFn.apply(x, conv.weight, conv.bias, self._tc[i], g)
            if i > 0:
                x = _DropINormFn.apply(x, scale, blk[3].weight, blk[3].bias)
            h.append(x)
        return _Linear1Fn.apply(x.reshape(B, -1), self.adv_layer.weight, self.adv_layer.bias), h


class MultiWindowDiscriminator(nn.Module):
    def __init__(self, time_lengths, cond_size=0, freq_length=80, kernel=(3, 3), c_in=1, hidden_size=128, norm_type='bn',
                 reduction='sum'):
        super().__init__()
        _check_config(norm_type, reduction, cond_size)
        self.win_lengths = time_lengths
        self.reduction = reduction
        self.conv_layers = nn.ModuleList([
            Discriminator2DFactory(t, freq_length, kernel, c_in=c_in, hidden_size=hidden_size, norm_type=norm_type, reduction=reduction)
            for t in time_lengths])

    def forward(self, x, x_len, cond=None, start_frames_wins=None, dropout_scales=None):
        """x [B, c_in, T, F], x_len [B] -> (validity or None when a window does not fit, start_frames_wins, h)."""
        if cond is not None:
            raise NotImplementedError('mel discriminator: the conditional discriminator is not implemented natively')
        x = _mel_input(x)
        if start_frames_wins is None:
            start_frames_wins = [None] * len(self.conv_layers)
        fits = clip_starts(int(x_len.max()), self.win_lengths, start_frames_wins, x.shape[0])    # the one host synchronisation
        validity, h = [], []
        for i, d in enumerate(self.conv_layers):
            if not fits[i]:
                continue
            s, win = start_frames_wins[i][0], self.win_lengths[i]
            v, h_ = d(x[:, :, s:s + win], None if dropout_scales is None else dropout_scales[i])
            h += h_
            validity.append(v)
        if len(validity) != len(self.conv_layers):
            return None, start_frames_wins, h
        if self.reduction == 'sum':
            return sum(validity), start_frames_wins, h
        return torch.stack(validity, -1), start_frames_wins, h


class Discriminator(nn.Module):
    def __init__(self, time_lengths=[32, 64, 128], freq_length=80, cond_size=0, kernel=(3, 3), c_in=1, hidden_size=128,
                 norm_type='bn', reduction='sum', uncond_disc=True):
        super().__init__()
        _check_config(norm_type, reduction, cond_size)
        self.time_lengths = time_lengths
        self.cond_size = cond_size
        self.reduction = reduction
        self.uncond_disc = uncond_disc
        if uncond_disc:
            self.discriminator = MultiWindowDiscriminator(freq_length=freq_length, time_lengths=time_lengths, kernel=kernel, c_in=c_in,
                                                          hidden_size=hidden_size, norm_type=norm_type, reduction=reduction)

    def forward(self, x, cond=None, start_frames_wins=None, dropout_scales=None):
        """x [B, T, F] (or [B, c_in, T, F]) -> {'y': [B, 1, n_win] ('stack') / [B, 1] ('sum') or None, 'y_c': None, 'h',
        'start_frames_wins'}.  ``x_len`` counts the frames whose bins do not sum to 0.  x must be float32 (TypeError otherwise)."""
        x = _mel_input(x)
        if x.dim() == 3:
            x = x[:, None, :, :]
        x_len = mel_x_len(x)
        ret = {'y_c': None, 'y': None}
        if self.uncond_disc:
            ret['y'], start_frames_wins, ret['h'] = self.discriminator(x, x_len, start_frames_wins=start_frames_wins,
                                                                       dropout_scales=dropout_scales)
        ret['start_frames_wins'] = start_frames_wins
        return ret

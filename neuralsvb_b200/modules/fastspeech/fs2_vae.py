"""WN gated dilated-conv stack of the GlobalFVAE -- first piece of the SVB acoustic step (SURVEY 8(f) N1).

Mirror of the reference class ``modules/fastspeech/fs2_vae.py:19-103`` (same constructor, ``state_dict`` names with
the weight-norm ``weight_g`` / ``weight_v`` pairs, ``remove_weight_norm``, ``forward(x, x_mask, g)``); the module only
holds parameters, the arithmetic is ``libsvb_vocoder.so`` (``svb_wn_*``, csrc/wn.cu: three wgmma convolutions per
layer plus the gate / residual-skip kernels).

Training is opt-in: ``trainable=True`` on ``WN``, ``FVAEDecoder`` / ``GlobalFVAEDecoder``, ``GlobalFVAEEncoder`` and
``GlobalFVAE``.  In ``train()`` mode with grad enabled the stacks are autograd nodes (``_WNTrainFn``,
``_FVAEDecTrainFn``) whose backward is ``svb_wn_backward`` / ``svb_fvae_decoder_backward``; weight norm is folded on the
device by ``_WeightNormFn`` so the ``weight_g`` / ``weight_v`` gradients come from ``svb_weight_norm_backward``.  Every
call owns its tape (a torch tensor kept by the autograd graph), so one module may run several training forwards before
one backward.  A trainable module keeps ONE native handle for its lifetime: after an optimizer step the folded weights
reach it on the device (``svb_wn_set_weight_dev`` + ``svb_wn_update_weights_dev``), never through the host.  With
``trainable=False`` (the default) the modules stay inference only and refuse to train.
"""
import ctypes

import torch
from torch import nn

from neuralsvb_b200 import _native


class _WNConv(nn.Module):
    """Parameter holder with the names ``torch.nn.utils.weight_norm(Conv1d)`` gives: bias, weight_g, weight_v."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(cout))
        self.weight_g = nn.Parameter(torch.ones(cout, 1, 1))
        self.weight_v = nn.Parameter(torch.randn(cout, cin, k) * 0.01)
        self.weight = None                      # set by remove_weight_norm

    def folded(self):
        if self.weight is not None:
            return self.weight
        return torch._weight_norm(self.weight_v, self.weight_g, 0)

    def folded_dev(self):
        """The folded weight as an autograd tensor: weight norm on the device (``_WeightNormFn``), or the weight itself."""
        if self.weight is not None:
            return self.weight
        from neuralsvb_b200.modules.hifigan.discriminators import _WeightNormFn
        return _WeightNormFn.apply(self.weight_v, self.weight_g)

    def remove_weight_norm(self):
        if self.weight is None:
            w = self.folded().detach()
            del self.weight_g, self.weight_v
            self.weight = nn.Parameter(w)


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class _NativeStack(nn.Module):
    """Handle management shared by WN and FVAEDecoder.  Subclasses provide ``_create(lib, device, handle_ref)`` (create +
    finalize from host copies of the folded tensors) and ``_train_tensors()`` ([(native name, folded autograd tensor)])."""

    def _init_native(self, trainable):
        self.trainable = bool(trainable)
        self._handle, self._versions, self._handle_dev = None, None, None
        self.host_uploads = 0           # handles built from host copies of the weights (a trainable module builds one)

    def _build(self, device):
        self._free()
        h = ctypes.c_void_p()
        self._create(_native.lib(), device, h)
        self._handle, self._handle_dev = h, str(device)
        self.host_uploads += 1
        return h

    def _native_handle(self, device):
        versions = tuple(p._version for p in self.parameters()) + (str(device),)
        if self._handle is not None and versions == self._versions:
            return self._handle
        h = self._build(device)
        self._versions = versions
        return h

    def _train_handle(self, device, training, tensors=None):
        """The module's one handle (trainable modules): created from host weights once, then kept in step on the device."""
        lib = _native.lib()
        versions = tuple(p._version for p in self.parameters()) + (str(device),)
        if self._handle is None or self._handle_dev != str(device):
            self._build(device)
            _native.check(lib.svb_wn_set_training(self._handle, 1), 'wn_set_training')
            self._versions = versions
        h = self._handle
        if versions != self._versions:
            _native.check(lib.svb_wn_set_training(h, 1), 'wn_set_training')
            st = _native.current_stream_ptr(device)
            if tensors is None:
                with torch.no_grad():
                    tensors = [t for _, t in self._train_tensors()]
            for name, t in zip(self._train_names(), tensors):
                t = t.detach().float().contiguous()
                _native.check(lib.svb_wn_set_weight_dev(h, name.encode(), _vp(t), t.numel(), st), f'wn_set_weight_dev({name})')
            _native.check(lib.svb_wn_update_weights_dev(h, st), 'wn_update_weights_dev')
            self._versions = versions
        _native.check(lib.svb_wn_set_training(h, 1 if training else 0), 'wn_set_training')
        return h

    def _native_backward(self, tape, B, T, dout, want_in, want_g, saved, backward_fn, din_shape, gin):
        """zero_grad, backward, then one gradient per saved tensor (same order)."""
        lib = _native.lib()
        h, dev = self._handle, dout.device
        dout = dout.contiguous().float()
        din = torch.empty(din_shape, device=dev, dtype=torch.float32) if want_in else None
        dg = torch.empty(B, gin, T, device=dev, dtype=torch.float32) if want_g else None
        with torch.cuda.device(dev):
            st = _native.current_stream_ptr(dev)
            _native.check(lib.svb_wn_zero_grad(h, st), 'wn_zero_grad')
            _native.check(backward_fn(h, _vp(tape), B, T, _vp(dout), _vp(din), _vp(dg), st), 'wn_backward')
            grads = []
            for name, like in zip(self._train_names(), saved):
                n = int(lib.svb_wn_grad_numel(h, name.encode()))
                if n != like.numel():
                    raise RuntimeError(f'gradient {name}: native {n} elements, parameter {like.numel()}')
                t = torch.empty(like.shape, device=dev, dtype=torch.float32)
                _native.check(lib.svb_wn_get_grad(h, name.encode(), _vp(t), n, st), f'wn_get_grad({name})')
                grads.append(t)
        return din, dg, grads

    def _free(self):
        if getattr(self, '_handle', None) is not None:
            _native.lib().svb_wn_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass


def check_frames(T, stride=4):
    """The frame counts a GlobalFVAE takes (vae_models.py:96-128): a multiple of the stride, because the decoder rebuilds T from the
    T / stride latent frames, and long enough that the encoder's three k = 3 stride-2 poolings leave at least one frame (T >= 60 at
    stride 4).  The reference's data loader crops every clip to a multiple of ``frames_multiple`` (4).  A shorter clip would leave
    the poolings an empty time axis, whose mean is NaN rather than an error."""
    n = T // stride
    for _ in range(3):
        n = (n - 3) // 2 + 1
    if T % stride or n < 1:
        raise ValueError(f'{T} frames: the GlobalFVAE takes a multiple of {stride} frames, at least {15 * stride} '
                         f'(its posterior encoder pools T / {stride} frames three times by 2)')


def _prep_mask_g(x_mask, g, B, T, gin):
    mask = None if not torch.is_tensor(x_mask) else x_mask.float().expand(B, 1, T).reshape(B, T).contiguous()
    gc = None if g is None else g.float().expand(B, gin, T).contiguous()
    return mask, gc


class _WNTrainFn(torch.autograd.Function):
    """Autograd node of one training forward of a native WN stack (replaces torch autograd through fs2_vae.py:62-94).
    ``tensors``: the folded weights and biases in ``WN._train_names()`` order."""

    @staticmethod
    def forward(ctx, mod, x, mask, g, *tensors):
        lib = _native.lib()
        B, H, T = x.shape
        with torch.cuda.device(x.device):
            h = mod._train_handle(x.device, True, tensors)
            tape = torch.empty(int(_native.check(lib.svb_wn_tape_bytes(h, B, T), 'wn_tape_bytes')), device=x.device, dtype=torch.uint8)
            out = torch.empty_like(x)
            _native.check(lib.svb_wn_forward_train(h, _vp(x), _vp(mask), _vp(g), B, T, _vp(out), _vp(tape),
                                                   _native.current_stream_ptr(x.device)), 'wn_forward_train')
        ctx.mod, ctx.tape, ctx.BT = mod, tape, (B, T)
        ctx.save_for_backward(*tensors)
        return out

    @staticmethod
    def backward(ctx, dout):
        saved = ctx.saved_tensors
        B, T = ctx.BT
        mod = ctx.mod
        dx, dg, grads = mod._native_backward(ctx.tape, B, T, dout, ctx.needs_input_grad[1], ctx.needs_input_grad[3], saved,
                                             _native.lib().svb_wn_backward, (B, mod.hidden_channels, T), mod.gin_channels)
        return (None, dx, None, dg) + tuple(grads)


class WN(_NativeStack):
    def __init__(self, hidden_channels, kernel_size, dilation_rate, n_layers, gin_channels=0, p_dropout=0,
                 share_cond_layers=False, is_BTC=False, precision='bf16x3', trainable=False):
        super().__init__()
        assert kernel_size % 2 == 1 and hidden_channels % 2 == 0          # fs2_vae.py:25-26
        if share_cond_layers:
            raise NotImplementedError('WN(share_cond_layers=True): the shared cond layer lives outside this module '
                                      '(glow-style use); the FVAE path of SURVEY 8(f) does not use it')
        self.is_BTC, self.hidden_channels, self.kernel_size = is_BTC, hidden_channels, kernel_size
        self.dilation_rate, self.n_layers, self.gin_channels, self.p_dropout = dilation_rate, n_layers, gin_channels, p_dropout
        self.share_cond_layers, self.precision = share_cond_layers, precision
        if gin_channels:
            self.cond_layer = _WNConv(gin_channels, 2 * hidden_channels * n_layers, 1)
        self.in_layers = nn.ModuleList(_WNConv(hidden_channels, 2 * hidden_channels, kernel_size) for _ in range(n_layers))
        self.res_skip_layers = nn.ModuleList(
            _WNConv(hidden_channels, 2 * hidden_channels if i < n_layers - 1 else hidden_channels, 1) for i in range(n_layers))
        self._init_native(trainable)

    def remove_weight_norm(self):
        for m in self.modules():
            if isinstance(m, _WNConv):
                m.remove_weight_norm()

    def _convs(self):
        out = [(f'in_layers.{i}', m) for i, m in enumerate(self.in_layers)]
        out += [(f'res_skip_layers.{i}', m) for i, m in enumerate(self.res_skip_layers)]
        if self.gin_channels:
            out.append(('cond_layer', self.cond_layer))
        return out

    def _train_names(self):
        return [f'{name}.{sfx}' for name, _ in self._convs() for sfx in ('weight', 'bias')]

    def _train_tensors(self):
        return [(f'{name}.{sfx}', t) for name, m in self._convs() for sfx, t in (('weight', m.folded_dev()), ('bias', m.bias))]

    def _create(self, lib, device, h):
        _native.check(lib.svb_wn_create(self.hidden_channels, self.kernel_size, self.dilation_rate, self.n_layers, self.gin_channels,
                                        _native.PREC[self.precision], device.index or 0, ctypes.byref(h)), 'wn_create')
        try:
            for name, m in self._convs():
                for suffix, t in (('weight', m.folded()), ('bias', m.bias)):
                    t = t.detach().float().cpu().contiguous()
                    shape = (ctypes.c_int64 * t.dim())(*t.shape)
                    _native.check(lib.svb_wn_set_weight(h, f'{name}.{suffix}'.encode(), ctypes.c_void_p(t.data_ptr()), shape, t.dim()),
                                  'wn_set_weight')
            _native.check(lib.svb_wn_finalize(h), 'wn_finalize')
        except Exception:
            lib.svb_wn_destroy(h)
            raise

    def forward(self, x, x_mask=None, g=None, **kwargs):
        """fs2_vae.py:62-94.  x [B, H, T] ([B, T, H] with is_BTC), x_mask [B, 1, T], g [B, gin, T]."""
        train = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()) and self.training
        # a trainable stack also tapes in eval mode when an input needs a gradient (a frozen stack between trainable layers)
        train = train or (self.trainable and torch.is_grad_enabled() and (x.requires_grad or (g is not None and g.requires_grad)))
        if train and not self.trainable:
            raise RuntimeError('neuralsvb_b200 WN is inference only: call .eval() and run under torch.no_grad() '
                               '(or construct it with trainable=True)')
        if train and self.training and self.p_dropout > 0:
            raise NotImplementedError(f'WN training with p_dropout={self.p_dropout}: the native stack has no dropout '
                                      '(the SVB configurations use 0)')
        if not x.is_cuda:
            raise RuntimeError('neuralsvb_b200 has no CPU path: move the module and its inputs to a CUDA device')
        if self.is_BTC:
            x = x.transpose(1, 2)
            x_mask = x_mask.transpose(1, 2) if x_mask is not None else None
        x = x.float().contiguous()
        B, H, T = x.shape
        assert H == self.hidden_channels, (H, self.hidden_channels)
        mask, gc = _prep_mask_g(x_mask, g, B, T, self.gin_channels)
        if train:
            out = _WNTrainFn.apply(self, x, mask, gc, *[t for _, t in self._train_tensors()])
            return out.transpose(1, 2) if self.is_BTC else out
        out = torch.empty_like(x)
        h = self._train_handle(x.device, False) if self.trainable else self._native_handle(x.device)
        st = torch.cuda.current_stream(x.device).cuda_stream
        _native.check(_native.lib().svb_wn_forward(h, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(mask.data_ptr()) if mask is not None else None,
                                                   ctypes.c_void_p(gc.data_ptr()) if gc is not None else None, B, T,
                                                   ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(st)), 'wn_forward')
        return out.transpose(1, 2) if self.is_BTC else out


class _FVAEDecTrainFn(torch.autograd.Function):
    """Autograd node of one training forward of the native FVAE decoder (fs2_vae.py:147-152): z, mask, g, then the folded
    weights and biases in ``FVAEDecoder._train_names()`` order."""

    @staticmethod
    def forward(ctx, mod, z, mask, g, T, *tensors):
        lib = _native.lib()
        B = z.shape[0]
        with torch.cuda.device(z.device):
            h = mod._train_handle(z.device, True, tensors)
            tape = torch.empty(int(_native.check(lib.svb_wn_tape_bytes(h, B, T), 'wn_tape_bytes')), device=z.device, dtype=torch.uint8)
            out = torch.empty(B, mod.out_channels, T, device=z.device, dtype=torch.float32)
            _native.check(lib.svb_fvae_decoder_forward_train(h, _vp(z), _vp(mask), _vp(g), B, T, _vp(out), _vp(tape),
                                                             _native.current_stream_ptr(z.device)), 'fvae_decoder_forward_train')
        ctx.mod, ctx.tape, ctx.BT, ctx.zshape = mod, tape, (B, T), tuple(z.shape)
        ctx.save_for_backward(*tensors)
        return out

    @staticmethod
    def backward(ctx, dout):
        saved = ctx.saved_tensors
        B, T = ctx.BT
        mod = ctx.mod
        dz, dg, grads = mod._native_backward(ctx.tape, B, T, dout, ctx.needs_input_grad[1], ctx.needs_input_grad[3], saved,
                                             _native.lib().svb_fvae_decoder_backward, ctx.zshape, mod.wn.gin_channels)
        return (None, dz, None, dg, None) + tuple(grads)


class FVAEDecoder(_NativeStack):
    """Mirror of ``modules/fastspeech/fs2_vae.py:130-152``: pre_net ConvTranspose1d(k = s, stride = s) -> * x_mask -> WN -> * x_mask
    -> out_proj.  One native call (``svb_fvae_decoder_forward``); ``pre_net`` / ``out_proj`` are parameter holders with the
    reference's ``state_dict`` names.  Inference only unless ``trainable=True`` (``_FVAEDecTrainFn``)."""

    def __init__(self, latent_channels, hidden_channels, out_channels, kernel_size, n_layers, gin_channels=0, p_dropout=0,
                 strides=[4], precision='bf16x3', trainable=False):
        super().__init__()
        if len(strides) != 1:
            raise NotImplementedError('FVAEDecoder: one up-sampling stride (the reference configs use strides=[4])')
        self.strides, self.hidden_size = list(strides), hidden_channels
        self.latent_channels, self.out_channels, self.precision = latent_channels, out_channels, precision
        self.pre_net = nn.Sequential(nn.ConvTranspose1d(latent_channels, hidden_channels, kernel_size=strides[0], stride=strides[0]))
        self.wn = WN(hidden_channels, kernel_size, 1, n_layers, gin_channels, p_dropout, precision=precision, trainable=trainable)
        self.out_proj = nn.Conv1d(hidden_channels, out_channels, 1)
        self._init_native(trainable)

    def _train_names(self):
        return self.wn._train_names() + ['pre_net.0.weight', 'pre_net.0.bias', 'out_proj.weight', 'out_proj.bias']

    def _train_tensors(self):
        return self.wn._train_tensors() + [('pre_net.0.weight', self.pre_net[0].weight), ('pre_net.0.bias', self.pre_net[0].bias),
                                           ('out_proj.weight', self.out_proj.weight), ('out_proj.bias', self.out_proj.bias)]

    def _create(self, lib, device, h):
        wn = self.wn
        _native.check(lib.svb_fvae_decoder_create(self.latent_channels, wn.hidden_channels, self.out_channels, wn.kernel_size, wn.n_layers,
                                                  wn.gin_channels, self.strides[0], _native.PREC[self.precision], device.index or 0,
                                                  ctypes.byref(h)), 'fvae_decoder_create')
        tensors = [(f'{name}.{sfx}', t) for name, m in wn._convs() for sfx, t in (('weight', m.folded()), ('bias', m.bias))]
        tensors += [('pre_net.0.weight', self.pre_net[0].weight), ('pre_net.0.bias', self.pre_net[0].bias),
                    ('out_proj.weight', self.out_proj.weight), ('out_proj.bias', self.out_proj.bias)]
        try:
            for name, t in tensors:
                t = t.detach().float().cpu().contiguous()
                shape = (ctypes.c_int64 * t.dim())(*t.shape)
                _native.check(lib.svb_wn_set_weight(h, name.encode(), ctypes.c_void_p(t.data_ptr()), shape, t.dim()), 'wn_set_weight')
            _native.check(lib.svb_wn_finalize(h), 'wn_finalize')
        except Exception:
            lib.svb_wn_destroy(h)
            raise

    def forward(self, x, x_mask, g):
        """x [B, latent, T / s]; x_mask [B, 1, T] (or the scalar 1 the reference passes at inference); g [B, gin, T] or None."""
        train = torch.is_grad_enabled() and self.training
        # a trainable decoder also tapes in eval mode when an input needs a gradient: the mapping step differentiates the mel
        # through the frozen eval-mode decoder (it has no dropout or BatchNorm, so the taped forward is the eval computation)
        train = train or (self.trainable and torch.is_grad_enabled() and (x.requires_grad or (torch.is_tensor(g) and g.requires_grad)))
        if train and not self.trainable:
            raise RuntimeError('neuralsvb_b200 FVAEDecoder is inference only: call .eval() and run under torch.no_grad() '
                               '(or construct it with trainable=True)')
        if train and self.training and self.wn.p_dropout > 0:
            raise NotImplementedError(f'FVAEDecoder training with p_dropout={self.wn.p_dropout}: the native stack has no dropout '
                                      '(the SVB configurations use 0)')
        if not x.is_cuda:
            raise RuntimeError('neuralsvb_b200 has no CPU path: move the module and its inputs to a CUDA device')
        x = x.float().contiguous()
        B, _, Tz = x.shape
        T = Tz * self.strides[0]
        mask, gc = _prep_mask_g(x_mask, g, B, T, self.wn.gin_channels)
        if train:
            return _FVAEDecTrainFn.apply(self, x, mask, gc, T, *[t for _, t in self._train_tensors()])
        out = torch.empty(B, self.out_channels, T, device=x.device, dtype=torch.float32)
        st = torch.cuda.current_stream(x.device).cuda_stream
        h = self._train_handle(x.device, False) if self.trainable else self._native_handle(x.device)
        _native.check(_native.lib().svb_fvae_decoder_forward(
            h, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(mask.data_ptr()) if mask is not None else None,
            ctypes.c_void_p(gc.data_ptr()) if gc is not None else None, B, T, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(st)),
            'fvae_decoder_forward')
        return out


class GlobalFVAEDecoder(FVAEDecoder):
    """``modules/voice_conversion/vae_models.py:108-128``: one latent vector per utterance, repeated over T / 4 frames."""

    def forward(self, x, x_mask, g):
        x = x.repeat(1, 1, g.shape[-1] // self.strides[0])          # [B, latent, 1] -> [B, latent, T // 4]   :122
        return super().forward(x, x_mask, g)


class GlobalFVAEEncoder(nn.Module):
    """``modules/voice_conversion/vae_models.py:81-106`` (FVAEEncoder, fs2_vae.py:106-127, plus the global pooling head):
    pre_net strided conv -> * mask -> WN (8 layers) -> * mask -> out_proj -> poolings (3 strided convs, ReLU, BatchNorm in eval
    mode) -> mean over time -> (m, logs) -> z = m + eps * exp(logs).  Every convolution is a native kernel (``svb_conv_nct_forward``
    for the strided / 1x1 layers, ``svb_wn_forward`` for the stack); the BatchNorm affine and the mean act on [B, 256, T / 32]
    tensors.  ``forward(..., eps=...)`` injects the posterior noise (parity tests); default: torch.randn_like.
    Inference only unless ``trainable=True``: then, in ``train()`` mode with grad enabled, the convolutions are the
    differentiable ``conv_nct`` / WN nodes and the poolings' BatchNorm runs in training mode (batch statistics, running
    statistics updated as the reference's nn.BatchNorm1d does)."""

    def __init__(self, in_channels, hidden_channels, latent_channels, kernel_size, n_layers, gin_channels=0, p_dropout=0, strides=[4],
                 precision='bf16x3', trainable=False):
        super().__init__()
        if len(strides) != 1:
            raise NotImplementedError('GlobalFVAEEncoder: one down-sampling stride (the reference configs use strides=[4])')
        s0 = strides[0]
        self.strides, self.hidden_size, self.latent_channels, self.trainable = list(strides), hidden_channels, latent_channels, trainable
        self.pre_net = nn.Sequential(nn.Conv1d(in_channels, hidden_channels, kernel_size=s0 * 2, stride=s0, padding=s0 // 2))
        self.wn = WN(hidden_channels, kernel_size, 1, n_layers, gin_channels, p_dropout, precision=precision, trainable=trainable)
        self.out_proj = nn.Conv1d(hidden_channels, latent_channels * 2, 1)
        c2 = latent_channels * 2
        self.poolings = nn.Sequential(nn.Conv1d(c2, c2, kernel_size=3, stride=2), nn.ReLU(), nn.BatchNorm1d(c2),
                                      nn.Conv1d(c2, c2, kernel_size=3, stride=2), nn.ReLU(), nn.BatchNorm1d(c2),
                                      nn.Conv1d(c2, c2, kernel_size=3, stride=2))

    @staticmethod
    def _bn_eval(bn, x):
        scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
        return x * scale[None, :, None] + (bn.bias - bn.running_mean * scale)[None, :, None]

    def forward(self, x, x_mask, g, eps=None, lens=None):
        """``lens`` (FrameLens of the mel frames; inference): each clip from its own frames only -- its convolutions treat the frames
        past its end as absent, and its latent is the mean over its own pooled frames (svb_global_latent_head_ragged)."""
        from neuralsvb_b200.modules.hifigan.discriminators import conv_nct
        if lens is not None:
            return self._forward_ragged(x, x_mask, g, eps, lens)
        train = torch.is_grad_enabled() and self.training
        if train and not self.trainable:
            raise RuntimeError('neuralsvb_b200 GlobalFVAEEncoder is inference only: call .eval() and run under torch.no_grad() '
                               '(or construct it with trainable=True)')
        if train and not x.is_cuda:
            raise RuntimeError('neuralsvb_b200 has no CPU path: move the module and its inputs to a CUDA device')
        s0 = self.strides[0]
        c = self.pre_net[0]
        x = conv_nct(x.float(), c.weight, c.bias, 2 * s0, stride=s0, pad=s0 // 2)                       # vae_models.py:97
        x_mask = x_mask[:, :, ::s0][:, :, :x.shape[-1]]                                                 # :98
        x = x * x_mask                                                                                  # :99
        x = self.wn(x, x_mask, g) * x_mask                                                              # :100
        x = conv_nct(x, self.out_proj.weight, self.out_proj.bias, 1)                                    # :101
        p = self.poolings
        bn = (lambda m, y: m(y)) if train else self._bn_eval                                           # BatchNorm: batch statistics / eval
        x = bn(p[2], conv_nct(x, p[0].weight, p[0].bias, 3, stride=2, slope=0.0))                       # conv + ReLU (slope 0), BatchNorm
        x = bn(p[5], conv_nct(x, p[3].weight, p[3].bias, 3, stride=2, slope=0.0))
        x = conv_nct(x, p[6].weight, p[6].bias, 3, stride=2)
        x = torch.mean(x, dim=-1, keepdim=True)                                                         # :102
        m, logs = torch.split(x, self.latent_channels, dim=1)                                           # :103
        z = m + (torch.randn_like(m) if eps is None else eps) * torch.exp(logs)                         # :104
        return z, m, logs, x_mask

    def _forward_ragged(self, x, x_mask, g, eps, lens):
        from neuralsvb_b200.modules.hifigan.discriminators import conv_nct_ragged
        s0 = self.strides[0]
        c = self.pre_net[0]
        enc = lens.map(lambda n: (n + 2 * (s0 // 2) - 2 * s0) // s0 + 1)
        x = conv_nct_ragged(x.float(), c.weight, c.bias, 2 * s0, s0, s0 // 2, 1, 1.0, lens)
        x_mask = x_mask[:, :, ::s0][:, :, :x.shape[-1]]
        x = self.wn(x * x_mask, x_mask, g) * x_mask
        x = conv_nct_ragged(x, self.out_proj.weight, self.out_proj.bias, 1, 1, 0, 1, 1.0, enc)
        p, n = self.poolings, enc
        for i, bn in ((0, p[2]), (3, p[5]), (6, None)):
            x = conv_nct_ragged(x, p[i].weight, p[i].bias, 3, 2, 0, 1, 0.0 if bn is not None else 1.0, n)
            n = n.map(lambda k: (k - 3) // 2 + 1)
            if bn is not None:
                x = self._bn_eval(bn, x).contiguous()
        B, L = x.shape[0], self.latent_channels
        eps = torch.randn(B, L, 1, device=x.device) if eps is None else eps.float().contiguous()
        m, logs, z = (torch.empty(B, L, 1, device=x.device) for _ in range(3))
        _native.check(_native.lib().svb_global_latent_head_ragged(
            _native.ptr(x.contiguous()), B, L, x.shape[-1], enc.c_host, _native.ptr(enc.dev), _native.ptr(eps), _native.ptr(m),
            _native.ptr(logs), _native.ptr(z), _native.current_stream_ptr(x.device)), 'global_latent_head_ragged')
        return z, m, logs, x_mask


class GlobalFVAE(nn.Module):
    """``modules/voice_conversion/vae_models.py:130-146`` (GlobalFVAE over TMPFVAE :11-52, FVAE fs2_vae.py:155-178) without the
    optional prior flow (``use_prior_glow: false`` in vae_global_mle_eng): ``g_pre_net`` strided conv on the condition, the global
    posterior encoder and the mel decoder -- every convolution native.  ``forward(x, x_mask, g, infer)`` returns what the reference
    returns; the KL term is computed in torch on the [B, latent, 1] statistics.  Inference / evaluation only unless
    ``trainable=True`` (passed to the encoder and the decoder)."""

    def __init__(self, in_out_channels, hidden_channels, latent_size, kernel_size, enc_n_layers, dec_n_layers, gin_channels, strides,
                 use_prior_glow=False, glow_hidden=None, glow_kernel_size=None, glow_n_blocks=None, precision='bf16x3', trainable=False):
        super().__init__()
        if use_prior_glow:
            raise NotImplementedError('GlobalFVAE(use_prior_glow=True): the prior flow is not part of the SVB configuration')
        self.strides, self.hidden_size, self.latent_size, self.use_prior_glow = list(strides), hidden_channels, latent_size, False
        self.g_pre_net = nn.Sequential(*[nn.Conv1d(gin_channels, gin_channels, kernel_size=s * 2, stride=s, padding=s // 2) for s in strides])
        self.encoder = GlobalFVAEEncoder(in_out_channels, hidden_channels, latent_size, kernel_size, enc_n_layers, gin_channels,
                                         strides=strides, precision=precision, trainable=trainable)
        self.decoder = GlobalFVAEDecoder(latent_size, hidden_channels, in_out_channels, kernel_size, dec_n_layers, gin_channels,
                                         strides=strides, precision=precision, trainable=trainable)

    def forward(self, x=None, x_mask=None, g=None, infer=False, eps=None, lens=None):
        """``lens`` (vc_modules.FrameLens of the mel frames; inference, infer=False): every clip from its own frames only (see
        MleSVBVAE.forward), x_mask then the lengths' mask."""
        from neuralsvb_b200.modules.hifigan.discriminators import conv_nct, conv_nct_ragged
        if not infer:
            check_frames(g.shape[-1], self.strides[0])
        g_sqz = g
        for c in self.g_pre_net:                                                                        # vae_models.py:20
            if lens is None:
                g_sqz = conv_nct(g_sqz.float(), c.weight, c.bias, c.kernel_size[0], stride=c.stride[0], pad=c.padding[0])
            else:
                g_sqz = conv_nct_ragged(g_sqz.float(), c.weight, c.bias, c.kernel_size[0], c.stride[0], c.padding[0], 1, 1.0, lens)
        if infer:                                                                                       # :45-52
            # the reference samples [B, latent, T / 4] here and its GlobalFVAEDecoder then repeats that T / 4 times (a shape
            # error: the SVB task never takes this branch, it calls vae_model.decoder directly, svb_vae.py:303); a GLOBAL
            # latent has one time step
            z_p = torch.randn(g_sqz.shape[0], self.latent_size, 1, device=g.device) if eps is None else eps
            return self.decoder(z_p, 1, g), z_p
        z_q, m_q, logs_q, x_mask_sqz = self.encoder(x, x_mask, g_sqz, eps=eps, lens=lens)               # :22
        x_recon = self.decoder(z_q, x_mask, g)                                                          # :23
        # validate_args=False: the argument check of torch.distributions is a device -> host synchronisation per call
        q_dist = torch.distributions.Normal(m_q, logs_q.exp(), validate_args=False)
        loss_kl = torch.distributions.kl_divergence(q_dist, torch.distributions.Normal(0.0, 1.0, validate_args=False))   # :38-39
        loss_kl = (loss_kl * x_mask_sqz).sum() / x_mask_sqz.sum() / z_q.shape[1]
        return x_recon, loss_kl, None, m_q, logs_q, x_mask_sqz, z_q

"""MultiPeriodDiscriminator / MultiScaleDiscriminator and the GAN losses, forward pass on the CUDA
operators of csrc/disc_ops.cu (reference: modules/hifigan/hifigan.py:181-365).

Same constructors, ``forward(y, y_hat, mel=None) -> (y_d_rs, y_d_gs, fmap_rs, fmap_gs)`` and
state_dict names (weight-norm ``weight_g/weight_v``; spectral-norm ``weight_orig/weight_u/weight_v``
for MSD[0]) as the reference.  With grad enabled every operator is a ``torch.autograd.Function`` whose
backward is a CUDA kernel of csrc/disc_bwd.cu (conv data / weight / bias gradients with the leaky-relu mask,
AvgPool1d, reflect pad, weight norm, loss gradients): torch only chains the nodes.  The one exception is the
spectral-norm re-parametrisation of MSD[0] (power iteration and sigma on the [Cout, Cin*K] weight matrix --
parameter-side arithmetic, a few small matrix-vector products in torch).
``use_cond=True`` (mel-conditioned discriminators, off in the shipped config): ``cond_net`` is the ConvTranspose1d
kernel pair ``svb_cond_net_forward / svb_cond_net_backward``; ``hparams['hop_size']`` is read at construction like the
reference does (hifigan.py:185-187, :292-301).
"""
import ctypes

import torch
from torch import nn

from neuralsvb_b200 import _native
from neuralsvb_b200.utils.synthetic import MPD_PERIODS, MSD_LAYERS

LRELU_SLOPE = 0.1


def _cuda(t):
    if not t.is_cuda:
        raise RuntimeError('discriminators need CUDA tensors: there is no CPU fallback')
    return t.contiguous().float()


def conv_nct(x, w, b, K, stride=1, dil=1, pad=0, groups=1, slope=1.0, W=1):
    """x [B, Cin, T(, W)] -> [B, Cout, Tout(, W)]: svb_conv_nct_forward, differentiable through svb_conv_nct_backward."""
    if torch.is_grad_enabled() and b is not None and (x.requires_grad or w.requires_grad or b.requires_grad):
        return _ConvNctFn.apply(x, w, b, K, stride, dil, pad, groups, slope, W)
    return _conv_nct_raw(x, w, b, K, stride, dil, pad, groups, slope, W)


class _ConvNctFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, K, stride, dil, pad, groups, slope, W):
        x, w, b = _cuda(x), _cuda(w), _cuda(b)
        y = _conv_nct_raw(x, w, b, K, stride, dil, pad, groups, slope, W)
        ctx.save_for_backward(x, w, y)
        ctx.cfg = (K, stride, dil, pad, groups, slope, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        K, stride, dil, pad, groups, slope, W = ctx.cfg
        lib = _native.lib()
        dy = _cuda(dy)
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        dz = torch.empty_like(y)
        dx = torch.empty_like(x) if need_x else None
        dw = torch.zeros_like(w) if need_w else None
        db = torch.zeros(w.shape[0], device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _native.check(lib.svb_conv_nct_backward(_native.ptr(x), _native.ptr(w), _native.ptr(y), _native.ptr(dy), x.shape[0],
                                                    x.shape[1], w.shape[0], x.shape[2], W, K, stride, dil, pad, groups,
                                                    ctypes.c_float(slope), _native.ptr(dz), _native.ptr(dx), _native.ptr(dw),
                                                    _native.ptr(db), _native.current_stream_ptr(x.device)), 'conv_nct_backward')
        return dx, dw, (db if need_b else None), None, None, None, None, None, None, None


USE_TC = True            # dense layers with >= 32 channels run on the wgmma kernel (svb_tc_layer_*); False: fp32 CUDA cores
TC_PRECISION = 'bf16x3'


USE_TC_GROUPED = True    # grouped k = 41 layers of the MSD on wgmma in polyphase form (svb_tc_layer_create_grouped)


def tc_eligible(cin, cout, K, stride, dil, pad, groups):
    if not USE_TC or dil != 1 or cout % 32 or cout > 1024:
        return False
    if groups != 1:
        if not USE_TC_GROUPED or cin % groups or cout % groups:
            return False
        ksp, pc, cg = -(-K // stride), cin // groups * stride, cout // groups
        gpt = 1
        while gpt <= groups and ((gpt * pc) % 32 or (gpt * cg) % 32):
            gpt *= 2
        return ksp % 2 == 1 and (ksp - 1) // 2 <= 64 and gpt <= groups and groups % gpt == 0 and gpt * pc <= 128 and gpt * cg <= 128
    if stride == 1:
        return cin % 32 == 0 and K % 2 == 1 and pad == (K - 1) // 2
    return (cin * K) % 32 == 0 and cin * K <= 3072


class TcLayer:
    """Owner of one svb_tc_layer handle (created lazily on the first CUDA call of its conv)."""

    def __init__(self):
        self.h, self.key = None, None
        self.wkey = None        # (data_ptr, version) of the weight / bias the handle holds: re-packed only when they change

    def get(self, cin, cout, K, stride, pad, device, groups=1):
        key = (cin, cout, K, stride, pad, device.index, TC_PRECISION, groups)
        if self.h is None or self.key != key:
            self.close()
            h = ctypes.c_void_p()
            dev = device.index if device.index is not None else torch.cuda.current_device()
            if groups == 1:
                _native.check(_native.lib().svb_tc_layer_create(cin, cout, K, stride, pad, _native.PREC[TC_PRECISION], dev,
                                                                ctypes.byref(h)), 'tc_layer_create')
            else:
                _native.check(_native.lib().svb_tc_layer_create_grouped(cin, cout, K, stride, pad, groups, _native.PREC[TC_PRECISION],
                                                                        dev, ctypes.byref(h)), 'tc_layer_create_grouped')
            self.h, self.key, self.wkey = h, key, None
        return self.h

    def close(self):
        if self.h is not None:
            _native.lib().svb_tc_layer_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def conv_tc(x, w, b, layer, K, stride, pad, slope, W, groups=1, wver=None):
    """Dense (or grouped, polyphase) conv through the tensor-core layer handle; same contract as conv_nct.
    ``wver``: hashable state the weight is a pure function of (see _tc_sync_weight)."""
    if torch.is_grad_enabled() and (x.requires_grad or w.requires_grad or b.requires_grad):
        return _TcConvFn.apply(x, w, b, layer, K, stride, pad, slope, W, groups, wver)
    return _tc_forward(_cuda(x), _cuda(w), _cuda(b), layer, K, stride, pad, slope, W, groups, wver)


def _tc_sync_weight(layer, h, w, b, st, wver=None):
    """Hand the effective weight to the layer handle only when it changed: the packings (gather + wgmma tiles for
    forward and data gradient) are rebuilt once per optimizer step, not on every forward / backward.  The effective
    weight is a pure function of the layer's parameters (and, for training-mode spectral norm, of its power-iteration
    count), so ``_NormConv.conv`` passes that state as ``wver``; tensors from elsewhere are keyed by identity and version."""
    key = wver or (w.data_ptr(), w._version, b.data_ptr(), b._version, tuple(w.shape))
    if layer.wkey == key:
        return
    _native.check(_native.lib().svb_tc_layer_set_weight_dev(h, _native.ptr(w), _native.ptr(b), st), 'tc_layer_set_weight')
    layer.wkey = key
    layer.wref = (w, b)         # keep the tensors alive: a freed-and-reused address must not look like the same weight


def _tc_forward(x, w, b, layer, K, stride, pad, slope, W, groups=1, wver=None):
    lib = _native.lib()
    B, Cin, Tin = x.shape[0], x.shape[1], x.shape[2]
    Cout = w.shape[0]
    with torch.cuda.device(x.device):
        st = _native.current_stream_ptr(x.device)
        h = layer.get(Cin, Cout, K, stride, pad, x.device, groups)
        _tc_sync_weight(layer, h, w, b, st, wver)
        Tout = int(lib.svb_tc_layer_out_len(h, Tin))
        y = torch.empty((B, Cout, Tout) + ((W,) if x.dim() == 4 else ()), device=x.device, dtype=torch.float32)
        _native.check(lib.svb_tc_layer_forward(h, _native.ptr(x), B, Tin, W, ctypes.c_float(slope), _native.ptr(y), st),
                      'tc_layer_forward')
    return y


class _TcConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, layer, K, stride, pad, slope, W, groups=1, wver=None):
        x, w, b = _cuda(x), _cuda(w), _cuda(b)
        y = _tc_forward(x, w, b, layer, K, stride, pad, slope, W, groups, wver)
        ctx.save_for_backward(x, w, b, y)
        ctx.cfg = (layer, K, stride, pad, slope, W, groups, wver)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, b, y = ctx.saved_tensors
        layer, K, stride, pad, slope, W, groups, wver = ctx.cfg
        lib = _native.lib()
        dy = _cuda(dy)
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        dx = torch.empty_like(x) if need_x else None
        dw = torch.zeros_like(w) if need_w else None
        db = torch.zeros_like(b) if need_b else None
        with torch.cuda.device(x.device):
            st = _native.current_stream_ptr(x.device)
            h = layer.get(x.shape[1], w.shape[0], K, stride, pad, x.device, groups)
            _tc_sync_weight(layer, h, w, b, st, wver)      # no-op unless the handle took other weights since the forward
            _native.check(lib.svb_tc_layer_backward(h, _native.ptr(x), _native.ptr(y), _native.ptr(dy), x.shape[0], x.shape[2], W,
                                                    ctypes.c_float(slope), _native.ptr(dx), _native.ptr(dw), _native.ptr(db), st),
                          'tc_layer_backward')
        return dx, dw, db, None, None, None, None, None, None, None, None


def conv_tc_ragged(x, w, b, layer, K, pad, slope, lens):
    """Stride-1 dense conv through the tensor-core layer handle on a ragged batch (inference): clip b is x[b][:, :n_b], frames past
    it absent; ``lens`` (vc_modules.FrameLens) holds n_b.  Output frames past n_b are zeros."""
    lib = _native.lib()
    x, w, b = _cuda(x), _cuda(w), _cuda(b)
    B, Cin, T = x.shape
    with torch.cuda.device(x.device):
        st = _native.current_stream_ptr(x.device)
        h = layer.get(Cin, w.shape[0], K, 1, pad, x.device)
        _tc_sync_weight(layer, h, w, b, st)
        y = torch.empty((B, w.shape[0], T), device=x.device, dtype=torch.float32)
        _native.check(lib.svb_tc_layer_forward_ragged(h, _native.ptr(x), B, T, lens.c_host, _native.ptr(lens.dev), ctypes.c_float(slope),
                                                      _native.ptr(y), st), 'tc_layer_forward_ragged')
    return y


def conv_nct_ragged(x, w, b, K, stride, pad, groups, slope, lens):
    """conv_nct on a ragged batch (inference): clip b is x[b][:, :n_b] (``lens``), its output (n_b + 2 pad - K) // stride + 1
    frames, zeros after them."""
    x = _cuda(x)
    B, Cin, Tin = x.shape
    Tout = (Tin + 2 * pad - (K - 1) - 1) // stride + 1
    y = torch.empty((B, w.shape[0], Tout), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _native.check(_native.lib().svb_conv_nct_forward_ragged(_native.ptr(x), _native.ptr(_cuda(w)), _native.ptr(_cuda(b)), _native.ptr(y),
                                                                B, Cin, w.shape[0], Tin, K, stride, 1, pad, groups, ctypes.c_float(slope),
                                                                lens.c_host, _native.ptr(lens.dev), _native.current_stream_ptr(x.device)),
                      'conv_nct_forward_ragged')
    return y


def _conv_nct_raw(x, w, b, K, stride=1, dil=1, pad=0, groups=1, slope=1.0, W=1):
    lib = _native.lib()
    x = _cuda(x)
    B, Cin, Tin = x.shape[0], x.shape[1], x.shape[2]
    Cout = w.shape[0]
    Tout = (Tin + 2 * pad - dil * (K - 1) - 1) // stride + 1
    y = torch.empty((B, Cout, Tout) + ((W,) if x.dim() == 4 else ()), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _native.check(lib.svb_conv_nct_forward(_native.ptr(x), _native.ptr(w), _native.ptr(b), _native.ptr(y), B, Cin, Cout, Tin,
                                               W, K, stride, dil, pad, groups, ctypes.c_float(slope),
                                               _native.current_stream_ptr(x.device)), 'conv_nct_forward')
    return y


class _NormConv(nn.Module):
    """Parameter container for a weight- or spectral-normalised conv; effective weight computed on the device."""

    def __init__(self, shape, spectral=False):
        super().__init__()
        cout = shape[0]
        inner = 1
        for s in shape[1:]:
            inner *= s
        self.spectral = spectral
        self.bias = nn.Parameter(torch.zeros(cout))
        v = torch.randn(*shape) * 0.02
        if spectral:
            self.weight_orig = nn.Parameter(v)
            self.register_buffer('weight_u', nn.functional.normalize(torch.randn(cout), dim=0))
            self.register_buffer('weight_v', nn.functional.normalize(torch.randn(inner), dim=0))
        else:
            self.weight_g = nn.Parameter(v.flatten(1).norm(dim=1).view(-1, *([1] * (len(shape) - 1))))
            self.weight_v = nn.Parameter(v)
        self._cache = None
        self.tc = TcLayer()

    def _wver(self):
        """State the effective weight depends on: parameter versions (+ the power-iteration count of spectral norm)."""
        wp = self.weight_orig if self.spectral else self.weight_v
        other = (self.weight_u._version, self.weight_v._version, getattr(self, '_sn_calls', 0), self.training) if self.spectral \
            else (self.weight_g._version, self.weight_g.data_ptr())
        return ('wver', id(self), wp._version, wp.data_ptr(), self.bias._version, self.bias.data_ptr()) + other

    def conv(self, x, K, stride=1, pad=0, groups=1, slope=1.0, W=1):
        """This layer's convolution on x: the tensor-core handle for dense >= 32-channel layers, else the fp32 kernel."""
        w, bias = self.effective(x.device)
        if tc_eligible(x.shape[1], w.shape[0], K, stride, 1, pad, groups) and x.is_cuda:
            return conv_tc(x, w, bias, self.tc, K, stride, pad, slope, W, groups, self._wver())
        return conv_nct(x, w, bias, K, stride=stride, pad=pad, groups=groups, slope=slope, W=W)

    def effective(self, device):
        """[Cout, Cin/groups, K] effective weight + bias on `device` (cached until parameters change).  With grad
        enabled the result is differentiable w.r.t. the parameters (weight norm: svb_weight_norm_backward)."""
        wp = self.weight_orig if self.spectral else self.weight_v
        diff = torch.is_grad_enabled() and (wp.requires_grad or self.bias.requires_grad)
        if self.spectral and self.training and wp.is_cuda:
            # torch.nn.utils.spectral_norm runs its power iteration on EVERY training-mode forward, also when this
            # discriminator's parameters are frozen (the generator step)
            eff = self._spectral_weight()
            if not diff:
                eff = eff.detach()
            return eff.reshape(eff.shape[0], eff.shape[1], -1), (self.bias if diff else self.bias.detach())
        if diff:
            if self.spectral:
                eff = self._spectral_weight()
            else:
                eff = _WeightNormFn.apply(self.weight_v, self.weight_g)
            return eff.reshape(eff.shape[0], eff.shape[1], -1), self.bias
        key = (str(device), self.bias._version, (self.weight_orig if self.spectral else self.weight_v)._version)
        if self._cache is not None and self._cache[0] == key:
            return self._cache[1], self._cache[2]
        if wp.is_cuda and wp.device == device:           # parameters already on the device: fold there, no host round trip
            with torch.no_grad():
                eff = self._spectral_weight() if self.spectral else _WeightNormFn.apply(self.weight_v, self.weight_g)
            eff = eff.detach().reshape(eff.shape[0], eff.shape[1], -1).contiguous()
            b = self.bias.detach().float()
            self._cache = (key, eff, b)
            return eff, b
        lib = _native.lib()
        dev_idx = device.index if device.index is not None else torch.cuda.current_device()
        if self.spectral:
            w = self.weight_orig.detach().float().cpu().contiguous()
            u, v = self.weight_u.float().cpu().contiguous(), self.weight_v.float().cpu().contiguous()
            sigma = ctypes.c_float()
            _native.check(lib.svb_spectral_sigma_host(_native.ptr(w), _native.ptr(u), _native.ptr(v), w.shape[0], w[0].numel(),
                                                      dev_idx, ctypes.byref(sigma)), 'spectral_sigma')
            eff = w / sigma.value
        else:
            v = self.weight_v.detach().float().cpu().contiguous()
            g = self.weight_g.detach().float().cpu().contiguous().view(-1)
            eff = torch.empty_like(v)
            _native.check(lib.svb_fold_weight_norm_host(_native.ptr(v), _native.ptr(g), v.shape[0], v[0].numel(), _native.ptr(eff),
                                                        dev_idx), 'fold_weight_norm')
        eff = eff.reshape(eff.shape[0], eff.shape[1], -1).contiguous().to(device)
        b = self.bias.detach().float().to(device)
        self._cache = (key, eff, b)
        return eff, b


    def _spectral_weight(self):
        """torch.nn.utils.spectral_norm semantics (hifigan.py:261 norm_f): in training mode one power iteration updates
        the u / v buffers in place, sigma = u . (W v) carries the gradient to weight_orig, u and v are constants."""
        wm = self.weight_orig.flatten(1)
        with torch.no_grad():
            if self.training:
                v = nn.functional.normalize(torch.mv(wm.t(), self.weight_u), dim=0, eps=1e-12)
                u = nn.functional.normalize(torch.mv(wm, v), dim=0, eps=1e-12)
                self.weight_v.copy_(v), self.weight_u.copy_(u)
                self._sn_calls = getattr(self, '_sn_calls', 0) + 1         # the effective weight changed
            u, v = self.weight_u.clone(), self.weight_v.clone()
        sigma = torch.dot(u, torch.mv(wm, v))
        return self.weight_orig / sigma


class _WeightNormFn(torch.autograd.Function):
    """w = g * v / ||v|| (norm over all dims but 0) on the device; backward = svb_weight_norm_backward."""

    @staticmethod
    def forward(ctx, v, g):
        lib = _native.lib()
        v, g = _cuda(v), _cuda(g)
        w = torch.empty_like(v)
        with torch.cuda.device(v.device):
            _native.check(lib.svb_fold_weight_norm_dev(_native.ptr(v), _native.ptr(g), v.shape[0], v[0].numel(), _native.ptr(w),
                                                       _native.current_stream_ptr(v.device)), 'fold_weight_norm_dev')
        ctx.save_for_backward(v, g)
        return w

    @staticmethod
    def backward(ctx, dw):
        v, g = ctx.saved_tensors
        lib = _native.lib()
        dw = _cuda(dw)
        dv, dg = torch.empty_like(v), torch.empty_like(g)
        with torch.cuda.device(v.device):
            _native.check(lib.svb_weight_norm_backward(_native.ptr(v), _native.ptr(g), _native.ptr(dw), v.shape[0], v[0].numel(),
                                                       _native.ptr(dv), _native.ptr(dg), _native.current_stream_ptr(v.device)),
                          'weight_norm_backward')
        return dv, dg


class _RowOpFn(torch.autograd.Function):
    """AvgPool1d(4,2,1) (kind 'pool') and the right reflect pad (kind 'pad') with their adjoint kernels."""

    @staticmethod
    def forward(ctx, x, kind, tpad):
        lib = _native.lib()
        x = _cuda(x)
        b, c, t = x.shape
        ctx.kind, ctx.shape, ctx.tpad = kind, (b, c, t), tpad
        with torch.cuda.device(x.device):
            st = _native.current_stream_ptr(x.device)
            if kind == 'pool':
                y = torch.empty(b, c, (t + 2 - 4) // 2 + 1, device=x.device)
                _native.check(lib.svb_avgpool1d_4_2_1(_native.ptr(x), _native.ptr(y), b * c, t, st), 'avgpool')
            else:
                y = torch.empty(b, c, tpad, device=x.device)
                _native.check(lib.svb_pad_reflect_right(_native.ptr(x), _native.ptr(y), b * c, t, tpad, st), 'pad_reflect_right')
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = _native.lib()
        dy = _cuda(dy)
        b, c, t = ctx.shape
        dx = torch.empty(b, c, t, device=dy.device)
        with torch.cuda.device(dy.device):
            st = _native.current_stream_ptr(dy.device)
            if ctx.kind == 'pool':
                _native.check(lib.svb_avgpool1d_4_2_1_backward(_native.ptr(dy), _native.ptr(dx), b * c, t, st), 'avgpool_backward')
            else:
                _native.check(lib.svb_pad_reflect_right_backward(_native.ptr(dy), _native.ptr(dx), b * c, t, ctx.tpad, st),
                              'pad_reflect_backward')
        return dx, None, None


class _CondNetFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mel, w, b, t):
        lib = _native.lib()
        mel, w, b = _cuda(mel), _cuda(w), _cuda(b)
        B, C, T = mel.shape
        y = torch.empty(B, 1, T * t, device=mel.device, dtype=torch.float32)
        with torch.cuda.device(mel.device):
            _native.check(lib.svb_cond_net_forward(_native.ptr(mel), _native.ptr(w), _native.ptr(b), B, C, T, 2 * t, t, t // 2,
                                                   _native.ptr(y), _native.current_stream_ptr(mel.device)), 'cond_net_forward')
        ctx.save_for_backward(mel, w)
        ctx.t = t
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = _native.lib()
        mel, w = ctx.saved_tensors
        dy = _cuda(dy)
        B, C, T = mel.shape
        dw, db = torch.zeros_like(w), torch.zeros(1, device=mel.device, dtype=torch.float32)
        with torch.cuda.device(mel.device):
            _native.check(lib.svb_cond_net_backward(_native.ptr(mel), _native.ptr(dy), B, C, T, 2 * ctx.t, ctx.t, ctx.t // 2,
                                                    _native.ptr(dw), _native.ptr(db), _native.current_stream_ptr(mel.device)),
                          'cond_net_backward')
        return None, dw, db, None


class _CondNet(nn.Module):
    """Parameters of ``cond_net = ConvTranspose1d(80, 1, 2t, stride=t, padding=t//2)`` (hifigan.py:188, :260)."""

    def __init__(self, t, n_mel=80):
        super().__init__()
        self.t = int(t)
        bound = 1.0 / (2 * self.t) ** 0.5
        self.weight = nn.Parameter(torch.empty(n_mel, 1, 2 * self.t).uniform_(-bound, bound))
        self.bias = nn.Parameter(torch.empty(1).uniform_(-bound, bound))

    def forward(self, mel):
        return _CondNetFn.apply(mel, self.weight, self.bias, self.t)


class DiscriminatorP(nn.Module):
    def __init__(self, period, kernel_size=5, stride=3, use_spectral_norm=False, use_cond=False, c_in=1):
        super().__init__()
        self.use_cond = use_cond
        if use_cond:
            from neuralsvb_b200.utils.hparams import hparams
            self.cond_net = _CondNet(hparams['hop_size'])
            c_in = 2
        self.period, self.kernel_size, self.stride = period, kernel_size, stride
        ch = [(c_in, 32), (32, 128), (128, 512), (512, 1024), (1024, 1024)]
        self.convs = nn.ModuleList([_NormConv((co, ci, kernel_size, 1), use_spectral_norm) for ci, co in ch])
        self.conv_post = _NormConv((1, 1024, 3, 1), use_spectral_norm)

    def forward(self, x, mel=None):
        x = _cuda(x)
        if self.use_cond:
            x = torch.cat([self.cond_net(mel), x], 1)                 # hifigan.py:204-206
        b, c, t = x.shape
        p = self.period
        if t % p != 0:                                   # reflect pad to a multiple of the period (:209-212)
            tp = t + (p - t % p)
            x, t = _RowOpFn.apply(x, 'pad', tp), tp
        x = x.view(b, c, t // p, p)
        fmap = []
        for i, l in enumerate(self.convs):
            x = l.conv(x, self.kernel_size, stride=(self.stride if i < 4 else 1), pad=2, slope=LRELU_SLOPE, W=p)
            fmap.append(x)
        x = self.conv_post.conv(x, 3, pad=1, W=p)
        fmap.append(x)
        return torch.flatten(x, 1, -1), fmap


BATCH_PAIRS = True       # run d(y) and d(y_hat) of a discriminator as ONE pass over [y; y_hat] when no input gradient is needed


def _pair_forward(d, y, y_hat, mel, stateful=False):
    """The reference runs every sub-discriminator twice, on y and on y_hat (hifigan.py:242-248, 314-323).  Convolutions act
    per sample, so when neither signal needs a gradient (the D step: y_hat is detached; inference) both run as one batch of 2B --
    half the launches, twice the rows per launch for the short late layers.  Not used when y_hat carries a gradient (the G step
    would pay the data gradient of the y half too) or for a module whose forward updates state per call (`stateful`: the
    spectral-norm power iteration of MSD[0] in training mode, hifigan.py:261,294)."""
    if (BATCH_PAIRS and not stateful and y.shape == y_hat.shape and
            not (torch.is_grad_enabled() and (y.requires_grad or y_hat.requires_grad))):
        B = y.shape[0]
        out, fmap = d(torch.cat([y, y_hat], 0), None if mel is None else torch.cat([mel, mel], 0))
        return out[:B], [f[:B] for f in fmap], out[B:], [f[B:] for f in fmap]
    r, fr = d(y, mel)
    g, fg = d(y_hat, mel)
    return r, fr, g, fg


class MultiPeriodDiscriminator(nn.Module):
    def __init__(self, use_cond=False, c_in=1):
        super().__init__()
        self.discriminators = nn.ModuleList([DiscriminatorP(p, use_cond=use_cond, c_in=c_in) for p in MPD_PERIODS])

    def forward(self, y, y_hat, mel=None):
        y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
        for d in self.discriminators:
            r, fr, g, fg = _pair_forward(d, y, y_hat, mel)
            y_d_rs.append(r), fmap_rs.append(fr), y_d_gs.append(g), fmap_gs.append(fg)
        return y_d_rs, y_d_gs, fmap_rs, fmap_gs


class DiscriminatorS(nn.Module):
    def __init__(self, use_spectral_norm=False, use_cond=False, upsample_rates=None, c_in=1):
        super().__init__()
        self.use_cond = use_cond
        if use_cond:
            t = 1
            for u in upsample_rates:
                t *= int(u)
            self.cond_net = _CondNet(t)
            c_in = 2
        self.convs = nn.ModuleList([_NormConv((co, (c_in if i == 0 else ci) // g, k), use_spectral_norm)
                                    for i, (ci, co, k, _, g, _) in enumerate(MSD_LAYERS)])
        self.conv_post = _NormConv((1, 1024, 3), use_spectral_norm)

    def forward(self, x, mel=None):
        fmap = []
        if self.use_cond:
            x = torch.cat([self.cond_net(mel), _cuda(x)], 1)          # hifigan.py:274-276
        for l, (_, _, k, s, g, p) in zip(self.convs, MSD_LAYERS):
            x = l.conv(x, k, stride=s, pad=p, groups=g, slope=LRELU_SLOPE)
            fmap.append(x)
        x = self.conv_post.conv(x, 3, pad=1)
        fmap.append(x)
        return torch.flatten(x, 1, -1), fmap


def avg_pool_4_2_1(x):
    return _RowOpFn.apply(x, 'pool', 0)


class MultiScaleDiscriminator(nn.Module):
    def __init__(self, use_cond=False, c_in=1):
        super().__init__()
        hop = 256
        if use_cond:
            from neuralsvb_b200.utils.hparams import hparams
            hop = hparams['hop_size']
        rates = [[4, 4, hop // 16], [4, 4, hop // 32], [4, 4, hop // 64]]          # hifigan.py:294-302
        self.discriminators = nn.ModuleList([
            DiscriminatorS(use_spectral_norm=True, use_cond=use_cond, upsample_rates=rates[0], c_in=c_in),
            DiscriminatorS(use_cond=use_cond, upsample_rates=rates[1], c_in=c_in),
            DiscriminatorS(use_cond=use_cond, upsample_rates=rates[2], c_in=c_in)])

    def forward(self, y, y_hat, mel=None):
        y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
        for i, d in enumerate(self.discriminators):
            if i != 0:
                y, y_hat = avg_pool_4_2_1(y), avg_pool_4_2_1(y_hat)
            r, fr, g, fg = _pair_forward(d, y, y_hat, mel, stateful=(i == 0 and self.training))
            y_d_rs.append(r), fmap_rs.append(fr), y_d_gs.append(g), fmap_gs.append(fg)
        return y_d_rs, y_d_gs, fmap_rs, fmap_gs


# ------------------------------------------------------------------ losses (device reductions)
def pair_stats(a, b=None, want_log=False):
    """float64 [6] on the host: sum (a-b)^2, sum a^2, sum |ln a - ln b|, sum |a-b|, sum (1-a)^2, sum b^2."""
    return pair_stats_dev(a, b, want_log).cpu()


def pair_stats_dev(a, b=None, want_log=False):
    """The same six sums as a float64 [6] DEVICE tensor (no host synchronisation: the training losses stay on the GPU)."""
    lib = _native.lib()
    a = _cuda(a)
    b = None if b is None else _cuda(b)
    out = torch.empty(6, device=a.device, dtype=torch.float64)
    with torch.cuda.device(a.device):
        _native.check(lib.svb_pair_stats(_native.ptr(a), _native.ptr(b), a.numel(), int(want_log), ctypes.c_void_p(out.data_ptr()),
                                         _native.current_stream_ptr(a.device)), 'pair_stats')
    return out


class _PairLossFn(torch.autograd.Function):
    """One reduction of the GAN losses as a differentiable scalar (float64 sum on the device, svb_pair_stats;
    gradient by svb_loss_grad).  kind: 'l1' mean |a - b|, 'one' mean (1 - a)^2, 'zero' mean a^2."""

    @staticmethod
    def forward(ctx, a, b, kind):
        a = _cuda(a)
        b = None if b is None else _cuda(b)
        s = pair_stats_dev(a, b)
        ctx.kind = kind
        ctx.save_for_backward(a, b) if b is not None else ctx.save_for_backward(a)
        return (s[{'l1': 3, 'one': 4, 'zero': 1}[kind]] / a.numel()).float()

    @staticmethod
    def backward(ctx, gout):
        lib = _native.lib()
        saved = ctx.saved_tensors
        a, b = saved[0], (saved[1] if len(saved) > 1 else None)
        n = a.numel()
        go = gout.detach().float().contiguous()          # upstream gradient: read by the kernel, never brought to the host
        da = torch.empty_like(a)
        db = None
        with torch.cuda.device(a.device):
            st = _native.current_stream_ptr(a.device)
            if ctx.kind == 'l1':
                _native.check(lib.svb_loss_grad_dev(_native.ptr(a), _native.ptr(b), 0, ctypes.c_float(1.0 / n), _native.ptr(go),
                                                    _native.ptr(da), n, 0, st), 'loss_grad')
                if ctx.needs_input_grad[1]:
                    db = torch.empty_like(b)
                    _native.check(lib.svb_loss_grad_dev(_native.ptr(b), _native.ptr(a), 0, ctypes.c_float(1.0 / n), _native.ptr(go),
                                                        _native.ptr(db), n, 0, st), 'loss_grad')
            else:
                _native.check(lib.svb_loss_grad_dev(_native.ptr(a), None, 1 if ctx.kind == 'one' else 2, ctypes.c_float(2.0 / n),
                                                    _native.ptr(go), _native.ptr(da), n, 0, st), 'loss_grad')
        return (da if ctx.needs_input_grad[0] else None), db, None


def _diff(*ts):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


def l1_loss(a, b):
    """mean |a - b| (F.l1_loss, the mel-spectrogram reconstruction loss of the vocoder G step); differentiable w.r.t. a."""
    if _diff(a, b):
        return _PairLossFn.apply(a, b, 'l1')
    return float(pair_stats(a, b)[3]) / a.numel()


def feature_loss(fmap_r, fmap_g):
    """2 * sum over discriminators and layers of mean |r - g|  (hifigan.py:328-334)."""
    loss = 0.0
    for dr, dg in zip(fmap_r, fmap_g):
        for rl, gl in zip(dr, dg):
            if _diff(rl, gl):
                loss = loss + _PairLossFn.apply(gl, rl, 'l1')
            else:
                loss += float(pair_stats(rl, gl)[3]) / rl.numel()
    return loss * 2


def discriminator_loss(disc_real_outputs, disc_generated_outputs):
    """(mean over discriminators of mean (1 - dr)^2, of mean dg^2)  (hifigan.py:337-347)."""
    r, g = 0.0, 0.0
    for dr, dg in zip(disc_real_outputs, disc_generated_outputs):
        if _diff(dr, dg):
            r = r + _PairLossFn.apply(dr, None, 'one')
            g = g + _PairLossFn.apply(dg, None, 'zero')
            continue
        s = pair_stats(dr, dg)
        r += float(s[4]) / dr.numel()
        g += float(s[5]) / dg.numel()
    n = len(disc_real_outputs)
    return r / n, g / n


def cond_discriminator_loss(outputs):
    """mean over discriminators of mean dg^2  (hifigan.py:350-356)."""
    if _diff(*outputs):
        return sum(_PairLossFn.apply(dg, None, 'zero') for dg in outputs) / len(outputs)
    return sum(float(pair_stats(dg)[1]) / dg.numel() for dg in outputs) / len(outputs)


def generator_loss(disc_outputs):
    """mean over discriminators of mean (1 - dg)^2  (hifigan.py:359-365)."""
    if _diff(*disc_outputs):
        return sum(_PairLossFn.apply(dg, None, 'one') for dg in disc_outputs) / len(disc_outputs)
    return sum(float(pair_stats(dg)[4]) / dg.numel() for dg in disc_outputs) / len(disc_outputs)

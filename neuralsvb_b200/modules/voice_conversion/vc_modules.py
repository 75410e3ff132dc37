"""PPG extractor of the SVB acoustic step (SURVEY 8(f) N1): the encoder half of the reference's ``VCASR``
(``modules/voice_conversion/vc_modules.py:56-80``) -- ``Prenet`` (``modules/fastspeech/pe.py:7-41``, mel_strides [2, 1, 1]) and two
conformer layers (``modules/fastspeech/conformer/conformer.py:9-52``, ``layers.py``, rel-pos attention
``modules/commons/espnet_transformer_attn.py:106-186``).  ``forward(mel)['h_content']`` is what ``SVBVAE.prepare_condition``
(``svb_vae.py:64-66``) consumes; the ASR token decoder is a training-time head and is not built (its checkpoint keys are ignored).

The module holds parameters under the reference's ``state_dict`` names; the arithmetic runs on [B, C, T] tensors through
``libsvb_vocoder.so``: every Conv1d / Linear is ``svb_conv_nct_forward`` (ReLU fused), LayerNorm is ``svb_layer_norm_nct``, the
attention core is ``svb_relpos_attention_nct``.  Element-wise glue (BatchNorm affine in eval mode, GLU, Swish, residual adds, masks)
is torch on the same tensors.  Inference only."""
import ctypes
import math

import torch
from torch import nn

from neuralsvb_b200 import _native


class _Holder(nn.Module):
    """Name-space node: carries sub-modules / parameters under the reference's attribute names, never called."""


USE_TC = True        # dense convolutions / linears with >= 32 frames run on the wgmma layer kernel (split-bf16, fp32 accumulate)


class FrameLens:
    """Per-clip frame counts of a ragged batch at one resolution (the length-aware inference mode): ``host`` ints, ``c_host`` the
    same as an int32 ctypes array (checked and planned by the native calls), ``dev`` an int32 device tensor (read by the kernels)."""

    def __init__(self, frames, device):
        self.host = [int(n) for n in frames]
        self.c_host = (ctypes.c_int32 * len(self.host))(*self.host)
        self.dev = torch.tensor(self.host, dtype=torch.int32, device=device)

    def map(self, f):
        """The frame counts after a layer that maps n frames to f(n)."""
        return FrameLens([f(n) for n in self.host], self.dev.device)

    def mask(self, T):
        """[B, T] float: 1 on each clip's frames, 0 after them."""
        return (torch.arange(T, device=self.dev.device)[None, :] < self.dev[:, None].long()).float()


def _conv(x, weight, bias, K=1, stride=1, pad=0, groups=1, relu=False, lens=None):
    """Conv1d / Linear on [B, C, T] through the C ABI: the tensor-core layer handle (svb_tc_layer_*, one per weight tensor, re-packed
    only when the weight changes) when the shape qualifies, else the fp32 CUDA-core kernel (svb_conv_nct_forward).
    ``lens`` (FrameLens of x): a ragged batch, each clip computed from its own frames only (svb_tc_layer_forward_ragged /
    svb_conv_nct_forward_ragged), output frames past a clip's end zero; the kernel is chosen by the layer alone, never by T."""
    from neuralsvb_b200.modules.hifigan import discriminators as D
    w = weight if weight.dim() == 3 else weight[:, :, None]
    if bias is None:
        bias = getattr(weight, '_svb_zero_bias', None)
        if bias is None or bias.device != x.device:
            bias = weight._svb_zero_bias = torch.zeros(w.shape[0], device=x.device)
    slope = 0.0 if relu else 1.0
    tc = USE_TC and groups == 1 and D.tc_eligible(w.shape[1], w.shape[0], K, stride, 1, pad, 1)
    if tc and (lens is None and x.shape[2] >= 32 or lens is not None and stride == 1):
        layer = getattr(weight, '_svb_tc_layer', None)
        if layer is None:
            layer = weight._svb_tc_layer = D.TcLayer()
        if lens is not None:
            return D.conv_tc_ragged(x, w, bias, layer, K, pad, slope, lens)
        return D.conv_tc(x, w, bias, layer, K, stride, pad, slope, 1)
    if lens is not None:
        return D.conv_nct_ragged(x, w, bias, K, stride, pad, groups, slope, lens)
    return D.conv_nct(x, w, bias, K, stride=stride, pad=pad, groups=groups, slope=slope)


def _bn_affine(bn, x):
    scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
    return x * scale[None, :, None] + (bn.bias - bn.running_mean * scale)[None, :, None]


def layer_norm_nct(x, ln):
    """nn.LayerNorm over the channel axis of [B, C, T] (svb_layer_norm_nct)."""
    x = x.contiguous()
    y = torch.empty_like(x)
    B, C, T = x.shape
    _native.check(_native.lib().svb_layer_norm_nct(_native.ptr(x), _native.ptr(ln.weight), _native.ptr(ln.bias), B, C, T, ctypes.c_float(ln.eps),
                                                   _native.ptr(y), _native.current_stream_ptr(x.device)), 'layer_norm_nct')
    return y


_PE_CACHE = {}


def rel_positions(T, H, device, max_len=5000):
    key = (T, H, str(device), max_len)
    if key not in _PE_CACHE:
        _PE_CACHE[key] = _rel_positions(T, H, device, max_len)
    return _PE_CACHE[key]


def _rel_positions(T, H, device, max_len=5000):
    """The reference's RelPositionalEncoding table (espnet_positional_embedding.py:24-46,98-112) is built once for max_len = 5000
    reversed positions and sliced from the front: row n encodes position max_len-1-n.  Returned as [H, T]."""
    assert T <= max_len
    pos = (max_len - 1 - torch.arange(T, dtype=torch.float32)).unsqueeze(1)
    div = torch.exp(torch.arange(0, H, 2, dtype=torch.float32) * -(math.log(10000.0) / H))
    pe = torch.zeros(T, H)
    pe[:, 0::2], pe[:, 1::2] = torch.sin(pos * div), torch.cos(pos * div)
    return pe.t().contiguous().to(device)


class VCASR(nn.Module):
    def __init__(self, dict_size=None, n_mel_bins=80, hidden_size=None, asr_enc_layers=None, mel_strides=None, asr_last_norm=None,
                 num_heads=4, kernel_size=31):
        super().__init__()
        if hidden_size is None or asr_enc_layers is None or mel_strides is None or asr_last_norm is None:
            from neuralsvb_b200.utils.hparams import hparams
            hidden_size = hparams['hidden_size'] if hidden_size is None else hidden_size
            asr_enc_layers = hparams['asr_enc_layers'] if asr_enc_layers is None else asr_enc_layers
            mel_strides = hparams['mel_strides'] if mel_strides is None else mel_strides
            asr_last_norm = hparams.get('asr_last_norm', True) if asr_last_norm is None else asr_last_norm
        H = self.hidden_size = hidden_size
        self.mel_strides, self.num_heads, self.kernel_size, self.asr_enc_layers = list(mel_strides), num_heads, kernel_size, asr_enc_layers
        self.mel_prenet = _Holder()
        self.mel_prenet.layers = nn.ModuleList(
            nn.Sequential(nn.Conv1d(n_mel_bins if i == 0 else H, H, kernel_size=5, padding=2, stride=s), nn.ReLU(), nn.BatchNorm1d(H))
            for i, s in enumerate(self.mel_strides))
        self.mel_prenet.out_proj = nn.Linear(H, H)
        enc = self.content_encoder = _Holder()
        enc.encoder_layers = nn.ModuleList()
        for _ in range(asr_enc_layers):
            l = _Holder()
            a = l.self_attn = _Holder()
            a.linear_q, a.linear_k, a.linear_v, a.linear_out = (nn.Linear(H, H) for _ in range(4))
            a.linear_pos = nn.Linear(H, H, bias=False)
            a.pos_bias_u, a.pos_bias_v = nn.Parameter(torch.zeros(num_heads, H // num_heads)), nn.Parameter(torch.zeros(num_heads, H // num_heads))
            for ff in ('feed_forward', 'feed_forward_macaron'):
                f = _Holder()
                f.w_1, f.w_2 = nn.Conv1d(H, 4 * H, 1), nn.Conv1d(4 * H, H, 1)
                setattr(l, ff, f)
            c = l.conv_module = _Holder()
            c.pointwise_conv1, c.depthwise_conv = nn.Conv1d(H, 2 * H, 1), nn.Conv1d(H, H, kernel_size, padding=(kernel_size - 1) // 2, groups=H)
            c.norm, c.pointwise_conv2 = nn.BatchNorm1d(H), nn.Conv1d(H, H, 1)
            l.norm_ff, l.norm_mha, l.norm_ff_macaron, l.norm_conv, l.norm_final = (nn.LayerNorm(H) for _ in range(5))
            enc.encoder_layers.append(l)
        enc.layer_norm = nn.LayerNorm(H) if asr_last_norm else nn.Linear(H, H)
        self.asr_last_norm = asr_last_norm

    def load_state_dict(self, state_dict, strict=True):
        """The token decoder / embedding of the reference checkpoint (``asr_decoder.*``, ``token_embed.*``) are training-time heads."""
        sd = {k: v for k, v in state_dict.items() if not k.startswith(('asr_decoder.', 'token_embed.'))}
        return super().load_state_dict(sd, strict=strict)

    # ---- conformer blocks on [B, C, T]
    def _ffn(self, f, x, lens=None):
        return _conv(_conv(x, f.w_1.weight, f.w_1.bias, relu=True, lens=lens), f.w_2.weight, f.w_2.bias, lens=lens)

    def _attention(self, a, x, p_emb, key_mask, lens=None):
        B, H, T = x.shape
        ver = tuple(t._version for t in (a.linear_q.weight, a.linear_k.weight, a.linear_v.weight, a.linear_q.bias)) + (str(x.device),)
        if getattr(a, '_qkv_ver', None) != ver:                     # one projection for q, k and v: weights concatenated once per update
            a._qkv_w = torch.cat([a.linear_q.weight, a.linear_k.weight, a.linear_v.weight], 0).detach()[:, :, None].contiguous()
            a._qkv_b = torch.cat([a.linear_q.bias, a.linear_k.bias, a.linear_v.bias], 0).detach().contiguous()
            a._qkv_ver = ver
        qkv = _conv(x, a._qkv_w, a._qkv_b, lens=lens)
        q, k, v = (t.contiguous() for t in qkv.split(H, 1))
        # linear_pos(pos_emb), [H, T]: row n is the same for every T, so with lengths one [T]-frame "clip" keeps the kernel choice
        p = _conv(p_emb[None], a.linear_pos.weight, None, lens=None if lens is None else FrameLens([T], x.device))[0].contiguous()
        ctx = torch.empty_like(q)
        args = (_native.ptr(q), _native.ptr(k), _native.ptr(v), _native.ptr(p), _native.ptr(a.pos_bias_u.contiguous()),
                _native.ptr(a.pos_bias_v.contiguous()), _native.ptr(key_mask), B, H, T, self.num_heads)
        if lens is None:
            _native.check(_native.lib().svb_relpos_attention_nct(*args, _native.ptr(ctx), _native.current_stream_ptr(x.device)),
                          'relpos_attention_nct')
        else:
            _native.check(_native.lib().svb_relpos_attention_nct_ragged(*args, lens.c_host, _native.ptr(lens.dev), _native.ptr(ctx),
                                                                        _native.current_stream_ptr(x.device)), 'relpos_attention_nct_ragged')
        return _conv(ctx, a.linear_out.weight, a.linear_out.bias, lens=lens)

    def _conv_module(self, c, x, lens=None):
        h = _conv(x, c.pointwise_conv1.weight, c.pointwise_conv1.bias, lens=lens)
        a, g = h.chunk(2, 1)
        h = (a * torch.sigmoid(g)).contiguous()                                                  # GLU over channels
        h = _conv(h, c.depthwise_conv.weight, c.depthwise_conv.bias, K=self.kernel_size, pad=(self.kernel_size - 1) // 2, groups=h.shape[1],
                  lens=lens)
        h = _bn_affine(c.norm, h)
        return _conv((h * torch.sigmoid(h)).contiguous(), c.pointwise_conv2.weight, c.pointwise_conv2.bias, lens=lens)   # Swish

    def forward(self, mel_input, prev_tokens=None, lens=None):
        """mel_input [B, T, 80] (all-zero frames = padding) -> {'h_content': [B, T / prod(mel_strides), H]}.
        ``lens`` (FrameLens of the mel frames): each clip is computed from its own frames only, whatever its padding holds; the
        masks come from the lengths, and frames past a clip's end are not part of the result."""
        if prev_tokens is not None:
            raise NotImplementedError('VCASR token decoder (ASR training head) is not part of the native path')
        if torch.is_grad_enabled() and self.training:
            raise RuntimeError('neuralsvb_b200 VCASR is inference only: call .eval() and run under torch.no_grad()')
        if not mel_input.is_cuda:
            raise RuntimeError('neuralsvb_b200 has no CPU path: move the module and its inputs to a CUDA device')
        mel = mel_input.float()
        if lens is None:
            nonpad = 1.0 - mel.abs().sum(-1).eq(0).float()[:, None, :]                           # pe.py:30-31
        x = mel.transpose(1, 2).contiguous()
        for seq, s in zip(self.mel_prenet.layers, self.mel_strides):                            # pe.py:34-36
            if lens is None:
                nonpad = nonpad[:, :, ::s]
                h = _conv(x, seq[0].weight, seq[0].bias, K=5, stride=s, pad=2, relu=True)
            else:
                h = _conv(x, seq[0].weight, seq[0].bias, K=5, stride=s, pad=2, relu=True, lens=lens)
                lens = lens.map(lambda n: (n - 1) // s + 1)
                nonpad = lens.mask(h.shape[2])[:, None, :]
            x = _bn_affine(seq[2], h) * nonpad
        x = _conv(x.contiguous(), self.mel_prenet.out_proj.weight, self.mel_prenet.out_proj.bias, lens=lens) * nonpad      # :40-41
        enc = self.content_encoder
        B, H, T = x.shape
        key_mask = (x.abs().sum(1) > 0).float().contiguous() if lens is None else nonpad[:, 0].contiguous()   # conformer.py:45
        p_emb = rel_positions(T, H, x.device)
        x = x * math.sqrt(H)                                                                     # RelPositionalEncoding xscale
        for l in enc.encoder_layers:                                                             # layers.py:181-260
            x = x + 0.5 * self._ffn(l.feed_forward_macaron, layer_norm_nct(x, l.norm_ff_macaron), lens)
            x = x + self._attention(l.self_attn, layer_norm_nct(x, l.norm_mha), p_emb, key_mask, lens)
            x = x + self._conv_module(l.conv_module, layer_norm_nct(x, l.norm_conv), lens)
            x = x + 0.5 * self._ffn(l.feed_forward, layer_norm_nct(x, l.norm_ff), lens)
            x = layer_norm_nct(x, l.norm_final)
        x = layer_norm_nct(x, enc.layer_norm) if self.asr_last_norm else _conv(x, enc.layer_norm.weight, enc.layer_norm.bias, lens=lens)
        return {'h_content': (x * key_mask[:, None, :]).transpose(1, 2)}                        # conformer.py:51

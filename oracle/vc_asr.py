"""ORACLE (test infrastructure only; see oracle/__init__.py): torch-CPU restatement of the PPG extractor of the SVB
acoustic step -- ``VCASR.forward(mel)['h_content']`` of the reference: modules/voice_conversion/vc_modules.py:56-80 =
Prenet (modules/fastspeech/pe.py:7-41) + ConformerLayers (modules/fastspeech/conformer/conformer.py:9-52, layers.py,
modules/commons/espnet_transformer_attn.py:106-186, espnet_positional_embedding.py:89-113).  Eval mode (dropout off, BatchNorm
running statistics).  Pinned by tests/golden/vc_asr.npz, written by oracle/gen_golden.py from the UNMODIFIED reference class."""
import math

import torch
import torch.nn.functional as F


def _bn(x, w, prefix):
    return F.batch_norm(x, w[prefix + '.running_mean'], w[prefix + '.running_var'], w[prefix + '.weight'], w[prefix + '.bias'], False, 0.0, 1e-5)


def prenet_forward(w, mel, strides):
    """pe.py:24-41.  mel [B, T, 80] -> x [B, T', H] (T' = T / prod(strides)), nonpadding [B, 1, T']."""
    nonpad = 1.0 - mel.abs().sum(-1).eq(0).float()[:, None, :]
    x = mel.transpose(1, 2)
    for i, s in enumerate(strides):
        nonpad = nonpad[:, :, ::s]
        x = F.conv1d(x, w[f'mel_prenet.layers.{i}.0.weight'], w[f'mel_prenet.layers.{i}.0.bias'], stride=s, padding=2)
        x = _bn(torch.relu(x), w, f'mel_prenet.layers.{i}.2') * nonpad
    x = F.linear(x.transpose(1, 2), w['mel_prenet.out_proj.weight'], w['mel_prenet.out_proj.bias'])
    return x * nonpad.transpose(1, 2)


def rel_positions(T, H, max_len=5000):
    """RelPositionalEncoding (espnet_positional_embedding.py:24-46,98-112): the table is built ONCE, at construction, for
    max_len = 5000 positions in reverse order, and forward slices its first T rows -- row n encodes position max_len-1-n
    (not T-1-n) for every T <= max_len."""
    assert T <= max_len
    pos = (max_len - 1 - torch.arange(T, dtype=torch.float32)).unsqueeze(1)
    div = torch.exp(torch.arange(0, H, 2, dtype=torch.float32) * -(math.log(10000.0) / H))
    pe = torch.zeros(T, H)
    pe[:, 0::2], pe[:, 1::2] = torch.sin(pos * div), torch.cos(pos * div)
    return pe


def shifted_bd(bd):
    """rel_shift (espnet_transformer_attn.py:127-145) written as the index map it performs on bd [B, h, T, T]:
    out[i][j] = bd[i][T-1-(i-j)] for j <= i ; 0 for j == i+1 ; bd[i+1][j-i-2] for j >= i+2."""
    T = bd.shape[-1]
    i = torch.arange(T, device=bd.device)[:, None]
    j = torch.arange(T, device=bd.device)[None, :]
    past = j <= i
    row = torch.where(past, i, (i + 1).clamp(max=T - 1)).expand(T, T)
    col = torch.where(past, T - 1 - (i - j), (j - i - 2).clamp(min=0))
    out = bd[..., row, col]
    return out.masked_fill((j == i + 1), 0.0)


def attention(w, pre, x, pos_emb, key_mask, n_head):
    """RelPositionMultiHeadedAttention.forward (:147-186) + forward_attention (:59-88).  x [B, T, H], key_mask [B, T] bool."""
    B, T, H = x.shape
    dk = H // n_head

    def heads(t):
        return t.view(t.shape[0], -1, n_head, dk).transpose(1, 2)
    q = heads(F.linear(x, w[pre + '.linear_q.weight'], w[pre + '.linear_q.bias']))
    k = heads(F.linear(x, w[pre + '.linear_k.weight'], w[pre + '.linear_k.bias']))
    v = heads(F.linear(x, w[pre + '.linear_v.weight'], w[pre + '.linear_v.bias']))
    p = heads(F.linear(pos_emb[None], w[pre + '.linear_pos.weight']))
    ac = torch.matmul(q + w[pre + '.pos_bias_u'][None, :, None, :], k.transpose(-2, -1))
    bd = shifted_bd(torch.matmul(q + w[pre + '.pos_bias_v'][None, :, None, :], p.transpose(-2, -1)))
    scores = (ac + bd) / math.sqrt(dk)
    dead = ~key_mask[:, None, None, :]
    attn = torch.softmax(scores.masked_fill(dead, torch.finfo(torch.float32).min), dim=-1).masked_fill(dead, 0.0)
    ctx = torch.matmul(attn, v).transpose(1, 2).reshape(B, T, H)
    return F.linear(ctx, w[pre + '.linear_out.weight'], w[pre + '.linear_out.bias'])


def _ln(w, pre, x):
    return F.layer_norm(x, (x.shape[-1],), w[pre + '.weight'], w[pre + '.bias'], 1e-5)


def _ffn(w, pre, x):
    """MultiLayeredConv1d with kernel 1 (layers.py:74-114)."""
    h = torch.relu(F.conv1d(x.transpose(1, 2), w[pre + '.w_1.weight'], w[pre + '.w_1.bias']))
    return F.conv1d(h, w[pre + '.w_2.weight'], w[pre + '.w_2.bias']).transpose(1, 2)


def _conv_module(w, pre, x, K):
    """ConvolutionModule (layers.py:7-71): pointwise -> GLU -> depthwise K -> BatchNorm -> Swish -> pointwise."""
    h = F.glu(F.conv1d(x.transpose(1, 2), w[pre + '.pointwise_conv1.weight'], w[pre + '.pointwise_conv1.bias']), dim=1)
    h = F.conv1d(h, w[pre + '.depthwise_conv.weight'], w[pre + '.depthwise_conv.bias'], padding=(K - 1) // 2, groups=h.shape[1])
    h = _bn(h, w, pre + '.norm')
    h = h * torch.sigmoid(h)
    return F.conv1d(h, w[pre + '.pointwise_conv2.weight'], w[pre + '.pointwise_conv2.bias']).transpose(1, 2)


def conformer_forward(w, pre, x, n_layers, n_head=4, K=31, last_norm=False):
    """ConformerLayers.forward (conformer.py:37-52) with EncoderLayer.forward (layers.py:181-260, macaron, normalize_before)."""
    B, T, H = x.shape
    key_mask = x.abs().sum(-1) > 0
    pos_emb = rel_positions(T, H).to(x.dtype)
    x = x * math.sqrt(H)
    for l in range(n_layers):
        e = f'{pre}.encoder_layers.{l}'
        x = x + 0.5 * _ffn(w, e + '.feed_forward_macaron', _ln(w, e + '.norm_ff_macaron', x))
        x = x + attention(w, e + '.self_attn', _ln(w, e + '.norm_mha', x), pos_emb, key_mask, n_head)
        x = x + _conv_module(w, e + '.conv_module', _ln(w, e + '.norm_conv', x), K)
        x = x + 0.5 * _ffn(w, e + '.feed_forward', _ln(w, e + '.norm_ff', x))
        x = _ln(w, e + '.norm_final', x)
    x = _ln(w, pre + '.layer_norm', x) if last_norm else F.linear(x, w[pre + '.layer_norm.weight'], w[pre + '.layer_norm.bias'])
    return x * key_mask.float()[:, :, None]


def vc_asr_h_content(w, mel, strides=(2, 1, 1), n_layers=2):
    """VCASR.forward(mel)['h_content'] (vc_modules.py:76-80)."""
    return conformer_forward(w, 'content_encoder', prenet_forward(w, mel, strides), n_layers)

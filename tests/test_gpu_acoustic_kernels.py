"""-m gpu: the kernels of the SVB acoustic model's inference forward (the PPG extractor VCASR and the MleSVBVAE glue), one at a
time, against float64 torch on the same fp32 inputs: LayerNorm over channels (svb_layer_norm_nct), relative-position attention
(svb_relpos_attention_nct), the fp32 CUDA-core convolution at the acoustic shapes (svb_conv_nct_forward), the tensor-core layer
at the acoustic shapes (svb_tc_layer_*, forward and backward), and the whole VCASR at encoder lengths on both sides of the
tensor-core gate.  Every tensor is compared in relative L2 and in L-inf relative to max |reference|; large references run on
the GPU in float64.  Test ids name the branch each case takes."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200 import _native
from neuralsvb_b200.utils import synthetic as S
from oracle import vc_asr as OV
from tests.test_gpu_disc_kernels import _conv_case, _gen, assert_within, conv_forward, errors

pytestmark = pytest.mark.gpu

f32 = ctypes.c_float

# Bars (rel L2, rel L-inf) per kernel class, about 5x the worst MEASURED over its cases on an H100 80GB HBM3 (700 W power
# limit); the worst measured value is in the comment.
TOL = {
    'ln': (5.5e-7, 9e-7),                                   # 1.1e-7 / 1.8e-7
    'ln_offset': (3e-4, 2e-4),                              # 6.2e-5 / 3.9e-5: x = 1e3 + N(0, 1), the fp32 mean near 1e3
    'att': (2.6e-6, 4.5e-6),                                # 5.2e-7 / 8.7e-7 (T 5000)
    'att_peaked': (1e-5, 6e-5),                             # 2.1e-6 / 1.2e-5: q x 30, nearly one-hot rows
    'conv': (3e-6, 7e-6),                                   # 5.8e-7 / 1.4e-6 (1024 -> 256, K 1)
    'tc_bf16x3': {'y': (3e-5, 3.6e-5), 'dx': (3e-5, 3.5e-5),  # 6.1e-6 / 7.2e-6, 6.2e-6 / 6.9e-6 (256 -> 256, K 5)
                  'dw': (1.8e-5, 2.7e-5), 'db': (6.6e-7, 8e-7)},    # 3.5e-6 / 5.5e-6, 1.3e-7 / 1.6e-7
    'tc_tf32x3': {'y': (4.5e-5, 4.7e-5), 'dx': (4.5e-5, 4.5e-5),    # 8.9e-6 / 9.5e-6, 9.0e-6 / 9.0e-6
                  'dw': (1.8e-5, 2.2e-5), 'db': (5.5e-7, 5e-7)},    # 3.5e-6 / 4.5e-6, 1.1e-7 / 9.4e-8
    'tc_tf32': {'y': (1.5e-3, 1.75e-3), 'dx': (1.5e-3, 1.7e-3),     # 2.9e-4 / 3.5e-4, 2.9e-4 / 3.4e-4
                'dw': (1.7e-5, 1.7e-5), 'db': (6e-7, 7e-7)},        # 3.5e-6 / 3.4e-6, 1.2e-7 / 1.4e-7
    'vc_asr_fp32': (5.3e-6, 8e-6),                          # 1.1e-6 / 1.6e-6
    'vc_asr_bf16x3': (4.8e-5, 6e-5),                        # 9.6e-6 / 1.2e-5
}


def _nan(*shape, like=None):
    return torch.full(shape if like is None else like.shape, float('nan'), device='cuda')


# ------------------------------------------------------------------ svb_layer_norm_nct
def layer_norm(x, gamma, beta, eps=1e-5):
    B, C, T = x.shape
    y = _nan(like=x)
    _native.check(_native.lib().svb_layer_norm_nct(_native.ptr(x), _native.ptr(gamma), _native.ptr(beta), B, C, T, f32(eps),
                                                   _native.ptr(y), None), 'layer_norm_nct')
    return y


def layer_norm_reference(x, gamma, beta, eps=1e-5):
    """nn.LayerNorm over the channel axis of [B, C, T], in float64."""
    return F.layer_norm(x.double().transpose(1, 2), (x.shape[1],), gamma.double(), beta.double(), eps).transpose(1, 2)


def _ln_params(C, key):
    g = _gen('ln-affine', C, key)
    return (0.5 + torch.rand(C, generator=g)).cuda(), (0.2 * torch.randn(C, generator=g)).cuda()


# C 100 does not split evenly over the 8 channel warps; 32 * C * 4 bytes of tile pass 48 KB for C > 384 (opt-in smem)
_LN_C = {256: 'C256', 100: 'C100_uneven_warps', 1000: 'C1000_optin_smem'}


@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('T', [1, 31, 32, 33, 77, 345, 700])
@pytest.mark.parametrize('C', list(_LN_C), ids=list(_LN_C.values()))
def test_layer_norm_matches_float64(C, T, B):
    x = torch.randn(B, C, T, generator=_gen('ln', C, T, B)).cuda()
    gamma, beta = _ln_params(C, 'rand')
    y = layer_norm(x, gamma, beta)
    assert_within(f'layer_norm C{C} T{T} B{B}', {'y': errors(y, layer_norm_reference(x, gamma, beta))}, {'y': TOL['ln']})


@pytest.mark.parametrize('C', list(_LN_C), ids=list(_LN_C.values()))
def test_layer_norm_large_common_offset(C):
    """A two-pass (centred) variance: 1e3 + N(0, 1) keeps its unit spread.  E[x^2] - E[x]^2 in fp32 would lose it."""
    B, T = 2, 45
    x = (1e3 + torch.randn(B, C, T, generator=_gen('ln-offset', C))).cuda()
    gamma, beta = _ln_params(C, 'offset')
    y = layer_norm(x, gamma, beta)
    assert_within(f'layer_norm offset 1e3 C{C}', {'y': errors(y, layer_norm_reference(x, gamma, beta))}, {'y': TOL['ln_offset']})


@pytest.mark.parametrize('C', list(_LN_C), ids=list(_LN_C.values()))
def test_layer_norm_zero_variance_columns_give_beta_exactly(C):
    """A padded (all-zero) frame and a constant frame have zero variance: (x - mean) is exactly 0, so y is exactly beta.
    The constant is dyadic so that its fp32 channel sum, and so the mean, is exact."""
    B, T = 2, 33
    x = torch.randn(B, C, T, generator=_gen('ln-zero', C)).cuda()
    x[1, :, T - 4:] = 0.0                 # the all-zero tail of a shorter clip
    x[0, :, 5] = -1.5
    gamma, beta = _ln_params(C, 'zero')
    y = layer_norm(x, gamma, beta)
    for b, t in [(1, T - 4), (1, T - 1), (0, 5)]:
        assert torch.equal(y[b, :, t], beta), (b, t, float((y[b, :, t] - beta).abs().max()))
    assert_within(f'layer_norm zero-variance C{C}', {'y': errors(y, layer_norm_reference(x, gamma, beta))}, {'y': TOL['ln']})


# ------------------------------------------------------------------ svb_relpos_attention_nct
def attention(q, k, v, p, u, bv, mask, n_head):
    B, C, T = q.shape
    out = torch.full_like(q, float('nan'))                     # on q's device, which need not be the current one
    with torch.cuda.device(q.device):
        _native.check(_native.lib().svb_relpos_attention_nct(
            _native.ptr(q), _native.ptr(k), _native.ptr(v), _native.ptr(p), _native.ptr(u), _native.ptr(bv), _native.ptr(mask),
            B, C, T, n_head, _native.ptr(out), _native.current_stream_ptr(q.device)), 'relpos_attention_nct')
    return out


def attention_reference(q, k, v, p, u, bv, mask, n_head):
    """float64 RelPositionMultiHeadedAttention core on [B, C, T] inputs, before linear_out: q, k, v [B, C, T], p = linear_pos(pos_emb)
    [C, T], u / bv the [n_head, dk] position biases, mask [B, T] (> 0: a valid key) or None.
    scores = ((q + u) k^T + rel_shift((q + bv) p^T)) / sqrt(dk), masked keys at finfo(float32).min before the softmax and 0 after."""
    B, C, T = q.shape
    dk = C // n_head

    def heads(t):                                             # [B, C, T] -> [B, h, T, dk]
        return t.double().reshape(t.shape[0], n_head, dk, T).transpose(2, 3)
    qh, kh, vh, ph = heads(q), heads(k), heads(v), heads(p[None])
    ac = (qh + u.double()[None, :, None, :]) @ kh.transpose(-2, -1)
    bd = OV.shifted_bd((qh + bv.double()[None, :, None, :]) @ ph.transpose(-2, -1))
    scores = (ac + bd) / math.sqrt(dk)
    if mask is None:
        attn = torch.softmax(scores, -1)
    else:
        dead = ~(mask > 0)[:, None, None, :]
        attn = torch.softmax(scores.masked_fill(dead, torch.finfo(torch.float32).min), -1).masked_fill(dead, 0.0)
    return (attn @ vh).transpose(2, 3).reshape(B, C, T)


def ragged_lengths(B, T):
    """clip b is T - b * max(1, T // 7) frames long (at least 1): T 45 gives 45 / 39, the former single-shape test."""
    return [max(1, T - b * max(1, T // 7)) for b in range(B)]


def attention_case(B, C, n_head, T, mask_kind, q_scale=1.0, key=()):
    g = _gen('att', B, C, n_head, T, mask_kind, q_scale, key)
    q, k, v = (torch.randn(B, C, T, generator=g) for _ in range(3))
    q = q * q_scale
    p = torch.randn(C, T, generator=g)
    u, bv = (0.3 * torch.randn(n_head, C // n_head, generator=g) for _ in range(2))
    mask = None
    if mask_kind == 'ragged':
        mask = torch.zeros(B, T)
        for b, n in enumerate(ragged_lengths(B, T)):
            mask[b, :n] = 1.0
    elif mask_kind == 'dead_clip':                            # clip 1 fully masked, clip 2 (if any) ragged
        mask = torch.ones(B, T)
        mask[1] = 0.0
        if B > 2:
            mask[2, ragged_lengths(3, T)[2]:] = 0.0
    return tuple(t.cuda() for t in (q, k, v, p, u, bv)) + (None if mask is None else mask.cuda(),)


def _att_tag(C, n_head, T, mask_kind, q_scale):
    dk = C // n_head
    tags = [f'C{C}_dk{dk}', f'T{T}', mask_kind]
    if T <= 2:
        tags.append('relshift_edges')
    if T % 8:
        tags.append(f'{8 - T % 8}idle_warps')
    if 8 * (3 * dk + T) * 4 > 48 * 1024:
        tags.append('optin_smem')
    if dk % 32:
        tags.append('dk_not_lane_multiple')
    if q_scale != 1.0:
        tags.append(f'peaked_q{q_scale:g}')
    return '_'.join(tags)


# (B, C, n_head, T, mask kind, q scale)
ATT_CASES = ([(2, 256, 4, T, 'ragged', 1.0) for T in (1, 2, 7, 8, 9, 31, 33, 45, 345, 700, 1345, 2600)] +
             [(1, 256, 4, T, 'none', 1.0) for T in (1, 2, 9, 345, 1345, 5000)] +
             [(2, 192, 4, T, 'ragged', 1.0) for T in (1, 2, 8, 33, 700, 1345, 2600)] +
             [(3, 256, 4, T, 'dead_clip', 1.0) for T in (2, 33, 1345)] +
             [(2, 256, 4, T, 'ragged', 30.0) for T in (9, 345, 1345)] +
             [(2, 192, 4, 700, 'ragged', 30.0)])


@pytest.mark.parametrize('case', ATT_CASES, ids=lambda c: _att_tag(*c[1:]))
def test_relpos_attention_matches_float64(case):
    """Every query row is compared, padded ones included: the conformer's k = 31 depthwise conv mixes them into valid rows."""
    B, C, n_head, T, mask_kind, q_scale = case
    q, k, v, p, u, bv, mask = attention_case(B, C, n_head, T, mask_kind, q_scale)
    out = attention(q, k, v, p, u, bv, mask, n_head)
    ref = attention_reference(q, k, v, p, u, bv, mask, n_head)
    if mask_kind == 'dead_clip':                             # a clip without a valid key attends to nothing
        assert torch.equal(out[1], torch.zeros_like(out[1]))
    assert_within(_att_tag(C, n_head, T, mask_kind, q_scale), {'out': errors(out, ref)},
                  {'out': TOL['att_peaked' if q_scale != 1.0 else 'att']})


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason=f'needs 2 CUDA devices, saw {torch.cuda.device_count()}')
def test_relpos_attention_optin_smem_on_a_second_device():
    """The opt-in shared-memory limit is a per-device function attribute: after cuda:0 raised it, cuda:1 must raise it too."""
    B, C, n_head, T = 2, 256, 4, 1345
    q, k, v, p, u, bv, mask = attention_case(B, C, n_head, T, 'ragged', key='dev')
    for dev in ('cuda:0', 'cuda:1'):
        args = [t.to(dev) for t in (q, k, v, p, u, bv, mask)]
        out = attention(*args, n_head)
        ref = attention_reference(*args, n_head)
        assert_within(f'attention T{T} on {dev}', {'out': errors(out, ref)}, {'out': TOL['att']})


# ------------------------------------------------------------------ svb_conv_nct_forward at the acoustic shapes (fp32 CUDA cores)
# (tag, B, Cin, Cout, Tin, W, K, stride, dil, pad, groups, slope) as in test_gpu_disc_kernels.CONV_SHAPES
def _lin(tag, cin, cout, T, slope, B=2):
    return (f'{tag}_{cin}to{cout}_T{T}_gconv16', B, cin, cout, T, 1, 1, 1, 1, 0, 1, slope)


ACOUSTIC_CONV_SHAPES = (
    [(f'prenet0_80to256_k5s2_relu_T{T}_gconv16', B, 80, 256, T, 1, 5, 2, 1, 2, 1, 0.0) for B, T in [(2, 63), (2, 64), (1, 1), (3, 1401)]] +
    [(f'depthwise_256g_k31_T{T}_gconv2_7of8lanes_masked', 2, 256, 256, T, 1, 31, 1, 1, 15, 256, 1.0) for T in (1, 7, 30, 345)] +
    [_lin('ffn_w1_relu', 256, 1024, T, 0.0) for T in (1, 5, 31)] +
    [_lin('ffn_w2', 1024, 256, T, 1.0) for T in (1, 5, 31)] +
    [_lin('qkv', 256, 768, T, 1.0) for T in (1, 5, 31)] +
    [_lin('768to256', 768, 256, T, 1.0) for T in (1, 5, 31)] +
    [_lin('pointwise_conv1', 256, 512, 31, 1.0), _lin('linear_out', 256, 256, 31, 1.0)] +
    [_lin('latent_map', 128, 128, 1, 1.0, B=3), _lin('latent_map_relu', 256, 128, 1, 0.0, B=3)])


@pytest.mark.parametrize('shape', ACOUSTIC_CONV_SHAPES, ids=lambda s: s[0])
def test_conv_nct_forward_at_acoustic_shapes_matches_float64(shape):
    _, B, Cin, Cout, Tin, W, K, s, dil, pad, grp, slope = shape
    x, w, b, _, Tout = _conv_case(shape)
    y = conv_forward(x, w, b, shape, Tout)[..., 0]
    z = F.conv1d(x[..., 0].double(), w.double(), b.double(), stride=s, padding=pad, dilation=dil, groups=grp)
    assert_within(shape[0], {'y': errors(y, F.leaky_relu(z, slope))}, {'y': TOL['conv']})


# ------------------------------------------------------------------ svb_tc_layer_* at the acoustic shapes
# (cin, cout, K) of the dense layers the acoustic model runs on wgmma once T >= 32
TC_SHAPES = [(256, 768, 1), (256, 1024, 1), (1024, 256, 1), (256, 512, 1), (768, 256, 1), (256, 256, 1), (256, 256, 5)]
_TB = [(1, 32), (2, 33), (3, 127), (1, 128), (2, 129), (3, 345), (1, 700)]
TC_CASES = [(cin, cout, K, slope) + _TB[(2 * n + r * 3) % len(_TB)]
            for n, (cin, cout, K, slope) in enumerate((c + (sl,)) for c in TC_SHAPES for sl in (1.0, 0.0)) for r in (0, 1)]


def _tc_tag(cin, cout, K, slope, B, T, prec='bf16x3'):
    return f'{cin}to{cout}_K{K}_{"linear" if slope == 1.0 else "relu"}_B{B}_T{T}_{prec}'


def tc_layer_forward_backward(cin, cout, K, slope, B, T, prec='bf16x3'):
    from neuralsvb_b200.modules.hifigan import discriminators as D
    g = _gen('tc', cin, cout, K, slope, B, T, prec)
    x = torch.randn(B, cin, T, generator=g)
    w = torch.randn(cout, cin, K, generator=g) / math.sqrt(cin * K)
    b = 0.1 * torch.randn(cout, generator=g)
    dy = torch.randn(B, cout, T, generator=g).cuda()
    pad = (K - 1) // 2
    assert D.tc_eligible(cin, cout, K, 1, 1, pad, 1)
    old = D.TC_PRECISION
    D.TC_PRECISION = prec
    try:
        xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
        y = D.conv_tc(xc, wc, bc, D.TcLayer(), K, 1, pad, slope, 1)
        y.backward(dy)
    finally:
        D.TC_PRECISION = old
    xr, wr, br = (t.double().cuda().requires_grad_(True) for t in (x, w, b))
    z = F.conv1d(xr, wr, br, padding=pad)
    # ReLU's derivative jumps at 0: the reference takes the mask of the CUDA output (as test_dense_tc_layers_match_torch does)
    mask = torch.where(y.detach() > 0, 1.0, slope).double()
    flips = int((mask != torch.where(z.detach() > 0, 1.0, slope)).sum())
    assert flips <= 1e-4 * mask.numel(), flips
    z.backward(dy.double() * mask)
    ref = z.detach() if slope == 1.0 else torch.relu(z.detach())
    return {'y': errors(y.detach(), ref), 'dx': errors(xc.grad, xr.grad), 'dw': errors(wc.grad, wr.grad), 'db': errors(bc.grad, br.grad)}


@pytest.mark.parametrize('case', TC_CASES, ids=lambda c: _tc_tag(*c))
def test_tc_layer_at_acoustic_shapes_matches_float64(case):
    assert_within(_tc_tag(*case), tc_layer_forward_backward(*case), TOL['tc_bf16x3'])


@pytest.mark.parametrize('prec', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('case', [(256, 1024, 1, 0.0, 2, 129), (256, 256, 5, 1.0, 1, 345)], ids=lambda c: _tc_tag(*c)[:-7])
def test_tc_layer_other_precisions_match_float64(case, prec):
    assert_within(_tc_tag(*case, prec), tc_layer_forward_backward(*case, prec), TOL[f'tc_{prec}'])


@pytest.mark.parametrize('T', [31, 32, 345])
def test_linear_pos_with_lazy_zero_bias_matches_float64(T):
    """linear_pos (bias=False) at B = 1 through vc_modules._conv: the zero bias is created on first use; T < 32 takes the
    fp32 kernel, T >= 32 the tensor-core layer."""
    from neuralsvb_b200.modules.voice_conversion import vc_modules as V
    H = 256
    g = _gen('linear_pos', T)
    w = (torch.randn(H, H, generator=g) / math.sqrt(H)).cuda()
    p_emb = V.rel_positions(T, H, 'cuda')
    with torch.no_grad():
        y = V._conv(p_emb[None], w, None)
    assert torch.equal(w._svb_zero_bias, torch.zeros(H, device='cuda'))
    ref = F.linear(p_emb.double().t(), w.double()).t()[None]
    assert_within(f'linear_pos T{T}', {'y': errors(y, ref)}, {'y': TOL['conv'] if T < 32 else TOL['tc_bf16x3']['y']})


def test_tc_layer_backward_without_y_at_slope_1_matches_the_call_with_y():
    """The ABI lets a linear layer (out_slope 1) pass y = NULL to the backward: no activation mask is needed.  dx is bit for bit
    the same.  The weight gradient adds its split-K partials with atomics, so dw / db differ in the last bits between any two
    calls; they are held to 1e-6."""
    from neuralsvb_b200.modules.hifigan import discriminators as D
    cin, cout, K, B, T = 256, 256, 5, 2, 129
    g = _gen('tc-null-y')
    x = torch.randn(B, cin, T, generator=g).cuda()
    w = (torch.randn(cout, cin, K, generator=g) / math.sqrt(cin * K)).cuda()
    b = (0.1 * torch.randn(cout, generator=g)).cuda()
    dy = torch.randn(B, cout, T, generator=g).cuda()
    layer = D.TcLayer()
    with torch.no_grad():
        y = D.conv_tc(x, w, b, layer, K, 1, 2, 1.0, 1)
    lib, st = _native.lib(), _native.current_stream_ptr()
    outs = []
    for y_arg in (y, None):
        dx, dw, db = _nan(like=x), torch.zeros_like(w), torch.zeros_like(b)
        _native.check(lib.svb_tc_layer_backward(layer.h, _native.ptr(x), _native.ptr(y_arg), _native.ptr(dy), B, T, 1, f32(1.0),
                                                _native.ptr(dx), _native.ptr(dw), _native.ptr(db), st), 'tc_layer_backward')
        outs.append((dx, dw, db))
    (dx_y, dw_y, db_y), (dx_n, dw_n, db_n) = outs
    assert torch.isfinite(dx_n).all() and torch.equal(dx_n, dx_y)
    e = {'dw': errors(dw_n, dw_y.double()), 'db': errors(db_n, db_y.double())}
    assert_within('tc_layer_backward y = NULL vs y', e, {'dw': (1e-6, 1e-6), 'db': (1e-6, 1e-6)})


# ------------------------------------------------------------------ the whole PPG extractor
@pytest.mark.parametrize('use_tc', [True, False], ids=['bf16x3', 'fp32'])
@pytest.mark.parametrize('T_enc,B', [(31, 2), (32, 2), (33, 3), (345, 2), (700, 2)], ids=lambda v: str(v))
def test_vc_asr_h_content_matches_float64_oracle(T_enc, B, use_tc):
    """VCASR(mel)['h_content'] against oracle.vc_asr in float64, at encoder lengths T' on both sides of the tensor-core gate
    (T' >= 32: the batch's padded length decides).  Clip b ends 9 b mel frames early (an all-zero tail)."""
    from neuralsvb_b200.modules.voice_conversion import vc_modules as V
    from tests.test_gpu_vc_asr import _model
    mel = S.make_vc_asr_mel(B, 2 * T_enc, 1234 + T_enc)
    old = V.USE_TC
    V.USE_TC = use_tc
    try:
        with torch.no_grad():
            h = _model()(mel.cuda())['h_content']
    finally:
        V.USE_TC = old
    w = {k: v.double() for k, v in S.make_vc_asr_state_dict(1234).items()}
    with torch.no_grad():
        ref = OV.vc_asr_h_content(w, mel.double())
    h = h.cpu()
    assert h.shape == ref.shape
    assert torch.equal(h[ref == 0], torch.zeros_like(h[ref == 0]))     # padded frames stay exactly zero
    assert_within(f'vc_asr T\'{T_enc} B{B} {"bf16x3" if use_tc else "fp32"}', {'h': errors(h, ref)},
                  {'h': TOL['vc_asr_bf16x3' if use_tc else 'vc_asr_fp32']})

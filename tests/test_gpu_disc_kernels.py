"""-m gpu: the fp32 CUDA-core kernels of the discriminator step, one kernel at a time, against float64 torch on the same
fp32 inputs: the general strided / dilated / grouped convolution (svb_conv_nct_forward, and svb_conv_nct_backward with its
leaky-relu mask, data, weight and bias gradients), AvgPool1d(4,2,1) and the right reflect pad with their adjoints, the
cond_net ConvTranspose1d pair, the loss reductions and element-wise loss gradients, the weight-norm backward and the
spectral-norm sigma.  Every tensor is compared in relative L2 and in L-inf relative to max |reference|; references are
computed on the GPU in float64 at test time."""
import ctypes
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200 import _native
from neuralsvb_b200.utils.synthetic import MPD_PERIODS, MSD_LAYERS

pytestmark = pytest.mark.gpu

f32 = ctypes.c_float


def errors(got, ref):
    d = got.double() - ref
    return float(d.norm() / ref.norm()), float(d.abs().max() / ref.abs().max())


def assert_within(what, e, tol):
    """e, tol: {tensor: (rel L2, rel L-inf)}.  Written as `not <=` so that a NaN error fails."""
    print('MEASURED', what, {k: f'{a:.2e}/{b:.2e}' for k, (a, b) in e.items()})
    bad = {k: v for k, v in e.items() if not (v[0] <= tol[k][0] and v[1] <= tol[k][1])}
    assert not bad, f'{what}: (rel L2, rel L-inf) {bad}, bars {tol}'


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


# ------------------------------------------------------------------ svb_conv_nct_forward / svb_conv_nct_backward
# (tag, B, Cin, Cout, Tin, W, K, stride, dil, pad, groups, slope); the tag names the branch each shape takes:
#   gconv<COQ> forward (COQ = 2/4/8/16 for cout_g <= 8/16/32/more) or conv_fewout<Cout> (stride 1, Cin >= 64, Cout <= 2),
#   dgrad<STRIDE, CIQ> (CIQ by cin_g <= 8/16/32/more; 'shared' taps when 256/CIQ is a multiple of the stride and dil == 1),
#   wgrad<K, kWC> (kWC by cout_g <= 16/32/more).
def _mpd0(cin, W):
    return (f'mpd0_c{cin}_W{W}_gconv8_dgrad3x2generic_wgrad5x32', 2, cin, 32, -(-8192 // W), W, 5, 3, 1, 2, 1, 0.1)


PRODUCT = [_mpd0(cin, W) for cin in (1, 2) for W in MPD_PERIODS] + [
    ('post_W1_fewout1_dgrad1x16shared_wgrad3x16', 2, 1024, 1, 256, 1, 3, 1, 1, 1, 1, 1.0),
    ('post_W11_fewout1_dgrad1x16shared_wgrad3x16', 2, 1024, 1, 10, 11, 3, 1, 1, 1, 1, 1.0),
    ('msd0_gconv16_dgrad1x2shared_wgrad15x64_2coltiles', 2, 1, 128, 8192, 1, 15, 1, 1, 7, 1, 0.1),
]
# the USE_TC = False fallback of the dense / grouped layers (they run on wgmma in the product)
_MSD_T = {1: 8192, 2: 4096, 3: 2048, 4: 512, 5: 128}
_CIQ = lambda c: 2 if c <= 8 else 4 if c <= 16 else 8 if c <= 32 else 16
_KWC = lambda c: 16 if c <= 16 else 32 if c <= 32 else 64
FALLBACK = [(f'msd{i}_g{g}_s{s}_dgrad{s}x{_CIQ(ci // g)}_wgrad41x{_KWC(co // g)}', 1, ci, co, _MSD_T[i], 1, k, s, 1, p, g, 0.1)
            for i, (ci, co, k, s, g, p) in enumerate(MSD_LAYERS) if 1 <= i <= 5] + [
    ('mpd2_dense_s3_W3_gconv16_dgrad3x16generic_wgrad5x64', 1, 128, 512, 304, 3, 5, 3, 1, 2, 1, 0.1),
    ('mpd4_1024x1024_s1_W2_dgrad1x16shared_wgrad5x64_wraps', 1, 1024, 1024, 51, 2, 5, 1, 1, 2, 1, 0.1),
]
OFF_PRODUCT = [
    ('dil2_dgrad1x4generic_wgrad5x16', 2, 16, 16, 300, 1, 5, 1, 2, 4, 1, 0.1),
    ('K1_W2_wgrad1x64_partial_tile', 2, 24, 40, 200, 2, 1, 1, 1, 0, 1, 0.1),
    ('K7_s2_dgrad2x4shared_wgrad7x32', 2, 12, 20, 150, 1, 7, 2, 1, 3, 1, 0.1),
    ('cout2_fewout2_W3', 2, 64, 2, 100, 3, 3, 1, 1, 1, 1, 0.1),
    ('tout1_s3_W2', 2, 4, 8, 3, 2, 5, 3, 1, 2, 1, 0.1),
    ('tin_lt_K7', 2, 8, 8, 3, 1, 7, 1, 1, 3, 1, 0.1),
    ('tin_lt_K15_msd0', 1, 1, 128, 5, 1, 15, 1, 1, 7, 1, 0.1),
    ('T209_not_dgrad_tile_multiple_dgrad1x8', 2, 32, 32, 209, 1, 3, 1, 1, 1, 1, 0.1),
    ('T1000_s4_g2_dgrad4x8shared', 2, 48, 24, 1000, 1, 5, 4, 1, 2, 2, 0.1),
    ('wgrad_grid_stride_wraps_c64_T8192', 2, 64, 64, 8192, 1, 3, 1, 1, 1, 1, 0.1),
]
CONV_SHAPES = PRODUCT + FALLBACK + OFF_PRODUCT

# Bars per tensor (rel L2, rel L-inf), about 5x the worst error measured over CONV_SHAPES (both tests below) on an H100 80GB
# HBM3 (400 W power limit):
#   y  1.3e-6 / 3.3e-6   dx 1.3e-6 / 2.8e-6   (both at 1024 -> 1024 k5: 5120-term sums)
#   dw 3.2e-7 / 4.7e-7   db 1.6e-7 / 1.8e-7
CONV_TOL = {'y': (6.5e-6, 1.7e-5), 'dx': (6.5e-6, 1.4e-5), 'dw': (1.6e-6, 2.4e-6), 'db': (8e-7, 1e-6)}


def _conv_case(shape):
    tag, B, Cin, Cout, Tin, W, K, s, dil, pad, grp, slope = shape
    g = _gen('conv', tag)
    x = torch.randn(B, Cin, Tin, W, generator=g).cuda()
    w = (torch.randn(Cout, Cin // grp, K, generator=g) / np.sqrt(Cin // grp * K)).cuda()
    b = (0.1 * torch.randn(Cout, generator=g)).cuda()
    Tout = (Tin + 2 * pad - dil * (K - 1) - 1) // s + 1
    dy = torch.randn(B, Cout, Tout, W, generator=g).cuda()
    return x, w, b, dy, Tout


def conv_forward(x, w, b, shape, Tout):
    _, B, Cin, Cout, Tin, W, K, s, dil, pad, grp, slope = shape
    y = torch.full((B, Cout, Tout, W), float('nan'), device='cuda')
    _native.check(_native.lib().svb_conv_nct_forward(_native.ptr(x), _native.ptr(w), _native.ptr(b), _native.ptr(y), B, Cin, Cout,
                                                     Tin, W, K, s, dil, pad, grp, f32(slope), None), 'conv_nct_forward')
    return y


def conv_backward(x, w, y, dy, shape, dw=None, db=None):
    _, B, Cin, Cout, Tin, W, K, s, dil, pad, grp, slope = shape
    dz = torch.full_like(dy, float('nan'))
    dx = torch.full_like(x, float('nan'))             # written in full, never read
    dw = torch.zeros_like(w) if dw is None else dw
    db = torch.zeros(Cout, device='cuda') if db is None else db
    _native.check(_native.lib().svb_conv_nct_backward(_native.ptr(x), _native.ptr(w), _native.ptr(y), _native.ptr(dy), B, Cin, Cout,
                                                      Tin, W, K, s, dil, pad, grp, f32(slope), _native.ptr(dz), _native.ptr(dx),
                                                      _native.ptr(dw), _native.ptr(db), None), 'conv_nct_backward')
    return dx, dw, db


def conv_reference(x, w, b, dy, y, shape):
    """float64: y_ref = lrelu(conv(x) + b) and the gradients of the LINEAR conv for dz = dy * where(y > 0, 1, slope), the mask
    taken from the kernel's own forward output so that a pre-activation within rounding of 0 cannot flip it."""
    _, B, Cin, Cout, Tin, W, K, s, dil, pad, grp, slope = shape
    xd, wd, bd = (t.double().requires_grad_(True) for t in (x, w, b))
    z = F.conv2d(xd, wd[..., None], bd, stride=(s, 1), padding=(pad, 0), dilation=(dil, 1), groups=grp)
    dz = dy.double() * torch.where(y > 0, 1.0, slope).double()
    z.backward(dz)
    return F.leaky_relu(z.detach(), slope), xd.grad, wd.grad, bd.grad


@pytest.mark.parametrize('shape', CONV_SHAPES, ids=lambda s: s[0])
def test_conv_nct_forward_and_backward_match_float64_torch(shape):
    x, w, b, dy, Tout = _conv_case(shape)
    y = conv_forward(x, w, b, shape, Tout)
    dx, dw, db = conv_backward(x, w, y, dy, shape)
    y_r, dx_r, dw_r, db_r = conv_reference(x, w, b, dy, y, shape)
    e = {'y': errors(y, y_r), 'dx': errors(dx, dx_r), 'dw': errors(dw, dw_r), 'db': errors(db, db_r)}
    assert_within(shape[0], e, CONV_TOL)


@pytest.mark.parametrize('shape', [PRODUCT[0], PRODUCT[10], FALLBACK[1], OFF_PRODUCT[-1]], ids=lambda s: s[0])
def test_conv_nct_backward_accumulates_into_nonzero_weight_and_bias_gradients(shape):
    """dw / db are ACCUMULATED (the caller zeroes them): started from random buffers they end at start + gradient."""
    x, w, b, dy, Tout = _conv_case(shape)
    y = conv_forward(x, w, b, shape, Tout)
    g = _gen('acc', shape[0])
    dw0, db0 = torch.randn(w.shape, generator=g).cuda() * 1e-2, torch.randn(b.shape, generator=g).cuda() * 1e-2
    _, dw, db = conv_backward(x, w, y, dy, shape, dw=dw0.clone(), db=db0.clone())
    _, _, dw_r, db_r = conv_reference(x, w, b, dy, y, shape)
    e = {'dw': errors(dw, dw0.double() + dw_r), 'db': errors(db, db0.double() + db_r)}
    assert_within(shape[0], e, CONV_TOL)


# ------------------------------------------------------------------ AvgPool1d(4, 2, 1) and the right reflect pad
# measured worst (H100 80GB HBM3, 400 W): avgpool y 4.1e-8 / 8.1e-8, dx 2.8e-8 / 4.5e-8; pad dx 3.1e-8 / 4.6e-8 (y: exact copy)
ROW_TOL = {'y': (2.5e-7, 4e-7), 'dx': (1.5e-7, 2.5e-7)}


def _row_call(fn, x, y, *args):
    _native.check(getattr(_native.lib(), fn)(_native.ptr(x), _native.ptr(y), *args, None), fn)
    return y


@pytest.mark.parametrize('Tin', [2, 3, 4, 5, 8191, 8192])
def test_avgpool_4_2_1_forward_and_backward_match_float64_torch(Tin):
    g = _gen('pool', Tin)
    rows = 6
    x = torch.randn(rows, Tin, generator=g).cuda()
    Tout = (Tin + 2 - 4) // 2 + 1
    dy = torch.randn(rows, Tout, generator=g).cuda()
    y = _row_call('svb_avgpool1d_4_2_1', x, torch.full((rows, Tout), float('nan'), device='cuda'), rows, Tin)
    dx = _row_call('svb_avgpool1d_4_2_1_backward', dy, torch.full_like(x, float('nan')), rows, Tin)
    xd = x.double().requires_grad_(True)
    y_r = F.avg_pool1d(xd[:, None], 4, 2, 1)[:, 0]
    y_r.backward(dy.double())
    assert_within(f'avgpool Tin {Tin}', {'y': errors(y, y_r.detach()), 'dx': errors(dx, xd.grad)}, ROW_TOL)


def _pad_cases():
    cases = []
    for p in MPD_PERIODS:
        for T in (3, 5, 7, 9, 13, 8191, 8193):
            if T % p and p - T % p < T:
                cases.append((p, T, T + p - T % p))
    return cases + [(0, T, 2 * T - 1) for T in (2, 3, 7, 8191)]      # the extreme Tpad - T = T - 1


@pytest.mark.parametrize('period,T,Tpad', _pad_cases(), ids=lambda v: str(v))
def test_pad_reflect_right_forward_and_backward_match_float64_torch(period, T, Tpad):
    g = _gen('pad', T, Tpad)
    rows = 4
    x = torch.randn(rows, T, generator=g).cuda()
    dy = torch.randn(rows, Tpad, generator=g).cuda()
    y = _row_call('svb_pad_reflect_right', x, torch.full((rows, Tpad), float('nan'), device='cuda'), rows, T, Tpad)
    dx = _row_call('svb_pad_reflect_right_backward', dy, torch.full_like(x, float('nan')), rows, T, Tpad)
    xd = x.double().requires_grad_(True)
    y_r = F.pad(xd[:, None], (0, Tpad - T), 'reflect')[:, 0]
    y_r.backward(dy.double())
    assert torch.equal(y.double(), y_r.detach())                   # a copy: exact
    assert_within(f'pad p{period} T{T} Tpad{Tpad}', {'y': errors(y, y_r.detach()), 'dx': errors(dx, xd.grad)}, ROW_TOL)


# ------------------------------------------------------------------ cond_net: ConvTranspose1d(80, 1, 2t, stride t, padding t // 2)
# measured worst (H100 80GB HBM3, 400 W): y 2.3e-7 / 5.7e-7, dw 1.7e-7 / 4.0e-7, db 1.1e-6 (a scalar: the sum of B * Tout
# random cotangents, relative to its own small value)
COND_TOL = {'y': (1.2e-6, 3e-6), 'dw': (9e-7, 2e-6), 'db': (6e-6, 6e-6)}


def cond_net_reference(mel, w, b, t):
    return F.conv_transpose1d(mel, w, b, stride=t, padding=t // 2)


@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('T', [1, 7, 32])
@pytest.mark.parametrize('t', [256, 128])
def test_cond_net_forward_and_backward_match_float64_torch(t, T, B):
    lib = _native.lib()
    g = _gen('cond', t, T, B)
    C, K, pad = 80, 2 * t, t // 2
    mel = torch.randn(B, C, T, generator=g).cuda()
    w = (torch.randn(C, 1, K, generator=g) / np.sqrt(C * 2.0)).cuda()
    b = (0.1 * torch.randn(1, generator=g)).cuda()
    Tout = (T - 1) * t - 2 * pad + K
    dy = torch.randn(B, 1, Tout, generator=g).cuda()
    y = torch.full((B, 1, Tout), float('nan'), device='cuda')
    _native.check(lib.svb_cond_net_forward(_native.ptr(mel), _native.ptr(w), _native.ptr(b), B, C, T, K, t, pad, _native.ptr(y), None),
                  'cond_net_forward')
    dw, db = torch.zeros_like(w), torch.zeros_like(b)
    _native.check(lib.svb_cond_net_backward(_native.ptr(mel), _native.ptr(dy), B, C, T, K, t, pad, _native.ptr(dw), _native.ptr(db),
                                            None), 'cond_net_backward')
    wd, bd = w.double().requires_grad_(True), b.double().requires_grad_(True)
    y_r = cond_net_reference(mel.double(), wd, bd, t)
    y_r.backward(dy.double())
    e = {'y': errors(y, y_r.detach()), 'dw': errors(dw, wd.grad), 'db': errors(db, bd.grad)}
    assert_within(f'cond_net t{t} T{T} B{B}', e, COND_TOL)


# ------------------------------------------------------------------ svb_pair_stats / svb_loss_grad(_dev)
N_LOSS = 2 * 132 * 8 * 256 + 77          # not a multiple of 256, more than one pass of the 132*8-block grid-stride loop


def _positive_pair(n, key):
    """a, b > 0 (the log-magnitude terms), every 17th pair an exact tie, the others at least 1e-3 apart in relative terms."""
    g = _gen('pair', key)
    a = torch.exp(torch.randn(n, generator=g))
    r = 1e-3 + torch.rand(n, generator=g)
    b = a * torch.where(torch.rand(n, generator=g) < 0.5, 1 + r, 1 / (1 + r))
    b[::17] = a[::17]
    return a.float().cuda(), b.float().cuda()


PAIR_TOL = 1.5e-8        # relative, per sum; measured worst 2.6e-9 (the fp32 logs), H100 80GB HBM3, 400 W


@pytest.mark.parametrize('with_b,want_log', [(True, True), (True, False), (False, True)])
def test_pair_stats_match_float64_sums(with_b, want_log):
    a, b = _positive_pair(N_LOSS, 'stats')
    if not want_log:
        a = a - 0.7                               # signed values (the log sum needs positive ones)
    out = torch.full((6,), float('nan'), dtype=torch.float64, device='cuda')
    _native.check(_native.lib().svb_pair_stats(_native.ptr(a), _native.ptr(b if with_b else None), N_LOSS, int(want_log),
                                               ctypes.c_void_p(out.data_ptr()), None), 'pair_stats')
    A = a.double().cpu().numpy()
    Bv = b.double().cpu().numpy() if with_b else np.zeros_like(A)
    ref = [((A - Bv) ** 2).sum(), (A ** 2).sum(),
           np.abs(np.log(A) - np.log(Bv)).sum() if (want_log and with_b) else 0.0,
           np.abs(A - Bv).sum(), ((1 - A) ** 2).sum(), (Bv ** 2).sum()]
    got = out.cpu().numpy()
    rel = [abs(gv - rv) / abs(rv) if rv else abs(gv) for gv, rv in zip(got, ref)]
    print('MEASURED pair_stats', with_b, want_log, [f'{r:.2e}' for r in rel])
    assert all(r <= PAIR_TOL for r in rel), (rel, got, ref)
    for i, rv in enumerate(ref):
        if rv == 0:
            assert got[i] == 0, (i, got)


def loss_expr(kind, a, b, scale):
    """The torch expression whose gradient w.r.t. a kind replaces (losses are scale * expression)."""
    if kind == 0:
        return scale * (a - b).abs().sum()                          # F.l1_loss
    if kind == 1:
        return scale * 0.5 * ((1 - a) ** 2).sum()                   # generator_loss / discriminator_loss (real)
    if kind == 2:
        return scale * 0.5 * (a ** 2).sum()                         # discriminator_loss (generated)
    if kind == 3:
        return scale * 0.5 * ((a - b) ** 2).sum()                   # spectral convergence numerator
    return scale * (torch.log(a) - torch.log(b)).abs().sum()       # log-magnitude L1


LOSS_GRAD_TOL = (3e-7, 5e-7)     # measured worst 5.8e-8 / 9.2e-8 (H100 80GB HBM3, 400 W)


@pytest.mark.parametrize('device_scale', [False, True])
@pytest.mark.parametrize('accumulate', [0, 1])
@pytest.mark.parametrize('kind', [0, 1, 2, 3, 4])
def test_loss_grad_matches_float64_autograd(kind, accumulate, device_scale):
    lib = _native.lib()
    a, b = _positive_pair(N_LOSS, ('grad', kind))
    use_b = kind in (0, 3, 4)
    scale, dev = 0.37, torch.tensor([1.75], device='cuda')
    da0 = torch.randn(N_LOSS, generator=_gen('da0', kind)).cuda()
    da = da0.clone() if accumulate else torch.full_like(a, float('nan'))
    bp = _native.ptr(b) if use_b else None
    if device_scale:
        rc = lib.svb_loss_grad_dev(_native.ptr(a), bp, kind, f32(scale), _native.ptr(dev), _native.ptr(da), N_LOSS, accumulate, None)
    else:
        rc = lib.svb_loss_grad(_native.ptr(a), bp, kind, f32(scale), _native.ptr(da), N_LOSS, accumulate, None)
    _native.check(rc, 'loss_grad')
    s = float(np.float32(scale)) * (float(dev) if device_scale else 1.0)
    ad = a.double().requires_grad_(True)
    loss_expr(kind, ad, b.double(), s).backward()
    ref = ad.grad + (da0.double() if accumulate else 0)
    e = {'da': errors(da, ref)}
    assert_within(f'loss_grad kind {kind} acc {accumulate} dev {device_scale}', e, {'da': LOSS_GRAD_TOL})
    if kind in (0, 4):                                              # exact ties: the gradient is exactly 0
        tie = (a == b)
        assert int(tie.sum()) == len(range(0, N_LOSS, 17))
        assert torch.equal(da[tie], da0[tie] if accumulate else torch.zeros_like(da[tie]))


# ------------------------------------------------------------------ weight norm backward, spectral-norm sigma
WN_SHAPES = [(co, ci, 5, 1) for ci, co in [(1, 32), (2, 32), (32, 128), (128, 512), (512, 1024), (1024, 1024)]] + [(1, 1024, 3, 1)] + \
            [(co, ci // g, k) for ci, co, k, _, g, _ in MSD_LAYERS] + [(1, 1024, 3)]
# measured worst (H100 80GB HBM3, 400 W): dv 8.0e-8 / 1.7e-7, dg 2.8e-7 / 2.8e-7
WN_TOL = {'dv': (4e-7, 8.5e-7), 'dg': (1.4e-6, 1.4e-6)}


@pytest.mark.parametrize('shape', WN_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_weight_norm_backward_matches_float64_autograd(shape):
    g = _gen('wn', shape)
    v = (torch.randn(*shape, generator=g) * 0.02).cuda()
    gv = (v.flatten(1).norm(dim=1) * (1 + 0.3 * torch.rand(shape[0], generator=g).cuda())).view(-1, *([1] * (len(shape) - 1)))
    dw = torch.randn(*shape, generator=g).cuda()
    dv, dg = torch.full_like(v, float('nan')), torch.full_like(gv, float('nan'))
    _native.check(_native.lib().svb_weight_norm_backward(_native.ptr(v), _native.ptr(gv.contiguous()), _native.ptr(dw), shape[0],
                                                         v[0].numel(), _native.ptr(dv), _native.ptr(dg), None), 'weight_norm_backward')
    vd, gd = v.double().requires_grad_(True), gv.double().requires_grad_(True)
    torch._weight_norm(vd, gd, 0).backward(dw.double())
    assert_within(f'weight_norm {shape}', {'dv': errors(dv, vd.grad), 'dg': errors(dg, gd.grad)}, WN_TOL)


SIGMA_TOL = 2.5e-7      # measured worst 4.7e-8 (H100 80GB HBM3, 400 W)


@pytest.mark.parametrize('layer', list(range(len(MSD_LAYERS) + 1)))
def test_spectral_sigma_matches_float64(layer):
    """sigma = u . (W v) on the MSD[0] weight matrices [Cout, Cin/groups * K], u / v one power iteration from a random start
    (what torch.nn.utils.spectral_norm keeps), so sigma is near the top singular value and has no cancellation."""
    ci, co, k, _, grp, _ = MSD_LAYERS[layer] if layer < len(MSD_LAYERS) else (1024, 1, 3, 1, 1, 1)
    g = _gen('sigma', layer)
    W = torch.randn(co, ci // grp * k, generator=g) / np.sqrt(ci // grp * k)
    u = F.normalize(torch.randn(co, generator=g, dtype=torch.float64), dim=0)
    v = F.normalize(W.double().t() @ u, dim=0)
    u = F.normalize(W.double() @ v, dim=0)
    W, u, v = W.contiguous(), u.float().contiguous(), v.float().contiguous()
    sigma = f32()
    _native.check(_native.lib().svb_spectral_sigma_host(_native.ptr(W), _native.ptr(u), _native.ptr(v), W.shape[0], W.shape[1], 0,
                                                        ctypes.byref(sigma)), 'spectral_sigma')
    ref = float(u.double() @ (W.double() @ v.double()))
    rel = abs(sigma.value - ref) / abs(ref)
    print('MEASURED sigma', layer, f'{rel:.2e}')
    assert rel <= SIGMA_TOL, (sigma.value, ref)

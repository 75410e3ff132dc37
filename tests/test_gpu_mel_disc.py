"""The mel discriminator on the native kernels against float64 torch: the 2-D wgmma layer, the fp32 2-D conv, the fused
Dropout2d + InstanceNorm2d and the adv_layer kernels one by one; the module against the reference fixture (train mode with the
captured Dropout2d masks, eval mode); the discriminator's part of the G and D steps through oracle/multi_window_disc.py with
needs_input_grad honoured; three alternating G / D AdamW rounds; the SVB model's phase-2 and phase-3 steps with their adversarial
terms; seeded repeatability of the starts and masks.
Errors are relative L2 and L-inf relative to max |reference|."""
import contextlib
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200 import _native
from neuralsvb_b200.modules.fastspeech import multi_window_disc as M
from neuralsvb_b200.utils import synthetic as S
from oracle import multi_window_disc as OD

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'mel_disc.npz'))
# (rel L2, rel L-inf) bars, about 5x the worst error measured on an H100 80GB HBM3 (DESIGN section 8 records the run)
KERNEL_BARS = {'fp32': (5e-6, 1e-5), 'tf32x3': (5e-5, 1e-4), 'bf16x3': (5e-5, 1e-4)}
MODULE_BARS = {False: (5e-5, 1e-4), True: (5e-4, 1e-3)}      # keyed by USE_TC; gradients through three instance norms
# G / D steps and the AdamW rounds, against float64 on the kernels' own leaky-relu masks (_native_masks).  Worst measured: fp32
# 2.6e-6 / 3.8e-6, bf16x3 2.9e-5 / 5.3e-5.  With F.leaky_relu in the reference instead, one pre-activation that rounds across zero
# moves a gradient by 0.8x that element's share: 2.6e-3 / 9.5e-3 on the bf16x3 D step, and 1.7e-2 on both paths (float32 torch
# too) for the D step right after an AdamW update of the mel.
STEP_BARS = {False: (1.5e-5, 2e-5), True: (1.5e-4, 3e-4)}


def _err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    d = got - ref
    return float(d.norm() / max(float(ref.norm()), 1e-30)), float(d.abs().max() / max(float(ref.abs().max()), 1e-30))


def _check(tag, got, ref, bars):
    assert got is not None and tuple(got.shape) == tuple(ref.shape), tag
    e2, ei = _err(got, ref)
    print(f'ERR {tag} {e2:.2e} {ei:.2e}')
    assert e2 < bars[0] and ei < bars[1], (tag, e2, ei)


def _rand(shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


# ---------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize('B,Cin,Cout,H,W', [(3, 64, 96, 37, 21), (2, 128, 128, 16, 40), (1, 32, 32, 5, 80)])
@pytest.mark.parametrize('prec', ['tf32x3', 'bf16x3'])
def test_tc_layer_2d_matches_float64(prec, B, Cin, Cout, H, W):
    x, w, b = _rand((B, Cin, H, W), 1), _rand((Cout, Cin, 3, 3), 2, (Cin * 9) ** -0.5), _rand((Cout,), 3, 0.1)
    x64, w64, b64 = (t.double().cuda().requires_grad_(True) for t in (x, w, b))
    y64 = F.leaky_relu(F.conv2d(x64, w64, b64, stride=2, padding=1), 0.2)
    dy = _rand(tuple(y64.shape), 4).cuda()
    y64.backward(dy.double())
    lib = _native.lib()
    h = ctypes.c_void_p()
    _native.check(lib.svb_tc_layer_create_2d(Cin, Cout, 3, 3, 2, 2, 1, 1, _native.PREC[prec], 0, ctypes.byref(h)), 'create_2d')
    try:
        xc, wc, bc = x.cuda(), w.cuda(), b.cuda()
        st = _native.current_stream_ptr()
        _native.check(lib.svb_tc_layer_set_weight_dev(h, _native.ptr(wc), _native.ptr(bc), st), 'set_weight')
        assert int(lib.svb_tc_layer_out_len(h, H)) == y64.shape[2]
        y = torch.empty(tuple(y64.shape), device='cuda')
        _native.check(lib.svb_tc_layer_forward(h, _native.ptr(xc), B, H, W, ctypes.c_float(0.2), _native.ptr(y), st), 'forward')
        dx, dw, db = torch.empty_like(xc), torch.zeros_like(wc), torch.zeros_like(bc)
        _native.check(lib.svb_tc_layer_backward(h, _native.ptr(xc), _native.ptr(y), _native.ptr(dy), B, H, W, ctypes.c_float(0.2),
                                                _native.ptr(dx), _native.ptr(dw), _native.ptr(db), st), 'backward')
        torch.cuda.synchronize()
    finally:
        lib.svb_tc_layer_destroy(h)
    tag = f'tc2d {prec} B{B} {Cin}->{Cout} {H}x{W}'
    for name, got, ref in (('y', y, y64), ('dx', dx, x64.grad), ('dw', dw, w64.grad), ('db', db, b64.grad)):
        _check(f'{tag} {name}', got, ref, KERNEL_BARS[prec])


def test_tc_layer_2d_rejects_bad_geometry():
    lib = _native.lib()
    h = ctypes.c_void_p()
    for args in ((128, 128, 3, 3, 2, 2, 2, 1), (128, 128, 3, 3, 0, 2, 1, 1), (1, 128, 3, 3, 2, 2, 1, 1), (128, 100, 3, 3, 2, 2, 1, 1)):
        assert lib.svb_tc_layer_create_2d(*args, _native.PREC['bf16x3'], 0, ctypes.byref(h)) == -1, args


@pytest.mark.parametrize('B,Cin,Cout,H,W', [(2, 1, 128, 33, 80), (3, 128, 128, 16, 40), (2, 5, 7, 9, 11)])
def test_conv2d_fp32_matches_float64(B, Cin, Cout, H, W):
    x, w, b = _rand((B, Cin, H, W), 11), _rand((Cout, Cin, 3, 3), 12, (Cin * 9) ** -0.5), _rand((Cout,), 13, 0.1)
    scale = (torch.rand(B, Cout, generator=torch.Generator().manual_seed(14)) > 0.25).float() / 0.75
    x64, w64, b64 = (t.double().cuda().requires_grad_(True) for t in (x, w, b))
    y64 = F.leaky_relu(F.conv2d(x64, w64, b64, stride=2, padding=1), 0.2) * scale.double().cuda()[:, :, None, None]
    dy = _rand(tuple(y64.shape), 15).cuda()
    y64.backward(dy.double())
    xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
    y = M._Conv2dFn.apply(xc, wc, bc, scale.cuda(), (3, 3, 2, 2, 1, 1))
    y.backward(dy)
    tag = f'conv2d fp32 B{B} {Cin}->{Cout} {H}x{W}'
    for name, got, ref in (('y', y, y64), ('dx', xc.grad, x64.grad), ('dw', wc.grad, w64.grad), ('db', bc.grad, b64.grad)):
        _check(f'{tag} {name}', got, ref, KERNEL_BARS['fp32'])


@pytest.mark.parametrize('B,C,H,W', [(2, 128, 8, 20), (3, 16, 4, 10), (1, 8, 64, 10)])
def test_drop_inorm_matches_float64(B, C, H, W):
    v = _rand((B, C, H, W), 21)
    v[0, 1] = 0.7                                                    # a constant plane: variance 0, gives beta
    scale = (torch.rand(B, C, generator=torch.Generator().manual_seed(22)) > 0.25).float() / 0.75
    scale[0, 2] = 0.0                                                # a dropped plane
    gamma, beta = 1 + _rand((C,), 23, 0.2), _rand((C,), 24, 0.1)
    v64, g64, b64 = (t.double().cuda().requires_grad_(True) for t in (v, gamma, beta))
    y64 = F.instance_norm(v64 * scale.double().cuda()[:, :, None, None], weight=g64, bias=b64, eps=1e-5)
    dy = _rand(tuple(y64.shape), 25).cuda()
    y64.backward(dy.double())
    vc, gc, bc = (t.cuda().requires_grad_(True) for t in (v, gamma, beta))
    y = M._DropINormFn.apply(vc, scale.cuda(), gc, bc)
    y.backward(dy)
    assert torch.isfinite(y).all() and torch.isfinite(vc.grad).all()
    assert torch.allclose(y[0, 2], bc[2].detach().expand(H, W)) and torch.allclose(y[0, 1], bc[1].detach().expand(H, W), atol=1e-3)
    assert float(vc.grad[0, 2].abs().max()) == 0.0
    tag = f'drop_inorm B{B} C{C} {H}x{W}'
    for name, got, ref in (('y', y, y64), ('dv', vc.grad, v64.grad), ('dgamma', gc.grad, g64.grad), ('dbeta', bc.grad, b64.grad)):
        _check(f'{tag} {name}', got, ref, KERNEL_BARS['fp32'])


def test_linear1_matches_float64():
    x, w, b = _rand((16, 20480), 31), _rand((1, 20480), 32, 20480 ** -0.5), _rand((1,), 33, 0.1)
    x64, w64, b64 = (t.double().cuda().requires_grad_(True) for t in (x, w, b))
    y64 = F.linear(x64, w64, b64)
    dy = _rand((16, 1), 34).cuda()
    y64.backward(dy.double())
    xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
    y = M._Linear1Fn.apply(xc, wc, bc)
    y.backward(dy)
    for name, got, ref in (('y', y, y64), ('dx', xc.grad, x64.grad), ('dw', wc.grad, w64.grad), ('db', bc.grad, b64.grad)):
        _check(f'linear1 {name}', got, ref, KERNEL_BARS['fp32'])


# ---------------------------------------------------------------------------------------------------------- module
@pytest.fixture(params=[False, True], ids=['fp32', 'tc'])
def use_tc(request, monkeypatch):
    monkeypatch.setattr(M, 'USE_TC', request.param)
    return request.param


def _disc():
    m = M.Discriminator(time_lengths=[32, 64, 128], freq_length=80, hidden_size=128, kernel=(3, 3), cond_size=0, norm_type='in',
                        reduction='stack')
    m.load_state_dict(S.make_mel_disc_state_dict(1234), strict=True)
    return m.cuda()


def _case(name):
    p = GOLD[f'{name}/params']
    B, T = int(p[0]), int(p[1])
    return B, T, [int(v) for v in p[2:2 + B]], [None if s < 0 else [int(s)] * B for s in p[2 + B:]]


def _gold_packed(prefix, k):
    return float(GOLD[f'{prefix}/{k}/norm']), torch.from_numpy(GOLD[f'{prefix}/{k}/sub']).double()


def _stride(n, s):
    return 1 if n <= 4096 else s


@pytest.mark.parametrize('mode', ['train', 'eval'])
@pytest.mark.parametrize('name', ['long', 'short'])
def test_module_matches_reference_fixture(use_tc, name, mode):
    from oracle.gen_golden import DISC_GRAD_STRIDE, GRAD_STRIDE
    B, T, pad, starts = _case(name)
    m = _disc().train(mode == 'train')
    scales = None
    if mode == 'train':
        s = torch.from_numpy(GOLD[f'{name}/train/scales']).reshape(-1, 3, B, 128).cuda()
        scales = [[s[w, j] for j in range(3)] for w in range(s.shape[0])] + [None] * (3 - s.shape[0])
    x = S.make_disc_mel(B, T, pad, 1234).cuda().requires_grad_(True)
    ret = m(x, start_frames_wins=[None if v is None else list(v) for v in starts], dropout_scales=scales)
    p, bars = f'{name}/{mode}', MODULE_BARS[use_tc]
    assert ret['y_c'] is None and len(ret['h']) == int(GOLD[f'{p}/n_h'])
    for i, h in enumerate(ret['h']):
        norm, sub = _gold_packed(f'{p}/h', str(i))
        hv = h.detach().double().reshape(-1).cpu()
        _check(f'module {use_tc} {p} h{i}', hv[::_stride(hv.numel(), DISC_GRAD_STRIDE)], sub, bars)
        assert abs(float(hv.norm()) - norm) < bars[0] * norm
    if f'{p}/y' not in GOLD:
        assert ret['y'] is None
        return
    y = ret['y']
    _check(f'module {use_tc} {p} y', y, torch.from_numpy(GOLD[f'{p}/y']), bars)
    F.mse_loss(y, torch.ones_like(y)).backward()
    g = x.grad.double().reshape(-1).cpu()
    _check(f'module {use_tc} {p} dmel', g[::GRAD_STRIDE], _gold_packed(f'{p}/dmel', 'x')[1], bars)
    for k, q in m.named_parameters():
        gv = q.grad.double().reshape(-1).cpu()
        _check(f'module {use_tc} {p} d{k}', gv[::_stride(gv.numel(), DISC_GRAD_STRIDE)], _gold_packed(f'{p}/grad', k)[1], bars)


def _draw(m, B, T_len, seed):
    """Starts and masks of one discriminator call, drawn the way the module draws them."""
    np.random.seed(seed)
    starts = [None] * 3
    M.clip_starts(T_len, (32, 64, 128), starts, B)
    torch.manual_seed(seed)
    scales = [d.draw_dropout_scales(B, torch.device('cuda')) for d in m.discriminator.conv_layers]
    return starts, [[s.reshape(B, -1) for s in w] for w in scales]


def _sd64(m, grad):
    return {k: v.detach().double().clone().requires_grad_(grad) for k, v in m.state_dict().items()}


@contextlib.contextmanager
def _native_masks(rec):
    """Record (output > 0) of every conv the module runs, in call order: the leaky-relu branch each output element took (block 1's
    Dropout2d factor is >= 0, and a dropped plane contributes nothing either way).  ``_masks(rec, k)`` groups them per call."""
    orig = {cls: cls.apply for cls in (M._Conv2dFn, M._Conv2dTcFn)}
    own = {cls: cls.__dict__.get('apply') for cls in orig}           # None: inherited from torch.autograd.Function

    def wrap(fn):
        def f(*a):
            y = fn(*a)
            rec.append(y.detach() > 0)
            return y
        return f
    try:
        for cls, fn in orig.items():
            cls.apply = wrap(fn)
        yield rec
    finally:
        for cls in orig:
            if own[cls] is None:
                del cls.apply
            else:
                cls.apply = own[cls]


def _masks(rec, n_calls):
    assert len(rec) == 9 * n_calls
    return [[[rec[9 * k + 3 * i + j] for j in range(3)] for i in range(3)] for k in range(n_calls)]


def test_g_and_d_steps_match_float64(use_tc):
    """G step: the discriminator is frozen and only d mel_out is wanted; D step: the mels are data and every discriminator
    parameter gets its gradient.  The adversarial terms are oracle/multi_window_disc.svb_adv_losses of both ways, run on the
    kernels' own leaky-relu masks."""
    B = 2
    m = _disc().train()
    mels = {w: S.make_disc_mel(B, 150, (0, 11 * i), 1234 + i).cuda() for i, w in enumerate(('a2a', 'p2p'))}
    gts = {w: S.make_disc_mel(B, 150, (0, 11 * i), 99 + i).cuda() for i, w in enumerate(('a2a', 'p2p'))}
    draws = [_draw(m, B, 150, 7 + k) for k in range(4)]
    sc64 = [[[s.double() for s in w] for w in d[1]] for d in draws]
    bars = STEP_BARS[use_tc]
    # G step
    m.requires_grad_(False)
    outs = {w: v.clone().requires_grad_(True) for w, v in mels.items()}
    total = 0
    with _native_masks([]) as rec:
        for k, (w, mel) in enumerate(outs.items()):
            y = m(mel, start_frames_wins=draws[k][0], dropout_scales=draws[k][1])['y']
            total = total + F.mse_loss(y, torch.ones_like(y)) * OD.LAMBDA_MEL_ADV
    total.backward()
    assert all(q.grad is None for q in m.parameters())
    outs64 = {w: v.double().clone().requires_grad_(True) for w, v in mels.items()}
    ref = OD.svb_adv_losses(_sd64(m, False), 'g', outs64, starts=[d[0] for d in draws], scales=sc64, masks=_masks(rec, 2))
    sum(ref.values()).backward()
    for w in outs:
        _check(f'G step {use_tc} d{w}', outs[w].grad, outs64[w].grad, bars)
    _check(f'G step {use_tc} loss', total.reshape(1), sum(ref.values()).reshape(1), bars)
    # D step
    m.requires_grad_(True)
    total = 0
    k = 0
    with _native_masks([]) as rec:
        for w in mels:
            y_r = m(gts[w], start_frames_wins=draws[k][0], dropout_scales=draws[k][1])['y']
            y_f = m(mels[w].detach(), start_frames_wins=draws[k + 1][0], dropout_scales=draws[k + 1][1])['y']
            total = total + F.mse_loss(y_r, torch.ones_like(y_r)) + F.mse_loss(y_f, torch.zeros_like(y_f))
            k += 2
    total.backward()
    sd = _sd64(m, True)
    ref = OD.svb_adv_losses(sd, 'd', {w: v.double() for w, v in mels.items()}, targets={w: v.double() for w, v in gts.items()},
                            starts=[d[0] for d in draws], scales=sc64, masks=_masks(rec, 4))
    sum(ref.values()).backward()
    assert set(ref) == {'a2a_r', 'a2a_f', 'p2p_r', 'p2p_f'}
    for n, q in m.named_parameters():
        _check(f'D step {use_tc} d{n}', q.grad, sd[n].grad, bars)


def test_three_alternating_adamw_steps(use_tc):
    """Three G / D rounds of AdamW on one module: a learnable mel plays the generator.  Every round's gradients match float64 at
    the parameters the native run reached, the 2-D layer handles are the ones built first and they are re-packed after each
    discriminator update."""
    B = 2
    m = _disc().train()
    mel = torch.nn.Parameter(S.make_disc_mel(B, 140, (0, 9), 5).cuda())
    gt = S.make_disc_mel(B, 140, (0, 9), 6).cuda()
    opt_g, opt_d = torch.optim.AdamW([mel], 1e-3), torch.optim.AdamW(list(m.parameters()), 2e-4, betas=(0.5, 0.9))
    bars = STEP_BARS[use_tc]
    layers = [L for d in m.discriminator.conv_layers for L in d._tc[1:]]
    handles, wkeys = None, None
    for step in range(3):
        d0, d1, d2 = (_draw(m, B, 140, 100 * step + k) for k in range(3))
        sc = [[[s.double() for s in w] for w in d[1]] for d in (d0, d1, d2)]
        m.requires_grad_(False)
        opt_g.zero_grad()
        mel64 = mel.detach().double().clone().requires_grad_(True)
        with _native_masks([]) as rec:
            y = m(mel, start_frames_wins=d0[0], dropout_scales=d0[1])['y']
        (F.mse_loss(y, torch.ones_like(y)) * OD.LAMBDA_MEL_ADV).backward()
        sum(OD.svb_adv_losses(_sd64(m, False), 'g', {'a2a': mel64}, starts=[d0[0]], scales=sc[:1], masks=_masks(rec, 1)).values()).backward()
        _check(f'adamw {use_tc} step {step} dmel', mel.grad, mel64.grad, bars)
        opt_g.step()
        m.requires_grad_(True)
        opt_d.zero_grad()
        with _native_masks([]) as rec:
            y_r = m(gt, start_frames_wins=d1[0], dropout_scales=d1[1])['y']
            y_f = m(mel.detach(), start_frames_wins=d2[0], dropout_scales=d2[1])['y']
        (F.mse_loss(y_r, torch.ones_like(y_r)) + F.mse_loss(y_f, torch.zeros_like(y_f))).backward()
        sd = _sd64(m, True)
        sum(OD.svb_adv_losses(sd, 'd', {'a2a': mel.detach().double()}, targets={'a2a': gt.double()}, starts=[d1[0], d2[0]],
                              scales=sc[1:], masks=_masks(rec, 2)).values()).backward()
        for n, q in m.named_parameters():
            _check(f'adamw {use_tc} step {step} d{n}', q.grad, sd[n].grad, bars)
        if use_tc:
            now = [L.h.value for L in layers]
            assert handles is None or now == handles
            handles = now
            assert wkeys is None or all(a != b for a, b in zip(wkeys, [L.wkey for L in layers]))      # re-packed after the update
            wkeys = [L.wkey for L in layers]
        opt_d.step()


# ------------------------------------------------------------------------------------------------- the SVB model's steps
@pytest.fixture(params=[False, True], ids=['fp32_cuda_cores', 'bf16x3_tensor_cores'])
def model_tc(request, monkeypatch):
    from neuralsvb_b200.modules.voice_conversion import vc_modules as V
    monkeypatch.setattr(V, 'USE_TC', request.param)
    monkeypatch.setattr(M, 'USE_TC', request.param)
    return request.param


@pytest.mark.parametrize('phase', [2, 3])
def test_svb_step_with_adversarial_terms_matches_float64(model_tc, phase):
    """The phase-2 generator step with {a2a,p2p}_a and the phase-3 mapping step with a2p_a: the MleSVBVAE on its native kernels
    plus the native discriminator (frozen, train mode: its Dropout2d stays active in phase 3), against float64 autograd through
    oracle/svb_vae_train.svb_train_losses plus oracle/multi_window_disc.svb_adv_losses, on the discriminator's own leaky-relu masks
    and, as tests/test_gpu_svb_vae_train._tied_step does, on the native PPG, train-mode BatchNorm inputs and ReLU masks.  Bars are the steps'
    own (tests/test_gpu_svb_vae_train.py)."""
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    from oracle import svb_vae_train as O
    from tests.test_gpu_svb_vae_train import MAP_BARS, MAP_ZERO_GRAD, _compare_step, _model, _native_relu, _recorded, _set_phase, _tie
    from tests.test_gpu_svb_vae_train import STEP_BARS as SVB_STEP_BARS
    Ta, Tp = 136, 140                                   # long enough for the 128-frame window: the adversarial terms exist
    batch = S.make_svb_batch(2, Ta, Tp, 1234)
    m = _model('bf16x3' if model_tc else 'fp32')
    _set_phase(m, phase)
    disc = _disc().train()
    disc.requires_grad_(False)
    ways = ['a2a', 'p2p'] if phase == 2 else ['a2a', 'p2p', 'a2p']
    adv = ['a2a', 'p2p'] if phase == 2 else ['a2p']
    draws = [_draw(disc, 2, Ta if w == 'a2a' else Tp, 50 + k) for k, w in enumerate(adv)]
    snap = {k: v.detach().clone() for k, v in m.state_dict().items()}
    b = {k: v.cuda() for k, v in batch.items()}
    targets = {'a2a': b['amateur_mel'], 'p2p': b['prof_mel'], 'a2p': b['prof_mel']}
    with _recorded(m) as trace:
        ret = m(**b, concurrent_ways=ways, eps=torch.zeros(2, 128, 1, device='cuda'))
    losses = {}
    for way in ways:
        if 'kl' in ret[way]:
            losses[f'{way}_kl'] = ret[way]['kl'] * 0.001
        l1, ss = mel_l1_ssim_loss(ret[way]['mel_out'], targets[way])
        losses[f'l1{way}'], losses[f'ssim{way}'] = 0.5 * l1, 0.5 * ss
    if phase == 3:
        losses['a2p_mle'] = ret['a2p']['mle'] * 1.0
    with _native_masks([]) as rec:
        for k, way in enumerate(adv):
            y = disc(ret[way]['mel_out'], start_frames_wins=draws[k][0], dropout_scales=draws[k][1])['y']
            losses[f'{way}_a'] = F.mse_loss(y, torch.ones_like(y)) * OD.LAMBDA_MEL_ADV
    sum(losses.values()).backward()
    assert all(q.grad is None for q in disc.parameters())
    req = {n for n, q in m.named_parameters() if q.requires_grad}
    p = {k: (v.double().clone().requires_grad_(k in req) if v.is_floating_point() else v.clone()) for k, v in snap.items()}
    b64 = {k: (v.double() if v.is_floating_point() else v) for k, v in b.items()}
    tie, left = _tie(trace['bn'])
    relu, masks_left = _native_relu(trace)
    ref, out = O.svb_train_losses(p, b64, torch.zeros(2, 128, 1, device='cuda', dtype=torch.float64), phase,
                                  ppg=dict(zip(('amateur', 'prof'), trace['ppg'])), tie=tie, relu=relu)
    assert not any(left.values()) and not any(masks_left.values())
    ref.update(OD.svb_adv_losses(_sd64(disc, False), 'g' if phase == 2 else 3, {w: out[w]['mel_out'] for w in adv},
                                 starts=[d[0] for d in draws], scales=[[[s.double() for s in w] for w in d[1]] for d in draws],
                                 masks=_masks(rec, len(adv))))
    assert {f'{w}_a' for w in adv} <= set(ref)
    sum(ref.values()).backward()
    bars = (SVB_STEP_BARS if phase == 2 else MAP_BARS)[model_tc]
    # The latent map's convs.0 / convs.3 biases feed train-mode BatchNorms directly (spk_proj.2's through convs.0): their exact
    # gradient is 0 (the norm removes any per-channel shift), so both sides hold only rounding.  They are checked to stay at that
    # level instead of relatively.
    shift_free = set(MAP_ZERO_GRAD) if phase == 3 else set()
    big = max(float(m.get_parameter(k).grad.abs().max()) for k in req)
    for k in shift_free:
        got, want = float(m.get_parameter(k).grad.abs().max()), float(p[k].grad.abs().max())
        print(f'ERR phase{phase} adv {model_tc} d{k} |native| {got / big:.2e} |float64| {want / big:.2e} of the largest gradient')
        assert got < 1e-4 * big and want < 1e-4 * big, k
        m.get_parameter(k).requires_grad_(False)
        m.get_parameter(k).grad = None
    n = _compare_step(f'phase{phase} adv {model_tc}', m, phase, losses, ref, p, bars)
    assert n + len(shift_free) > 100 if phase == 2 else n + len(shift_free) == len(list(m.z_mapping_function.parameters()))


def test_seeded_draws_repeat_and_follow_torch_dropout2d():
    m = _disc().train()
    B = 3
    a, b = _draw(m, B, 150, 42), _draw(m, B, 150, 42)
    assert a[0] == b[0]
    assert all(torch.equal(s, t) for w, v in zip(a[1], b[1]) for s, t in zip(w, v))
    # the masks are the ones nn.Dropout2d would draw from the same generator state, in the reference's layer order
    torch.manual_seed(42)
    ref = []
    for _ in range(9):
        o = F.dropout2d(torch.ones(B, 128, 2, 2, device='cuda'), 0.25, training=True)
        ref.append(o[:, :, 0, 0])
    got = [s for w in a[1] for s in w]
    assert all(torch.equal(g, r) for g, r in zip(got, ref))
    # a seeded module forward draws the same starts and masks as the injected ones
    x = S.make_disc_mel(B, 150, (0, 3, 9), 1)
    np.random.seed(42)
    torch.manual_seed(42)
    with torch.no_grad():
        r1 = m(x.cuda())
    with torch.no_grad():
        r2 = m(x.cuda(), start_frames_wins=a[0], dropout_scales=a[1])
    assert r1['start_frames_wins'] == a[0] and torch.equal(r1['y'], r2['y'])

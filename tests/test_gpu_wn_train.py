"""GlobalFVAE training on the native kernels: every gradient of the WN stack, the FVAE decoder, the K = 8 strided conv and
the whole GlobalFVAE against float64 torch autograd through oracle/fs2_vae.py, on the same fp32 inputs and cotangents.
Errors are relative L2 and L-inf relative to max |reference|."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200.utils import synthetic as S

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
PRECISIONS = ['fp32', 'tf32', 'tf32x3', 'bf16x3']
# (rel L2, rel L-inf) bars per precision: about 5x (fp32 L-inf 4x) the worst error any test of this file measured on an H100 80GB HBM3 at
# 400 W (worst: fp32 3.4e-6 / 5.0e-6, tf32 1.1e-3 / 1.7e-3, tf32x3 3.9e-5 / 4.5e-5, bf16x3 4.0e-5 / 4.2e-5; the deepest
# graphs -- the whole GlobalFVAE and the 8-layer conditioned stack -- set them)
BARS = {'fp32': (1.7e-5, 2e-5), 'tf32': (6e-3, 8e-3), 'tf32x3': (2e-4, 2.2e-4), 'bf16x3': (2e-4, 2.1e-4)}
# one strided fp32 conv (svb_conv_nct_backward, K = 8): worst dx 4.1e-7 / 1.1e-6, dw 1.4e-7 / 3.8e-7, db 7.3e-8 / 7.4e-8
CONV_BARS = {'dx': (2e-6, 5.5e-6), 'dw': (7.5e-7, 2e-6), 'db': (4e-7, 4e-7)}


def _err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    d = got - ref
    return float(d.norm() / ref.norm()), float(d.abs().max() / ref.abs().max())


def _check(tag, got, ref, bars):
    l2, li = _err(got, ref)
    print(f'ERR {tag} {l2:.2e} {li:.2e}')
    assert l2 < bars[0] and li < bars[1], (tag, l2, li, bars)


def _cot(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).randn(*shape).astype(np.float32))


def _leaf64(t):
    return None if t is None else t.double().requires_grad_(True)


def _check_params(tag, module, ref, bars, prefix=''):
    n = 0
    for name, p in module.named_parameters():
        _check(f'{tag} d{name}', p.grad, ref[prefix + name].grad, bars)
        n += 1
    assert n > 0


# ---------------------------------------------------------------------------------------------------------- WN stack
# (H, K, dilation_rate, L, gin, B, T, mask): the three wn.npz shapes, then L = 1, no mask, T shorter than the receptive field
# (dilations 1, 2, 4, 8 reach 30 rows each side), B = 3 with an odd T
WN_CASES = {
    'fvae_dec': (192, 5, 1, 4, 0, 2, 100, True),
    'fvae_enc_cond': (192, 5, 1, 8, 256, 2, 61, True),
    'dilated_cond': (64, 3, 2, 3, 32, 1, 300, True),
    'one_layer': (64, 5, 1, 1, 32, 2, 50, True),
    'no_mask': (64, 3, 1, 2, 0, 2, 40, False),
    'short_T': (64, 5, 2, 4, 16, 2, 9, True),
    'B3_oddT': (64, 5, 1, 3, 16, 3, 77, True),
}


def _wn_reference(sd, case, x, mask, g, cot):
    from oracle import fs2_vae as OW
    H, K, dr, L = case[:4]
    p = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    xd, gd = _leaf64(x), _leaf64(g)
    y = OW.wn_forward(OW.fold_weight_norm(p), H, K, dr, L, xd, None if mask is None else mask.double(), gd)
    (y * cot.double()).sum().backward()
    return y, xd, gd, p


def _wn_native(sd, case, x, mask, g, cot, precision, m=None):
    from neuralsvb_b200.modules.fastspeech.fs2_vae import WN
    H, K, dr, L, gin = case[:5]
    if m is None:
        m = WN(H, K, dr, L, gin_channels=gin, precision=precision, trainable=True)
        m.load_state_dict(sd, strict=True)
        m = m.cuda().train()
    xc = x.cuda().requires_grad_(True)
    gc = None if g is None else g.cuda().requires_grad_(True)
    y = m(xc, None if mask is None else mask.cuda(), gc)
    (y * cot.cuda()).sum().backward()
    return m, y, xc, gc


@pytest.mark.parametrize('name', list(WN_CASES))
@pytest.mark.parametrize('precision', PRECISIONS)
def test_wn_backward_matches_float64(name, precision):
    case = WN_CASES[name]
    H, K, dr, L, gin, B, T, use_mask = case
    sd = S.make_wn_state_dict(H, K, L, gin, 1234)
    x, mask, g = S.make_wn_inputs(B, T, H, gin, 1234)
    mask = mask if use_mask else None
    cot = _cot((B, H, T), 7)
    y_ref, xd, gd, p = _wn_reference(sd, case, x, mask, g, cot)
    m, y, xc, gc = _wn_native(sd, case, x, mask, g, cot, precision)
    bars = BARS[precision]
    _check(f'wn {name} {precision} y', y, y_ref, bars)
    _check(f'wn {name} {precision} dx', xc.grad, xd.grad, bars)
    if gin:
        _check(f'wn {name} {precision} dg', gc.grad, gd.grad, bars)
    _check_params(f'wn {name} {precision}', m, p, bars)


# ---------------------------------------------------------------------------------------------------------- decoder
def _decoder_setup(name):
    g = np.load(os.path.join(GOLDEN, 'fvae_decoder.npz'))
    lat, H, oc, K, L, gin, B, T, glob = [int(v) for v in g[f'{name}/params']]
    sd = S.make_fvae_decoder_state_dict(lat, H, oc, K, L, gin, 4, 1234)
    _, mask, cond = S.make_wn_inputs(B, T, H, gin, 1234)
    z = torch.from_numpy(np.random.RandomState(1234 + 5).randn(B, lat, 1 if glob else T // 4).astype(np.float32))
    return (lat, H, oc, K, L, gin, B, T, glob), sd, z, (mask if glob else 1), cond


def _decoder_reference(cfg, sd, z, mask, cond, cot):
    from oracle import fs2_vae as OW
    lat, H, oc, K, L, gin, B, T, glob = cfg
    p = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    zd, gd = _leaf64(z), _leaf64(cond)
    y = OW.fvae_decoder_forward(OW.fold_weight_norm(p), H, K, L, 4, zd, mask.double() if torch.is_tensor(mask) else mask, gd, bool(glob))
    (y * cot.double()).sum().backward()
    return y, zd, gd, p


def _decoder_native(cfg, m, z, mask, cond, cot):
    zc = z.cuda().requires_grad_(True)
    gc = None if cond is None else cond.cuda().requires_grad_(True)
    y = m(zc, mask.cuda() if torch.is_tensor(mask) else mask, gc)
    (y * cot.cuda()).sum().backward()
    return y, zc, gc


def _make_decoder(cfg, sd, precision):
    from neuralsvb_b200.modules.fastspeech.fs2_vae import FVAEDecoder, GlobalFVAEDecoder
    lat, H, oc, K, L, gin, B, T, glob = cfg
    m = (GlobalFVAEDecoder if glob else FVAEDecoder)(lat, H, oc, K, L, gin, strides=[4], precision=precision, trainable=True)
    m.load_state_dict(sd, strict=True)
    return m.cuda().train()


@pytest.mark.parametrize('name', ['global_dec', 'local_dec_nocond_mask1'])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_fvae_decoder_backward_matches_float64(name, precision):
    cfg, sd, z, mask, cond = _decoder_setup(name)
    lat, H, oc, K, L, gin, B, T, glob = cfg
    cot = _cot((B, oc, T), 11)
    y_ref, zd, gd, p = _decoder_reference(cfg, sd, z, mask, cond, cot)
    m = _make_decoder(cfg, sd, precision)
    y, zc, gc = _decoder_native(cfg, m, z, mask, cond, cot)
    bars = BARS[precision]
    _check(f'dec {name} {precision} y', y, y_ref, bars)
    _check(f'dec {name} {precision} dz', zc.grad, zd.grad, bars)
    if gin:
        _check(f'dec {name} {precision} dg', gc.grad, gd.grad, bars)
    _check_params(f'dec {name} {precision}', m, p, bars)


# ---------------------------------------------------------------------------------------------------------- K = 8 conv
@pytest.mark.parametrize('cin,cout', [(80, 192), (256, 256)])
def test_conv_nct_backward_k8_stride4(cin, cout):
    """svb_conv_nct_backward at the GlobalFVAE's pre_net (80 -> 192) and g_pre_net (256 -> 256): k 8, stride 4, pad 2."""
    from neuralsvb_b200.modules.hifigan.discriminators import conv_nct
    rs = np.random.RandomState(cin)
    B, T = 2, 240
    x = torch.from_numpy(rs.randn(B, cin, T).astype(np.float32))
    w = torch.from_numpy((rs.rand(cout, cin, 8).astype(np.float32) - 0.5) * 0.1)
    b = torch.from_numpy(rs.randn(cout).astype(np.float32) * 0.1)
    cot = _cot((B, cout, 60), 3)
    xd, wd, bd = _leaf64(x), _leaf64(w), _leaf64(b)
    (F.conv1d(xd, wd, bd, stride=4, padding=2) * cot.double()).sum().backward()
    xc, wc, bc = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    y = conv_nct(xc, wc, bc, 8, stride=4, pad=2)
    assert tuple(y.shape) == (B, cout, 60)
    (y * cot.cuda()).sum().backward()
    for tag, got, ref in (('dx', xc.grad, xd.grad), ('dw', wc.grad, wd.grad), ('db', bc.grad, bd.grad)):
        _check(f'conv_k8 {cin}->{cout} {tag}', got, ref, CONV_BARS[tag])


# ---------------------------------------------------------------------------------------------------------- GlobalFVAE
def _global_fvae_reference(p, cfg, x, mask, cond, eps, cot):
    """GlobalFVAE.forward(infer=False) in float64 with the poolings' BatchNorm in training mode (running statistics of ``p``
    updated in place), then x_recon . cot + kl backward."""
    from oracle import fs2_vae as OW
    io_c, H, lat, K, Le, Ld, gin, B, T = cfg
    w = OW.fold_weight_norm(p)
    g_sqz = F.conv1d(cond, w['g_pre_net.0.weight'], w['g_pre_net.0.bias'], stride=4, padding=2)
    e = {k[8:]: v for k, v in w.items() if k.startswith('encoder.')}
    h = F.conv1d(x, e['pre_net.0.weight'], e['pre_net.0.bias'], stride=4, padding=2)
    xm = mask[:, :, ::4][:, :, :h.shape[-1]]
    h = OW.wn_forward({k[3:]: v for k, v in e.items() if k.startswith('wn.')}, H, K, 1, Le, h * xm, xm, g_sqz) * xm
    h = F.conv1d(h, e['out_proj.weight'], e['out_proj.bias'])
    for i in (0, 3):
        h = torch.relu(F.conv1d(h, e[f'poolings.{i}.weight'], e[f'poolings.{i}.bias'], stride=2))
        j = i + 2
        h = F.batch_norm(h, p[f'encoder.poolings.{j}.running_mean'], p[f'encoder.poolings.{j}.running_var'], e[f'poolings.{j}.weight'],
                         e[f'poolings.{j}.bias'], training=True, momentum=0.1, eps=1e-5)
    h = F.conv1d(h, e['poolings.6.weight'], e['poolings.6.bias'], stride=2).mean(-1, keepdim=True)
    m_q, logs_q = torch.split(h, lat, dim=1)
    z = m_q + eps * torch.exp(logs_q)
    dec = {k[8:]: v for k, v in w.items() if k.startswith('decoder.')}
    x_recon = OW.fvae_decoder_forward(dec, H, K, Ld, 4, z, mask, cond, True)
    kl = torch.distributions.kl_divergence(torch.distributions.Normal(m_q, logs_q.exp()), torch.distributions.Normal(0.0, 1.0))
    kl = (kl * xm).sum() / xm.sum() / lat
    ((x_recon * cot).sum() + kl).backward()
    return x_recon, kl


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
def test_global_fvae_training_step_matches_float64(precision):
    from neuralsvb_b200.modules.fastspeech.fs2_vae import GlobalFVAE
    from tests.test_oracle_golden import _global_fvae_inputs
    g = np.load(os.path.join(GOLDEN, 'global_fvae.npz'))
    cfg, x, mask, cond = _global_fvae_inputs(g)
    io_c, H, lat, K, Le, Ld, gin, B, T = cfg
    sd = S.make_global_fvae_state_dict(io_c, H, lat, K, Le, Ld, gin, 4, 1234)
    eps = _cot((B, lat, 1), 5)
    cot = _cot((B, io_c, T), 13)
    p = {k: (v.double().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v.clone().double()) for k, v in sd.items()}
    cd = _leaf64(cond)
    xr_ref, kl_ref = _global_fvae_reference(p, cfg, x.double(), mask.double(), cd, eps.double(), cot.double())
    m = GlobalFVAE(io_c, H, lat, K, Le, Ld, gin, [4], precision=precision, trainable=True)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    cc = cond.cuda().requires_grad_(True)
    xr, kl, _, m_q, logs_q, xm, z_q = m(x.cuda(), mask.cuda(), cc, infer=False, eps=eps.cuda())
    ((xr * cot.cuda()).sum() + kl).backward()
    bars = BARS[precision]
    _check(f'gfvae {precision} x_recon', xr, xr_ref, bars)
    _check(f'gfvae {precision} kl', kl.reshape(1), kl_ref.reshape(1), bars)
    _check(f'gfvae {precision} dg', cc.grad, cd.grad, bars)
    _check_params(f'gfvae {precision}', m, p, bars)
    for j in (2, 5):
        for s in ('running_mean', 'running_var'):
            _check(f'gfvae {precision} bn{j} {s}', getattr(m.encoder.poolings[j], s), p[f'encoder.poolings.{j}.{s}'], bars)
        assert int(m.encoder.poolings[j].num_batches_tracked) == int(sd[f'encoder.poolings.{j}.num_batches_tracked']) + 1


# ---------------------------------------------------------------------------------------------------------- tape per call
def test_two_forwards_before_one_backward():
    """The a2a + p2p pattern: one module, two training forwards, then one backward.  The gradients are the float64 sum of
    both calls, so each call differentiated its own tape."""
    case = WN_CASES['fvae_enc_cond']
    H, K, dr, L, gin, B, T, _ = case
    sd = S.make_wn_state_dict(H, K, L, gin, 1234)
    x1, mask1, g1 = S.make_wn_inputs(B, T, H, gin, 1234)
    x2, mask2, g2 = S.make_wn_inputs(B, T + 16, H, gin, 99, ragged=False)
    c1, c2 = _cot((B, H, T), 1), _cot((B, H, T + 16), 2)
    from oracle import fs2_vae as OW
    p = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    w = OW.fold_weight_norm(p)
    ((OW.wn_forward(w, H, K, dr, L, x1.double(), mask1.double(), g1.double()) * c1.double()).sum()
     + (OW.wn_forward(w, H, K, dr, L, x2.double(), mask2.double(), g2.double()) * c2.double()).sum()).backward()
    from neuralsvb_b200.modules.fastspeech.fs2_vae import WN
    m = WN(H, K, dr, L, gin_channels=gin, precision='fp32', trainable=True)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    y1 = m(x1.cuda(), mask1.cuda(), g1.cuda())
    y2 = m(x2.cuda(), mask2.cuda(), g2.cuda())
    ((y1 * c1.cuda()).sum() + (y2 * c2.cuda()).sum()).backward()
    _check_params('two_calls fp32', m, p, BARS['fp32'])


# ---------------------------------------------------------------------------------------------------------- same forward
@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
def test_training_forward_equals_inference_forward(precision):
    from neuralsvb_b200.modules.fastspeech.fs2_vae import WN
    H, K, dr, L, gin, B, T, _ = WN_CASES['fvae_enc_cond']
    sd = S.make_wn_state_dict(H, K, L, gin, 1234)
    x, mask, g = S.make_wn_inputs(B, T, H, gin, 1234)
    mods = []
    for trainable in (False, True):
        m = WN(H, K, dr, L, gin_channels=gin, precision=precision, trainable=trainable)
        m.load_state_dict(sd, strict=True)
        m.remove_weight_norm()
        mods.append(m.cuda())
    with torch.no_grad():
        y_inf = mods[0].eval()(x.cuda(), mask.cuda(), g.cuda())
    y_train = mods[1].train()(x.cuda(), mask.cuda(), g.cuda())
    assert y_train.requires_grad and torch.equal(y_train.detach(), y_inf)
    cfg, dsd, z, dmask, cond = _decoder_setup('global_dec')
    decs = []
    for trainable in (False, True):
        d = _make_decoder(cfg, dsd, precision)
        d.trainable = trainable
        d.wn.remove_weight_norm()
        decs.append(d)
    with torch.no_grad():
        o_inf = decs[0].eval()(z.cuda(), dmask.cuda(), cond.cuda())
    o_train = decs[1].train()(z.cuda(), dmask.cuda(), cond.cuda())
    assert torch.equal(o_train.detach(), o_inf)


# ---------------------------------------------------------------------------------------------------------- optimizer steps
@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
def test_three_adamw_steps_repack_on_the_device(precision):
    """After every step the next training forward and its gradients match float64 at the module's current parameters (so
    every packing, the data-gradient twins included, was rebuilt on the device), the handle is the one built at the first
    call, no host upload happened, and an eval forward matches the oracle too."""
    cfg, sd, z, mask, cond = _decoder_setup('global_dec')
    lat, H, oc, K, L, gin, B, T, glob = cfg
    m = _make_decoder(cfg, sd, precision)
    opt = torch.optim.AdamW(m.parameters(), lr=2e-2)
    cot = _cot((B, oc, T), 17)
    bars = BARS[precision]
    handle = None
    for step in range(4):
        cur = {k: v.detach().cpu() for k, v in m.state_dict().items()}
        y_ref, zd, gd, p = _decoder_reference(cfg, cur, z, mask, cond, cot)
        opt.zero_grad()
        y, zc, gc = _decoder_native(cfg, m, z, mask, cond, cot)
        handle = handle or m._handle.value
        assert m._handle.value == handle and m.host_uploads == 1
        _check(f'adamw {precision} step {step} y', y, y_ref, bars)
        _check(f'adamw {precision} step {step} dz', zc.grad, zd.grad, bars)
        _check_params(f'adamw {precision} step {step}', m, p, bars)
        if step:
            with torch.no_grad():
                y_eval = m.eval()(z.cuda(), mask.cuda(), cond.cuda())
            m.train()
            _check(f'adamw {precision} step {step} eval y', y_eval, y_ref, bars)
        if step < 3:
            opt.step()
    assert m._handle.value == handle and m.host_uploads == 1


# ---------------------------------------------------------------------------------------------------------- ABI rejects
def test_training_abi_rejects_leave_buffers_untouched():
    from neuralsvb_b200 import _native
    from neuralsvb_b200.modules.fastspeech.fs2_vae import WN
    lib = _native.lib()
    m = WN(64, 3, 1, 2, trainable=True).cuda()
    x = torch.randn(2, 64, 32, device='cuda')
    with torch.no_grad():
        m.eval()(x)
    h = m._handle
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    src = torch.zeros(64 * 128 * 3 + 1, device='cuda')
    # a handle with training switched off takes no new weights
    assert lib.svb_wn_set_weight_dev(h, b'in_layers.0.weight', vp(src), 64 * 128 * 3, None) < 0 and b'only a training handle' in lib.svb_last_error()
    assert lib.svb_wn_set_training(h, 1) == 0
    assert lib.svb_wn_set_weight_dev(h, b'in_layers.0.weight', vp(src), 64 * 128 * 3 + 1, None) < 0 and b'elements' in lib.svb_last_error()
    assert lib.svb_wn_set_weight_dev(h, b'nope.weight', vp(src), 4, None) < 0 and b'no tensor' in lib.svb_last_error()
    tape = torch.empty(int(lib.svb_wn_tape_bytes(h, 2, 32)), device='cuda', dtype=torch.uint8)
    dout = torch.randn(2, 64, 32, device='cuda')
    dx = torch.full((2, 64, 32), 7.0, device='cuda')
    dg = torch.full((2, 8, 32), 7.0, device='cuda')
    # backward of a tape no training forward wrote
    assert lib.svb_wn_backward(h, vp(tape), 2, 32, vp(dout), vp(dx), None, None) < 0 and b'no training forward' in lib.svb_last_error()
    out = torch.empty_like(x)
    assert lib.svb_wn_forward_train(h, vp(x), None, None, 2, 32, vp(out), vp(tape), None) == 0
    assert lib.svb_wn_backward(h, vp(tape), 2, 16, vp(dout), vp(dx), None, None) < 0 and b'B 2 T 32' in lib.svb_last_error()
    assert lib.svb_wn_backward(h, vp(tape), 2, 32, vp(dout), vp(dx), vp(dg), None) < 0 and b'unconditioned' in lib.svb_last_error()
    assert lib.svb_fvae_decoder_backward(h, vp(tape), 2, 32, vp(dout), vp(dx), None, None) < 0 and b'not a decoder' in lib.svb_last_error()
    torch.cuda.synchronize()
    assert bool((dx == 7.0).all()) and bool((dg == 7.0).all())
    assert lib.svb_wn_backward(h, vp(tape), 2, 32, vp(dout), vp(dx), None, None) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all() and not bool((dx == 7.0).all())

"""-m gpu: MPD / MSD forward, GAN / feature losses and the multi-resolution STFT loss on the CUDA
operators, against the fixtures the reference modules produced (tests/golden/discriminators.npz,
losses.npz) and against the oracle."""
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200.utils import synthetic as S
from oracle import hifigan as O

pytestmark = pytest.mark.gpu
SEED = 1234
REL = 2e-4          # fp32 kernels, different summation order than cuDNN / MKL: relative L-inf per tensor


def _signals():
    y = S.make_wave_batch(2, 8192, seed=SEED)[:, None]
    y_hat = (y + 0.1 * S.make_wave_batch(2, 8192, seed=SEED + 5)[:, None]).clamp(-1, 1)
    return y, y_hat


@pytest.mark.parametrize('name', ['mpd', 'msd'])
def test_discriminator_forward_matches_reference_fixture(golden_dir, name):
    from neuralsvb_b200.modules.hifigan import discriminators as D
    g = np.load(os.path.join(golden_dir, 'discriminators.npz'))
    if name == 'mpd':
        m, sd = D.MultiPeriodDiscriminator(), S.make_mpd_state_dict(SEED)
    else:
        m, sd = D.MultiScaleDiscriminator(), S.make_msd_state_dict(SEED)
    m.load_state_dict(sd, strict=True)                    # reference key names and shapes
    m = m.eval().cuda()
    y, y_hat = _signals()
    with torch.no_grad():
        rs, gs, fr, fg = m(y.cuda(), y_hat.cuda())
        losses = [D.feature_loss(fr, fg), *D.discriminator_loss(rs, gs), D.generator_loss(gs)]
    torch.cuda.synchronize()
    for i, (r, gg) in enumerate(zip(rs, gs)):
        ref_r, ref_g = g[f'{name}/logit_r{i}'], g[f'{name}/logit_g{i}']
        assert tuple(r.shape) == ref_r.shape                                  # bit-exact logit / fmap indexing
        assert np.abs(r.cpu().numpy() - ref_r).max() <= REL * np.abs(ref_r).max() + 1e-6
        assert np.abs(gg.cpu().numpy() - ref_g).max() <= REL * np.abs(ref_g).max() + 1e-6
        for j, f in enumerate(fr[i]):
            assert tuple(f.shape) == tuple(g[f'{name}/fmap_r{i}_{j}_shape'])
            sub = f.cpu().numpy().reshape(-1)[::211]
            ref = g[f'{name}/fmap_r{i}_{j}_sub']
            assert np.abs(sub - ref).max() <= REL * np.abs(ref).max() + 1e-6, (i, j)
    np.testing.assert_allclose(losses, g[f'{name}/losses'], rtol=1e-4)


def test_multi_resolution_stft_loss_matches_reference_fixture(golden_dir):
    from neuralsvb_b200.modules.parallel_wavegan.losses.stft_loss import multi_resolution_stft_loss
    g = np.load(os.path.join(golden_dir, 'losses.npz'))
    y = S.make_wave_batch(2, 8192, seed=SEED)
    x = (y + 0.05 * S.make_wave_batch(2, 8192, seed=SEED + 1)).clamp(-1, 1)
    sc, mag = multi_resolution_stft_loss(x.cuda(), y.cuda())
    np.testing.assert_allclose([sc, mag], g['mr_stft/sc_mag'], rtol=1e-3)      # north star: 1e-3 on spectral features
    sc_o, mag_o = O.mr_stft_loss(x, y)
    np.testing.assert_allclose([sc, mag], [float(sc_o), float(mag_o)], rtol=1e-3)


def test_generic_conv_edge_cases_against_torch():
    """ragged / tiny shapes of the general conv: odd lengths, stride > 1, groups, W > 1, no bias."""
    import torch.nn.functional as F
    from neuralsvb_b200.modules.hifigan.discriminators import avg_pool_4_2_1, conv_nct
    g = torch.Generator().manual_seed(3)
    for (B, Cin, Cout, T, K, s, p, grp) in [(1, 1, 5, 17, 15, 1, 7, 1), (2, 8, 12, 101, 41, 4, 20, 4), (1, 6, 6, 9, 5, 2, 2, 3),
                                           (2, 3, 7, 64, 3, 1, 1, 1)]:
        x = torch.randn(B, Cin, T, generator=g)
        w = torch.randn(Cout, Cin // grp, K, generator=g) * 0.2
        b = torch.randn(Cout, generator=g)
        ref = F.leaky_relu(F.conv1d(x.double(), w.double(), b.double(), stride=s, padding=p, groups=grp), 0.1)
        got = conv_nct(x.cuda(), w.cuda(), b.cuda(), K, stride=s, pad=p, groups=grp, slope=0.1).cpu().double()
        assert got.shape == ref.shape and (got - ref).abs().max() < 1e-4 * ref.abs().max()
    x = torch.randn(2, 4, 30, 3, generator=g)                 # W = 3 inner columns, (5,1) kernel, stride (3,1)
    w = torch.randn(6, 4, 5, generator=g) * 0.2
    ref = F.conv2d(x.double(), w.double()[..., None], None, stride=(3, 1), padding=(2, 0))
    got = conv_nct(x.cuda(), w.cuda(), None, 5, stride=3, pad=2, W=3).cpu().double()
    assert got.shape == ref.shape and (got - ref).abs().max() < 1e-4 * ref.abs().max()
    x = torch.randn(2, 1, 33, generator=g)
    assert torch.allclose(avg_pool_4_2_1(x.cuda()).cpu(), F.avg_pool1d(x, 4, 2, padding=1), atol=1e-6)


@pytest.mark.parametrize('name', ['mpd', 'msd'])
def test_cond_discriminators_forward_and_backward(golden_dir, name):
    """use_cond=True: logits / losses against the reference fixture, parameter gradients (incl. cond_net) against
    torch autograd through the oracle."""
    from neuralsvb_b200.modules.hifigan import discriminators as D
    from neuralsvb_b200.utils.hparams import hparams
    hparams['hop_size'] = 256
    g = np.load(os.path.join(golden_dir, 'discriminators_cond.npz'))
    if name == 'mpd':
        m, sd, fwd = D.MultiPeriodDiscriminator(use_cond=True), S.make_mpd_state_dict(SEED, use_cond=True), O.mpd_forward
    else:
        m, sd, fwd = D.MultiScaleDiscriminator(use_cond=True), S.make_msd_state_dict(SEED, use_cond=True), O.msd_forward
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    y, y_hat = _signals()
    mel, _ = S.make_mel_f0(2, 32, SEED)
    with torch.no_grad():
        rs, gs, fr, fg = m(y.cuda(), y_hat.cuda(), mel.cuda())
        losses = [D.feature_loss(fr, fg), *D.discriminator_loss(rs, gs), D.generator_loss(gs), D.cond_discriminator_loss(gs)]
    np.testing.assert_allclose(losses, g[f'{name}/losses'], rtol=2e-4)
    for i, (r, gg) in enumerate(zip(rs, gs)):
        ref_r, ref_g = g[f'{name}/logit_r{i}'], g[f'{name}/logit_g{i}']
        assert np.abs(r.cpu().numpy() - ref_r).max() <= 5e-4 * np.abs(ref_r).max() + 1e-6
        assert np.abs(gg.cpu().numpy() - ref_g).max() <= 5e-4 * np.abs(ref_g).max() + 1e-6
    # gradients
    is_buf = lambda k: k.endswith('weight_u') or (k.endswith('weight_v') and k[:-1] + 'orig' in sd)
    p = {k: (v.clone() if is_buf(k) else v.clone().requires_grad_(True)) for k, v in sd.items()}
    rs, gs, fr, fg = fwd(y, y_hat, O.fold_discriminator_weights(p), mel=mel)
    dr, dg = O.discriminator_loss(rs, gs)
    (dr + dg + O.feature_loss(fr, fg)).backward()
    # fp32 kernels pin the logic; with the dense layers on split-bf16 tensor cores the cond_net weight gradient (a
    # correlation of the mel with an oscillating dy: heavy cancellation) amplifies their 1e-5 rounding to ~1e-2
    # (and a leaky-relu mask flipped by the forward's rounding moves one discriminator's gradient by ~1e-2: measured
    # fp32 errors 1.3e-4 on an unaffected discriminator, 8.7e-3 on an affected one)
    for use_tc, cond_tol in ((False, 3e-2), (True, 6e-2)):
        D.USE_TC = use_tc
        try:
            m.zero_grad()
            rs, gs, fr, fg = m(y.cuda(), y_hat.cuda(), mel.cuda())
            dr, dg = D.discriminator_loss(rs, gs)
            (dr + dg + D.feature_loss(fr, fg)).backward()
        finally:
            D.USE_TC = True
        errs = {k: float((q.grad.cpu().double() - p[k].grad.double()).norm() / p[k].grad.double().norm().clamp_min(1e-30))
                for k, q in m.named_parameters()}
        cond = {k: e for k, e in errs.items() if 'cond_net' in k}
        print(name, 'tc' if use_tc else 'fp32', 'cond_net grad errors', {k[15:]: f'{e:.1e}' for k, e in cond.items()})
        assert cond and max(cond.values()) < cond_tol and (use_tc or min(cond.values()) < 1e-3), cond
        assert float(np.median(list(errs.values()))) < 1e-2 and max(errs.values()) < 8e-2, sorted(errs.items(), key=lambda kv: -kv[1])[:4]


@pytest.mark.parametrize('T', [700, 2051])
@pytest.mark.parametrize('layer', range(1, 6))
def test_grouped_polyphase_tc_layers_match_torch(layer, T):
    """The grouped k = 41 layers of DiscriminatorS (hifigan.py:263-267) on wgmma in polyphase form
    (svb_tc_layer_create_grouped): forward, data / weight / bias gradients against torch fp64 grouped convolution."""
    import torch.nn.functional as F
    from neuralsvb_b200.modules.hifigan import discriminators as D
    cin, cout, k, s, g, p = S.MSD_LAYERS[layer]
    assert D.tc_eligible(cin, cout, k, s, 1, p, g)
    B = 2
    gen = torch.Generator().manual_seed(100 + layer)
    x = torch.randn(B, cin, T, generator=gen)
    w = torch.randn(cout, cin // g, k, generator=gen) * (1.0 / (cin // g * k) ** 0.5)
    b = torch.randn(cout, generator=gen) * 0.1
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, w, b))
    ref_lin = F.conv1d(xr, wr, br, stride=s, padding=p, groups=g)
    ref = F.leaky_relu(ref_lin, 0.1)
    cot = torch.randn(ref.shape, generator=gen)
    xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
    got = D.conv_tc(xc, wc, bc, D.TcLayer(), k, s, p, 0.1, 1, g)
    assert got.shape == ref.shape
    rel = lambda a, r: float((a.detach().cpu().double() - r.detach()).norm() / r.detach().norm())
    assert rel(got, ref) < 2e-5, rel(got, ref)
    (got * cot.cuda()).sum().backward()
    # leaky-relu's derivative is discontinuous at 0: with ~10^6 outputs a few pre-activations within the forward's 1e-6
    # of zero flip their mask and each flip moves the gradients by ~1e-3 relative.  The reference therefore applies the
    # mask of the CUDA forward itself -- what is compared is the convolution's data / weight / bias gradient.
    mask = torch.where(got.detach().cpu() > 0, 1.0, 0.1).double()
    flips = int((mask != torch.where(ref.detach() > 0, 1.0, 0.1)).sum())
    assert flips <= 1e-4 * mask.numel(), flips
    (ref_lin * (cot.double() * mask)).sum().backward()
    e = {'dx': rel(xc.grad, xr.grad), 'dw': rel(wc.grad, wr.grad), 'db': rel(bc.grad, br.grad)}
    assert max(e.values()) < 1e-4, e
    # and the fp32 CUDA-core kernel agrees (the path USE_TC_GROUPED = False takes)
    got32 = D.conv_nct(x.cuda(), w.cuda(), b.cuda(), k, stride=s, pad=p, groups=g, slope=0.1)
    assert rel(got32, ref) < 2e-5


# the dense MPD layers on wgmma (k5 s3 p2: tap-major expansion, wgrad_tc with K = 1, col2im; k5 s1 p2: the generator's
# kernel as is) with the input lengths a 600-sample column gives along the stack
DENSE_TC_LAYERS = [(32, 128, 5, 3, 2, 600), (128, 512, 5, 3, 2, 200), (512, 1024, 5, 3, 2, 67), (1024, 1024, 5, 1, 2, 23)]


@pytest.mark.parametrize('W', [1, 2, 3, 5, 7, 11, 13])          # 13 > the 11 period columns of one output tile: W slices
@pytest.mark.parametrize('layer', range(len(DENSE_TC_LAYERS)))
def test_dense_tc_layers_match_torch(layer, W):
    """The dense (groups = 1) discriminator layers through svb_tc_layer_create: forward, data / weight / bias gradients
    against torch fp64 F.conv2d with a (K, 1) kernel over W period columns (F.conv1d for W = 1)."""
    import torch.nn.functional as F
    from neuralsvb_b200.modules.hifigan import discriminators as D
    cin, cout, k, s, p, T = DENSE_TC_LAYERS[layer]
    assert D.tc_eligible(cin, cout, k, s, 1, p, 1)
    B = 2
    gen = torch.Generator().manual_seed(200 + 10 * layer + W)
    x = torch.randn((B, cin, T) + ((W,) if W > 1 else ()), generator=gen)
    w = torch.randn(cout, cin, k, generator=gen) * (1.0 / (cin * k) ** 0.5)
    b = torch.randn(cout, generator=gen) * 0.1
    xr, wr, br = (t.double().cuda().requires_grad_(True) for t in (x, w, b))
    if W > 1:
        ref_lin = F.conv2d(xr, wr[..., None], br, stride=(s, 1), padding=(p, 0))
    else:
        ref_lin = F.conv1d(xr, wr, br, stride=s, padding=p)
    ref = F.leaky_relu(ref_lin, 0.1)
    cot = torch.randn(ref.shape, generator=gen).cuda()
    xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
    got = D.conv_tc(xc, wc, bc, D.TcLayer(), k, s, p, 0.1, W, 1)
    assert got.shape == ref.shape
    rel = lambda a, r: (float((a.detach().double() - r.detach()).norm() / r.detach().norm()),
                        float((a.detach().double() - r.detach()).abs().max() / r.detach().abs().max()))
    e_y = rel(got, ref)
    (got * cot).sum().backward()
    # the reference takes the leaky-relu mask of the CUDA forward (see test_grouped_polyphase_tc_layers_match_torch)
    mask = torch.where(got.detach() > 0, 1.0, 0.1).double()
    flips = int((mask != torch.where(ref.detach() > 0, 1.0, 0.1)).sum())
    assert flips <= 1e-4 * mask.numel(), flips
    (ref_lin * (cot.double() * mask)).sum().backward()
    e = {'y': e_y, 'dx': rel(xc.grad, xr.grad), 'dw': rel(wc.grad, wr.grad), 'db': rel(bc.grad, br.grad)}
    print('MEASURED', DENSE_TC_LAYERS[layer], W, {n: f'{a:.2e}/{b:.2e}' for n, (a, b) in e.items()})
    bad = {n: v for n, v in e.items() if v[0] > DENSE_TOL[n][0] or v[1] > DENSE_TOL[n][1]}
    assert not bad, f'{DENSE_TC_LAYERS[layer]} W {W}: (rel L2, rel L-inf) {bad}'


# (relative L2, relative L-inf) per tensor, split-bf16 on wgmma (bf16x3, the discriminators' mode): about 5x the worst
# measured on an H100 80GB HBM3 (400 W power limit) -- y 1.7e-5 / 2.2e-5 and dx 1.8e-5 / 2.1e-5 (both on the 1024 -> 1024
# layer: 5120 products per output), dw 4.1e-6 / 5.2e-6, db 1.5e-7 / 1.9e-7
DENSE_TOL = {'y': (9e-5, 1.1e-4), 'dx': (9e-5, 1.1e-4), 'dw': (2.5e-5, 3e-5), 'db': (1e-6, 1e-6)}

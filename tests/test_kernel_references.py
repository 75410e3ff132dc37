"""CPU: the float64 references of the kernel-level GPU tests (tests/test_gpu_stft_kernels.py, test_gpu_disc_kernels.py,
test_gpu_acoustic_kernels.py, test_gpu_generator_backward.py) against the oracle (oracle/hifigan.py, oracle/frontend.py,
oracle/vc_asr.py), which is pinned to the reference fixtures.  A wrong reference
would let a wrong kernel pass its test; here it fails without a GPU."""
import os

import numpy as np
import torch
import torch.nn.functional as F

from neuralsvb_b200.utils import synthetic as S
from oracle import frontend as FE
from oracle import hifigan as O
from oracle import vc_asr as OV
from tests import test_gpu_acoustic_kernels as A
from tests import test_gpu_disc_kernels as D
from tests import test_gpu_generator_backward as G
from tests import test_gpu_stft_kernels as T


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


def test_stft_reference_matches_the_oracle_mel_spectrogram_stft_and_wav2spec():
    hp = S.hifigan_config()
    y = T.make_wave(2, 8192, 'oracle', 'loud')                # clamp_input matters: samples beyond +-1
    # mel loss: clamp, half reflect pad, hann(win), sqrt(|X|^2 + 1e-9), fmin 80 / fmax 7600 basis, ln(clamp(1e-5))
    cfg = (hp['fft_size'], hp['hop_size'], hp['win_size'], T.HALF, T.LN_MEL, 1, 80, 0, 1e-5)
    ref, _ = T.stft_reference(y, cfg, T.make_basis('loss80', hp['fft_size'], 80))
    assert _rel(ref, O.mel_spectrogram(y, hp)) < 1e-5
    # MR-STFT magnitude: torch.stft defaults (centre, reflect), sqrt(clamp(|X|^2, 1e-7)), frames-major
    x = T.make_wave(2, 8192, 'oracle-mag')
    ref, _ = T.stft_reference(x, (1024, 120, 600, T.REFLECT, T.MAG, 0, 0, 1, 1e-7), None)
    assert _rel(ref, O.stft_mag(x, 1024, 120, 600)) < 1e-5
    # wav2spec: librosa.stft(centre, zero pad) -> |.| -> mel -> log10(max(eps, .))
    cfg = (hp['fft_size'], hp['hop_size'], hp['win_size'], T.ZERO, T.LOG10_MEL, 0, 80, 1, 1e-10)
    ref, _ = T.stft_reference(x[:1], cfg, T.make_basis('loss80', hp['fft_size'], 80))
    _, mel = FE.wav2spec(x[0].numpy(), hp)
    assert _rel(ref[0], mel) < 1e-5


def test_cond_net_reference_matches_the_oracle():
    g = torch.Generator().manual_seed(5)
    t = 128
    mel = torch.randn(2, 80, 7, generator=g, dtype=torch.float64)
    x = torch.randn(2, 1, 7 * t, generator=g, dtype=torch.float64)
    w = {'d.cond_net.weight': torch.randn(80, 1, 2 * t, generator=g, dtype=torch.float64),
         'd.cond_net.bias': torch.randn(1, generator=g, dtype=torch.float64)}
    ref = D.cond_net_reference(mel, w['d.cond_net.weight'], w['d.cond_net.bias'], t)
    assert torch.equal(O._cond(x, w, 'd', mel)[:, :1], ref)


def _grad(f, a):
    a = a.clone().requires_grad_(True)
    f(a).backward()
    return a.grad


def test_loss_gradient_references_match_the_oracle_losses(monkeypatch):
    """Each svb_loss_grad kind, at the scale its call site passes, is the gradient of the oracle loss it replaces."""
    g = torch.Generator().manual_seed(9)
    n = 1000
    a = torch.exp(torch.randn(n, generator=g, dtype=torch.float64))
    b = torch.exp(torch.randn(n, generator=g, dtype=torch.float64))
    b[::7] = a[::7]                                            # ties: sign(0) = 0 on both sides
    kind = lambda k, scale, b_=b: _grad(lambda t: D.loss_expr(k, t, b_, scale), a)
    # feature_loss (2 * mean |r - g|, w.r.t. g), generator_loss, discriminator_loss (real / generated terms)
    assert _rel(kind(0, 2 / n), _grad(lambda t: O.feature_loss([[b]], [[t]]), a)) < 1e-12
    assert _rel(kind(1, 2 / n), _grad(lambda t: O.generator_loss([t]), a)) < 1e-12
    assert _rel(kind(1, 2 / n), _grad(lambda t: O.discriminator_loss([t], [b])[0], a)) < 1e-12
    assert _rel(kind(2, 2 / n), _grad(lambda t: O.discriminator_loss([b], [t])[1], a)) < 1e-12
    # the STFT losses on given magnitudes: spectral convergence (kind 3) and log-magnitude L1 (kind 4), w.r.t. the prediction
    monkeypatch.setattr(O, 'stft_mag', lambda x, *args: x)
    sc_scale = float(1 / ((b - a).norm() * b.norm()))
    assert _rel(kind(3, sc_scale), _grad(lambda t: O.stft_loss(t, b, 0, 0, 0)[0], a)) < 1e-12
    assert _rel(kind(4, 1 / n), _grad(lambda t: O.stft_loss(t, b, 0, 0, 0)[1], a)) < 1e-12
    assert (kind(4, 1 / n)[::7] == 0).all() and (kind(0, 1.0)[::7] == 0).all()


def _rel_shift(x):
    """espnet's rel_shift as written: prepend a zero column, view [T, T + 1] as [T + 1, T], drop the first row."""
    *lead, T, _ = x.shape
    padded = torch.cat([x.new_zeros(*lead, T, 1), x], -1).view(*lead, T + 1, T)
    return padded[..., 1:, :].reshape(x.shape)


def test_shifted_bd_is_rel_shift():
    for T in (1, 2, 3, 8):
        x = torch.randn(2, 3, T, T, generator=torch.Generator().manual_seed(T), dtype=torch.float64)
        assert torch.equal(OV.shifted_bd(x), _rel_shift(x)), T


def test_attention_reference_matches_the_oracle_attention():
    """The float64 attention core of test_gpu_acoustic_kernels on the fixture's weights and shape (B 2, T' 48, the shorter
    clip's last 4 keys masked), against oracle.vc_asr.attention in fp32 with linear_out set to the identity."""
    B, T, H, nh = 2, 48, 256, 4
    pre = 'content_encoder.encoder_layers.0.self_attn'
    w = {k: v for k, v in S.make_vc_asr_state_dict(1234).items() if k.startswith(pre)}
    w[pre + '.linear_out.weight'], w[pre + '.linear_out.bias'] = torch.eye(H), torch.zeros(H)
    x = torch.randn(B, T, H, generator=torch.Generator().manual_seed(11))
    mask = torch.ones(B, T, dtype=torch.bool)
    mask[1, T - 4:] = False
    pos = OV.rel_positions(T, H)
    with torch.no_grad():
        ctx = OV.attention(w, pre, x, pos, mask, nh)
        q, k, v = (F.linear(x, w[f'{pre}.linear_{n}.weight'], w[f'{pre}.linear_{n}.bias']).transpose(1, 2).contiguous() for n in 'qkv')
        p = F.linear(pos, w[pre + '.linear_pos.weight']).t().contiguous()
        ref = A.attention_reference(q, k, v, p, w[pre + '.pos_bias_u'], w[pre + '.pos_bias_v'], mask.float(), nh)
    assert ref.dtype == torch.float64
    assert _rel(ref.transpose(1, 2), ctx) < 1e-5


def test_vc_asr_oracle_runs_in_float64_and_matches_the_fixture():
    """The float64 PPG-extractor reference of test_gpu_acoustic_kernels is the oracle run on double weights and mel."""
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'vc_asr.npz'))
    B, T = [int(v) for v in g['params']]
    w = {k: v.double() for k, v in S.make_vc_asr_state_dict(1234).items()}
    with torch.no_grad():
        h = OV.vc_asr_h_content(w, S.make_vc_asr_mel(B, T, 1234).double())
    assert h.dtype == torch.float64
    assert _rel(h, g['h_content']) < 1e-5


def test_masked_generator_reference_with_its_own_masks_is_autograd():
    """test_gpu_generator_backward's reference (leaky relus at given masks, NSF sines passed in) fed the masks of its own
    pre-activations is plain float64 autograd through the oracle: the same waveform and every gradient to 1e-12."""
    h = S.small_config(True)
    B, T, hop = 2, 24, 16
    sd = S.make_generator_state_dict(h, 1234)
    mel, f0 = (t.double() for t in S.make_mel_f0(B, T, 1234))
    ri, nz = (t.double() for t in S.make_nsf_noise(B, T * hop, 1234))
    cot = torch.randn(B, 1, T * hop, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    pre = {}

    def record(site, x, slope):
        assert site not in pre, site
        pre[site] = x.detach()
        return F.leaky_relu(x, slope)
    p = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    y = O.generator_forward(O.fold_weight_norm(p), h, mel, f0, ri, nz, act=record)
    (y * cot).sum().backward()
    nk, nd, n_ups = len(h['resblock_kernel_sizes']), len(h['resblock_dilation_sizes'][0]), len(h['upsample_rates'])
    assert len(pre) == 1 + n_ups + n_ups * nk * nd * 2
    with torch.no_grad():
        assert torch.equal(y, O.generator_forward(O.fold_weight_norm(p), h, mel, f0, ri, nz))
    y_m, _, g_m, _ = G.reference(h, sd, mel, f0, G.nsf_sines(h, f0, ri, nz), cot, G.masked_act(pre.__getitem__))
    assert _rel(y_m, y.detach()) < 1e-12
    assert set(g_m) == set(p)
    for k, t in p.items():
        assert _rel(g_m[k], t.grad) < 1e-12, k


def test_generator_launch_group_references_chain_to_the_oracle_taps():
    """test_gpu_generator_forward's per-launch-group references (O.upsample_forward, O.stage_forward, O.post_forward)
    fed the float32 oracle's own taps give back each next tap and the waveform: ``ups{i}`` is the upsampler of
    ``conv_pre`` / ``stage{i-1}`` with the noise conv of ``har_source`` added, ``stage{i}`` the ResBlock mean of
    ``ups{i}``."""
    for h, T in ((S.small_config(True), 24), (S.hifigan_config(True), 3), (S.hifigan_config(False), 3)):
        hop = int(np.prod(h['upsample_rates']))
        B = 2
        w = O.fold_weight_norm(S.make_generator_state_dict(h, 1234))
        mel, f0 = S.make_mel_f0(B, T, 1234)
        ri, nz = S.make_nsf_noise(B, T * hop, 1234)
        nsf = h['use_pitch_embed']
        taps = {}
        with torch.no_grad():
            y = O.generator_forward(w, h, mel, f0 if nsf else None, ri, nz, taps)
            har = taps.get('har_source')
            assert (har is not None) == nsf
            n = len(h['upsample_rates'])
            assert set(taps) == {'conv_pre', *(f'ups{i}' for i in range(n)), *(f'stage{i}' for i in range(n))} | (
                {'har_source'} if nsf else set())
            for i in range(n):
                x = taps['conv_pre' if i == 0 else f'stage{i - 1}']
                assert torch.equal(O.upsample_forward(w, h, i, x, har), taps[f'ups{i}']), (h['hop_size'], i)
                assert torch.equal(O.stage_forward(w, h, i, taps[f'ups{i}']), taps[f'stage{i}']), (h['hop_size'], i)
                if nsf:     # the noise conv is part of ups{i}: without it the tap is not reproduced
                    assert not torch.allclose(O.upsample_forward(w, h, i, x, None), taps[f'ups{i}'])
            assert torch.equal(O.post_forward(w, h, taps[f'stage{n - 1}']), y)
            assert y.shape == (B, 1, T * hop)

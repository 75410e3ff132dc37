"""MleSVBVAE training on the native kernels against float64 torch: the fused mel-loss kernel (values and d mel_out), the phase-2
generator step and the phase-3 mapping step through the train-mode oracle (oracle/svb_vae_train.py, oracle/mel_loss.py), the eval-mode
decoder the mapping step differentiates through, and three AdamW steps on one set of native handles.  Errors are relative L2 and
L-inf relative to max |reference|."""
import numpy as np
import pytest
import torch

from neuralsvb_b200.utils import synthetic as S
from tests.test_gpu_wn_train import _check, _cot, _decoder_reference, _decoder_setup, _make_decoder
from tests.test_oracle_golden import SVB_HP

pytestmark = pytest.mark.gpu
# (rel L2, rel L-inf) bars, about 5x the worst error measured on an H100 80GB HBM3 (see DESIGN section 8 for the run)
MEL_VALUE_BAR = 2.5e-5             # worst l1 3.2e-8, ssim 4.4e-6 (T = 1)
MEL_GRAD_BARS = (2.7e-6, 1.2e-5)   # worst 5.3e-7 / 2.4e-6
# The steps run B = 2 clips with random weights, so the train-mode BatchNorms (upsample_layer after a ReLU, the latent map over two
# [128, 1] latents) amplify rounding.  Worst measured, H100 80GB HBM3 at a 400 W power limit:
#   phase 2, every dense convolution on the fp32 CUDA cores (vc_modules.USE_TC = False, WN stacks fp32): 3.4e-5 / 4.1e-5;
#   phase 2 on the default bf16x3 tensor-core convolutions (about 5e-6 each, test_gpu_acoustic_kernels.py): 1.0e-2 / 3.4e-2, on
#     upsample_layer.0.1 (the BatchNorm after its ReLU divides by small batch deviations); every other tensor 3.4e-3 / 7.5e-3 or less;
#   phase 3 (BatchNorm over two latents): 1.0e-3 / 1.0e-3 on the CUDA cores, 8.9e-3 / 8.9e-3 on the tensor cores -- float32 torch
#     on the CPU is 5.4e-4 off there too (tests/test_svb_vae_train_host.py);
#   loss values 7.7e-6, running statistics 2.7e-5.
# Errors of a tensor whose reference gradient is (nearly) zero -- the biases in front of a BatchNorm -- are taken relative to 1e-3
# of the step's largest gradient.
STEP_BARS = {False: (1.7e-4, 2e-4), True: (5e-2, 1.7e-1)}          # keyed by USE_TC
MAP_BARS = {False: (5e-3, 1e-2), True: (4.5e-2, 4.5e-2)}
RUNNING = ['upsample_layer.0.3', 'vae_model.encoder.poolings.2', 'vae_model.encoder.poolings.5']
MAP_RUNNING = ['z_mapping_function.convs.1', 'z_mapping_function.convs.4']


# ---------------------------------------------------------------------------------------------------------- mel loss
def _pads(B, T):
    """Trailing padding per clip: none on clip 0, an all-padding clip 1 when B > 2, ragged tails elsewhere."""
    return [0 if b == 0 else (T if b == 1 and B > 2 else (7 * b) % T) for b in range(B)]


@pytest.mark.parametrize('T', [1, 5, 11, 12, 37, 1000, 1024, 1031])
@pytest.mark.parametrize('B', [1, 3, 16])
def test_mel_loss_kernel_matches_float64(B, T):
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    from oracle import mel_loss as OM
    mel_out, target = S.make_mel_pair(B, T, _pads(B, T), 1234 + T)
    g1, g2 = 0.7, -1.3                                              # upstream gradients != 1, read by the kernel from the device
    x64 = mel_out.cuda().double().requires_grad_(True)
    l1_r, ss_r = OM.mel_l1_ssim_loss(x64, target.cuda().double())
    (g1 * l1_r + g2 * ss_r).backward()
    x = mel_out.cuda().requires_grad_(True)
    l1, ss = mel_l1_ssim_loss(x, target.cuda())
    assert l1.dtype == torch.float32 and l1.is_cuda and l1.dim() == 0
    torch.autograd.backward([l1, ss], [torch.tensor(g1, device='cuda'), torch.tensor(g2, device='cuda')])
    for tag, got, ref in (('l1', l1, l1_r), ('ssim', ss, ss_r)):
        err = abs(float(got) - float(ref)) / abs(float(ref))
        print(f'ERR mel B{B} T{T} {tag} {err:.2e}')
        assert err < MEL_VALUE_BAR, (tag, err)
    _check(f'mel B{B} T{T} dmel', x.grad, x64.grad, MEL_GRAD_BARS)


def test_mel_loss_all_padding_batch_is_nan():
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    mel_out, target = S.make_mel_pair(2, 20, [20, 20], 1234)
    l1, ss = mel_l1_ssim_loss(mel_out.cuda(), target.cuda())
    assert bool(torch.isnan(l1)) and bool(torch.isnan(ss))


# ---------------------------------------------------------------------------------------------------------- model steps
def _model(precision):
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    m = MleSVBVAE(80, hp=SVB_HP, precision=precision, trainable=True)
    m.load_state_dict(S.make_svb_state_dict(1234), strict=True)
    return m.cuda()


def _set_phase(m, phase):
    """requires_grad as the trainer leaves it for the phase's optimizer, train / eval flags as SVBVAEMleTask sets them."""
    for n, p in m.named_parameters():
        p.requires_grad_(n.startswith('z_mapping_function.') if phase == 3 else not n.startswith(('vc_asr.', 'z_mapping_function.')))
    if phase == 2:
        m.train()
        m.z_mapping_function.eval()
    else:
        m.eval()
        m.z_mapping_function.train()
    m.vc_asr.eval()


def _batch():
    return S.make_svb_batch(2, 96, 120, 1234)


def _native_step(m, phase, batch):
    """The step's loss (the task's terms without the adversarial ones) and its backward."""
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    ways = ['a2a', 'p2p'] if phase == 2 else ['a2a', 'p2p', 'a2p']
    b = {k: v.cuda() for k, v in batch.items()}
    ret = m(**b, concurrent_ways=ways, eps=torch.zeros(2, 128, 1, device='cuda'))
    targets = {'a2a': b['amateur_mel'], 'p2p': b['prof_mel'], 'a2p': b['prof_mel']}
    losses = {}
    for way in ways:
        if 'kl' in ret[way]:
            losses[f'{way}_kl'] = ret[way]['kl'] * 0.001
        l1, ss = mel_l1_ssim_loss(ret[way]['mel_out'], targets[way])
        losses[f'l1{way}'], losses[f'ssim{way}'] = 0.5 * l1, 0.5 * ss
    if phase == 3:
        losses['a2p_mle'] = ret['a2p']['mle'] * 1.0
    sum(losses.values()).backward()
    return losses


def _oracle_step(m, phase, batch):
    """float64 autograd through the train-mode oracle at the module's current parameters and running statistics (updated in place)."""
    from oracle import svb_vae_train as O
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    req = {n for n, p in m.named_parameters() if p.requires_grad}
    p = {k: (v.double().clone().requires_grad_(k in req) if v.is_floating_point() else v.clone()) for k, v in sd.items()}
    b = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in batch.items()}
    losses, _ = O.svb_train_losses(p, b, torch.zeros(2, 128, 1, device='cuda', dtype=torch.float64), phase)
    sum(losses.values()).backward()
    return losses, p


def _compare_step(tag, m, phase, losses, ref_losses, p, bars):
    assert sorted(losses) == sorted(ref_losses)
    for k in losses:
        _check(f'{tag} loss {k}', losses[k].detach().reshape(1), ref_losses[k].detach().reshape(1), bars)
    req = [(name, q) for name, q in m.named_parameters() if q.requires_grad]
    floor = 1e-3 * max(float(p[name].grad.norm()) for name, _ in req)
    for name, q in m.named_parameters():
        if not q.requires_grad:
            assert q.grad is None, name
    for name, q in req:
        ref = p[name].grad.detach().double()
        d = q.grad.detach().double() - ref
        l2 = float(d.norm()) / max(float(ref.norm()), floor)
        li = float(d.abs().max()) / max(float(ref.abs().max()), floor / ref.numel() ** 0.5)
        print(f'ERR {tag} d{name} {l2:.2e} {li:.2e}')
        assert l2 < bars[0] and li < bars[1], (tag, name, l2, li, bars)
    return len(req)


@pytest.fixture(params=[False, True], ids=['fp32_cuda_cores', 'bf16x3_tensor_cores'])
def use_tc(request, monkeypatch):
    from neuralsvb_b200.modules.voice_conversion import vc_modules as V
    monkeypatch.setattr(V, 'USE_TC', request.param)
    return request.param


def test_phase2_generator_step_matches_float64(use_tc):
    precision = 'bf16x3' if use_tc else 'fp32'
    m = _model(precision)
    _set_phase(m, 2)
    batch = _batch()
    before = {k: int(v) for k, v in m.state_dict().items() if k.endswith('num_batches_tracked')}
    ref_losses, p = _oracle_step(m, 2, batch)
    losses = _native_step(m, 2, batch)
    n = _compare_step(f'phase2 {precision}', m, 2, losses, ref_losses, p, STEP_BARS[use_tc])
    assert n > 100
    assert bool((m.pitch_embed.weight.grad[0] == 0).all())
    assert all(q.grad is None for q in m.vc_asr.parameters())
    sd = m.state_dict()
    for pre in RUNNING:
        for s in ('running_mean', 'running_var'):
            _check(f'phase2 {precision} {pre}.{s}', sd[f'{pre}.{s}'], p[f'{pre}.{s}'], STEP_BARS[use_tc])
        assert int(sd[f'{pre}.num_batches_tracked']) == before[f'{pre}.num_batches_tracked'] + 2      # amateur + professional calls


def test_phase3_mapping_step_matches_float64(use_tc):
    m = _model('bf16x3' if use_tc else 'fp32')
    _set_phase(m, 3)
    batch = _batch()
    ref_losses, p = _oracle_step(m, 3, batch)
    frozen = {k: v.clone() for k, v in m.state_dict().items() if 'running' in k and not k.startswith('z_mapping_function.')}
    losses = _native_step(m, 3, batch)
    n = _compare_step('phase3', m, 3, losses, ref_losses, p, MAP_BARS[use_tc])
    assert n == len(list(m.z_mapping_function.parameters()))
    sd = m.state_dict()
    for pre in MAP_RUNNING:
        for s in ('running_mean', 'running_var'):
            _check(f'phase3 {pre}.{s}', sd[f'{pre}.{s}'], p[f'{pre}.{s}'], MAP_BARS[use_tc])
    for k, v in frozen.items():                                    # eval-mode BatchNorms keep their statistics
        assert torch.equal(sd[k], v), k


def test_eval_mode_decoder_is_differentiable_and_unchanged():
    cfg, sd, z, mask, cond = _decoder_setup('global_dec')
    lat, H, oc, K, L, gin, B, T, glob = cfg
    m = _make_decoder(cfg, sd, 'bf16x3').eval()
    for q in m.parameters():
        q.requires_grad_(False)
    with torch.no_grad():
        y_ref = m(z.cuda(), mask.cuda(), cond.cuda())
    zc = z.cuda().requires_grad_(True)
    y = m(zc, mask.cuda(), cond.cuda())
    assert y.requires_grad and torch.equal(y.detach(), y_ref)
    cot = _cot((B, oc, T), 11)
    (y * cot.cuda()).sum().backward()
    _, zd, _, _ = _decoder_reference(cfg, sd, z, mask, cond, cot)
    _check('eval decoder dz', zc.grad, zd.grad, (8e-5, 8e-5))          # worst 1.6e-5 / 1.6e-5
    assert all(q.grad is None for q in m.parameters())


def test_three_adamw_phase2_steps(use_tc):
    """Each step's gradients match float64 at the current parameters; the WN and decoder handles are the ones built first."""
    precision = 'bf16x3' if use_tc else 'fp32'
    m = _model(precision)
    _set_phase(m, 2)
    opt = torch.optim.AdamW([q for q in m.parameters() if q.requires_grad], lr=1e-3)
    batch = _batch()
    stacks = [m.vae_model.encoder.wn, m.vae_model.decoder]
    handles = None
    for step in range(3):
        opt.zero_grad()
        ref_losses, p = _oracle_step(m, 2, batch)
        # the oracle updated ITS copy of the running statistics; the native step updates the module's
        losses = _native_step(m, 2, batch)
        handles = handles or [s._handle.value for s in stacks]
        assert [s._handle.value for s in stacks] == handles and all(s.host_uploads == 1 for s in stacks)
        _compare_step(f'adamw {precision} step {step}', m, 2, losses, ref_losses, p, STEP_BARS[use_tc])
        opt.step()

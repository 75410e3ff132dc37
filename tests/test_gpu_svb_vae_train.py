"""MleSVBVAE training on the native kernels against float64 torch: the fused mel-loss kernel (values and d mel_out), the phase-2
generator step and the phase-3 mapping step through the train-mode oracle (oracle/svb_vae_train.py, oracle/mel_loss.py), the eval-mode
decoder the mapping step differentiates through, and three AdamW steps on one set of native handles.  Errors are relative L2 and
L-inf relative to max |reference|."""
import contextlib

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
# The steps run B = 2 clips with random weights; the float64 reference runs on the native PPG, train-mode BatchNorm inputs and ReLU
# masks (_tied_step).  Without them, the BatchNorms over two clips amplified the bf16x3 rounding to 1.0e-2 / 3.4e-2 (phase 2) and
# 8.9e-3 (phase 3), and a pre-activation rounding across zero moved single gradients by up to 7.5e-2, differently from run to run.
# Worst over three runs on an H100 80GB HBM3 (400 W power limit), this file and the adversarial steps of test_gpu_mel_disc.py
# together, gradients / loss values:
#   phase 2 fp32 (vc_modules.USE_TC = False, WN stacks fp32): 4.2e-6 / 1.2e-5 and 2.7e-7;
#   phase 2 bf16x3: 3.9e-5 / 6.6e-5 (the posterior encoder) and 5.6e-6;
#   phase 3: 3.8e-5 / 3.8e-5 (either precision; 1.8e-5 fp32, 5.5e-5 bf16x3 with the adversarial term) and 1.2e-6 fp32, 1.4e-5 bf16x3;
#   running statistics 1.6e-7.
# The biases in front of a train-mode BatchNorm have an exact gradient of 0 (MAP_ZERO_GRAD, _compare_step's zero_grad).
STEP_BARS = {False: {None: (2.1e-5, 6e-5), 'loss': (1.4e-6, 1.4e-6)}, True: {None: (2e-4, 3.3e-4), 'loss': (2.8e-5, 2.8e-5)}}   # keyed by USE_TC
MAP_BARS = {False: {None: (2e-4, 2e-4), 'loss': (6e-6, 6e-6)}, True: {None: (2.8e-4, 2.8e-4), 'loss': (7e-5, 7e-5)}}
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


def _native_step(m, phase, batch, extra=None):
    """The step's loss (the task's terms without the adversarial ones, plus ``extra(ret)`` when given) and its backward."""
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    ways = ['a2a', 'p2p'] if phase == 2 else ['a2a', 'p2p', 'a2p']
    b = {k: v.cuda() for k, v in batch.items()}
    ret = m(**b, concurrent_ways=ways, eps=torch.zeros(b['amateur_mel'].shape[0], 128, 1, device='cuda'))
    targets = {'a2a': b['amateur_mel'], 'p2p': b['prof_mel'], 'a2p': b['prof_mel']}
    losses = {}
    for way in ways:
        if 'kl' in ret[way]:
            losses[f'{way}_kl'] = ret[way]['kl'] * 0.001
        l1, ss = mel_l1_ssim_loss(ret[way]['mel_out'], targets[way])
        losses[f'l1{way}'], losses[f'ssim{way}'] = 0.5 * l1, 0.5 * ss
    if phase == 3:
        losses['a2p_mle'] = ret['a2p']['mle'] * 1.0
    if extra is not None:
        losses.update(extra(ret))
    sum(losses.values()).backward()
    return losses


def _oracle_step(m, phase, batch, sd=None, ppg=None, tie=None, relu=None, extra=None):
    """float64 autograd through the train-mode oracle at the module's current parameters and running statistics (updated in place),
    or at ``sd`` (a state_dict taken before the native step).  ``ppg`` / ``tie`` / ``relu``: see oracle/svb_vae_train.py; ``extra(out)`` adds
    loss terms."""
    from oracle import svb_vae_train as O
    sd = {k: v.detach() for k, v in (sd or m.state_dict()).items()}
    req = {n for n, p in m.named_parameters() if p.requires_grad}
    p = {k: (v.double().clone().requires_grad_(k in req) if v.is_floating_point() else v.clone()) for k, v in sd.items()}
    b = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in batch.items()}
    eps = torch.zeros(b['amateur_mel'].shape[0], 128, 1, device='cuda', dtype=torch.float64)
    losses, out = O.svb_train_losses(p, b, eps, phase, ppg=ppg, tie=tie, relu=relu)
    if extra is not None:
        losses.update(extra(out))
    sum(losses.values()).backward()
    return losses, p


def _bar(bars, name):
    return bars.get(name, bars[None]) if isinstance(bars, dict) else bars


def _compare_step(tag, m, phase, losses, ref_losses, p, bars, zero_grad=()):
    """Loss values and every trainable gradient against float64.  ``bars``: (rel L2, rel L-inf), or {'loss': bars of the loss values,
    None: bars of the gradients}.  ``zero_grad``: parameters whose exact gradient is 0 (a bias straight in front of a train-mode BatchNorm): both
    sides must stay below 1e-4 of the step's largest gradient, and they are left out of the relative comparison."""
    assert sorted(losses) == sorted(ref_losses)
    bar = (lambda name: _bar(bars, name))
    for k in losses:
        _check(f'{tag} loss {k}', losses[k].detach().reshape(1), ref_losses[k].detach().reshape(1), bar('loss'))
    for name, q in m.named_parameters():
        if not q.requires_grad:
            assert q.grad is None, name
    req = [(name, q) for name, q in m.named_parameters() if q.requires_grad]
    big = max(float(q.grad.abs().max()) for _, q in req)
    for name in zero_grad:
        got, want = float(m.get_parameter(name).grad.abs().max()), float(p[name].grad.abs().max())
        print(f'ERR {tag} d{name} |native| {got / big:.2e} |float64| {want / big:.2e} of the largest gradient')
        assert got < 1e-4 * big and want < 1e-4 * big, (tag, name, got / big, want / big)
    req = [(name, q) for name, q in req if name not in zero_grad]
    floor = 1e-3 * max(float(p[name].grad.norm()) for name, _ in req)
    for name, q in req:
        ref = p[name].grad.detach().double()
        d = q.grad.detach().double() - ref
        l2 = float(d.norm()) / max(float(ref.norm()), floor)
        li = float(d.abs().max()) / max(float(ref.abs().max()), floor / ref.numel() ** 0.5)
        print(f'ERR {tag} d{name} {l2:.2e} {li:.2e}')
        assert l2 < bar(name)[0] and li < bar(name)[1], (tag, name, l2, li, bar(name))
    return len(req) + len(zero_grad)


@contextlib.contextmanager
def _recorded(m):
    """Record what the native forward computed, per module name in call order: the PPG extractor's outputs (amateur, then
    professional), the input and output of every BatchNorm1d that runs as a module call (i.e. in train mode) and the output of every
    GroupNorm (the pitch encoder's, each followed by a ReLU)."""
    rec = {'ppg': [], 'bn': {}, 'bn_out': {}, 'gn': {}}

    def keep(key, name):
        return lambda mod, inp, out=None: rec[key].setdefault(name, []).append((inp[0] if out is None else out).detach().clone())
    hooks = [m.vc_asr.register_forward_hook(lambda mod, inp, out: rec['ppg'].append(out['h_content'].detach().clone()))]
    for name, mod in m.named_modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            hooks += [mod.register_forward_pre_hook(keep('bn', name)), mod.register_forward_hook(keep('bn_out', name))]
        elif isinstance(mod, torch.nn.GroupNorm):
            hooks.append(mod.register_forward_hook(keep('gn', name)))
    try:
        yield rec
    finally:
        for h in hooks:
            h.remove()


def _tie(bn_inputs):
    """The oracle's ``tie``: each BatchNorm input takes the native value in its forward, x64 + (x_native - x64).detach(), so the
    float64 gradient is evaluated where the native one was.  Returns (tie, what is left unused)."""
    left = {k: list(v) for k, v in bn_inputs.items()}

    def tie(name, x):
        if name not in left:
            return x
        xn = left[name].pop(0)
        assert tuple(xn.shape) == tuple(x.shape), (name, xn.shape, x.shape)
        return x + (xn.to(x.dtype) - x).detach()
    return tie, left


# the oracle's ReLU (named by the layer it follows) -> where the native forward's mask is recorded
_RELU_AFTER_BN_INPUT = {'upsample_layer.0.1': 'upsample_layer.0.3', 'vae_model.encoder.poolings.0': 'vae_model.encoder.poolings.2',
                        'vae_model.encoder.poolings.3': 'vae_model.encoder.poolings.5'}


def _native_relu(rec):
    """The oracle's ``relu``: x * (native pre-activation > 0), so the float64 gradient takes the branch the native one took.  The
    masks come from the native GroupNorm outputs (pitch encoder), the BatchNorm inputs that are ReLU outputs (the ReLU is fused into
    the conv in front: upsample_layer.0, the posterior encoder's poolings) and the latent map's BatchNorm outputs.  ReLUs without a
    recorded mask (eval-mode BatchNorms, spk_proj's fused ReLU) stay torch.relu.  Returns (relu, what is left unused)."""
    left = {k: [o > 0 for o in v] for k, v in rec['gn'].items()}
    left.update({relu: [x > 0 for x in rec['bn'][bn]] for relu, bn in _RELU_AFTER_BN_INPUT.items() if bn in rec['bn']})
    left.update({k: [o > 0 for o in v] for k, v in rec['bn_out'].items() if k.startswith('z_mapping_function.')})

    def relu(name, x):
        if name not in left:
            return torch.relu(x)
        mask = left[name].pop(0)
        assert tuple(mask.shape) == tuple(x.shape), (name, mask.shape, x.shape)
        return x * mask.to(x.dtype)
    return relu, left


def _tied_step(m, phase, batch, native_extra=None, oracle_extra=None):
    """The native step, then float64 autograd through the oracle at the parameters and running statistics the native step started
    from, on what the native forward computed:
      - the native PPG extractor's outputs (detached in both, pinned on their own by test_gpu_vc_asr.py), so the PPG extractor's
        bf16x3 rounding does not enter the BatchNorms as input noise;
      - every train-mode BatchNorm input (_tie): BatchNorm over a few clips divides by small batch deviations and amplifies the
        rounding in front of it by orders of magnitude;
      - every ReLU mask (_native_relu): a pre-activation within rounding of zero takes a different branch on each side and moves its
        element's gradient by its whole share.  The training kernels reduce with atomics, so which element flips changes from run to
        run; on the native masks the comparison no longer depends on it.
    The comparison then sees the rounding of the kernels themselves.  A wrong forward value in front of a BatchNorm is not seen here,
    only in its gradients: the eval-mode forward against float64 (test_gpu_svb_vae_shapes.py) covers those values."""
    snap = {k: v.detach().clone() for k, v in m.state_dict().items()}
    with _recorded(m) as rec:
        losses = _native_step(m, phase, batch, native_extra)
    ref_losses, p = _oracle_on_native(m, phase, batch, snap, rec, oracle_extra)
    return losses, ref_losses, p


def _oracle_on_native(m, phase, batch, snap, rec, extra=None):
    """_oracle_step at ``snap`` on the native PPG, BatchNorm inputs and ReLU masks in ``rec`` (_recorded); all of them are used."""
    assert len(rec['ppg']) == 2
    tie, left = _tie(rec['bn'])
    relu, masks_left = _native_relu(rec)
    out = _oracle_step(m, phase, batch, sd=snap, ppg=dict(zip(('amateur', 'prof'), rec['ppg'])), tie=tie, relu=relu, extra=extra)
    assert not any(left.values()) and not any(masks_left.values()), ({k: len(v) for k, v in left.items()},
                                                                     {k: len(v) for k, v in masks_left.items()})
    return out


# spk_proj.2's bias too: it is added to the latent in front of convs.0, so its gradient is convs.0's weight applied to convs.0.bias's
MAP_ZERO_GRAD = ('z_mapping_function.convs.0.bias', 'z_mapping_function.convs.3.bias', 'z_mapping_function.spk_proj.2.bias')


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
    losses, ref_losses, p = _tied_step(m, 2, batch)
    n = _compare_step(f'phase2 {precision}', m, 2, losses, ref_losses, p, STEP_BARS[use_tc])
    assert n > 100
    assert bool((m.pitch_embed.weight.grad[0] == 0).all())
    assert all(q.grad is None for q in m.vc_asr.parameters())
    sd = m.state_dict()
    for pre in RUNNING:
        for s in ('running_mean', 'running_var'):
            _check(f'phase2 {precision} {pre}.{s}', sd[f'{pre}.{s}'], p[f'{pre}.{s}'], STEP_BARS[use_tc][None])
        assert int(sd[f'{pre}.num_batches_tracked']) == before[f'{pre}.num_batches_tracked'] + 2      # amateur + professional calls


def test_phase3_mapping_step_matches_float64(use_tc):
    m = _model('bf16x3' if use_tc else 'fp32')
    _set_phase(m, 3)
    batch = _batch()
    frozen = {k: v.clone() for k, v in m.state_dict().items() if 'running' in k and not k.startswith('z_mapping_function.')}
    losses, ref_losses, p = _tied_step(m, 3, batch)
    n = _compare_step('phase3', m, 3, losses, ref_losses, p, MAP_BARS[use_tc], zero_grad=MAP_ZERO_GRAD)
    assert n == len(list(m.z_mapping_function.parameters()))
    sd = m.state_dict()
    for pre in MAP_RUNNING:
        for s in ('running_mean', 'running_var'):
            _check(f'phase3 {pre}.{s}', sd[f'{pre}.{s}'], p[f'{pre}.{s}'], MAP_BARS[use_tc][None])
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
        losses, ref_losses, p = _tied_step(m, 2, batch)
        handles = handles or [s._handle.value for s in stacks]
        assert [s._handle.value for s in stacks] == handles and all(s.host_uploads == 1 for s in stacks)
        _compare_step(f'adamw {precision} step {step}', m, 2, losses, ref_losses, p, STEP_BARS[use_tc])
        opt.step()

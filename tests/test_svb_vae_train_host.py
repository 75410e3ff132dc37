"""Host-side checks of the SVB acoustic model's training path (no GPU needed): the float64 oracles of the mel loss and of the phase-2 /
phase-3 steps against the fixtures written from the reference, the mel-loss C entry points rejecting bad arguments before any CUDA
call, and the module refusing what it cannot do."""
import ctypes
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.utils import synthetic as S
from tests.test_oracle_golden import SVB_HP

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
# the fixtures are float32 reference runs: the float64 oracle meets them to float32 rounding of the reference's arithmetic
VALUE_BAR, GRAD_BAR = 2e-5, 1e-4
# phase 3's gradients pass through BatchNorm over a batch of two [128, 1] latents, which amplifies the reference's float32 rounding
# (worst measured 5.4e-4); the biases in front of those BatchNorms have an exactly zero gradient in exact arithmetic, so errors are
# taken relative to at least 1e-3 of the step's largest gradient norm
PHASE3_GRAD_BAR = 2e-3


def _rel(a, b, floor=1e-30):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), floor))


def _check_grad(fx, prefix, name, g, bar, floor):
    g = g.detach().double().reshape(-1)
    sub, norm = fx[f'{prefix}/{name}/sub'], float(fx[f'{prefix}/{name}/norm'])
    stride = 1 if g.numel() <= 4096 else 211
    assert abs(float(g.norm()) - norm) <= bar * max(norm, floor), name
    assert _rel(g[::stride].numpy(), sub, floor) < bar, (name, _rel(g[::stride].numpy(), sub))


def test_mel_loss_oracle_matches_reference_fixture():
    from oracle import mel_loss as OM
    from oracle.gen_golden_train import MEL_LOSS_CASES
    fx = np.load(os.path.join(GOLDEN, 'mel_loss.npz'))
    for name, (B, T, pad) in MEL_LOSS_CASES.items():
        assert list(fx[f'{name}/params']) == [B, T] + list(pad)
        mel_out, target = S.make_mel_pair(B, T, pad, 1234)
        for key, fn in (('l1', OM.l1_loss), ('ssim', OM.ssim_loss)):
            x = mel_out.double().requires_grad_(True)
            loss = fn(x, target.double())
            loss.backward()
            assert _rel(float(loss.detach()), float(fx[f'{name}/{key}'])) < VALUE_BAR, (name, key)
            g = x.grad.reshape(-1)
            stride = 1 if g.numel() <= 4096 else 7
            assert _rel(g[::stride].numpy(), fx[f'{name}/grad/{key}/sub']) < GRAD_BAR, (name, key)


def _oracle_params(sd, trainable):
    return {k: (v.double().requires_grad_(True) if v.is_floating_point() and trainable(k) and 'running' not in k else v.clone().double())
            for k, v in sd.items()}


@pytest.mark.parametrize('phase', [2, 3])
def test_svb_train_oracle_matches_reference_fixture(phase):
    from oracle import svb_vae_train as O
    fx = np.load(os.path.join(GOLDEN, 'svb_vae_train.npz'))
    sd = S.make_svb_state_dict(1234)
    if phase == 2:
        p = _oracle_params(sd, lambda k: not k.startswith(('vc_asr.', 'z_mapping_function.')))
    else:
        p = _oracle_params(sd, lambda k: k.startswith('z_mapping_function.'))
    batch = {k: (v.double() if v.is_floating_point() else v) for k, v in S.make_svb_batch(2, 96, 120, 1234).items()}
    losses, _ = O.svb_train_losses(p, batch, torch.zeros(2, 128, 1, dtype=torch.float64), phase)
    keys = sorted(k.split('/')[-1] for k in fx.files if k.startswith(f'p{phase}/loss/'))
    assert sorted(losses) == keys
    for k, v in losses.items():
        assert _rel(float(v.detach()), float(fx[f'p{phase}/loss/{k}'])) < VALUE_BAR, k
    sum(losses.values()).backward()
    names = list(fx[f'p{phase}/grad_names'])
    assert sorted(names) == sorted(k for k, v in p.items() if v.requires_grad)
    floor = 1e-3 * max(float(fx[f'p{phase}/grad/{n}/norm']) for n in names) if phase == 3 else 1e-30
    for n in names:
        _check_grad(fx, f'p{phase}/grad', n, p[n].grad, GRAD_BAR if phase == 2 else PHASE3_GRAD_BAR, floor)
    if phase == 2:
        assert np.all(fx['p2/pitch_embed_row0'] == 0) and bool((p['pitch_embed.weight'].grad[0] == 0).all())
    bns = ['upsample_layer.0.3', 'vae_model.encoder.poolings.2', 'vae_model.encoder.poolings.5'] if phase == 2 else \
        ['z_mapping_function.convs.1', 'z_mapping_function.convs.4']
    for pre in bns:
        for s in ('running_mean', 'running_var'):
            assert _rel(p[f'{pre}.{s}'].numpy(), fx[f'p{phase}/{pre}.{s}']) < VALUE_BAR, (pre, s)


@pytest.fixture(scope='module')
def lib():
    try:
        _native.build()
    except RuntimeError as e:          # no nvcc on this box: the prebuilt library must already be there
        if not os.path.exists(_native.LIB_PATH):
            pytest.fail(str(e))
    return _native.lib()


def test_mel_loss_entry_points_reject_bad_arguments(lib):
    """Every rejection happens before a launch: host buffers stand in for the device ones and are left untouched."""
    buf = np.full(1 << 12, 7.0, np.float32)
    dbl = np.full(8, 7.0, np.float64)
    p, d = ctypes.c_void_p(buf.ctypes.data), ctypes.c_void_p(dbl.ctypes.data)
    f = ctypes.c_float(6.0)
    err = lambda: lib.svb_last_error()
    fwd = lambda pp, tt, B, T, M, ws=d, out=d: lib.svb_mel_loss_forward(pp, tt, B, T, M, f, ws, out, None)
    bwd = lambda pp, tt, B, T, M, st=d, dp=p: lib.svb_mel_loss_backward(pp, tt, B, T, M, f, st, p, p, dp, None)
    for call in (fwd, bwd):
        assert call(None, p, 1, 8, 80) < 0 and b'null argument' in err()
        assert call(p, None, 1, 8, 80) < 0 and b'null argument' in err()
        for B, T, M in ((0, 8, 80), (1, 0, 80), (1, 8, 0), (-2, 8, 80), (1, -1, 80), (1, 8, -80)):
            assert call(p, p, B, T, M) < 0 and b'bad shape' in err(), (B, T, M)
        assert call(p, p, 1, 8, 129) < 0 and b'do not fit the tile' in err()
    assert fwd(p, p, 1, 8, 80, ws=None) < 0 and b'null argument' in err()
    assert fwd(p, p, 1, 8, 80, out=None) < 0 and b'null argument' in err()
    assert bwd(p, p, 1, 8, 80, st=None) < 0 and b'null argument' in err()
    assert bwd(p, p, 1, 8, 80, dp=None) < 0 and b'null argument' in err()
    assert lib.svb_mel_loss_workspace_bytes(2, 33, 80) == 2 * 3 * 3 * 8          # 3 tiles of 16 frames per clip, 3 doubles each
    for B, T, M in ((0, 8, 80), (1, 0, 80), (1, 8, 0), (1, 8, 129)):
        assert lib.svb_mel_loss_workspace_bytes(B, T, M) == -1
    assert np.all(buf == 7.0) and np.all(dbl == 7.0)


def test_default_model_still_refuses_to_train():
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    m = MleSVBVAE(80, hp=SVB_HP).train()
    assert not m.trainable and not m.vae_model.encoder.trainable and not m.z_mapping_function.trainable
    batch = S.make_svb_batch(2, 16, 16, 1234)
    with pytest.raises(RuntimeError, match='MleSVBVAE is inference only: call .eval'):
        m(**batch, concurrent_ways=['a2a', 'p2p'])


def test_trainable_model_has_no_cpu_path():
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    m = MleSVBVAE(80, hp=SVB_HP, trainable=True)
    assert m.trainable and m.vae_model.encoder.trainable and m.vae_model.decoder.trainable and m.z_mapping_function.trainable
    batch = S.make_svb_batch(2, 16, 16, 1234)
    for mode in (m.train, m.eval):
        mode()
        with pytest.raises(RuntimeError, match='no CPU path'):
            m(**batch, concurrent_ways=['a2a', 'p2p'])
    with pytest.raises(RuntimeError, match='no CPU path'):
        mel_l1_ssim_loss(torch.zeros(1, 4, 80), torch.zeros(1, 4, 80))

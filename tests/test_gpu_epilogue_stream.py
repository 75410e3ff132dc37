"""-m gpu: the streamed epilogue of the wgmma conv kernel (conv_tc.cu: residual and running-sum pieces bulk-copied into
shared memory while the item's MMAs run) against the same generator forced onto per-thread epilogue loads (SVB_EPI=0,
read when the handle is created).  Both compute the same expression in the same order, so the waveform, the stage
outputs and the training-mode forward must be the same bits."""
import contextlib
import io

import pytest
import torch

from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
from neuralsvb_b200.utils import synthetic as S
from tests import gpu_util as U

pytestmark = pytest.mark.gpu

# (B, T frames): the bench shape; one clip of 1 / 3 frames (one-tile items, odd tile counts, rows per stage that are not
# a multiple of 16, 64 or 128); 37 frames (too few items to fuse); 77 frames (stage 3 fused, its rows not a multiple of
# the fused P = 246); and a batch long enough that stage 3 falls back to one launch per layer
SHAPES = [(16, 128), (1, 1), (1, 3), (1, 37), (3, 77), (8, 689)]


def _model(h, precision, epi, monkeypatch, train=False):
    monkeypatch.setenv('SVB_EPI', '1' if epi else '0')
    m = HifiGanGenerator(h, precision=precision)
    m.load_state_dict(S.make_generator_state_dict(h, U.SEED), strict=True)
    if not train:
        with contextlib.redirect_stdout(io.StringIO()):
            m.remove_weight_norm()
    m = (m.train() if train else m.eval()).cuda()
    m.native_handle(torch.device('cuda', 0))            # the handle reads SVB_EPI now
    monkeypatch.delenv('SVB_EPI')
    return m


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3', 'tf32'])
def test_streamed_epilogue_is_bit_identical(precision, monkeypatch, capfd):
    h = S.hifigan_config()
    new = _model(h, precision, True, monkeypatch)
    ref = _model(h, precision, False, monkeypatch)
    for B, T in SHAPES:
        mel, f0 = S.make_mel_f0(B, T, U.SEED)
        ri, nz = S.make_nsf_noise(B, T * 256, U.SEED)
        args, kw = (mel.cuda(), f0.cuda()), dict(rand_ini=ri.cuda(), noise=nz.cuda())
        with torch.no_grad():
            monkeypatch.setenv('SVB_TC_VERBOSE', '1')
            y_n = new(*args, **kw).clone()
            torch.cuda.synchronize()
            monkeypatch.delenv('SVB_TC_VERBOSE')
            plan = capfd.readouterr().err
            taps_n = {n: new.get_tap(n) for n in ('stage0', 'stage1', 'stage2', 'stage3')}
            y_r = ref(*args, **kw).clone()
            taps_r = {n: ref.get_tap(n) for n in taps_n}
        assert torch.isfinite(y_n).all(), (B, T)
        assert torch.equal(y_n, y_r), (precision, B, T, float((y_n - y_r).abs().max()))
        for n in taps_n:
            assert torch.equal(taps_n[n], taps_r[n]), (precision, B, T, n)
        if (B, T) == (16, 128) and precision != 'tf32x3':
            # the bench shape streams the epilogue of the fused steps of stages 2 and 3
            assert any(' epi ' in l and not l.endswith(' epi 0') for l in plan.splitlines()), plan[-2000:]


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32'])
def test_streamed_epilogue_training_forward_and_gradients(precision, monkeypatch):
    h = S.hifigan_config()
    B, T = 2, 24
    mel, f0 = S.make_mel_f0(B, T, U.SEED)
    ri, nz = S.make_nsf_noise(B, T * 256, U.SEED)
    cot = torch.randn(B, 1, T * 256, generator=torch.Generator().manual_seed(7)).cuda()
    out = []
    for epi in (True, False):
        m = _model(h, precision, epi, monkeypatch, train=True)
        y = m(mel.cuda(), f0.cuda(), rand_ini=ri.cuda(), noise=nz.cuda())
        (y * cot).sum().backward()
        out.append((y.detach().clone(), {k: p.grad.clone() for k, p in m.named_parameters()}))
    (y_n, g_n), (y_r, g_r) = out
    assert torch.equal(y_n, y_r), float((y_n - y_r).abs().max())
    # the forward is the same bits; backward sums some gradients with fp32 atomics, whose order varies from run to run
    for k in g_r:
        err = float((g_n[k] - g_r[k]).norm() / g_r[k].norm().clamp_min(1e-30))
        assert err < 1e-5, (k, err)


def test_streamed_epilogue_single_layer_with_residual(monkeypatch):
    """One svb_conv1d_layer call with a residual: the per-layer path of the C ABI takes the streamed epilogue too."""
    from tests.test_gpu_conv_kernels import run_layer
    g = torch.Generator().manual_seed(U.SEED)
    B, C, T, K, dil = 3, 64, 1000, 7, 3
    x, res = torch.randn(B, C, T, generator=g).cuda(), torch.randn(B, C, T, generator=g).cuda()
    w, b = (torch.randn(C, C, K, generator=g) * 0.05).cuda(), torch.randn(C, generator=g).cuda()
    monkeypatch.setenv('SVB_TC_EPI_SLOTS', '0')
    y_ref, _ = run_layer(x, w, b, res, K, dil, 0, 0.1, 0.5, 'bf16x3')
    monkeypatch.delenv('SVB_TC_EPI_SLOTS')
    y_new, _ = run_layer(x, w, b, res, K, dil, 0, 0.1, 0.5, 'bf16x3')
    assert torch.equal(y_new, y_ref)

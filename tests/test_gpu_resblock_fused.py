"""-m gpu: fused ResBlock1 steps (conv_tc.cu, FUSED items: c1 and c2 of one dilation step in one launch for the C <= 64
stages) against the same generator forced onto two launches per step (SVB_FUSE=0, read when the handle is created).  The
fused path must give the same bits: the waveform and the stage outputs are compared with torch.equal."""
import contextlib
import io

import pytest
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
from neuralsvb_b200.utils import synthetic as S
from tests import gpu_util as U

pytestmark = pytest.mark.gpu

# (B, T frames): the bench shape; one clip of 1 / 2 / 3 / 37 frames (too few items per SM to fuse: both handles must take
# the same two-launch path); an odd length whose stage-3 rows (T x 256) are not a multiple of P = 246, fused in stage 3
# only; and a batch long enough that stage 3 falls back from merged and fused launches to one launch per layer
SHAPES = [(16, 128), (1, 1), (1, 2), (1, 3), (1, 37), (3, 77), (8, 689)]


def _model(h, precision, fuse, monkeypatch):
    if fuse:
        monkeypatch.delenv('SVB_FUSE', raising=False)
    else:
        monkeypatch.setenv('SVB_FUSE', '0')
    m = HifiGanGenerator(h, precision=precision)
    m.load_state_dict(S.make_generator_state_dict(h, U.SEED), strict=True)
    with contextlib.redirect_stdout(io.StringIO()):
        m.remove_weight_norm()
    m = m.eval().cuda()
    m.native_handle(torch.device('cuda', 0))            # the handle reads SVB_FUSE now
    return m


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3', 'tf32'])
def test_fused_resblock_steps_are_bit_identical_to_two_launches(precision, monkeypatch, capfd):
    h = S.hifigan_config()
    fused = _model(h, precision, True, monkeypatch)
    plain = _model(h, precision, False, monkeypatch)
    lib = _native.lib()
    for B, T in SHAPES:
        mel, f0 = S.make_mel_f0(B, T, U.SEED)
        ri, nz = S.make_nsf_noise(B, T * 256, U.SEED)
        args, kw = (mel.cuda(), f0.cuda()), dict(rand_ini=ri.cuda(), noise=nz.cuda())
        with torch.no_grad():
            monkeypatch.setenv('SVB_TC_VERBOSE', '1')
            y_f = fused(*args, **kw).clone()
            torch.cuda.synchronize()
            monkeypatch.delenv('SVB_TC_VERBOSE')
            plan = capfd.readouterr().err
            taps_f = {n: fused.get_tap(n) for n in ('stage2', 'stage3')}
            n_f = lib.svb_gen_last_launches(fused.native_handle())
            y_p = plain(*args, **kw).clone()
            taps_p = {n: plain.get_tap(n) for n in ('stage2', 'stage3')}
            n_p = lib.svb_gen_last_launches(plain.native_handle())
        assert torch.isfinite(y_f).all(), (B, T)
        assert torch.equal(y_f, y_p), (precision, B, T, float((y_f - y_p).abs().max()))
        for n in taps_f:
            assert torch.equal(taps_f[n], taps_p[n]), (precision, B, T, n)
        if precision != 'tf32x3' and (B, T) == (16, 128):
            # the bench shape runs both C <= 64 stages fused: 3 launches per stage instead of 6
            assert '[tc] fused 3 chain(s) C 64' in plan and '[tc] fused 3 chain(s) C 32' in plan, plan[-2000:]
            assert n_p - n_f == 6, (n_f, n_p)
        if precision != 'tf32x3' and (B, T) == (3, 77):
            assert '[tc] fused 3 chain(s) C 32' in plan and '[tc] fused 3 chain(s) C 64' not in plan
        if precision == 'tf32x3' and (B, T) == (16, 128):
            assert '[tc] fused' not in plan                 # the doubled planes do not fit next to the intermediate at every step

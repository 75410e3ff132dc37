"""-m gpu: the fused C = 32 ResBlock1 steps at two CTAs per SM (conv_tc.cu: tc_plan with ctas = 2) against the same
generator held at one CTA per SM (SVB_TC_FUSED_CTAS=1, read when the handle is created).  Every item still runs in one CTA
in the same order, so the waveform and the stage outputs must be the same bits (torch.equal)."""
import contextlib
import io

import pytest
import torch

from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
from neuralsvb_b200.utils import synthetic as S
from tests import gpu_util as U

pytestmark = pytest.mark.gpu

# (B, T frames, CTAs per SM of stage 3's fused launches with the default handle, with SVB_TC_FUSED_CTAS=1; 0 = not fused).
# The bench shape first: the one-CTA handle launches the fused C = 32 kernel with its larger layout before the default
# handle asks the occupancy calculator about the smaller one, and then launches it again.  Odd lengths whose stage-3
# rows (T x 256) end inside the last P = 246-row item (16 x 77 / 41: 32 / 164 rows in the last item); clips too few for 264 CTAs (one CTA
# per SM, or no fused launch); and a batch whose stage 3 exceeds the one-CTA item table (fused only at two CTAs per SM).
SHAPES = [(16, 128, 2, 1), (16, 77, 2, 1), (16, 41, 2, 1), (3, 77, 1, 1), (1, 1, 0, 0), (1, 37, 0, 0), (2, 41, 0, 0),
          (8, 689, 2, 0)]


def _model(h, precision, ctas, monkeypatch):
    monkeypatch.setenv('SVB_TC_FUSED_CTAS', str(ctas))
    m = HifiGanGenerator(h, precision=precision)
    m.load_state_dict(S.make_generator_state_dict(h, U.SEED), strict=True)
    with contextlib.redirect_stdout(io.StringIO()):
        m.remove_weight_norm()
    m = m.eval().cuda()
    m.native_handle(torch.device('cuda', 0))            # the handle reads SVB_TC_FUSED_CTAS now
    monkeypatch.delenv('SVB_TC_FUSED_CTAS')
    return m


def _run(m, args, kw, monkeypatch, capfd):
    monkeypatch.setenv('SVB_TC_VERBOSE', '1')
    y = m(*args, **kw).clone()
    torch.cuda.synchronize()
    monkeypatch.delenv('SVB_TC_VERBOSE')
    plan = [l for l in capfd.readouterr().err.splitlines() if l.startswith('[tc] fused 3 chain(s) C 32')]
    return y, {n: m.get_tap(n) for n in ('stage2', 'stage3')}, plan


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32'])
def test_two_ctas_per_sm_are_bit_identical_to_one(precision, monkeypatch, capfd):
    h = S.hifigan_config()
    one = _model(h, precision, 1, monkeypatch)
    two = _model(h, precision, 2, monkeypatch)
    for B, T, ctas_two, ctas_one in SHAPES:
        mel, f0 = S.make_mel_f0(B, T, U.SEED)
        ri, nz = S.make_nsf_noise(B, T * 256, U.SEED)
        args, kw = (mel.cuda(), f0.cuda()), dict(rand_ini=ri.cuda(), noise=nz.cuda())
        with torch.no_grad():
            y_1, taps_1, plan_1 = _run(one, args, kw, monkeypatch, capfd)
            y_2, taps_2, plan_2 = _run(two, args, kw, monkeypatch, capfd)
            y_1b, _, plan_1b = _run(one, args, kw, monkeypatch, capfd)     # after the other handle's plans
        assert torch.isfinite(y_2).all(), (B, T)
        assert torch.equal(y_2, y_1), (precision, B, T, float((y_2 - y_1).abs().max()))
        assert torch.equal(y_1b, y_1), (precision, B, T)
        for n in taps_2:
            assert torch.equal(taps_2[n], taps_1[n]), (precision, B, T, n)
        for plan, ctas in ((plan_2, ctas_two), (plan_1, ctas_one), (plan_1b, ctas_one)):
            if ctas:
                assert len(plan) == 3 and all(f' ctas/SM {ctas} ' in l for l in plan), (B, T, plan)
            else:
                assert not plan, (B, T, plan)

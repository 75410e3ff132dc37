"""-m gpu: the staged epilogue of the 128-column wgmma conv (conv_tc.cu: epilogue_staged, the C = 256 and C = 128 ResBlock
launches of stages 0 and 1) against the same generator forced onto per-thread epilogue loads (SVB_EPI=0, read when the
handle is created).  Both compute ((acc + b) + res) * out_scale (+ old) in the same order with the same row masks, so the
stage-0 and stage-1 outputs and the waveform must be the same bits.  The plan is read back from SVB_TC_VERBOSE: the
residual launches of stages 0 and 1 take two staging slots per math warp ("stage 2") in bf16x3 and tf32; tf32x3 has no
room for them and keeps the L2-prefetch path."""
import contextlib
import io
import re

import pytest
import torch

from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
from neuralsvb_b200.utils import synthetic as S
from tests import gpu_util as U

pytestmark = pytest.mark.gpu

# (B, T frames, ResBlock layers per launch of stage 1).  The bench shape; 4 x 41 frames (stage 0: 328 rows = 3 tiles per
# clip, stage 1: 2624 rows = 21 tiles, so one-tile items at the end of each clip, LPT splits, and a last tile whose rows
# end inside a 16-row piece); clips shorter than one tile in stage 0 (1 / 3 frames: 8 / 24 rows) and in stage 1 (1 frame:
# 64 rows); and a batch whose stage-1 work list would overflow the per-CTA item table, so stage 1 runs one launch per
# layer.  Every forward ends each stage with the running-sum step (chain-ordered, read-modify-write of the sum).
SHAPES = [(16, 128, 3), (4, 41, 3), (1, 1, 3), (1, 3, 3), (8, 1111, 1)]
PLAN = re.compile(r'\[tc\] (\d) layer\(s\) Cin (\d+) CoutP (\d+) .* l2pf (\d) stage (\d)$')


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


def _run(m, args, kw, monkeypatch, capfd, taps=('stage0', 'stage1')):
    monkeypatch.setenv('SVB_TC_VERBOSE', '1')
    y = m(*args, **kw).detach().clone()
    torch.cuda.synchronize()
    monkeypatch.delenv('SVB_TC_VERBOSE')
    # the ResBlock launches of stages 0 and 1: Cin = CoutP = 256 / 128 (the upsamplers have CoutP = rate x C)
    plans = [PLAN.search(l) for l in capfd.readouterr().err.splitlines()]
    plans = [tuple(int(x) for x in p.groups()) for p in plans if p and p.group(2) == p.group(3) and p.group(2) in ('256', '128')]
    return y, {n: m.get_tap(n).clone() for n in taps}, plans


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3', 'tf32'])
def test_staged_epilogue_is_bit_identical(precision, monkeypatch, capfd):
    h = S.hifigan_config()
    new = _model(h, precision, True, monkeypatch)
    ref = _model(h, precision, False, monkeypatch)
    staged = precision != 'tf32x3'
    for B, T, layers1 in SHAPES:
        mel, f0 = S.make_mel_f0(B, T, U.SEED)
        ri, nz = S.make_nsf_noise(B, T * 256, U.SEED)
        args, kw = (mel.cuda(), f0.cuda()), dict(rand_ini=ri.cuda(), noise=nz.cuda())
        with torch.no_grad():
            y_n, taps_n, plan_n = _run(new, args, kw, monkeypatch, capfd)
            y_r, taps_r, plan_r = _run(ref, args, kw, monkeypatch, capfd)
        assert torch.isfinite(y_n).all(), (B, T)
        for n in taps_n:
            assert torch.equal(taps_n[n], taps_r[n]), (precision, B, T, n, float((taps_n[n] - taps_r[n]).abs().max()))
        assert torch.equal(y_n, y_r), (precision, B, T, float((y_n - y_r).abs().max()))
        # The c2 launches read a residual (and the running sum on the last step; the middle step runs in place), so the plan
        # prefetches their rows into L2 ("l2pf 1") and, but in tf32x3, stages them.  Stage 0 always merges its 3 chains;
        # stage 1 merges them unless the work list overflows.  c1 launches and the upsamplers (the stage-2 one also has
        # Cin = CoutP = 128) read no residual and are never staged.
        for C, layers in ((256, 3), (128, layers1)):
            c2 = [p for p in plan_n if p[1] == C and p[3]]
            assert c2 and all(p[0] == layers and p[4] == (2 if staged else 0) for p in c2), (precision, B, T, C, c2)
        assert all(p[4] == 0 for p in plan_n if not p[3]), (precision, B, T, plan_n)
        # the reference handle keeps per-thread loads everywhere (no staging slots, no L2 prefetch)
        assert plan_r and all(p[3] == 0 and p[4] == 0 for p in plan_r), (precision, B, T, plan_r)


def test_staged_epilogue_training_forward(monkeypatch, capfd):
    """The training forward runs the same merged launches: its waveform and its tape (every ResBlock input x{m} and c1
    output t{m} of stages 0 and 1) are the same bits with the staged epilogue."""
    h = S.hifigan_config()
    B, T = 2, 24
    mel, f0 = S.make_mel_f0(B, T, U.SEED)
    ri, nz = S.make_nsf_noise(B, T * 256, U.SEED)
    args, kw = (mel.cuda(), f0.cuda()), dict(rand_ini=ri.cuda(), noise=nz.cuda())
    tape = ['stage0', 'stage1'] + [f'resblocks.{r}.{v}{m}' for r in range(6) for v in 'xt' for m in range(3)]
    out = []
    for epi in (True, False):
        m = _model(h, 'bf16x3', epi, monkeypatch, train=True)
        out.append(_run(m, args, kw, monkeypatch, capfd, taps=tape))
    (y_n, taps_n, plan_n), (y_r, taps_r, _) = out
    assert any(p[4] == 2 for p in plan_n), plan_n
    assert torch.equal(y_n, y_r), float((y_n - y_r).abs().max())
    for n in tape:
        assert torch.equal(taps_n[n], taps_r[n]), n

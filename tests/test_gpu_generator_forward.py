"""-m gpu: the generator's inference forward (svb_gen_forward: conv_tc.cu / conv_ffma.cu, the NSF source, conv_post) launch
group by launch group against float64 torch on the kernels' own inputs, at the shapes and schedules that run in production.

Each group is recomputed in float64 from the taps the CUDA forward left behind, with the oracle's own statement of the model
(oracle/hifigan.py: upsample_forward, stage_forward, post_forward) and the weights the handle was given (folded_state):
  conv_pre   from the mel
  ups{i}     from conv_pre / stage{i-1} and har_source (the upsampler plus the noise conv)
  stage{i}   from ups{i} (every ResBlock of the stage, summed and divided by their number)
  waveform   from the last stage
so what a check sees is the rounding of one group, not errors compounded from the mel onwards.  A training handle keeps every
conv input (the tape, resblocks.{r}.x{m} / .t{m}), which makes single-conv checks of the merged, staged, chain-ordered
launches possible as well.

Errors are measured per tap as the L-inf error relative to max |reference| of a clip, taking the worst clip, and as the
relative L2 error over the batch.  The per-clip L-inf is the check: a fault confined to one 16-row piece of one clip is
diluted in any norm over the batch (test_per_clip_linf_sees_a_fault_that_batch_l2_dilutes).  A failure names the clip,
channel, row and the row's 128-row tile and 16-row piece.  The schedule every stage ran is read back from the SVB_TC_VERBOSE
plan lines (conv_tc.cu: tc_plan and launch_conv_tc_multi)."""
import contextlib
import io
import math
import re
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
from neuralsvb_b200.utils import synthetic as S
from oracle import hifigan as O
from tests import gpu_util as U
from tests.test_gpu_conv_kernels import TOL

pytestmark = pytest.mark.gpu

# (L-inf relative to max |reference| of the worst clip, relative L2 over the batch) per tap, about 3x the worst values
# measured (in the comments) on an H100 80GB HBM3 at a 700 W power limit over every shape, knob handle and architecture of
# this file that runs the precision.  Stage 0 (C = 256) contracts over the most terms and has the largest split-mode error.
BARS = {
    'bf16x3': {'conv_pre': (2.0e-5, 1.4e-5),       # 7.2e-6 / 4.9e-6
               'ups0': (2.0e-5, 1.6e-5),           # 6.8e-6 / 5.6e-6
               'ups1': (1.9e-5, 1.4e-5),           # 6.5e-6 / 4.7e-6
               'ups2': (2.1e-5, 1.3e-5),           # 7.3e-6 / 4.6e-6
               'ups3': (2.5e-5, 1.3e-5),           # 8.4e-6 / 4.6e-6
               'stage0': (4.2e-5, 3.4e-5),         # 1.4e-5 / 1.2e-5
               'stage1': (2.4e-5, 1.9e-5),         # 8.1e-6 / 6.5e-6
               'stage2': (1.6e-5, 1.3e-5),         # 5.7e-6 / 4.5e-6
               'stage3': (2.1e-5, 1.3e-5),         # 7.2e-6 / 4.6e-6
               'wave': (2.1e-6, 7.0e-7)},          # 7.2e-7 / 2.4e-7
    'tf32x3': {'conv_pre': (1.5e-5, 1.1e-5),       # 5.1e-6 / 3.9e-6
               'ups0': (2.5e-5, 2.0e-5),           # 8.6e-6 / 6.7e-6
               'ups1': (1.2e-5, 9.0e-6),           # 4.2e-6 / 3.1e-6
               'ups2': (7.0e-6, 4.0e-6),           # 2.3e-6 / 1.4e-6
               'ups3': (3.5e-6, 1.7e-6),           # 1.2e-6 / 6.0e-7
               'stage0': (7.5e-5, 6.5e-5),         # 2.5e-5 / 2.2e-5
               'stage1': (2.6e-5, 2.6e-5),         # 8.7e-6 / 8.7e-6
               'stage2': (1.7e-5, 1.4e-5),         # 5.9e-6 / 4.8e-6
               'stage3': (9.0e-6, 8.0e-6),         # 3.2e-6 / 2.8e-6
               'wave': (2.3e-6, 6.0e-7)},          # 7.7e-7 / 2.1e-7
    # 1xTF32, the opt-in fast mode (10-bit operands); conv_post runs on CUDA cores in every mode
    'tf32': {'conv_pre': (1.2e-3, 9.0e-4),         # 4.2e-4 / 3.0e-4
             'ups0': (1.0e-3, 8.4e-4),             # 3.4e-4 / 2.8e-4
             'ups1': (1.0e-3, 8.0e-4),             # 3.5e-4 / 2.7e-4
             'ups2': (1.1e-3, 7.0e-4),             # 3.8e-4 / 2.3e-4
             'ups3': (1.2e-3, 6.0e-4),             # 4.0e-4 / 2.0e-4
             'stage0': (1.0e-3, 8.0e-4),           # 3.4e-4 / 2.7e-4
             'stage1': (9.5e-4, 7.0e-4),           # 3.2e-4 / 2.4e-4
             'stage2': (9.0e-4, 7.5e-4),           # 3.1e-4 / 2.6e-4
             'stage3': (1.2e-3, 8.5e-4),           # 4.1e-4 / 2.9e-4
             'wave': (2.0e-6, 6.0e-7)},            # 6.6e-7 / 2.0e-7
    # every kernel on CUDA cores (conv_ffma)
    'fp32': {'conv_pre': (3.4e-6, 1.2e-6),         # 1.1e-6 / 4.2e-7
             'ups0': (5.0e-6, 1.6e-6),             # 1.7e-6 / 5.3e-7
             'ups1': (3.2e-6, 1.0e-6),             # 1.1e-6 / 3.6e-7
             'ups2': (2.4e-6, 7.0e-7),             # 8.0e-7 / 2.3e-7
             'ups3': (1.8e-6, 4.2e-7),             # 6.1e-7 / 1.4e-7
             'stage0': (3.1e-6, 2.1e-6),           # 1.1e-6 / 7.2e-7
             'stage1': (1.9e-6, 1.3e-6),           # 6.4e-7 / 4.5e-7
             'stage2': (1.5e-6, 1.0e-6),           # 5.3e-7 / 3.4e-7
             'stage3': (1.4e-6, 7.5e-7),           # 4.6e-7 / 2.5e-7
             'wave': (1.8e-6, 6.4e-7)},            # 6.1e-7 / 2.2e-7
}
# A conv weight scaled by 1 + 2e-3 must fail its split-mode stage bar by this factor (test_a_2e_3_weight_error_fails_its_stage_bar:
# measured 7.0x (tf32x3, stage 0) to 57x); so must 2e-3 x max |ref| added to one piece.
MARGIN = 5.0

# (B, T frames, what the shape reaches).  Stage i has T x prod(rates[:i+1]) rows per clip: 8 / 64 / 128 / 256 x T.
SHAPES = [
    (16, 128, 'bench.py headline: stages 0-1 merged with the staged epilogue (bf16x3, tf32), stages 2-3 fused, stage 3 '
              'at two CTAs per SM; tf32x3 merged and unfused'),
    (8, 688, "pipeline_cfg5's generator (8 clips of 8 s)"),
    (4, 41, 'MT = 2 and one-tile items in one list; the last rows of a clip end inside a 16-row piece'),
    (16, 77, 'two-CTA fused launches whose last item is partial'),
    (16, 41, 'two-CTA fused launches whose last item is partial'),
    (3, 77, 'stage 3 fused at one CTA per SM, stage 2 not fused'),
    (1, 37, 'too few items to fuse'),
    (1, 1, 'clips shorter than one tile'),
    (1, 3, 'clips shorter than one tile'),
    (8, 1111, 'stage 1 falls back to one launch per layer (its work list overflows the per-CTA item table)'),
]
SHORT = [(16, 128), (4, 41), (1, 1)]                        # tf32 and fp32 (conv_ffma) run these
# Per-stage schedules of the bench shape, as test_gpu_epilogue_stream_n128.py, test_gpu_resblock_fused.py and
# test_gpu_fused_two_ctas.py pin them.
BENCH_SCHEDULE = {'bf16x3': ['merged-staged', 'merged-staged', 'fused1', 'fused2'],
                  'tf32': ['merged-staged', 'merged-staged', 'fused1', 'fused2'],
                  'tf32x3': ['merged', 'merged', 'merged', 'merged'],
                  'fp32': ['ffma'] * 4}
KINDS = {'fused2', 'fused1', 'merged-staged', 'merged', 'single'}
# tf32x3 has no room for the staging slots and does not fuse at the bench shape; over SHAPES it reaches these kinds:
TF32X3_KINDS = {'merged', 'single'}

PLAN = re.compile(r'\[tc\] (\d+) layer\(s\) Cin (\d+) CoutP (\d+) KS \d+\.\. halo \d+ Tq (\d+) \|.* stage (\d+)$')
FUSED = re.compile(r'\[tc\] fused (\d+) chain\(s\) C (\d+) KS .* Tq (\d+) \|.* ctas/SM (\d+) ')


def say(capfd, msg):
    with capfd.disabled():
        print(msg, flush=True)


def config(name):
    if name == 'hop256':
        return S.hifigan_config(True)
    if name == 'hop128':
        return S.hifigan_config(True, hop=128)
    if name == 'no_nsf':
        return S.hifigan_config(False)
    h = S.hifigan_config(True)                     # 'resblock2': ResBlock2 with two dilations
    h['resblock'] = '2'
    h['resblock_dilation_sizes'] = [[1, 3], [1, 3], [1, 3]]
    return h


def make_model(name, precision, monkeypatch, train=False, env=None):
    """A generator on cuda:0 whose handle is created now, under the knobs ``env`` (read at handle creation)."""
    h = config(name)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    m = HifiGanGenerator(h, precision=precision)
    m.load_state_dict(S.make_generator_state_dict(h, U.SEED), strict=True)
    if not train:
        with contextlib.redirect_stdout(io.StringIO()):
            m.remove_weight_norm()
    m = (m.train() if train else m.eval()).cuda()
    m.native_handle(torch.device('cuda', 0))
    for k in env or {}:
        monkeypatch.delenv(k)
    return m, h


def ref_weights(m):
    """The folded tensors the handle was given, as float64 on the GPU."""
    return {k: v.to('cuda', torch.float64) for k, v in m.folded_state().items()}


def forward(m, h, B, T, monkeypatch, capfd):
    """One forward at (B, T) with the NSF draws injected; returns the mel, the waveform and the plan lines."""
    hop = int(np.prod(h['upsample_rates']))
    mel, f0 = S.make_mel_f0(B, T, U.SEED)
    args, kw = [mel.cuda(), None], {}
    if h['use_pitch_embed']:
        ri, nz = S.make_nsf_noise(B, T * hop, U.SEED)
        args[1], kw = f0.cuda(), dict(rand_ini=ri.cuda(), noise=nz.cuda())
    capfd.readouterr()
    monkeypatch.setenv('SVB_TC_VERBOSE', '1')
    with torch.enable_grad() if m.training else torch.no_grad():
        y = m(*args, **kw).detach()
    torch.cuda.synchronize()
    monkeypatch.delenv('SVB_TC_VERBOSE')
    return mel, y, capfd.readouterr().err.splitlines()


def schedules(h, T, plan):
    """The schedule of each stage's ResBlock launches: 'fused1' / 'fused2' (fused c1 + c2 items at 1 / 2 CTAs per SM),
    'merged-staged' / 'merged' (one launch per step over all chains, with / without the staged epilogue), 'single' (one
    launch per conv) or 'ffma' (no wgmma launch).  ResBlock launches have Cin = CoutP = C and Tq = the stage's rows; the
    next stage's upsampler can match that too (Cin = 2 C, CoutP = rate x C), but it is one launch, never a stage's worth."""
    nk, nd = len(h['resblock_kernel_sizes']), len(h['resblock_dilation_sizes'][0])
    per_conv = nk * nd * (2 if h['resblock'] == '1' else 1)
    lines = [tuple(int(x) for x in p.groups()) for p in map(PLAN.search, plan) if p]
    fused = [tuple(int(x) for x in f.groups()) for f in map(FUSED.search, plan) if f]
    out, Ti, C = [], T, h['upsample_initial_channel']
    for u in h['upsample_rates']:
        Ti, C = Ti * u, C // 2
        rb = [p for p in lines if p[1] == C and p[2] == C and p[3] == Ti]
        kinds = [f'fused{c}' for c in sorted({f[3] for f in fused if f[1] == C and f[2] == Ti})]
        multi = [p for p in rb if p[0] == nk]
        if multi:
            kinds.append('merged-staged' if any(p[4] for p in multi) else 'merged')
        if sum(p[0] == 1 for p in rb) >= per_conv:
            kinds.append('single')
        out.append('+'.join(kinds) if kinds else ('ffma' if not lines and not fused else '?'))
    return out


def compare(got, ref_fn):
    """(worst per-clip L-inf relative to max |ref| of that clip, batch relative L2, (clip, channel, row)) of ``got``
    [B, C, T] against the float64 references ``ref_fn(b)`` [1, C, T], computed one clip at a time."""
    worst, where, d2, r2 = -1.0, (0, 0, 0), 0.0, 0.0
    for b in range(got.shape[0]):
        ref = ref_fn(b)[0]
        g = got[b].double()
        assert g.shape == ref.shape, (tuple(g.shape), tuple(ref.shape))
        d = (g - ref).abs()
        if not torch.isfinite(g).all():
            d = torch.where(torch.isfinite(d), d, torch.full_like(d, math.inf))
        e = float(d.max()) / max(float(ref.abs().max()), 1e-30)
        if e > worst:
            c, t = divmod(int(d.argmax()), d.shape[-1])
            worst, where = e, (b, c, t)
        d2 += float((d * d).sum())
        r2 += float((ref * ref).sum())
    return worst, math.sqrt(d2 / max(r2, 1e-300)), where


def describe(tag, tap, res):
    e, l2, (b, c, t) = res
    return (f'{tag} {tap}: L-inf {e:.2e} at clip {b} channel {c} row {t} (128-row tile {t // 128}, 16-row piece '
            f'{t % 128 // 16}), relative L2 {l2:.2e}')


def group_errors(m, h, w, mel, y):
    """{tap: compare(...)} of every launch group of the last forward of ``m``, each on the kernels' own input."""
    n = len(h['upsample_rates'])
    mel = mel.to(w['conv_pre.weight'].device, torch.float64)
    har = m.get_tap('har_source') if h['use_pitch_embed'] else None
    hb = (lambda b: None) if har is None else (lambda b: har[b:b + 1].double())
    out = {'conv_pre': compare(m.get_tap('conv_pre'),
                               lambda b: F.conv1d(mel[b:b + 1], w['conv_pre.weight'], w['conv_pre.bias'], padding=3))}
    x = m.get_tap('conv_pre')
    for i in range(n):
        ups = m.get_tap(f'ups{i}')
        out[f'ups{i}'] = compare(ups, lambda b: O.upsample_forward(w, h, i, x[b:b + 1].double(), hb(b)))
        x = m.get_tap(f'stage{i}')
        out[f'stage{i}'] = compare(x, lambda b: O.stage_forward(w, h, i, ups[b:b + 1].double()))
        del ups
    out['wave'] = compare(y, lambda b: O.post_forward(w, h, x[b:b + 1].double()))
    return out


def judge(tag, precision, errs, capfd, bad):
    """Print a MEASURED line per tap and collect the taps over their bars in ``bad``."""
    for tap, res in errs.items():
        say(capfd, 'MEASURED ' + describe(tag, tap, res))
        li, l2 = BARS[precision][tap]
        if not (res[0] <= li and res[1] <= l2):
            bad.append(describe(tag, tap, res) + f' > bars ({li:.0e}, {l2:.0e})')


# ------------------------------------------------------------------ eval forward, every schedule
@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3', 'tf32', 'fp32'])
def test_eval_forward_launch_groups_match_float64(precision, monkeypatch, capfd):
    m, h = make_model('hop256', precision, monkeypatch)
    w = ref_weights(m)
    shapes = [s for s in SHAPES if precision in ('bf16x3', 'tf32x3') or s[:2] in SHORT]
    bad, table = [], {}
    for B, T, what in shapes:
        t0 = time.time()
        mel, y, plan = forward(m, h, B, T, monkeypatch, capfd)
        table[(B, T)] = schedules(h, T, plan)
        judge(f'B{B}xT{T} {precision}', precision, group_errors(m, h, w, mel, y), capfd, bad)
        say(capfd, f'SCHEDULE B{B}xT{T} {precision}: {table[(B, T)]} ({what}; {time.time() - t0:.1f} s)')
        torch.cuda.empty_cache()
    assert not bad, '\n'.join(bad)
    assert table[(16, 128)] == BENCH_SCHEDULE[precision], table[(16, 128)]
    reached = {k for t in table.values() for s in t for k in s.split('+')}
    assert reached <= KINDS | {'ffma'}, table
    if precision == 'bf16x3':
        assert reached == KINDS, table
    if precision == 'tf32x3':
        assert reached == TF32X3_KINDS, table


# ------------------------------------------------------------------ the anchors of the bit-equality tests
@pytest.mark.parametrize('env', [{'SVB_FUSE': '0'}, {'SVB_MERGE': '0'}, {'SVB_EPI': '0'}, {'SVB_TC_FUSED_CTAS': '1'}],
                         ids=lambda e: '_'.join(f'{k}={v}' for k, v in e.items()))
def test_knob_handles_match_float64(env, monkeypatch, capfd):
    """The handles test_gpu_resblock_fused.py, test_gpu_epilogue_stream*.py and test_gpu_fused_two_ctas.py compare the
    default schedule with, held to the same bars."""
    m, h = make_model('hop256', 'bf16x3', monkeypatch, env=env)
    w = ref_weights(m)
    bad = []
    for B, T in ((16, 128), (4, 41)):
        mel, y, plan = forward(m, h, B, T, monkeypatch, capfd)
        tag = f'B{B}xT{T} bf16x3 {env}'
        judge(tag, 'bf16x3', group_errors(m, h, w, mel, y), capfd, bad)
        say(capfd, f'SCHEDULE {tag}: {schedules(h, T, plan)}')
    assert not bad, '\n'.join(bad)


# ------------------------------------------------------------------ other architectures
@pytest.mark.parametrize('name,B,T', [pytest.param('hop128', 2, 75, id='hop128_singing'),
                                      pytest.param('resblock2', 2, 40, id='resblock2_two_dilations'),
                                      pytest.param('no_nsf', 2, 40, id='hop256_without_nsf')])
def test_other_architectures_match_float64(name, B, T, monkeypatch, capfd):
    m, h = make_model(name, 'bf16x3', monkeypatch)
    mel, y, plan = forward(m, h, B, T, monkeypatch, capfd)
    bad = []
    judge(f'{name} B{B}xT{T} bf16x3', 'bf16x3', group_errors(m, h, ref_weights(m), mel, y), capfd, bad)
    say(capfd, f'SCHEDULE {name} B{B}xT{T} bf16x3: {schedules(h, T, plan)}')
    assert not bad, '\n'.join(bad)


# ------------------------------------------------------------------ training forward, one launch at a time
def tape_errors(m, h, w):
    """{tap: compare(...)} of every conv launch of the ResBlocks of the last training forward, each on its own tape input:
    ResBlock1 t{m} = c1(lrelu(x{m})), x{m+1} = c2(lrelu(t{m})) + x{m}; ResBlock2 x{m+1} = c(lrelu(x{m})) + x{m}; and
    stage{i} = sum over chains of the last step's output / nk (the chain-ordered running sum)."""
    nk = len(h['resblock_kernel_sizes'])
    r1 = h['resblock'] == '1'
    out = {}

    def conv(name, x, k, d):
        return F.conv1d(F.leaky_relu(x, O.LRELU_SLOPE), w[name + '.weight'], w[name + '.bias'], dilation=d,
                        padding=O.get_padding(k, d))
    for i in range(len(h['upsample_rates'])):
        last = []
        for j, (k, dil) in enumerate(zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes'])):
            rb = f'resblocks.{i * nk + j}'
            for mm, d in enumerate(dil):
                x = m.get_tap(f'{rb}.x{mm}')
                c2_in = x
                if r1:
                    t = m.get_tap(f'{rb}.t{mm}')
                    out[f'{rb}.t{mm}'] = compare(t, lambda b: conv(f'{rb}.convs1.{mm}', x[b:b + 1].double(), k, d))
                    c2_in, name, d2 = t, f'{rb}.convs2.{mm}', 1
                else:
                    name, d2 = f'{rb}.convs.{mm}', d

                def step(b, c2_in=c2_in, x=x, name=name, k=k, d2=d2):
                    return conv(name, c2_in[b:b + 1].double(), k, d2) + x[b:b + 1].double()
                if mm + 1 < len(dil):
                    out[f'{rb}.x{mm + 1}'] = compare(m.get_tap(f'{rb}.x{mm + 1}'), step)
                else:
                    last.append(step)
        out[f'stage{i}'] = compare(m.get_tap(f'stage{i}'), lambda b: sum(s(b) for s in last) / nk)
    return out


# Single-conv launches are held to test_gpu_conv_kernels.py's TOL with the per-clip normalisation as it is.  Worst per-clip
# L-inf measured on the H100 above over both shapes: fp32 3.1e-6, tf32 5.8e-4, tf32x3 2.3e-5, bf16x3 1.5e-5 (ResBlock2
# 9.2e-6), every one a c1 output t{m}.
def judge_tape(tag, precision, errs, capfd, bad):
    worst = max(errs.items(), key=lambda kv: kv[1][0])
    for tap, res in errs.items():
        if tap.startswith('stage'):
            say(capfd, 'MEASURED ' + describe(tag, tap, res))
        if not res[0] <= TOL[precision]:
            bad.append(describe(tag, tap, res) + f' > {TOL[precision]:.0e}')
    say(capfd, f'MEASURED {tag}: {len(errs)} launches, worst ' + describe('', worst[0], worst[1]).strip())


_train = {}


def train_model(name, precision, monkeypatch):
    """One training handle per architecture, shared by its cases (set_precision switches the kernels' mode)."""
    if name not in _train:
        _train.clear()
        _train[name] = make_model(name, precision, monkeypatch, train=True)
    m, h = _train[name]
    m.set_precision(precision)
    return m, h


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'tf32x3', 'bf16x3'])
@pytest.mark.parametrize('B,T', [pytest.param(16, 128, id='B16xT128_bench'), pytest.param(3, 37, id='B3xT37_odd')])
def test_training_forward_tape_matches_float64_launch_by_launch(B, T, precision, monkeypatch, capfd):
    m, h = train_model('hop256', precision, monkeypatch)
    _, _, plan = forward(m, h, B, T, monkeypatch, capfd)
    bad = []
    judge_tape(f'tape B{B}xT{T} {precision}', precision, tape_errors(m, h, ref_weights(m)), capfd, bad)
    say(capfd, f'SCHEDULE tape B{B}xT{T} {precision}: {schedules(h, T, plan)}')
    assert not bad, '\n'.join(bad)


def test_resblock2_training_tape_matches_float64(monkeypatch, capfd):
    m, h = train_model('resblock2', 'bf16x3', monkeypatch)
    forward(m, h, 2, 40, monkeypatch, capfd)
    bad = []
    judge_tape('tape resblock2 B2xT40 bf16x3', 'bf16x3', tape_errors(m, h, ref_weights(m)), capfd, bad)
    assert not bad, '\n'.join(bad)


# ------------------------------------------------------------------ the NSF source at the timed lengths
@pytest.mark.parametrize('B,T', [(16, 128), (8, 688)])
def test_nsf_source_at_the_timed_lengths_matches_oracle(B, T, monkeypatch, capfd):
    """nsf_source.cu reproduces the float32 reference's phase sums exactly by keeping every partial sum exact in double;
    the bits left for that shrink as the clip grows.  16 x 128 frames is 32k samples a clip, 8 x 688 is 176k."""
    m, h = make_model('hop256', 'bf16x3', monkeypatch)
    forward(m, h, B, T, monkeypatch, capfd)
    har = m.get_tap('har_source')[:, 0].cpu()
    _, f0 = S.make_mel_f0(B, T, U.SEED)
    ri, nz = S.make_nsf_noise(B, T * 256, U.SEED)
    f0_up = torch.repeat_interleave(f0, 256, dim=1)[:, :, None]
    ref, _ = O.source_module(f0_up, m.folded_state(), ri, nz, sr=h['audio_sample_rate'])
    d = (har - ref[:, :, 0]).abs()
    b, t = divmod(int(d.argmax()), d.shape[1])
    say(capfd, f'MEASURED har_source B{B}xT{T}: L-inf {float(d.max()):.2e} at clip {b} sample {t}')
    assert float(d.max()) < 5e-6, (float(d.max()), b, t)     # test_gpu_parity.py::test_nsf_source_matches_oracle


# ------------------------------------------------------------------ the bars bite
# (stage, conv, schedule class at the bench shape in bf16x3)
PERTURB = [(0, 'resblocks.2.convs2.2', 'merged, staged, accumulating into the running sum (c2 of the last step)'),
           (1, 'resblocks.3.convs2.1', 'merged, staged, in place (c2 of the middle dilation)'),
           (2, 'resblocks.6.convs1.0', 'fused, one CTA per SM (a c1)'),
           (3, 'resblocks.11.convs2.2', 'fused, two CTAs per SM, accumulating into the running sum (c2 of the last step)')]


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3'])
@pytest.mark.parametrize('stage,conv,what', PERTURB, ids=[p[1] for p in PERTURB])
def test_a_2e_3_weight_error_fails_its_stage_bar(stage, conv, what, precision, monkeypatch, capfd):
    """One conv's weight scaled by 1 + 2e-3 in the module: the handle is rebuilt from the new weights, the reference keeps
    the old ones.  The affected stage must fail its bar by MARGIN, every other group must still pass."""
    m, h = make_model('hop256', precision, monkeypatch)
    w = ref_weights(m)
    with torch.no_grad():
        m.get_parameter(conv + '.weight').mul_(1 + 2e-3)
    mel, y, _ = forward(m, h, 16, 128, monkeypatch, capfd)
    errs = group_errors(m, h, w, mel, y)
    tag = f'B16xT128 {precision} {conv} x (1 + 2e-3)'
    res = errs.pop(f'stage{stage}')
    li = BARS[precision][f'stage{stage}'][0]
    say(capfd, f'MEASURED {describe(tag, f"stage{stage}", res)}: {res[0] / li:.1f} x the bar ({what})')
    assert res[0] >= MARGIN * li, (tag, res, li)
    bad = []
    judge(tag, precision, errs, capfd, bad)
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3'])
def test_per_clip_linf_sees_a_fault_that_batch_l2_dilutes(precision, monkeypatch, capfd):
    """2e-3 x max |ref| added to one 16-row x 32-channel piece of the last clip of the bench shape's stage-3 tap (a copy).
    The per-clip L-inf check fails it by MARGIN.  The relative L2 over the batch sees the piece through the 1 / 32768 share
    of the rows it covers: measured on the H100 above it moves to 3x (bf16x3) / 5x (tf32x3) its bar while L-inf moves to
    95x / 220x, so a fault a few times smaller, or a batch a few times longer, passes a norm over the batch.  Asserted: L2
    sees the fault at least 10x less clearly than per-clip L-inf, relative to their bars."""
    m, h = make_model('hop256', precision, monkeypatch)
    w = ref_weights(m)
    forward(m, h, 16, 128, monkeypatch, capfd)
    ups, got = m.get_tap('ups3'), m.get_tap('stage3')
    refs = [O.stage_forward(w, h, 3, ups[b:b + 1].double()) for b in range(got.shape[0])]
    li, l2 = BARS[precision]['stage3']
    clean = compare(got, refs.__getitem__)
    assert clean[0] <= li and clean[1] <= l2, describe('clean', 'stage3', clean)
    b, r0 = got.shape[0] - 1, 5 * 128 + 3 * 16
    faulty = got.clone()
    faulty[b, :32, r0:r0 + 16] += 2e-3 * float(refs[b].abs().max())
    res = compare(faulty, refs.__getitem__)
    say(capfd, f'MEASURED {describe(f"B16xT128 {precision} one faulty piece", "stage3", res)}: L-inf {res[0] / li:.1f} x '
               f'its bar, relative L2 {res[1] / l2:.2f} x its bar')
    assert res[2][0] == b and r0 <= res[2][2] < r0 + 16, res
    assert res[0] >= MARGIN * li, res
    assert res[1] / l2 * 10 <= res[0] / li, res

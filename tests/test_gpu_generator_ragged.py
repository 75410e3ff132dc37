"""-m gpu: ragged batches through the generator (svb_gen_forward_ragged, svb_gen_spec2wav_ragged_host[_i16], the lengths of
HifiGanGenerator.forward and the list form of HifiGAN.spec2wav_batch).

Every clip of a ragged call must be bit-identical to a B = 1 forward of that clip alone, whatever schedule either call picks
(fused, merged, one launch per conv, MT = 1 or 2, one or two CTAs per SM): a row's value does not depend on which work item
computes it.  Frames past a clip's length are never read (NaN there changes nothing) and its samples past length * hop are 0."""
import contextlib
import io

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
from neuralsvb_b200.utils import synthetic as S
from neuralsvb_b200.vocoders.hifigan import HifiGAN
from oracle import hifigan as O
from tests import gpu_util as U
from tests.test_gpu_generator_forward import BARS, compare, config, make_model, ref_weights

pytestmark = pytest.mark.gpu

PRECISIONS = ['fp32', 'tf32', 'tf32x3', 'bf16x3']
ARCHS = ['hop256', 'hop128', 'resblock2']
# 1 frame, odd counts, 128 k +- 1 frames (and, at every stage, rows just around a multiple of the 128-row tile), and one clip
# of T_max
LENGTHS = [1, 37, 129, 64, 3, 127, 130]
T_MAX = 130


def hop_of(h):
    return int(np.prod(h['upsample_rates']))


def inputs(h, lengths, T, seed=U.SEED):
    """mel [B, n_mel, T], f0 [B, T], rand_ini [B, 9], noise [B, T*hop, 9] (CPU), valid frames / samples finite."""
    B = len(lengths)
    mel, f0 = S.make_mel_f0(B, T, seed)
    ri, nz = S.make_nsf_noise(B, T * hop_of(h), seed)
    return mel, f0, ri, nz


def run(m, mel, f0, ri, nz, lengths=None, seed=7):
    kw = {} if ri is None else dict(rand_ini=ri.cuda(), noise=nz.cuda())
    with torch.no_grad():
        y = m(mel.cuda(), None if f0 is None else f0.cuda(), seed=seed, lengths=lengths, **kw)
    torch.cuda.synchronize()
    return y[:, 0].cpu()


def alone(m, h, mel, f0, ri, nz, b, L, nsf):
    """clip b on its own: B = 1, its first L frames, the same draws"""
    hop = hop_of(h)
    return run(m, mel[b:b + 1, :, :L].contiguous(), f0[b:b + 1, :L].contiguous() if nsf else None,
               ri[b:b + 1] if nsf else None, nz[b:b + 1, :L * hop].contiguous() if nsf else None)[0]


def bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.numpy().view(np.int32), b.numpy().view(np.int32))


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('arch', ARCHS)
def test_each_clip_is_bit_identical_to_its_batch_of_one(arch, precision, monkeypatch):
    """1 (injected NSF draws and the non-NSF call) and 2 (NaN in every padded mel and f0 frame)."""
    m, h = make_model(arch, precision, monkeypatch)
    hop = hop_of(h)
    mel, f0, ri, nz = inputs(h, LENGTHS, T_MAX)
    bad = []
    for nsf in (True, False):
        y = run(m, mel, f0 if nsf else None, ri if nsf else None, nz if nsf else None, LENGTHS)
        melp, f0p = mel.clone(), f0.clone()
        for b, L in enumerate(LENGTHS):
            melp[b, :, L:] = float('nan')
            f0p[b, L:] = float('nan')
        yp = run(m, melp, f0p if nsf else None, ri if nsf else None, nz if nsf else None, LENGTHS)
        assert bits_equal(y, yp), f'{arch} {precision} nsf={nsf}: NaN in padded frames changed the output'
        for b, L in enumerate(LENGTHS):
            one = alone(m, h, mel, f0, ri, nz, b, L, nsf)
            got = y[b, :L * hop]
            if not bits_equal(got, one):
                d = (got - one).abs()
                t = int(d.argmax())
                bad.append(f'{arch} {precision} nsf={nsf} clip {b} (L {L}): {int((d > 0).sum())} samples differ, max '
                           f'{float(d.max()):.3e} at sample {t} (frame {t // hop})')
            assert torch.isfinite(yp[b, :L * hop]).all()
            assert (y[b, L * hop:] == 0).all() and (yp[b, L * hop:] == 0).all()
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('precision', PRECISIONS)
def test_equal_lengths_reproduce_the_uniform_call_in_philox_mode(precision, monkeypatch):
    """3: lengths all T_max give the uniform svb_gen_forward's output bit for bit, NSF draws from the seed."""
    m, h = make_model('hop256', precision, monkeypatch)
    B, T = 4, 129
    mel, f0, _, _ = inputs(h, [T] * B, T)
    y0 = run(m, mel, f0, None, None, None, seed=11)
    y1 = run(m, mel, f0, None, None, [T] * B, seed=11)
    assert bits_equal(y0, y1)


@pytest.mark.parametrize('precision', ['bf16x3', 'fp32'])
def test_a_short_call_after_a_long_one_on_one_handle(precision, monkeypatch):
    """4: rows a longer call left behind past a clip's new end are zeroed before they reach a halo."""
    m, h = make_model('hop256', precision, monkeypatch)
    T = 130
    mel, f0, ri, nz = inputs(h, [T] * 3, T)
    run(m, mel, f0, ri, nz, [130, 64, 3])
    run(m, mel, f0, ri, nz, None)                                   # the uniform call leaves every row live
    y_short = run(m, mel, f0, ri, nz, [5, 64, 129])
    fresh, _ = make_model('hop256', precision, monkeypatch)
    y_fresh = run(fresh, mel, f0, ri, nz, [5, 64, 129])
    assert bits_equal(y_short, y_fresh)


def clip_errors(m, h, w, mel, y, lengths):
    """compare(...) of every launch group of clip b of the last ragged forward, on its own valid rows, against the float64
    oracle run on that clip alone (test_gpu_generator_forward.group_errors, one clip at a time)."""
    n = len(h['upsample_rates'])
    hop = hop_of(h)
    mel = mel.to(w['conv_pre.weight'].device, torch.float64)
    taps = {k: m.get_tap(k) for k in ['conv_pre'] + [f'{p}{i}' for i in range(n) for p in ('ups', 'stage')]}
    har = m.get_tap('har_source') if h['use_pitch_embed'] else None
    worst = {}

    def put(name, res):
        if name not in worst or res[0] > worst[name][0]:
            worst[name] = res
    for b, L in enumerate(lengths):
        hb = None if har is None else har[b:b + 1, ..., :L * hop].double()
        put('conv_pre', compare(taps['conv_pre'][b:b + 1, :, :L],
                                lambda _: F.conv1d(mel[b:b + 1, :, :L], w['conv_pre.weight'], w['conv_pre.bias'], padding=3)))
        x, r = taps['conv_pre'][b:b + 1, :, :L], L
        for i in range(n):
            r *= h['upsample_rates'][i]
            ups = taps[f'ups{i}'][b:b + 1, :, :r]
            put(f'ups{i}', compare(ups, lambda _: O.upsample_forward(w, h, i, x.double(), hb)))
            x = taps[f'stage{i}'][b:b + 1, :, :r]
            put(f'stage{i}', compare(x, lambda _: O.stage_forward(w, h, i, ups.double())))
        put('wave', compare(y[b:b + 1, None, :L * hop].cuda(), lambda _: O.post_forward(w, h, x.double())))
    return worst


@pytest.mark.parametrize('arch,precision', [('hop256', p) for p in PRECISIONS] + [('hop128', 'bf16x3'), ('resblock2', 'bf16x3')])
def test_each_clip_matches_float64_on_its_own(arch, precision, monkeypatch):
    """5: every launch group of every clip, on the kernels' own inputs cut to the clip, against the float64 oracle on that clip
    alone, within the bars of test_gpu_generator_forward.py."""
    m, h = make_model(arch, precision, monkeypatch)
    mel, f0, ri, nz = inputs(h, LENGTHS, T_MAX)
    y = run(m, mel, f0, ri, nz, LENGTHS)
    bad = []
    for tap, res in clip_errors(m, h, ref_weights(m), mel, y, LENGTHS).items():
        li, _ = BARS[precision][tap]
        print(f'MEASURED {arch} {precision} {tap}: worst per-clip L-inf {res[0]:.2e} at {res[2]}')
        if not res[0] <= li:
            bad.append(f'{arch} {precision} {tap}: L-inf {res[0]:.2e} > {li:.0e}')
    assert not bad, '\n'.join(bad)


def vocoder(precision='bf16x3'):
    h = S.hifigan_config(True)
    m = HifiGanGenerator(h, precision=precision)
    m.load_state_dict(S.make_generator_state_dict(h, U.SEED), strict=True)
    with contextlib.redirect_stdout(io.StringIO()):
        m.remove_weight_norm()
    return HifiGAN.from_model(m.eval().cuda(), h), h


def test_list_spec2wav_batch_equals_spec2wav_clip_by_clip():
    """6: float, int16 and int16 with per-clip peak normalisation; the list form with f0 equals the ragged forward."""
    voc, h = vocoder()
    mel, f0, _, _ = inputs(h, LENGTHS, T_MAX)
    mels = [mel[b, :, :L].T.contiguous().numpy() for b, L in enumerate(LENGTHS)]
    f0s = [f0[b, :L].numpy() for b, L in enumerate(LENGTHS)]
    hop = hop_of(h)
    got = voc.spec2wav_batch(mels)
    assert [g.shape for g in got] == [(L * hop,) for L in LENGTHS]
    for g, m1 in zip(got, mels):
        assert bits_equal(torch.from_numpy(g), torch.from_numpy(voc.spec2wav(m1)))
    for norm in (False, True):
        got16 = voc.spec2wav_batch(mels, int16=True, norm=norm)
        for g, m1 in zip(got16, mels):
            want = voc.spec2wav_batch(m1[None], int16=True, norm=norm)[0]
            assert g.dtype == np.int16 and np.array_equal(g, want)
            if norm:
                assert np.abs(g.astype(np.int32)).max() == 32767       # each clip at its own peak
    # with f0: the same as the ragged forward with the same seed (Philox draws keyed by clip and sample)
    got_f0 = voc.spec2wav_batch(mels, f0s, seed=5)
    want = run(voc.model, mel, f0, None, None, LENGTHS, seed=5)
    for b, L in enumerate(LENGTHS):
        assert bits_equal(torch.from_numpy(got_f0[b]), want[b, :L * hop])
    # an array batch behaves exactly as before
    arr = voc.spec2wav_batch(mel[:2].transpose(1, 2).contiguous().numpy())
    assert arr.shape == (2, T_MAX * hop)


def test_training_handles_and_bad_lengths_raise(monkeypatch):
    """7"""
    m, h = make_model('hop256', 'fp32', monkeypatch, train=True)
    mel, f0, ri, nz = inputs(h, [8, 5], 8)
    with pytest.raises(RuntimeError):
        m(mel.cuda(), f0.cuda(), lengths=[8, 5])                     # autograd needed
    m2, _ = make_model('hop256', 'bf16x3', monkeypatch)
    for bad in ([0, 5], [9, 5], [8]):
        with pytest.raises(ValueError):
            run(m2, mel, f0, None, None, bad)
    voc, _ = vocoder()
    with pytest.raises(ValueError):
        voc.spec2wav_batch([mel[0].T.numpy(), np.zeros((0, 80), np.float32)])
    # the C ABI checks the lengths itself, before the GPU is touched
    import ctypes
    from neuralsvb_b200 import _native
    lib = _native.lib()
    g = m2.native_handle(torch.device('cuda', 0))
    y = torch.empty(2, 8 * hop_of(h), device='cuda')
    for bad in ([0, 5], [9, 5]):
        ln = np.array(bad, np.int32)
        rc = lib.svb_gen_forward_ragged(g, _native.ptr(mel.cuda()), None, None, None, ctypes.c_uint64(1), 2, 8,
                                        ln.ctypes.data_as(ctypes.c_void_p), _native.ptr(y), None)
        assert rc == -1                                             # SVB_ERR_INVALID
    # a training handle (after a training forward) given lengths: SVB_ERR_STATE
    m(mel.cuda(), f0.cuda(), rand_ini=ri.cuda(), noise=nz.cuda()).sum().backward()
    ln = np.array([8, 5], np.int32)
    rc = lib.svb_gen_forward_ragged(m.native_handle(torch.device('cuda', 0)), _native.ptr(mel.cuda()), None, None, None,
                                    ctypes.c_uint64(1), 2, 8, ln.ctypes.data_as(ctypes.c_void_p), _native.ptr(y), None)
    assert rc == -3

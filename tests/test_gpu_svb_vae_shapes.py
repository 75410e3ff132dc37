"""MleSVBVAE at the shapes the benchmarks time and on ragged batches, against float64 torch (oracle/svb_vae.py, oracle/svb_vae_train.py
with every weight and input cast to float64 on the GPU).  bench.py's pipeline_cfg5 runs the eval-mode forward (a2a + p2p + a2p) on
make_svb_batch(8, 688, 688, 1234); tools/svb_train_bench.py runs the phase-2 and phase-3 steps on make_svb_batch(16, 1024, 1024).

  A  the eval-mode forward, every output and the conditions, at those shapes, on ragged batches, at the shortest clip and a long one;
  B  every clip of a ragged batch equals the same clip run alone;
  C  frame counts the float64 oracle rejects are rejected by the model too, before any launch;
  D  the training steps (with and without the adversarial terms) on a ragged batch of 8 and at 16 x 1024;
  E  the tensor-core step bars fail on a 2e-3 error in one convolution, on one stale weight packing and on a 2e-3 error of the decoder;
  F  three AdamW steps per phase leave no stale packing or running statistic behind.

Errors are relative L2 and L-inf relative to max |reference|."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200.utils import synthetic as S
from tests.test_gpu_svb_vae_train import MAP_ZERO_GRAD, _compare_step, _set_phase, _tied_step
from tests.test_gpu_wn_train import _check
from tests.test_oracle_golden import SVB_HP

# (rel L2, rel L-inf) bars, about 5x the worst error measured on an H100 80GB HBM3 (DESIGN section 8), keyed by vc_modules.USE_TC
# (False: fp32 CUDA cores, True: bf16x3 tensor cores).
# Eval forward, every output of every shape (700 W power limit): worst 1.6e-6 / 2.1e-6 fp32, 1.5e-5 / 1.7e-5 bf16x3 (h_content of the
# cfg-5 batch).
FWD_BARS = {False: (8e-6, 1e-5), True: (7.5e-5, 9e-5)}
# Steps, on the native PPG, BatchNorm inputs and ReLU masks (tests/test_gpu_svb_vae_train._tied_step), worst over three runs at a
# 400 W power limit (gradients / loss values):
#   ragged 8 x 688, phase 2: fp32 4.0e-6 / 6.2e-6 and 3.3e-7; bf16x3 4.1e-5 / 5.1e-5 (the posterior encoder) and 4.0e-6;
#   16 x 1024, phase 2 bf16x3: 3.9e-4 / 8.5e-4 (upsample_layer.0.1 and pitch_embed, whose weight gradients sum over 16k frames);
#   phase 3, both shapes: fp32 2.9e-6 / 3.6e-6 and 3.3e-7; bf16x3 2.1e-5 / 2.6e-5 and 5.9e-6; running statistics 1.5e-7.
# The E tests inject 2e-3 errors on the ragged batch, 8x or more above its bf16x3 bars.  At 16 x 1024 the bf16x3 phase-2 gradient
# bar is the size of such an error.
STEP_BARS = {False: {None: (2e-5, 3e-5), 'loss': (1.7e-6, 1.7e-6)}, True: {None: (2e-4, 2.6e-4), 'loss': (2e-5, 2e-5)}}
TRAIN_BENCH_STEP_BARS = {False: STEP_BARS[False], True: {None: (2e-3, 4.3e-3), 'loss': (2e-5, 2e-5)}}
MAP_BARS = {False: {None: (1.5e-5, 1.8e-5), 'loss': (1.7e-6, 1.7e-6)}, True: {None: (1.1e-4, 1.3e-4), 'loss': (3e-5, 3e-5)}}
FRAMES_MULTIPLE = 4                  # vae_global_mle_eng's frames_multiple: the reference's loader crops every clip to a multiple of it
SHORTEST = 60                        # the posterior encoder's three k = 3 stride-2 poolings need T / 4 >= 15 frames


# ---------------------------------------------------------------------------------------------------------- batches
def _ragged(La, Lp, seed, Ta=None, Tp=None, n_mel=80):
    """A batch whose clip b has La[b] amateur and Lp[b] professional frames (multiples of FRAMES_MULTIPLE), each row padded to Ta / Tp
    (default: the longest clip) as the reference's collate pads: zero mel frames, pitch 0, alignment 0.  Pitch ids in [1, 255] inside
    a clip, different amateur and professional speakers, and an a2p alignment that follows the tempo ratio of each clip with a jitter
    of one frame and stays inside that clip's amateur frames."""
    B = len(La)
    Ta, Tp = Ta or max(La), Tp or max(Lp)
    assert all(n % FRAMES_MULTIPLE == 0 for n in list(La) + list(Lp) + [Ta, Tp])
    rs = np.random.RandomState(seed)
    a_mel, p_mel = np.zeros((B, Ta, n_mel), np.float32), np.zeros((B, Tp, n_mel), np.float32)
    a_pitch, p_pitch = np.zeros((B, Ta), np.int64), np.zeros((B, Tp), np.int64)
    align = np.zeros((B, Tp), np.int64)
    for b in range(B):
        a_mel[b, :La[b]] = (rs.randn(La[b], n_mel) * 1.2 - 2.5).clip(-6, 1.5)
        p_mel[b, :Lp[b]] = (rs.randn(Lp[b], n_mel) * 1.2 - 2.5).clip(-6, 1.5)
        a_pitch[b, :La[b]], p_pitch[b, :Lp[b]] = rs.randint(1, 256, La[b]), rs.randint(1, 256, Lp[b])
        align[b, :Lp[b]] = np.minimum((np.arange(Lp[b]) * La[b] / Lp[b]).astype(np.int64) + rs.randint(0, 2, Lp[b]), La[b] - 1)
    t = torch.from_numpy
    return dict(amateur_mel=t(a_mel), prof_mel=t(p_mel), amateur_pitch=t(a_pitch), prof_pitch=t(p_pitch),
                amateur_spk_id=t((rs.randn(B, 256) * 0.5).astype(np.float32)), prof_spk_id=t((rs.randn(B, 256) * 0.5).astype(np.float32)),
                a2p_alignment=t(align))


def _lengths(B, seed, T=688, spread=0.15):
    """Clip lengths of T +- spread (8 s at hop 256 is 688 frames), cropped to FRAMES_MULTIPLE as the reference's loader does."""
    rs = np.random.RandomState(seed)
    return [int(T * rs.uniform(1 - spread, 1 + spread)) // FRAMES_MULTIPLE * FRAMES_MULTIPLE for _ in range(B)]


def _ragged8():
    return _ragged(_lengths(8, 1), _lengths(8, 2), 11)


SHAPES = {
    'cfg5_8x688': lambda: S.make_svb_batch(8, 688, 688, 1234),                # exactly the batch pipeline_cfg5 times
    'ragged_8x688': _ragged8,
    'b1_shortest': lambda: _ragged([SHORTEST], [SHORTEST], 12),
    'b3_uneven': lambda: _ragged([300, 212, 76], [236, 332, 68], 13),          # Ta != Tp, no multiple of 32; clip 2 fills a quarter of its rows
    'long_pair': lambda: _ragged([1376], [1380], 14),
}


def _eps(B, kind):
    if kind == 'zero':
        return torch.zeros(B, 128, 1)
    return torch.randn(B, 128, 1, generator=torch.Generator().manual_seed(B + 5))


# ---------------------------------------------------------------------------------------------------------- models
@pytest.fixture(params=[False, True], ids=['fp32_cuda_cores', 'bf16x3_tensor_cores'])
def use_tc(request, monkeypatch):
    from neuralsvb_b200.modules.fastspeech import multi_window_disc as M
    from neuralsvb_b200.modules.voice_conversion import vc_modules as V
    monkeypatch.setattr(V, 'USE_TC', request.param)
    monkeypatch.setattr(M, 'USE_TC', request.param)
    return request.param


def _model(use_tc, trainable=False, sd=None):
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    m = MleSVBVAE(80, hp=SVB_HP, precision='bf16x3' if use_tc else 'fp32', trainable=trainable)
    m.load_state_dict(S.make_svb_state_dict(1234) if sd is None else sd, strict=True)
    return m.cuda()


def _native_forward(m, batch, eps):
    """Every output of the eval-mode forward plus the amateur conditions, keyed as _oracle_forward keys them."""
    b = {k: v.cuda() for k, v in batch.items()}
    with torch.no_grad():
        r = m(**b, infer=False, concurrent_ways=['a2a', 'p2p', 'a2p'], eps=eps.cuda())
        c = m.prepare_condition(b['amateur_mel'], b['amateur_pitch'], spk_ids=b['amateur_spk_id'])
    return _outputs(r, c)


def _outputs(r, c):
    out = {f'{w} mel_out': r[w]['mel_out'] for w in ('a2a', 'p2p', 'a2p')}
    for w in ('a2a', 'p2p'):
        out.update({f'{w} {k}': r[w][k] for k in ('m_q', 'logs_q', 'kl')})
    out.update({'a2p mle': r['a2p']['mle'], 'h_content': c['h_content'], 'h_pitch': c['h_pitch']})
    return out


def _oracle_forward(batch, eps, sd=None):
    """The float64 oracle's outputs, keyed as _native_forward keys them, at ``sd`` (a model's state_dict; default the weights
    _model loads)."""
    from oracle import fs2_vae as OF
    from oracle import svb_vae as OS
    sd = S.make_svb_state_dict(1234) if sd is None else sd
    w = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in sd.items()}
    b = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in batch.items()}
    with torch.no_grad(), torch.device('cuda'):            # oracle/vc_asr.py builds its position table on the default device
        r = OS.mle_svb_vae_forward(w, b, eps.cuda().double())
        c = OS.prepare_condition(OF.fold_weight_norm(w), b['amateur_mel'], b['amateur_pitch'], b['amateur_spk_id'])
    return _outputs(r, c)


# ---------------------------------------------------------------------------------------------------------- A: eval forward
@pytest.mark.gpu
@pytest.mark.parametrize('eps_kind', ['zero', 'randn'])
@pytest.mark.parametrize('shape', list(SHAPES))
def test_eval_forward_matches_float64(use_tc, shape, eps_kind):
    batch = SHAPES[shape]()
    eps = _eps(batch['amateur_mel'].shape[0], eps_kind)
    got = _native_forward(_model(use_tc).eval(), batch, eps)
    ref = _oracle_forward(batch, eps)
    assert tuple(got['a2p mel_out'].shape) == tuple(batch['prof_mel'].shape)
    for k in ref:                       # conditions first: a failure there points at the stage
        _check(f'fwd {shape} {eps_kind} tc={use_tc} {k}', got[k].reshape(-1), ref[k].reshape(-1), FWD_BARS[use_tc])


# ---------------------------------------------------------------------------------------------------------- B: batch independence
@pytest.mark.gpu
def test_ragged_batch_clips_equal_clips_run_alone(use_tc):
    """Each clip's outputs in the ragged batch of 8 are bit-identical to the same clip run alone in a row of the same length: no
    kernel mixes clips or orders a reduction by the batch size.  The KL and MLE terms are batch means and are left out."""
    batch = _ragged8()
    B = batch['amateur_mel'].shape[0]
    eps = _eps(B, 'randn')
    m = _model(use_tc).eval()
    full = _native_forward(m, batch, eps)
    for b in range(B):
        one = _native_forward(m, {k: v[b:b + 1] for k, v in batch.items()}, eps[b:b + 1])
        for k, v in one.items():
            if v.dim() == 0:
                continue
            d = float((full[k][b:b + 1] - v).abs().max())
            assert torch.equal(full[k][b:b + 1], v), (b, k, d)


# ---------------------------------------------------------------------------------------------------------- C: length contract
BAD_FRAMES = [(62, 64), (64, 62), (61, SHORTEST), (56, SHORTEST), (SHORTEST, 56), (28, 64)]


def _cpu_model_and_oracle_weights():
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    sd = S.make_svb_state_dict(1234)
    m = MleSVBVAE(80, hp=SVB_HP).eval()
    m.load_state_dict(sd, strict=True)
    return m, {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


def _cpu_batch(Ta, Tp):
    batch = S.make_svb_batch(1, Ta, Tp, 3)
    return batch, {k: (v.double() if v.is_floating_point() else v) for k, v in batch.items()}


@pytest.mark.parametrize('Ta,Tp', BAD_FRAMES)
def test_oracle_and_model_reject_the_same_frame_counts(Ta, Tp):
    """On the CPU: the float64 oracle fails on a frame count that is not a multiple of 4 (the decoder rebuilds 4 * (T // 4) frames,
    which do not meet the mask) and below 60 frames (a pooling finds fewer frames than its kernel); the model raises on the same
    counts before it launches anything."""
    from oracle import svb_vae as OS
    m, w = _cpu_model_and_oracle_weights()
    batch, b64 = _cpu_batch(Ta, Tp)
    with torch.no_grad():
        with pytest.raises(RuntimeError):
            OS.mle_svb_vae_forward(w, b64, torch.zeros(1, 128, 1, dtype=torch.float64))
        with pytest.raises(ValueError, match='frames'):
            m(**batch, concurrent_ways=['a2a', 'p2p', 'a2p'])


def test_oracle_and_model_take_the_shortest_clip():
    """60 x 60 runs through the float64 oracle, and the model's frame check lets it pass (to the first convolution, which has no
    CPU path)."""
    from oracle import svb_vae as OS
    m, w = _cpu_model_and_oracle_weights()
    batch, b64 = _cpu_batch(SHORTEST, SHORTEST)
    with torch.no_grad():
        assert OS.mle_svb_vae_forward(w, b64, torch.zeros(1, 128, 1, dtype=torch.float64))['a2p']['mel_out'].shape == (1, SHORTEST, 80)
        with pytest.raises(RuntimeError, match='CUDA'):
            m(**batch, concurrent_ways=['a2a', 'p2p', 'a2p'])


@pytest.mark.gpu
@pytest.mark.parametrize('Ta,Tp', BAD_FRAMES)
def test_model_on_gpu_rejects_frame_counts_the_oracle_rejects(Ta, Tp):
    """Inference and training alike raise; before this check 28-56 frames returned NaN latents (the last pooling produced no frame
    and its mean was taken over an empty axis) instead of failing as the reference does."""
    batch = {k: v.cuda() for k, v in S.make_svb_batch(1, Ta, Tp, 3).items()}
    m = _model(True).eval()
    with torch.no_grad(), pytest.raises(ValueError, match='frames'):
        m(**batch, concurrent_ways=['a2a', 'p2p', 'a2p'])
    t = _model(True, trainable=True)
    _set_phase(t, 2)
    with pytest.raises(ValueError, match='frames'):
        t(**batch, concurrent_ways=['a2a', 'p2p'])


# ---------------------------------------------------------------------------------------------------------- D: training steps
def _disc():
    from tests.test_gpu_mel_disc import _disc as make
    d = make().train()
    d.requires_grad_(False)
    return d


def _adv_terms(disc, phase, batch, seed=50):
    """(native extra, oracle extra): the adversarial terms of the step ({a2a,p2p}_a in phase 2, a2p_a in phase 3) from the frozen
    train-mode discriminator, the oracle on the discriminator's own leaky-relu masks and the same starts and Dropout2d masks."""
    from oracle import multi_window_disc as OD
    from tests.test_gpu_mel_disc import _draw, _masks, _native_masks, _sd64
    B, Ta, Tp = batch['amateur_mel'].shape[0], batch['amateur_mel'].shape[1], batch['prof_mel'].shape[1]
    adv = ['a2a', 'p2p'] if phase == 2 else ['a2p']
    draws = [_draw(disc, B, Ta if w == 'a2a' else Tp, seed + k) for k, w in enumerate(adv)]
    rec = []

    def native(ret):
        out = {}
        with _native_masks(rec):
            for k, w in enumerate(adv):
                y = disc(ret[w]['mel_out'], start_frames_wins=draws[k][0], dropout_scales=draws[k][1])['y']
                out[f'{w}_a'] = F.mse_loss(y, torch.ones_like(y)) * OD.LAMBDA_MEL_ADV
        return out

    def oracle(out):
        return OD.svb_adv_losses(_sd64(disc, False), 'g' if phase == 2 else 3, {w: out[w]['mel_out'] for w in adv},
                                 starts=[d[0] for d in draws], scales=[[[s.double() for s in w] for w in d[1]] for d in draws],
                                 masks=_masks(rec, len(adv)))
    return native, oracle


def _train_step(m, phase, batch, disc=None):
    """One tied step (tests/test_gpu_svb_vae_train._tied_step), with the adversarial terms when ``disc`` is given."""
    ne, oe = _adv_terms(disc, phase, batch) if disc is not None else (None, None)
    return _tied_step(m, phase, batch, native_extra=ne, oracle_extra=oe)


def _compare(tag, m, phase, step, use_tc, step_bars=STEP_BARS):
    losses, ref, p = step
    bars = (step_bars if phase == 2 else MAP_BARS)[use_tc]
    return _compare_step(tag, m, phase, losses, ref, p, bars, zero_grad=MAP_ZERO_GRAD if phase == 3 else ())


def _trainable(use_tc, phase):
    m = _model(use_tc, trainable=True)
    _set_phase(m, phase)
    return m


@pytest.mark.gpu
@pytest.mark.parametrize('adv', [False, True], ids=['mel_losses', 'with_adversarial'])
@pytest.mark.parametrize('phase', [2, 3])
def test_steps_on_ragged_batch_match_float64(use_tc, phase, adv):
    batch = _ragged8()
    m = _trainable(use_tc, phase)
    step = _train_step(m, phase, batch, _disc() if adv else None)
    n = _compare(f'ragged8 phase{phase} adv={adv} tc={use_tc}', m, phase, step, use_tc)
    assert n > 100 if phase == 2 else n == len(list(m.z_mapping_function.parameters()))
    sd, p = m.state_dict(), step[2]
    running = ['upsample_layer.0.3', 'vae_model.encoder.poolings.2', 'vae_model.encoder.poolings.5'] if phase == 2 else \
        ['z_mapping_function.convs.1', 'z_mapping_function.convs.4']
    for pre in running:
        for s in ('running_mean', 'running_var'):
            _check(f'ragged8 phase{phase} adv={adv} tc={use_tc} {pre}.{s}', sd[f'{pre}.{s}'], p[f'{pre}.{s}'],
                   (STEP_BARS if phase == 2 else MAP_BARS)[use_tc][None])


@pytest.mark.gpu
@pytest.mark.parametrize('phase', [2, 3])
def test_steps_at_train_bench_shape_match_float64(use_tc, phase):
    """make_svb_batch(16, 1024, 1024), the batch tools/svb_train_bench.py times."""
    m = _trainable(use_tc, phase)
    n = _compare(f'16x1024 phase{phase} tc={use_tc}', m, phase, _train_step(m, phase, S.make_svb_batch(16, 1024, 1024, 1234)), use_tc,
                 TRAIN_BENCH_STEP_BARS)
    assert n > 100 if phase == 2 else n == len(list(m.z_mapping_function.parameters()))


# ---------------------------------------------------------------------------------------------------------- E: the bars can fail
def _fails(tag, m, phase, step):
    with pytest.raises(AssertionError) as e:
        _compare(tag, m, phase, step, True)
    print(f'FAILS {tag}: {e.value}')


@pytest.fixture
def bf16x3(monkeypatch):
    from neuralsvb_b200.modules.voice_conversion import vc_modules as V
    monkeypatch.setattr(V, 'USE_TC', True)


@pytest.mark.gpu
@pytest.mark.parametrize('layer', ['upsample_layer.1.weight', 'encoded_embed_proj.weight'])
def test_bars_fail_on_one_conv_off_by_2e_3(bf16x3, monkeypatch, layer):
    """One tensor-core convolution whose output is 2e-3 too large, the size of a dropped hi x lo cross term of bf16x3.  (A
    convolution straight in front of a BatchNorm would be invisible: the norm removes a per-channel scale, forward and backward.)"""
    from neuralsvb_b200.modules.hifigan import discriminators as D
    m = _trainable(True, 2)
    target, orig, hits = m.get_parameter(layer), D.conv_tc, []

    def conv_tc(x, w, *a, **k):
        y = orig(x, w, *a, **k)
        if w is target or (w.dim() == 3 and target.dim() == 2 and w._base is target):
            hits.append(1)
            return y * (1 + 2e-3)
        return y
    monkeypatch.setattr(D, 'conv_tc', conv_tc)
    step = _train_step(m, 2, _ragged8())
    assert hits
    _fails(f'conv {layer} x (1 + 2e-3)', m, 2, step)


@pytest.mark.gpu
@pytest.mark.parametrize('what', ['tc_layer', 'decoder_versions'])
def test_bars_fail_on_one_stale_packing_after_adamw(bf16x3, monkeypatch, what):
    """One AdamW step, then one layer keeps the packing of the weights before it: the tensor-core handle of
    encoded_embed_proj (_tc_sync_weight skipped), or the mel decoder's WN handle (its parameter versions marked current)."""
    from neuralsvb_b200.modules.hifigan import discriminators as D
    batch = _ragged8()
    m = _trainable(True, 2)
    opt = torch.optim.AdamW([q for q in m.parameters() if q.requires_grad], lr=1e-3)
    _train_step(m, 2, batch)
    opt.step()
    opt.zero_grad(set_to_none=True)
    if what == 'tc_layer':
        layer, orig = m.encoded_embed_proj.weight._svb_tc_layer, D._tc_sync_weight
        monkeypatch.setattr(D, '_tc_sync_weight', lambda lay, *a, **k: None if lay is layer else orig(lay, *a, **k))
    else:
        dec = m.vae_model.decoder
        dec._versions = tuple(q._version for q in dec.parameters()) + (str(torch.device('cuda', torch.cuda.current_device())),)
    _fails(f'stale {what}', m, 2, _train_step(m, 2, batch))


@pytest.mark.gpu
@pytest.mark.parametrize('phase', [2, 3])
def test_bars_fail_on_decoder_output_off_by_2e_3(bf16x3, monkeypatch, phase):
    """The mel decoder's output 2e-3 too large at the Python boundary (every a2a / p2p / a2p decode)."""
    from neuralsvb_b200.modules.fastspeech import fs2_vae as FV
    orig = FV.FVAEDecoder.forward
    monkeypatch.setattr(FV.FVAEDecoder, 'forward', lambda self, *a: orig(self, *a) * (1 + 2e-3))
    m = _trainable(True, phase)
    _fails(f'decoder x (1 + 2e-3) phase{phase}', m, phase, _train_step(m, phase, _ragged8()))


# ---------------------------------------------------------------------------------------------------------- F: no stale packings
@pytest.mark.gpu
def test_adamw_steps_leave_no_stale_packing(use_tc):
    """Three AdamW steps of phase 2, then three of phase 3, on one model; its eval-mode forward is then bit-identical to a new model
    loaded with the same state_dict: the tensor-core handles of every dense conv (the PPG extractor's included), the WN and decoder
    handles and the BatchNorm running statistics all hold what the parameters and buffers say."""
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    batch = _ragged(_lengths(4, 21), _lengths(4, 22), 23)
    b = {k: v.cuda() for k, v in batch.items()}
    B = b['amateur_mel'].shape[0]
    m = _model(use_tc, trainable=True)
    for phase in (2, 3):
        _set_phase(m, phase)
        opt = torch.optim.AdamW([q for q in m.parameters() if q.requires_grad], lr=1e-3)
        ways = ['a2a', 'p2p'] if phase == 2 else ['a2a', 'p2p', 'a2p']
        for _ in range(3):
            opt.zero_grad(set_to_none=True)
            ret = m(**b, concurrent_ways=ways, eps=torch.zeros(B, 128, 1, device='cuda'))
            loss = sum(sum(mel_l1_ssim_loss(ret[w]['mel_out'], b['amateur_mel' if w == 'a2a' else 'prof_mel'])) for w in ways)
            loss = loss + (ret['a2p']['mle'] if phase == 3 else 0)
            loss.backward()
            opt.step()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    assert not torch.equal(sd['vae_model.decoder.out_proj.weight'], S.make_svb_state_dict(1234)['vae_model.decoder.out_proj.weight'].cuda())
    eps = _eps(B, 'randn')
    got = _native_forward(m.eval(), batch, eps)
    # A new model builds its WN and decoder handles from weights folded by torch (weight_g * v / |v|); after an optimizer step a
    # trained one receives them folded on the device (_WeightNormFn), which rounds differently (1.6e-5 on a2a mel_out).  So the new
    # model takes the same route: one forward builds its handles, a version bump of every parameter (values unchanged) makes the
    # next forward hand them the device-folded weights.
    new = _model(use_tc, trainable=True, sd=sd).eval()
    _native_forward(new, batch, eps)
    with torch.no_grad():
        for q in new.parameters():
            q.mul_(1)
    ref = _native_forward(new, batch, eps)
    diffs = {k: float((got[k] - ref[k]).abs().max()) for k in ref}
    print(f'ERR stale tc={use_tc} max |trained - new| {diffs}')
    assert all(torch.equal(got[k], ref[k]) for k in ref), diffs

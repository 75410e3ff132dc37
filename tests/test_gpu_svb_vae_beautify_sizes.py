"""MleSVBVAE at the sizes the beautifier runs it, against float64 torch (oracle/svb_vae.py, oracle/svb_vae_train.py on the GPU in
float64, called with the model's own state_dict).  beautify_batch takes pairs of up to max_frames = 5000 frames; beautify_songs
runs the model once per song on all of that song's segments of up to 5000 frames, the short tail segment padded to the longest.

  A  max_frames clips (B = 1): (Ta, Tp) = (5000, 5000), (5000, 2996), (3000, 5000), eps zero and randn.  The mel decoder runs its
     WN at the full frame rate, so T > 4224 takes the second pass of the WN elementwise kernels' grid-stride loops (528 blocks of 8
     frames), and the conformer runs at 2500 frames, 4999 rows of its 5000-position table;
  B  the batches the beautifier builds, recorded at the model's forward: the segment batch of one 4-minute song (beautify_songs)
     and 64 pairs of 8 s +- 15 % at hop 128 with one max_frames pair and one 60-frame pair (beautify_batch);
  C  every row of those batches equals the same clip run alone at the same padded lengths, bit for bit; and how far the float64
     oracle's own output moves between a clip padded in its batch and the same clip alone and unpadded;
  D  one phase-2 and one phase-3 step on [5000, 1236, 60] amateur x [4996, 1300, 60] professional frames: the WN backward
     grid-stride loops and weight-gradient sums over ~6300 frames;
  E  the bars catch a 2e-3 error in the decoder rows only the grid-stride pass writes, and in the song's short tail segment alone.

Every output of _outputs is checked, the conditions first, at fp32 (CUDA cores) and bf16x3 (tensor cores, the beautifier's
svb_precision), two ways: per clip (over that clip's own frames, relative to that clip's own max |reference|, so the long clips
cannot hide a fault in a short one) and on the whole tensor, padded rows included.  Errors are relative L2 and L-inf relative to
max |reference|.

The batches of B and C are compared with the oracle run one clip at a time, each padded to the batch's Ta / Tp (eval-mode BatchNorm
keeps the oracle per clip, so this gives the batch's values, and a whole-batch float64 attention at 64 x 2500 frames would need
tens of GB).  The KL and MLE terms are batch means and are recombined from the per-clip terms: the MLE as the mean over clips, each
KL weighted by the clip's latent frames (the mask the KL averages over).

Worst errors measured on an H100 80GB HBM3 at a 700 W power limit (DESIGN section 8), identical over three runs:
  forward, every output, per clip and whole (A and B): fp32 1.6e-6 / 2.8e-6, bf16x3 1.7e-5 / 2.1e-5 (h_content); the benchmark
  shapes' FWD_BARS hold;
  steps (gradients / loss values / running statistics): phase 2 fp32 2.1e-5 / 5.0e-5 (the pitch encoder's convolution weights),
  bf16x3 4.7e-5 / 6.3e-5 (the same), losses 1.3e-7, running statistics 1.8e-7; phase 3 fp32 1.3e-6 / 1.9e-6, bf16x3 4.8e-6 /
  4.5e-6.  The fp32 phase-2 gradient is 5x its value on 8 x 688 frames and sits at STEP_BARS[False]: the fp32 weight gradients
  (svb_conv_nct_backward) are float32 sums over the batch's frames, each partial sum here a few thousand frames long.  So that
  step takes its own bar, 5x the measured error; every other check uses the bars of the benchmark shapes unchanged;
  E: the grid-stride rows miss the bf16x3 forward bar 38x, the song's tail 89x (its whole-tensor L2 only 13x).
Wall time about 2.5 minutes; torch.cuda.max_memory_allocated peaks at 6.2 GiB (the 64-pair batch)."""
import numpy as np
import pytest
import torch

from neuralsvb_b200.inference import beautify as BF
from neuralsvb_b200.utils import hparams as H
from tests.test_gpu_beautify import Spy as BatchSpy
from tests.test_gpu_beautify import make_experiment
from tests.test_gpu_song import Spy as SongSpy
from tests.test_gpu_song import song
from tests.test_gpu_svb_vae_shapes import FWD_BARS, _eps, _model, _native_forward, _oracle_forward, _ragged, bf16x3, use_tc  # noqa: F401
from tests.test_gpu_svb_vae_train import MAP_BARS, MAP_ZERO_GRAD, STEP_BARS, _compare_step, _set_phase, _tied_step
from tests.test_gpu_wn_train import _check, _err

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='needs a CUDA device')]

MAX_FRAMES = 5000
GRID_STRIDE_FRAMES = 528 * 8         # frames one pass of the WN elementwise kernels covers (min(528, (T + 7) / 8) blocks of 8 warps)
BATCH_KEYS = ('amateur_mel', 'prof_mel', 'amateur_pitch', 'prof_pitch', 'amateur_spk_id', 'prof_spk_id', 'a2p_alignment')
CONDITIONS = ('h_content', 'h_pitch')
AMATEUR_ROWS = ('h_content', 'h_pitch', 'a2a mel_out')
PROF_ROWS = ('p2p mel_out', 'a2p mel_out')
SONG = (41, 41000, 40000)            # (seed, amateur frames, professional frames): 238 s at 22.05 kHz / hop 128
N_PAIRS, MAX_PAIR, MIN_PAIR = 64, 17, 40      # the max_frames pair and the 60-frame pair sit inside the batch
INJECT = 2e-3                        # the E errors, times max |reference|
MISS = 8                             # ... must miss their bar by at least this factor
# the phase-2 step at max_frames on the fp32 CUDA cores: 5x the 2.1e-5 / 5.0e-5 measured (header); the rest as STEP_BARS
MAX_FRAMES_STEP_BARS = {False: {None: (1e-4, 2.5e-4), 'loss': STEP_BARS[False]['loss']}, True: STEP_BARS[True]}

_REFS = {}                           # float64 oracle outputs (host), shared by both precisions and the E tests


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f'PEAK max_memory_allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB')


# ---------------------------------------------------------------------------------------------------------- references and checks
def _host(out):
    return {k: v.detach().cpu() for k, v in out.items()}


def _oracle_clip(key, batch, eps, sd, b):
    """The float64 oracle on clip b of ``batch`` alone, at the batch's padded lengths (cached under ``key``)."""
    k = (key, b)
    if k not in _REFS:
        _REFS[k] = _host(_oracle_forward({n: v[b:b + 1] for n, v in batch.items()}, eps[b:b + 1], sd))
    return _REFS[k]


def _oracle_batch(key, batch, eps, sd):
    """The float64 oracle of ``batch``, one clip at a time: rows stacked, the MLE the mean of the clips' terms (a sum over the
    batch divided by B), each KL the clips' terms weighted by their latent frames (pitch > 0 at every 4th frame: the mask the KL
    averages over)."""
    B = batch['amateur_mel'].shape[0]
    outs = [_oracle_clip(key, batch, eps, sd, b) for b in range(B)]
    ref = {k: torch.cat([o[k] for o in outs]) for k in outs[0] if outs[0][k].dim() > 0}
    for k, pitch in (('a2a kl', batch['amateur_pitch']), ('p2p kl', batch['prof_pitch'])):
        n = (pitch[:, ::4] > 0).sum(1).double()
        ref[k] = sum(o[k] * n[b] for b, o in enumerate(outs)) / n.sum()
    ref['a2p mle'] = sum(o['a2p mle'] for o in outs) / B
    return ref


def _lengths(pitch):
    """Each row's frame count: pitch ids are >= 1 inside a clip and 0 on its padding."""
    n = (pitch > 0).sum(1)
    for b, L in enumerate(n.tolist()):
        assert bool((pitch[b, :L] > 0).all()), (b, L)
    return n.tolist()


def _check_outputs(tag, got, ref, batch, bars):
    """Every output per clip and whole, the conditions first; every error is printed before the first failure (in that order)
    is raised."""
    La, Lp = _lengths(batch['amateur_pitch']), _lengths(batch['prof_pitch'])
    assert sorted(got) == sorted(ref)
    bad = []

    def check(name, g, r):
        try:
            _check(name, g, r, bars)
        except AssertionError as e:
            bad.append(e)
    for k in list(CONDITIONS) + [k for k in ref if k not in CONDITIONS]:
        g, r = got[k].cpu(), ref[k]
        assert g.shape == r.shape, (k, g.shape, r.shape)
        if r.dim() > 0:
            for b in range(r.shape[0]):
                n = La[b] if k in AMATEUR_ROWS else Lp[b] if k in PROF_ROWS else r.shape[1]
                check(f'{tag} {k} clip {b} ({n} frames)', g[b, :n].reshape(-1), r[b, :n].reshape(-1))
        check(f'{tag} {k} whole', g.reshape(-1), r.reshape(-1))
    assert not bad, bad[0]


def _decoder_frames(m):
    """A hook recording the frame count of every mel-decoder call; returns (list, handle)."""
    seen = []
    return seen, m.vae_model.decoder.register_forward_pre_hook(lambda mod, a: seen.append(a[2].shape[-1]))


# ---------------------------------------------------------------------------------------------------------- A: max_frames clips
A_CASES = {'5000x5000': (5000, 5000), '5000x2996': (5000, 2996), '3000x5000': (3000, 5000)}


def _a_batch(case):
    Ta, Tp = A_CASES[case]
    return _ragged([Ta], [Tp], 31 + list(A_CASES).index(case))


@pytest.mark.parametrize('eps_kind', ['zero', 'randn'])
@pytest.mark.parametrize('case', list(A_CASES))
def test_max_frames_clip_matches_float64(use_tc, case, eps_kind):
    batch, eps = _a_batch(case), _eps(1, eps_kind)
    m = _model(use_tc).eval()
    frames, hook = _decoder_frames(m)
    got = _native_forward(m, batch, eps)
    hook.remove()
    assert max(frames) > GRID_STRIDE_FRAMES, frames          # the WN elementwise kernels' second grid-stride pass runs
    ref = _oracle_batch(('A', case, eps_kind), batch, eps, m.state_dict())
    _check_outputs(f'A {case} {eps_kind} tc={use_tc}', got, ref, batch, FWD_BARS[use_tc])


# ---------------------------------------------------------------------------------------------------------- B: the beautifier's batches
class _Inputs:
    """Records the keyword inputs of every call of ``model``'s forward (host copies)."""

    def __init__(self, model):
        self.calls, fwd = [], model.forward

        def forward(**kw):
            self.calls.append({k: (v.detach().cpu().clone() if torch.is_tensor(v) else v) for k, v in kw.items()})
            return fwd(**kw)
        model.forward = forward


def _pairs(seed=1234):
    """tools/beautify_bench.py's pairs: 8 s +- 15 % at 22.05 kHz / hop 128, the professional take +- 15 % of the amateur one, an
    embedding per pair; pair MAX_PAIR has max_frames in both takes and pair MIN_PAIR 60 frames, the shortest the model takes."""
    rs = np.random.RandomState(seed)
    fps = 22050 / 128
    ama, prof, emb = [], [], []
    for i in range(N_PAIRS):
        Sf = int(8.0 * rs.uniform(0.85, 1.15) * fps)
        Tf = int(Sf * rs.uniform(0.85, 1.15))
        Sf, Tf = {MAX_PAIR: (MAX_FRAMES, MAX_FRAMES), MIN_PAIR: (60, 60)}.get(i, (Sf, Tf))
        a, p = song(int(rs.randint(0, 2 ** 31 - 1)), Sf, Tf)
        ama.append(a)
        prof.append(p)
        emb.append(rs.normal(0, 0.5, 256).astype(np.float32))
    return ama, prof, emb


@pytest.fixture(scope='module')
def beautifier_batches(tmp_path_factory):
    """{'song': ..., 'pairs64': ...}: (batch, eps, the beautifier's own a2p mel_out) of the model call of beautify_songs on one
    4-minute song and of beautify_batch on 64 pairs, and 'sd': the beautifier model's state_dict, 'plan': the song's segments."""
    from neuralsvb_b200.modules.fastspeech import multi_window_disc as M
    from neuralsvb_b200.modules.voice_conversion import vc_modules as V
    saved = dict(H.hparams)
    work, pairs = make_experiment(str(tmp_path_factory.mktemp('beautify_sizes')))
    emb = np.load(pairs[0][3])
    out = {}
    try:
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(V, 'USE_TC', True)
            mp.setattr(M, 'USE_TC', True)
            b = BF.SVBBeautifier(work)
            # the vocoder is not under test here, and its workspace for 64 rows of 5000 frames is tens of GB
            hop = int(b.hp['hop_size'])
            b._vocode = lambda mel_out, f0, Tp, seed, first_clip=0: torch.zeros(sum(Tp) * hop, device=b.device)
            rec = _Inputs(b.model)
            spy = SongSpy(b)
            a, p = song(*SONG)
            b.beautify_songs([a], [p], [emb], seed=3)
            out['song'] = (rec.calls[-1], spy.seen['_model_on'][0].cpu())
            out['plan'] = b.song_plans[0]
            spy = BatchSpy(b)
            b.beautify_batch(*_pairs(), seed=4)
            out['pairs64'] = (rec.calls[-1], spy.seen['_acoustic'].cpu())
            assert len(rec.calls) == 2
            out['sd'] = {k: v.detach().clone() for k, v in b.model.state_dict().items()}
        del b, rec, spy
    finally:
        H.hparams.clear()
        H.hparams.update(saved)
    torch.cuda.empty_cache()
    res = {'sd': out['sd'], 'plan': out['plan']}
    for name in ('song', 'pairs64'):
        call, mel_out = out[name]
        assert call['infer'] is False and not call['disable_map'] and list(call['concurrent_ways']) == ['a2a', 'p2p', 'a2p']
        res[name] = ({k: call[k] for k in BATCH_KEYS}, call['eps'], mel_out)
    return res


def _assert_coverage(name, batch, plan=None):
    La, Lp = _lengths(batch['amateur_pitch']), _lengths(batch['prof_pitch'])
    Ta, Tp = batch['amateur_mel'].shape[1], batch['prof_mel'].shape[1]
    print(f'COVERAGE {name}: B = {len(La)}, rows {Ta} x {Tp}, amateur frames {La}, professional frames {Lp}')
    if name == 'song':
        assert len(La) >= 8 and len(plan) == len(La)                      # >= 8 segments, one row each
        assert Lp[-1] < Tp / 4, (Lp[-1], Tp)                               # the tail fills under a quarter of its padded row
        assert any(a != p for a, p in zip(La, Lp))                         # segments whose Ta differs from Tp
        assert Tp == MAX_FRAMES
    else:
        assert len(La) == N_PAIRS and (La[MAX_PAIR], Lp[MAX_PAIR]) == (MAX_FRAMES, MAX_FRAMES) and (La[MIN_PAIR], Lp[MIN_PAIR]) == (60, 60)
        assert (Ta, Tp) == (MAX_FRAMES, MAX_FRAMES)


@pytest.mark.parametrize('name', ['song', 'pairs64'])
def test_beautifier_batches_match_float64(use_tc, beautifier_batches, name):
    batch, eps, mel_out = beautifier_batches[name]
    _assert_coverage(name, batch, beautifier_batches['plan'])
    sd = beautifier_batches['sd']
    m = _model(use_tc, sd=sd).eval()
    got = _native_forward(m, batch, eps)
    if use_tc:                                           # the recording is what the beautifier ran: its own a2p mel, bit for bit
        assert torch.equal(got['a2p mel_out'].cpu(), mel_out)
    ref = _oracle_batch(('B', name), batch, eps, sd)
    _check_outputs(f'B {name} tc={use_tc}', got, ref, batch, FWD_BARS[use_tc])


# ---------------------------------------------------------------------------------------------------------- C: padding
@pytest.mark.parametrize('name', ['song', 'pairs64'])
def test_rows_equal_clips_run_alone_at_the_same_padding(use_tc, beautifier_batches, name):
    """Each row of the beautifier's batch is bit-identical to its clip run alone in a row of the batch's lengths: no kernel mixes
    clips or orders a reduction by the batch size at 5000 frames and B = 64.  The KL and MLE batch means are left out."""
    batch, eps, _ = beautifier_batches[name]
    m = _model(use_tc, sd=beautifier_batches['sd']).eval()
    full = _host(_native_forward(m, batch, eps))
    for b in range(batch['amateur_mel'].shape[0]):
        one = _native_forward(m, {k: v[b:b + 1] for k, v in batch.items()}, eps[b:b + 1])
        for k, v in one.items():
            if v.dim() == 0:
                continue
            v = v.cpu()
            assert torch.equal(full[k][b:b + 1], v), (name, b, k, float((full[k][b:b + 1] - v).abs().max()))


def _movement(tag, padded, alone, L):
    """How far the oracle's output over a clip's own L frames moves when the clip's padding is removed: the largest change, the
    frame it is at, and the largest change over the clip's last 64 frames and over the rest."""
    d = (padded[0, :L] - alone[0, :L]).abs().flatten(1).max(1).values
    scale = float(alone[0, :L].abs().max())
    rel = float(d.max()) / scale
    print(f'MOVED {tag}: max |padded - alone| {float(d.max()):.3e} ({rel:.2e} of max |ref|) at frame {int(d.argmax())} of {L}; '
          f'last 64 frames {float(d[-64:].max()):.3e}, frames before {float(d[:-64].max()) if L > 64 else 0.0:.3e}, '
          f'median over frames {float(d.median()):.3e}')
    return rel


def test_oracle_moves_with_the_padding(beautifier_batches):
    """The float64 oracle on a padded row against the same clip alone and unpadded: the song's tail segment (padded to 5000) and the
    60-frame pair (in a 5000-frame row).  The model is not blind to padding (the posterior's mean over time takes in the padded
    frames), so the reference of a padded row must be the oracle on that padded row; its movement must be far above the forward
    bars, or the batch tests above would not see the padding."""
    sd = beautifier_batches['sd']
    worst = []
    for name, b in (('song', None), ('pairs64', MIN_PAIR)):
        batch, eps, _ = beautifier_batches[name]
        b = batch['amateur_mel'].shape[0] - 1 if b is None else b
        La, Lp = _lengths(batch['amateur_pitch'])[b], _lengths(batch['prof_pitch'])[b]
        padded = _oracle_clip(('B', name), batch, eps, sd, b)
        one = {k: v[b:b + 1] for k, v in batch.items()}
        for k in ('amateur_mel', 'amateur_pitch'):
            one[k] = one[k][:, :La]
        for k in ('prof_mel', 'prof_pitch', 'a2p_alignment'):
            one[k] = one[k][:, :Lp]
        alone = _host(_oracle_forward(one, eps[b:b + 1], sd))
        tag = f'{name} clip {b} ({La} x {Lp} frames in {batch["amateur_mel"].shape[1]} x {batch["prof_mel"].shape[1]} rows)'
        for k in ('h_content', 'a2a mel_out'):
            _movement(f'{tag} {k}', padded[k], alone[k], La)
        _movement(f'{tag} p2p mel_out', padded['p2p mel_out'], alone['p2p mel_out'], Lp)
        worst.append(_movement(f'{tag} a2p mel_out', padded['a2p mel_out'], alone['a2p mel_out'], Lp))
        for k in ('a2a m_q', 'p2p m_q'):
            print(f'MOVED {tag} {k}: max |padded - alone| {float((padded[k] - alone[k]).abs().max()):.3e}')
    assert min(worst) > 100 * FWD_BARS[True][1], worst


# ---------------------------------------------------------------------------------------------------------- D: training steps
def _d_batch():
    return _ragged([MAX_FRAMES, 1236, 60], [MAX_FRAMES - 4, 1300, 60], 41)


@pytest.mark.parametrize('phase', [2, 3])
def test_steps_at_max_frames_match_float64(use_tc, phase):
    m = _model(use_tc, trainable=True)
    _set_phase(m, phase)
    frames, hook = _decoder_frames(m)
    losses, ref, p = _tied_step(m, phase, _d_batch())
    hook.remove()
    assert max(frames) > GRID_STRIDE_FRAMES, frames
    bars = (MAX_FRAMES_STEP_BARS if phase == 2 else MAP_BARS)[use_tc]
    n = _compare_step(f'D phase{phase} tc={use_tc}', m, phase, losses, ref, p, bars, zero_grad=MAP_ZERO_GRAD if phase == 3 else ())
    assert n > 100 if phase == 2 else n == len(list(m.z_mapping_function.parameters()))
    sd = m.state_dict()
    running = ['upsample_layer.0.3', 'vae_model.encoder.poolings.2', 'vae_model.encoder.poolings.5'] if phase == 2 else \
        ['z_mapping_function.convs.1', 'z_mapping_function.convs.4']
    for pre in running:
        for s in ('running_mean', 'running_var'):
            _check(f'D phase{phase} tc={use_tc} {pre}.{s}', sd[f'{pre}.{s}'], p[f'{pre}.{s}'], bars[None])


# ---------------------------------------------------------------------------------------------------------- E: the bars can fail
def _inject(monkeypatch, clip, frames, delta):
    """Every mel-decoder output [B, 80, T] gets ``delta`` added on row ``clip``, frames [frames[0], frames[1])."""
    from neuralsvb_b200.modules.fastspeech import fs2_vae as FV
    orig, hits = FV.FVAEDecoder.forward, []

    def forward(self, *a):
        y = orig(self, *a).clone()
        y[clip, :, frames[0]:frames[1]] += delta
        hits.append(y.shape[-1])
        return y
    monkeypatch.setattr(FV.FVAEDecoder, 'forward', forward)
    return hits


def _misses(tag, got, ref, bars):
    """The check must fail, by at least MISS times its bar in L2 or L-inf; prints the factor."""
    with pytest.raises(AssertionError):
        _check(tag, got, ref, bars)
    l2, li = _err(got, ref)
    factor = max(l2 / bars[0], li / bars[1])
    print(f'MISSES {tag}: {factor:.1f}x its bar (rel L2 {l2:.2e} / {bars[0]:.1e}, rel L-inf {li:.2e} / {bars[1]:.1e})')
    return factor


def test_bars_fail_on_the_grid_stride_rows_off_by_2e_3(bf16x3, monkeypatch):
    """Frames [4224, 5000) of the decoder output of a 5000 x 5000 clip: the rows only the second grid-stride pass writes."""
    batch, eps = _a_batch('5000x5000'), _eps(1, 'zero')
    m = _model(True).eval()
    ref = _oracle_batch(('A', '5000x5000', 'zero'), batch, eps, m.state_dict())
    hits = _inject(monkeypatch, 0, (GRID_STRIDE_FRAMES, MAX_FRAMES), INJECT * float(ref['a2p mel_out'].abs().max()))
    got = _native_forward(m, batch, eps)
    assert hits and max(hits) == MAX_FRAMES
    assert _misses('E grid-stride rows a2p mel_out', got['a2p mel_out'].cpu().reshape(-1), ref['a2p mel_out'].reshape(-1),
                   FWD_BARS[True]) >= MISS


def test_bars_fail_on_the_song_tail_segment_off_by_2e_3(bf16x3, monkeypatch, beautifier_batches):
    """The song batch's short tail segment alone: its per-clip check fails although the whole tensor is mostly the long clips."""
    batch, eps, _ = beautifier_batches['song']
    sd = beautifier_batches['sd']
    tail = batch['amateur_mel'].shape[0] - 1
    Lp = _lengths(batch['prof_pitch'])[tail]
    ref = _oracle_batch(('B', 'song'), batch, eps, sd)['a2p mel_out']
    _inject(monkeypatch, tail, (0, Lp), INJECT * float(ref[tail, :Lp].abs().max()))
    got = _native_forward(_model(True, sd=sd).eval(), batch, eps)['a2p mel_out'].cpu()
    l2, li = _err(got.reshape(-1), ref.reshape(-1))
    print(f'ERR E song tail, whole tensor {l2:.2e} {li:.2e} (bars {FWD_BARS[True]})')
    assert _misses(f'E song tail a2p mel_out clip {tail} ({Lp} frames)', got[tail, :Lp].reshape(-1), ref[tail, :Lp].reshape(-1),
                   FWD_BARS[True]) >= MISS

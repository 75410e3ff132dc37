"""-m gpu: whole songs.  The cluster DTW of align_long against the one-CTA kernel of align_batch bit for bit (SVB_DTW_CTA_CELLS puts
pairs of up to 5000 frames on clusters of 2 .. 8 CTAs) and against the oracle past 8192 frames; beautify_songs against its
composition (align_long, plan_song, condition(), MleSVBVAE, the numpy stitch, spec2wav_batch), against beautify on a song of one
segment, its independence of the other songs, its errors and the --song CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from neuralsvb_b200.inference import beautify as BF
from neuralsvb_b200.inference.song_plan import plan_song, stitch_weights
from neuralsvb_b200.modules.voice_conversion.dtw import core
from neuralsvb_b200.tasks.singing.dataset_utils import clip_alignment
from neuralsvb_b200.utils import audio
from neuralsvb_b200.utils import hparams as H
from neuralsvb_b200.utils import synthetic as S
from neuralsvb_b200.utils.pitch_utils import denorm_f0, norm_interp_f0
from oracle import sadtw as O
from tests.test_gpu_beautify import CONFIG, ROOT, make_experiment

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'sadtw.npz')


@pytest.fixture(autouse=True)
def keep_hparams():
    saved = dict(H.hparams)
    yield
    H.hparams.clear()
    H.hparams.update(saved)


def both(pairs, method='EHSADTW', dtype=np.float32):
    srcs = [a.astype(dtype) for a, _ in pairs]
    tgts = [b.astype(dtype) for _, b in pairs]
    return core.align_batch(srcs, tgts, method), core.align_long(srcs, tgts, method)


def assert_same(r1, r2):
    for p, (x, y) in enumerate(zip(r1.split(), r2.split())):
        assert np.array_equal(x, y), f'pair {p}: alignment'
    assert torch.equal(r1.path_cost, r2.path_cost), (r1.path_cost, r2.path_cost)


# SVB_DTW_CTA_CELLS -> shapes (S, T): min(S, T) > cells puts the pair on a cluster of ceil(min / max(cells, ceil(min / 8))) CTAs
CLUSTER_SHAPES = {
    64: [(449, 449), (130, 700), (700, 130), (5000, 5000), (65, 3000)],    # 449 = 7 x 64 + 1: one cell in the last CTA
    625: [(5000, 5000), (4376, 4900), (4900, 4376), (626, 626), (1251, 5000)],
    1000: [(5000, 5000), (1001, 1001), (2500, 4000), (4000, 2500), (3001, 3200)],   # 1001, 3001: one cell in the last CTA
    4096: [(4097, 4097), (5000, 4200), (4200, 5000), (4097, 5000)],
}


@pytest.mark.parametrize('cells', sorted(CLUSTER_SHAPES))
def test_cluster_dtw_equals_the_one_cta_kernel(monkeypatch, cells):
    monkeypatch.setenv('SVB_DTW_CTA_CELLS', str(cells))
    shapes = CLUSTER_SHAPES[cells]
    pairs = [S.make_f0_pair(300 + k, s, t) for k, (s, t) in enumerate(shapes)]
    for method in ('EHSADTW', 'SADTW'):
        assert_same(*both(pairs, method))
    # a ragged batch mixing cluster pairs with one-CTA pairs (min(S, T) <= cells), float64
    mixed = [pairs[0], S.make_f0_pair(7, 40, 60), pairs[-1], S.make_f0_pair(8, cells, 2 * cells), S.make_f0_pair(9, 2, 90)]
    assert_same(*both(mixed, dtype=np.float64))


def test_cluster_dtw_on_the_fixture_pairs(monkeypatch):
    from oracle.gen_golden_sadtw import SADTW_CASES
    g = np.load(GOLDEN)
    pairs = [S.make_f0_pair(*SADTW_CASES[name]) for name in SADTW_CASES]
    monkeypatch.setenv('SVB_DTW_CTA_CELLS', '16')
    r1, r2 = both(pairs)
    assert_same(r1, r2)
    for name, al in zip(SADTW_CASES, r2.split()):
        key = f'{name}/EHSADTW/np32/alignment'
        if key in g:
            assert np.array_equal(al, g[key]), name


def test_cta_cells_hook_is_validated(monkeypatch):
    a, b = S.make_f0_pair(1, 100, 100)
    for bad in ('0', '8193', 'x'):
        monkeypatch.setenv('SVB_DTW_CTA_CELLS', bad)
        with pytest.raises(ValueError, match='SVB_DTW_CTA_CELLS'):
            core.align_long([a], [b])


@pytest.mark.parametrize('shape,dtype', [((8193, 8193), np.float32), ((9000, 16500), np.float64), ((16500, 9000), np.float32),
                                         ((16385, 17000), np.float64)])
def test_align_long_equals_the_oracle_past_8192_frames(shape, dtype):
    a, b = S.make_f0_pair(77, *shape)
    got = core.align_long([a.astype(dtype)], [b.astype(dtype)])
    al, last = O.shape_aware_align(a.astype(dtype), b.astype(dtype), 'EHSADTW')
    assert np.array_equal(got.split()[0], al)
    assert got.path_cost.cpu().numpy()[0] == np.float32(last)


# ---- beautify_songs ----------------------------------------------------------------------------------------------------------
def song(seed, Ta, Tp, hop=128, sr=22050):
    """(amateur, professional) float32 takes at sr of Ta / Tp frames: make_f0_pair's contours through make_sung_take."""
    a, p = S.make_f0_pair(seed, Ta - 1, Tp - 1)
    return S.make_sung_take(a, seed, sr, hop)[0], S.make_sung_take(p, seed + 1, sr, hop)[0]


@pytest.fixture(scope='module')
def exp(tmp_path_factory):
    work, pairs = make_experiment(str(tmp_path_factory.mktemp('song')))
    songs = [song(41, 10400, 10200), song(42, 6000, 6900), song(43, 900, 860)]
    return work, songs, np.load(pairs[0][3])


class Spy:
    def __init__(self, b):
        self.seen = {'_model_on': []}
        for name in ('_front_end', '_pitch', '_align_songs', '_model_on', '_vocode'):
            setattr(b, name, self._wrap(name, getattr(b, name)))

    def _wrap(self, name, fn):
        def call(*a, **kw):
            r = fn(*a, **kw)
            if name == '_model_on':
                self.seen[name].append(r)
            else:
                self.seen[name] = r
            return r
        return call


def restated_stitch(mels, plan, ov):
    w = stitch_weights(ov)[:, None]
    out = np.zeros((plan[-1][1], mels[0].shape[1]), np.float32)
    for k, (s, e, _, _) in enumerate(plan):
        out[s:e] = mels[k][:e - s]
    for k in range(len(plan) - 1):
        s0, s1 = plan[k][0], plan[k + 1][0]
        out[s1:s1 + ov] = (np.float32(1) - w) * mels[k][s1 - s0:s1 - s0 + ov] + w * mels[k + 1][:ov]
    return out


def test_beautify_songs_equals_its_composition(exp):
    work, songs, emb = exp
    b = BF.SVBBeautifier(work)
    hp, B, seed = b.hp, len(songs), 5
    eps = torch.randn(B, hp['latent_size'], 1, generator=torch.Generator().manual_seed(3))
    spy = Spy(b)
    got = b.beautify_songs([s[0] for s in songs], [s[1] for s in songs], [emb] * B, seed=seed, eps=eps)
    f0_dev, f0s = spy.seen['_pitch']
    frames = [len(f) for f in f0s]
    assert frames[0] > 8192 and frames[B] > 8192 and hp['max_frames'] < frames[1] <= 8192 and frames[2] < hp['max_frames']
    t = torch.split(f0_dev.double(), frames)
    ref = core.align_long(list(t[:B]), list(t[B:])).split()
    fm, mels, f0v = hp['frames_multiple'], [], []
    for i in range(B):
        assert np.array_equal(spy.seen['_align_songs'][i], ref[i]), f'song {i}: alignment'
        Ta, Tp = frames[i] // fm * fm, frames[B + i] // fm * fm
        a2p = clip_alignment(ref[i], Tp, Ta).numpy()
        pf0, puv = norm_interp_f0(f0s[B + i][:Tp], hp)
        plan = plan_song(Tp, Ta, a2p, puv.numpy(), hp)
        assert plan == b.song_plans[i], f'song {i}: plan'
        assert (len(plan) > 1) == (i < 2)
        f2c = BF.f0_to_coarse
        sample, sa, sp = BF.condition([a1 - a0 for _, _, a0, a1 in plan] + [e - s for s, e, _, _ in plan],
                                      [f0s[i][a0:a1] for _, _, a0, a1 in plan] + [f0s[B + i][s:e] for s, e, _, _ in plan],
                                      [f2c(f0s[i])[a0:a1] for _, _, a0, a1 in plan] + [f2c(f0s[B + i])[s:e] for s, e, _, _ in plan],
                                      [a2p[s:e] - a0 for s, e, a0, _ in plan], [torch.FloatTensor(emb)] * len(plan), hp)
        out = spy.seen['_model_on'][i]
        assert tuple(out.shape[:2]) == (len(plan), max(sp))
        mels.append(restated_stitch([out[k].cpu().numpy() for k in range(len(plan))], plan, 64))
        assert np.array_equal(b.song_mels[i].cpu().numpy(), mels[-1]), f'song {i}: stitched mel'
        f0v.append(denorm_f0(pf0, puv, hp).numpy())
        # the segment batch the model saw: condition()'s rules on the plan's slices
        with torch.no_grad():
            rows = np.concatenate([[0], np.cumsum(frames)])
            wav_mel = spy.seen['_front_end'][0]
            pad = lambda rs, T: torch.stack([torch.nn.functional.pad(wav_mel[r:r + n], (0, 0, 0, max(T) - n)) for r, n in zip(rs, T)])
            d = b.device
            o2 = b.model(amateur_mel=pad([rows[i] + a0 for _, _, a0, _ in plan], sa), prof_mel=pad([rows[B + i] + s for s, _, _, _ in plan], sp),
                         amateur_pitch=sample['pitch'].to(d), prof_pitch=sample['prof_pitch'].to(d), amateur_spk_id=sample['spk'].to(d),
                         prof_spk_id=sample['spk'].to(d), a2p_alignment=sample['a2p_f0_alignment'].to(d), infer=False,
                         concurrent_ways=['a2a', 'p2p', 'a2p'], disable_map=hp['disable_map'],
                         eps=eps[i:i + 1].expand(len(plan), -1, -1).contiguous().to(d))['a2p']['mel_out']
        assert torch.equal(o2, out), f'song {i}: segment mels'
    wavs = b.vocoder.spec2wav_batch(mels, f0v, seed=seed)
    for i in range(B):
        assert got[i].dtype == np.float32 and np.array_equal(got[i], wavs[i]), f'song {i}: waveform'


def test_a_one_segment_song_is_beautify_and_songs_do_not_depend_on_each_other(exp):
    work, songs, emb = exp
    b = BF.SVBBeautifier(work)
    eps = torch.randn(3, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(8))
    one = b.beautify(songs[2][0], songs[2][1], emb, seed=4, eps=eps[:1])
    alone = b.beautify_songs([songs[2][0]], [songs[2][1]], [emb], seed=4, eps=eps[:1])[0]
    assert np.array_equal(one, alone)
    both_ = b.beautify_songs([songs[1][0], songs[2][0]], [songs[1][1], songs[2][1]], [emb] * 2, seed=4, eps=eps[1:])
    mel_b, plan_b = b.song_mels[0].clone(), b.song_plans[0]
    b.beautify_songs([songs[1][0]], [songs[1][1]], [emb], seed=4, eps=eps[1:2])
    assert plan_b == b.song_plans[0] and torch.equal(mel_b, b.song_mels[0])
    assert len(both_) == 2


def test_errors_raise_before_the_model(exp):
    work, songs, emb = exp
    b = BF.SVBBeautifier(work)
    spy = Spy(b)
    with pytest.raises(ValueError, match='song 0: the professional take has 65537 frames'):
        b.beautify_songs([songs[2][0]], [np.zeros(65536 * 128, np.float32)], [emb])
    with pytest.raises(ValueError, match='song 1: the amateur take'):
        b.beautify_songs([songs[2][0], songs[2][0][:50 * 128]], [songs[2][1]] * 2, [emb] * 2)
    with pytest.raises(ValueError, match='beautify_songs: overlap_frames = 66'):
        b.beautify_songs([songs[1][0]], [songs[1][1]], [emb], overlap_frames=66)
    with pytest.raises(ValueError, match='beautify_songs: segment_frames = 5001'):
        b.beautify_songs([songs[1][0]], [songs[1][1]], [emb], segment_frames=5001)
    assert '_front_end' not in spy.seen                            # argument and take checks: before any device work
    # a real planning failure: song 1's alignment piles its 6000 amateur frames onto the first allowed window
    align = b._align_songs
    b._align_songs = lambda f0, frames, st: [a if i == 0 else np.where(np.arange(len(a)) < 100, 0, 5999)
                                             for i, a in enumerate(align(f0, frames, st))]
    with pytest.raises(ValueError, match='song 1: cannot plan the segments at professional frame 0: every segment end'):
        b.beautify_songs([songs[2][0], songs[1][0]], [songs[2][1], songs[1][1]], [emb] * 2)
    assert '_pitch' in spy.seen and spy.seen['_model_on'] == [] and '_vocode' not in spy.seen
    with pytest.raises(ValueError, match='max_frames'):
        b.beautify(songs[1][0], songs[1][1], emb)


def test_cli_song_writes_one_file_per_pair(exp, tmp_path):
    work, songs, emb = exp
    root = os.path.dirname(os.path.dirname(work))
    ins = []
    for i, (a, p) in enumerate(songs[1:]):
        ins.append((str(tmp_path / f'a{i}.wav'), str(tmp_path / f'p{i}.wav'), str(tmp_path / f'e{i}.npy')))
        audio.save_wav(a, ins[-1][0], 22050, norm=False)
        audio.save_wav(p, ins[-1][1], 22050, norm=False)
        np.save(ins[-1][2], emb)
    outs = [str(tmp_path / f'o{i}.wav') for i in range(len(ins))]
    r = subprocess.run([sys.executable, '-m', 'neuralsvb_b200.inference.beautify', '--config', CONFIG, '--exp_name', 'svb_bf', '--song',
                        '--amateur'] + [x[0] for x in ins] + ['--prof'] + [x[1] for x in ins] + ['--spk_emb'] + [x[2] for x in ins] +
                       ['--out'] + outs, cwd=root, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    for fn, (_, p, _) in zip(outs, ins):
        assert audio.wav_info(fn)[1] == (audio.wav_info(p)[1] // 128 + 1) // 4 * 4 * 128


def test_songs_vocoded_in_several_groups_draw_by_song_index(exp, monkeypatch):
    """Songs split over several generator calls (SONG_VOCODE_FRAMES forced small) still draw their NSF noise by (seed, song
    index): every waveform equals spec2wav_batch of all the stitched mels in one call with the same seed."""
    work, songs, emb = exp
    b = BF.SVBBeautifier(work)
    monkeypatch.setattr(BF, 'SONG_VOCODE_FRAMES', 12000)
    spy = Spy(b)
    got = b.beautify_songs([s[0] for s in songs], [s[1] for s in songs], [emb] * 3, seed=6)
    Tps = [p[-1][1] for p in b.song_plans]
    assert BF._groups([1] * 3, 12000, lambda a, c: (c - a) * max(Tps[a:c])) == [(0, 1), (1, 2), (2, 3)]
    f0s = spy.seen['_pitch'][1]
    f0v = []
    for i, Tp in enumerate(Tps):
        pf0, puv = norm_interp_f0(f0s[3 + i][:Tp], b.hp)
        f0v.append(denorm_f0(pf0, puv, b.hp).numpy())
    ref = b.vocoder.spec2wav_batch([m.cpu().numpy() for m in b.song_mels], f0v, seed=6)
    for i in range(3):
        assert np.array_equal(got[i], ref[i]), f'song {i}: waveform'


def test_normalize_pitch_normalises_each_whole_take_once(exp):
    """normalize_pitch on: a one-segment song is still beautify of the pair, and a multi-segment song's segments get the pitch ids
    and f0 of the whole take's normalised contour, sliced (one key per song), not of each slice normalised on its own."""
    from neuralsvb_b200.tasks.singing.dataset_utils import normalized_take_f0
    work, songs, emb = exp
    b = BF.SVBBeautifier(work)
    b.hp['normalize_pitch'] = True
    eps = torch.randn(2, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(2))
    one = b.beautify(songs[2][0], songs[2][1], emb, seed=3, eps=eps[:1])
    assert np.array_equal(one, b.beautify_songs([songs[2][0]], [songs[2][1]], [emb], seed=3, eps=eps[:1])[0])
    seen = []
    model_on = b._model_on
    b._model_on = lambda sample, *a: seen.append(sample) or model_on(sample, *a)
    spy = Spy(b)
    b.beautify_songs([songs[1][0]], [songs[1][1]], [emb], seed=3, eps=eps[1:])
    f0s, plan, hp = spy.seen['_pitch'][1], b.song_plans[0], b.hp
    assert len(plan) > 1
    fa, fp = normalized_take_f0(f0s[0], hp, 500), normalized_take_f0(f0s[1], hp, 900)
    ref, _, _ = BF.condition([a1 - a0 for _, _, a0, a1 in plan] + [e - s for s, e, _, _ in plan],
                             [fa[a0:a1] for _, _, a0, a1 in plan] + [fp[s:e] for s, e, _, _ in plan],
                             [BF.f0_to_coarse(fa)[a0:a1] for _, _, a0, a1 in plan] + [BF.f0_to_coarse(fp)[s:e] for s, e, _, _ in plan],
                             [np.zeros(e - s, np.int64) for s, e, _, _ in plan], [torch.FloatTensor(emb)] * len(plan),
                             dict(hp, normalize_pitch=False))
    for k in ('pitch', 'f0', 'uv', 'prof_pitch', 'prof_f0', 'prof_uv'):
        assert torch.equal(seen[0][k], ref[k]), k
    per_clip, _, _ = BF.condition([a1 - a0 for _, _, a0, a1 in plan] + [e - s for s, e, _, _ in plan],
                                  [f0s[0][a0:a1] for _, _, a0, a1 in plan] + [f0s[1][s:e] for s, e, _, _ in plan],
                                  [BF.f0_to_coarse(f0s[0])[a0:a1] for _, _, a0, a1 in plan] +
                                  [BF.f0_to_coarse(f0s[1])[s:e] for s, e, _, _ in plan],
                                  [np.zeros(e - s, np.int64) for s, e, _, _ in plan], [torch.FloatTensor(emb)] * len(plan), hp)
    assert not torch.equal(seen[0]['prof_f0'], per_clip['prof_f0'])     # the departure from per-clip conditioning is real

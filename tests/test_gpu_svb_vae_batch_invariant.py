"""MleSVBVAE's length-aware mode (forward(..., amateur_lens=, prof_lens=)) and the beautifier's batch_invariant: every clip computed
from its own frames only.

  kernels   the masked GroupNorm + ReLU + residual, the global latent head and the ragged tensor-core / fp32 convolutions against
            float64 torch, each clip bit-identical to the clip alone and unpadded, zeros past its length;
  model     a ragged batch (Ta != Tp, a 60-frame clip, a 5000-frame clip, a clip filling under a quarter of its row): each clip's
            conditions, mels and latent statistics equal, bit for bit, the clip alone and unpadded, at another row, padded to 5000
            and with garbage in every padding frame; and each clip is within FWD_BARS of the float64 oracle of the clip alone;
  song      the 4-minute song's tail segment against its unpadded oracle, in both modes;
  beautifier beautify_batch / beautify_songs with batch_invariant=True against the pairs and segments run alone, and the
            refusals of bad lengths."""
import ctypes

import numpy as np
import pytest
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.inference import beautify as BF
from neuralsvb_b200.modules.voice_conversion.vc_modules import FrameLens
from neuralsvb_b200.utils import hparams as H
from tests.test_gpu_beautify import Spy as BatchSpy
from tests.test_gpu_beautify import make_experiment, regular
from tests.test_gpu_song import Spy as SongSpy
from tests.test_gpu_song import song
from tests.test_gpu_svb_vae_beautify_sizes import _Inputs, _lengths, SONG
from tests.test_gpu_svb_vae_shapes import FWD_BARS, _eps, _model, _oracle_forward, _ragged, use_tc  # noqa: F401
from tests.test_gpu_wn_train import _check, _err

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='needs a CUDA device')]

WAYS = ['a2a', 'p2p', 'a2p']
AMATEUR = ('h_content', 'h_pitch', 'a2a mel_out')
PROF = ('p2p mel_out', 'a2p mel_out')
LATENT = ('a2a m_q', 'a2a logs_q', 'a2a z_q', 'p2p m_q', 'p2p logs_q', 'p2p z_q')
LA = [5000, 60, 1236, 300, 212, 76, 688, 1024, 412]
LP = [4996, 60, 1300, 236, 332, 68, 720, 980, 400]
_REFS = {}


@pytest.fixture(autouse=True)
def keep_hparams():
    saved = dict(H.hparams)
    yield
    H.hparams.clear()
    H.hparams.update(saved)


def _fl(n):
    return FrameLens(n, torch.device('cuda'))


# ---------------------------------------------------------------------------------------------------------- kernels
def test_group_norm_relu_add_matches_float64_and_ignores_padding():
    torch.manual_seed(0)
    C, G, T, lens = 256, 16, 5000, [15, 60, 4999, 5000]
    B = len(lens)
    x, h = torch.randn(B, C, T, device='cuda'), torch.randn(B, C, T, device='cuda') * 3 + 1
    gamma, beta = torch.randn(C, device='cuda'), torch.randn(C, device='cuda')

    def run(x, h, n):
        y = torch.full_like(h, float('nan'))
        _native.check(_native.lib().svb_group_norm_relu_add_ragged(
            _native.ptr(x), _native.ptr(h), _native.ptr(gamma), _native.ptr(beta), x.shape[0], C, x.shape[2], G,
            ctypes.c_float(1e-5), n.c_host, _native.ptr(n.dev), _native.ptr(y), _native.current_stream_ptr()), 'gn')
        return y
    y = run(x, h, _fl(lens))
    for b, L in enumerate(lens):
        hd = h[b:b + 1, :, :L].double()
        ref = x[b:b + 1, :, :L].double() + torch.relu(torch.nn.functional.group_norm(hd, G, gamma.double(), beta.double(), 1e-5))
        _check(f'gn L={L}', y[b:b + 1, :, :L].reshape(-1), ref.reshape(-1), FWD_BARS[False])
        assert bool((y[b, :, L:] == 0).all()), L
        alone = run(x[b:b + 1, :, :L].contiguous(), h[b:b + 1, :, :L].contiguous(), _fl([L]))
        assert torch.equal(alone, y[b:b + 1, :, :L]), L


def test_latent_head_matches_float64():
    torch.manual_seed(1)
    latent, enc = 128, [15, 1250]                  # 60 mel frames (n3 = 1) and 5000 (n3 = 155)
    n3 = [1, 155]
    T = max(n3) + 7
    x = torch.randn(2, 2 * latent, T, device='cuda')
    eps = torch.randn(2, latent, 1, device='cuda')
    m, logs, z = (torch.empty(2, latent, 1, device='cuda') for _ in range(3))
    n = _fl(enc)
    _native.check(_native.lib().svb_global_latent_head_ragged(_native.ptr(x), 2, latent, T, n.c_host, _native.ptr(n.dev), _native.ptr(eps),
                                                              _native.ptr(m), _native.ptr(logs), _native.ptr(z),
                                                              _native.current_stream_ptr()), 'latent_head')
    for b, k in enumerate(n3):
        mean = x[b, :, :k].double().mean(-1)
        rm, rl = mean[:latent], mean[latent:]
        for name, g, r in (('m', m[b, :, 0], rm), ('logs', logs[b, :, 0], rl), ('z', z[b, :, 0], rm + eps[b, :, 0].double() * rl.exp())):
            _check(f'latent head n3={k} {name}', g, r, FWD_BARS[False])


def _garbage_rows(x, lens):
    x = x.clone()
    for b, L in enumerate(lens):
        x[b, :, L:] = torch.randn_like(x[b, :, L:]) * 50
    return x


# (Cin, Cout, K, stride, pad, groups): every convolution form of the model's length-aware path
CONVS = {
    'tc_1x1_256': (256, 256, 1, 1, 0, 1, True), 'tc_k5_256': (256, 256, 5, 1, 2, 1, True), 'tc_1x1_768': (768, 256, 1, 1, 0, 1, True),
    'tc_1x1_256_1024': (256, 1024, 1, 1, 0, 1, True),
    'fp32_prenet_k5_s2': (80, 256, 5, 2, 2, 1, False), 'fp32_k5_256': (256, 256, 5, 1, 2, 1, False),
    'fp32_enc_k8_s4': (80, 192, 8, 4, 2, 1, False), 'fp32_pool_k3_s2': (256, 256, 3, 2, 0, 1, False),
    'fp32_depthwise_k31': (256, 256, 31, 1, 15, 256, False), 'fp32_1x1': (192, 256, 1, 1, 0, 1, False),
}


@pytest.mark.parametrize('name', list(CONVS))
def test_ragged_convs_equal_the_clip_alone_and_zero_its_padding(name):
    from neuralsvb_b200.modules.hifigan import discriminators as D
    Cin, Cout, K, s, p, g, tc = CONVS[name]
    torch.manual_seed(2)
    lens, T = [60, 5000, 1236, 301, 33], 5000
    x = _garbage_rows(torch.randn(len(lens), Cin, T, device='cuda'), lens)
    w = torch.randn(Cout, Cin // g, K, device='cuda') / (Cin // g * K) ** 0.5
    bias = torch.randn(Cout, device='cuda')
    layer = D.TcLayer() if tc else None

    def run(x, n):
        if tc:
            return D.conv_tc_ragged(x, w, bias, layer, K, p, 0.0, _fl(n))
        return D.conv_nct_ragged(x, w, bias, K, s, p, g, 0.0, _fl(n))
    y = run(x, lens)
    for b, L in enumerate(lens):
        Lo = (L + 2 * p - K) // s + 1
        one = run(x[b:b + 1, :, :L].contiguous(), [L])
        assert one.shape[-1] == Lo
        assert torch.equal(one, y[b:b + 1, :, :Lo]), (name, b, L)
        assert bool((y[b, :, Lo:] == 0).all()), (name, b, L)
        ref = torch.relu(torch.nn.functional.conv1d(x[b:b + 1, :, :L].double(), w.double(), bias.double(), s, p, 1, g))
        _check(f'{name} L={L}', one.reshape(-1), ref.reshape(-1), FWD_BARS[tc])


def test_ragged_tc_layer_refuses_strided_layers_and_bad_lengths():
    from neuralsvb_b200.modules.hifigan import discriminators as D
    x = torch.randn(1, 256, 64, device='cuda')
    layer = D.TcLayer()
    y = D.conv_tc(x, torch.randn(256, 256, 4, device='cuda'), torch.zeros(256, device='cuda'), layer, 4, 2, 1, 1.0, 1)   # strided handle
    n = _fl([64])
    with pytest.raises(RuntimeError, match='stride-1'):
        _native.check(_native.lib().svb_tc_layer_forward_ragged(layer.h, _native.ptr(x), 1, 64, n.c_host, _native.ptr(n.dev),
                                                                ctypes.c_float(1.0), _native.ptr(y), _native.current_stream_ptr()), 'ragged')
    with pytest.raises(RuntimeError, match='clip 0 has 65 frames'):
        D.conv_tc_ragged(x, torch.randn(256, 256, 1, device='cuda'), torch.zeros(256, device='cuda'), D.TcLayer(), 1, 0, 1.0, _fl([65]))


# ---------------------------------------------------------------------------------------------------------- the model
def _forward(m, batch, eps, La, Lp):
    b = {k: v.cuda() for k, v in batch.items()}
    with torch.no_grad():
        r = m(**b, infer=False, concurrent_ways=WAYS, eps=eps.cuda(), amateur_lens=La, prof_lens=Lp)
        c = m.prepare_condition(b['amateur_mel'], b['amateur_pitch'], spk_ids=b['amateur_spk_id'], lens=La)
    out = {f'{w} mel_out': r[w]['mel_out'] for w in WAYS}
    out.update({f'{w} {k}': r[w][k] for w in ('a2a', 'p2p') for k in ('m_q', 'logs_q', 'z_q')})
    out.update({'h_content': c['h_content'], 'h_pitch': c['h_pitch']})
    return {k: v.cpu() for k, v in out.items()}


def _clip(out, row, La, Lp):
    """Clip `row`'s outputs on its own frames."""
    r = {k: out[k][row, :La] for k in AMATEUR}
    r.update({k: out[k][row, :Lp] for k in PROF})
    r.update({k: out[k][row] for k in LATENT})
    return r


def _slice(batch, rows, La, Lp, Ta=None, Tp=None, garbage=None):
    """Rows `rows` of `batch`, cropped (or zero-padded) to Ta x Tp; garbage: a seed for random values in every padding frame."""
    Ta, Tp = Ta or max(La), Tp or max(Lp)
    out = {}
    for k, v in batch.items():
        v = v[rows]
        if v.dim() == 1 or k.endswith('spk_id'):
            out[k] = v
            continue
        T = Ta if k.startswith('amateur') else Tp
        pad = torch.zeros((v.shape[0], T) + tuple(v.shape[2:]), dtype=v.dtype)
        n = min(T, v.shape[1])
        pad[:, :n] = v[:, :n]
        out[k] = pad
    lens_of = {'amateur_mel': La, 'amateur_pitch': La, 'prof_mel': Lp, 'prof_pitch': Lp, 'a2p_alignment': Lp}
    for k, lens in lens_of.items():
        for b, L in enumerate(lens):
            out[k][b, L:] = 0
            if garbage is not None:
                g = torch.Generator().manual_seed(garbage + b)
                n = out[k].shape[1] - L
                if k.endswith('mel'):
                    out[k][b, L:] = torch.randn(n, out[k].shape[2], generator=g) * 3
                elif k.endswith('pitch'):
                    out[k][b, L:] = torch.randint(1, 300, (n,), generator=g)
                else:
                    out[k][b, L:] = torch.randint(0, out['amateur_mel'].shape[1], (n,), generator=g)
    return out


def _batch():
    return _ragged(LA, LP, 71)


def test_each_clip_is_bit_identical_wherever_it_runs(use_tc):
    batch, B = _batch(), len(LA)
    eps = _eps(B, 'randn')
    m = _model(use_tc).eval()
    full = _forward(m, batch, eps, LA, LP)
    rev = list(range(B))[::-1]
    flipped = _forward(m, _slice(batch, rev, [LA[i] for i in rev], [LP[i] for i in rev]), eps[rev], [LA[i] for i in rev], [LP[i] for i in rev])
    junk = _forward(m, _slice(batch, list(range(B)), LA, LP, garbage=5), eps, LA, LP)
    for b in range(B):
        La, Lp = LA[b], LP[b]
        want = _clip(full, b, La, Lp)
        alone = _clip(_forward(m, _slice(batch, [b], [La], [Lp]), eps[b:b + 1], [La], [Lp]), 0, La, Lp)
        padded = _clip(_forward(m, _slice(batch, [b], [La], [Lp], 5000, 5000), eps[b:b + 1], [La], [Lp]), 0, La, Lp)
        for tag, got in (('alone', alone), ('padded to 5000', padded), ('at another row', _clip(flipped, B - 1 - b, La, Lp)),
                         ('garbage padding', _clip(junk, b, La, Lp))):
            for k in want:
                assert torch.equal(got[k], want[k]), (tag, b, La, Lp, k, float((got[k] - want[k]).abs().max()))


def _oracle_alone(batch, eps, b):
    if b not in _REFS:
        one = _slice(batch, [b], [LA[b]], [LP[b]])
        r = _oracle_forward(one, eps[b:b + 1])
        _REFS[b] = {k: v.cpu() for k, v in r.items()}
    return _REFS[b]


def test_each_clip_matches_the_float64_oracle_of_the_clip_alone(use_tc):
    batch, B = _batch(), len(LA)
    eps = _eps(B, 'randn')
    got = _forward(_model(use_tc).eval(), batch, eps, LA, LP)
    for b in range(B):
        ref = dict(_oracle_alone(batch, eps, b))
        for w in ('a2a', 'p2p'):                                  # z = m + eps * exp(logs) of the oracle's statistics
            ref[f'{w} z_q'] = ref[f'{w} m_q'] + eps[b:b + 1].double() * ref[f'{w} logs_q'].exp()
        g = _clip(got, b, LA[b], LP[b])
        for k in g:
            _check(f'clip {b} ({LA[b]} x {LP[b]}) tc={use_tc} {k}', g[k].reshape(-1), ref[k][0].reshape(-1), FWD_BARS[use_tc])


def test_bad_lengths_raise_before_any_launch(monkeypatch):
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    batch = _ragged([300, 212], [236, 332], 3)
    b = {k: v.cuda() for k, v in batch.items()}
    m = _model(True).eval()
    calls = []
    monkeypatch.setattr(MleSVBVAE, 'prepare_condition', lambda *a, **k: calls.append(1))
    kw = dict(b, infer=False, concurrent_ways=WAYS, eps=_eps(2, 'zero').cuda())
    for la, lp, match in (([300, 212], None, 'both'), ([300, 59], [236, 332], r'amateur_lens\[1\]'),
                          ([300, 210], [236, 332], r'amateur_lens\[1\].*multiple of 4'), ([300, 212], [236, 336], r'prof_lens\[1\] = 336'),
                          ([300.0, 212], [236, 332], r'amateur_lens\[0\] = 300.0'), ([300], [236, 332], 'amateur_lens: 1 frame counts')):
        with torch.no_grad(), pytest.raises(ValueError, match=match):
            m(**kw, amateur_lens=la, prof_lens=lp)
    assert not calls
    t = _model(True, trainable=True).train()
    with pytest.raises(RuntimeError, match='inference only'):
        t(**kw, amateur_lens=[300, 212], prof_lens=[236, 332])
    assert not calls


# ---------------------------------------------------------------------------------------------------------- the beautifier
@pytest.fixture(scope='module')
def experiment(tmp_path_factory):
    return make_experiment(str(tmp_path_factory.mktemp('batch_invariant')))


def _beautifier(work):
    from neuralsvb_b200.modules.fastspeech import multi_window_disc as M
    from neuralsvb_b200.modules.voice_conversion import vc_modules as V
    V.USE_TC, M.USE_TC = True, True
    return BF.SVBBeautifier(work)


def test_song_tail_segment_matches_its_unpadded_oracle(experiment):
    work, pairs = experiment
    b = _beautifier(work)
    hop = int(b.hp['hop_size'])
    b._vocode = lambda mel_out, f0, Tp, seed, first_clip=0: torch.zeros(sum(Tp) * hop, device=b.device)
    rec, spy = _Inputs(b.model), SongSpy(b)
    a, p = song(*SONG)
    emb = np.load(pairs[0][3])
    b.beautify_songs([a], [p], [emb], seed=3)
    call, default_mel = rec.calls[-1], spy.seen['_model_on'][0].cpu()
    keys = ('amateur_mel', 'prof_mel', 'amateur_pitch', 'prof_pitch', 'amateur_spk_id', 'prof_spk_id', 'a2p_alignment')
    batch, eps = {k: call[k] for k in keys}, call['eps'].cpu()
    La, Lp = _lengths(batch['amateur_pitch']), _lengths(batch['prof_pitch'])
    tail = len(La) - 1
    assert Lp[tail] < batch['prof_mel'].shape[1] / 4, (Lp, batch['prof_mel'].shape)
    sd = {k: v.detach().clone() for k, v in b.model.state_dict().items()}
    got = _forward(b.model, batch, eps, La, Lp)['a2p mel_out'][tail, :Lp[tail]]
    one = _slice(batch, [tail], [La[tail]], [Lp[tail]])
    ref = _oracle_forward(one, eps[tail:tail + 1], sd)['a2p mel_out'][0].cpu()
    _check(f'song tail a2p mel_out ({La[tail]} x {Lp[tail]} frames) length-aware', got.reshape(-1), ref.reshape(-1), FWD_BARS[True])
    l2, li = _err(default_mel[tail, :Lp[tail]].reshape(-1), ref.reshape(-1))
    print(f'DEFAULT MODE song tail vs its unpadded oracle: rel L2 {l2:.2e}, rel L-inf {li:.2e} '
          f'({max(l2 / FWD_BARS[True][0], li / FWD_BARS[True][1]):.0f}x the bf16x3 forward bar)')
    assert li > 100 * FWD_BARS[True][1]
    # the beautifier's own length-aware call on that song gives those bits for its tail
    spy2 = SongSpy(b)
    b.beautify_songs([a], [p], [emb], seed=3, batch_invariant=True)
    assert torch.equal(spy2.seen['_model_on'][0].cpu()[tail, :Lp[tail]], got)


class _VocodeArgs:
    def __init__(self, b):
        self.f0, fn = [], b._vocode

        def call(mel_out, f0, Tp, seed, first_clip=0):
            self.f0.append((f0.detach().cpu().clone(), list(Tp), seed))
            return fn(mel_out, f0, Tp, seed, first_clip)
        b._vocode = call


def test_beautify_batch_pairs_equal_the_pairs_alone(experiment):
    work, pairs = experiment
    b = _beautifier(work)
    pairs = regular(pairs)
    B = len(pairs)
    assert B >= 8
    eps = torch.randn(B, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(9))
    spy, voc = BatchSpy(b), _VocodeArgs(b)
    got = b.beautify_batch([p[1] for p in pairs], [p[2] for p in pairs], [p[3] for p in pairs], seed=9, eps=eps, batch_invariant=True)
    mel = spy.seen['_acoustic'].cpu()
    f0, Tp, seed = voc.f0[-1]
    ref_wavs = b.vocoder.spec2wav_batch([mel[i, :t].numpy() for i, t in enumerate(Tp)], [f0[i, :t].numpy() for i, t in enumerate(Tp)],
                                        seed=seed)
    for i, p in enumerate(pairs):
        assert np.array_equal(got[i], ref_wavs[i]), f'pair {i}: waveform'
        alone = BatchSpy(b)
        one = b.beautify(p[1], p[2], p[3], seed=9, eps=eps[i:i + 1], batch_invariant=True)
        assert torch.equal(alone.seen['_acoustic'][0, :Tp[i]].cpu(), mel[i, :Tp[i]]), f'pair {i}: a2p mel'
        if i == 0:
            assert np.array_equal(one, got[0]), 'pair 0: waveform alone'
    # one pair: the two modes differ by rounding only
    default = BatchSpy(b)
    b.beautify(pairs[1][1], pairs[1][2], pairs[1][3], seed=9, eps=eps[1:2])
    d = float((default.seen['_acoustic'][0, :Tp[1]].cpu() - mel[1, :Tp[1]]).abs().max()) / float(mel[1, :Tp[1]].abs().max())
    print(f'one pair, default vs length-aware a2p mel: {d:.2e} of max |mel|')
    assert d < FWD_BARS[True][1] * 10


def test_beautify_songs_segments_equal_segments_alone(experiment):
    work, pairs = experiment
    b = _beautifier(work)
    emb = np.load(pairs[0][3])
    hop = int(b.hp['hop_size'])
    # one-segment song: exactly beautify(..., batch_invariant=True) of the pair
    a, p = song(43, 900, 860)
    one_song = b.beautify_songs([a], [p], [emb], seed=4, batch_invariant=True)[0]
    one_pair = b.beautify(a, p, emb, seed=4, batch_invariant=True)
    assert np.array_equal(one_song, one_pair)
    # a multi-segment song: every segment's a2p mel equals that segment run alone
    b._vocode = lambda mel_out, f0, Tp, seed, first_clip=0: torch.zeros(sum(Tp) * hop, device=b.device)
    rec, spy = _Inputs(b.model), SongSpy(b)
    a, p = song(41, 10400, 10200)
    b.beautify_songs([a], [p], [emb], seed=5, batch_invariant=True)
    call, out = rec.calls[-1], spy.seen['_model_on'][0].cpu()
    assert call['amateur_lens'] is not None
    La, Lp = [int(x) for x in call['amateur_lens']], [int(x) for x in call['prof_lens']]
    assert len(La) >= 2
    keys = ('amateur_mel', 'prof_mel', 'amateur_pitch', 'prof_pitch', 'amateur_spk_id', 'prof_spk_id', 'a2p_alignment')
    batch = {k: call[k] for k in keys}
    for k in range(len(La)):
        one = _slice(batch, [k], [La[k]], [Lp[k]])
        alone = _forward(b.model, one, call['eps'][k:k + 1].cpu(), [La[k]], [Lp[k]])['a2p mel_out'][0]
        assert torch.equal(alone, out[k, :Lp[k]]), k

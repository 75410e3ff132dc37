"""Shape-aware DTW on the GPU (csrc/sadtw.cu) against the oracle (oracle/sadtw.py) and tests/golden/sadtw.npz, bit for bit:
histograms, the skewed cost, the DTW matrix through the time_warp drop-in, the direction-derived alignments and the path cost."""
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200.modules.voice_conversion.dtw import a2p_alignment_batch, align_pitch
from neuralsvb_b200.modules.voice_conversion.dtw import align as A
from neuralsvb_b200.modules.voice_conversion.dtw import core
from neuralsvb_b200.modules.voice_conversion.dtw import enhance_sadtw as EH
from neuralsvb_b200.modules.voice_conversion.dtw import shape_aware_dtw as SA
from neuralsvb_b200.utils import synthetic as S
from oracle import sadtw as O
from oracle.gen_golden_sadtw import KINDS, METHODS, SADTW_CASES, make_input

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'sadtw.npz')
DROP_IN = {'SADTW': (SA, SA.SADTW), 'EHSADTW': (EH, EH.EHSADTW)}


def _as(kind, f):
    """f0 as numpy / torch, float32 / float64, host / device."""
    dt, where = kind.split('_')
    a = f.astype(np.float32 if dt == 'f32' else np.float64)
    if where == 'np':
        return a
    t = torch.from_numpy(a)
    return t.cuda() if where == 'dev' else t


INPUT_KINDS = ('f32_np', 'f64_np', 'f32_torch', 'f64_torch', 'f32_dev', 'f64_dev')
# (seed, S, T): T / S below, at and above 1, lengths 2 .. 1400
SHAPES = [(31, 2, 2), (32, 2, 5), (33, 5, 2), (34, 17, 14), (35, 40, 40), (36, 90, 113), (37, 300, 240), (38, 700, 701),
          (39, 1378, 1400), (40, 1100, 1500)]


def skew_order(R, C):
    """(i, j) of the cells of an R x C matrix in the kernels' anti-diagonal-major order."""
    ii = [np.arange(max(0, d - C + 1), min(d, R - 1) + 1) for d in range(R + C - 1)]
    i = np.concatenate(ii)
    j = np.concatenate([d - x for d, x in enumerate(ii)])
    return i, j


@pytest.mark.parametrize('method', METHODS)
@pytest.mark.parametrize('kind', INPUT_KINDS)
def test_histogram_kernel_matches_oracle(method, kind):
    for seed, Sn, Tn in SHAPES[:8]:
        a, b = S.make_f0_pair(seed, Sn, Tn)
        fa, fb = _as(kind, a), _as(kind, b)
        h, c = core.histogram([fa, fb], method, [1.0, Tn / Sn], counts=True)
        h, c = h.cpu().numpy(), c.cpu().numpy()
        assert np.array_equal(h[:Sn], O.histogram(fa, method)), (seed, 'src')
        assert np.array_equal(h[Sn:], O.histogram(fb, method, Tn / Sn)), (seed, 'tgt')
        assert np.array_equal(c[:Sn], O.counts(fa, method))


@pytest.mark.parametrize('method', METHODS)
@pytest.mark.parametrize('kind', ('f32_np', 'f64_dev'))
def test_batched_pipeline_is_the_oracle_bit_for_bit(method, kind):
    """One ragged batch: histograms, skewed cost, alignments and path costs against the oracle, pair by pair."""
    pairs = [S.make_f0_pair(seed, Sn, Tn) for seed, Sn, Tn in SHAPES]
    srcs, tgts = [_as(kind, a) for a, _ in pairs], [_as(kind, b) for _, b in pairs]
    r = core.align_batch(srcs, tgts, method, keep_workspace=True)
    ws = r.workspace.cpu().numpy()
    sec = r.sections
    hist = ws[sec[2]:sec[3]].view(np.float32)
    cost = ws[sec[3]:sec[4]].view(np.float32)
    rows_src = sum(r.src_len)
    got = r.split()
    pc = r.path_cost.cpu().numpy()
    hs_off = ht_off = cell = 0
    for p, (a, b) in enumerate(zip(srcs, tgts)):
        Sn, Tn = len(a), len(b)
        al, last, m = O.shape_aware_align(a, b, method, full=True)
        hs = hist[(hs_off) * 48:(hs_off + Sn) * 48].reshape(Sn, 48)
        ht = hist[(rows_src + ht_off) * 48:(rows_src + ht_off + Tn) * 48].reshape(Tn, 48)
        assert np.array_equal(hs, m['hist_src']) and np.array_equal(ht, m['hist_tgt']), p
        i, j = skew_order(Tn, Sn)
        assert np.array_equal(cost[cell:cell + Sn * Tn], m['cost'][i, j]), p
        assert np.array_equal(got[p], al), p
        assert pc[p] == np.float32(last) or (np.isinf(pc[p]) and np.isinf(last)), (p, pc[p], last)
        hs_off += Sn
        ht_off += Tn
        cell += Sn * Tn


@pytest.mark.parametrize('dtype', (np.float32, np.float64))
@pytest.mark.parametrize('shape', ((1, 1), (1, 7), (7, 1), (2, 2), (3, 50), (50, 3), (64, 64), (300, 200), (257, 1031)))
def test_time_warp_drop_in_on_arbitrary_costs(dtype, shape):
    rs = np.random.RandomState(shape[0] * 1000 + shape[1])
    c = rs.rand(*shape).astype(dtype)
    c[rs.rand(*shape) < 0.2] = 0.25                                      # exact ties between paths
    dtw = A.time_warp(c)
    assert dtw.dtype == dtype and np.array_equal(dtw, O.time_warp(c))
    for where in ('np', 'host', 'dev'):
        x = c if where == 'np' else (torch.from_numpy(c).cuda() if where == 'dev' else torch.from_numpy(c))
        got = A.align_from_distances(x)
        assert isinstance(got, list) and got == O.align_from_distances(c), where
    al, pc, full = core.dtw(torch.from_numpy(c).cuda(), matrix=True)
    assert pc.dtype == torch.from_numpy(c).dtype and pc.cpu().numpy()[0] == dtw[-1, -1]


def test_time_warp_on_the_reference_matrix():
    g = np.load(GOLDEN)
    assert np.array_equal(A.time_warp(g['matrix/cost']), g['matrix/dtw'])
    assert A.align_from_distances(g['matrix/cost']) == g['matrix/alignment'].tolist()


@pytest.mark.parametrize('method', METHODS)
@pytest.mark.parametrize('kind', KINDS)
def test_drop_ins_reproduce_the_reference_fixture(method, kind):
    g = np.load(GOLDEN)
    mod, fn = DROP_IN[method]
    for name, (seed, Sn, Tn) in SADTW_CASES.items():
        a, b = S.make_f0_pair(seed, Sn, Tn)
        fa, fb = make_input(kind, a), make_input(kind, b)
        out, alignment = fn(fa, fb, fa)
        ref = g[f'{name}/{method}/{kind}/alignment']
        assert isinstance(alignment, list) and alignment == ref.tolist(), name
        assert type(out) is type(fa) and np.array_equal(np.asarray(out), np.asarray(fa)[ref])
        if f'{name}/{method}/{kind}/hist_src' in g:
            hs = mod.cal_hist_of_f0(fa, normalize_hist=True)
            ht = mod.cal_hist_of_f0(fb, normalize_hist=True, scale_factor=Tn / Sn)
            assert isinstance(hs, list) and np.array_equal(torch.tensor(hs).numpy(), g[f'{name}/{method}/{kind}/hist_src'])
            assert np.array_equal(torch.tensor(ht).numpy(), g[f'{name}/{method}/{kind}/hist_tgt'])
            d = mod.cal_shape_dist(fa, fb, Sn, Tn)
            assert tuple(d.shape) == (1, Sn, Tn) and d.dtype == torch.float32
            assert np.array_equal(d[0].cpu().numpy().T, O.cost(O.histogram(fa, method), O.histogram(fb, method, Tn / Sn)))


def test_dtw_align_batch_drop_in():
    """SADTW's DTW_align: padded [B, S, 1] f0 with true lengths; the histograms run over the padded rows, as in the reference."""
    pairs = [S.make_f0_pair(50 + b, 60 + 7 * b, 70 - 3 * b) for b in range(3)]
    Sm, Tm = max(len(a) for a, _ in pairs), max(len(t) for _, t in pairs)
    srcs, tgts = torch.zeros(3, Sm, 1), torch.zeros(3, Tm, 1)
    for b, (a, t) in enumerate(pairs):
        srcs[b, :len(a), 0], tgts[b, :len(t), 0] = torch.from_numpy(a), torch.from_numpy(t)
    inputs = torch.arange(3 * Sm).reshape(3, Sm, 1).float()
    sl, tl = torch.tensor([len(a) for a, _ in pairs]), torch.tensor([len(t) for _, t in pairs])
    out = SA.DTW_align(srcs, tgts, inputs, srcs_lens=sl, tgt_lens=tl)
    assert tuple(out.shape) == (3, Tm, 1)
    for b in range(3):
        al, _ = O.shape_aware_align(srcs[b], tgts[b], 'SADTW', scale=int(tl[b]) / int(sl[b]))
        assert torch.equal(out[b], inputs[b][al])


def test_ragged_batch_equals_single_calls_and_repeats():
    rs = np.random.RandomState(7)
    shapes = []
    for b in range(64):                       # T / S in [0.5, 2]: a much shorter professional take has frames without neighbours
        Sn = int(rs.randint(2, 400))
        shapes.append((100 + b, Sn, max(2, int(Sn * rs.uniform(0.5, 2.0)))))
    pairs = [S.make_f0_pair(*s) for s in shapes]
    srcs, tgts = [torch.from_numpy(a).float().cuda() for a, _ in pairs], [torch.from_numpy(t).float().cuda() for _, t in pairs]
    r1, r2 = core.align_batch(srcs, tgts), core.align_batch(srcs, tgts)
    assert torch.equal(r1.alignment, r2.alignment) and torch.equal(r1.path_cost, r2.path_cost)
    got = r1.split()
    for p in range(64):
        one = core.align_batch([srcs[p]], [tgts[p]])
        assert np.array_equal(one.split()[0], got[p]) and one.path_cost[0] == r1.path_cost[p], p
    assert [len(x) for x in align_pitch(srcs, tgts)] == [s[2] for s in shapes]


@pytest.mark.parametrize('shape', ((5000, 5000), (5000, 320), (2, 5000), (4000, 5000)))
def test_long_pairs(shape):
    a, b = S.make_f0_pair(77, *shape)
    got = core.align_batch([a.astype(np.float32)], [b.astype(np.float32)])
    al, last = O.shape_aware_align(a.astype(np.float32), b.astype(np.float32), 'EHSADTW')
    assert np.array_equal(got.split()[0], al)
    assert got.path_cost.cpu().numpy()[0] == np.float32(last)


def test_a2p_alignment_batch_clips_pads_and_feeds_mle_svb_vae():
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    from tests.test_oracle_golden import SVB_HP
    B, Ta, Tp = 2, 96, 120
    la, lp = [96, 88], [120, 108]
    af, pf = torch.zeros(B, Ta), torch.zeros(B, Tp)
    for b in range(B):
        a, p = S.make_f0_pair(90 + b, la[b], lp[b])
        af[b, :la[b]], pf[b, :lp[b]] = torch.from_numpy(a), torch.from_numpy(p)
    align = a2p_alignment_batch(af.cuda(), pf.cuda(), torch.tensor(la), torch.tensor(lp))
    assert align.dtype == torch.int64 and align.is_cuda and tuple(align.shape) == (B, Tp)
    for b in range(B):
        ref, _ = O.shape_aware_align(af[b, :la[b]], pf[b, :lp[b]], 'EHSADTW')
        assert np.array_equal(align[b, :lp[b]].cpu().numpy(), np.minimum(ref, la[b] - 1))
        assert (align[b, lp[b]:] == 0).all() and int(align[b].max()) <= la[b] - 1
    batch = {k: v.cuda() for k, v in S.make_svb_batch(B, Ta, Tp, 1234).items()}
    batch['a2p_alignment'] = align
    m = MleSVBVAE(80, hp=SVB_HP)
    m.load_state_dict(S.make_svb_state_dict(1234), strict=True)
    with torch.no_grad():
        out = m.eval().cuda()(**batch, infer=False, concurrent_ways=['a2a', 'p2p', 'a2p'])
    assert tuple(out['a2p']['mel_out'].shape) == (B, Tp, 80) and torch.isfinite(out['a2p']['mel_out']).all()


def test_device_inputs_rejected_before_launch():
    with pytest.raises(ValueError, match='NaN or inf'):
        EH.EHSADTW(torch.tensor([200.0, float('inf'), 201.0]).cuda(), torch.ones(4).cuda(), torch.ones(3))
    with pytest.raises(ValueError, match='at least 2'):
        SA.SADTW(np.ones(1), np.ones(4), np.ones(1))
    with pytest.raises(ValueError, match='no neighbour'):
        core.align_batch([np.linspace(200, 210, 200)], [np.linspace(200, 210, 200)], 'SADTW', scales=[0.01])
    with pytest.raises(ValueError, match='no neighbour'):           # scale 2 / 5000: the reference divides by zero
        EH.EHSADTW(np.linspace(200, 210, 5000), np.linspace(200, 210, 2), np.ones(5000))

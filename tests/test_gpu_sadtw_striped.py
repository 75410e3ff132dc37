"""-m gpu: the striped shape-aware DTW (align_songs, svb_sadtw_align_striped) against align_long bit for bit, alignment and path
cost: single pass and checkpointed at forced stripe widths (SVB_DTW_STRIPE_DIAGS), the one-CTA and the cluster kernel, SADTW and
EHSADTW, float32 and float64 f0; against the oracle past 8192 frames; its device memory within the budget; and beautify_songs with
an alignment budget that forces the checkpointed passes."""
import numpy as np
import pytest
import torch

from neuralsvb_b200.inference import beautify as BF
from neuralsvb_b200.modules.voice_conversion.dtw import core
from neuralsvb_b200.utils import synthetic as S
from oracle import sadtw as O
from tests.test_gpu_song import Spy, exp, keep_hparams  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
GiB = 1 << 30


@pytest.fixture(autouse=True)
def no_hooks(monkeypatch):
    monkeypatch.delenv('SVB_DTW_STRIPE_DIAGS', raising=False)
    monkeypatch.delenv('SVB_DTW_CTA_CELLS', raising=False)


def contours(shapes, dtype=np.float32, seed=500):
    pairs = [S.make_f0_pair(seed + k, s, t) for k, (s, t) in enumerate(shapes)]
    return [a.astype(dtype) for a, _ in pairs], [b.astype(dtype) for _, b in pairs]


def striped(monkeypatch, srcs, tgts, method='EHSADTW', K=None, budget=core.SONGS_WORKSPACE_BYTES):
    if K is None:
        monkeypatch.delenv('SVB_DTW_STRIPE_DIAGS', raising=False)
    else:
        monkeypatch.setenv('SVB_DTW_STRIPE_DIAGS', str(K))
    r = core.align_songs(srcs, tgts, method, workspace_bytes=budget)
    monkeypatch.delenv('SVB_DTW_STRIPE_DIAGS', raising=False)
    assert r.mode == ('single_pass' if K is None and budget == core.SONGS_WORKSPACE_BYTES else 'checkpointed')
    assert K is None or r.stripe_diags == K
    return r


def assert_same(ref, got):
    for p, (x, y) in enumerate(zip(ref.split(), got.split())):
        assert np.array_equal(x, y), f'pair {p}: alignment'
    assert torch.equal(ref.path_cost, got.path_cost), (ref.path_cost, got.path_cost)


# R = professional frames (T), C = amateur frames (S): R < C, R > C, R = C, 2-frame takes, one-CTA pairs and one over 8192 frames
MIXED = [(40, 60), (60, 40), (300, 300), (2, 2), (2, 90), (5, 2), (1500, 1100), (8300, 8500), (700, 5000)]


@pytest.mark.parametrize('K', (None, 64, 1000))
@pytest.mark.parametrize('dtype', (np.float32, np.float64))
@pytest.mark.parametrize('method', ('EHSADTW', 'SADTW'))
def test_ragged_batch_equals_align_long(monkeypatch, method, dtype, K):
    srcs, tgts = contours(MIXED, dtype)
    ref = core.align_long(srcs, tgts, method)
    assert_same(ref, striped(monkeypatch, srcs, tgts, method, K))


# SVB_DTW_CTA_CELLS=64 puts pairs over 64 frames on clusters of up to 8 CTAs (449 = 7 x 64 + 1: one cell in the last CTA)
SMALL = [(449, 449), (130, 700), (700, 130), (65, 300), (2, 2), (2, 90), (40, 60), (20, 10)]


@pytest.mark.parametrize('cells', (None, 64))
@pytest.mark.parametrize('K', (1, 2, 3))
def test_one_two_and_three_diagonal_stripes(monkeypatch, K, cells):
    if cells:
        monkeypatch.setenv('SVB_DTW_CTA_CELLS', str(cells))
    for method, dtype in (('EHSADTW', np.float32), ('SADTW', np.float64)):
        srcs, tgts = contours(SMALL, dtype, seed=40)
        assert_same(core.align_long(srcs, tgts, method), striped(monkeypatch, srcs, tgts, method, K))


@pytest.mark.parametrize('cells', (None, 64))
@pytest.mark.parametrize('K', (100, 150, 300))
def test_stripe_boundaries_where_the_diagonal_length_changes(monkeypatch, K, cells):
    """Pairs of 301 x 601 and 601 x 301 frames: diagonals start shrinking or stop growing at d = 300 and d = 600, which every
    K here puts on a stripe boundary."""
    if cells:
        monkeypatch.setenv('SVB_DTW_CTA_CELLS', str(cells))
    srcs, tgts = contours([(301, 601), (601, 301), (301, 301), (601, 601)], seed=70)
    assert_same(core.align_long(srcs, tgts), striped(monkeypatch, srcs, tgts, K=K))


@pytest.mark.parametrize('K', (None, 3, 64))
def test_thousand_frame_pairs_on_clusters(monkeypatch, K):
    monkeypatch.setenv('SVB_DTW_CTA_CELLS', '1000')
    srcs, tgts = contours([(1001, 1001), (2500, 4000), (4000, 2500), (3001, 3200), (999, 1200), (30, 40)], seed=310)
    assert_same(core.align_long(srcs, tgts), striped(monkeypatch, srcs, tgts, K=K))


@pytest.mark.parametrize('K', (None, 500))
def test_equals_the_oracle_past_8192_frames(monkeypatch, K):
    a, b = S.make_f0_pair(77, 9000, 16500)
    got = striped(monkeypatch, [a], [b], K=K)
    al, last = O.shape_aware_align(a, b, 'EHSADTW')
    assert np.array_equal(got.split()[0], al)
    assert got.path_cost.cpu().numpy()[0] == np.float32(last)


def test_a_four_minute_pair_checkpointed_in_one_gib(monkeypatch):
    srcs, tgts = contours([(40000, 36000)], seed=9)
    ref = core.align_long(srcs, tgts)
    got = striped(monkeypatch, srcs, tgts, budget=GiB)
    assert got.workspace_bytes <= GiB
    assert_same(ref, got)


def test_a_65536_frame_pair_stays_within_its_budget(monkeypatch):
    a, b = S.make_f0_pair(12, 65536, 60000)
    a, b = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ck = striped(monkeypatch, [a], [b], budget=GiB)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    out = ck.alignment.numel() * 8 + 512            # the alignment and the path cost (one 512-byte allocator block)
    assert peak <= GiB + out, (peak, GiB + out)
    assert ck.stripe_diags > 1 and ck.workspace_bytes <= GiB
    single = striped(monkeypatch, [a], [b])
    assert_same(single, ck)
    r = core.align_songs([a], [b], workspace_bytes=GiB, stage_ms=True)
    assert len(r.stage_ms) == 4 and min(r.stage_ms) >= 0 and r.stage_ms[2] > 0
    assert_same(single, r)


def song_frames(songs, hop=128):
    return [len(s[0]) // hop + 1 for s in songs], [len(s[1]) // hop + 1 for s in songs]


def test_beautify_songs_checkpointed_equals_the_default(exp):  # noqa: F811
    work, songs, emb = exp
    b = BF.SVBBeautifier(work)
    B, budget = len(songs), 64 << 20
    assert core.striped_plan(*song_frames(songs), budget).mode == 1             # checkpointed at this budget
    assert core.striped_plan(*song_frames(songs), BF.SONG_ALIGN_BYTES).mode == 0
    eps = torch.randn(B, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(11))
    call = ([s[0] for s in songs], [s[1] for s in songs], [emb] * B)
    ref = b.beautify_songs(*call, seed=7, eps=eps)
    b.timing = True
    got = b.beautify_songs(*call, seed=7, eps=eps, align_bytes=budget)
    assert len(b.align_ms) == 1 and len(b.align_ms[0]) == 4 and b.align_ms[0][2] > 0
    for i in range(B):
        assert got[i].dtype == np.float32 and np.array_equal(got[i], ref[i]), f'song {i}'


def test_beautify_songs_refuses_a_budget_below_the_minimum_before_the_front_end(exp):  # noqa: F811
    work, songs, emb = exp
    b = BF.SVBBeautifier(work)
    spy = Spy(b)
    with pytest.raises(ValueError, match=r'align_bytes = 100000: .*below the minimum of [0-9]+ bytes'):
        b.beautify_songs([songs[1][0]], [songs[1][1]], [emb], align_bytes=100000)
    assert '_front_end' not in spy.seen

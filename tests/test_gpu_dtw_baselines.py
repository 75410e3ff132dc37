"""Baseline pitch alignments on the GPU (csrc/sadtw.cu: LoNDTW, NaiveDTW, ZMNaiveDTW, NNaiveDTW, NInterpo) against a host
emulation of the kernels' own operation order, the oracle (oracle/dtw_baselines.py) and tests/golden/dtw_baselines.npz."""
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200.modules.voice_conversion.dtw import a2p_alignment_batch, alignment_accuracy, core
from neuralsvb_b200.modules.voice_conversion.dtw import local_norm_dtw as LN
from neuralsvb_b200.modules.voice_conversion.dtw import naive_dtw as ND
from neuralsvb_b200.modules.voice_conversion.dtw import naive_interpo as NI
from neuralsvb_b200.utils import synthetic as S
from oracle import dtw_baselines as O
from oracle import sadtw as OS
from oracle.gen_golden_dtw_baselines import DTW_METHODS, INTERPO_CASES, KINDS, make_input, mel_pair
from oracle.gen_golden_sadtw import SADTW_CASES

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'dtw_baselines.npz')
DROP_IN = {'LoNDTW': LN.LoNDTW, 'NaiveDTW': ND.NaiveDTW, 'ZMNaiveDTW': ND.ZMNaiveDTW, 'NNaiveDTW': ND.NNaiveDTW}


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


def _emulate_features(method, x):
    """The kernels' per-frame features in the input's type, host torch, same operation order: [S, K]."""
    dt = x.dtype
    if method == 'LoNDTW':
        ctx = O.local_context(x)
        m = torch.zeros(x.shape[0], dtype=dt)
        for k in range(64):
            m = m + ctx[:, k]
        m = m / 64
        return ctx - m[:, None]
    if method == 'NaiveDTW':
        return x if x.dim() == 2 else x[:, None]
    x = x.reshape(-1)
    mu = x.double().sum().to(dt) / x.shape[0]
    f = x - mu
    if method == 'NNaiveDTW':
        std = torch.sqrt(((x.double() - x.double().sum() / x.shape[0]) ** 2).sum() / (x.shape[0] - 1)).to(dt)
        f = f / (std + 1e-8)
    return f[:, None]


def _emulate_cost(method, a, b):
    """[S, T] in the input's type with the kernel's order: the product form (sum_k (-2 x_k) y_k, then + |x|^2, then + |y|^2) or,
    with at most 25 frames on both sides, sqrt(sum_k (x_k - y_k)^2)."""
    x, y = _emulate_features(method, a), _emulate_features(method, b)
    S_, T_ = x.shape[0], y.shape[0]
    acc = torch.zeros(S_, T_, dtype=x.dtype)
    if S_ <= 25 and T_ <= 25:
        for k in range(x.shape[1]):
            d = x[:, k, None] - y[None, :, k]
            acc = acc + d * d
        return torch.sqrt(acc)
    xn = torch.zeros(S_, dtype=x.dtype)
    yn = torch.zeros(T_, dtype=x.dtype)
    for k in range(x.shape[1]):
        acc = acc + (-2 * x[:, k, None]) * y[None, :, k]
        xn = xn + x[:, k] * x[:, k]
        yn = yn + y[:, k] * y[:, k]
    return torch.sqrt(((acc + xn[:, None]) + yn[None, :]).clamp_min(0))


def _mean_shift(method, a, b):
    """A bound on how far one frame's ZM / NN feature may move between the kernel and torch: both round the contour's mean (and
    std) once, but torch's CPU sum runs in an order that depends on the host's vector width, so the two may differ by an ulp of
    the mean, and NN divides that by the std.  0 for the other methods (their per-frame context means are covered by the
    cancellation bound)."""
    if method not in ('ZMNaiveDTW', 'NNaiveDTW'):
        return 0.0
    eps = float(torch.finfo(a.dtype).eps)
    d = 0.0
    for x in (a.double().reshape(-1), b.double().reshape(-1)):
        mu = float(x.mean().abs())
        if method == 'ZMNaiveDTW':
            d += 4 * eps * mu
        else:
            sd = float(x.std())
            d += 4 * eps * (mu / sd + float((x - x.mean()).abs().max()) / sd)
    return d


def _pairs():
    out = [(name, *S.make_f0_pair(seed, Sn, Tn)) for name, (seed, Sn, Tn) in SADTW_CASES.items()]
    a, b = mel_pair()
    return out, (a, b)


@pytest.mark.parametrize('dt', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', DTW_METHODS)
def test_cost_kernel_against_emulated_formula_and_oracle(method, dt):
    f0s, mel = _pairs()
    cases = [(name, torch.from_numpy(a).to(dt), torch.from_numpy(b).to(dt)) for name, a, b in f0s]
    if method == 'NaiveDTW':
        cases = [(n, a[:, None], b[:, None]) for n, a, b in cases] + [('mel', mel[0].to(dt), mel[1].to(dt))]
    f0_cases = [c for c in cases if c[0] != 'mel']      # a batch has one feature width
    got = core.baseline_costs([a.cuda() for _, a, _ in f0_cases], [b.cuda() for _, _, b in f0_cases], method)
    if method == 'NaiveDTW':
        got += core.baseline_costs([cases[-1][1].cuda()], [cases[-1][2].cuda()], method)
    tol = 1e-6 if dt == torch.float32 else 1e-12
    eps = float(torch.finfo(dt).eps)
    for (name, a, b), g in zip(cases, got):
        g = g.cpu()
        e = _emulate_cost(method, a, b)
        assert g.dtype == dt and g.shape == e.shape, name
        x = _emulate_features(method, a).double()
        y = _emulate_features(method, b).double()
        K, d = x.shape[1], _mean_shift(method, a, b)

        def within_cancellation(ref):
            # the squared costs differ by at most the product form's cancellation bound plus the features' shift
            ref = ref.double()
            bound = 4 * (K + 2) * eps * ((x * x).sum(1)[:, None] + (y * y).sum(1)[None, :]) + 2 * (ref + d) * d + 1e-30
            return bool(((g.double() ** 2 - ref ** 2).abs() <= bound).all())
        if method in ('ZMNaiveDTW', 'NNaiveDTW') and dt == torch.float64:
            # the kernel sums the float64 contour in a block order the emulation cannot follow: the mean may differ by an ulp,
            # which the product form's cancellation turns into more than 1e-12 near zero cost
            assert within_cancellation(e), (method, dt, name)
        else:
            err = float((g - e).abs().max() / e.abs().max())
            assert err <= tol, (method, dt, name, err)
        # against torch.cdist, the reference's own cost, which sums in another order
        assert within_cancellation(O.cdist_cost(method, a, b)), (method, dt, name)


def _native_path_cost_ok(method, a, b, al_native, golden_al):
    """The fallback when a near tie went the other way: the native path, evaluated under the reference's cost matrix (the
    oracle's, which reproduces it), costs what the reference's DTW value says, within 1e-6 relative plus, for ZM / NN, the
    mean's rounding (_mean_shift) on every cell of a path."""
    ref_cost = O.cost(method, a, b)
    ref_val = OS.time_warp(ref_cost)[-1, -1]
    nat_cost = core.baseline_costs([a.cuda() if torch.is_tensor(a) else a], [b.cuda() if torch.is_tensor(b) else b],
                                   method)[0].T.contiguous().cpu().numpy()
    nat_dtw = OS.time_warp(nat_cost)
    assert np.array_equal(np.asarray(OS.align_from_dtw(nat_dtw)), al_native), 'the DTW kernel disagrees with its own cost'
    val = O.path_cost(ref_cost.astype(np.float64), nat_dtw)
    ta, tb = (torch.as_tensor(np.asarray(a)), torch.as_tensor(np.asarray(b))) if not torch.is_tensor(a) else (a, b)
    slack = 2 * (ref_cost.shape[0] + ref_cost.shape[1]) * _mean_shift(method, ta, tb)
    return abs(val - float(ref_val)) <= 1e-6 * abs(float(ref_val)) + slack


def test_drop_ins_against_reference_fixture(golden):
    fallbacks, total = [], 0
    for name, (seed, Sn, Tn) in SADTW_CASES.items():
        src, tgt = S.make_f0_pair(seed, Sn, Tn)
        for method in DTW_METHODS:
            for kind in KINDS[method]:
                a, b = make_input(kind, src, method), make_input(kind, tgt, method)
                for where in ('host', 'dev'):
                    if where == 'dev' and not torch.is_tensor(a):
                        continue
                    aa, bb = (a.cuda(), b.cuda()) if where == 'dev' else (a, b)
                    out, al = DROP_IN[method](aa, bb, aa)
                    ref = golden[f'{name}/{method}/{kind}/alignment']
                    total += 1
                    assert isinstance(al, list) and len(al) == Tn
                    assert type(out) is type(aa) and out.shape[0] == Tn
                    if not np.array_equal(np.asarray(al), ref):
                        assert _native_path_cost_ok(method, a, b, np.asarray(al), ref), (name, method, kind, where)
                        fallbacks.append((name, method, kind, where))
    a, b = mel_pair()
    _, al = ND.NaiveDTW(a.cuda(), b.cuda(), a)
    total += 1
    if not np.array_equal(np.asarray(al), golden['mel/alignment']):
        assert _native_path_cost_ok('NaiveDTW', a, b, np.asarray(al), golden['mel/alignment'])
        fallbacks.append(('mel',))
    print(f'drop-ins: {total} cases, {len(fallbacks)} decided by a near tie (path cost checked instead): {fallbacks}')
    assert len(fallbacks) <= total // 4


def test_ninterpo_index_map_is_the_reference(golden):
    for name, (Sn, Tn) in {**{k: v[1:] for k, v in SADTW_CASES.items()}, **INTERPO_CASES}.items():
        if Sn < 2 or Tn < 2:
            continue
        src = torch.linspace(100, 300, Sn).cuda()
        mel2ph = torch.arange(Sn).cuda()
        mel = torch.randn(Sn, 80).cuda()
        out, m2p, amel = NI.NInterpo(src, torch.zeros(Tn).cuda(), src, mel2ph, amateur_mel=mel)
        idx = golden[f'ninterpo/{name}/index']
        assert m2p.dtype == torch.int64 and tuple(m2p.shape) == (Tn, 1) and tuple(out.shape) == (Tn, 1)
        assert np.array_equal(m2p[:, 0].cpu().numpy(), idx), name
        assert torch.equal(out[:, 0], src[torch.from_numpy(idx).cuda()]) and torch.equal(amel, mel[torch.from_numpy(idx).cuda()])
        r = core.align_batch([src], [torch.zeros(Tn).cuda()], 'NInterpo')
        assert np.array_equal(r.alignment.cpu().numpy(), idx) and r.path_cost is None


def test_cal_localnorm_dist_and_dtw_align():
    src, tgt = S.make_f0_pair(21, 300, 330)
    d = LN.cal_localnorm_dist(torch.from_numpy(src), torch.from_numpy(tgt), 300, 330)
    assert tuple(d.shape) == (1, 300, 330) and d.dtype == torch.float64 and d.device.type == 'cpu'
    o = O.cdist_cost('LoNDTW', src, tgt)
    assert float((d[0] - o).abs().max()) <= 1e-9 * float(o.abs().max())
    ctx = LN.get_local_context(src[:40])
    assert len(ctx) == 40 and len(ctx[0]) == 64 and np.array_equal(np.asarray(ctx), O.local_context(src[:40]).numpy())
    B, L = 3, 200
    srcs = torch.zeros(B, L, dtype=torch.float64)
    tgts = torch.zeros(B, L, dtype=torch.float64)
    for k in range(B):
        a, b = S.make_f0_pair(40 + k, L, L)
        srcs[k], tgts[k] = torch.from_numpy(a), torch.from_numpy(b)
    inputs = torch.arange(B * L).view(B, L, 1)
    out = LN.DTW_align(srcs, tgts, inputs, torch.tensor([L] * B), torch.tensor([L] * B))
    for k in range(B):
        _, al = LN.LoNDTW(srcs[k], tgts[k], inputs[k])
        assert torch.equal(out[k], inputs[k][al])


@pytest.mark.parametrize('method', DTW_METHODS + ('NInterpo',))
def test_ragged_batch_equals_single_pairs_and_repeats(method):
    rs = np.random.RandomState(5)
    lens = [(int(rs.randint(2, 40)), int(rs.randint(2, 40))) for _ in range(12)] + [(1378, 1400), (700, 1500), (1500, 650)]
    pairs = [S.make_f0_pair(200 + p, s, t) for p, (s, t) in enumerate(lens)]
    for dt in (torch.float32, torch.float64):
        xs = [torch.from_numpy(a).to(dt).cuda() for a, _ in pairs]
        ys = [torch.from_numpy(b).to(dt).cuda() for _, b in pairs]
        r = core.align_batch(xs, ys, method)
        r2 = core.align_batch(xs, ys, method)
        assert torch.equal(r.alignment, r2.alignment)
        if method != 'NInterpo':
            assert torch.equal(r.path_cost, r2.path_cost) and r.path_cost.dtype == dt
        for p, al in enumerate(r.split()):
            one = core.align_batch([xs[p]], [ys[p]], method)
            assert np.array_equal(one.alignment.cpu().numpy(), al), (method, dt, p)
            if method != 'NInterpo':
                assert torch.equal(one.path_cost[0], r.path_cost[p])
    # NaiveDTW on a ragged batch of [S, 80] mels
    if method == 'NaiveDTW':
        ms = [S.make_mel_pair(1, s, [0], 77 + p)[1][0].cuda() for p, (s, _) in enumerate(lens[-5:])]
        mt = [S.make_mel_pair(1, t, [0], 99 + p)[1][0].cuda() for p, (_, t) in enumerate(lens[-5:])]
        r = core.align_batch(ms, mt, method)
        for p, al in enumerate(r.split()):
            assert np.array_equal(core.align_batch([ms[p]], [mt[p]], method).alignment.cpu().numpy(), al)


@pytest.mark.parametrize('method', core.METHODS)
def test_a2p_alignment_batch_feeds_mle_svb_vae(method):
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    from tests.test_oracle_golden import SVB_HP
    B, Ta, Tp = 2, 96, 120
    la, lp = [96, 88], [120, 108]
    af, pf = torch.zeros(B, Ta), torch.zeros(B, Tp)
    for b in range(B):
        a, p = S.make_f0_pair(90 + b, la[b], lp[b])
        af[b, :la[b]], pf[b, :lp[b]] = torch.from_numpy(a), torch.from_numpy(p)
    align = a2p_alignment_batch(af.cuda(), pf.cuda(), torch.tensor(la), torch.tensor(lp), method=method)
    assert align.dtype == torch.int64 and align.is_cuda and tuple(align.shape) == (B, Tp)
    for b in range(B):
        ref = core.align_batch([af[b, :la[b]]], [pf[b, :lp[b]]], method).alignment.cpu().numpy()
        assert np.array_equal(align[b, :lp[b]].cpu().numpy(), np.minimum(ref, la[b] - 1)), (method, b)
        assert (align[b, lp[b]:] == 0).all()
    al = core.align_pitch([af[b, :la[b]].numpy() for b in range(B)], [pf[b, :lp[b]].numpy() for b in range(B)], method=method)
    assert [len(x) for x in al] == lp
    batch = {k: v.cuda() for k, v in S.make_svb_batch(B, Ta, Tp, 1234).items()}
    batch['a2p_alignment'] = align
    m = MleSVBVAE(80, hp=SVB_HP)
    m.load_state_dict(S.make_svb_state_dict(1234), strict=True)
    with torch.no_grad():
        out = m.eval().cuda()(**batch, infer=False, concurrent_ways=['a2a', 'p2p', 'a2p'])
    assert tuple(out['a2p']['mel_out'].shape) == (B, Tp, 80) and torch.isfinite(out['a2p']['mel_out']).all()


def test_alignment_accuracy_equals_job(golden):
    als, ams, pms, want = [], [], [], []
    for name, (seed, Sn, Tn) in SADTW_CASES.items():
        m_src, m_tgt = S.make_mel2ph_pair(seed, Sn, Tn)
        for method in DTW_METHODS:
            for kind in KINDS[method]:
                key = f'{name}/{method}/{kind}'
                als.append(golden[f'{key}/alignment'])
                ams.append(torch.from_numpy(m_src).cuda())
                pms.append(m_tgt)
                want.append(float(golden[f'{key}/accuracy']))
    got = alignment_accuracy(als, ams, pms)
    assert got.dtype == np.float64 and np.array_equal(got, np.asarray(want))
    with pytest.raises(ValueError, match='outside'):
        alignment_accuracy([np.array([0, 5])], [np.array([1, 1])], [np.array([1, 1])])


def test_pitch_align_eval_end_to_end(tmp_path):
    import importlib.util
    from neuralsvb_b200.utils.indexed_datasets import IndexedDatasetBuilder
    spec = importlib.util.spec_from_file_location('pitch_align_eval', os.path.join(os.path.dirname(os.path.dirname(__file__)),
                                                                                    'tools', 'pitch_align_eval.py'))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    path = str(tmp_path / 'paired')
    b = IndexedDatasetBuilder(path)
    for k, (Sn, Tn) in enumerate([(300, 330), (410, 380), (250, 260)]):
        f0, pf0 = S.make_f0_pair(300 + k, Sn, Tn)
        m, pm = S.make_mel2ph_pair(300 + k, Sn, Tn)
        b.add_item({'item_name': f'item{k}', 'f0': f0, 'mel2ph': m, 'prof_f0': pf0, 'prof_mel2ph': pm})
    b.finalize()
    save = tmp_path / 'out'
    res = tool.main(['--data', path, '--batch', '2', '--save', str(save)])
    assert set(res) == set(core.METHODS)
    for method, acc in res.items():
        assert acc.shape == (3,) and ((acc >= 0) & (acc <= 1)).all()
        items = tool.load_items(path, dict(pitch_norm='log', use_uv=True, f0_mean=0.0, f0_std=1.0))
        for k, it in enumerate(items):
            al = np.load(save / f'a2p_alignments_by_{method}' / f'item{k}_alignment.npy')
            f0a = it['f0'] if method != 'NaiveDTW' else it['f0'][:, None]
            f0p = it['prof_f0'] if method != 'NaiveDTW' else it['prof_f0'][:, None]
            assert len(al) == len(it['prof_f0'])
            if method == 'NInterpo':
                assert np.array_equal(al, O.align(method, f0a, f0p)[0])
            assert acc[k] == O.alignment_accuracy(al, it['mel2ph'].numpy(), it['prof_mel2ph'].numpy())

"""ORACLE tooling (test infrastructure only; see oracle/__init__.py): writes tests/golden/dtw_baselines.npz from the UNMODIFIED
reference baseline pitch alignments (modules/voice_conversion/dtw/local_norm_dtw.py: LoNDTW, naive_dtw.py: NaiveDTW / ZMNaiveDTW /
NNaiveDTW, naive_interpo.py: NInterpo, over align.py) and utils/pitch_utils.py's f0 round trip.

    NEURALSVB_REFERENCE=/path/to/NeuralSVB python -m oracle.gen_golden_dtw_baselines

The stubs are gen_golden_sadtw.install_stubs().  Inputs are regenerated from seeds (synthetic.make_f0_pair, make_mel_pair,
make_mel2ph_pair), never stored.  Per case and input kind: the alignment and job()'s accuracy; for one small case per method the
[T, S] cost and time_warp's DTW matrix; NInterpo's index map up to 7001 frames; denorm_f0(norm_interp_f0(f0)) for two pitch norms.
The script fails when oracle/dtw_baselines.py does not reproduce a reference alignment or cost.
"""
import os
import sys

import numpy as np
import torch

from neuralsvb_b200.utils import synthetic as S
from oracle import dtw_baselines as O
from oracle import ref_harness as R
from oracle.gen_golden import OUT
from oracle.gen_golden_sadtw import SADTW_CASES, install_stubs

DTW_METHODS = ('LoNDTW', 'NaiveDTW', 'ZMNaiveDTW', 'NNaiveDTW')
KINDS = {'LoNDTW': ('np64', 'np32', 'torch32', 'torch64'), 'NaiveDTW': ('torch32', 'torch64'),
         'ZMNaiveDTW': ('torch32', 'torch64'), 'NNaiveDTW': ('torch32', 'torch64')}
MATRIX_CASE = 's17_t21'          # costs and DTW matrices stored for every method and kind
MATRIX_CASE_MM = 's60_t48'       # and for one case in cdist's matrix-product form (more than 25 rows)
MEL_CASE = (31, 300, 340)        # NaiveDTW on [S, 80] mels: seed, S, T
INTERPO_CASES = {'s5000_t4999': (5000, 4999), 's4999_t5000': (4999, 5000), 's4321_t5000': (4321, 5000), 's3000_t7001': (3000, 7001),
                 's1400_t2800': (1400, 2800)}
ROUND_TRIPS = {'log': dict(pitch_norm='log', use_uv=True), 'standard': dict(pitch_norm='standard', use_uv=True, f0_mean=250.0,
                                                                              f0_std=90.0)}


def make_input(kind, f, method):
    if kind == 'np64':
        return f.astype(np.float64)
    if kind == 'np32':
        return f.astype(np.float32)
    t = torch.from_numpy(f.astype(np.float64 if kind == 'torch64' else np.float32))
    return t[:, None] if method == 'NaiveDTW' and t.dim() == 1 else t


def mel_pair():
    seed, Sn, Tn = MEL_CASE
    a = S.make_mel_pair(1, Sn, [0], seed)[1][0]
    b = S.make_mel_pair(1, Tn, [0], seed + 1)[1][0]
    return a, b


def gen():
    install_stubs()
    from modules.voice_conversion.dtw import align as ref_align
    from modules.voice_conversion.dtw import local_norm_dtw as ref_lo
    from modules.voice_conversion.dtw import naive_dtw as ref_naive
    from modules.voice_conversion.dtw import naive_interpo as ref_interp
    from utils import pitch_utils as ref_pu
    fns = {'LoNDTW': ref_lo.LoNDTW, 'NaiveDTW': ref_naive.NaiveDTW, 'ZMNaiveDTW': ref_naive.ZMNaiveDTW,
           'NNaiveDTW': ref_naive.NNaiveDTW}
    out = {}
    for name, (seed, Sn, Tn) in SADTW_CASES.items():
        src, tgt = S.make_f0_pair(seed, Sn, Tn)
        m_src, m_tgt = S.make_mel2ph_pair(seed, Sn, Tn)
        out[f'{name}/params'] = np.array([seed, Sn, Tn], np.int64)
        out[f'{name}/mel2ph_src'], out[f'{name}/mel2ph_tgt'] = m_src, m_tgt
        for method in DTW_METHODS:
            for kind in KINDS[method]:
                a, b = make_input(kind, src, method), make_input(kind, tgt, method)
                key = f'{name}/{method}/{kind}'
                _, alignment = fns[method](a, b, a)
                alignment = np.asarray(alignment, np.int64)
                out[f'{key}/alignment'] = alignment
                mine, _ = O.align(method, a, b)
                assert np.array_equal(mine, alignment), f'{key}: the oracle alignment differs from the reference'
                acc = (torch.from_numpy(m_tgt) == torch.from_numpy(m_src)[alignment]).sum().cpu().numpy() / (
                    torch.from_numpy(m_tgt) != 0).sum().cpu().numpy()
                out[f'{key}/accuracy'] = np.float64(acc)
                if name in (MATRIX_CASE, MATRIX_CASE_MM):
                    if method == 'LoNDTW':
                        ref_cost = ref_lo.cal_localnorm_dist(a, b, Sn, Tn).squeeze(0).T.contiguous().numpy()
                    elif method == 'NaiveDTW':
                        ref_cost = torch.cdist(a.unsqueeze(0), b.unsqueeze(0)).squeeze(0).T.contiguous().numpy()
                    else:
                        ref_cost = None
                    mc = O.cost(method, a, b)
                    if ref_cost is not None:
                        assert np.array_equal(mc, ref_cost), f'{key}: the oracle cost differs from the reference'
                    out[f'{key}/cost'] = mc
                    out[f'{key}/dtw'] = ref_align.time_warp(mc)
                print(key, 'ok', flush=True)
    a, b = mel_pair()
    _, alignment = ref_naive.NaiveDTW(a, b, a)
    alignment = np.asarray(alignment, np.int64)
    assert np.array_equal(O.align('NaiveDTW', a, b)[0], alignment), 'mel: the oracle alignment differs from the reference'
    out['mel/alignment'], out['mel/params'] = alignment, np.array(MEL_CASE, np.int64)
    print('mel ok', flush=True)
    for name, (Sn, Tn) in {**{k: v[1:] for k, v in SADTW_CASES.items()}, **INTERPO_CASES}.items():
        src = torch.from_numpy(S.make_f0_pair(7, Sn, 2)[0].astype(np.float32))
        tgt = torch.zeros(Tn)
        mel2ph = torch.arange(Sn, dtype=torch.int64)
        _, idx, _ = ref_interp.NInterpo(src, tgt, src, mel2ph)
        idx = idx[:, 0].numpy().astype(np.int64)
        assert np.array_equal(O.nearest_index(Sn, Tn), idx), f'NInterpo {name}: the oracle index map differs from the reference'
        out[f'ninterpo/{name}/index'] = idx
        out[f'ninterpo/{name}/params'] = np.array([Sn, Tn], np.int64)
    print('ninterpo ok', flush=True)
    for norm, hp in ROUND_TRIPS.items():
        for name in ('s60_t48', 's8s'):
            seed, Sn, Tn = SADTW_CASES[name]
            f0 = S.make_f0_pair(seed, Sn, Tn)[0]
            mel2ph = S.make_mel2ph_pair(seed, Sn, Tn)[0]
            f, uv = ref_pu.norm_interp_f0(f0, hp)
            f, uv = torch.FloatTensor(f), torch.FloatTensor(uv)
            out[f'roundtrip/{norm}/{name}'] = ref_pu.denorm_f0(f, uv, hp, pitch_padding=torch.from_numpy(mel2ph) == 0).numpy()
    np.savez_compressed(os.path.join(OUT, 'dtw_baselines.npz'), **out)
    print('dtw_baselines.npz', os.path.getsize(os.path.join(OUT, 'dtw_baselines.npz')), 'bytes')


def main():
    if not R.available():
        sys.exit('gen_golden_dtw_baselines needs NEURALSVB_REFERENCE = a checkout of the reference NeuralSVB')
    os.makedirs(OUT, exist_ok=True)
    gen()


if __name__ == '__main__':
    main()

"""-m gpu: the autocorrelation pitch tracker (csrc/pitch_ac.cu) against the float64 oracle (oracle/pitch_ac.py), and the paired
binarizer end to end.

  * ragged batches of 2-12 s clips, with a clip exactly one window plus one hop long, digital silence, noise and f0 near the floor and
    the ceiling: r(tau) within 2e-5, candidates within 1e-5 relative (frequency) and 2e-5 (strength), path f0 equal on every frame
    where the oracle's best path is more than 1e-4 ahead of the best path through another candidate;
  * every clip bit-identical alone and in the batch; get_pitch equal to get_pitch_batch;
  * write_svb_raw -> the binarize CLI -> the dataset on disk (keys, mel / f0 / alignment against the single-clip calls, the stats
    files, the skipped items, the f0 accuracy against the ground truth) -> tasks/run.py trains, resumes and infers on it."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from neuralsvb_b200.data_gen.tts import data_gen_utils as DG
from neuralsvb_b200.utils import synthetic as S
from oracle import pitch_ac as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR, HOP = 22050, 128
FPS = SR / HOP
HP = {'audio_sample_rate': SR, 'hop_size': HOP}


def tone(f, seconds, seed):
    rs = np.random.RandomState(seed)
    t = np.arange(int(seconds * SR)) / SR
    f = f * (1 + 0.01 * np.sin(2 * np.pi * 5 * t))
    ph = 2 * np.pi * np.cumsum(f) / SR
    return (0.4 * np.sin(ph) + 0.15 * np.sin(2 * ph) + 0.002 * rs.standard_normal(len(t))).astype(np.float32)


def clips():
    out = []
    for i, sec in enumerate((2.0, 5.3, 12.0, 3.1)):
        fa, _ = S.make_f0_pair(i, int(sec * FPS), int(sec * FPS), FPS)
        out.append(S.make_sung_take(fa * 2 ** ((3 * i - 4) / 12), i, SR, HOP)[0])
    out.append(tone(220.0, 1.0, 5)[:827 + HOP])                                               # one window plus one hop
    out.append(np.zeros(int(2.5 * SR), np.float32))                                           # digital silence
    out.append((0.05 * np.random.RandomState(9).standard_normal(int(2.2 * SR))).astype(np.float32))
    out.append(tone(84.0, 3.0, 11))                                                           # near the floor
    out.append(tone(720.0, 2.4, 12))                                                          # near the ceiling
    return out


@pytest.fixture(scope='module')
def batch():
    torch.cuda.set_device(0)
    ws = clips()
    lens = np.array([len(w) for w in ws])
    n_mel = lens // HOP + 1
    cat = torch.from_numpy(np.concatenate(ws)).cuda()
    tr = DG.pitch_ac_device(cat, lens, n_mel, HP, want_cand=True, want_r=True)
    torch.cuda.synchronize()
    return ws, lens, n_mel, tr


def split(tr, lens, n_mel):
    fo = np.concatenate([[0], np.cumsum(tr.frames)])
    oo = np.concatenate([[0], np.cumsum(n_mel)])
    r, cand, cnt, f0 = tr.r.cpu().numpy(), tr.cand.cpu().numpy(), tr.count.cpu().numpy(), tr.f0.cpu().numpy()
    return [(r[fo[c]:fo[c + 1]], cand[fo[c]:fo[c + 1]], cnt[fo[c]:fo[c + 1]], f0[oo[c]:oo[c + 1]]) for c in range(len(lens))]


def test_autocorrelation_and_candidates_match_the_oracle(batch):
    ws, lens, n_mel, tr = batch
    compared = total = 0
    for c, (r, cand, cnt, _) in enumerate(split(tr, lens, n_mel)):
        ro, lp, ra0, gp = P.normalised_autocorr(ws[c], SR, HOP / SR)
        assert r.shape == ro.shape
        live = ra0 > 0
        assert np.abs(r[live] - ro[live]).max(initial=0) < 2e-5, (c, np.abs(r[live] - ro[live]).max())
        fo, so, co = P.candidates_from_r(ro, lp, ra0, gp, SR)
        for j in range(len(r)):
            total += 1
            # frames whose candidate list hangs on a comparison closer than the r tolerance are not compared
            d = np.abs(np.diff(ro[j]))
            s_all, lag, h = P.peaks(ro[j], SR, P.DEFAULTS)
            near = (d.min() < 4e-5 or (np.abs(h - 0.3) < 1e-4).any() or (np.abs(lag - SR / 750) < 1e-3).any()
                    or (np.abs(lag - SR / 80) < 1e-3).any() or (len(s_all) > 14 and np.sort(s_all)[-14] - np.sort(s_all)[-15] < 1e-4))
            if near and cnt[j] != co[j]:
                continue
            assert cnt[j] == co[j], (c, j, cnt[j], co[j])
            k = cnt[j]
            if near and not np.allclose(cand[j, 1:k, 0], fo[j, 1:k], rtol=1e-5, atol=0):
                continue
            compared += 1
            assert np.allclose(cand[j, :k, 0], fo[j, :k], rtol=1e-5, atol=0), (c, j, cand[j, :k, 0], fo[j, :k])
            assert np.abs(cand[j, :k, 1] - so[j, :k]).max() < 2e-5, (c, j)
    assert compared > 0.97 * total, (compared, total)


def test_path_matches_the_oracle(batch):
    ws, lens, n_mel, tr = batch
    differ = 0
    for c, (_, _, _, f0) in enumerate(split(tr, lens, n_mel)):
        fo, marg = P.track(ws[c], SR, HOP, margins=True)
        placed = P.place(fo, n_mel[c], HOP)
        pm = P.place(marg, n_mel[c], HOP)
        pm[:8] = np.inf
        same = ((placed > 0) == (f0 > 0)) & (np.abs(f0 - placed) <= 1e-5 * placed)
        bad = ~same
        differ += int(bad.sum())
        assert (pm[bad] < 1e-4).all(), (c, np.nonzero(bad)[0][:10], pm[bad][:10])
    assert differ < 10, differ
    sil = split(tr, lens, n_mel)[5][3]
    noise = split(tr, lens, n_mel)[6][3]
    assert (sil == 0).all() and (noise == 0).all()


def test_each_clip_is_bit_identical_alone_and_in_the_batch(batch):
    ws, lens, n_mel, tr = batch
    parts = split(tr, lens, n_mel)
    for c, w in enumerate(ws):
        one = DG.pitch_ac_device(torch.from_numpy(w).cuda(), lens[c:c + 1], n_mel[c:c + 1], HP, want_cand=True, want_r=True)
        r, cand, cnt, f0 = parts[c]
        assert np.array_equal(one.r.cpu().numpy(), r) and np.array_equal(one.cand.cpu().numpy(), cand)
        assert np.array_equal(one.count.cpu().numpy(), cnt) and np.array_equal(one.f0.cpu().numpy(), f0)
    # the same batch reversed
    rev = ws[::-1]
    tr2 = DG.pitch_ac_device(torch.from_numpy(np.concatenate(rev)).cuda(), lens[::-1], n_mel[::-1], HP)
    oo = np.concatenate([[0], np.cumsum(n_mel[::-1])])
    for i, c in enumerate(range(len(ws) - 1, -1, -1)):
        assert np.array_equal(tr2.f0.cpu().numpy()[oo[i]:oo[i + 1]], parts[c][3])


def test_get_pitch_equals_get_pitch_batch(batch):
    ws, lens, n_mel, tr = batch
    mels = [np.zeros((int(t), 80), np.float32) for t in n_mel]
    many = DG.get_pitch_batch(ws, mels, HP)
    for c in (0, 3, 5, 8):
        f0, pitch = DG.get_pitch(ws[c], mels[c], HP)
        assert np.array_equal(f0, many[c][0]) and np.array_equal(pitch, many[c][1])
        assert np.array_equal(f0, split(tr, lens, n_mel)[c][3].astype(np.float64))
    with pytest.raises(ValueError, match='clip 0'):
        DG.get_pitch(np.zeros(800, np.float32), np.zeros((7, 80)), HP)


# ------------------------------------------------------------------------------------------------- binarizer end to end
def _cli(module, args, cwd, timeout=1200):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, '-m', module] + args, cwd=cwd, env=env, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_binarize_cli_then_train_and_infer(tmp_path):
    from scipy.io import wavfile

    from neuralsvb_b200.modules.voice_conversion.dtw.core import align_pitch
    from neuralsvb_b200.tasks.singing.dataset_utils import MultiSpkEmbDataset
    from neuralsvb_b200.utils import hparams as H
    from neuralsvb_b200.utils.indexed_datasets import IndexedDataset
    from neuralsvb_b200.vocoders.hifigan import HifiGAN
    raw, binary = str(tmp_path / 'raw'), str(tmp_path / 'bin')
    truth = S.write_svb_raw(raw, binary)
    ov = f'processed_data_dir={raw},binary_data_dir={binary},spk_emb_data_dir={raw}/spk_emb'
    out = _cli('neuralsvb_b200.data_gen.tts.bin.binarize', ['--config', os.path.join(ROOT, 'egs', 'svb_binarize_synthetic.yaml'),
                                                            '--hparams', ov], tmp_path)
    assert '| Skip item (Empty f0). item_name: Male1#singing#Song_A_Amateur_1' in out
    with open(os.path.join(binary, 'bad_case.txt')) as f:
        assert f.read().startswith('Gap is too large: Female2#singing#Song_B_Amateur_1')
    hp = H.set_hparams(os.path.join(ROOT, 'egs', 'svb_binarize_synthetic.yaml'), '', ov, print_hparams=False, global_hparams=False)
    keys = {'item_name', 'mel', 'prof_mel', 'f0', 'prof_f0', 'pitch', 'prof_pitch', 'a2p_f0_alignment', 'multi_spk_emb'}
    expect = {'train': ['Female1#singing#Song_A_Amateur_0', 'Female1#singing#Song_A_Amateur_1', 'Female1#singing#Song_B_Amateur_0',
                        'Female1#singing#Song_B_Amateur_1', 'Female2#singing#Song_A_Amateur_0', 'Female2#singing#Song_A_Amateur_1',
                        'Female2#singing#Song_B_Amateur_0'],
              'test': ['Male1#singing#Song_A_Amateur_0', 'Male1#singing#Song_B_Amateur_0', 'Male1#singing#Song_B_Amateur_1']}
    pairs = []
    for prefix in ('train', 'valid', 'test'):
        ds = IndexedDataset(os.path.join(binary, prefix))
        items = [ds[i] for i in range(len(ds))]
        assert [it['item_name'] for it in items] == expect['train' if prefix == 'train' else 'test']
        f0s = []
        for it in items:
            assert set(it) == keys
            name = it['item_name']
            wav_fn = glob.glob(os.path.join(raw, 'data', '*', name + '.wav'))[0]
            prof_fn = wav_fn.replace('Amateur', 'Professional')
            for fn, mk, fk in ((wav_fn, 'mel', 'f0'), (prof_fn, 'prof_mel', 'prof_f0')):
                wav, mel = HifiGAN.wav2spec(fn, hp=hp)
                assert np.array_equal(it[mk], mel), name
                f0, pitch = DG.get_pitch(wav, mel, hp)
                assert np.array_equal(it[fk], f0) and np.array_equal(it[fk.replace('f0', 'pitch')], pitch), name
                tv = truth[os.path.splitext(os.path.basename(fn))[0]]
                # placed frame i >= 8 is analysis frame i - 8 centred on sample c0 + (i - 8) hop
                n, L, c0, _ = P.grid(len(wav), SR, HOP / SR)
                idx = np.arange(8, len(f0))
                centre = np.minimum(c0 + (idx - 8) * HOP, len(tv) - 1)
                t = np.zeros(len(f0))
                t[idx] = tv[centre]
                ok = np.zeros(len(f0), bool)
                ok[idx] = True
                v = t > 0
                for e in np.nonzero(np.diff(v.astype(int)))[0]:
                    ok[max(0, e - 3):e + 5] = False
                pairs.append((f0, t, ok))
            assert np.array_equal(it['a2p_f0_alignment'], align_pitch([it['f0']], [it['prof_f0']], 'EHSADTW')[0])
            f0s += [it['f0'], it['prof_f0']]
        lengths = np.load(os.path.join(binary, f'{prefix}_lengths.npy'))
        assert lengths.tolist() == [max(len(it['mel']), len(it['prof_mel'])) for it in items]
        f = np.concatenate(f0s)
        assert np.allclose(np.load(os.path.join(binary, f'{prefix}_f0s_mean_std.npy')), [f[f > 0].mean(), f[f > 0].std()])
    gross = voiced = verr = total = 0
    cents = []
    for est, t, ok in pairs:
        both = ok & (t > 0) & (est > 0)
        gross += int((np.abs(est[both] / t[both] - 1) > 0.2).sum())
        voiced += int((ok & (t > 0)).sum())
        verr += int((ok & ((t > 0) != (est > 0))).sum())
        total += int(ok.sum())
        cents += list(np.abs(1200 * np.log2(est[both] / t[both])))
    assert gross < 0.01 * voiced and np.median(cents) < 10 and verr < 0.05 * total, (gross, voiced, np.median(cents), verr, total)
    # the dataset reads it
    hp_train = H.set_hparams(os.path.join(ROOT, 'egs', 'svb_vae_train_synthetic.yaml'), '', f'binary_data_dir={binary}',
                             print_hparams=False, global_hparams=False)
    ds = MultiSpkEmbDataset('train', hp_train)
    assert len(ds) == 7 and ds[0]['multi_spk_emb'].shape == (5, 256)
    # tasks/run.py: train, resume, infer
    cfg = os.path.join(ROOT, 'egs', 'svb_vae_train_synthetic.yaml')
    tov = (f'binary_data_dir={binary},pretrain_asr_ckpt={binary}/asr,vocoder_ckpt={binary}/hifigan,max_updates=6,phase_2_steps=4,'
           'val_check_interval=3,valid_infer_interval=3,tb_log_interval=1')
    out = _cli('neuralsvb_b200.tasks.run', ['--config', cfg, '--exp_name', 'svb_raw', '--reset', '--hparams', tov], tmp_path)
    assert 'Training end' in out
    out = _cli('neuralsvb_b200.tasks.run', ['--config', cfg, '--exp_name', 'svb_raw', '--hparams', 'max_updates=8'], tmp_path)
    assert '| step 6:' in out and '| step 5:' not in out and 'Training end' in out
    _cli('neuralsvb_b200.tasks.run', ['--config', cfg, '--exp_name', 'svb_raw', '--infer'], tmp_path)
    wavs = sorted(glob.glob(str(tmp_path / 'checkpoints' / 'svb_raw' / 'generated_*_' / 'wavs' / 'a2p_wavout' / '*.wav')))
    assert len(wavs) == 3, wavs
    assert wavfile.read(wavs[0])[0] == SR

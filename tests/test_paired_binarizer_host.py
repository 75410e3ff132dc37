"""Host logic of the paired singing binarizer (data_gen/singing/binarize_para.py) with the three device calls replaced by fakes:
pairing, splits, the speaker map, the length-gap skip and bad_case.txt, the empty-f0 skip, the missing phone_set.json error, the
seeded embedding selection and the per-batch call pattern.  CPU only."""
import json
import os

import numpy as np
import pytest

from neuralsvb_b200.data_gen.singing import binarize_para as BP
from neuralsvb_b200.utils import hparams as H
from neuralsvb_b200.utils import synthetic as S
from neuralsvb_b200.utils.indexed_datasets import IndexedDataset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, 'egs', 'svb_binarize_synthetic.yaml')


@pytest.fixture
def hp():
    saved = dict(H.hparams)
    yield H.hparams
    H.hparams.clear()
    H.hparams.update(saved)


class FakeDevice:
    """wav2spec_batch: frames = 1 + n // hop, zero mels; get_pitch_batch: 200 Hz wherever the take is not silent;
    align_pitch: the linear map.  Counts the calls."""

    def __init__(self, hop):
        self.hop, self.calls = hop, {'wav2spec': 0, 'pitch': 0, 'align': 0}

    def wav2spec_batch(self, wavs):
        from scipy.io import wavfile
        self.calls['wav2spec'] += 1
        out = []
        for w in wavs:
            x = wavfile.read(w)[1].astype(np.float32) / 32768.0
            T = len(x) // self.hop + 1
            wo = np.zeros(T * self.hop, np.float32)
            wo[:len(x)] = x
            out.append((wo, np.zeros((T, 80), np.float32)))
        return out

    def get_pitch_batch(self, wavs, mels, hparams):
        self.calls['pitch'] += 1
        res = []
        for w, m in zip(wavs, mels):
            f0 = np.full(len(m), 200.0 if np.abs(w).max() > 0 else 0.0)
            f0[:8] = 0
            res.append((f0, np.ones(len(m), np.int64)))
        return res

    def align_pitch(self, srcs, tgts, method):
        self.calls['align'] += 1
        assert method == 'EHSADTW'
        return [np.round(np.arange(len(t)) * (len(s) - 1) / max(len(t) - 1, 1)).astype(np.int64) for s, t in zip(srcs, tgts)]


def setup(tmp_path, hp, monkeypatch, extra=''):
    raw, binary = str(tmp_path / 'raw'), str(tmp_path / 'bin')
    S.write_svb_raw(raw, seconds=(0.6, 0.9), gap_frames=240)
    os.makedirs(binary, exist_ok=True)
    with open(os.path.join(binary, 'phone_set.json'), 'w') as f:
        json.dump(['a'], f)
    H.set_hparams(CONFIG, '', f'processed_data_dir={raw},binary_data_dir={binary},spk_emb_data_dir={raw}/spk_emb' +
                  (',' + extra if extra else ''), print_hparams=False)
    fake = FakeDevice(hp['hop_size'])

    class Voc:
        wav2spec_batch = staticmethod(fake.wav2spec_batch)
    monkeypatch.setattr(BP, 'get_vocoder_cls', lambda hparams: Voc)
    monkeypatch.setattr(BP, 'get_pitch_batch', fake.get_pitch_batch)
    monkeypatch.setattr(BP, 'align_pitch', fake.align_pitch)
    return raw, binary, fake


def test_pairing_splits_and_outputs(tmp_path, hp, monkeypatch, capsys):
    raw, binary, fake = setup(tmp_path, hp, monkeypatch)
    b = BP.PopBuTFyENSpkEMBinarizer()
    b.process()
    out = capsys.readouterr().out
    # pairing: singing amateur takes with a professional take; no Song_C (unpaired), no #speech#, no Professional items
    names = sorted(b.item_names)
    assert all('#singing#' in n and 'Amateur' in n for n in names)
    assert not any('Song_C' in n for n in names)
    assert len(names) == 3 * 2 * 2
    assert b.test_item_names == [n for n in b.item_names if n.startswith('Male1#singing#')]
    assert set(b.train_item_names) | set(b.test_item_names) == set(b.item_names)
    with open(os.path.join(binary, 'spk_map.json')) as f:
        assert json.load(f) == {'Female1#': 0, 'Female2#': 1, 'Male1#': 2}
    # the gap pair is skipped and logged, the silent take is skipped as Empty f0
    with open(os.path.join(binary, 'bad_case.txt')) as f:
        bad = f.read()
    assert 'Gap is too large: Female2#singing#Song_B_Amateur_1' in bad and bad.count('\n') == 1
    assert '| Skip item (Empty f0). item_name: Male1#singing#Song_A_Amateur_1' in out
    # one group per split: three device calls each
    assert fake.calls == {'wav2spec': 3, 'pitch': 3, 'align': 3}
    for prefix, expect in (('train', [n for n in b.train_item_names if n != 'Female2#singing#Song_B_Amateur_1']),
                           ('test', [n for n in b.test_item_names if n != 'Male1#singing#Song_A_Amateur_1'])):
        ds = IndexedDataset(os.path.join(binary, prefix))
        items = [ds[i] for i in range(len(ds))]
        assert [it['item_name'] for it in items] == expect                      # metadata order
        lengths = np.load(os.path.join(binary, f'{prefix}_lengths.npy'))
        assert lengths.tolist() == [max(len(it['mel']), len(it['prof_mel'])) for it in items]
        f = np.concatenate([np.concatenate([it['f0'], it['prof_f0']]) for it in items])
        ms = np.load(os.path.join(binary, f'{prefix}_f0s_mean_std.npy'))
        assert np.allclose(ms, [f[f != 0].mean(), f[f != 0].std()])
        for it in items:
            assert set(it) == {'item_name', 'mel', 'prof_mel', 'f0', 'prof_f0', 'pitch', 'prof_pitch', 'a2p_f0_alignment', 'multi_spk_emb'}
            assert it['multi_spk_emb'].shape == (5, 256)
            own = np.load(os.path.join(raw, 'spk_emb', it['item_name'] + '.npy'))
            assert np.array_equal(it['multi_spk_emb'][0], own)
            assert len(it['a2p_f0_alignment']) == len(it['prof_mel'])


def test_small_groups_cost_three_calls_each(tmp_path, hp, monkeypatch):
    raw, binary, fake = setup(tmp_path, hp, monkeypatch, 'binarize_batch_seconds=2.0')
    BP.PopBuTFyENSpkEMBinarizer().process()
    n = fake.calls['wav2spec']
    assert n > 3 and fake.calls['pitch'] <= n and fake.calls['align'] <= n


def test_missing_phone_set_is_named(tmp_path, hp, monkeypatch):
    raw, binary, fake = setup(tmp_path, hp, monkeypatch)
    os.remove(os.path.join(binary, 'phone_set.json'))
    with pytest.raises(FileNotFoundError, match='phone_set.json'):
        BP.PopBuTFyENSpkEMBinarizer().process()
    assert fake.calls['wav2spec'] == 0


def test_mp3_only_input_names_the_conversion(tmp_path, hp, monkeypatch):
    raw, binary, fake = setup(tmp_path, hp, monkeypatch)
    d = tmp_path / 'mp3' / 'data' / 'Female1#singing#X'
    d.mkdir(parents=True)
    (d / 'Female1#singing#X_Amateur_0.mp3').write_bytes(b'')
    hp['processed_data_dir'] = str(tmp_path / 'mp3')
    with pytest.raises(ValueError, match='ffmpeg'):
        BP.PopBuTFyENSpkEMBinarizer().process()


def test_embedding_selection_is_seeded_by_item_name():
    names = [f'F#singing#Song_X_Amateur_{i}' for i in range(7)] + ['F#singing#Song_Y_Amateur_0', 'G#singing#Song_X_Amateur_0']
    a = BP.select_spk_emb_items(names[2], names, 4)
    assert a == BP.select_spk_emb_items(names[2], list(names), 4)               # reproducible
    assert all(n.startswith('F#singing#Song_X_Amateur_') for n in a) and len(set(a)) == 4
    # fewer pieces than spk_emb_num: the last one repeats
    two = ['F#singing#Song_Z_Amateur_0', 'F#singing#Song_Z_Amateur_1']
    sel = BP.select_spk_emb_items(two[0], two, 4)
    assert sorted(set(sel)) == two and sel[2] == sel[1] == sel[3]
    assert BP.song_pieces('F#singing#Song_X_Amateur_1', names) == names[:7]

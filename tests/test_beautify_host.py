"""Host logic of the beautifier (neuralsvb_b200/inference/beautify.py) with its device stages replaced by fakes: CLI parsing, the
input checks, the f0-statistics error, checkpoint discovery, the dataset's crop rule, and that a bad pair raises with its index
before any model or vocoder call.  CPU only."""
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200.inference import beautify as BF
from neuralsvb_b200.tasks.singing.dataset_utils import MultiSpkEmbDataset
from neuralsvb_b200.utils import hparams as H
from neuralsvb_b200.utils import synthetic as S

SR, HOP = 22050, 128


@pytest.fixture
def hp():
    saved = dict(H.hparams)
    H.hparams.clear()
    H.hparams.update({'audio_sample_rate': SR, 'hop_size': HOP, 'max_frames': 5000, 'frames_multiple': 4, 'pitch_norm': 'standard',
                      'use_uv': True, 'f0_mean': 300.0, 'f0_std': 80.0, 'latent_size': 128, 'disable_map': False,
                      'vocoder_denoise_c': 0.0})
    yield H.hparams
    H.hparams.clear()
    H.hparams.update(saved)


class FakeBeautifier(BF.SVBBeautifier):
    """The host code of SVBBeautifier; front end: frames = 1 + n // hop; pitch: 200 Hz wherever the take is not silent; alignment:
    the linear map; model and vocoder: zeros.  Records the device stages it reaches."""

    def __init__(self, hp):
        self.hp, self.device, self.timing, self.stage_ms, self.calls = hp, torch.device('cpu'), False, None, []
        self.vocoder = type('V', (), {})()
        self.vocoder.model = type('M', (), {'seed': 0})()

    def _front_end(self, dec, rates, lens, st):
        self.calls.append('front_end')
        self.dec = dec
        return None, None

    def _pitch(self, wav, frames):
        self.calls.append('pitch')
        return None, [np.full(int(T), 200.0 if np.abs(w).max() > 0 else 0.0) for (w, _), T in zip(self.dec, frames)]

    def _align(self, f0_dev, frames):
        self.calls.append('align')
        B = len(frames) // 2
        return [np.round(np.arange(frames[B + i]) * (frames[i] - 1) / (frames[B + i] - 1)).astype(np.int64) for i in range(B)]

    def _acoustic(self, sample, mel, frames, Ta, Tp, eps):
        self.calls.append('model')
        self.sample, self.eps = sample, eps
        return torch.zeros(len(Ta), max(Tp), 80)

    def _vocode(self, mel_out, f0, Tp, seed):
        self.calls.append('vocoder')
        self.seed = seed
        return torch.zeros(sum(Tp) * HOP)


def take(frames, seed=0, silent=False):
    w = S.make_clip((frames - 1) * HOP, SR, seed)
    return np.zeros_like(w) if silent else w


EMB = np.zeros(256, np.float32)


def test_cli_parses_one_value_per_pair_and_refuses_mismatched_counts(capsys):
    a = BF.parse_args(['--config', 'c.yaml', '--exp_name', 'x', '--hparams', 'a=1', '--amateur', 'a0.wav', 'a1.wav', '--prof', 'p0.wav',
                       'p1.wav', '--spk_emb', 'e0.npy', 'e1.npy', '--out', 'o0.wav', 'o1.wav'])
    assert (a.config, a.exp_name, a.hparams) == ('c.yaml', 'x', 'a=1')
    assert a.amateur == ['a0.wav', 'a1.wav'] and a.prof == ['p0.wav', 'p1.wav'] and a.out == ['o0.wav', 'o1.wav']
    with pytest.raises(SystemExit):
        BF.parse_args(['--exp_name', 'x', '--amateur', 'a0.wav', 'a1.wav', '--prof', 'p0.wav', '--spk_emb', 'e.npy', '--out', 'o.wav'])
    assert 'one value per pair' in capsys.readouterr().err


def test_mismatched_lists_and_bad_embeddings_raise_before_any_device_stage(hp):
    b = FakeBeautifier(hp)
    with pytest.raises(ValueError, match='one of each per pair'):
        b._run([take(200)], [take(200), take(210)], [EMB], None, None)
    for bad in (np.zeros(255), np.zeros((1, 256)), np.full(256, np.nan), np.array(['x'] * 256)):
        with pytest.raises(ValueError, match='pair 1: the speaker embedding'):
            b._run([take(200), take(200)], [take(200), take(200)], [EMB, bad], None, None)
    assert b.calls == []


def test_missing_f0_statistics_file_is_named(tmp_path, hp):
    hp['binary_data_dir'] = str(tmp_path)
    with pytest.raises(FileNotFoundError, match='train_f0s_mean_std.npy'):
        BF.SVBBeautifier(str(tmp_path), hp=hp)
    np.save(tmp_path / 'train_f0s_mean_std.npy', [250.0, 60.0])
    BF.load_f0_stats(hp)
    assert (hp['f0_mean'], hp['f0_std']) == (250.0, 60.0)


def test_newest_checkpoint_is_the_largest_step(tmp_path):
    with pytest.raises(FileNotFoundError, match='model_ckpt_steps'):
        BF.newest_checkpoint(str(tmp_path))
    for step in (9, 120, 30):
        (tmp_path / f'model_ckpt_steps_{step}.ckpt').write_bytes(b'')
    (tmp_path / 'model_ckpt_steps_x.ckpt').write_bytes(b'')
    assert BF.newest_checkpoint(str(tmp_path)) == os.path.join(str(tmp_path), 'model_ckpt_steps_120.ckpt')


def test_conditioning_is_the_datasets_crop_and_collate_rule(tmp_path, hp):
    """condition() on the binarized items equals MultiSpkEmbDataset's collated batch, with max_frames and frames_multiple biting."""
    S.write_svb_binary(str(tmp_path), n_items=4, seed=7, n_valid=1, n_test=1, frames=(60, 256))
    dhp = dict(hp, binary_data_dir=str(tmp_path), infer=False, num_test_samples=0, min_frames=0, max_frames=150, frames_multiple=8,
               test_ids=[], sort_by_len=False)
    ds = MultiSpkEmbDataset('train', dhp)
    items = [ds._get_item(i) for i in range(len(ds))]
    ref = ds.collater([ds[i] for i in range(len(ds))])
    frames = [len(it['mel']) for it in items] + [len(it['prof_mel']) for it in items]
    f0s = [it['f0'] for it in items] + [it['prof_f0'] for it in items]
    pitches = [it['pitch'] for it in items] + [it['prof_pitch'] for it in items]
    spk = [torch.FloatTensor(it['multi_spk_emb'][0]) for it in items]
    got, Ta, Tp = BF.condition(frames, f0s, pitches, [it['a2p_f0_alignment'] for it in items], spk, dhp)
    assert max(frames) > 150 and all(t <= 150 and t % 8 == 0 for t in Ta + Tp)
    for k in ('pitch', 'f0', 'uv', 'prof_pitch', 'prof_f0', 'prof_uv', 'a2p_f0_alignment'):
        assert got[k].dtype == ref[k].dtype and torch.equal(got[k], ref[k]), k
    assert torch.equal(got['spk'], ref['multi_spk_emb'][:, 0, :])
    assert max(Ta) == ref['mels'].shape[1] and max(Tp) == ref['prof_mels'].shape[1]


@pytest.mark.parametrize('case', ['short_amateur', 'short_prof', 'long_prof', 'silent_amateur', 'silent_prof'])
def test_a_bad_pair_raises_with_its_index_before_the_model(hp, case):
    b = FakeBeautifier(hp)
    ama, prof = [take(300, 1), take(260, 2), take(280, 3)], [take(310, 4), take(250, 5), take(290, 6)]
    bad = {'short_amateur': ('amateur', take(58)), 'short_prof': ('prof', take(59)), 'long_prof': ('prof', take(5001)),
           'silent_amateur': ('amateur', take(300, silent=True)), 'silent_prof': ('prof', take(300, silent=True))}[case]
    (ama if bad[0] == 'amateur' else prof)[1] = bad[1]
    msg = {'short': 'too short', 'long': 'max_frames', 'silent': 'no voiced f0'}[case.split('_')[0]]
    with pytest.raises(ValueError, match=f'pair 1: the {"amateur" if bad[0] == "amateur" else "professional"} take .*{msg}'):
        b._run(ama, prof, [EMB] * 3, 5, None)
    assert 'model' not in b.calls and 'vocoder' not in b.calls
    assert b.calls == ([] if case.split('_')[0] in ('short', 'long') else ['front_end', 'pitch'])


def test_a_good_batch_returns_the_cropped_professional_length_and_keys_the_draws_by_seed(hp):
    b = FakeBeautifier(hp)
    out = b._run([take(300, 1), take(64, 2)], [take(301, 3), take(70, 4)], [EMB, EMB], 11, None)
    assert [len(o) for o in out] == [300 * HOP, 68 * HOP]           # 1 + n // hop frames, cropped to a multiple of 4
    assert b.seed == 11 and tuple(b.eps.shape) == (2, 128, 1)
    assert torch.equal(b.eps, torch.randn(2, 128, 1, generator=torch.Generator('cpu').manual_seed(11)))
    b._run([take(300, 1)], [take(300, 3)], [EMB], None, None)
    assert b.seed == 1                                                # the vocoder's next seed, as spec2wav
    assert b.calls[-5:] == ['front_end', 'pitch', 'align', 'model', 'vocoder']

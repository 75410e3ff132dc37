"""-m gpu: the beautifier (neuralsvb_b200/inference/beautify.py) against the existing route on a write_svb_raw set: the paired
binarizer's wav2spec_batch / get_pitch_batch / align_pitch, MultiSpkEmbDataset's take and collate rules, MleSVBVAE on the collated
batch and HifiGAN.spec2wav_batch.  Every quantity must match bit for bit; also the ragged batch, the error paths, the CLI and the
device front end."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

from neuralsvb_b200 import _native
from neuralsvb_b200.data_gen.tts.data_gen_utils import get_pitch_batch
from neuralsvb_b200.inference import beautify as BF
from neuralsvb_b200.modules.voice_conversion.dtw.core import align_pitch
from neuralsvb_b200.tasks.singing.dataset_utils import MultiSpkEmbDataset
from neuralsvb_b200.utils import audio, move_to_cuda
from neuralsvb_b200.utils import hparams as H
from neuralsvb_b200.utils import synthetic as S
from neuralsvb_b200.utils.pitch_utils import denorm_f0

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, 'egs', 'svb_vae_train_synthetic.yaml')
SILENT = 'Male1#singing#Song_A_Amateur_1'


@pytest.fixture(autouse=True)
def keep_hparams():
    saved = dict(H.hparams)
    yield
    H.hparams.clear()
    H.hparams.update(saved)


def make_experiment(root, **raw_kw):
    """A raw set, the vocoder / ASR checkpoints, f0 statistics and checkpoints/svb_bf/ holding config.yaml and a random MleSVBVAE."""
    raw, binary = os.path.join(root, 'raw'), os.path.join(root, 'binary')
    S.write_svb_raw(raw, binary, seed=1234, **raw_kw)
    np.save(os.path.join(binary, 'train_f0s_mean_std.npy'), [300.0, 80.0])
    with open(CONFIG) as f:
        cfg = yaml.safe_load(f)
    cfg.update(binary_data_dir=binary, vocoder_ckpt=os.path.join(binary, 'hifigan'), pretrain_asr_ckpt=os.path.join(binary, 'asr'))
    work = os.path.join(root, 'checkpoints', 'svb_bf')
    os.makedirs(work)
    with open(os.path.join(work, 'config.yaml'), 'w') as f:
        yaml.safe_dump(cfg, f)
    torch.save({'state_dict': {'model': S.make_svb_state_dict(1234)}, 'global_step': 5}, os.path.join(work, 'model_ckpt_steps_5.ckpt'))
    pairs = []
    for d in sorted(os.listdir(os.path.join(raw, 'data'))):
        for fn in sorted(os.listdir(os.path.join(raw, 'data', d))):
            name = fn[:-4]
            prof = os.path.join(raw, 'data', d, fn.replace('Amateur', 'Professional'))
            if '#singing#' in name and 'Amateur' in name and os.path.exists(prof):
                pairs.append((name, os.path.join(raw, 'data', d, fn), prof, os.path.join(raw, 'spk_emb', name + '.npy')))
    return work, pairs


class Spy:
    """Records what each device stage of a beautifier returns."""

    def __init__(self, b):
        self.seen = {}
        for name in ('_front_end', '_pitch', '_align', '_acoustic', '_vocode'):
            setattr(b, name, self._wrap(name, getattr(b, name)))

    def _wrap(self, name, fn):
        def call(*a, **kw):
            r = fn(*a, **kw)
            self.seen[name] = r
            return r
        return call


def existing_route(b, pairs, eps, seed):
    """The composition of section 2: the binarizer's three calls, the dataset's items and collater, the model, spec2wav_batch."""
    from neuralsvb_b200.vocoders.hifigan import HifiGAN
    hp, B = b.hp, len(pairs)
    specs = HifiGAN.wav2spec_batch([p[1] for p in pairs] + [p[2] for p in pairs])
    pitches = get_pitch_batch([s[0] for s in specs], [s[1] for s in specs], hp)
    aligns = align_pitch([pitches[i][0] for i in range(B)], [pitches[B + i][0] for i in range(B)], 'EHSADTW')
    items = [{'item_name': p[0], 'mel': specs[i][1], 'prof_mel': specs[B + i][1], 'f0': pitches[i][0], 'pitch': pitches[i][1],
              'prof_f0': pitches[B + i][0], 'prof_pitch': pitches[B + i][1], 'a2p_f0_alignment': aligns[i],
              'multi_spk_emb': np.load(p[3])[None]} for i, p in enumerate(pairs)]
    ds = MultiSpkEmbDataset.__new__(MultiSpkEmbDataset)
    ds.hparams, ds.sizes = hp, [max(len(it['mel']), len(it['prof_mel'])) for it in items]
    ds._get_item = lambda i: items[i]
    sample = move_to_cuda(ds.collater([ds[i] for i in range(B)]))
    spk = sample['multi_spk_emb'][:, 0, :]
    with torch.no_grad():
        out = b.model(amateur_mel=sample['mels'], prof_mel=sample['prof_mels'], amateur_pitch=sample['pitch'], prof_pitch=sample['prof_pitch'],
                      amateur_spk_id=spk, prof_spk_id=spk, a2p_alignment=sample['a2p_f0_alignment'], infer=False,
                      concurrent_ways=['a2a', 'p2p', 'a2p'], disable_map=hp['disable_map'], eps=eps.cuda())
    mel_out = out['a2p']['mel_out']
    f0 = denorm_f0(sample['prof_f0'], sample['prof_uv'], hp)
    Tp = [int((sample['prof_pitch'][b_] > 0).sum()) for b_ in range(B)]
    wavs = b.vocoder.spec2wav_batch([mel_out[i, :t].cpu().numpy() for i, t in enumerate(Tp)],
                                    [f0[i, :t].cpu().numpy() for i, t in enumerate(Tp)], seed=seed)
    return specs, pitches, aligns, mel_out, wavs


def check_equivalent(b, pairs, seed=77):
    B = len(pairs)
    eps = torch.randn(B, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(seed))
    spy = Spy(b)
    got = b.beautify_batch([p[1] for p in pairs], [p[2] for p in pairs], [p[3] for p in pairs], seed=seed, eps=eps)
    specs, pitches, aligns, mel_out, wavs = existing_route(b, pairs, eps, seed)
    mel, wav = (t.cpu().numpy() for t in spy.seen['_front_end'])
    f0s = spy.seen['_pitch'][1]
    o = ow = 0
    for k, (w_ref, m_ref) in enumerate(specs):
        assert np.array_equal(mel[o:o + len(m_ref)], m_ref), f'take {k}: mel'
        assert np.array_equal(wav[ow:ow + len(w_ref)], w_ref), f'take {k}: padded waveform'
        assert np.array_equal(f0s[k], pitches[k][0]) and f0s[k].dtype == pitches[k][0].dtype, f'take {k}: f0'
        o, ow = o + len(m_ref), ow + len(w_ref)
    for i in range(B):
        assert np.array_equal(spy.seen['_align'][i], aligns[i]), f'pair {i}: alignment'
    assert torch.equal(spy.seen['_acoustic'], mel_out), 'a2p mel_out'
    for i in range(B):
        assert got[i].dtype == np.float32 and np.array_equal(got[i], wavs[i]), f'pair {i}: waveform'
    return got, spy


@pytest.fixture(scope='module')
def exp22(tmp_path_factory):
    return make_experiment(str(tmp_path_factory.mktemp('bf22')))


def regular(pairs):
    return [p for p in pairs if p[0] != SILENT]


def test_equivalent_to_the_existing_route_at_22050_hz_int16(exp22):
    work, pairs = exp22
    b = BF.SVBBeautifier(work)
    got, _ = check_equivalent(b, regular(pairs)[:4])
    assert all(np.abs(g).max() > 0 for g in got)


def test_equivalent_to_the_existing_route_at_44100_hz_float32_stereo(tmp_path):
    work, pairs = make_experiment(str(tmp_path), file_sr=44100, channels=2, sample_format='float32')
    b = BF.SVBBeautifier(work)
    assert audio.wav_info(pairs[0][1])[0] == 44100
    check_equivalent(b, regular(pairs)[:4], seed=5)


def test_ragged_batch_stages_match_each_pair_alone(exp22):
    """One call over every regular pair: the stages before the model are per pair, bit for bit the pair run alone; the model runs
    on the collated batch (check_equivalent) and the waveforms equal spec2wav_batch's list form on the batch's mels.  The a2p mel of
    a pair in the batch and alone differ (the model sees the padding); the largest difference is printed."""
    work, pairs = exp22
    b = BF.SVBBeautifier(work)
    pairs = regular(pairs)
    assert len(pairs) >= 8 and len({audio.wav_info(p[2])[1] for p in pairs}) == len(pairs)
    got, spy = check_equivalent(b, pairs, seed=9)
    mel_b = spy.seen['_front_end'][0].cpu().numpy()
    f0_b, al_b, mo_b = spy.seen['_pitch'][1], spy.seen['_align'], spy.seen['_acoustic']
    B = len(pairs)
    eps = torch.randn(B, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(9))
    frames = [len(f) for f in f0_b]
    offs = np.concatenate([[0], np.cumsum(frames)])
    worst = 0.0
    for i, p in enumerate(pairs):
        alone = Spy(b)
        one = b.beautify_batch([p[1]], [p[2]], [p[3]], seed=9, eps=eps[i:i + 1])[0]
        mel1 = alone.seen['_front_end'][0].cpu().numpy()
        for k, src in ((i, 0), (B + i, 1)):                       # the alone run's takes: amateur, then professional
            start = 0 if src == 0 else frames[i]
            assert np.array_equal(mel_b[offs[k]:offs[k + 1]], mel1[start:start + frames[k]]), (i, k)
            assert np.array_equal(f0_b[k], alone.seen['_pitch'][1][src]), (i, k)
        assert np.array_equal(al_b[i], alone.seen['_align'][0]), i
        assert len(one) == len(got[i])
        Tp = len(one) // b.hp['hop_size']
        worst = max(worst, float((mo_b[i, :Tp] - alone.seen['_acoustic'][0, :Tp]).abs().max()))
    print(f'MEASURED ragged: largest |a2p mel in batch - alone| = {worst:.3e}')


def test_bad_pairs_raise_naming_the_pair_and_vocode_nothing(exp22):
    work, pairs = exp22
    b = BF.SVBBeautifier(work)
    spy = Spy(b)
    silent = [p for p in pairs if p[0] == SILENT][0]
    batch = regular(pairs)[:2] + [silent]
    with pytest.raises(ValueError, match='pair 2: the amateur take has no voiced f0'):
        b.beautify_batch([p[1] for p in batch], [p[2] for p in batch], [p[3] for p in batch], seed=1)
    assert '_acoustic' not in spy.seen and '_vocode' not in spy.seen
    short = S.make_clip(58 * 128, 22050, 3)                      # 59 frames
    good = regular(pairs)[0]
    with pytest.raises(ValueError, match='pair 1: the professional take is too short: 59 frames'):
        b.beautify_batch([good[1], good[1]], [good[2], short], [good[3], good[3]], seed=1)
    assert '_acoustic' not in spy.seen and '_vocode' not in spy.seen


def test_cli_writes_what_save_wav_writes_from_the_api(exp22, tmp_path):
    work, pairs = exp22
    pairs = regular(pairs)[:2]
    root = os.path.dirname(os.path.dirname(work))
    outs = [str(tmp_path / f'o{i}.wav') for i in range(2)]
    r = subprocess.run([sys.executable, '-m', 'neuralsvb_b200.inference.beautify', '--config', CONFIG, '--exp_name', 'svb_bf',
                        '--amateur'] + [p[1] for p in pairs] + ['--prof'] + [p[2] for p in pairs] + ['--spk_emb'] +
                       [p[3] for p in pairs] + ['--out'] + outs, cwd=root, env=dict(os.environ, PYTHONPATH=ROOT),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    b = BF.SVBBeautifier(work)                                    # a fresh vocoder: the same first seed as the CLI's
    got = b.beautify_batch([p[1] for p in pairs], [p[2] for p in pairs], [p[3] for p in pairs])
    for w, fn in zip(got, outs):
        ref = str(tmp_path / 'ref.wav')
        audio.save_wav(w, ref, b.hp['audio_sample_rate'], norm=b.hp['out_wav_norm'])
        assert open(fn, 'rb').read() == open(ref, 'rb').read(), fn


def test_device_front_end_matches_per_clip_calls_and_the_host_wrapper_on_a_ragged_batch():
    from neuralsvb_b200.vocoders.hifigan import HifiGAN, stft_config
    hp = {'fft_size': 512, 'hop_size': 128, 'win_size': 512, 'audio_num_mel_bins': 80, 'audio_sample_rate': 22050, 'fmin': 50,
          'fmax': 11025}
    lengths = [22050, 1, 130, 4000, 257, 12345, 128]
    clips = [S.make_clip(n, 22050, i) for i, n in enumerate(lengths)]
    cat = np.ascontiguousarray(np.concatenate(clips))
    mel_d, wav_d, frames = HifiGAN.wav2spec_device(torch.from_numpy(cat).cuda(), lengths, hp)
    lib = _native.lib()
    cfg = stft_config(hp, _native.PAD_CENTER_ZERO, _native.OUT_LOG10_MEL, 1e-10)
    lens = np.array(lengths, np.int64)
    assert frames.tolist() == [1 + n // 128 for n in lengths]
    offs = np.concatenate([[0], np.cumsum(frames)])
    for k, c in enumerate(clips):
        mel1, wav1, _ = HifiGAN.wav2spec_device(torch.from_numpy(c).cuda(), lengths[k:k + 1], hp)
        assert torch.equal(mel_d[offs[k]:offs[k + 1]], mel1) and torch.equal(wav_d[offs[k] * 128:offs[k + 1] * 128], wav1), k
    host = HifiGAN.wav2spec_batch(clips, hp)
    assert np.array_equal(np.concatenate([m for _, m in host]), mel_d.cpu().numpy())
    assert np.array_equal(np.concatenate([w for w, _ in host]), wav_d.cpu().numpy())
    pad = np.concatenate([np.concatenate([c, np.zeros(f * 128 - len(c), np.float32)]) for c, f in zip(clips, frames)])
    assert np.array_equal(wav_d.cpu().numpy(), pad)
    basis = np.ascontiguousarray(audio.build_mel_basis(hp))
    ws = lib.svb_wav2spec_workspace_bytes(ctypes.byref(cfg), lens.ctypes.data_as(ctypes.c_void_p), len(lens), None)
    assert ws > 0
    buf = torch.empty(int(ws), dtype=torch.uint8, device='cuda')
    x = torch.from_numpy(cat).cuda()
    assert lib.svb_wav2spec_batch(ctypes.byref(cfg), _native.ptr(x), lens.ctypes.data_as(ctypes.c_void_p), len(lens), None,
                                  _native.ptr(mel_d), None, None, ctypes.c_void_p(buf.data_ptr()), int(ws), None) == -1   # no filters
    assert lib.svb_wav2spec_batch(ctypes.byref(cfg), _native.ptr(x), lens.ctypes.data_as(ctypes.c_void_p), len(lens),
                                  _native.ptr(torch.from_numpy(basis).cuda()), _native.ptr(mel_d), None, None,
                                  ctypes.c_void_p(buf.data_ptr()), int(ws) - 1, None) == -1                        # short workspace

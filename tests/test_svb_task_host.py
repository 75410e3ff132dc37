"""CPU: the SVB task's paired-singing dataset against the reference's own MultiSpkEmbDataset (tests/golden/svb_dataset.npz,
oracle/gen_golden_svb_dataset.py), the task's phase / way / gating logic, its optimizer partition and schedules, and the
synthetic config against the reference's resolved vae_global_mle_eng hyper-parameters."""
import json
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200.tasks.singing import svb_vae_task as T
from neuralsvb_b200.tasks.singing.dataset_utils import BATCH_KEYS, MultiSpkEmbDataset, build_batches, build_dataloader
from neuralsvb_b200.utils import hparams as H
from neuralsvb_b200.utils.synthetic import write_svb_binary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, 'egs', 'svb_vae_train_synthetic.yaml')
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'svb_dataset.npz')


@pytest.fixture
def hp():
    saved = dict(H.hparams)
    yield H.hparams
    H.hparams.clear()
    H.hparams.update(saved)


@pytest.fixture(scope='module')
def fixture_data(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('svb_golden'))
    write_svb_binary(d, 12, 1234, n_valid=1, n_test=1)        # the dataset oracle/gen_golden_svb_dataset.py read
    return d


@pytest.fixture(scope='module')
def small_data(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('svb_small'))
    write_svb_binary(d, 4, 7, n_valid=1, n_test=1)
    return d


def _config(hp, data_dir, extra=''):
    H.set_hparams(CONFIG, '', f'binary_data_dir={data_dir},pretrain_asr_ckpt={data_dir}/asr' + (',' + extra if extra else ''),
                  print_hparams=False)
    return hp


# ---------------------------------------------------------------------------------------------------------- dataset
def test_dataset_batches_match_the_reference_dataset_bit_for_bit(hp, fixture_data):
    g = np.load(GOLDEN)
    _config(hp, fixture_data)
    np.random.seed(1234)
    ds = MultiSpkEmbDataset('train', hp, shuffle=True)
    assert (hp['f0_mean'], hp['f0_std']) == tuple(g['f0_mean_std'])
    batches = build_batches(ds, True, 600, 4)
    assert [len(b) for b in batches] == list(g['batches_w1_r0'])
    assert np.array_equal(np.concatenate(batches), g['indices_w1_r0'])
    for i, batch in enumerate(build_dataloader(ds, batches)):
        if i == 4:
            break
        assert set(batch) == set(BATCH_KEYS) | {'item_name', 'nsamples'}
        assert list(batch['item_name']) == list(g[f'b{i}_item_name']) and batch['nsamples'] == len(batch['item_name'])
        for k in BATCH_KEYS:
            ref = g[f'b{i}_{k}']
            assert batch[k].dtype == torch.from_numpy(ref).dtype and np.array_equal(batch[k].numpy(), ref), (i, k)


def test_rank_shards_match_the_reference_and_are_disjoint(hp, fixture_data):
    g = np.load(GOLDEN)
    _config(hp, fixture_data)
    ds = MultiSpkEmbDataset('train', hp, shuffle=True)
    shards = []
    for rank in range(2):
        np.random.seed(1234)
        b = build_batches(ds, True, 600, 4, rank=rank, world=2)
        assert [len(x) for x in b] == list(g[f'batches_w2_r{rank}'])
        assert np.array_equal(np.concatenate(b), g[f'indices_w2_r{rank}'])
        shards.append(set(np.concatenate(b).tolist()))
    assert not shards[0] & shards[1]


def test_endless_training_batches_repeat_reshuffled_epochs(hp, small_data):
    _config(hp, small_data)
    ds = MultiSpkEmbDataset('train', hp, shuffle=True)
    np.random.seed(0)
    one = build_batches(ds, True, 40000, 2)
    np.random.seed(0)
    many = build_batches(ds, True, 40000, 2, endless=True)
    assert len(many) == 1000 * len(one)
    assert sorted(map(tuple, many[:len(one)])) == sorted(map(tuple, one))


def test_alignment_is_clipped_to_the_cropped_amateur_take(hp, small_data):
    _config(hp, small_data, 'max_frames=64')
    s = MultiSpkEmbDataset('train', hp)[0]
    assert s['mel'].shape[0] == s['pitch'].shape[0] == 64 and s['prof_mel'].shape[0] == 64
    assert s['a2p_f0_alignment'].shape == (64,) and int(s['a2p_f0_alignment'].max()) <= 63


# ---------------------------------------------------------------------------------------------------------- task logic
def test_phase_and_ways_around_the_phase_boundaries(hp):
    hp.update(phase_1_steps=5, phase_2_steps=10, phase_1_concurrent_ways='p2p', phase_2_concurrent_ways='a2a,p2p',
              phase_3_concurrent_ways='a2p')
    got = {s: T.phase_of(s, hp) for s in (0, 4, 5, 6, 10, 11, 50)}
    assert got == {0: (1, ['p2p']), 4: (1, ['p2p']), 5: (1, ['p2p']), 6: (2, ['a2a', 'p2p']), 10: (2, ['a2a', 'p2p']),
                   11: (3, ['a2p']), 50: (3, ['a2p'])}
    assert [T.valid_ways(s, hp) for s in (5, 6, 10, 11)] == [['p2p'], ['a2a', 'p2p'], ['a2a', 'p2p'], ['a2a', 'p2p', 'a2p']]
    hp.update(phase_1_steps=-1)                 # vae_global_mle_eng: no phase 1
    assert T.phase_of(0, hp)[0] == 2 and T.valid_ways(0, hp) == ['a2a', 'p2p']


class _FakeTask(T.SVBVAEMleTask):
    """The step's control flow with the model and the discriminator replaced by recorders (no device work)."""

    def __init__(self):
        super().__init__()
        self.model = torch.nn.Module()
        self.model.z_mapping_function = torch.nn.Module()
        self.mel_disc, self.calls = object(), []

    def run_model(self, sample, concurrent_ways, infer=False, disable_map=False):
        self.calls.append(('run', tuple(concurrent_ways)))
        losses = {f'{w}_kl': torch.tensor(1.0) for w in concurrent_ways if w != 'a2p'}
        out = {w: {'mel_out': torch.zeros(1), 'mle': torch.tensor(2.0)} for w in concurrent_ways}
        return losses, out

    def _adv(self, mel, target_one):
        self.calls.append(('disc', target_one))
        return torch.tensor(3.0)


def _step(task, step, opt):
    task.global_step, task.calls = step, []
    ret = task._training_step({'mels': torch.zeros(2, 4, 80), 'prof_mels': torch.zeros(2, 4, 80)}, 0, opt)
    return None if ret is None else ret[1], task.calls


def test_disc_start_and_interval_gating(hp):
    _config(hp, '/nonexistent', 'disc_start_steps=3,disc_interval=2,phase_2_steps=100')
    task = _FakeTask()
    log, _ = _step(task, 3, 0)                               # disc_start needs global_step > disc_start_steps
    assert not any(k.endswith('_a') for k in log)
    assert _step(task, 3, 1)[0] is None
    log, calls = _step(task, 4, 0)
    assert {'a2a_a', 'p2p_a'} <= set(log) and calls.count(('disc', True)) == 2
    log, calls = _step(task, 4, 1)                           # 4 % disc_interval == 0
    assert set(log) == {'a2a_r', 'a2a_f', 'p2p_r', 'p2p_f', 'bs'} and calls == [('disc', True), ('disc', False)] * 2
    assert _step(task, 5, 1)[0] is None                      # 5 % 2 != 0
    assert _step(task, 5, 2)[0] is None                      # the map optimizer waits for phase 3
    hp['lambda_mel_adv'] = 0.0
    assert not any(k.endswith('_a') for k in _step(task, 4, 0)[0]) and _step(task, 4, 1)[0] is None


def test_phase_3_runs_the_map_step_only(hp):
    _config(hp, '/nonexistent', 'phase_2_steps=10')
    task = _FakeTask()
    assert _step(task, 11, 0)[0] is None and _step(task, 11, 1)[0] is None
    log, calls = _step(task, 11, 2)
    assert calls[0] == ('run', ('a2a', 'p2p', 'a2p')) and {'a2p_mle', 'a2p_a'} <= set(log)
    total, _ = task._training_step({'mels': torch.zeros(2, 4, 80)}, 0, 2)
    assert float(total) == pytest.approx(1.0 + 1.0 + 2.0 * hp['lambda_mle'] + 3.0 * hp['lambda_mel_adv'])


def test_non_finite_kl_is_detached(hp):
    _config(hp, '/nonexistent')
    task = _FakeTask()
    w = torch.tensor(1.0, requires_grad=True)
    task.run_model = lambda s, ways, **k: ({'a2a_kl': w * float('inf'), 'p2p_kl': w * 2}, {x: {'mel_out': None} for x in ways})
    task.global_step = 0
    _, log = task._training_step({'mels': torch.zeros(1, 4, 80)}, 0, 0)
    assert not log['a2a_kl'].requires_grad and log['p2p_kl'].requires_grad


def test_optimizer_partition_and_frozen_asr(hp, small_data):
    _config(hp, small_data)
    task = T.SVBVAEMleTask()
    task.build_model()
    opts = task.configure_optimizers()
    ids = [{id(p) for g in o.param_groups for p in g['params']} for o in opts]
    assert not (ids[0] & ids[1] or ids[0] & ids[2] or ids[1] & ids[2])
    names = {id(p): n for n, p in task.model.named_parameters()}
    assert all(not names[i].startswith(('vc_asr.', 'z_mapping_function.')) for i in ids[0])
    assert {names[i] for i in ids[0]} | {n for n in names.values() if n.startswith(('vc_asr.', 'z_mapping_function.'))} == set(names.values())
    assert ids[2] == {id(p) for p in task.model.z_mapping_function.parameters()}
    assert ids[1] == {id(p) for p in task.mel_disc.parameters()}
    asr = list(task.model.vc_asr.parameters())
    assert asr and all(not p.requires_grad for p in asr) and not any(id(p) in i for p in asr for i in ids)
    assert [o.defaults['lr'] for o in opts[1:]] == [hp['disc_lr'], hp['map_lr']]
    assert opts[1].defaults['eps'] == 1e-6 and opts[0].defaults['betas'] == (0.5, 0.999)
    assert len(task.model.state_dict()) == 259


def test_scheduler_stepping(hp, small_data):
    _config(hp, small_data, 'scheduler=rsqrt,lr=1.0,disc_start_steps=10')
    hp['discriminator_scheduler_params'] = {'gamma': 0.5, 'step_size': 4}
    hp['map_scheduler_params'] = {'gamma': 0.1, 'step_size': 3}
    task = T.SVBVAEMleTask()
    task.build_model()
    opts = task.configure_optimizers()
    rsqrt = lambda n: max(min(n / 2000, 1.0) * max(2000, n) ** -0.5 * 256 ** -0.5, 1e-7)
    assert opts[0].param_groups[0]['lr'] == rsqrt(0) == 1e-7
    for step in (1, 1000, 2000, 8000):
        task.global_step = step
        task.on_after_optimization(0, 0, opts[0], 0)
        assert opts[0].param_groups[0]['lr'] == pytest.approx(rsqrt(step), rel=1e-12)
    task.global_step = 12                                    # disc: StepLR at max(12 - 10, 1) = 2 -> no decay yet
    task.on_after_optimization(0, 0, opts[1], 1)
    assert opts[1].param_groups[0]['lr'] == pytest.approx(hp['disc_lr'])
    task.global_step = 14                                    # 4 -> one decay
    task.on_after_optimization(0, 0, opts[1], 1)
    assert opts[1].param_groups[0]['lr'] == pytest.approx(hp['disc_lr'] * 0.5)
    task.global_step = 7                                     # map: StepLR at global_step 7 -> two decays of 0.1
    task.on_after_optimization(0, 0, opts[2], 2)
    assert opts[2].param_groups[0]['lr'] == pytest.approx(hp['map_lr'] * 0.01)
    hp['scheduler'] = 'none'
    opts = task.configure_optimizers()
    task.global_step = 5
    task.on_after_optimization(0, 0, opts[0], 0)
    assert opts[0].param_groups[0]['lr'] == 1.0


@pytest.mark.parametrize('key', ['use_cond_disc', 'rerun_gen'])
def test_unsupported_options_raise(hp, small_data, key):
    _config(hp, small_data, f'{key}=True')
    with pytest.raises(NotImplementedError, match=key):
        T.SVBVAEMleTask().build_model()


# ---------------------------------------------------------------------------------------------------------- config
TASK_KEYS = [
    'hidden_size', 'audio_num_mel_bins', 'latent_size', 'fvae_enc_dec_hidden', 'fvae_kernel_size', 'fvae_enc_n_layers',
    'fvae_dec_n_layers', 'asr_enc_layers', 'asr_last_norm', 'mel_strides', 'phase_1_steps', 'phase_2_steps', 'phase_1_concurrent_ways',
    'phase_2_concurrent_ways', 'phase_3_concurrent_ways', 'disable_map', 'mel_loss', 'lambda_kl', 'lambda_mle', 'lambda_mel_adv',
    'cross_way_no_recon_loss', 'cross_way_no_disc_loss', 'mel_gan', 'use_cond_disc', 'rerun_gen', 'disc_win_num',
    'mel_disc_hidden_size', 'disc_norm', 'disc_reduction', 'disc_start_steps', 'disc_interval', 'lr', 'scheduler', 'warmup_updates',
    'optimizer_adam_beta1', 'optimizer_adam_beta2', 'weight_decay', 'disc_lr', 'discriminator_optimizer_params',
    'discriminator_scheduler_params', 'map_lr', 'map_scheduler_params', 'generator_grad_norm', 'discriminator_grad_norm', 'max_frames',
    'frames_multiple', 'min_frames', 'max_tokens', 'max_sentences', 'max_valid_tokens', 'max_valid_sentences', 'endless_ds',
    'sort_by_len', 'num_test_samples', 'test_ids', 'normalize_pitch', 'pitch_norm', 'use_uv', 'audio_sample_rate', 'hop_size',
    'out_wav_norm', 'gen_dir_name', 'load_ckpt', 'train_set_name', 'valid_set_name', 'test_set_name', 'seed', 'max_updates',
    'val_check_interval', 'valid_infer_interval', 'num_valid_plots', 'num_sanity_val_steps', 'tb_log_interval', 'accumulate_grad_batches',
    'amp', 'valid_monitor_key', 'valid_monitor_mode', 'num_ckpt_keep', 'save_best', 'binary_data_dir', 'pretrain_asr_ckpt', 'vocoder',
    'vocoder_ckpt', 'task_cls']
# the values egs/svb_vae_train_synthetic.yaml changes, each with its reason in the YAML's comments
DEVIATIONS = {'phase_2_steps', 'lr', 'scheduler', 'max_sentences', 'max_updates', 'val_check_interval', 'valid_infer_interval',
              'num_valid_plots', 'num_sanity_val_steps', 'tb_log_interval', 'binary_data_dir', 'pretrain_asr_ckpt', 'vocoder',
              'vocoder_ckpt'}


def test_synthetic_config_resolves_the_reference_hyper_parameters(hp):
    with open(os.path.join(ROOT, 'tests', 'golden', 'hparams', 'expected.json')) as f:
        ref = json.load(f)['egs/datasets/audio/PopBuTFy/vae_global_mle_eng.yaml']
    got = H.set_hparams(CONFIG, '', '', print_hparams=False, global_hparams=False)
    for k in TASK_KEYS:
        assert k in got, k
        if k not in DEVIATIONS | {'task_cls'}:
            assert got[k] == ref[k], (k, got[k], ref[k])
    with open(CONFIG) as f:
        commented = {line.split(':')[0] for line in f if '# reference' in line}
    assert DEVIATIONS == commented
    assert got['task_cls'].endswith('svb_vae_task.SVBVAEMleTask') and ref['task_cls'].endswith('svb_vae_task.SVBVAEMleTask')

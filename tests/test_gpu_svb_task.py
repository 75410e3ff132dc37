"""-m gpu: SVBVAEMleTask on the device.

  * each kind of training step (phase-2 G and D, phase-3 map, phase-1) against the same loss terms assembled by hand from the
    MleSVBVAE / Discriminator / mel_l1_ssim_loss calls of tools/svb_train_bench.py::native_step, with the same random draws, and
    gradients only in that optimizer's parameters;
  * ``tasks/run.py`` end to end on a synthetic dataset: training across phases 2 and 3 with validation audio, the checkpoint
    layout, resuming, and ``--infer`` writing the five wav and mel sets;
  * two ranks through the trainer's mp.spawn path when two GPUs are visible.
Sizes stay small (B <= 4, T <= 256 frames)."""
import glob
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200.utils import hparams as H
from neuralsvb_b200.utils.synthetic import write_svb_binary

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, 'egs', 'svb_vae_train_synthetic.yaml')


@pytest.fixture(scope='module')
def data_dir(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('svb_data'))
    write_svb_binary(d, 4, 1234, n_valid=1, n_test=2, frames=(60, 160))
    return d


def _overrides(d, extra=''):
    return f'binary_data_dir={d},pretrain_asr_ckpt={d}/asr,vocoder_ckpt={d}/hifigan' + (',' + extra if extra else '')


# ------------------------------------------------------------------------------------------------- one step of each kind
@pytest.fixture(scope='module')
def task_and_batch(data_dir):
    from neuralsvb_b200.tasks.singing.svb_vae_task import SVBVAEMleTask
    from neuralsvb_b200.utils import move_to_cuda
    saved = dict(H.hparams)
    H.set_hparams(CONFIG, '', _overrides(data_dir, 'phase_1_steps=5,phase_2_steps=10,disc_start_steps=0'), print_hparams=False)
    torch.cuda.set_device(0)
    task = SVBVAEMleTask()
    task.build_model()
    task.cuda()
    opts = task.configure_optimizers()
    batch = move_to_cuda(next(iter(task.train_dataloader())))
    yield task, opts, batch
    H.hparams.clear()
    H.hparams.update(saved)


def _task_loss(task, opts, batch, step, opt_idx, seed):
    mine = {id(p) for g in opts[opt_idx].param_groups for p in g['params']}
    for p in task.parameters():                              # what Trainer.run_training_batch does before each optimizer
        p.requires_grad = id(p) in mine
        p.grad = None
    task.global_step = step
    np.random.seed(seed)
    torch.manual_seed(seed)
    loss = task.training_step(batch, 0, opt_idx)['loss']
    loss.backward()
    with_grad = {id(p) for p in task.parameters() if p.grad is not None}
    assert with_grad and with_grad <= mine, 'gradients outside the stepped optimizer'
    assert any(float(p.grad.abs().sum()) > 0 for p in task.parameters() if p.grad is not None)
    return loss.detach()


def _hand(task, batch, ways, seed, disc_ways=(), mle=False):
    """tools/svb_train_bench.py::native_step's loss assembly with the task's hyper-parameters (λ_kl 1e-3, l1 / ssim 0.5,
    λ_mle 1, λ_mel_adv 0.1), the speaker embedding drawn as the task draws it."""
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    hp = H.hparams
    np.random.seed(seed)
    torch.manual_seed(seed)
    idx = np.random.randint(1, batch['multi_spk_emb'].shape[1])
    spk = batch['multi_spk_emb'][:, idx]
    # grad mode on, as in a training step: the train-mode BatchNorms use batch statistics only then
    ret = task.model(amateur_mel=batch['mels'], prof_mel=batch['prof_mels'], amateur_pitch=batch['pitch'], prof_pitch=batch['prof_pitch'],
                     amateur_spk_id=spk, prof_spk_id=spk, a2p_alignment=batch['a2p_f0_alignment'], concurrent_ways=ways)
    targets = {'a2a': batch['mels'], 'p2p': batch['prof_mels'], 'a2p': batch['prof_mels']}
    loss = 0
    for way in ways:
        if 'kl' in ret[way]:
            loss = loss + ret[way]['kl'] * hp['lambda_kl']
        l1, ss = mel_l1_ssim_loss(ret[way]['mel_out'], targets[way])
        loss = loss + 0.5 * l1 + 0.5 * ss
    if mle:
        loss = loss + ret['a2p']['mle'] * hp['lambda_mle']
    for way in disc_ways:
        y = task.mel_disc(ret[way]['mel_out'])['y']
        loss = loss + F.mse_loss(y, torch.ones_like(y)) * hp['lambda_mel_adv']
    return loss.detach(), ret


def _hand_d(task, batch, ret, ways, seed):
    np.random.seed(seed)
    torch.manual_seed(seed)
    targets = {'a2a': batch['mels'], 'p2p': batch['prof_mels']}
    loss = 0
    for way in ways:
        y_r, y_f = task.mel_disc(targets[way])['y'], task.mel_disc(ret[way]['mel_out'].detach())['y']
        loss = loss + F.mse_loss(y_r, torch.ones_like(y_r)) + F.mse_loss(y_f, torch.zeros_like(y_f))
    return loss.detach()


def _close(a, b):
    assert abs(float(a) - float(b)) <= 1e-6 * abs(float(b)), (float(a), float(b))


def test_phase_2_g_and_d_steps_match_hand_assembled_losses(task_and_batch):
    task, opts, batch = task_and_batch
    task.train()
    g = _task_loss(task, opts, batch, 7, 0, 11)
    d = _task_loss(task, opts, batch, 7, 1, 12)
    want_g, ret = _hand(task, batch, ['a2a', 'p2p'], 11, disc_ways=('a2a', 'p2p'))
    _close(g, want_g)
    _close(d, _hand_d(task, batch, ret, ['a2a', 'p2p'], 12))
    assert task.training_step(batch, 0, 2)['loss'] is None


def test_phase_3_map_step_matches_hand_assembled_loss(task_and_batch):
    task, opts, batch = task_and_batch
    task.train()
    m = _task_loss(task, opts, batch, 11, 2, 13)
    assert not task.model.training and task.model.z_mapping_function.training
    _close(m, _hand(task, batch, ['a2a', 'p2p', 'a2p'], 13, disc_ways=('a2p',), mle=True)[0])
    assert task.training_step(batch, 0, 0)['loss'] is None and task.training_step(batch, 0, 1)['loss'] is None


def test_phase_1_step_matches_hand_assembled_loss(task_and_batch):
    task, opts, batch = task_and_batch
    task.train()
    g = _task_loss(task, opts, batch, 3, 0, 14)
    want, ret = _hand(task, batch, ['p2p'], 14, disc_ways=('p2p',))
    _close(g, want)
    _close(_task_loss(task, opts, batch, 3, 1, 15), _hand_d(task, batch, ret, ['p2p'], 15))


# ------------------------------------------------------------------------------------------------- tasks/run.py end to end
def _run(cwd, args, timeout):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, '-m', 'neuralsvb_b200.tasks.run', '--config', CONFIG, '--exp_name', 'svb_cli'] + args,
                       cwd=cwd, env=env, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_run_py_trains_resumes_and_infers(tmp_path, data_dir):
    from scipy.io import wavfile
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    ov = _overrides(data_dir, 'max_updates=12,phase_2_steps=8,val_check_interval=6,valid_infer_interval=6,tb_log_interval=1,lr=0.001')
    out = _run(tmp_path, ['--reset', '--hparams', ov], 900)
    assert 'Training end' in out and '| valid results' in out
    steps = {int(m.group(1)): m.group(2) for m in re.finditer(r'\| step (\d+): (.*)', out)}
    mel = lambda s: sum(float(v) for k, v in re.findall(r'(\w+) ([0-9.eE+-]+)', steps[s]) if k in ('l1a2a', 'ssima2a', 'l1p2p', 'ssimp2p'))
    p2 = sorted(s for s in steps if s <= 8 and 'l1a2a' in steps[s])
    assert len(p2) >= 6 and mel(p2[-1]) < mel(p2[0]), [mel(s) for s in p2]
    assert any('a2p_mle' in steps[s] for s in steps if s > 8)                  # phase 3 ran
    work = tmp_path / 'checkpoints' / 'svb_cli'
    ev = EventAccumulator(str(work / 'lightning_logs' / 'version_lastest'), size_guidance={'audio': 0})
    ev.Reload()
    tags = ev.Tags()['audio']
    assert all(any(t.startswith(x) for t in tags) for x in ('a2a_wavout_0', 'p2p_wavout_0', 'gt_a_wav_0', 'gt_p_wav_0')), tags
    ck = torch.load(work / 'model_ckpt_steps_12.ckpt', map_location='cpu', weights_only=False)
    assert set(ck['state_dict']) == {'model', 'mel_disc'} and len(ck['optimizer_states']) == 3
    assert len(ck['state_dict']['model']) == 259
    H.set_hparams(CONFIG, '', _overrides(data_dir), print_hparams=False)
    MleSVBVAE(70).load_state_dict(ck['state_dict']['model'], strict=True)             # the README snippet's load
    out = _run(tmp_path, ['--hparams', 'max_updates=14'], 900)                        # resumes from step 12
    assert '| step 12:' in out and '| step 11:' not in out and 'Training end' in out
    out = _run(tmp_path, ['--infer'], 900)
    gen = work / 'generated_12_'
    hop, sr = 128, 22050
    for key in ('gt_a', 'gt_p', 'a2a', 'p2p', 'a2p'):
        wavs = sorted(glob.glob(str(gen / 'wavs' / f'{key}_wavout' / '*.wav')))
        mels = sorted(glob.glob(str(gen / 'mels' / f'{key}_mel' / '*.npy')))
        assert len(wavs) == len(mels) == 2, (key, wavs, mels)
        for w, m in zip(wavs, mels):
            rate, data = wavfile.read(w)
            assert rate == sr and len(data) == np.load(m).shape[0] * hop and np.abs(data).max() > 10, (w, len(data))


# ------------------------------------------------------------------------------------------------- two ranks
def _ddp_worker(rank, world, data_dir, out_dir, port):
    from neuralsvb_b200.tasks.singing.svb_vae_task import SVBVAEMleTask
    from neuralsvb_b200.utils.trainer import Trainer
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    os.chdir(out_dir)                                        # ranks > 0 write their TensorBoard logs under ./tmp
    H.set_hparams(CONFIG, '', _overrides(data_dir, 'max_sentences=2'), print_hparams=False)
    H.hparams['work_dir'] = out_dir
    names = []

    class Task(SVBVAEMleTask):
        def training_step(self, sample, batch_idx, optimizer_idx=-1):
            if optimizer_idx == 0:
                names.extend(sample['item_name'])
            return super().training_step(sample, batch_idx, optimizer_idx)

        def on_train_end(self):
            torch.save({'params': {n: p.detach().cpu() for n, p in self.named_parameters()}, 'names': names,
                        'collectives': [r.collectives if r is not None else 0 for r in self.trainer.reducers]},
                       os.path.join(out_dir, f'rank{rank}.pt'))
    tr = Trainer(work_dir=out_dir, val_check_interval=1000, max_updates=3, num_sanity_val_steps=0, seed=1234, tb_log_interval=1000)
    np.random.seed(1234)
    tr._ddp_worker(rank, Task, None, rank, world)
    torch.distributed.destroy_process_group()


def test_two_ranks_stay_identical(tmp_path, data_dir):
    if torch.cuda.device_count() < 2:
        pytest.skip(f'needs 2 GPUs, {torch.cuda.device_count()} visible')
    import torch.multiprocessing as mp
    ctx = mp.start_processes(_ddp_worker, args=(2, data_dir, str(tmp_path), 29000 + os.getpid() % 1000), nprocs=2, join=False,
                             start_method='spawn')
    deadline = time.time() + 900
    try:
        while not ctx.join(timeout=5):
            assert time.time() < deadline, 'two-rank run timed out'
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.kill()
            p.join()
    r0, r1 = (torch.load(tmp_path / f'rank{r}.pt') for r in range(2))
    for n, p in r0['params'].items():
        assert torch.equal(p, r1['params'][n]), n
    # steps 0..3 in phase 2: one gen exchange per step, one disc exchange from step 1 (disc_start_steps 0), no map exchange
    assert r0['collectives'] == r1['collectives'] == [4, 3, 0]
    assert not set(r0['names']) & set(r1['names'])

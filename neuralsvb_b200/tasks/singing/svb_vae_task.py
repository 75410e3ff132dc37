"""``SVBVAEMleTask``: training, validation and inference of the SVB acoustic model through ``tasks/run.py`` (reference:
tasks/singing/svb_vae_task.py:543-726 with the parts of ``SVBVAETask`` / ``SVBVAEBoostTask`` (:48-165, :302-404),
``gen_cheat_disc`` / ``disc_judge_gen`` / ``get_corresponding_gtmel`` (svb_para.py:118-170) and ``build_disc_model``
(fs2_adv.py:22-35) that it uses), written as one class on this package's ``BaseTask``.

Three optimizers, in the trainer's order:
  0  gen   every MleSVBVAE parameter outside ``vc_asr`` and ``z_mapping_function``; phases 1 and 2
  1  disc  the mel discriminator; phases 1 and 2, from ``disc_start_steps`` on, every ``disc_interval`` steps
  2  map   ``z_mapping_function``; phase 3, with the rest of the model in eval mode
Phase p runs while ``global_step <= phase_p_steps`` (phase 3 after ``phase_2_steps``) with the ways ``phase_p_concurrent_ways``.

Every forward and backward of the step is a CUDA kernel of this package (``MleSVBVAE(trainable=True)``, the native mel
discriminator, ``mel_l1_ssim_loss``); torch adds the loss sums, ``F.mse_loss`` on the discriminator outputs, AdamW and gradient
clipping.  ``vc_asr`` is loaded from ``pretrain_asr_ckpt`` and frozen.  ``use_cond_disc`` and ``rerun_gen`` are not supported."""
import json
import os

import numpy as np
import torch
import torch.nn.functional as F

from neuralsvb_b200.tasks.base_task import BaseTask
from neuralsvb_b200.tasks.singing.dataset_utils import MultiSpkEmbDataset, build_batches, build_dataloader
from neuralsvb_b200.utils import audio, ddp_utils, tensors_to_scalars
from neuralsvb_b200.utils.ckpt_utils import load_ckpt
from neuralsvb_b200.utils.common_schedulers import NoneSchedule, RSQRTSchedule
from neuralsvb_b200.utils.hparams import hparams
from neuralsvb_b200.utils.pitch_utils import denorm_f0
from neuralsvb_b200.vocoders.base_vocoder import get_vocoder_cls

WAYS = ('a2a', 'p2p', 'a2p')


def phase_of(step, hp):
    """(phase, ways) of the training step ``step``."""
    if step <= hp['phase_1_steps']:
        return 1, hp['phase_1_concurrent_ways'].split(',')
    if step <= hp['phase_2_steps']:
        return 2, hp['phase_2_concurrent_ways'].split(',')
    return 3, hp['phase_3_concurrent_ways'].split(',')


def valid_ways(step, hp):
    """Ways a validation step runs at training step ``step`` (svb_vae_task.py:694-700)."""
    if step <= hp['phase_1_steps']:
        return ['p2p']
    return ['a2a', 'p2p'] if step <= hp['phase_2_steps'] else list(WAYS)


def mel_loss_lambdas(spec):
    """'ssim:0.5|l1:0.5' -> {'ssim': 0.5, 'l1': 0.5}; the native mel loss computes l1 and ssim only."""
    out = {}
    for part in spec.split('|'):
        name, lbd = part.split(':')
        if name not in ('l1', 'ssim'):
            raise NotImplementedError(f'mel_loss {name!r}: only l1 and ssim are implemented')
        out[name] = float(lbd)
    return out


class SVBVAEMleTask(BaseTask):
    def __init__(self):
        super().__init__()
        self.vocoder, self.mel_disc, self.model_out = None, None, None
        self.loss_and_lambda = mel_loss_lambdas(hparams['mel_loss'])
        self._loaders = {}

    # ------------------------------------------------------------------ model and optimizers
    def build_model(self):
        from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
        if hparams['use_cond_disc']:
            raise NotImplementedError('use_cond_disc: the conditional mel discriminator is not implemented; set use_cond_disc: false')
        if hparams['rerun_gen']:
            raise NotImplementedError('rerun_gen: the discriminator step judges the generator step\'s detached output '
                                      '(the reference exits on rerun_gen too); set rerun_gen: false')
        with open(os.path.join(hparams['binary_data_dir'], 'phone_set.json')) as f:
            phone_list = json.load(f)
        self.model = MleSVBVAE(len(phone_list) + 10, trainable=True, precision=hparams.get('svb_precision', 'bf16x3'))
        load_ckpt(self.model.vc_asr, hparams['pretrain_asr_ckpt'], model_name='model')
        self.model.vc_asr.eval()
        for p in self.model.vc_asr.parameters():
            p.requires_grad = False
        if hparams['load_ckpt'] != '':
            self.load_ckpt(hparams['load_ckpt'], strict=False)
        self.build_disc_model()
        self.gen_params = [p for n, p in self.model.named_parameters() if 'vc_asr' not in n and 'z_mapping_function' not in n]
        self.mapping_params = list(self.model.z_mapping_function.parameters())
        return self.model

    def build_disc_model(self):
        self.disc_params = []
        if hparams['mel_gan']:
            from neuralsvb_b200.modules.fastspeech.multi_window_disc import Discriminator
            self.mel_disc = Discriminator(time_lengths=[32, 64, 128][:hparams['disc_win_num']], freq_length=80,
                                          hidden_size=hparams['mel_disc_hidden_size'], kernel=(3, 3), cond_size=0,
                                          norm_type=hparams['disc_norm'], reduction=hparams['disc_reduction'])
            self.disc_params = list(self.mel_disc.parameters())

    def configure_optimizers(self):
        betas = (hparams['optimizer_adam_beta1'], hparams['optimizer_adam_beta2'])
        opt_gen = torch.optim.AdamW(self.gen_params, lr=hparams['lr'], betas=betas, weight_decay=hparams['weight_decay'])
        opt_disc = torch.optim.AdamW(self.disc_params, lr=hparams['disc_lr'], betas=betas,
                                     **hparams['discriminator_optimizer_params']) if self.disc_params else None
        opt_map = torch.optim.AdamW(self.mapping_params, lr=hparams['map_lr'], betas=betas, weight_decay=hparams['weight_decay'])
        self.scheduler = {
            'gen': RSQRTSchedule(opt_gen) if hparams['scheduler'] == 'rsqrt' else NoneSchedule(opt_gen),
            'disc': torch.optim.lr_scheduler.StepLR(opt_disc, **hparams['discriminator_scheduler_params']) if opt_disc else None,
            'map': torch.optim.lr_scheduler.StepLR(opt_map, **hparams['map_scheduler_params']),
        }
        return [opt_gen, opt_disc, opt_map]

    def on_before_optimization(self, opt_idx):
        params, norm = [(self.gen_params, 'generator_grad_norm'), (self.disc_params, 'discriminator_grad_norm'),
                        (self.mapping_params, 'generator_grad_norm')][opt_idx]
        torch.nn.utils.clip_grad_norm_(params, hparams[norm])

    def on_after_optimization(self, epoch, batch_idx, optimizer, optimizer_idx):
        if optimizer_idx == 0:
            self.scheduler['gen'].step(self.global_step)
        elif optimizer_idx == 1:
            self.scheduler['disc'].step(max(self.global_step - hparams['disc_start_steps'], 1))
        else:
            self.scheduler['map'].step(self.global_step)

    # ------------------------------------------------------------------ data
    def _loader(self, prefix, shuffle, max_tokens, max_sentences, endless=False, by_size=True):
        if prefix not in self._loaders:
            ds = MultiSpkEmbDataset(prefix, hparams, shuffle=shuffle)
            rank, world, _ = ddp_utils.dist_env()
            self._loaders[prefix] = build_dataloader(ds, build_batches(ds, shuffle, max_tokens, max_sentences, rank, world, endless,
                                                                       by_size))
        return self._loaders[prefix]

    def _valid_limits(self):
        return (hparams['max_tokens'] if hparams['max_valid_tokens'] == -1 else hparams['max_valid_tokens'],
                hparams['max_sentences'] if hparams['max_valid_sentences'] == -1 else hparams['max_valid_sentences'])

    def train_dataloader(self):
        return self._loader(hparams['train_set_name'], True, hparams['max_tokens'], hparams['max_sentences'], hparams['endless_ds'])

    def val_dataloader(self):
        return self._loader(hparams['valid_set_name'], False, *self._valid_limits())

    def test_dataloader(self):
        return self._loader(hparams['test_set_name'], False, *self._valid_limits(), by_size=False)

    # ------------------------------------------------------------------ the step
    @staticmethod
    def get_corresponding_gtmel(way, sample):
        return sample['mels'] if way in ('a2a', 'p2a') else sample['prof_mels']

    def add_mel_loss(self, mel_out, target, losses, postfix):
        from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
        l1, ssim = mel_l1_ssim_loss(mel_out, target)
        for name, lbd in self.loss_and_lambda.items():
            losses[f'{name}{postfix}'] = (l1 if name == 'l1' else ssim) * lbd

    def run_model(self, sample, concurrent_ways, infer=False, disable_map=False):
        """The model on both takes with one speaker embedding (a random one of rows 1-4 in training, row 0 in inference) and
        the per-way KL and mel losses."""
        self.model.vc_asr.eval()
        idx = 0 if infer else np.random.randint(1, sample['multi_spk_emb'].shape[1])
        spk = sample['multi_spk_emb'][:, idx, :]
        out = self.model(amateur_mel=sample['mels'], prof_mel=sample['prof_mels'], amateur_pitch=sample['pitch'],
                         prof_pitch=sample['prof_pitch'], amateur_spk_id=spk, prof_spk_id=spk, a2p_alignment=sample['a2p_f0_alignment'],
                         infer=False, concurrent_ways=concurrent_ways, disable_map=disable_map)
        losses = {}
        for way in concurrent_ways:
            if 'kl' in out[way]:
                losses[f'{way}_kl'] = out[way]['kl'] * hparams['lambda_kl']
            if way in ('a2a', 'p2p') or not hparams['cross_way_no_recon_loss']:
                self.add_mel_loss(out[way]['mel_out'], self.get_corresponding_gtmel(way, sample), losses, way)
        return losses, out

    def _adv(self, mel, target_one):
        y = self.mel_disc(mel)['y']
        if y is None:
            return None
        return F.mse_loss(y, torch.ones_like(y) if target_one else torch.zeros_like(y))

    def _training_step(self, sample, batch_idx, optimizer_idx):
        log, weights = {}, {}
        disc_start = hparams['mel_gan'] and self.global_step > hparams['disc_start_steps'] and hparams['lambda_mel_adv'] > 0
        phase, ways = phase_of(self.global_step, hparams)
        if optimizer_idx == 0 and phase in (1, 2):
            self.model.z_mapping_function.eval()
            log, out = self.run_model(sample, ways)
            self.model_out = {w: {k: v.detach() for k, v in out[w].items() if isinstance(v, torch.Tensor)} for w in out}
            if disc_start:
                for way in ways:
                    a = self._adv(out[way]['mel_out'], True)
                    if a is not None:
                        log[f'{way}_a'], weights[f'{way}_a'] = a, hparams['lambda_mel_adv']
        elif optimizer_idx == 1 and phase in (1, 2):
            self.model.z_mapping_function.eval()
            if disc_start and self.global_step % hparams['disc_interval'] == 0:
                for way in ways:
                    r = self._adv(self.get_corresponding_gtmel(way, sample), True)
                    f = self._adv(self.model_out[way]['mel_out'], False)
                    if f is not None:
                        log[f'{way}_r'], log[f'{way}_f'] = r, f
        elif optimizer_idx == 2 and phase == 3:
            self.model.eval()
            self.model.z_mapping_function.train()
            log, out = self.run_model(sample, ['a2a', 'p2p'] + ways)
            for way in ways:
                log[f'{way}_mle'], weights[f'{way}_mle'] = out[way]['mle'], hparams['lambda_mle']
                if not hparams['cross_way_no_disc_loss'] and self.mel_disc is not None:
                    a = self._adv(out[way]['mel_out'], True)
                    if a is not None:
                        log[f'{way}_a'], weights[f'{way}_a'] = a, hparams['lambda_mel_adv']
        if not log:
            return None
        for k in [f'{w}_{t}' for w in WAYS for t in ('kl', 'mle')]:
            if k in log and not bool(torch.isfinite(log[k]).all()):
                log[k] = log[k].detach()
        total = sum(weights.get(k, 1) * v for k, v in log.items())
        log['bs'] = sample['mels'].shape[0]
        return total, log

    def training_step(self, sample, batch_idx, optimizer_idx=-1):
        ret = self._training_step(sample, batch_idx, optimizer_idx)
        if ret is None:
            return {'loss': None}
        total, log = ret
        # device scalars: the trainer reads them only when it prints / writes TensorBoard
        log = {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in log.items()}
        if optimizer_idx >= 0 and self.trainer is not None:
            log[f'lr_{optimizer_idx}'] = self.trainer.optimizers[optimizer_idx].param_groups[0]['lr']
        return {'loss': total, 'progress_bar': log, 'tb_log': {f'tr/{k}': v for k, v in log.items()}}

    # ------------------------------------------------------------------ validation
    def _vocoder(self):
        if self.vocoder is None:
            self.vocoder = get_vocoder_cls(hparams)()
        return self.vocoder

    def _f0s(self, sample):
        a = denorm_f0(sample['f0'], sample['uv'], hparams)
        p = denorm_f0(sample['prof_f0'], sample['prof_uv'], hparams)
        return {'a2a': a, 'p2p': p, 'a2p': p}

    def validation_step(self, sample, batch_idx):
        ways = valid_ways(self.global_step, hparams)
        losses, out = self.run_model(sample, ways, infer=True, disable_map=hparams['disable_map'])
        for way in ways:
            if 'mle' in out[way]:
                losses[f'{way}_mle'] = out[way]['mle']
        outputs = tensors_to_scalars({'losses': losses, 'total_loss': sum(losses.values()), 'nsamples': sample['nsamples']})
        if self.global_step % hparams['valid_infer_interval'] == 0 and batch_idx < hparams['num_valid_plots'] \
                and self.logger is not None:
            sr, f0s = hparams['audio_sample_rate'], self._f0s(sample)
            clips = {f'{way}_wavout_{batch_idx}': (out[way]['mel_out'][0], f0s[way][0]) for way in ways}
            clips[f'gt_a_wav_{batch_idx}'] = (sample['mels'][0], f0s['a2a'][0])
            clips[f'gt_p_wav_{batch_idx}'] = (sample['prof_mels'][0], f0s['p2p'][0])
            for tag, (mel, f0) in clips.items():
                wav = self._vocoder().spec2wav(mel.float().cpu().numpy(), f0=f0.cpu().numpy())
                self.logger.add_audio(tag, torch.from_numpy(wav)[None], self.global_step, sr)
        return outputs

    def validation_end(self, outputs):
        sums, n_all = {'total_loss': 0.0}, 0
        for o in outputs:
            n = o['nsamples']
            n_all += n
            for k, v in list(o['losses'].items()) + [('total_loss', o['total_loss'])]:
                sums[k] = sums.get(k, 0.0) + v * n
        res = {k: round(v / max(n_all, 1), 4) for k, v in sums.items()}
        print(f'| valid results: {res}', flush=True)
        return {'tb_log': {f'val/{k}': v for k, v in res.items()}, 'val_loss': res['total_loss'], 'nsamples': n_all}

    def on_train_end(self):
        if self.logger is not None:              # the audio and scalars of the last validation reach the event file
            self.logger.flush()

    # ------------------------------------------------------------------ inference
    def test_start(self):
        self._vocoder()
        self.gen_dir = os.path.join(hparams['work_dir'], f'generated_{self.trainer.global_step}_{hparams["gen_dir_name"]}')

    def test_step(self, sample, batch_idx):
        assert sample['nsamples'] == 1, 'Only support batch_size=1 in inference.'
        _, out = self.run_model(sample, list(WAYS), infer=True, disable_map=hparams['disable_map'])
        f0s = self._f0s(sample)
        item_name = sample['item_name'][0]
        np0 = lambda t: t[0].float().cpu().numpy()
        mels = {'gt_a': np0(sample['mels']), 'gt_p': np0(sample['prof_mels'])}
        mels.update({way: np0(out[way]['mel_out']) for way in WAYS})
        f0 = {'gt_a': f0s['a2a'], 'gt_p': f0s['p2p'], **f0s}
        base_fn = f'[{0:06d}][{item_name}][P]'.replace(' ', '_')
        prefix = 'disable_map_' if hparams['disable_map'] else ''
        for key, mel in mels.items():
            wav = self._vocoder().spec2wav(mel, f0=np0(f0[key]))
            wkey, mkey = prefix + (f'{key}_wavout'), prefix + (f'{key}_mel')
            os.makedirs(f'{self.gen_dir}/wavs/{wkey}', exist_ok=True)
            os.makedirs(f'{self.gen_dir}/mels/{mkey}', exist_ok=True)
            audio.save_wav(wav, f'{self.gen_dir}/wavs/{wkey}/{base_fn}.wav', hparams['audio_sample_rate'], norm=hparams['out_wav_norm'])
            np.save(f'{self.gen_dir}/mels/{mkey}/{base_fn}.npy', mel)
        return {'item_name': item_name}

    def test_end(self, outputs):
        print(f'| SVB infer: {len(outputs)} items -> {self.gen_dir}', flush=True)
        return {}

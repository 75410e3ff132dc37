"""Time the SVB acoustic model's training steps (BASELINE config 4, per GPU: B = 16, T = 1024 mel frames, vae_global_mle_eng sizes):

  phase2    the generator step: a2a + p2p forward, the KL and mel losses, backward into every parameter outside vc_asr and the latent map
  phase3    the mapping step: model in eval mode, latent map in train mode, a2a + p2p + a2p forward, losses, backward into the latent map
  mel_loss  the masked L1 + SSIM mel loss alone on one [16, 1024, 80] pair, forward and backward

By default both steps are the reference step (SVBVAEMleTask) minus the adversarial terms.  With --mel-gan they include them (the mel
discriminator of vae_global_mle_eng: 3 windows, instance norm, 'stack', lambda_mel_adv 0.1):

  phase2    the G step with {a2a,p2p}_a, then the D step ({way}_r / {way}_f on the ground-truth and the detached mel_out)
  phase3    the mapping step with a2p_a through the eval-mode model
  mel_disc  one discriminator forward + backward (d mel and every parameter gradient) on a [16, 1024, 80] mel

Native path (MleSVBVAE(trainable=True) with the WN stacks in bf16x3 or fp32, mel_l1_ssim_loss) against the same graph in PyTorch
eager on the same GPU, built from the oracle (oracle/svb_vae_train.py, oracle/mel_loss.py), with cuDNN TF32 on and off.  Prints one JSON line
per configuration with the GPU name and power limit read in the same run.

    python tools/svb_train_bench.py --steps 50 --warmup 5 [--mel-gan]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.fvae_train_bench import gpu_info, timeit  # noqa: E402

HP = {'hidden_size': 256, 'audio_num_mel_bins': 80, 'asr_enc_layers': 2, 'mel_strides': [2, 1, 1], 'asr_last_norm': False, 'latent_size': 128,
      'fvae_enc_dec_hidden': 192, 'fvae_kernel_size': 5, 'fvae_enc_n_layers': 8, 'fvae_dec_n_layers': 4}
LAMBDAS = {'kl': 0.001, 'mle': 1.0, 'l1': 0.5, 'ssim': 0.5}
LAMBDA_MEL_ADV = 0.1


def set_phase(m, phase):
    for n, p in m.named_parameters():
        p.requires_grad_(n.startswith('z_mapping_function.') if phase == 3 else not n.startswith(('vc_asr.', 'z_mapping_function.')))
    if phase == 2:
        m.train()
        m.z_mapping_function.eval()
    else:
        m.eval()
        m.z_mapping_function.train()
    m.vc_asr.eval()


def _targets(batch):
    return {'a2a': batch['amateur_mel'], 'p2p': batch['prof_mel'], 'a2p': batch['prof_mel']}


def native_step(m, batch, phase, disc=None):
    """One step; with ``disc`` (the native mel discriminator) the adversarial terms, and in phase 2 the D step after the G step."""
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    ways = ['a2a', 'p2p'] if phase == 2 else ['a2a', 'p2p', 'a2p']
    ret = m(**batch, concurrent_ways=ways)
    targets = _targets(batch)
    loss = 0
    for way in ways:
        if 'kl' in ret[way]:
            loss = loss + ret[way]['kl'] * LAMBDAS['kl']
        l1, ss = mel_l1_ssim_loss(ret[way]['mel_out'], targets[way])
        loss = loss + LAMBDAS['l1'] * l1 + LAMBDAS['ssim'] * ss
    if phase == 3:
        loss = loss + ret['a2p']['mle'] * LAMBDAS['mle']
    if disc is not None:
        disc.requires_grad_(False)
        for way in (['a2a', 'p2p'] if phase == 2 else ['a2p']):
            y = disc(ret[way]['mel_out'])['y']
            loss = loss + F.mse_loss(y, torch.ones_like(y)) * LAMBDA_MEL_ADV
    loss.backward()
    if disc is not None and phase == 2:
        disc.requires_grad_(True)
        loss_d = 0
        for way in ways:
            y_r, y_f = disc(targets[way])['y'], disc(ret[way]['mel_out'].detach())['y']
            loss_d = loss_d + F.mse_loss(y_r, torch.ones_like(y_r)) + F.mse_loss(y_f, torch.zeros_like(y_f))
        loss_d.backward()


def eager_draws(n_calls, B, T, dev):
    """Window starts and Dropout2d factors of n discriminator calls, drawn as the reference draws them."""
    starts, scales = [], []
    for _ in range(n_calls):
        starts.append([[np.random.randint(0, T - w + 1)] * B for w in (32, 64, 128)])
        scales.append([[torch.empty(B, 128, device=dev).bernoulli_(0.75).div_(0.75) for _ in range(3)] for _ in range(3)])
    return starts, scales


def eager_step(p, batch, eps, phase, dsd=None):
    from oracle import multi_window_disc as OD
    from oracle import svb_vae_train as O
    losses, out = O.svb_train_losses(p, batch, eps, phase)
    if dsd is not None:
        B, T = batch['amateur_mel'].shape[:2]
        g = 'g' if phase == 2 else 3
        mels = {w: out[w]['mel_out'] for w in (['a2a', 'p2p'] if phase == 2 else ['a2p'])}
        frozen = {k: v.detach() for k, v in dsd.items()}
        losses.update(OD.svb_adv_losses(frozen, g, mels, None, *eager_draws(len(mels), B, T, eps.device)))
    sum(losses.values()).backward()
    if dsd is not None and phase == 2:
        sum(OD.svb_adv_losses(dsd, 'd', mels, _targets(batch), *eager_draws(4, B, T, eps.device)).values()).backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--frames', type=int, default=1024)
    ap.add_argument('--mel-gan', action='store_true', help='include the mel discriminator (adversarial terms, D step, mel_disc leg)')
    a = ap.parse_args()
    from neuralsvb_b200.modules.commons.mel_loss import mel_l1_ssim_loss
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    from neuralsvb_b200.utils import synthetic as SY
    from oracle import mel_loss as OM
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    B, T = a.batch, a.frames
    sd = SY.make_svb_state_dict(1234)
    batch = {k: v.to(dev) for k, v in SY.make_svb_batch(B, T, T, 1234).items()}
    eps = torch.randn(B, HP['latent_size'], 1, device=dev)
    name, power = gpu_info()
    results = []
    disc, dsd = None, None
    if a.mel_gan:
        from neuralsvb_b200.modules.fastspeech.multi_window_disc import Discriminator
        disc_sd = SY.make_mel_disc_state_dict(1234)
        disc = Discriminator(time_lengths=[32, 64, 128], freq_length=80, hidden_size=128, kernel=(3, 3), cond_size=0, norm_type='in',
                             reduction='stack')
        disc.load_state_dict(disc_sd, strict=True)
        disc = disc.to(dev).train()
        dsd = {k: v.to(dev).requires_grad_(True) for k, v in disc_sd.items()}
    for phase in (2, 3):
        for precision in ('bf16x3', 'fp32'):
            m = MleSVBVAE(80, hp=HP, precision=precision, trainable=True)
            m.load_state_dict(sd, strict=True)
            m = m.to(dev)
            set_phase(m, phase)
            ms = timeit(lambda: native_step(m, batch, phase, disc), a.steps, a.warmup,
                        lambda: (m.zero_grad(set_to_none=True), disc is not None and disc.zero_grad(set_to_none=True)))
            results.append({'step': f'phase{phase}', 'path': f'native {precision}', 'ms': round(ms, 3)})
            del m
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            gen = lambda k: not k.startswith(('vc_asr.', 'z_mapping_function.')) if phase == 2 else k.startswith('z_mapping_function.')
            p = {k: (v.to(dev).float().requires_grad_(gen(k)) if v.is_floating_point() and 'running' not in k else v.to(dev).clone())
                 for k, v in sd.items()}
            eb = {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()}

            def zero():
                for v in list(p.values()) + list((dsd or {}).values()):
                    v.grad = None
            ms = timeit(lambda: eager_step(p, eb, eps, phase, dsd), a.steps, a.warmup, zero)
            results.append({'step': f'phase{phase}', 'path': f'eager cudnn tf32={tf32}', 'ms': round(ms, 3)})
    mel_out, target = SY.make_mel_pair(B, T, [0] + [8 * b for b in range(1, B)], 1234)
    mel_out, target = mel_out.to(dev).requires_grad_(True), target.to(dev)

    def mel_native():
        l1, ss = mel_l1_ssim_loss(mel_out, target)
        (LAMBDAS['l1'] * l1 + LAMBDAS['ssim'] * ss).backward()

    def mel_eager():
        l1, ss = OM.mel_l1_ssim_loss(mel_out, target)
        (LAMBDAS['l1'] * l1 + LAMBDAS['ssim'] * ss).backward()

    def zero_mel():
        mel_out.grad = None
    mel_steps = max(a.steps, 200)
    results.append({'step': 'mel_loss', 'path': 'native', 'ms': round(timeit(mel_native, mel_steps, a.warmup, zero_mel), 4)})
    for tf32 in (True, False):
        torch.backends.cudnn.allow_tf32 = tf32
        results.append({'step': 'mel_loss', 'path': f'eager cudnn tf32={tf32}', 'ms': round(timeit(mel_eager, mel_steps, a.warmup, zero_mel), 4)})
    if a.mel_gan:
        from oracle import multi_window_disc as OD
        mel = SY.make_disc_mel(B, T, [0] + [8 * b for b in range(1, B)], 1234).to(dev).requires_grad_(True)

        def disc_native():
            y = disc(mel)['y']
            F.mse_loss(y, torch.ones_like(y)).backward()

        def disc_eager():
            starts, scales = eager_draws(1, B, T, dev)
            y = OD.disc_forward(dsd, mel, starts[0], scales[0])[0]
            F.mse_loss(y, torch.ones_like(y)).backward()

        def zero_disc():
            mel.grad = None
            disc.zero_grad(set_to_none=True)
            for v in dsd.values():
                v.grad = None
        disc.requires_grad_(True)
        results.append({'step': 'mel_disc', 'path': 'native', 'ms': round(timeit(disc_native, a.steps, a.warmup, zero_disc), 4)})
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            results.append({'step': 'mel_disc', 'path': f'eager cudnn tf32={tf32}', 'ms': round(timeit(disc_eager, a.steps, a.warmup, zero_disc), 4)})
    torch.backends.cudnn.allow_tf32 = True
    step_note = 'reference step with the adversarial terms (phase2: G step + D step)' if a.mel_gan else 'reference step minus the adversarial terms'
    for r in results:
        print(json.dumps(dict(r, B=B, T=T, steps=a.steps, gpu=name, power_limit=power,
                              note=step_note if r['step'] not in ('mel_loss', 'mel_disc') else 'forward + backward')))


if __name__ == '__main__':
    main()

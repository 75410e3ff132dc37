"""ORACLE tooling (test infrastructure only; see oracle/__init__.py): writes the fixtures of the SVB acoustic model's training path
from the UNMODIFIED reference, the same way oracle/gen_golden.py writes the others.

    NEURALSVB_REFERENCE=/path/to/NeuralSVB python -m oracle.gen_golden_train     # mel_loss.npz and svb_vae_train.npz

Inputs and weights are never stored: neuralsvb_b200/utils/synthetic.py regenerates them from the seeds.
"""
import os
import sys
import warnings

import numpy as np
import torch

from neuralsvb_b200.utils import synthetic as S
from oracle import ref_harness as R
from oracle.gen_golden import DISC_GRAD_STRIDE, OUT, SEED, SVB_HPARAMS, _pack_grads

MEL_LOSS_CASES = {
    # name: (B, T, padding frames per clip)   ragged padding with an all-padding clip, T < 11 (the window is wider than the clip), T ~ 1000
    'ragged': (3, 37, (0, 5, 37)),
    'short': (2, 5, (0, 2)),
    'long': (2, 1000, (0, 123)),
}


def _reference_mel_losses():
    """``FastSpeech2Task.l1_loss`` and ``ssim_loss`` (tasks/tts/fs2.py:158-175) as unbound methods of the UNMODIFIED reference class on a
    stand-in ``self`` that only provides ``TtsTask.weights_nonzero_speech`` (tasks/tts/tts.py:127-131).  The task module imports plotting
    and text front-end packages the losses never use; absent ones are replaced by inert stubs."""
    import types

    class _Inert(types.ModuleType):
        def __getattr__(self, k):
            if k.startswith('__'):
                raise AttributeError(k)
            return _Inert(k)

        def __call__(self, *a, **k):
            return _Inert('call')
    R.install()
    for name in ('matplotlib', 'matplotlib.pyplot', 'tensorboardX', 'g2p_en', 'pypinyin'):
        try:
            __import__(name)
        except Exception:
            sys.modules[name] = _Inert(name)
    from tasks.tts.fs2 import FastSpeech2Task
    from tasks.tts.tts import TtsTask
    me = types.SimpleNamespace(weights_nonzero_speech=lambda t: TtsTask.weights_nonzero_speech(None, t))
    return (lambda o, t: FastSpeech2Task.l1_loss(me, o, t)), (lambda o, t: FastSpeech2Task.ssim_loss(me, o, t))


def gen_mel_loss():
    """l1 / ssim (bias 6) of the reference and d(l1)/d mel_out, d(ssim)/d mel_out by reference autograd, float32 on the CPU, for the
    inputs of synthetic.make_mel_pair (MEL_LOSS_CASES).  Gradients stored subsampled with their exact norms (_pack_grads)."""
    l1_fn, ssim_fn = _reference_mel_losses()
    out = {}
    for name, (B, T, pad) in MEL_LOSS_CASES.items():
        mel_out, target = S.make_mel_pair(B, T, pad, SEED)
        res = {}
        for key, fn in (('l1', l1_fn), ('ssim', ssim_fn)):
            x = mel_out.clone().requires_grad_(True)
            loss = fn(x, target)
            loss.backward()
            out[f'{name}/{key}'] = np.float64(loss.detach())
            res[key] = x.grad
        _pack_grads(out, f'{name}/grad', [(k, g) for k, g in res.items()])
        out[f'{name}/params'] = np.array([B, T] + list(pad), np.int64)
    np.savez_compressed(os.path.join(OUT, 'mel_loss.npz'), **out)
    print('mel_loss.npz', {k: float(v) for k, v in out.items() if k.endswith(('/l1', '/ssim'))})


SVB_TRAIN_RUNNING = ['upsample_layer.0.3', 'vae_model.encoder.poolings.2', 'vae_model.encoder.poolings.5']


def gen_svb_vae_train():
    """One phase-2 (generator) and one phase-3 (mapping function) step of the reference MleSVBVAE (svb_vae.py:251-312) with the
    requires_grad / train / eval flags SVBVAEMleTask and the trainer set (tasks/singing/svb_vae_task.py:543-676, vc_asr frozen and in
    eval mode), posterior noise replaced by zeros, the synthetic state_dict with weight norm live, batch make_svb_batch(2, 96, 120)
    (its last clips end in pitch-0 frames).  Loss terms are the task's (lambda_kl 0.001, lambda_mle 1, ssim:0.5|l1:0.5) without the
    adversarial ones.  Stored: the weighted loss terms, strided parameter gradients (_pack_grads) plus pitch_embed's row-0 gradient,
    BatchNorm running statistics after each step."""
    l1_fn, ssim_fn = _reference_mel_losses()
    from utils.hparams import hparams
    hparams.update(SVB_HPARAMS)
    from modules.voice_conversion.svb_vae import MleSVBVAE
    batch = S.make_svb_batch(2, 96, 120, SEED)
    targets = {'a2a': batch['amateur_mel'], 'p2p': batch['prof_mel'], 'a2p': batch['prof_mel']}
    out = {}
    for phase, ways in ((2, ['a2a', 'p2p']), (3, ['a2a', 'p2p', 'a2p'])):
        torch.manual_seed(SEED)
        m = MleSVBVAE(80)
        res = m.load_state_dict(S.make_svb_state_dict(SEED), strict=False)
        assert not res.unexpected_keys
        for n, p in m.named_parameters():
            p.requires_grad_(('z_mapping_function' in n) if phase == 3 else ('vc_asr' not in n and 'z_mapping_function' not in n))
        if phase == 2:
            m.train()
            m.z_mapping_function.eval()
        else:
            m.eval()
            m.z_mapping_function.train()
        m.vc_asr.eval()
        orig = torch.randn_like
        torch.randn_like = lambda t, **k: torch.zeros_like(t)
        try:
            ret = m(**batch, infer=False, concurrent_ways=ways)
        finally:
            torch.randn_like = orig
        losses = {}
        for way in ways:
            if 'kl' in ret[way]:
                losses[f'{way}_kl'] = ret[way]['kl'] * 0.001
            losses[f'ssim{way}'] = ssim_fn(ret[way]['mel_out'], targets[way]) * 0.5
            losses[f'l1{way}'] = l1_fn(ret[way]['mel_out'], targets[way]) * 0.5
        if phase == 3:
            losses['a2p_mle'] = ret['a2p']['mle'] * 1.0
        sum(losses.values()).backward()
        for k, v in losses.items():
            out[f'p{phase}/loss/{k}'] = np.float64(v.detach())
        grads = [(n, p.grad) for n, p in m.named_parameters() if p.requires_grad]
        _pack_grads(out, f'p{phase}/grad', grads, DISC_GRAD_STRIDE)
        out[f'p{phase}/grad_names'] = np.array([n for n, _ in grads])
        if phase == 2:
            out['p2/pitch_embed_row0'] = m.pitch_embed.weight.grad[0].numpy()
        bns = SVB_TRAIN_RUNNING if phase == 2 else ['z_mapping_function.convs.1', 'z_mapping_function.convs.4']
        sd = m.state_dict()
        for pre in bns:
            for s in ('running_mean', 'running_var', 'num_batches_tracked'):
                out[f'p{phase}/{pre}.{s}'] = sd[f'{pre}.{s}'].numpy()
    np.savez_compressed(os.path.join(OUT, 'svb_vae_train.npz'), **out)
    print('svb_vae_train.npz', {k: float(v) for k, v in out.items() if '/loss/' in k})


def main():
    if not R.available():
        sys.exit('gen_golden_train needs NEURALSVB_REFERENCE = a checkout of the reference NeuralSVB')
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    warnings.simplefilter('ignore')
    for w in sys.argv[1:] or ['mel_loss', 'svb_vae_train']:
        globals()[f'gen_{w}']()


if __name__ == '__main__':
    main()

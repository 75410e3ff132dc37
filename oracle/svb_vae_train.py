"""ORACLE (test infrastructure only; see oracle/__init__.py): torch restatement of the two optimizer steps of SVBVAEMleTask
(tasks/singing/svb_vae_task.py:543-676 of the reference) without the adversarial terms -- phase 2 (generator: ways a2a + p2p, everything
but the latent map in train mode) and phase 3 (mapping function: ways a2a + p2p + a2p, the model in eval mode, the latent map in train
mode) -- built on the eval-mode pieces of oracle/svb_vae.py with train-mode BatchNorm (batch statistics, running statistics updated in
place), the pitch embedding's padding_idx 0 and the PPG detached.  ``w`` is the state_dict with weight_g / weight_v pairs (autograd
leaves where the caller wants gradients).  Runs in the dtype of its inputs.

Three optional inputs let a test hold the reference to values the model under test computed without changing the gradient graph:
``ppg`` replaces the PPG extractor's output (detached in the reference, so it only enters as data); ``tie(name, x)`` is applied
to the input of every BatchNorm, named by its state_dict prefix (a straight-through substitution keeps its forward values on the
tested model's and its gradient on ``x``); ``relu(name, x)`` replaces each ReLU, named by the layer whose output it takes
(``pitch_encoder.conv.{i}.norm``, ``upsample_layer.0.1``, ``vae_model.encoder.poolings.{0,3}``, ``z_mapping_function.convs.{1,4}``),
so that it can apply the tested model's ReLU masks: a pre-activation within rounding of zero otherwise takes a different branch
on each side and moves its element's gradient by its whole share.  Pinned by tests/golden/svb_vae_train.npz, which
oracle/gen_golden_train.py writes from the UNMODIFIED reference class."""
import torch
import torch.nn.functional as F

from oracle import fs2_vae as OF
from oracle import vc_asr as OV
from oracle.svb_vae import _cond_sum, _sub, conv_stacks

LAMBDA_KL, LAMBDA_MLE, LAMBDA_L1, LAMBDA_SSIM = 0.001, 1.0, 0.5, 0.5       # vae_global_mle_eng: lambda_kl, lambda_mle, ssim:0.5|l1:0.5


def _bn(w, pre, x, train, tie=None, name=None):
    if tie is not None:
        x = tie(name or pre, x)
    return F.batch_norm(x, w[pre + '.running_mean'], w[pre + '.running_var'], w[pre + '.weight'], w[pre + '.bias'], train, 0.1, 1e-5)


def _relu(relu, name, x):
    return torch.relu(x) if relu is None else relu(name, x)


def prepare_condition_train(w, mel, pitch, spk, bn_train, ppg=None, tie=None, relu=None):
    """prepare_condition with Embedding(300, H, padding_idx=0), the PPG detached (svb_vae.py:68) and upsample_layer's BatchNorm in train
    mode when ``bn_train``.  ``ppg`` [B, T / 2, H]: the PPG extractor's output to use instead of computing it."""
    T = pitch.shape[1]
    h_pitch = conv_stacks(w, 'pitch_encoder', F.embedding(pitch, w['pitch_embed.weight'], padding_idx=0), relu=relu)
    if ppg is None:
        with torch.device(mel.device):                   # oracle/vc_asr.py builds its position table with the default device
            ppg = OV.vc_asr_h_content(_sub(w, 'vc_asr.'), mel)
    h = ppg.to(mel.dtype).detach().transpose(1, 2)
    h = _relu(relu, 'upsample_layer.0.1', F.conv1d(F.interpolate(h, scale_factor=2, mode='nearest'), w['upsample_layer.0.1.weight'],
                                                   w['upsample_layer.0.1.bias'], padding=2))
    h = F.conv1d(_bn(w, 'upsample_layer.0.3', h, bn_train, tie), w['upsample_layer.1.weight'], w['upsample_layer.1.bias'], padding=2)
    h_style = F.linear(spk, w['spk_embed_proj.weight'], w['spk_embed_proj.bias'])[:, None, :].repeat(1, T, 1)
    return dict(h_pitch=h_pitch, h_content=h.transpose(1, 2)[:, :mel.shape[1]], h_style=h_style,
                tgt_nonpadding=(pitch > 0).to(mel.dtype)[:, :, None])


def normal_vae_train(w, mel, c, eps, bn_train, H=192, lat=128, K=5, Le=8, Ld=4, tie=None, relu=None):
    """normal_vae(infer=False) with the posterior encoder's BatchNorms in train mode when ``bn_train``."""
    g = _cond_sum(w, [c['h_pitch'], c['h_content'], c['h_style']])
    mask = c['tgt_nonpadding'].transpose(1, 2)
    v = _sub(w, 'vae_model.')
    e = _sub(v, 'encoder.')
    g_sqz = F.conv1d(g, v['g_pre_net.0.weight'], v['g_pre_net.0.bias'], stride=4, padding=2)
    h = F.conv1d(mel.transpose(1, 2), e['pre_net.0.weight'], e['pre_net.0.bias'], stride=4, padding=2)
    xm = mask[:, :, ::4][:, :, :h.shape[-1]]
    h = OF.wn_forward(_sub(e, 'wn.'), H, K, 1, Le, h * xm, xm, g_sqz) * xm
    h = F.conv1d(h, e['out_proj.weight'], e['out_proj.bias'])
    for i in (0, 3):
        h = _relu(relu, f'vae_model.encoder.poolings.{i}', F.conv1d(h, e[f'poolings.{i}.weight'], e[f'poolings.{i}.bias'], stride=2))
        h = _bn(e, f'poolings.{i + 2}', h, bn_train, tie, f'vae_model.encoder.poolings.{i + 2}')
    h = F.conv1d(h, e['poolings.6.weight'], e['poolings.6.bias'], stride=2).mean(-1, keepdim=True)
    m_q, logs_q = torch.split(h, lat, dim=1)
    z_q = m_q + eps * torch.exp(logs_q)
    x_recon = OF.fvae_decoder_forward(_sub(v, 'decoder.'), H, K, Ld, 4, z_q, mask, g, True)
    kl = torch.distributions.kl_divergence(torch.distributions.Normal(m_q, logs_q.exp()), torch.distributions.Normal(0.0, 1.0))
    return dict(mel_out=x_recon.transpose(1, 2), kl=(kl * xm).sum() / xm.sum() / lat, m_q=m_q, logs_q=logs_q, z_q=z_q)


def latent_map_train(w, pre, x, spk_emb, bn_train, tie=None, relu=None):
    """GlobalLatentMap.forward with its BatchNorms on [B, latent, 1] in train mode when ``bn_train``."""
    s = F.conv1d(spk_emb[:, :, :x.shape[-1]], w[pre + '.spk_proj.0.weight'], w[pre + '.spk_proj.0.bias'])
    x = x + F.conv1d(_relu(relu, pre + '.spk_proj.0', s), w[pre + '.spk_proj.2.weight'], w[pre + '.spk_proj.2.bias'])
    for i in (0, 3):
        x = _relu(relu, f'{pre}.convs.{i + 1}', _bn(w, f'{pre}.convs.{i + 1}', F.conv1d(x, w[f'{pre}.convs.{i}.weight'], w[f'{pre}.convs.{i}.bias']),
                                                    bn_train, tie))
    return F.conv1d(x, w[pre + '.convs.6.weight'], w[pre + '.convs.6.bias'])


def svb_train_losses(w, batch, eps, phase, ppg=None, tie=None, relu=None):
    """The weighted loss terms of one phase-2 (generator) or phase-3 (mapping) step, keyed as the task logs them
    (``{way}_kl``, ``l1{way}``, ``ssim{way}``, ``a2p_mle``), the mel loss from oracle/mel_loss.py.  Sum them for the step's loss.
    ``ppg``: {'amateur': ..., 'prof': ...} PPG extractor outputs to use; ``tie``, ``relu``: see the module docstring."""
    from oracle import mel_loss as OM
    wf = OF.fold_weight_norm(w)
    gen_train = phase == 2
    ppg = ppg or {}
    ac = prepare_condition_train(wf, batch['amateur_mel'], batch['amateur_pitch'], batch['amateur_spk_id'], gen_train, ppg.get('amateur'), tie,
                                 relu)
    pc = prepare_condition_train(wf, batch['prof_mel'], batch['prof_pitch'], batch['prof_spk_id'], gen_train, ppg.get('prof'), tie, relu)
    out = {'a2a': normal_vae_train(wf, batch['amateur_mel'], ac, eps, gen_train, tie=tie, relu=relu),
           'p2p': normal_vae_train(wf, batch['prof_mel'], pc, eps, gen_train, tie=tie, relu=relu)}
    targets = {'a2a': batch['amateur_mel'], 'p2p': batch['prof_mel'], 'a2p': batch['prof_mel']}
    losses = {}
    if phase == 3:
        a2a, p2p = out['a2a'], out['p2p']
        mapped = latent_map_train(wf, 'z_mapping_function', a2a['z_q'], ac['h_style'].transpose(1, 2), True, tie, relu)
        mle = -torch.distributions.Normal(p2p['m_q'], p2p['logs_q'].exp()).log_prob(mapped).sum() / mapped.shape[0] / mapped.shape[1]
        H = ac['h_content'].shape[-1]
        align = batch['a2p_alignment'][:, :, None].repeat(1, 1, H)
        g = _cond_sum(wf, [pc['h_pitch'], torch.gather(ac['h_content'], 1, align), ac['h_style'][:, :1, :].repeat(1, pc['h_pitch'].shape[1], 1)])
        mel = OF.fvae_decoder_forward(_sub(wf, 'vae_model.decoder.'), 192, 5, 4, 4, mapped, pc['tgt_nonpadding'].transpose(1, 2), g, True)
        out['a2p'] = dict(mel_out=mel.transpose(1, 2))
        losses['a2p_mle'] = mle * LAMBDA_MLE
    for way, o in out.items():
        if 'kl' in o:
            losses[f'{way}_kl'] = o['kl'] * LAMBDA_KL
        l1, ss = OM.mel_l1_ssim_loss(o['mel_out'], targets[way])
        losses[f'l1{way}'], losses[f'ssim{way}'] = l1 * LAMBDA_L1, ss * LAMBDA_SSIM
    return losses, out

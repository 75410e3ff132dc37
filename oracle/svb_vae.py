"""ORACLE (test infrastructure only; see oracle/__init__.py): torch-CPU restatement of the SVB acoustic model's forward
(``MleSVBVAE.forward(..., infer=False, concurrent_ways=['a2a', 'p2p', 'a2p'])``, modules/voice_conversion/svb_vae.py:57-84,155-165,
258-312 of the reference) in eval mode, composed from oracle/vc_asr.py (PPG extractor) and oracle/fs2_vae.py (GlobalFVAE).  Pinned by
tests/golden/svb_vae.npz, which oracle/gen_golden.py writes from the UNMODIFIED reference class."""
import torch
import torch.nn.functional as F

from oracle import fs2_vae as OF
from oracle import vc_asr as OV


def _sub(w, prefix):
    return {k[len(prefix):]: v for k, v in w.items() if k.startswith(prefix)}


def conv_stacks(w, pre, x, n_layers=3, relu=None):
    """ConvStacks (modules/commons/common_layers.py:672-707) with ConvBlock norm 'gn' (:739-773), res=True.  x [B, T, H].
    ``relu(name, x)``, when given, replaces the ReLU on the output of the GroupNorm ``name`` (see oracle/svb_vae_train.py)."""
    x = F.linear(x, w[pre + '.in_proj.weight'], w[pre + '.in_proj.bias']).transpose(1, 2)
    for i in range(n_layers):
        h = F.conv1d(x, w[f'{pre}.conv.{i}.conv.conv.weight'], w[f'{pre}.conv.{i}.conv.conv.bias'], padding=2)
        h = F.group_norm(h, h.shape[1] // 16, w[f'{pre}.conv.{i}.norm.weight'], w[f'{pre}.conv.{i}.norm.bias'], 1e-5)
        x = x + (torch.relu(h) if relu is None else relu(f'{pre}.conv.{i}.norm', h))
    return F.linear(x.transpose(1, 2), w[pre + '.out_proj.weight'], w[pre + '.out_proj.bias'])


def prepare_condition(w, mel, pitch, spk):
    """SVBVAE.prepare_condition (svb_vae.py:57-84)."""
    T = pitch.shape[1]
    h_pitch = conv_stacks(w, 'pitch_encoder', F.embedding(pitch, w['pitch_embed.weight']))
    h = OV.vc_asr_h_content(_sub(w, 'vc_asr.'), mel).transpose(1, 2)
    h = F.interpolate(h, scale_factor=2, mode='nearest')                                            # upsample_layer[0]: Upsample, Conv, ReLU, BN
    h = torch.relu(F.conv1d(h, w['upsample_layer.0.1.weight'], w['upsample_layer.0.1.bias'], padding=2))
    h = F.batch_norm(h, w['upsample_layer.0.3.running_mean'], w['upsample_layer.0.3.running_var'], w['upsample_layer.0.3.weight'],
                     w['upsample_layer.0.3.bias'], False, 0.0, 1e-5)
    h = F.conv1d(h, w['upsample_layer.1.weight'], w['upsample_layer.1.bias'], padding=2)
    h_content = h.transpose(1, 2)[:, :mel.shape[1]]
    h_style = F.linear(spk, w['spk_embed_proj.weight'], w['spk_embed_proj.bias'])[:, None, :].repeat(1, T, 1)
    return dict(h_pitch=h_pitch, h_content=h_content, h_style=h_style, tgt_nonpadding=(pitch > 0).float()[:, :, None])


def _cond_sum(w, parts):
    return F.linear(torch.cat(parts, -1), w['encoded_embed_proj.weight'], w['encoded_embed_proj.bias']).transpose(1, 2)


def normal_vae(w, vae_w, mel, c, eps):
    """SVBVAE.normal_vae (svb_vae.py:155-165), infer=False."""
    g = _cond_sum(w, [c['h_pitch'], c['h_content'], c['h_style']])
    x_recon, kl, m_q, logs_q = OF.global_fvae_forward(vae_w, 80, 192, 128, 5, 8, 4, 4, mel.transpose(1, 2), c['tgt_nonpadding'].transpose(1, 2), g, eps)
    return dict(mel_out=x_recon.transpose(1, 2), kl=kl, m_q=m_q, logs_q=logs_q, z_q=m_q + eps * torch.exp(logs_q))


def latent_map(w, pre, x, spk_emb):
    """GlobalLatentMap.forward (vae_models.py:149-172) in eval mode."""
    s = F.conv1d(spk_emb[:, :, :x.shape[-1]], w[pre + '.spk_proj.0.weight'], w[pre + '.spk_proj.0.bias'])
    x = x + F.conv1d(torch.relu(s), w[pre + '.spk_proj.2.weight'], w[pre + '.spk_proj.2.bias'])
    for i in (0, 3):
        x = F.conv1d(x, w[f'{pre}.convs.{i}.weight'], w[f'{pre}.convs.{i}.bias'])
        j = i + 1
        x = torch.relu(F.batch_norm(x, w[f'{pre}.convs.{j}.running_mean'], w[f'{pre}.convs.{j}.running_var'], w[f'{pre}.convs.{j}.weight'],
                                    w[f'{pre}.convs.{j}.bias'], False, 0.0, 1e-5))
    return F.conv1d(x, w[pre + '.convs.6.weight'], w[pre + '.convs.6.bias'])


def mle_svb_vae_forward(w, batch, eps=None):
    """MleSVBVAE.forward(infer=False, concurrent_ways=['a2a', 'p2p', 'a2p']) (svb_vae.py:258-312); ``eps`` = posterior noise [B, 128, 1]."""
    w = OF.fold_weight_norm(w)
    vae_w = _sub(w, 'vae_model.')
    B = batch['amateur_mel'].shape[0]
    eps = torch.zeros(B, 128, 1) if eps is None else eps
    ac = prepare_condition(w, batch['amateur_mel'], batch['amateur_pitch'], batch['amateur_spk_id'])
    pc = prepare_condition(w, batch['prof_mel'], batch['prof_pitch'], batch['prof_spk_id'])
    a2a = normal_vae(w, vae_w, batch['amateur_mel'], ac, eps)
    p2p = normal_vae(w, vae_w, batch['prof_mel'], pc, eps)
    H = ac['h_content'].shape[-1]
    mapped = latent_map(w, 'z_mapping_function', a2a['z_q'], ac['h_style'].transpose(1, 2))
    mle = -torch.distributions.Normal(p2p['m_q'], p2p['logs_q'].exp()).log_prob(mapped).sum() / mapped.shape[0] / mapped.shape[1]
    align = batch['a2p_alignment'][:, :, None].repeat(1, 1, H)
    g = _cond_sum(w, [pc['h_pitch'], torch.gather(ac['h_content'], 1, align), ac['h_style'][:, :1, :].repeat(1, pc['h_pitch'].shape[1], 1)])
    dec_w = _sub(vae_w, 'decoder.')
    mel = OF.fvae_decoder_forward(dec_w, 192, 5, 4, 4, mapped, pc['tgt_nonpadding'].transpose(1, 2), g, True).transpose(1, 2)
    return dict(a2a=a2a, p2p=p2p, a2p=dict(mel_out=mel, mle=mle))

"""The SVB acoustic model (SURVEY 8(f) N1, BASELINE cfg 5's middle step): drop-in for the reference's ``MleSVBVAE``
(``modules/voice_conversion/svb_vae.py:13-56,178-199,251-312``) on the inference / evaluation path the SVB task takes
(``forward(..., infer=False, concurrent_ways=['a2a', 'p2p', 'a2p'])``, ``tasks/singing/svb_vae_task.py:120-150,303-305``):

    conditions   pitch_embed -> pitch_encoder (ConvStacks) ; vc_asr (PPG extractor) -> upsample_layer ; spk_embed_proj
    a2a / p2p    encoded_embed_proj -> GlobalFVAE (posterior encoder + mel decoder + KL)
    a2p          z_mapping_function (GlobalLatentMap) -> decoder with the professional pitch / aligned amateur content -> mel_out

Same constructor (``dict_size`` + hparams) and ``state_dict`` names as the reference.  Every Conv1d / Linear runs as a native kernel
(``svb_conv_nct_forward``; the WN stacks and the PPG extractor through their own entry points, see ``modules/fastspeech/fs2_vae.py`` and
``vc_modules.py``); embedding lookup, GroupNorm / BatchNorm(eval) affine maps, nearest up-sampling, gathers and concatenations are torch
ops on the same device tensors.

Training is opt-in: ``MleSVBVAE(..., trainable=True)`` makes the generator and the latent map differentiable (the phase-2 generator
step and the phase-3 mapping step of ``SVBVAEMleTask``, tasks/singing/svb_vae_task.py:543-676).  Every convolution then runs as an
autograd node with a native backward (``_conv`` -> ``_TcConvFn`` / ``_ConvNctFn``, the GlobalFVAE through ``_WNTrainFn`` /
``_FVAEDecTrainFn``); the BatchNorms of ``upsample_layer`` and of the latent map use batch statistics in ``train()`` mode and update
their running statistics as ``nn.BatchNorm1d`` does; ``vc_asr`` always runs without grad (the reference ``.detach()``es its output).
The mel reconstruction loss is ``neuralsvb_b200.modules.commons.mel_loss.mel_l1_ssim_loss``; the task that drives the steps
(single GPU or data parallel) is ``neuralsvb_b200.tasks.singing.svb_vae_task.SVBVAEMleTask``."""
import ctypes
import numbers

import torch
import torch.nn.functional as F
from torch import nn

from neuralsvb_b200 import _native
from neuralsvb_b200.modules.fastspeech.fs2_vae import GlobalFVAE, check_frames
from neuralsvb_b200.modules.voice_conversion.vc_modules import VCASR, FrameLens, _bn_affine, _conv, _Holder


def frame_counts(L, mel_strides, stride=4):
    """A clip's frame count at every resolution MleSVBVAE computes at, for a clip of L mel frames: 'mel' L; 'ppg' the PPG extractor's
    (the mel prenet's k = 5, pad 2 convolutions at mel_strides); 'enc' the posterior encoder's and g_pre_net's (k = 2 stride,
    pad stride / 2); 'pool' the three valid k = 3 stride-2 poolings after it."""
    ppg = L
    for s in mel_strides:
        ppg = (ppg - 1) // s + 1
    enc = (L + 2 * (stride // 2) - 2 * stride) // stride + 1
    pool, n = [], enc
    for _ in range(3):
        n = (n - 3) // 2 + 1
        pool.append(n)
    return {'mel': L, 'ppg': ppg, 'enc': enc, 'pool': tuple(pool)}


def _linear_btc(x, lin, lens=None):
    """nn.Linear on [B, T, C] as a native 1x1 convolution on [B, C, T]."""
    return _conv(x.transpose(1, 2).contiguous(), lin.weight, lin.bias, lens=lens).transpose(1, 2)


def _bn_train(m):
    """Batch-statistics BatchNorm (running statistics updated, as nn.BatchNorm1d in train mode) for a trainable module in training."""
    return m.trainable and m.training and torch.is_grad_enabled()


class _ConvStacks(nn.Module):
    """Parameter names of ``ConvStacks`` / ``ConvBlock(norm='gn')`` (modules/commons/common_layers.py:672-707,739-773)."""

    def __init__(self, H, n_layers=3, K=5):
        super().__init__()
        self.K = K
        self.in_proj = nn.Linear(H, H)
        self.conv = nn.ModuleList()
        for _ in range(n_layers):
            blk, cn = _Holder(), _Holder()
            cn.conv = nn.Conv1d(H, H, K, padding=K // 2)
            blk.conv, blk.norm = cn, nn.GroupNorm(H // 16, H)
            self.conv.append(blk)
        self.out_proj = nn.Linear(H, H)

    def forward(self, x, lens=None):
        x = _conv(x.transpose(1, 2).contiguous(), self.in_proj.weight, self.in_proj.bias, lens=lens)
        for blk in self.conv:
            h = _conv(x, blk.conv.conv.weight, blk.conv.conv.bias, K=self.K, pad=self.K // 2, lens=lens)
            if lens is None:
                x = x + torch.relu(blk.norm(h))                     # nn.GroupNorm: F.group_norm with its parameters
            else:                                                   # statistics over each clip's own frames
                n = blk.norm
                y = torch.empty_like(h)
                _native.check(_native.lib().svb_group_norm_relu_add_ragged(
                    _native.ptr(x), _native.ptr(h), _native.ptr(n.weight), _native.ptr(n.bias), h.shape[0], h.shape[1], h.shape[2],
                    n.num_groups, ctypes.c_float(n.eps), lens.c_host, _native.ptr(lens.dev), _native.ptr(y),
                    _native.current_stream_ptr(h.device)), 'group_norm_relu_add_ragged')
                x = y
        return _conv(x.contiguous(), self.out_proj.weight, self.out_proj.bias, lens=lens).transpose(1, 2)


class _GlobalLatentMap(nn.Module):
    """``GlobalLatentMap`` (modules/voice_conversion/vae_models.py:149-172): 1x1 convs on the [B, latent, 1] latent, eval-mode BatchNorm
    (batch statistics in ``train()`` mode with grad enabled when ``trainable``)."""

    def __init__(self, latent, trainable=False):
        super().__init__()
        self.trainable = trainable
        self.convs = nn.Sequential(nn.Conv1d(latent, latent, 1), nn.BatchNorm1d(latent), nn.ReLU(), nn.Conv1d(latent, latent, 1),
                                   nn.BatchNorm1d(latent), nn.ReLU(), nn.Conv1d(latent, latent, 1))
        self.spk_proj = nn.Sequential(nn.Conv1d(256, latent, 1), nn.ReLU(), nn.Conv1d(latent, latent, 1))

    def forward(self, x, spk_emb):
        s = spk_emb[:, :, :x.shape[-1]].contiguous()
        s = _conv(_conv(s, self.spk_proj[0].weight, self.spk_proj[0].bias, relu=True), self.spk_proj[2].weight, self.spk_proj[2].bias)
        x = (x + s).contiguous()
        c = self.convs
        bn = (lambda m, y: m(y)) if _bn_train(self) else _bn_affine
        x = torch.relu(bn(c[1], _conv(x, c[0].weight, c[0].bias))).contiguous()
        x = torch.relu(bn(c[4], _conv(x, c[3].weight, c[3].bias))).contiguous()
        return _conv(x, c[6].weight, c[6].bias)


class MleSVBVAE(nn.Module):
    def __init__(self, dict_size=None, hp=None, precision='bf16x3', trainable=False):
        super().__init__()
        self.trainable = bool(trainable)
        if hp is None:
            from neuralsvb_b200.utils.hparams import hparams as hp
        H = self.hidden_size = hp['hidden_size']
        self.c_content = self.c_out = hp['audio_num_mel_bins']
        self.vae_model = GlobalFVAE(self.c_content, hp['fvae_enc_dec_hidden'], hp['latent_size'], hp['fvae_kernel_size'],
                                    hp['fvae_enc_n_layers'], hp['fvae_dec_n_layers'], H, [4], False, precision=precision,
                                    trainable=self.trainable)
        self.pitch_embed = nn.Embedding(300, H, 0)
        self.pitch_encoder = _ConvStacks(H, 3)
        self.vc_asr = VCASR(dict_size, self.c_content, hidden_size=H, asr_enc_layers=hp['asr_enc_layers'], mel_strides=hp['mel_strides'],
                            asr_last_norm=hp.get('asr_last_norm', True))
        self.mel_strides = list(hp['mel_strides'])
        self.upsample_layer = nn.Sequential(*([nn.Sequential(nn.Upsample(scale_factor=s, mode='nearest'), nn.Conv1d(H, H, s * 2 + 1, padding=s),
                                                            nn.ReLU(), nn.BatchNorm1d(H)) for s in self.mel_strides if s > 1] +
                                              [nn.Conv1d(H, H, 5, padding=2)]))
        self.spk_embed_proj = nn.Linear(256, H)
        self.encoded_embed_proj = nn.Linear(3 * H, H)
        self.z_mapping_function = _GlobalLatentMap(hp['latent_size'], self.trainable)

    def load_state_dict(self, state_dict, strict=True):
        sd = {k: v for k, v in state_dict.items() if not k.startswith(('vc_asr.asr_decoder.', 'vc_asr.token_embed.'))}
        return super().load_state_dict(sd, strict=strict)

    def prepare_condition(self, mels_content=None, pitch=None, spk_ids=None, lens=None):
        """svb_vae.py:57-84.  ``lens``: the clips' mel frame counts (checked as forward checks them), for the length-aware mode:
        every condition computed from its clip's own frames, ``tgt_nonpadding`` from the lengths."""
        T = pitch.shape[1]
        if lens is not None and not isinstance(lens, FrameLens):
            lens = FrameLens(self._check_lens('lens', lens, pitch.shape[0], T), pitch.device)
        # padding_idx 0 as the reference's Embedding(300, H, 0): unvoiced / padding frames (pitch 0) give row 0 no gradient
        h_pitch = self.pitch_encoder(F.embedding(pitch, self.pitch_embed.weight, padding_idx=0), lens)
        with torch.no_grad():                                       # the reference detaches h_content (svb_vae.py:68)
            h = self.vc_asr(mels_content, lens=lens)['h_content'].transpose(1, 2)
        bn = (lambda m, y: m(y)) if _bn_train(self) else _bn_affine
        up = None if lens is None else lens.map(lambda n: frame_counts(n, self.mel_strides)['ppg'])
        for m in self.upsample_layer:
            if isinstance(m, nn.Sequential):                        # Upsample(nearest) -> Conv1d -> ReLU -> BatchNorm1d
                s = int(m[0].scale_factor)
                up = None if up is None else up.map(lambda n: n * s)
                h = bn(m[3], _conv(h.repeat_interleave(s, dim=2).contiguous(), m[1].weight, m[1].bias, K=2 * s + 1, pad=s, relu=True,
                                   lens=up))
            else:
                h = _conv(h.contiguous(), m.weight, m.bias, K=5, pad=2, lens=up)
        h_content = h.transpose(1, 2)[:, :mels_content.shape[1]]
        h_style = _linear_btc(spk_ids[:, None, :].float(), self.spk_embed_proj).repeat(1, T, 1)
        nonpad = (pitch > 0).float() if lens is None else lens.mask(T)
        return {'h_pitch': h_pitch, 'h_content': h_content, 'h_style': h_style, 'tgt_nonpadding': nonpad[:, :, None]}

    def _cond_sum(self, parts, lens=None):
        return _linear_btc(torch.cat(parts, -1), self.encoded_embed_proj, lens).transpose(1, 2).contiguous()

    def _check_lens(self, name, lens, B, T):
        """Per-clip frame counts of the length-aware mode, checked on the host before any launch: B ints, each a frame count the
        GlobalFVAE takes (check_frames: a multiple of frames_multiple, >= 60) within the batch's T frames."""
        if torch.is_tensor(lens):
            lens = lens.tolist()
        lens = list(lens)
        if len(lens) != B:
            raise ValueError(f'{name}: {len(lens)} frame counts for a batch of {B} clips')
        for b, n in enumerate(lens):
            if isinstance(n, bool) or not isinstance(n, numbers.Integral):
                raise ValueError(f'{name}[{b}] = {n!r}: a frame count is an int')
            if not 0 < n <= T:
                raise ValueError(f'{name}[{b}] = {n}: clip {b} must have 1 to {T} frames (the batch\'s padded length)')
            try:
                check_frames(int(n), self.vae_model.strides[0])
            except ValueError as e:
                raise ValueError(f'{name}[{b}]: clip {b}: {e}') from None
        return [int(n) for n in lens]

    def normal_vae(self, tgt_mel, pitch_cond, content_cond, timbre_cond, padding_cond, infer, eps=None, lens=None):
        """svb_vae.py:155-165 (infer=False: the branch the SVB task uses for validation and test as well)."""
        if infer:
            raise NotImplementedError('normal_vae(infer=True) samples a [B, latent, T / 4] prior that the reference GlobalFVAEDecoder cannot '
                                      'consume (vae_models.py:120-122); the SVB task always calls it with infer=False')
        g = self._cond_sum([pitch_cond, content_cond, timbre_cond], lens)
        x_recon, kl, z_p, m_q, logs_q, x_mask_sqz, z_q = self.vae_model(tgt_mel.transpose(1, 2).contiguous(), padding_cond.transpose(1, 2), g, eps=eps,
                                                                         lens=lens)
        return {'mel_out': x_recon.transpose(1, 2), 'kl': kl, 'z_p': z_p, 'm_q': m_q, 'logs_q': logs_q, 'x_mask_sqz': x_mask_sqz, 'z_q': z_q}

    def forward(self, amateur_mel=None, prof_mel=None, amateur_pitch=None, prof_pitch=None, amateur_spk_id=None, prof_spk_id=None,
                a2p_alignment=None, p2a_alignment=None, infer=False, disable_map=False, eps=None, amateur_lens=None, prof_lens=None,
                **kwargs):
        """svb_vae.py:258-312.  ``eps`` [B, latent, 1] replaces the posterior noise (parity tests); default torch.randn_like.

        ``amateur_lens`` / ``prof_lens`` (both or neither; inference only): each clip's frame count in its row of amateur_mel /
        prof_mel.  Every clip is then computed from its own frames only, as the reference computes that clip alone and unpadded
        (batch size 1): its conditions, mels and latent statistics are the same bits in any batch, at any row, at any padded length
        and whatever the padding holds.  Frames past a clip's length are not part of the result; ``kl`` and ``mle`` stay batch
        means.  Without them (the default) the clips share the padded batch as the task's collated batches do."""
        if torch.is_grad_enabled() and self.training and not self.trainable:
            raise RuntimeError('neuralsvb_b200 MleSVBVAE is inference only: call .eval() and run under torch.no_grad()')
        if (amateur_lens is None) != (prof_lens is None):
            raise ValueError('MleSVBVAE: pass both amateur_lens and prof_lens, or neither')
        if amateur_lens is not None and self.training and torch.is_grad_enabled():
            raise RuntimeError('MleSVBVAE(amateur_lens=..., prof_lens=...) is inference only: call .eval() and run under '
                               'torch.no_grad()')
        if self.trainable and not amateur_mel.is_cuda:
            raise RuntimeError('neuralsvb_b200 has no CPU path: move the module and its inputs to a CUDA device')
        for mel in (amateur_mel, prof_mel):                         # before any launch: both clips go through the GlobalFVAE
            check_frames(mel.shape[1], self.vae_model.strides[0])
        la = lp = None
        if amateur_lens is not None:
            la = FrameLens(self._check_lens('amateur_lens', amateur_lens, amateur_mel.shape[0], amateur_mel.shape[1]), amateur_mel.device)
            lp = FrameLens(self._check_lens('prof_lens', prof_lens, prof_mel.shape[0], prof_mel.shape[1]), prof_mel.device)
        ways = kwargs['concurrent_ways']
        ret = {}
        ac = self.prepare_condition(amateur_mel, amateur_pitch, spk_ids=amateur_spk_id, lens=la)
        pc = self.prepare_condition(prof_mel, prof_pitch, spk_ids=prof_spk_id, lens=lp)
        if 'a2a' in ways:
            a2a = ret['a2a'] = self.normal_vae(amateur_mel, ac['h_pitch'], ac['h_content'], ac['h_style'], ac['tgt_nonpadding'], infer, eps,
                                               lens=la)
        if 'p2p' in ways:
            p2p = ret['p2p'] = self.normal_vae(prof_mel, pc['h_pitch'], pc['h_content'], pc['h_style'], pc['tgt_nonpadding'], infer, eps,
                                               lens=lp)
        if 'a2p' in ways:
            z = a2a['z_q']
            mapped = z if disable_map else self.z_mapping_function(z, ac['h_style'].transpose(1, 2))
            prof = torch.distributions.Normal(p2p['m_q'], p2p['logs_q'].exp(), validate_args=False)      # no host sync
            out = {'mle': -prof.log_prob(mapped).sum() / mapped.shape[0] / mapped.shape[1]}
            align = a2p_alignment[:, :, None].repeat(1, 1, self.hidden_size)
            g = self._cond_sum([pc['h_pitch'], torch.gather(ac['h_content'], 1, align),
                                ac['h_style'][:, :1, :].repeat(1, pc['h_pitch'].shape[1], 1)], lp)
            out['mel_out'] = self.vae_model.decoder(mapped.contiguous(), pc['tgt_nonpadding'].transpose(1, 2), g).transpose(1, 2)
            out['logs_amateur_zq'], out['logs_prof_zq'] = a2a['z_q'], p2p['z_q']
            ret['a2p'] = out
        return ret

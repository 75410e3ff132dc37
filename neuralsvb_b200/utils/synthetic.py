"""Deterministic synthetic weights and inputs for the mel-to-waveform path.

There is no network on the build or GPU boxes, so no pretrained vocoder
checkpoint and no dataset.  Everything here is generated from
``numpy.random.RandomState`` (bit-stable across numpy versions and machines),
so the oracle, the golden fixtures, the CUDA parity tests and ``bench.py`` all
see identical tensors.

Shapes and key names follow the reference checkpoint layout
(``vocoders/hifigan.py:17-33`` loads ``ckpt['state_dict']['model_gen']`` into
``HifiGanGenerator`` with weight-norm key names; layer shapes from
``modules/hifigan/hifigan.py:105-142``).
"""
from collections import OrderedDict

import numpy as np
import torch


def hifigan_config(nsf=True, hop=256):
    """The hop-256 HiFi-GAN(-NSF) architecture of
    ``egs/egs_bases/tts/vocoder/hifigan.yaml:3-10`` (+ ``use_pitch_embed``,
    SURVEY D7) or the hop-128 variant used by the singing configs."""
    if hop == 256:
        rates, ksz = [8, 8, 2, 2], [16, 16, 4, 4]
    elif hop == 128:
        rates, ksz = [8, 4, 2, 2], [16, 8, 4, 4]
    else:
        raise ValueError(f'no stock architecture for hop {hop}')
    return {
        'resblock': '1',
        'upsample_rates': rates,
        'upsample_kernel_sizes': ksz,
        'upsample_initial_channel': 512,
        'resblock_kernel_sizes': [3, 7, 11],
        'resblock_dilation_sizes': [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
        'use_pitch_embed': bool(nsf),
        'audio_sample_rate': 22050,
        'audio_num_mel_bins': 80,
        'hop_size': hop,
        'fft_size': 1024,
        'win_size': 512,
        'fmin': 80,
        'fmax': 7600,
    }


def small_config(nsf=True):
    """A narrow generator (64 initial channels, hop 16) for quick CPU-side
    parity cases; same topology, every code path exercised."""
    return {
        'resblock': '1',
        'upsample_rates': [4, 2, 2],
        'upsample_kernel_sizes': [8, 4, 4],
        'upsample_initial_channel': 64,
        'resblock_kernel_sizes': [3, 7, 11],
        'resblock_dilation_sizes': [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
        'use_pitch_embed': bool(nsf),
        'audio_sample_rate': 22050,
        'audio_num_mel_bins': 80,
        'hop_size': 16,
    }


def _normal(rs, shape, std):
    return (rs.standard_normal(size=shape) * std).astype(np.float32)


def _uniform(rs, shape, bound):
    return rs.uniform(-bound, bound, size=shape).astype(np.float32)


def _wn_pair(rs, shape, std, norm_dims):
    """weight_v ~ N(0, std) and a weight_g that is NOT equal to ||v|| so that
    weight-norm folding is actually exercised (g = ||v|| * U(0.7, 1.4))."""
    v = _normal(rs, shape, std)
    nrm = np.sqrt((v.astype(np.float64) ** 2).sum(axis=norm_dims, keepdims=True))
    g = (nrm * rs.uniform(0.7, 1.4, size=nrm.shape)).astype(np.float32)
    return g, v


def make_generator_state_dict(h, seed=1234, n_mel=80):
    """state_dict with the reference's weight-norm key names
    (``conv_pre.weight_g/weight_v``, ``ups.{i}.*``, ``noise_convs.{i}.*``,
    ``resblocks.{n}.convs{1,2}.{j}.*``, ``conv_post.*``,
    ``m_source.l_linear.*``).  Conv weights ~ N(0, 0.01..0.05) in the spirit of
    ``init_weights`` (``hifigan.py:14-17``); ConvTranspose1d weight-norm is
    over dim 0 = in-channels (SURVEY K13)."""
    rs = np.random.RandomState(seed)
    sd = OrderedDict()
    c0 = h['upsample_initial_channel']
    rates = h['upsample_rates']
    if h['use_pitch_embed']:
        sd['m_source.l_linear.weight'] = _uniform(rs, (1, 9), 1.0)
        sd['m_source.l_linear.bias'] = _uniform(rs, (1,), 1.0 / 3.0)
        for i in range(len(rates)):
            c_cur = c0 // (2 ** (i + 1))
            if i + 1 < len(rates):
                s = int(np.prod(rates[i + 1:]))
                k = 2 * s
            else:
                k = 1
            b = 4.0 / np.sqrt(k)
            sd[f'noise_convs.{i}.weight'] = _uniform(rs, (c_cur, 1, k), b)
            sd[f'noise_convs.{i}.bias'] = _uniform(rs, (c_cur,), b)
    b = 1.0 / np.sqrt(n_mel * 7)
    sd['conv_pre.bias'] = _uniform(rs, (c0,), b)
    g, v = _wn_pair(rs, (c0, n_mel, 7), b, (1, 2))
    sd['conv_pre.weight_g'], sd['conv_pre.weight_v'] = g, v
    for i, (u, k) in enumerate(zip(rates, h['upsample_kernel_sizes'])):
        cin = c0 // (2 ** i)
        cout = cin // 2
        sd[f'ups.{i}.bias'] = _uniform(rs, (cout,), 0.05)
        g, v = _wn_pair(rs, (cin, cout, k), 1.0 / np.sqrt(cin * k / u), (1, 2))
        sd[f'ups.{i}.weight_g'], sd[f'ups.{i}.weight_v'] = g, v
    nk = len(h['resblock_kernel_sizes'])
    for i in range(len(rates)):
        ch = c0 // (2 ** (i + 1))
        for j, (k, dil) in enumerate(zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes'])):
            n = i * nk + j
            groups = ['convs1', 'convs2'] if h['resblock'] == '1' else ['convs']
            for grp in groups:
                for m in range(len(dil)):
                    sd[f'resblocks.{n}.{grp}.{m}.bias'] = _uniform(rs, (ch,), 0.05)
                    g, v = _wn_pair(rs, (ch, ch, k), 1.0 / np.sqrt(ch * k), (1, 2))
                    sd[f'resblocks.{n}.{grp}.{m}.weight_g'] = g
                    sd[f'resblocks.{n}.{grp}.{m}.weight_v'] = v
    ch = c0 // (2 ** len(rates))
    sd['conv_post.bias'] = _uniform(rs, (1,), 0.05)
    g, v = _wn_pair(rs, (1, ch, 7), 0.2 / np.sqrt(ch * 7), (1, 2))
    sd['conv_post.weight_g'], sd['conv_post.weight_v'] = g, v
    return OrderedDict((k, torch.from_numpy(np.ascontiguousarray(v))) for k, v in sd.items())


def make_mel_f0(batch, frames, seed=1234, n_mel=80):
    """SURVEY 8(d) cfg 2 inputs: log10-mel ~ clamp(N(-2.5, 1.2^2), -6, 1.5)
    (range of ``tts/base.yaml:59-60``), f0 piecewise constant over 8..32-frame
    segments, voiced w.p. 0.8 with Hz ~ U(100, 500), 0 = unvoiced."""
    rs = np.random.RandomState(seed)
    mel = np.clip(rs.standard_normal((batch, n_mel, frames)) * 1.2 - 2.5, -6.0, 1.5).astype(np.float32)
    f0 = np.zeros((batch, frames), np.float32)
    for b in range(batch):
        t = 0
        while t < frames:
            seg = int(rs.randint(8, 33))
            hz = float(rs.uniform(100.0, 500.0)) if rs.uniform() < 0.8 else 0.0
            f0[b, t:t + seg] = hz
            t += seg
    return torch.from_numpy(mel), torch.from_numpy(f0)


def make_nsf_noise(batch, samples, seed=1234, harmonics=9):
    """The three RNG draws of the NSF source in reference order (SURVEY D8;
    ``source.py:53-56,131-132,397``): rand_ini[B,9] with column 0 zeroed,
    sine noise randn[B,T,9]; the third draw (noise branch, unused by the
    generator) is skipped."""
    rs = np.random.RandomState(seed + 7)
    rand_ini = rs.uniform(0.0, 1.0, size=(batch, harmonics)).astype(np.float32)
    rand_ini[:, 0] = 0.0
    noise = rs.standard_normal(size=(batch, samples, harmonics)).astype(np.float32)
    return torch.from_numpy(rand_ini), torch.from_numpy(noise)


def make_clip(n=44100, sr=22050, seed=1234, f_base=220.0):
    """SURVEY 8(d) cfg 1 clip: tone + chirp + noise, float32 in [-1, 1]."""
    rs = np.random.RandomState(seed)
    t = np.arange(n, dtype=np.float64) / sr
    wav = 0.3 * np.sin(2 * np.pi * f_base * t) + 0.1 * np.sin(2 * np.pi * (f_base + 330.0 * t) * t) \
        + 0.01 * rs.standard_normal(n)
    return np.clip(wav, -1.0, 1.0).astype(np.float32)


def make_wave_batch(batch, samples, sr=22050, seed=1234):
    """Harmonic + noise clips [B, samples] for the STFT-loss / discriminator cases."""
    rs = np.random.RandomState(seed + 11)
    out = np.zeros((batch, samples), np.float32)
    t = np.arange(samples, dtype=np.float64) / sr
    for b in range(batch):
        f = rs.uniform(100.0, 400.0)
        sig = np.zeros(samples)
        for hnum in range(1, 6):
            sig += (0.25 / hnum) * np.sin(2 * np.pi * f * hnum * t + rs.uniform(0, 2 * np.pi))
        sig += 0.02 * rs.standard_normal(samples)
        out[b] = np.clip(sig, -1.0, 1.0)
    return torch.from_numpy(out)


# ---------------------------------------------------------------------------------- discriminators
MPD_PERIODS = (2, 3, 5, 7, 11)
_MPD_CH = [(1, 32), (32, 128), (128, 512), (512, 1024), (1024, 1024)]
MSD_LAYERS = [(1, 128, 15, 1, 1, 7), (128, 128, 41, 2, 4, 20), (128, 256, 41, 2, 16, 20), (256, 512, 41, 4, 16, 20),
              (512, 1024, 41, 4, 16, 20), (1024, 1024, 41, 1, 16, 20), (1024, 1024, 5, 1, 1, 2)]


def _cond_net(rs, sd, prefix, t):
    """cond_net = ConvTranspose1d(80, 1, 2t, stride=t, padding=t//2), plain (hifigan.py:185-189, :257-260)."""
    sd[prefix + 'cond_net.weight'] = _normal(rs, (80, 1, 2 * t), 0.3 / np.sqrt(80 * 2.0))
    sd[prefix + 'cond_net.bias'] = _uniform(rs, (1,), 0.05)


def make_mpd_state_dict(seed=1234, use_cond=False, hop=256):
    """MultiPeriodDiscriminator state_dict: 5 x DiscriminatorP, weight-normed Conv2d [Cout, Cin, 5, 1]
    (+ conv_post [1, 1024, 3, 1]) -- modules/hifigan/hifigan.py:181-235.  ``use_cond``: + cond_net, 2 input channels."""
    rs = np.random.RandomState(seed + 101 + (1000 if use_cond else 0))
    sd = OrderedDict()
    for d in range(len(MPD_PERIODS)):
        if use_cond:
            _cond_net(rs, sd, f'discriminators.{d}.', hop)
        layers = [(f'convs.{i}', (2 if use_cond and i == 0 else cin), cout, 5) for i, (cin, cout) in enumerate(_MPD_CH)] + \
                 [('conv_post', 1024, 1, 3)]
        for name, cin, cout, k in layers:
            sd[f'discriminators.{d}.{name}.bias'] = _uniform(rs, (cout,), 0.05)
            g, v = _wn_pair(rs, (cout, cin, k, 1), 1.3 / np.sqrt(cin * k), (1, 2, 3))
            sd[f'discriminators.{d}.{name}.weight_g'], sd[f'discriminators.{d}.{name}.weight_v'] = g, v
    return OrderedDict((k, torch.from_numpy(np.ascontiguousarray(v))) for k, v in sd.items())


def make_msd_state_dict(seed=1234, use_cond=False, hop=256):
    """MultiScaleDiscriminator state_dict: discriminator 0 is spectral-normed (weight_orig / weight_u / weight_v),
    1 and 2 weight-normed -- modules/hifigan/hifigan.py:253-302.  ``use_cond``: + cond_net with stride
    hop / 2**d (upsample_rates [4, 4, hop // (16 * 2**d)], :294-302), 2 input channels."""
    rs = np.random.RandomState(seed + 202 + (1000 if use_cond else 0))
    sd = OrderedDict()
    for d in range(3):
        if use_cond:
            _cond_net(rs, sd, f'discriminators.{d}.', hop // (2 ** d))
        layers = [(f'convs.{i}', (2 if use_cond and i == 0 else cin), cout, k, g)
                  for i, (cin, cout, k, _, g, _) in enumerate(MSD_LAYERS)] + [('conv_post', 1024, 1, 3, 1)]
        for name, cin, cout, k, groups in layers:
            cg = cin // groups
            sd[f'discriminators.{d}.{name}.bias'] = _uniform(rs, (cout,), 0.05)
            if d == 0:
                w = _normal(rs, (cout, cg, k), 1.3 / np.sqrt(cg * k))
                # u, v as one power iteration from a random start leaves them (what spectral_norm stores),
                # so sigma = u . (W v) is a sensible estimate of the top singular value
                wm = w.reshape(cout, -1).astype(np.float64)
                u = rs.standard_normal(cout)
                v = wm.T @ (u / np.linalg.norm(u))
                v /= np.linalg.norm(v)
                u = wm @ v
                u /= np.linalg.norm(u)
                sd[f'discriminators.{d}.{name}.weight_orig'] = w
                sd[f'discriminators.{d}.{name}.weight_u'] = u.astype(np.float32)
                sd[f'discriminators.{d}.{name}.weight_v'] = v.astype(np.float32)
            else:
                g, v = _wn_pair(rs, (cout, cg, k), 1.3 / np.sqrt(cg * k), (1, 2))
                sd[f'discriminators.{d}.{name}.weight_g'], sd[f'discriminators.{d}.{name}.weight_v'] = g, v
    return OrderedDict((k, torch.from_numpy(np.ascontiguousarray(v))) for k, v in sd.items())


def make_wn_state_dict(hidden=192, kernel_size=5, n_layers=4, gin_channels=0, seed=1234):
    """state_dict of the reference's WN (modules/fastspeech/fs2_vae.py:19-60) with its weight-norm key names:
    ``in_layers.{i}.{bias,weight_g,weight_v}``, ``res_skip_layers.{i}.*``, ``cond_layer.*``; g != ||v||."""
    rs = np.random.RandomState(seed)
    sd = OrderedDict()

    def conv(prefix, cout, cin, k):
        b = 1.0 / np.sqrt(cin * k)
        sd[f'{prefix}.bias'] = _uniform(rs, (cout,), b)
        g, v = _wn_pair(rs, (cout, cin, k), b, (1, 2))
        sd[f'{prefix}.weight_g'], sd[f'{prefix}.weight_v'] = g, v
    if gin_channels:
        conv('cond_layer', 2 * hidden * n_layers, gin_channels, 1)
    for i in range(n_layers):
        conv(f'in_layers.{i}', 2 * hidden, hidden, kernel_size)
        conv(f'res_skip_layers.{i}', 2 * hidden if i < n_layers - 1 else hidden, hidden, 1)
    return OrderedDict((k, torch.from_numpy(v)) for k, v in sd.items())


def make_wn_inputs(B, T, hidden=192, gin_channels=0, seed=1234, ragged=True):
    """x [B, H, T] ~ N(0, 1), x_mask [B, 1, T] (clip b keeps T - 7 b frames when ``ragged``), g [B, gin, T] or None."""
    rs = np.random.RandomState(seed + 17)
    x = torch.from_numpy(_normal(rs, (B, hidden, T), 1.0))
    mask = torch.ones(B, 1, T)
    if ragged:
        for b in range(B):
            mask[b, :, T - min(7 * b, T - 1):] = 0.0 if b else 1.0
    g = torch.from_numpy(_normal(rs, (B, gin_channels, T), 1.0)) if gin_channels else None
    return x * mask, mask, g


def make_fvae_decoder_state_dict(latent=128, hidden=192, out_channels=80, kernel_size=5, n_layers=4, gin_channels=256, stride=4, seed=1234):
    """state_dict of the reference's FVAEDecoder / GlobalFVAEDecoder (fs2_vae.py:130-146): ``pre_net.0.*`` (ConvTranspose1d),
    ``wn.*`` (weight-normed), ``out_proj.*``."""
    rs = np.random.RandomState(seed + 3)
    sd = OrderedDict()
    b = 1.0 / np.sqrt(latent)
    sd['pre_net.0.weight'] = torch.from_numpy(_uniform(rs, (latent, hidden, stride), b))
    sd['pre_net.0.bias'] = torch.from_numpy(_uniform(rs, (hidden,), b))
    for k, v in make_wn_state_dict(hidden, kernel_size, n_layers, gin_channels, seed).items():
        sd[f'wn.{k}'] = v
    b = 1.0 / np.sqrt(hidden)
    sd['out_proj.weight'] = torch.from_numpy(_uniform(rs, (out_channels, hidden, 1), b))
    sd['out_proj.bias'] = torch.from_numpy(_uniform(rs, (out_channels,), b))
    return sd


def make_fvae_encoder_state_dict(in_channels=80, hidden=192, latent=128, kernel_size=5, n_layers=8, gin_channels=256, stride=4, seed=1234):
    """state_dict of the reference's GlobalFVAEEncoder (vae_models.py:81-95): ``pre_net.0.*``, ``wn.*`` (weight-normed),
    ``out_proj.*``, ``poolings.{0,3,6}.*`` (convs) and ``poolings.{2,5}.*`` (BatchNorm with non-trivial running statistics)."""
    rs = np.random.RandomState(seed + 9)
    sd = OrderedDict()

    def t(a):
        return torch.from_numpy(a)
    b = 1.0 / np.sqrt(in_channels * 2 * stride)
    sd['pre_net.0.weight'], sd['pre_net.0.bias'] = t(_uniform(rs, (hidden, in_channels, 2 * stride), b)), t(_uniform(rs, (hidden,), b))
    for k, v in make_wn_state_dict(hidden, kernel_size, n_layers, gin_channels, seed).items():
        sd[f'wn.{k}'] = v
    b = 1.0 / np.sqrt(hidden)
    c2 = 2 * latent
    sd['out_proj.weight'], sd['out_proj.bias'] = t(_uniform(rs, (c2, hidden, 1), b)), t(_uniform(rs, (c2,), b))
    b = 1.0 / np.sqrt(c2 * 3)
    for i in (0, 3, 6):
        sd[f'poolings.{i}.weight'], sd[f'poolings.{i}.bias'] = t(_uniform(rs, (c2, c2, 3), b)), t(_uniform(rs, (c2,), b))
    for i in (2, 5):
        sd[f'poolings.{i}.weight'], sd[f'poolings.{i}.bias'] = t(rs.uniform(0.5, 1.5, c2).astype(np.float32)), t(_uniform(rs, (c2,), 0.2))
        sd[f'poolings.{i}.running_mean'] = t(_uniform(rs, (c2,), 0.1))
        sd[f'poolings.{i}.running_var'] = t(rs.uniform(0.05, 0.5, c2).astype(np.float32))
        sd[f'poolings.{i}.num_batches_tracked'] = torch.tensor(100)
    return sd


def make_global_fvae_state_dict(in_out=80, hidden=192, latent=128, kernel_size=5, enc_layers=8, dec_layers=4, gin=256, stride=4, seed=1234):
    """state_dict of the reference's GlobalFVAE (vae_models.py:130-146): ``g_pre_net.0.*``, ``encoder.*``, ``decoder.*``."""
    rs = np.random.RandomState(seed + 21)
    sd = OrderedDict()
    b = 1.0 / np.sqrt(gin * 2 * stride)
    sd['g_pre_net.0.weight'] = torch.from_numpy(_uniform(rs, (gin, gin, 2 * stride), b))
    sd['g_pre_net.0.bias'] = torch.from_numpy(_uniform(rs, (gin,), b))
    for k, v in make_fvae_encoder_state_dict(in_out, hidden, latent, kernel_size, enc_layers, gin, stride, seed).items():
        sd[f'encoder.{k}'] = v
    for k, v in make_fvae_decoder_state_dict(latent, hidden, in_out, kernel_size, dec_layers, gin, stride, seed).items():
        sd[f'decoder.{k}'] = v
    return sd


def make_vc_asr_state_dict(seed=1234, hidden=256, n_mel=80, n_layers=2, n_head=4, K=31):
    """state_dict of the encoder half of the reference's VCASR (vc_modules.py:56-75): ``mel_prenet.*`` (Prenet, pe.py:7-22) and
    ``content_encoder.*`` (ConformerLayers with asr_last_norm false: the last ``layer_norm`` is a Linear).  BatchNorm layers get
    non-trivial running statistics, LayerNorms non-trivial affine parameters."""
    rs = np.random.RandomState(seed + 31)
    sd = OrderedDict()

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))

    def lin(prefix, cout, cin, k=None, bias=True):
        shape = (cout, cin) if k is None else (cout, cin, k)
        b = 1.0 / np.sqrt(cin * (k or 1))
        sd[prefix + '.weight'] = t(_uniform(rs, shape, b))
        if bias:
            sd[prefix + '.bias'] = t(_uniform(rs, (cout,), b))

    def bn(prefix, c):
        sd[prefix + '.weight'], sd[prefix + '.bias'] = t(rs.uniform(0.5, 1.5, c)), t(_uniform(rs, (c,), 0.2))
        sd[prefix + '.running_mean'], sd[prefix + '.running_var'] = t(_uniform(rs, (c,), 0.1)), t(rs.uniform(0.2, 1.0, c))
        sd[prefix + '.num_batches_tracked'] = torch.tensor(100)

    def ln(prefix, c):
        sd[prefix + '.weight'], sd[prefix + '.bias'] = t(rs.uniform(0.7, 1.3, c)), t(_uniform(rs, (c,), 0.1))
    cin = n_mel
    for i in range(3):
        lin(f'mel_prenet.layers.{i}.0', hidden, cin, 5)
        bn(f'mel_prenet.layers.{i}.2', hidden)
        cin = hidden
    lin('mel_prenet.out_proj', hidden, hidden)
    for l in range(n_layers):
        e = f'content_encoder.encoder_layers.{l}'
        for name in ('linear_q', 'linear_k', 'linear_v', 'linear_out'):
            lin(f'{e}.self_attn.{name}', hidden, hidden)
        lin(f'{e}.self_attn.linear_pos', hidden, hidden, bias=False)
        sd[f'{e}.self_attn.pos_bias_u'] = t(_uniform(rs, (n_head, hidden // n_head), 0.1))
        sd[f'{e}.self_attn.pos_bias_v'] = t(_uniform(rs, (n_head, hidden // n_head), 0.1))
        for ff in ('feed_forward', 'feed_forward_macaron'):
            lin(f'{e}.{ff}.w_1', 4 * hidden, hidden, 1)
            lin(f'{e}.{ff}.w_2', hidden, 4 * hidden, 1)
        lin(f'{e}.conv_module.pointwise_conv1', 2 * hidden, hidden, 1)
        lin(f'{e}.conv_module.depthwise_conv', hidden, 1, K)
        bn(f'{e}.conv_module.norm', hidden)
        lin(f'{e}.conv_module.pointwise_conv2', hidden, hidden, 1)
        for name in ('norm_ff', 'norm_mha', 'norm_ff_macaron', 'norm_conv', 'norm_final'):
            ln(f'{e}.{name}', hidden)
    lin('content_encoder.layer_norm', hidden, hidden)
    return sd


def make_vc_asr_mel(B, T, seed=1234, n_mel=80):
    """mel [B, T, 80] in the log10-mel range; clip b ends 9 b frames early (all-zero frames = padding, pe.py:30)."""
    rs = np.random.RandomState(seed + 37)
    mel = torch.from_numpy((rs.randn(B, T, n_mel) * 1.2 - 2.5).clip(-6, 1.5).astype(np.float32))
    for b in range(B):
        if b:
            mel[b, T - 9 * b:] = 0.0
    return mel


def make_svb_state_dict(seed=1234, hidden=256, latent=128, n_mel=80):
    """state_dict of the reference's MleSVBVAE (modules/voice_conversion/svb_vae.py:13-56,178-199,251-256) at the
    vae_global_mle_eng sizes, without the ASR token decoder (``vc_asr.asr_decoder.*``, ``vc_asr.token_embed.*``: training heads)."""
    rs = np.random.RandomState(seed + 41)
    sd = OrderedDict()

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))

    def lin(prefix, cout, cin, k=None):
        shape = (cout, cin) if k is None else (cout, cin, k)
        b = 1.0 / np.sqrt(cin * (k or 1))
        sd[prefix + '.weight'], sd[prefix + '.bias'] = t(_uniform(rs, shape, b)), t(_uniform(rs, (cout,), b))

    def bn(prefix, c):
        sd[prefix + '.weight'], sd[prefix + '.bias'] = t(rs.uniform(0.5, 1.5, c)), t(_uniform(rs, (c,), 0.2))
        sd[prefix + '.running_mean'], sd[prefix + '.running_var'] = t(_uniform(rs, (c,), 0.1)), t(rs.uniform(0.2, 1.0, c))
        sd[prefix + '.num_batches_tracked'] = torch.tensor(100)
    emb = _normal(rs, (300, hidden), hidden ** -0.5)
    emb[0] = 0
    sd['pitch_embed.weight'] = t(emb)
    lin('pitch_encoder.in_proj', hidden, hidden)
    for i in range(3):
        lin(f'pitch_encoder.conv.{i}.conv.conv', hidden, hidden, 5)
        sd[f'pitch_encoder.conv.{i}.norm.weight'], sd[f'pitch_encoder.conv.{i}.norm.bias'] = t(rs.uniform(0.7, 1.3, hidden)), t(_uniform(rs, (hidden,), 0.1))
    lin('pitch_encoder.out_proj', hidden, hidden)
    for k, v in make_vc_asr_state_dict(seed, hidden, n_mel).items():
        sd[f'vc_asr.{k}'] = v
    lin('upsample_layer.0.1', hidden, hidden, 5)
    bn('upsample_layer.0.3', hidden)
    lin('upsample_layer.1', hidden, hidden, 5)
    lin('spk_embed_proj', hidden, 256)
    lin('encoded_embed_proj', hidden, 3 * hidden)
    for k, v in make_global_fvae_state_dict(n_mel, 192, latent, 5, 8, 4, hidden, 4, seed).items():
        sd[f'vae_model.{k}'] = v
    for i in (0, 3, 6):
        lin(f'z_mapping_function.convs.{i}', latent, latent, 1)
    for i in (1, 4):
        bn(f'z_mapping_function.convs.{i}', latent)
    lin('z_mapping_function.spk_proj.0', latent, 256, 1)
    lin('z_mapping_function.spk_proj.2', latent, latent, 1)
    return sd


def make_mel_pair(B, T, pad, seed=1234, n_mel=80):
    """(mel_out, target) [B, T, n_mel] for the mel reconstruction loss: a log10-mel-range target whose clip b has its last pad[b]
    frames zero (padding; pad[b] = T is an all-padding clip) and a prediction = target + noise everywhere, padding frames included."""
    rs = np.random.RandomState(seed + 47)
    tgt = (rs.randn(B, T, n_mel) * 1.2 - 2.5).clip(-6, 1.5)
    out = tgt + rs.randn(B, T, n_mel) * 0.3
    for b, p in enumerate(pad):
        if p:
            tgt[b, T - p:] = 0.0
    return torch.from_numpy(out.astype(np.float32)), torch.from_numpy(tgt.astype(np.float32))


def make_svb_batch(B=2, Ta=96, Tp=120, seed=1234, n_mel=80):
    """A PopBuTFy-shaped batch (SURVEY 8(d) cfg 4 / 5): amateur / professional mels [B, T, 80] (zero frames = padding), coarse pitch
    ids in [1, 255] (0 = padding), one speaker embedding [B, 256], the a2p alignment [B, Tp] into the amateur frames."""
    rs = np.random.RandomState(seed + 43)

    def mel(T, short):
        m = (rs.randn(B, T, n_mel) * 1.2 - 2.5).clip(-6, 1.5).astype(np.float32)
        m[B - 1, T - short:] = 0.0
        return torch.from_numpy(m)

    def pitch(T, short):
        p = rs.randint(1, 256, size=(B, T))
        p[B - 1, T - short:] = 0
        return torch.from_numpy(p.astype(np.int64))
    a_mel, p_mel = mel(Ta, 8), mel(Tp, 12)
    a_pitch, p_pitch = pitch(Ta, 8), pitch(Tp, 12)
    spk = torch.from_numpy(_normal(rs, (B, 256), 0.5))
    align = torch.from_numpy(np.minimum((np.arange(Tp)[None, :] * Ta / Tp).astype(np.int64) + rs.randint(0, 2, size=(B, Tp)), Ta - 1))
    return dict(amateur_mel=a_mel, prof_mel=p_mel, amateur_pitch=a_pitch, prof_pitch=p_pitch, amateur_spk_id=spk, prof_spk_id=spk,
                a2p_alignment=align)


def make_mel_disc_state_dict(seed=1234, wins=(32, 64, 128), hidden=128, n_mel=80):
    """state_dict of the reference's mel discriminator (modules/fastspeech/multi_window_disc.py, Discriminator with
    norm_type 'in', c_in 1, kernel 3x3; tasks/tts/fs2_adv.py:22-34): per window three Conv2d blocks, InstanceNorm2d affine
    parameters on blocks 2 and 3, adv_layer = Linear(hidden * win/8 * ceil(n_mel/8), 1).  Uniform weights at PyTorch's default
    fan-in bounds, norm scales around 1."""
    rs = np.random.RandomState(seed + 53)
    sd = OrderedDict()

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    for i, win in enumerate(wins):
        p = f'discriminator.conv_layers.{i}.'
        for j in range(3):
            cin = 1 if j == 0 else hidden
            b = 1.0 / np.sqrt(cin * 9)
            sd[f'{p}model.{j}.0.weight'] = t(_uniform(rs, (hidden, cin, 3, 3), b))
            sd[f'{p}model.{j}.0.bias'] = t(_uniform(rs, (hidden,), b))
            if j > 0:
                sd[f'{p}model.{j}.3.weight'] = t(rs.uniform(0.7, 1.3, hidden))
                sd[f'{p}model.{j}.3.bias'] = t(_uniform(rs, (hidden,), 0.1))
        n = hidden * (win // 8) * ((n_mel + 7) // 8)
        sd[p + 'adv_layer.weight'] = t(_uniform(rs, (1, n), 1.0 / np.sqrt(n)))
        sd[p + 'adv_layer.bias'] = t(_uniform(rs, (1,), 1.0 / np.sqrt(n)))
    return sd


def make_disc_mel(B, T, pad, seed=1234, n_mel=80):
    """A log10-mel-range mel [B, T, n_mel] whose clip b has its last pad[b] frames zero (padding, not counted by x_len)."""
    rs = np.random.RandomState(seed + 59)
    m = (rs.randn(B, T, n_mel) * 1.2 - 2.5).clip(-6, 1.5)
    for b, p in enumerate(pad):
        if p:
            m[b, T - p:] = 0.0
    return torch.from_numpy(m.astype(np.float32))


def make_f0_pair(seed, S, T, fps=172.27):
    """(amateur [S], professional [T]) float64 f0 contours in Hz for the shape-aware DTW: one melody of held notes (note steps of
    a few semitones), sung twice.  The professional take has 5.5 Hz vibrato; the amateur one is detuned by up to half a semitone,
    drifts, has slower vibrato and different note timing.  Both have unvoiced gaps (f0 = 0) between some notes, like a denormed
    pitch track.  fps: frames per second (22050 Hz / hop 128)."""
    rs = np.random.RandomState(seed + 61)
    n_notes = max(1, int(round(max(S, T) / fps * 2.5)))
    notes = 57 + np.cumsum(rs.randint(-4, 5, size=n_notes)).clip(-12, 12)
    gaps = rs.rand(n_notes) < 0.3
    base = rs.dirichlet(np.full(n_notes, 4.0))

    def take(n, jitter, vib_hz, vib_st, detune, drift):
        w = base * np.exp(rs.randn(n_notes) * jitter)
        edges = np.concatenate([[0], np.cumsum(w / w.sum())]) * n
        t = np.arange(n)
        idx = np.searchsorted(edges[1:-1], t, side='right')
        semis = notes[idx] + detune + drift * t / max(n - 1, 1) + vib_st * np.sin(2 * np.pi * vib_hz * t / fps + rs.rand() * 6.28)
        f0 = 440.0 * 2.0 ** ((semis - 69) / 12.0)
        pos = (t - edges[idx]) / np.maximum(edges[idx + 1] - edges[idx], 1)
        f0[gaps[idx] & (pos > 0.75)] = 0.0
        return f0
    prof = take(T, 0.05, 5.5, 0.35, 0.0, 0.0)
    ama = take(S, 0.35, 4.5, 0.15, rs.uniform(-0.5, 0.5), rs.uniform(-0.4, 0.4))
    return ama, prof


def make_mel2ph_pair(seed, S, T):
    """(amateur [S], professional [T]) int64 mel2ph tracks for scoring a pitch alignment: the same phoneme sequence (ids 1 ..
    n_ph) sung with different durations, monotone runs, and a few trailing frames of zero padding per take."""
    rs = np.random.RandomState(seed + 67)
    n_ph = max(1, min(S, T) // 12)

    def take(n):
        pad = rs.randint(0, max(1, n // 10) + 1) if n > n_ph + 1 else 0
        w = rs.dirichlet(np.full(n_ph, 3.0))
        edges = np.floor(np.concatenate([[0], np.cumsum(w)]) * (n - pad)).astype(np.int64)
        m = np.zeros(n, np.int64)
        m[:n - pad] = np.searchsorted(edges[1:-1], np.arange(n - pad), side='right') + 1
        return m
    return take(S), take(T)


def write_svb_binary(data_dir, n_items=8, seed=1234, n_valid=2, n_test=2, frames=(60, 256)):
    """Write a paired-singing dataset in the layout data_gen/singing/binarize_para.py writes (``{train,valid,test}.data`` / ``.idx``,
    ``{prefix}_lengths.npy``, ``train_f0s_mean_std.npy``, ``phone_set.json``), plus what the SVB config points at next to it:
    ``asr/model_ckpt_steps_0.ckpt`` (a random VCASR encoder as ``state_dict.model``, the pretrain_asr_ckpt layout) and
    ``hifigan/`` (config.yaml + a random hop-128 HiFi-GAN-NSF in the vocoder checkpoint layout).

    Each item: an amateur and a professional take of independent lengths (multiples of 4 in ``frames``), log10-range mels,
    f0 from ``make_f0_pair`` with coarse pitch ids, ``a2p_f0_alignment`` = the monotone linear map from professional to amateur
    frames, and ``multi_spk_emb`` [5, 256].  Runs on the CPU."""
    import json
    import os

    from neuralsvb_b200.utils.indexed_datasets import IndexedDatasetBuilder
    from neuralsvb_b200.utils.pitch_utils import f0_to_coarse
    os.makedirs(data_dir, exist_ok=True)
    rs = np.random.RandomState(seed + 71)
    lo, hi = frames[0] // 4, frames[1] // 4
    with open(os.path.join(data_dir, 'phone_set.json'), 'w') as f:
        json.dump([f'ph{i}' for i in range(60)], f)
    train_f0s = []
    for prefix, n in (('train', n_items), ('valid', n_valid), ('test', n_test)):
        builder = IndexedDatasetBuilder(os.path.join(data_dir, prefix))
        lengths = []
        for i in range(n):
            Ta, Tp = 4 * int(rs.randint(lo, hi + 1)), 4 * int(rs.randint(lo, hi + 1))
            f0, prof_f0 = make_f0_pair(int(rs.randint(0, 2 ** 31 - 1)), Ta, Tp)
            mel = lambda T: (rs.randn(T, 80) * 1.2 - 2.5).clip(-6, 1.5).astype(np.float32)
            item = {'item_name': f'{prefix}_{i:04d}#Amateur', 'mel': mel(Ta), 'prof_mel': mel(Tp), 'f0': f0, 'prof_f0': prof_f0,
                    'pitch': f0_to_coarse(f0), 'prof_pitch': f0_to_coarse(prof_f0),
                    'a2p_f0_alignment': np.round(np.arange(Tp) * (Ta - 1) / max(Tp - 1, 1)).astype(np.int64),
                    'multi_spk_emb': _normal(rs, (5, 256), 0.5), 'len': Ta, 'prof_len': Tp}
            builder.add_item(item)
            lengths.append(max(Ta, Tp))
            if prefix == 'train':
                train_f0s += [f0, prof_f0]
        builder.finalize()
        np.save(os.path.join(data_dir, f'{prefix}_lengths.npy'), lengths)
    f0s = np.concatenate(train_f0s)
    f0s = f0s[f0s != 0]
    np.save(os.path.join(data_dir, 'train_f0s_mean_std.npy'), [np.mean(f0s).item(), np.std(f0s).item()])
    write_svb_checkpoints(data_dir, seed)


def write_svb_checkpoints(data_dir, seed=1234):
    """What the SVB config points at next to a dataset: ``asr/model_ckpt_steps_0.ckpt`` (a random VCASR encoder) and ``hifigan/``
    (config.yaml + a random hop-128 HiFi-GAN-NSF checkpoint)."""
    import os

    import yaml
    os.makedirs(os.path.join(data_dir, 'asr'), exist_ok=True)
    torch.save({'state_dict': {'model': make_vc_asr_state_dict(seed)}, 'global_step': 0},
               os.path.join(data_dir, 'asr', 'model_ckpt_steps_0.ckpt'))
    voc = os.path.join(data_dir, 'hifigan')
    os.makedirs(voc, exist_ok=True)
    h = hifigan_config(hop=128)
    with open(os.path.join(voc, 'config.yaml'), 'w') as f:
        yaml.safe_dump(h, f)
    torch.save({'state_dict': {'model_gen': make_generator_state_dict(h, seed)}, 'global_step': 0, 'epoch': 0,
                'checkpoint_callback_best': 0.0, 'optimizer_states': []}, os.path.join(voc, 'model_ckpt_steps_0.ckpt'))


def make_sung_take(f0_frames, seed, sr=22050, hop=128, breath=True):
    """(wav float32 [len(f0_frames) * hop], true f0 float64 per sample, 0 = unvoiced) of one singing-like take: a harmonic source
    whose phase integrates the frame contour (linearly interpolated over voiced frames), with a per-take spectral tilt, a slow
    amplitude envelope and 10 ms fades at every voicing edge, over silence or low-level breath noise in the gaps."""
    rs = np.random.RandomState(seed + 73)
    f0_frames = np.asarray(f0_frames, np.float64)
    n = len(f0_frames) * hop
    voiced_fr = f0_frames > 0
    k = np.arange(n)
    voiced = voiced_fr[k // hop]
    if voiced_fr.any():
        pos = np.nonzero(voiced_fr)[0] * hop + hop / 2.0
        f0 = np.interp(k, pos, f0_frames[voiced_fr])
    else:
        f0 = np.zeros(n)
    f0 = np.where(voiced, f0, 0.0)
    phase = 2 * np.pi * np.cumsum(f0) / sr + rs.uniform(0, 2 * np.pi)
    tilt = rs.uniform(0.8, 1.6)
    src = np.zeros(n)
    for h in range(1, 40):
        amp = h ** -tilt * rs.uniform(0.7, 1.3)
        src += np.where(h * f0 < 0.45 * sr, amp * np.sin(h * phase + rs.uniform(0, 2 * np.pi)), 0.0)
    fade = int(0.01 * sr)
    ramp = np.convolve(voiced.astype(np.float64), np.hanning(2 * fade + 1) / np.hanning(2 * fade + 1).sum(), mode='same')
    env = (0.55 + 0.25 * np.sin(2 * np.pi * k / sr * rs.uniform(0.3, 1.2) + rs.uniform(0, 6.28))) * ramp
    wav = 0.35 * env * src / max(1.0, np.abs(src).max() / 2.5)
    if breath:
        wav += (1.0 - ramp) * 0.004 * rs.standard_normal(n)
    return np.clip(wav, -1, 1).astype(np.float32), f0


def write_svb_raw(processed_dir, binary_data_dir=None, seed=1234, sr=22050, hop=128, seconds=(1.5, 3.0), gap_frames=None,
                  file_sr=None, channels=1, sample_format='int16'):
    """Write a raw paired-singing set in PopBuTFy's layout, for the paired binarizer (egs/svb_binarize_synthetic.yaml):
    ``{processed_dir}/data/{spk}#singing#{song}/{spk}#singing#{song}_{Amateur|Professional}_{k}.wav`` (16-bit mono WAV at sr),
    ``{processed_dir}/spk_emb/{item_name}.npy`` (256-d, one per amateur take) and ``{processed_dir}/phone_set.json``.

    Three speakers (Female1, Female2, Male1) sing two songs in two pieces each; each pair is ``make_f0_pair``'s two takes through
    ``make_sung_take``.  Besides the regular pairs: ``Female2#singing#Song_B_Amateur_1``'s professional take is ``gap_frames`` frames
    (default 240) longer than the amateur one; ``Male1#singing#Song_A_Amateur_1`` is digital silence; ``Female1#singing#Song_C_Amateur_0``
    has no professional take; ``Female1#speech#Talk_Amateur_0`` is not singing.  With ``binary_data_dir``, phone_set.json and the
    checkpoints of ``write_svb_checkpoints`` are written there too.

    ``sr`` / ``hop`` are the model's rate and hop (the f0 contours have sr / hop frames per second).  The files are recorded at
    ``file_sr`` (default sr; the takes are synthesised at that rate, round(hop file_sr / sr) samples per contour frame) with
    ``channels`` channels (channel c is the take times 1 - 0.2 c) as ``sample_format`` 'int16' or 'float32' samples.

    Returns {item_name: true f0 per sample of the file (float64, 0 = unvoiced)} for every file written."""
    import json
    import os

    from scipy.io import wavfile
    if sample_format not in ('int16', 'float32') or channels < 1:
        raise ValueError(f'write_svb_raw writes int16 or float32 samples on 1 or more channels, not {sample_format} x {channels}')
    rs = np.random.RandomState(seed + 79)
    fps = sr / hop
    file_sr = sr if file_sr is None else int(file_sr)
    file_hop = hop if file_sr == sr else int(round(hop * file_sr / sr))
    gap_frames = 240 if gap_frames is None else gap_frames
    truth = {}

    def write(name, wav, f0):
        d = os.path.join(processed_dir, 'data', name.rsplit('_', 2)[0])
        os.makedirs(d, exist_ok=True)
        wav = np.clip(wav, -1, 1)
        if channels > 1:
            wav = np.stack([wav * np.float32(1 - 0.2 * c) for c in range(channels)], axis=1)
        data = np.round(wav * 32767).astype(np.int16) if sample_format == 'int16' else wav.astype(np.float32)
        wavfile.write(os.path.join(d, name + '.wav'), file_sr, data)
        truth[name] = f0

    emb_dir = os.path.join(processed_dir, 'spk_emb')
    os.makedirs(emb_dir, exist_ok=True)
    spk_shift = {'Female1': 5, 'Female2': 3, 'Male1': -4}
    for spk, shift in spk_shift.items():
        songs = [('Song_A', 2), ('Song_B', 2)] + ([('Song_C', 1)] if spk == 'Female1' else [])
        for song, pieces in songs:
            for piece in range(pieces):
                base = f'{spk}#singing#{song}'
                ama, prof = f'{base}_Amateur_{piece}', f'{base}_Professional_{piece}'
                S = int(rs.uniform(*seconds) * fps)
                T = S + gap_frames if ama == 'Female2#singing#Song_B_Amateur_1' else int(S * rs.uniform(0.85, 1.15))
                fa, fp = make_f0_pair(int(rs.randint(0, 2 ** 31 - 1)), S, T, fps)
                fa, fp = fa * 2 ** (shift / 12), fp * 2 ** (shift / 12)
                wa, ta = make_sung_take(fa, int(rs.randint(0, 2 ** 31 - 1)), file_sr, file_hop)
                if ama == 'Male1#singing#Song_A_Amateur_1':
                    wa, ta = np.zeros_like(wa), np.zeros_like(ta)
                write(ama, wa, ta)
                np.save(os.path.join(emb_dir, ama + '.npy'), _normal(rs, (256,), 0.5))
                if song != 'Song_C':
                    wp, tp = make_sung_take(fp, int(rs.randint(0, 2 ** 31 - 1)), file_sr, file_hop)
                    write(prof, wp, tp)
    f0, _ = make_f0_pair(int(rs.randint(0, 2 ** 31 - 1)), int(2 * fps), int(2 * fps), fps)
    w, t = make_sung_take(f0, int(rs.randint(0, 2 ** 31 - 1)), file_sr, file_hop)
    write('Female1#speech#Talk_Amateur_0', w, t)
    phones = [f'ph{i}' for i in range(60)]
    for d in [processed_dir] + ([binary_data_dir] if binary_data_dir else []):
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, 'phone_set.json'), 'w') as f:
            json.dump(phones, f)
    if binary_data_dir:
        write_svb_checkpoints(binary_data_dir, seed)
    return truth

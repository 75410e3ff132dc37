"""ORACLE (test infrastructure only; see oracle/__init__.py).

torch-CPU fp32 restatement of the HiFi-GAN-NSF generator, the NSF source, the
MPD / MSD discriminators, the GAN losses, the torch mel_spectrogram and the
multi-resolution STFT loss.  Functional style over a plain ``{name: tensor}``
weight dict (the reference's state_dict names), no nn.Module, no RNG inside:
the three random draws of the NSF source are explicit arguments (SURVEY D8).

Follows, in order:
  modules/parallel_wavegan/models/source.py:7-137,351-398   SineGen, SourceModuleHnNSF
  modules/hifigan/hifigan.py:11-178                          ResBlock1/2, HifiGanGenerator
  modules/hifigan/hifigan.py:181-365                         MPD, MSD, GAN losses
  modules/hifigan/mel_utils.py:45-80                         mel_spectrogram
  modules/parallel_wavegan/losses/stft_loss.py:12-153        stft, SC / log-mag, MR-STFT
  modules/parallel_wavegan/stft_loss.py:13-100               use_mel_loss variant
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import frontend

LRELU_SLOPE = 0.1          # hifigan.py:11


# ------------------------------------------------------------------ weight norm
def fold_weight_norm(sd):
    """remove_weight_norm (hifigan.py:63-67,171-178): weight = g * v / ||v||
    with the norm over every dim except 0 (torch.nn.utils.weight_norm dim=0;
    for ConvTranspose1d dim 0 is IN-channels, SURVEY K13).  Plain tensors pass
    through."""
    out = {}
    for k, v in sd.items():
        if k.endswith('.weight_g'):
            continue
        if k.endswith('.weight_v'):
            g = sd[k[:-1] + 'g']
            out[k[:-2]] = torch._weight_norm(v, g, 0)
        else:
            out[k] = v
    return out


def get_padding(kernel_size, dilation=1):
    """hifigan.py:26-27."""
    return int((kernel_size * dilation - dilation) / 2)


# ------------------------------------------------------------------ NSF source
def sine_gen(f0, rand_ini, noise, sr=22050, harmonic_num=8, sine_amp=0.1, noise_std=0.003,
             voiced_threshold=0.0):
    """SineGen.forward (source.py:104-137) with _f02sine (:44-73) and _f02uv
    (:38-42).  f0 [B,T,1]; rand_ini [B,9] with column 0 == 0 (draw 1,
    :53-55); noise [B,T,9] standard normal (draw 2, :132)."""
    dim = harmonic_num + 1
    f0_buf = torch.zeros(f0.shape[0], f0.shape[1], dim)
    f0_buf[:, :, 0] = f0[:, :, 0]
    for idx in range(harmonic_num):
        f0_buf[:, :, idx + 1] = f0_buf[:, :, 0] * (idx + 2)
    rad_values = (f0_buf / sr) % 1
    rad_values[:, 0, :] = rad_values[:, 0, :] + rand_ini
    tmp_over_one = torch.cumsum(rad_values, 1) % 1
    tmp_over_one_idx = (tmp_over_one[:, 1:, :] - tmp_over_one[:, :-1, :]) < 0
    cumsum_shift = torch.zeros_like(rad_values)
    cumsum_shift[:, 1:, :] = tmp_over_one_idx * -1.0
    sines = torch.sin(torch.cumsum(rad_values + cumsum_shift, dim=1) * 2 * np.pi)
    sine_waves = sines * sine_amp
    uv = torch.ones_like(f0) * (f0 > voiced_threshold)
    noise_amp = uv * noise_std + (1 - uv) * sine_amp / 3
    sine_waves = sine_waves * uv + noise_amp * noise
    return sine_waves, uv


def source_module(f0_up, w, rand_ini, noise, sr=22050):
    """SourceModuleHnNSF.forward (source.py:385-398): tanh(Linear(9->1)(sines)).
    The noise branch (draw 3, :397) is returned by the reference but never used
    by the generator, so it is not produced here."""
    sine_wavs, uv = sine_gen(f0_up, rand_ini, noise, sr=sr)
    merged = torch.tanh(F.linear(sine_wavs, w['m_source.l_linear.weight'], w['m_source.l_linear.bias']))
    return merged, uv


# ------------------------------------------------------------------ generator
def _leaky_relu(site, x, slope):
    return F.leaky_relu(x, slope)


def resblock1(x, w, prefix, k, dil, act=_leaky_relu):
    """ResBlock1.forward (hifigan.py:54-61).  ``act(site, x, slope)`` is every leaky relu; the sites are
    ``{prefix}.x{m}`` (the input of step m) and ``{prefix}.t{m}`` (convs1's output)."""
    for m, d in enumerate(dil):
        xt = act(f'{prefix}.x{m}', x, LRELU_SLOPE)
        xt = F.conv1d(xt, w[f'{prefix}.convs1.{m}.weight'], w[f'{prefix}.convs1.{m}.bias'],
                      dilation=d, padding=get_padding(k, d))
        xt = act(f'{prefix}.t{m}', xt, LRELU_SLOPE)
        xt = F.conv1d(xt, w[f'{prefix}.convs2.{m}.weight'], w[f'{prefix}.convs2.{m}.bias'],
                      padding=get_padding(k, 1))
        x = xt + x
    return x


def resblock2(x, w, prefix, k, dil, act=_leaky_relu):
    """ResBlock2.forward (hifigan.py:81-86); ``act`` as in resblock1, sites ``{prefix}.x{m}``."""
    for m, d in enumerate(dil):
        xt = act(f'{prefix}.x{m}', x, LRELU_SLOPE)
        xt = F.conv1d(xt, w[f'{prefix}.convs.{m}.weight'], w[f'{prefix}.convs.{m}.bias'],
                      dilation=d, padding=get_padding(k, d))
        x = xt + x
    return x


def upsample_forward(w, h, i, x, har=None, act=_leaky_relu):
    """Upsampler ``i`` (hifigan.py:153-157): leaky relu of ``x`` (``conv_pre`` or ``stage{i-1}``), ``ups.{i}``, plus
    ``noise_convs.{i}(har)`` when ``har`` [B,1,T*hop] is given.  Returns the ``ups{i}`` tap."""
    rates, u, k = h['upsample_rates'], h['upsample_rates'][i], h['upsample_kernel_sizes'][i]
    x = act('conv_pre' if i == 0 else f'stage{i - 1}', x, LRELU_SLOPE)
    x = F.conv_transpose1d(x, w[f'ups.{i}.weight'], w[f'ups.{i}.bias'], stride=u, padding=(k - u) // 2)
    if har is not None:
        if i + 1 < len(rates):
            s = int(np.prod(rates[i + 1:]))
            x = x + F.conv1d(har, w[f'noise_convs.{i}.weight'], w[f'noise_convs.{i}.bias'], stride=s, padding=s // 2)
        else:
            x = x + F.conv1d(har, w[f'noise_convs.{i}.weight'], w[f'noise_convs.{i}.bias'])
    return x


def stage_forward(w, h, i, x, act=_leaky_relu):
    """The ResBlocks of stage ``i`` on ``x`` (the ``ups{i}`` tap), summed and divided by their number
    (hifigan.py:158-164).  Returns the ``stage{i}`` tap."""
    nk = len(h['resblock_kernel_sizes'])
    fn = resblock1 if h['resblock'] == '1' else resblock2
    xs = None
    for j, (rk, dil) in enumerate(zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes'])):
        r = fn(x, w, f'resblocks.{i * nk + j}', rk, dil, act)
        xs = r if xs is None else xs + r
    return xs / nk


def post_forward(w, h, x, act=_leaky_relu):
    """tanh(conv_post(leaky_relu(x, 0.01))) of the last stage's output (hifigan.py:165-167)."""
    x = act(f'stage{len(h["upsample_rates"]) - 1}', x, 0.01)   # F.leaky_relu's default slope (SURVEY D9)
    x = F.conv1d(x, w['conv_post.weight'], w['conv_post.bias'], padding=3)
    return torch.tanh(x)


def generator_forward(w, h, mel, f0=None, rand_ini=None, noise=None, taps=None, act=_leaky_relu):
    """HifiGanGenerator.forward (hifigan.py:144-169) on FOLDED weights ``w``
    (see fold_weight_norm).  mel [B,80,T]; f0 [B,T] Hz or None.  ``taps``: an
    optional dict that receives named intermediates for layer-level checks.
    ``act(site, x, slope)`` is called at every leaky relu, named after the tap
    that holds its input: ``conv_pre`` and ``stage{i}`` (upsampler inputs, the
    last stage's at slope 0.01 before conv_post) and the ResBlock sites of
    resblock1 / resblock2."""
    rates = h['upsample_rates']
    har = None
    if f0 is not None:
        scale = int(np.prod(rates))
        f0_up = F.interpolate(f0[:, None], scale_factor=scale, mode='nearest').transpose(1, 2)   # :113,147
        har, _ = source_module(f0_up, w, rand_ini, noise, sr=h['audio_sample_rate'])
        har = har.transpose(1, 2)                                                                # [B,1,T*hop]
        if taps is not None:
            taps['har_source'] = har
    x = F.conv1d(mel, w['conv_pre.weight'], w['conv_pre.bias'], padding=3)
    if taps is not None:
        taps['conv_pre'] = x
    for i in range(len(rates)):
        x = upsample_forward(w, h, i, x, har, act)
        if taps is not None:
            taps[f'ups{i}'] = x
        x = stage_forward(w, h, i, x, act)
        if taps is not None:
            taps[f'stage{i}'] = x
    return post_forward(w, h, x, act)


# ------------------------------------------------------------------ discriminators
def _cond(x, w, prefix, mel):
    """cond_net + concat (hifigan.py:204-206, :274-276): x_mel = ConvTranspose1d(80, 1, 2t, t, t//2)(mel)."""
    cw = w[f'{prefix}.cond_net.weight']
    t = cw.shape[2] // 2
    x_mel = F.conv_transpose1d(mel, cw, w[f'{prefix}.cond_net.bias'], stride=t, padding=t // 2)
    return torch.cat([x_mel, x], 1)


def disc_p_forward(x, w, prefix, period, mel=None):
    """DiscriminatorP.forward (hifigan.py:202-223).  ``w`` holds folded Conv2d weights [Cout,Cin,k,1];
    ``mel`` [B,80,T] switches on the use_cond branch."""
    fmap = []
    if mel is not None:
        x = _cond(x, w, prefix, mel)
    b, c, t = x.shape
    if t % period != 0:
        n_pad = period - (t % period)
        x = F.pad(x, (0, n_pad), 'reflect')
        t = t + n_pad
    x = x.view(b, c, t // period, period)
    strides = [3, 3, 3, 3, 1]
    for i, s in enumerate(strides):
        x = F.conv2d(x, w[f'{prefix}.convs.{i}.weight'], w[f'{prefix}.convs.{i}.bias'],
                     stride=(s, 1), padding=(2, 0))
        x = F.leaky_relu(x, LRELU_SLOPE)
        fmap.append(x)
    x = F.conv2d(x, w[f'{prefix}.conv_post.weight'], w[f'{prefix}.conv_post.bias'], padding=(1, 0))
    fmap.append(x)
    return torch.flatten(x, 1, -1), fmap


MPD_PERIODS = (2, 3, 5, 7, 11)                  # hifigan.py:229-235


def mpd_forward(y, y_hat, w, prefix='', mel=None):
    """MultiPeriodDiscriminator.forward (hifigan.py:237-250)."""
    y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
    for i, p in enumerate(MPD_PERIODS):
        r, fr = disc_p_forward(y, w, f'{prefix}discriminators.{i}', p, mel)
        g, fg = disc_p_forward(y_hat, w, f'{prefix}discriminators.{i}', p, mel)
        y_d_rs.append(r), fmap_rs.append(fr), y_d_gs.append(g), fmap_gs.append(fg)
    return y_d_rs, y_d_gs, fmap_rs, fmap_gs


MSD_LAYERS = [  # (cin, cout, k, stride, groups, pad)   hifigan.py:262-270
    (1, 128, 15, 1, 1, 7), (128, 128, 41, 2, 4, 20), (128, 256, 41, 2, 16, 20), (256, 512, 41, 4, 16, 20),
    (512, 1024, 41, 4, 16, 20), (1024, 1024, 41, 1, 16, 20), (1024, 1024, 5, 1, 1, 2)]


def disc_s_forward(x, w, prefix, mel=None):
    """DiscriminatorS.forward (hifigan.py:273-286), effective (already normalised) weights; ``mel`` switches on
    the use_cond branch."""
    fmap = []
    if mel is not None:
        x = _cond(x, w, prefix, mel)
    for i, (_, _, _, s, g, p) in enumerate(MSD_LAYERS):
        x = F.conv1d(x, w[f'{prefix}.convs.{i}.weight'], w[f'{prefix}.convs.{i}.bias'],
                     stride=s, padding=p, groups=g)
        x = F.leaky_relu(x, LRELU_SLOPE)
        fmap.append(x)
    x = F.conv1d(x, w[f'{prefix}.conv_post.weight'], w[f'{prefix}.conv_post.bias'], padding=1)
    fmap.append(x)
    return torch.flatten(x, 1, -1), fmap


def msd_forward(y, y_hat, w, prefix='', mel=None):
    """MultiScaleDiscriminator.forward (hifigan.py:309-325): AvgPool1d(4,2,1)
    between scales (count_include_pad default True)."""
    y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
    for i in range(3):
        if i != 0:
            y = F.avg_pool1d(y, 4, 2, padding=1)
            y_hat = F.avg_pool1d(y_hat, 4, 2, padding=1)
        r, fr = disc_s_forward(y, w, f'{prefix}discriminators.{i}', mel)
        g, fg = disc_s_forward(y_hat, w, f'{prefix}discriminators.{i}', mel)
        y_d_rs.append(r), fmap_rs.append(fr), y_d_gs.append(g), fmap_gs.append(fg)
    return y_d_rs, y_d_gs, fmap_rs, fmap_gs


# ------------------------------------------------------------------ GAN losses
def feature_loss(fmap_r, fmap_g):
    """hifigan.py:328-334."""
    loss = 0
    for dr, dg in zip(fmap_r, fmap_g):
        for rl, gl in zip(dr, dg):
            loss = loss + torch.mean(torch.abs(rl - gl))
    return loss * 2


def discriminator_loss(disc_real_outputs, disc_generated_outputs):
    """hifigan.py:337-347."""
    r_losses, g_losses = 0, 0
    for dr, dg in zip(disc_real_outputs, disc_generated_outputs):
        r_losses = r_losses + torch.mean((1 - dr) ** 2)
        g_losses = g_losses + torch.mean(dg ** 2)
    n = len(disc_real_outputs)
    return r_losses / n, g_losses / n


def generator_loss(disc_outputs):
    """hifigan.py:359-365."""
    loss = 0
    for dg in disc_outputs:
        loss = loss + torch.mean((1 - dg) ** 2)
    return loss / len(disc_outputs)


# ------------------------------------------------------------------ torch mel / STFT losses
def mel_spectrogram(y, hp, center=False):
    """modules/hifigan/mel_utils.py:45-80 (non-complex branch): clamp, reflect
    pad (n_fft-hop)/2, torch.stft(center=False, hann(win)), sqrt(re^2+im^2+1e-9),
    mel matmul, ln(clamp(., 1e-5)).  y [B, T] -> [B, 80, T/hop]."""
    n_fft, hop, win = hp['fft_size'], hp['hop_size'], hp['win_size']
    y = y.clamp(min=-1., max=1.)
    mel_basis = torch.from_numpy(frontend.mel_filterbank(
        hp['audio_sample_rate'], n_fft, hp['audio_num_mel_bins'], hp['fmin'], hp['fmax'])).float()
    window = torch.hann_window(win)
    pad = int((n_fft - hop) / 2)
    y = F.pad(y.unsqueeze(1), (pad, pad), mode='reflect').squeeze(1)
    spec = torch.view_as_real(torch.stft(y, n_fft, hop_length=hop, win_length=win, window=window, center=center,
                                         pad_mode='reflect', normalized=False, onesided=True,
                                         return_complex=True))
    spec = torch.sqrt(spec.pow(2).sum(-1) + 1e-9)
    spec = torch.matmul(mel_basis, spec)
    return torch.log(torch.clamp(spec, min=1e-5))


def stft_mag(x, fft_size, hop_size, win_length):
    """losses/stft_loss.py:12-31: torch.stft defaults (center=True, reflect),
    sqrt(clamp(re^2+im^2, 1e-7)), transposed to [B, frames, bins]."""
    window = torch.hann_window(win_length)
    x_stft = torch.view_as_real(torch.stft(x, fft_size, hop_size, win_length, window, return_complex=True))
    real, imag = x_stft[..., 0], x_stft[..., 1]
    return torch.sqrt(torch.clamp(real ** 2 + imag ** 2, min=1e-7)).transpose(2, 1)


def stft_loss(x, y, fft_size, hop_size, win_length, mel_basis=None):
    """STFTLoss.forward (losses/stft_loss.py:89-106; parallel_wavegan/stft_loss.py:29-52
    when ``mel_basis`` [bins, 80] is given): spectral convergence + log-mag L1."""
    x_mag = stft_mag(x, fft_size, hop_size, win_length)
    y_mag = stft_mag(y, fft_size, hop_size, win_length)
    if mel_basis is not None:
        x_mag, y_mag = x_mag @ mel_basis, y_mag @ mel_basis
    sc = torch.norm(y_mag - x_mag, p='fro') / torch.norm(y_mag, p='fro')
    mag = F.l1_loss(torch.log(y_mag), torch.log(x_mag))
    return sc, mag


MR_STFT = ((1024, 120, 600), (2048, 240, 1200), (512, 50, 240))     # losses/stft_loss.py:113-115


def mr_stft_loss(x, y, resolutions=MR_STFT, use_mel_loss=False):
    """MultiResolutionSTFTLoss.forward (losses/stft_loss.py:130-153)."""
    sc_loss, mag_loss = 0.0, 0.0
    for fs, ss, wl in resolutions:
        mb = None
        if use_mel_loss:   # parallel_wavegan/stft_loss.py:43-47: mel(22050, fft, 80), full band
            mb = torch.from_numpy(frontend.mel_filterbank(22050, fs, 80)).T
        sc, mag = stft_loss(x, y, fs, ss, wl, mb)
        sc_loss, mag_loss = sc_loss + sc, mag_loss + mag
    n = len(resolutions)
    return sc_loss / n, mag_loss / n


def fold_discriminator_weights(sd):
    """Effective conv weights of an MPD / MSD state_dict: weight norm folded (dim 0) and, for the
    spectral-normed MSD[0], weight_orig / sigma with sigma = u . (W v) -- torch.nn.utils.spectral_norm
    in eval mode (no power iteration; hifigan.py:294-296 wraps DiscriminatorS(use_spectral_norm=True))."""
    out = {}
    for k, v in sd.items():
        if k.endswith('.weight_g') or k.endswith('.weight_u'):
            continue
        if k.endswith('.weight_orig'):
            p = k[:-len('weight_orig')]
            w_mat = v.reshape(v.shape[0], -1)
            sigma = torch.dot(sd[p + 'weight_u'], torch.mv(w_mat, sd[p + 'weight_v']))
            out[p + 'weight'] = v / sigma
        elif k.endswith('.weight_v'):
            p = k[:-len('weight_v')]
            if p + 'weight_orig' in sd:
                continue
            out[p + 'weight'] = torch._weight_norm(v, sd[p + 'weight_g'], 0)
        else:
            out[k] = v
    return out


# ------------------------------------------------------------------ spectral norm, training mode
def spectral_power_iteration(sd, prefix):
    """One power iteration of torch.nn.utils.spectral_norm (the forward pre-hook runs it on EVERY training-mode
    forward, under no_grad): v <- normalize(W^T u), u <- normalize(W v); the buffers in ``sd`` are updated in
    place.  hifigan.py:261 (norm_f = spectral_norm) + :294 (DiscriminatorS(use_spectral_norm=True))."""
    with torch.no_grad():
        wm = sd[prefix + 'weight_orig'].detach().flatten(1)
        v = F.normalize(torch.mv(wm.t(), sd[prefix + 'weight_u']), dim=0, eps=1e-12)
        u = F.normalize(torch.mv(wm, v), dim=0, eps=1e-12)
        sd[prefix + 'weight_u'], sd[prefix + 'weight_v'] = u, v


def disc_s_train_weights(sd, d):
    """Effective weights of MSD discriminator ``d`` for ONE training-mode forward: spectral-normed layers run their
    power iteration first (buffers of ``sd`` updated), sigma = u . (W v) with u, v constants (the gradient reaches
    weight_orig through both the numerator and sigma)."""
    out = {}
    pre = f'discriminators.{d}.'
    for k in [k for k in sd if k.startswith(pre)]:
        v = sd[k]
        if k.endswith('.weight_orig'):
            p = k[:-len('weight_orig')]
            spectral_power_iteration(sd, p)
            sigma = torch.dot(sd[p + 'weight_u'], torch.mv(v.flatten(1), sd[p + 'weight_v']))
            out[p + 'weight'] = v / sigma
        elif k.endswith('.weight_v') and k[:-1] + 'g' in sd:
            out[k[:-2]] = torch._weight_norm(v, sd[k[:-1] + 'g'], 0)
        elif k.endswith('.weight_g') or k.endswith('.weight_u') or k.endswith('.weight_v'):
            continue
        else:
            out[k] = v
    return out


def msd_forward_train(y, y_hat, sd, mel=None):
    """MultiScaleDiscriminator.forward in train() mode (hifigan.py:309-325): every DiscriminatorS call is its own
    forward, so discriminator 0 runs one power iteration for ``y`` and another for ``y_hat``."""
    y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
    for i in range(3):
        if i != 0:
            y = F.avg_pool1d(y, 4, 2, padding=1)
            y_hat = F.avg_pool1d(y_hat, 4, 2, padding=1)
        r, fr = disc_s_forward(y, disc_s_train_weights(sd, i), f'discriminators.{i}', mel)
        g, fg = disc_s_forward(y_hat, disc_s_train_weights(sd, i), f'discriminators.{i}', mel)
        y_d_rs.append(r), fmap_rs.append(fr), y_d_gs.append(g), fmap_gs.append(fg)
    return y_d_rs, y_d_gs, fmap_rs, fmap_gs

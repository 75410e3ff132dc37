"""ORACLE (test infrastructure only; see oracle/__init__.py): torch restatement of the mel discriminator
(modules/fastspeech/multi_window_disc.py, built by tasks/tts/fs2_adv.py:22-34 with disc_norm 'in') and of the adversarial
terms of the SVB training steps (tasks/singing/svb_para.py:118-170, svb_vae_task.py:621-660).

Runs in the dtype of its inputs.  The window starts (``start_frames_wins``) and the Dropout2d factors (``dropout_scales``:
per window, per block, [B, C] of 0 or 1/(1-p); None = eval mode) are injected, never drawn.
"""
import torch
import torch.nn.functional as F

WINDOWS = (32, 64, 128)
LAMBDA_MEL_ADV = 0.1


def x_len(x):
    """Frames whose bins do not sum to 0, x [B, T, F] (Discriminator.forward)."""
    return x.sum(-1).ne(0).int().sum(-1)


def window_forward(sd, prefix, x, scales=None, slope=0.2, eps=1e-5, masks=None):
    """Discriminator2DFactory.forward: x [B, 1, win, F] -> (validity [B, 1], h = three block outputs).
    ``masks`` (per block, bool like the conv output; None = F.leaky_relu) fixes which elements take the leaky relu's identity branch:
    a test passes the masks of the run it checks, so that a pre-activation that rounds across zero in one of the two runs does not
    move the gradient by (1 - slope) of that element's value."""
    h = []
    for j in range(3):
        p = f'{prefix}model.{j}.'
        z = F.conv2d(x, sd[p + '0.weight'], sd[p + '0.bias'], stride=2, padding=1)
        x = F.leaky_relu(z, slope) if masks is None else torch.where(masks[j], z, slope * z)
        if scales is not None:
            x = x * scales[j].reshape(x.shape[0], x.shape[1], 1, 1)
        if j > 0:
            x = F.instance_norm(x, weight=sd[p + '3.weight'], bias=sd[p + '3.bias'], eps=eps)
        h.append(x)
    return F.linear(x.reshape(x.shape[0], -1), sd[prefix + 'adv_layer.weight'], sd[prefix + 'adv_layer.bias']), h


def disc_forward(sd, x, start_frames_wins, dropout_scales=None, wins=WINDOWS, reduction='stack', masks=None):
    """Discriminator(uncond).forward on mel x [B, T, F] -> (y or None, h).  ``start_frames_wins[i][0]`` is window i's start;
    ``masks[i]``: window i's leaky-relu masks (window_forward)."""
    x4 = x[:, None]
    len_max = int(x_len(x).max())
    ys, h = [], []
    for i, win in enumerate(wins):
        if len_max < win:
            continue
        s = start_frames_wins[i][0]
        y, h_ = window_forward(sd, f'discriminator.conv_layers.{i}.', x4[:, :, s:s + win],
                               None if dropout_scales is None else dropout_scales[i], masks=None if masks is None else masks[i])
        ys.append(y)
        h += h_
    if len(ys) != len(wins):
        return None, h
    return (torch.stack(ys, -1) if reduction == 'stack' else sum(ys)), h


def svb_adv_losses(sd, step, mel_outs, targets=None, starts=None, scales=None, masks=None):
    """The adversarial terms of one SVBVAEMleTask step, added to oracle/svb_vae_train.svb_train_losses by the caller.
      step 'g' (optimizer 0): {way}_a = MSE(D(mel_out), 1) * lambda_mel_adv for each way of ``mel_outs``;
      step 'd' (optimizer 1): {way}_r = MSE(D(target), 1), {way}_f = MSE(D(mel_out.detach()), 0);
      step 3   (optimizer 2): a2p_a = MSE(D(mel_out of a2p), 1) * lambda_mel_adv.
    Every discriminator call k (in the reference's order) uses ``starts[k]``, ``scales[k]`` (None: eval-mode dropout) and, when
    given, the leaky-relu masks ``masks[k]`` (disc_forward)."""
    calls = iter(range(1 << 30))

    def d(mel):
        k = next(calls)
        return disc_forward(sd, mel, starts[k], None if scales is None else scales[k], masks=None if masks is None else masks[k])[0]
    out = {}
    if step == 'g' or step == 3:
        for way, mel in mel_outs.items():
            if step == 3 and way != 'a2p':
                continue
            y = d(mel)
            if y is not None:
                out[f'{way}_a'] = F.mse_loss(y, torch.ones_like(y)) * LAMBDA_MEL_ADV
    elif step == 'd':
        for way, mel in mel_outs.items():
            y_r = d(targets[way])
            y_f = d(mel.detach())
            if y_f is not None:
                out[f'{way}_r'] = F.mse_loss(y_r, torch.ones_like(y_r))
                out[f'{way}_f'] = F.mse_loss(y_f, torch.zeros_like(y_f))
    else:
        raise ValueError(step)
    return out

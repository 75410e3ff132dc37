"""ORACLE tooling (test infrastructure only; see oracle/__init__.py): writes tests/golden/mel_disc.npz from the UNMODIFIED reference
mel discriminator (modules/fastspeech/multi_window_disc.py) the way oracle/gen_golden.py writes the other fixtures.

    NEURALSVB_REFERENCE=/path/to/NeuralSVB python -m oracle.gen_golden_mel_disc

Weights and mels are never stored: neuralsvb_b200/utils/synthetic.py regenerates them from the seeds.  Per case and mode:
y (None is stored as an absent key), the block outputs h, d mel and every parameter gradient of MSE(y, 1) by reference autograd,
float32 on the CPU.  h, d mel and the gradients are stored subsampled with their exact norms (_pack_grads).  Train-mode
Dropout2d factors are read back with forward hooks on the reference's Dropout2d modules (a plane is all zero or input / (1 - p)).
"""
import os
import sys
import warnings

import numpy as np
import torch

from neuralsvb_b200.utils import synthetic as S
from oracle import ref_harness as R
from oracle.gen_golden import DISC_GRAD_STRIDE, GRAD_STRIDE, OUT, SEED, _pack_grads

MEL_DISC_CASES = {
    # name: (B, T, trailing padding per clip, start frame per window (None: the window does not fit))
    'long': (2, 150, (0, 23), (5, 40, 13)),        # x_len = (150, 127): every window fits; x_len.max() = 150, not T - pad
    'short': (2, 60, (0, 7), (10, None, None)),    # x_len.max() = 60: the 64- and 128-frame windows are skipped, y is None
}


def build_reference():
    R.install()
    from modules.fastspeech.multi_window_disc import Discriminator
    m = Discriminator(time_lengths=[32, 64, 128], freq_length=80, hidden_size=128, kernel=(3, 3), cond_size=0, norm_type='in',
                      reduction='stack')
    m.load_state_dict(S.make_mel_disc_state_dict(SEED), strict=True)
    return m


def gen_mel_disc():
    m = build_reference()
    out = {}
    for name, (B, T, pad, starts) in MEL_DISC_CASES.items():
        mel = S.make_disc_mel(B, T, pad, SEED)
        for mode in ('train', 'eval'):
            m.train(mode == 'train')
            m.zero_grad()
            scales = []

            def hook(mod, inp, outp):
                a, o = inp[0].detach(), outp.detach()
                scales.append(((o.abs().sum((2, 3)) > 0) | (a.abs().sum((2, 3)) == 0)).float() / (1 - mod.p))
            hooks = [mod.register_forward_hook(hook) for mod in m.modules() if isinstance(mod, torch.nn.Dropout2d)]
            torch.manual_seed(SEED)
            x = mel.clone().requires_grad_(True)
            ret = m(x, start_frames_wins=[None if s is None else [s] * B for s in starts])
            for h in hooks:
                h.remove()
            p = f'{name}/{mode}'
            _pack_grads(out, f'{p}/h', [(str(i), t) for i, t in enumerate(ret['h'])], DISC_GRAD_STRIDE)
            out[f'{p}/n_h'] = np.int64(len(ret['h']))
            if ret['y'] is not None:
                y = ret['y']
                out[f'{p}/y'] = y.detach().numpy()
                torch.nn.functional.mse_loss(y, torch.ones_like(y)).backward()
                _pack_grads(out, f'{p}/dmel', [('x', x.grad)], GRAD_STRIDE)
                _pack_grads(out, f'{p}/grad', [(k, q.grad) for k, q in m.named_parameters()], DISC_GRAD_STRIDE)
            if mode == 'train':
                out[f'{p}/scales'] = torch.stack([s.reshape(-1) for s in scales]).numpy()
                assert ((out[f'{p}/scales'] == 0) | np.isclose(out[f'{p}/scales'], 4 / 3)).all()
        out[f'{name}/params'] = np.array([B, T] + list(pad) + [-1 if s is None else s for s in starts], np.int64)
    out['state_dict_keys'] = np.array(list(m.state_dict().keys()))
    out['state_dict_shapes'] = np.array([list(v.shape) + [0] * (4 - v.dim()) for v in m.state_dict().values()], np.int64)
    np.savez_compressed(os.path.join(OUT, 'mel_disc.npz'), **out)
    print('mel_disc.npz', {k: v.tolist() for k, v in out.items() if k.endswith('/y')})


def main():
    if not R.available():
        sys.exit('gen_golden_mel_disc needs NEURALSVB_REFERENCE = a checkout of the reference NeuralSVB')
    os.makedirs(OUT, exist_ok=True)
    warnings.simplefilter('ignore')
    gen_mel_disc()


if __name__ == '__main__':
    main()

"""The mel discriminator without a GPU: the float64 oracle (oracle/multi_window_disc.py) against the fixture written from the
unmodified reference (tests/golden/mel_disc.npz, oracle/gen_golden_mel_disc.py), the drop-in's state_dict names and shapes,
the x_len / window-start logic, and its refusals."""
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200.modules.fastspeech import multi_window_disc as M
from neuralsvb_b200.utils import synthetic as S
from oracle import multi_window_disc as OD
from oracle.gen_golden import DISC_GRAD_STRIDE, GRAD_STRIDE, grad_stride

GOLD = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'mel_disc.npz'))
CASES = ('long', 'short')


def case(name):
    p = GOLD[f'{name}/params']
    B, T = int(p[0]), int(p[1])
    pad, starts = [int(v) for v in p[2:2 + B]], [int(v) for v in p[2 + B:]]
    return B, T, pad, [None if s < 0 else [s] * B for s in starts]


def fixture_scales(name, B, C=128):
    """The captured train-mode Dropout2d factors as dropout_scales: per window that ran, per block, [B, C]."""
    s = torch.from_numpy(GOLD[f'{name}/train/scales']).reshape(-1, 3, B, C)
    return [[s[w, j] for j in range(3)] for w in range(s.shape[0])]


def rel(got, ref):
    return float(np.linalg.norm(np.asarray(got, np.float64) - ref) / max(np.linalg.norm(ref), 1e-30))


def check_packed(prefix, named, tol, stride=DISC_GRAD_STRIDE):
    """Against oracle/gen_golden._pack_grads: the exact norm and every stride-th element (all of a tensor up to 4096)."""
    for k, g in named:
        g = g.detach().double().reshape(-1)
        sub = GOLD[f'{prefix}/{k}/sub'].astype(np.float64)
        st = grad_stride(g.numel(), stride)
        assert g[::st].numel() == sub.size, (k, g.numel(), sub.size)
        assert abs(float(g.norm()) - float(GOLD[f'{prefix}/{k}/norm'])) <= tol * max(float(GOLD[f'{prefix}/{k}/norm']), 1e-30), k
        assert rel(g[::st].numpy(), sub) < tol, (k, rel(g[::st].numpy(), sub))


@pytest.mark.parametrize('mode', ['train', 'eval'])
@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference_fixture(name, mode):
    B, T, pad, starts = case(name)
    sd = {k: v.double().requires_grad_(True) for k, v in S.make_mel_disc_state_dict(1234).items()}
    x = S.make_disc_mel(B, T, pad, 1234).double().requires_grad_(True)
    scales = [[s.double() for s in w] for w in fixture_scales(name, B)] if mode == 'train' else None
    if scales is not None:       # windows that were skipped have no masks: pad the list to one entry per window
        scales = scales + [None] * (3 - len(scales))
    y, h = OD.disc_forward(sd, x, starts, scales)
    p = f'{name}/{mode}'
    assert len(h) == int(GOLD[f'{p}/n_h'])
    check_packed(f'{p}/h', [(str(i), t) for i, t in enumerate(h)], 1e-5)
    if f'{p}/y' not in GOLD:
        assert y is None
        return
    assert tuple(y.shape) == GOLD[f'{p}/y'].shape == (B, 1, 3)
    assert rel(y.detach().numpy(), GOLD[f'{p}/y']) < 1e-5
    torch.nn.functional.mse_loss(y, torch.ones_like(y)).backward()
    check_packed(f'{p}/dmel', [('x', x.grad)], 1e-5, GRAD_STRIDE)
    check_packed(f'{p}/grad', [(k, v.grad) for k, v in sd.items()], 2e-5)


def test_state_dict_names_and_shapes_match_reference():
    m = M.Discriminator(time_lengths=[32, 64, 128], freq_length=80, hidden_size=128, kernel=(3, 3), cond_size=0, norm_type='in',
                        reduction='stack')
    sd = m.state_dict()
    assert list(sd.keys()) == [str(k) for k in GOLD['state_dict_keys']]
    shapes = [[d for d in s if d] for s in GOLD['state_dict_shapes'].tolist()]
    assert [list(v.shape) for v in sd.values()] == shapes
    m.load_state_dict(S.make_mel_disc_state_dict(1234), strict=True)


def test_x_len_counts_nonzero_frames():
    x = S.make_disc_mel(3, 40, (0, 5, 40), 1234)
    x[0, 10] = 0.0                                    # an interior silent frame is not counted either
    x[0, 11, :2] = torch.tensor([1.0, -1.0])
    x[0, 11, 2:] = 0.0                                # bins that sum to 0 count as padding, as in the reference
    assert M.mel_x_len(x[:, None]).tolist() == [38, 35, 0]
    assert OD.x_len(x).tolist() == [38, 35, 0]


def test_clip_starts_range_skip_and_given():
    np.random.seed(0)
    seen = set()
    for _ in range(400):
        sfw = [None, None, None]
        fits = M.clip_starts(100, (32, 64, 128), sfw, 4)
        assert fits == [True, True, False] and sfw[2] is None
        assert len(sfw[0]) == 4 and len(set(sfw[0])) == 1 and 0 <= sfw[0][0] <= 68 and 0 <= sfw[1][0] <= 36
        seen.add(sfw[1][0])
    assert seen == set(range(37))                     # high end inclusive: randint(0, x_len.max() - win + 1)
    sfw = [[7, 7], None, [3, 3]]
    assert M.clip_starts(64, (32, 64, 128), sfw, 2) == [True, True, False]
    assert sfw[0] == [7, 7] and sfw[1] == [0, 0] and sfw[2] == [3, 3]
    # the reference draws exactly one numpy integer per window that fits, so a seeded run reproduces its starts
    np.random.seed(5)
    a = [None] * 3
    M.clip_starts(130, (32, 64, 128), a, 1)
    np.random.seed(5)
    assert a == [[np.random.randint(0, 99)], [np.random.randint(0, 67)], [np.random.randint(0, 3)]]


@pytest.mark.parametrize('kw', [dict(norm_type='bn'), dict(norm_type='sn'), dict(reduction='none'), dict(cond_size=256),
                                dict(reduction='mean')])
def test_unsupported_settings_raise_at_construction(kw):
    args = dict(time_lengths=[32, 64, 128], norm_type='in', reduction='stack')
    args.update(kw)
    with pytest.raises(NotImplementedError):
        M.Discriminator(**args)


def test_reduction_sum_and_cpu_refusal():
    m = M.Discriminator(norm_type='in', reduction='sum')
    assert m.discriminator.reduction == 'sum'
    with pytest.raises(RuntimeError, match='CUDA'):
        m(S.make_disc_mel(1, 40, (0,), 1234))


def test_oracle_with_its_own_masks_reproduces_leaky_relu():
    """The masked oracle (the form the GPU step tests use with the kernels' masks) given the float64 forward's own masks is
    plain float64 autograd: value and every gradient to 1e-12."""
    B, T, pad, starts = case('long')
    sd0 = S.make_mel_disc_state_dict(1234)
    x0 = S.make_disc_mel(B, T, pad, 1234).double()
    masks = []
    for i, win in enumerate(OD.WINDOWS):
        h, ms = x0[:, None, starts[i][0]:starts[i][0] + win], []
        for j in range(3):
            p = f'discriminator.conv_layers.{i}.model.{j}.'
            z = torch.nn.functional.conv2d(h, sd0[p + '0.weight'].double(), sd0[p + '0.bias'].double(), stride=2, padding=1)
            ms.append(z > 0)
            h = torch.nn.functional.leaky_relu(z, 0.2)
            if j > 0:
                h = torch.nn.functional.instance_norm(h, weight=sd0[p + '3.weight'].double(), bias=sd0[p + '3.bias'].double(), eps=1e-5)
        masks.append(ms)
    res = []
    for mk in (None, masks):
        sd = {k: v.double().requires_grad_(True) for k, v in sd0.items()}
        x = x0.clone().requires_grad_(True)
        y = OD.disc_forward(sd, x, starts, masks=mk)[0]
        torch.nn.functional.mse_loss(y, torch.ones_like(y)).backward()
        res.append([y.detach(), x.grad] + [v.grad for v in sd.values()])
    for a, b in zip(*res):
        assert float((a - b).abs().max()) <= 1e-12 * max(float(b.abs().max()), 1.0)


def test_non_float32_mel_is_refused():
    m = M.Discriminator(norm_type='in', reduction='stack')
    for dt in (torch.float16, torch.bfloat16, torch.float64):
        with pytest.raises(TypeError, match='float32'):
            m.discriminator(S.make_disc_mel(1, 40, (0,), 1234).to(dt)[:, None], torch.tensor([40]))

"""Host side of MleSVBVAE's length-aware mode (forward(..., amateur_lens=, prof_lens=)): the per-resolution frame counts against the
output lengths of the float64 oracle's convolutions, the refusal of bad lengths before any device work, the new C entries, and the
live tiles the ragged planner schedules for the beautifier's batches.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200 import _native
from tests.test_oracle_golden import SVB_HP

NEW_ENTRIES = ('svb_tc_layer_forward_ragged', 'svb_conv_nct_forward_ragged', 'svb_relpos_attention_nct_ragged',
               'svb_group_norm_relu_add_ragged', 'svb_global_latent_head_ragged')


def test_frame_counts_match_the_oracle_convolutions():
    """Every L from 60 to 5000 in steps of 4: the lengths oracle/vc_asr.py's mel prenet and oracle/fs2_vae.py's pre_net / g_pre_net
    and poolings produce on one unpadded clip (one channel, zeros: only the shapes matter)."""
    from neuralsvb_b200.modules.voice_conversion.svb_vae import frame_counts
    strides, s0 = SVB_HP['mel_strides'], 4
    for L in range(60, 5001, 4):
        c = frame_counts(L, strides, s0)
        x = torch.zeros(1, 1, L)
        for s in strides:                                    # oracle/vc_asr.py:prenet_forward
            x = F.conv1d(x, torch.zeros(1, 1, 5), stride=s, padding=2)
        assert c['ppg'] == x.shape[-1], L
        e = F.conv1d(torch.zeros(1, 1, L), torch.zeros(1, 1, 2 * s0), stride=s0, padding=s0 // 2)     # pre_net / g_pre_net
        assert c['enc'] == e.shape[-1] == L // s0, L
        pools = []
        for _ in range(3):
            e = F.conv1d(e, torch.zeros(1, 1, 3), stride=2)
            pools.append(e.shape[-1])
        assert c['pool'] == tuple(pools) and pools[-1] >= 1, L
        assert c['mel'] == L


def _model():
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    return MleSVBVAE(80, hp=SVB_HP).eval()


def _batch(Ta=312, Tp=336):
    z = lambda *s: torch.zeros(*s)
    return dict(amateur_mel=z(2, Ta, 80), prof_mel=z(2, Tp, 80), amateur_pitch=torch.ones(2, Ta, dtype=torch.long),
                prof_pitch=torch.ones(2, Tp, dtype=torch.long), amateur_spk_id=z(2, 256), prof_spk_id=z(2, 256),
                a2p_alignment=torch.zeros(2, Tp, dtype=torch.long), infer=False, concurrent_ways=['a2a', 'p2p', 'a2p'])


@pytest.mark.parametrize('la, lp, match', [
    ([300, 212], None, 'both'),
    (None, [236, 332], 'both'),
    ([300, 56], [236, 332], r'amateur_lens\[1\]: clip 1: 56 frames'),
    ([300, 210], [236, 332], r'amateur_lens\[1\]: clip 1: 210 frames: .*multiple of 4'),
    ([300, 212], [236, 340], r'prof_lens\[1\] = 340: clip 1 must have 1 to 336 frames'),
    ([300, 212.0], [236, 332], r'amateur_lens\[1\] = 212.0: a frame count is an int'),
    ([True, 212], [236, 332], r'amateur_lens\[0\] = True'),
    ([300], [236, 332], 'amateur_lens: 1 frame counts for a batch of 2 clips'),
])
def test_bad_lengths_raise_before_any_device_work(monkeypatch, la, lp, match):
    """CPU tensors: anything past the checks would raise a different error (there is no CPU path)."""
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    monkeypatch.setattr(MleSVBVAE, 'prepare_condition', lambda *a, **k: pytest.fail('device work before the checks'))
    with torch.no_grad(), pytest.raises(ValueError, match=match):
        _model()(**_batch(), amateur_lens=la, prof_lens=lp)


def test_lengths_accept_ints_numpy_ints_and_tensors():
    m = _model()
    assert m._check_lens('x', [np.int64(300), 212], 2, 312) == [300, 212]
    assert m._check_lens('x', torch.tensor([300, 60]), 2, 312) == [300, 60]


def test_length_mode_is_inference_only():
    from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
    m = MleSVBVAE(80, hp=SVB_HP, trainable=True).train()
    b = _batch()
    with pytest.raises(RuntimeError, match='inference only'):
        m(**{**b, 'amateur_mel': b['amateur_mel'].requires_grad_(False)}, amateur_lens=[300, 212], prof_lens=[236, 332])


def test_new_entries_are_declared_bound_and_exported():
    lib = ctypes.CDLL(_native.LIB_PATH if os.path.exists(_native.LIB_PATH) else _native.build())
    for name in NEW_ENTRIES:
        assert name in _native.declared_symbols(), name
        assert name in _native._PROTOS, name
        assert hasattr(lib, name), name


def _live_items(lengths, Cin=256):
    from tests.test_tc_ragged_schedule import ragged
    items, _, _, _ = ragged([5], [0], [0], lengths, MT=1, Cin=Cin)
    return items


def test_ragged_planner_schedules_only_live_tiles():
    """The song batch of tests/test_gpu_svb_vae_beautify_sizes (a 780-frame tail padded to 5000 frames) and a 60-frame clip beside a
    5000-frame one: the planner's items cover each clip's ceil(L / 128) tiles and nothing of its padding."""
    for lengths in ([4996] * 9 + [780], [60, 5000]):
        items = _live_items(lengths)
        live = sum(-(-L // 128) for L in lengths)
        padded = len(lengths) * -(-max(lengths) // 128)
        assert len(items) == live, (lengths, len(items), live)
        for it in items:
            assert it[3] < lengths[it[2]], it                 # no item starts at or past its clip's end
        print(f'TILES {lengths}: {live} live of {padded} padded 128-row tiles per layer')

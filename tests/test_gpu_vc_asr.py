"""PPG extractor (SURVEY 8(f) N1): the encoder half of VCASR (modules/voice_conversion/vc_modules.py:56-80) on the native convs,
LayerNorm and rel-pos attention kernels, against the fixture generated from the reference class."""
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200.utils import synthetic as S

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'vc_asr.npz')


def _model():
    from neuralsvb_b200.modules.voice_conversion.vc_modules import VCASR
    m = VCASR(80, 80, hidden_size=256, asr_enc_layers=2, mel_strides=[2, 1, 1], asr_last_norm=False)
    sd = S.make_vc_asr_state_dict(1234)
    sd['asr_decoder.layers.0.dummy'] = torch.zeros(1)          # checkpoint keys of the training head are ignored
    m.load_state_dict(sd, strict=True)
    return m.eval().cuda()


def test_vc_asr_h_content_matches_reference_fixture():
    g = np.load(GOLDEN)
    B, T = [int(v) for v in g['params']]
    with torch.no_grad():
        h = _model()(S.make_vc_asr_mel(B, T, 1234).cuda())['h_content'].cpu().numpy()
    ref = g['h_content']
    assert h.shape == ref.shape
    rel = float(np.abs(h - ref).max() / np.abs(ref).max())
    assert rel < 1e-4, rel                    # fp32 kernels throughout; the north-star asks 1e-3 relative L-inf on spectral features
    assert np.all(h[1, -9 // 2:] == 0.0)      # padded frames stay exactly zero (conformer.py:51)

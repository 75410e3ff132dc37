"""-m gpu: two-tile work items of the wgmma convolution (conv_tc.cu), with the one-tile item at the end of a clip whose
tile count is odd, in the same launch: a single layer on the implicit round-robin list and the merged ResBlock launches
of the generator on host-built lists.  The plan is read back from SVB_TC_VERBOSE to make sure MT = 2 was taken."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200.utils import synthetic as S
from oracle import hifigan as O
from tests import gpu_util as U
from tests.test_gpu_conv_kernels import TOL, run_layer

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('precision', ['tf32', 'tf32x3', 'bf16x3'])
def test_two_tile_items_with_an_odd_tile_tail_match_float64_torch(precision, monkeypatch, capfd):
    """Cin = Cout = 64, k 11 d 5, 334 rows = 3 tiles per clip (the third partial): items (2 tiles, 1 tile) per clip.
    B = SMs / 2 clips keep the two-tile list at one wave, so the plan takes MT = 2."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B, C, T, K, dil = sms // 2, 64, 3 * 128 - 50, 11, 5
    g = torch.Generator().manual_seed(4321)
    x = torch.randn(B, C, T, generator=g).cuda() * 2
    w = (torch.randn(C, C, K, generator=g) / np.sqrt(C * K)).cuda()
    b = torch.randn(C, generator=g).cuda() * 0.1
    res = torch.randn(B, C, T, generator=g).cuda()
    monkeypatch.setenv('SVB_TC_VERBOSE', '1')
    y, _ = run_layer(x, w, b, res, K, dil, 0, 0.1, 0.5, precision)
    torch.cuda.synchronize()
    plan = capfd.readouterr().err
    assert 'MT 2' in plan, plan
    ref = (F.conv1d(F.leaky_relu(x.double(), 0.1), w.double(), b.double(), dilation=dil, padding=dil * (K - 1) // 2) + res.double()) * 0.5
    err = float((y.double() - ref).abs().max() / ref.abs().max())
    assert err < TOL[precision], f'{precision}: rel L-inf {err:.3e}'


@pytest.mark.parametrize('precision', ['bf16x3', 'tf32x3'])
def test_merged_launches_with_an_odd_tile_tail_match_oracle(precision, monkeypatch, capfd):
    """hop-256 generator, 4 clips x 41 frames: stage 2 (C = 64) runs 5248 rows = 41 tiles per clip, and its merged c1 and
    (chain-ordered) c2 work lists mix two-tile and one-tile items; every stage boundary against the oracle at the bar of
    test_generator_layers_match_oracle."""
    from tests.test_native_abi import _schedule
    cfg, B, T = 'hop256', 4, 41
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for chain in (False, True):
        items, _, _ = _schedule([3, 7, 11], [int(chain)] * 3, [0, int(chain), int(chain)], B, T * 128, 2, 1, chain, grid=sms, Cin=64)
        assert set(items[:, 4].tolist()) == {1, 2}, (chain, sms)
    h, hop, mel, f0, ri, nz = U.inputs(cfg, True, B, T)
    m = U.cuda_generator(cfg, True, precision)
    monkeypatch.setenv('SVB_TC_VERBOSE', '1')
    y = m(mel.cuda(), f0.cuda(), rand_ini=ri.cuda(), noise=nz.cuda()).cpu().numpy()
    plan = capfd.readouterr().err
    assert any('3 layer(s)' in l and f'Tq {T * 128} ' in l and 'MT 2' in l for l in plan.splitlines()), plan
    w = O.fold_weight_norm(S.make_generator_state_dict(h, U.SEED))
    taps = {}
    with torch.no_grad():
        y_o = O.generator_forward(w, h, mel, f0, ri, nz, taps).numpy()
    for name, ref in taps.items():
        got = m.get_tap(name).cpu().numpy()
        assert got.shape == tuple(ref.shape), name
        rel = np.abs(got - ref.numpy()).max() / np.abs(ref.numpy()).max()
        assert rel < 5e-5, f'{name}: rel L-inf {rel:.3e}'
    assert U.rms(y, y_o) < 1e-4

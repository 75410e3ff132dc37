"""-m gpu: single conv layers through the C ABI (svb_conv1d_run) -- the CUDA-core kernel and the
wgmma kernel (1xTF32, 3xTF32) against a float64 torch convolution of the same layer."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200 import _native

pytestmark = pytest.mark.gpu

# (B, Cin, Cout, T, K, dil, transposed stride u, residual[, in_slope = 0.1])
LAYERS = [
    (2, 32, 32, 300, 3, 1, 0, True),
    (2, 32, 32, 700, 11, 5, 0, True),
    (1, 64, 64, 513, 7, 3, 0, False),
    (2, 128, 128, 384, 11, 1, 0, True),
    (2, 256, 256, 256, 3, 3, 0, True),
    (1, 256, 256, 1024, 11, 5, 0, True),
    (2, 64, 32, 200, 4, 0, 2, False),
    (1, 512, 256, 96, 16, 0, 8, False),
    (1, 80, 512, 60, 7, 1, 0, False),          # conv_pre shape: Cin padded to 96 on the tensor-core path
    (2, 64, 96, 300, 5, 1, 0, True),           # the N = 96 instantiation
    (2, 64, 160, 300, 3, 1, 0, False),         # n_tile 32 x 5 column blocks
    (2, 48, 64, 300, 7, 1, 0, True),           # a partial 32-channel input chunk
    (1, 32, 32, 1, 3, 1, 0, True),             # a single row
    (2, 32, 64, 5, 11, 5, 0, True),            # halo (25 rows) wider than the clip
    (3, 64, 64, 200, 3, 1, 0, True, 1.0),      # odd batch, identity slope
]
TOL = {'fp32': 2e-5, 'tf32x3': 3e-5, 'bf16x3': 1e-4, 'tf32': 3e-3}   # relative to max |y|


def run_layer(x, w, b, res, K, dil, u, slope, scale, precision, iters=1):
    lib = _native.lib()
    B, Cin, T = x.shape
    Cout = w.shape[1] if u else w.shape[0]
    Tout = T * u if u else T
    y = torch.empty(B, Cout, Tout, device='cuda')
    ms = ctypes.c_float(0)
    wc, bc = w.cpu().contiguous(), b.cpu().contiguous()
    rc = lib.svb_conv1d_run(_native.ptr(x), _native.ptr(wc), _native.ptr(bc), _native.ptr(res), B, Cin, Cout, T, K,
                            dil, u, slope, scale, _native.PREC[precision], iters, _native.ptr(y), ctypes.byref(ms),
                            _native.current_stream_ptr())
    _native.check(rc, 'conv1d_run')
    return y, ms.value


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'tf32x3', 'bf16x3'])
@pytest.mark.parametrize('layer', LAYERS)
def test_conv_layer_matches_float64_torch(layer, precision):
    B, Cin, Cout, T, K, dil, u, with_res = layer[:8]
    slope = layer[8] if len(layer) > 8 else 0.1
    g = torch.Generator().manual_seed(1234 + Cin + K)
    x = torch.randn(B, Cin, T, generator=g).cuda() * 2
    wshape = (Cin, Cout, K) if u else (Cout, Cin, K)
    w = (torch.randn(*wshape, generator=g) / np.sqrt(Cin * K / max(u, 1))).cuda()
    b = torch.randn(Cout, generator=g).cuda() * 0.1
    Tout = T * u if u else T
    res = torch.randn(B, Cout, Tout, generator=g).cuda() if with_res else None
    scale = 1.0 / 3
    y, _ = run_layer(x, w, b, res, K, dil, u, slope, scale, precision)
    xd = F.leaky_relu(x.double(), slope)
    if u:
        ref = F.conv_transpose1d(xd, w.double(), b.double(), stride=u, padding=(K - u) // 2)
    else:
        ref = F.conv1d(xd, w.double(), b.double(), dilation=dil, padding=dil * (K - 1) // 2)
    if res is not None:
        ref = ref + res.double()
    ref = ref * scale
    err = float((y.double() - ref).abs().max() / ref.abs().max())
    assert err < TOL[precision], f'{layer} {precision}: rel L-inf {err:.3e}'


@pytest.mark.parametrize('precision', ['tf32', 'tf32x3', 'bf16x3'])
def test_conv_layer_batch_slicing_matches_float64_torch(precision):
    """A launch with more work items per CTA than the kernel's shared-memory list holds (kMaxItems = 120, conv_tc.cu)
    runs the batch in slices of clips.  Cin 32 -> Cout 1024 (8 column blocks of 128), 16000 rows = 125 tiles per clip;
    the batch is sized from this GPU's SM count so that the launch slices on any H100."""
    B_items = 125 * 8
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 120 * sms // B_items + 1
    assert -(-B * B_items // sms) > 120
    Cin, Cout, T, K = 32, 1024, 16000, 3
    g = torch.Generator().manual_seed(99)
    x = torch.randn(B, Cin, T, generator=g).cuda()
    w = (torch.randn(Cout, Cin, K, generator=g) / np.sqrt(Cin * K)).cuda()
    b = torch.randn(Cout, generator=g).cuda() * 0.1
    res = torch.randn(B, Cout, T, generator=g).cuda()
    y, _ = run_layer(x, w, b, res, K, 1, 0, 0.1, 0.5, precision)
    ref = F.conv1d(F.leaky_relu(x.double(), 0.1), w.double(), b.double(), padding=1).add_(res.double()).mul_(0.5)
    ref_max = float(ref.abs().max())
    per_clip = ref.sub_(y.double()).abs_().amax(dim=(1, 2))      # a slice at the wrong offset shows in its clips
    del ref
    worst = float(per_clip.max()) / ref_max
    assert worst < TOL[precision], f'B {B} {precision}: rel L-inf {worst:.3e} (worst clip {int(per_clip.argmax())})'

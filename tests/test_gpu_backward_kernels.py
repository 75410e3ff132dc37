"""-m gpu: the backward of single conv layers through svb_conv1d_backward_run -- the launchers and argument mappings
the generator's backward uses (wgrad_tc.cu or the fp32 weight-gradient kernel, the column sum, the data-gradient conv on
flipped weights plus the leaky-relu mask, the ConvTranspose1d data gradient) -- against float64 torch autograd of
F.conv1d / F.conv_transpose1d on the same tensors.  Every gradient is compared per tensor in relative L2 and in
L-inf relative to max |reference|."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from neuralsvb_b200 import _native

pytestmark = pytest.mark.gpu

PRECISIONS = ['fp32', 'tf32', 'tf32x3', 'bf16x3']

# (B, Cin, Cout, T, K, dil, slope), stride 1: each shape takes one branch of wgrad_tc.cu
STRIDE1 = [
    (2, 32, 32, 300, 3, 1, .1),         # N = 64, one A group (nxa = 1), tap sets 2 + 1
    (2, 32, 32, 700, 11, 5, .1),        # reach 50 rows, 6 tap sets, A slab of 178 rows
    (1, 64, 64, 513, 7, 3, .1),         # N = 128, one full pair of A groups
    (3, 96, 96, 257, 5, 1, .1),         # odd group count: last pair nxa = 1, last coset ng = 1 under N = 128 (masked half tile)
    (2, 128, 128, 384, 11, 1, .1),      # the generator's ResBlock shapes
    (2, 256, 256, 1000, 3, 3, .1),
    (1, 256, 256, 1024, 11, 5, .1),
    (1, 512, 512, 96, 7, 1, .1),        # Tq < 128 (hop-256 stage 0 at 12 frames)
    (2, 80, 512, 60, 7, 1, 1.0),        # conv_pre: 80 channels padded to 96, identity slope
    (1, 32, 32, 1, 3, 1, .1),           # a single row
    (16, 128, 128, 1024, 11, 1, .1),    # many units per CTA (splits < units): ring wrap-around and stage parity
]
# (B, Cin, Cout, T, K, u): the hop-256 upsamplers (ConvTranspose1d, padding (K - u) / 2), fp32 kernels in every mode
TRANSPOSED = [
    (2, 512, 256, 12, 16, 8),
    (2, 256, 128, 96, 16, 8),
    (2, 128, 64, 768, 4, 2),
    (2, 64, 32, 1536, 4, 2),
]

# Bars per (tensor, precision): (relative L2, relative L-inf), about 5x the worst error measured over STRIDE1 on an
# H100 80GB HBM3 (400 W power limit):
#   dw  fp32 5.0e-7 / 6.0e-7   tf32, tf32x3, bf16x3 (all split-bf16 on wgrad_tc) 5.3e-6 / 5.7e-6
#   db  every mode (fp32 column sum) 2.3e-7 / 3.6e-7
#   dx  fp32 1.1e-6 / 2.9e-6   tf32 3.8e-4 / 5.4e-4   tf32x3 2.5e-5 / 2.6e-5   bf16x3 1.3e-5 / 1.3e-5
# The data gradient follows the forward kernel's mode (conv_pre's 80 output channels take the fp32 kernel in every mode).
# A dropped hi*lo cross term costs ~2^-9 = 2e-3 relative: 60x the tensor-core dw bar (and 25x the bf16x3 dx bar).
_DW_TC, _DB = (3e-5, 3e-5), (2e-6, 2e-6)
TOL = {
    ('dw', 'fp32'): (3e-6, 3e-6), ('dw', 'tf32'): _DW_TC, ('dw', 'tf32x3'): _DW_TC, ('dw', 'bf16x3'): _DW_TC,
    ('db', 'fp32'): _DB, ('db', 'tf32'): _DB, ('db', 'tf32x3'): _DB, ('db', 'bf16x3'): _DB,
    ('dx', 'fp32'): (6e-6, 1.5e-5), ('dx', 'tf32'): (2e-3, 3e-3), ('dx', 'tf32x3'): (1.3e-4, 1.3e-4), ('dx', 'bf16x3'): (7e-5, 7e-5),
}
# transposed layers, fp32 kernels in every mode; measured worst dx 1.1e-6 / 2.1e-6, dw 2.1e-7 / 3.7e-7, db 1.8e-7 / 2.6e-7
TOL_T = {'dx': (6e-6, 1.1e-5), 'dw': (1e-6, 2e-6), 'db': (1e-6, 1.5e-6)}


def run_backward(x, w, dy, K, dil, u, slope, precision, dw=None, db=None):
    """One call of svb_conv1d_backward_run; dw / db are accumulated into (zeros unless given), dx is returned."""
    lib = _native.lib()
    B, Cin, T = x.shape
    Cout = w.shape[1] if u else w.shape[0]
    dx = torch.full_like(x, float('nan'))          # written in full, never read
    dw = torch.zeros(w.shape, device='cuda') if dw is None else dw
    db = torch.zeros(Cout, device='cuda') if db is None else db
    wc = w.cpu().contiguous()
    rc = lib.svb_conv1d_backward_run(_native.ptr(x), _native.ptr(wc), _native.ptr(dy), B, Cin, Cout, T, K, dil, u,
                                     ctypes.c_float(slope), _native.PREC[precision], _native.ptr(dx), _native.ptr(dw),
                                     _native.ptr(db), _native.current_stream_ptr())
    _native.check(rc, 'conv1d_backward_run')
    return dx, dw, db


def make_case(B, Cin, Cout, T, K, dil, u, slope):
    g = torch.Generator().manual_seed(4321 + Cin + 7 * Cout + K + T)
    x = (torch.randn(B, Cin, T, generator=g) * 2).cuda()
    wshape = (Cin, Cout, K) if u else (Cout, Cin, K)
    w = (torch.randn(*wshape, generator=g) / np.sqrt(Cin * K / max(u, 1))).cuda()
    Tout = T * u if u else T
    dy = torch.randn(B, Cout, Tout, generator=g).cuda()
    return x, w, dy


def reference(x, w, dy, K, dil, u, slope):
    """float64 autograd on the GPU.  The mask is lrelu'(x) as the kernels see it (x >= 0 -> 1): x is an input, so it is the
    exact mask -- what is compared is the convolution's gradient."""
    a = F.leaky_relu(x.double(), slope).requires_grad_(True)
    wd = w.double().requires_grad_(True)
    bd = torch.zeros(w.shape[1] if u else w.shape[0], dtype=torch.float64, device='cuda', requires_grad=True)
    if u:
        y = F.conv_transpose1d(a, wd, bd, stride=u, padding=(K - u) // 2)
    else:
        y = F.conv1d(a, wd, bd, dilation=dil, padding=dil * (K - 1) // 2)
    y.backward(dy.double())
    mask = torch.where(x >= 0, 1.0, slope).double()
    return a.grad * mask, wd.grad, bd.grad


def errors(got, ref):
    d = got.double() - ref
    return float(d.norm() / ref.norm()), float(d.abs().max() / ref.abs().max())


_refs = {}


def _case(key, K, dil, u, slope, build):
    if key not in _refs:
        _refs.clear()                   # one shape at a time: the references of the large shapes are big
        x, w, dy = build()
        _refs[key] = (x, w, dy, reference(x, w, dy, K, dil, u, slope))
    return _refs[key]


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('shape', STRIDE1, ids=lambda s: 'B{}_C{}x{}_T{}_K{}_d{}_s{}'.format(*s))
def test_conv_backward_matches_float64_torch(shape, precision):
    B, Cin, Cout, T, K, dil, slope = shape
    x, w, dy, (dx_r, dw_r, db_r) = _case(shape, K, dil, 0, slope, lambda: make_case(B, Cin, Cout, T, K, dil, 0, slope))
    dx, dw, db = run_backward(x, w, dy, K, dil, 0, slope, precision)
    e = {'dx': errors(dx, dx_r), 'dw': errors(dw, dw_r), 'db': errors(db, db_r)}
    print('MEASURED', shape, precision, {k: f'{a:.2e}/{b:.2e}' for k, (a, b) in e.items()})
    bad = {k: v for k, v in e.items() if v[0] > TOL[k, precision][0] or v[1] > TOL[k, precision][1]}
    assert not bad, f'{shape} {precision}: (rel L2, rel L-inf) {bad}'


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('shape', TRANSPOSED, ids=lambda s: 'B{}_C{}x{}_T{}_K{}_u{}'.format(*s))
def test_conv_transpose_backward_matches_float64_torch(shape, precision):
    B, Cin, Cout, T, K, u = shape
    x, w, dy, (dx_r, dw_r, db_r) = _case(shape, K, 1, u, 0.1, lambda: make_case(B, Cin, Cout, T, K, 1, u, 0.1))
    dx, dw, db = run_backward(x, w, dy, K, 1, u, 0.1, precision)
    e = {'dx': errors(dx, dx_r), 'dw': errors(dw, dw_r), 'db': errors(db, db_r)}
    print('MEASURED', shape, precision, {k: f'{a:.2e}/{b:.2e}' for k, (a, b) in e.items()})
    bad = {k: v for k, v in e.items() if v[0] > TOL_T[k][0] or v[1] > TOL_T[k][1]}
    assert not bad, f'{shape} {precision}: (rel L2, rel L-inf) {bad}'


@pytest.mark.parametrize('shape,precision', [((2, 64, 64, 513, 7, 3, 0, .1), 'bf16x3'),      # wgrad_tc
                                             ((2, 32, 32, 300, 3, 1, 0, .1), 'fp32'),        # fp32 weight-gradient kernel
                                             ((2, 128, 64, 768, 4, 1, 2, .1), 'fp32')])      # ConvTranspose1d
def test_backward_accumulates_weight_and_bias_gradients(shape, precision):
    """dw / db are accumulated (the generator sums the gradients of a step into one buffer), dx is overwritten."""
    B, Cin, Cout, T, K, dil, u, slope = shape
    x, w, dy = make_case(B, Cin, Cout, T, K, dil, u, slope)
    dx1, dw1, db1 = run_backward(x, w, dy, K, dil, u, slope, precision)
    dw, db = dw1.clone(), db1.clone()
    dx2, dw2, db2 = run_backward(x, w, dy, K, dil, u, slope, precision, dw=dw, db=db)
    assert dw2 is dw and db2 is db
    for got, once in ((dw2, dw1), (db2, db1)):
        assert errors(got, 2 * once.double())[1] < 1e-6
    assert errors(dx2, dx1.double())[1] < 1e-6

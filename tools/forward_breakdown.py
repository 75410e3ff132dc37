#!/usr/bin/env python
"""Per-launch time breakdown of the benchmark's generator forward (bench.py: config 2, 16 clips x 128 frames).

    python tools/forward_breakdown.py [--precision bf16x3] [--steps 10] [--mt 2] [--json OUT]

svb_gen_enable_timing(handle, 2) records one CUDA-event pair around every launch, in launch order (the NSF source
then runs on the main stream, so the records are serial).  Each record is labelled from the generator config:
mel layout, NSF source, conv_pre, and per upsampling stage the upsampler, noise_conv_add and, per dilation step m,
the merged c1 and c2 launches of the three ResBlock chains -- or, in the C <= 64 stages, ONE fused launch per step that
runs c1 and c2 (not in tf32x3, whose layout does not fit; SVB_FUSE=0 labels a build or handle without fused launches);
conv_post last.  Per launch class it prints:

* ms (mean over the timed forwards);
* tensor fraction: algorithmic FLOPs / (ms x the operand mode's dense peak), the peak (H100 SXM data sheet, 989 TFLOP/s
  bf16 at a 1980 MHz boost clock) scaled to the SM clock sampled during the timed forwards;
* GB/s of the layer-streaming byte model (input once, output once, residual / running sum once);
* modelled L2 -> shared-memory weight bytes: every work item streams the (column block, input chunk, tap) tiles
  of its layer once, so the bytes scale with 1 / tiles per item (MT, `--mt`; balance splits into one-tile items are
  not modelled); resident-weight launches (C = 32) load each layer's tiles once per CTA.  A fused item (P = 246
  output rows, 256 c1 rows) streams the tiles of both convolutions through the ring.
"""
import argparse
import contextlib
import ctypes
import io
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import B_CLIPS, T_FRAMES, ClockSampler  # noqa: E402
from neuralsvb_b200.utils import synthetic as S  # noqa: E402

BF16_PEAK_TFLOPS, PEAK_MHZ = 989.0, 1980.0
MODE_DIV = {'tf32': 2.0, 'tf32x3': 6.0, 'bf16x3': 3.0}     # dense peak of the operand mode = bf16 peak / this
PLANES = {'tf32': 1, 'tf32x3': 2, 'bf16x3': 1}


def n_tile_of(coutp):
    if coutp <= 128:
        return coutp
    return next(n for n in range(128, 31, -32) if coutp % n == 0)


def weight_bytes(precision, cin, coutp, ks_list, B, rows, mt, grid=132):
    """Modelled L2 -> smem weight bytes of one launch over the layers with taps `ks_list` (same shape class)."""
    n = n_tile_of(coutp)
    tile = n * 128 * PLANES[precision]
    chunks, blocks = (cin + 31) // 32, coutp // n
    tiles = (rows + 127) // 128
    m = mt if tiles >= 2 else 1
    if chunks == 1 and blocks == 1:                        # resident: every CTA loads all layers' tiles once
        return grid * sum(ks_list) * tile
    items = blocks * B * ((tiles + m - 1) // m)
    return sum(items * chunks * k * tile for k in ks_list)


def fused_weight_bytes(precision, C, ks_list, B, rows, P=246):
    """Modelled L2 -> smem weight bytes of one fused launch: every item streams c1's and c2's tiles once."""
    tile = C * 128 * PLANES[precision]
    items = B * ((rows + P - 1) // P)
    return sum(items * (C // 32) * 2 * k * tile for k in ks_list)


def labels(h, B, T, precision, mt, fuse=True):
    """(label, class, modelled weight bytes) per record, in the generator's launch order (every stage merged; the C <= 64
    stages fused unless `fuse` is off or the precision is tf32x3)."""
    out = [('mel layout', 'mel layout', 0.0), ('nsf source', 'nsf source', 0.0)]
    C0 = h['upsample_initial_channel']
    out.append(('conv_pre', 'conv_pre', weight_bytes(precision, h['audio_num_mel_bins'], C0, [7], B, T, mt)))
    Tin, Cin = T, C0
    ks = h['resblock_kernel_sizes']
    for i, (u, k) in enumerate(zip(h['upsample_rates'], h['upsample_kernel_sizes'])):
        C = Cin // 2
        out.append((f'stage{i} ups', f'stage{i} (C={C}) upsampler', weight_bytes(precision, Cin, u * C, [3], B, Tin, mt)))
        out.append((f'stage{i} noise_conv_add', 'noise_conv_add', 0.0))
        Ti = Tin * u
        for m, _ in enumerate(h['resblock_dilation_sizes'][0]):
            if fuse and C <= 64 and precision != 'tf32x3':
                out.append((f'stage{i} m{m} c1+c2', f'stage{i} (C={C}) c1+c2 fused', fused_weight_bytes(precision, C, ks, B, Ti)))
                continue
            wb = weight_bytes(precision, C, C, ks, B, Ti, mt)
            out.append((f'stage{i} m{m} c1', f'stage{i} (C={C}) c1', wb))
            out.append((f'stage{i} m{m} c2', f'stage{i} (C={C}) c2', wb))
        Tin, Cin = Ti, C
    out.append(('conv_post', 'conv_post', 0.0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--precision', default='bf16x3', choices=['tf32', 'tf32x3', 'bf16x3'])
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--mt', type=int, default=2, choices=[1, 2], help='tiles per work item in the weight-byte model')
    ap.add_argument('--json', help='also write the table as JSON to this path')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('forward_breakdown.py: no CUDA device')
    from neuralsvb_b200 import _native
    from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator

    dev = torch.device('cuda', 0)
    h = S.hifigan_config()
    model = HifiGanGenerator(h, precision=args.precision)
    model.load_state_dict(S.make_generator_state_dict(h, 1234), strict=True)
    with contextlib.redirect_stdout(io.StringIO()):
        model.remove_weight_norm()
    model = model.eval().to(dev)
    lib, handle = _native.lib(), model.native_handle(dev)
    mel, f0 = (t.to(dev) for t in S.make_mel_f0(B_CLIPS, T_FRAMES, 1234))
    lab = labels(h, B_CLIPS, T_FRAMES, args.precision, args.mt, fuse=os.environ.get('SVB_FUSE', '1') != '0')
    name = ctypes.create_string_buffer(64)
    ms, by, fl = ctypes.c_float(), ctypes.c_double(), ctypes.c_double()
    rec = None
    with torch.no_grad():
        for _ in range(3):
            model(mel, f0)
        torch.cuda.synchronize()
        _native.check(lib.svb_gen_enable_timing(handle, 2), 'enable_timing')
        with ClockSampler(0) as clk:
            for s in range(args.steps):
                model(mel, f0)
                torch.cuda.synchronize()
                n = lib.svb_gen_profile_count(handle)
                if n != len(lab):
                    sys.exit(f'forward_breakdown.py: {n} timed launches, the config predicts {len(lab)} (a stage did not merge?)')
                if rec is None:
                    rec = np.zeros((n, 3))
                for i in range(n):
                    _native.check(lib.svb_gen_profile_get(handle, i, name, 64, ctypes.byref(ms), ctypes.byref(by), ctypes.byref(fl)),
                                  'profile_get')
                    rec[i] += (ms.value, by.value, fl.value)
        _native.check(lib.svb_gen_enable_timing(handle, 0), 'enable_timing')
    rec /= args.steps
    clocks = clk.summary()
    mhz = clocks['sm_mhz'] or PEAK_MHZ
    peak = BF16_PEAK_TFLOPS / MODE_DIV[args.precision] * mhz / PEAK_MHZ
    classes = {}
    for (label, cls, wb), (t, b, f) in zip(lab, rec):
        d = classes.setdefault(cls, {'launches': 0, 'ms': 0.0, 'bytes': 0.0, 'flops': 0.0, 'l2_weight_bytes': 0.0})
        d['launches'] += 1
        d['ms'] += t
        d['bytes'] += b
        d['flops'] += f
        d['l2_weight_bytes'] += wb
    total = float(rec[:, 0].sum())
    print(f'{torch.cuda.get_device_name(dev)}, power limit {clocks["power_limit_w"]} W, SM clock median {clocks["sm_mhz"]} MHz '
          f'({clocks["samples"]} samples), {args.precision}, {args.steps} timed forwards, sum of launch times {total:.3f} ms')
    print(f'{"launch class":28s} {"n":>3s} {"ms":>8s} {"share":>6s} {"tensor":>7s} {"GB/s":>7s} {"L2 wgt GB":>9s}')
    for cls, d in classes.items():
        d['tensor_frac'] = d['flops'] / (d['ms'] * 1e-3) / (peak * 1e12) if d['flops'] else 0.0
        d['gbs'] = d['bytes'] / (d['ms'] * 1e-3) / 1e9
        print(f'{cls:28s} {d["launches"]:3d} {d["ms"]:8.3f} {d["ms"] / total:6.1%} {d["tensor_frac"]:7.3f} {d["gbs"]:7.0f} '
              f'{d["l2_weight_bytes"] / 1e9:9.2f}')
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as fh:
            json.dump({'gpu': torch.cuda.get_device_name(dev), 'clocks': clocks, 'precision': args.precision, 'mt_model': args.mt,
                       'tensor_peak_tflops_at_clock': peak, 'total_ms': total, 'classes': classes,
                       'launches': [{'label': l, 'ms': float(t), 'bytes': float(b), 'flops': float(f), 'l2_weight_bytes': wb}
                                    for (l, _, wb), (t, b, f) in zip(lab, rec)]}, fh, indent=1)


if __name__ == '__main__':
    main()

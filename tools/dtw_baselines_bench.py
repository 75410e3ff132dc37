"""Baseline pitch alignments on the GPU (csrc/sadtw.cu: LoNDTW, NaiveDTW, ZMNaiveDTW, NNaiveDTW, NInterpo): prints one JSON line.

    python tools/dtw_baselines_bench.py [--pairs 256] [--frames 1378] [--reps 10] [--oracle-pairs 2] [--out result.json]

Per method, on `pairs` pairs of about 8 s (frames +- 15 %, float32 f0; NaiveDTW also on [S, 80] float32 mels, the paper's
clean-mel upper bound):
  * device_ms_per_batch: align_batch on inputs already on the device, CUDA events around the call (metadata upload included);
  * stage_ms (per-frame features, cost, dtw, backtrack) from the entry point's CUDA events;
  * the cost kernel's achieved FLOP/s against the FP32 data-sheet rate and its bytes/s against HBM bandwidth, and which bounds it;
  * the CPU baseline is the oracle (oracle/dtw_baselines.py: torch.cdist and the vectorised numpy DTW) on this host, per pair.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from neuralsvb_b200.modules.voice_conversion.dtw import core  # noqa: E402
from neuralsvb_b200.utils import synthetic as S  # noqa: E402

HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet
FP32_FLOP_PER_S = 67e12              # H100 SXM data sheet, dense FP32


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:           # the query is informational
        q = f'unavailable ({e})'
    return name, q


def events_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def cost_work(method, K, cells, frames, esz):
    """(FLOP, bytes) the cost kernel needs: per cell K products and K + 2 additions, a clamp and a square root (counted as 1);
    bytes: the cost written once plus every input row and per-frame value read once."""
    flop = cells * (2 * K + 3)
    return flop, cells * esz + frames * (K if method == 'NaiveDTW' else 1) * esz * 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=256)
    ap.add_argument('--frames', type=int, default=1378)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--oracle-pairs', type=int, default=2)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('dtw_baselines_bench needs a CUDA device')
    name, power = card()
    rs = np.random.RandomState(2026)
    lens = [(int(a.frames * rs.uniform(0.85, 1.15)), int(a.frames * rs.uniform(0.85, 1.15))) for _ in range(a.pairs)]
    host = [S.make_f0_pair(1000 + p, s, t) for p, (s, t) in enumerate(lens)]
    f0_src = [torch.from_numpy(x.astype(np.float32)).cuda() for x, _ in host]
    f0_tgt = [torch.from_numpy(y.astype(np.float32)).cuda() for _, y in host]
    mel_src = [S.make_mel_pair(1, s, [0], 3000 + p)[1][0].cuda() for p, (s, _) in enumerate(lens)]
    mel_tgt = [S.make_mel_pair(1, t, [0], 5000 + p)[1][0].cuda() for p, (_, t) in enumerate(lens)]
    cells = sum(s * t for s, t in lens)
    frames = sum(s + t for s, t in lens)
    runs = {'LoNDTW': (f0_src, f0_tgt, 'LoNDTW', 64), 'NaiveDTW_f0': (f0_src, f0_tgt, 'NaiveDTW', 1),
            'NaiveDTW_mel80': (mel_src, mel_tgt, 'NaiveDTW', 80), 'ZMNaiveDTW': (f0_src, f0_tgt, 'ZMNaiveDTW', 1),
            'NNaiveDTW': (f0_src, f0_tgt, 'NNaiveDTW', 1), 'NInterpo': (f0_src, f0_tgt, 'NInterpo', 0)}
    from oracle import dtw_baselines as O
    methods = {}
    for key, (xs, ys, method, K) in runs.items():
        run = lambda: core.align_batch(xs, ys, method)  # noqa: E731
        for _ in range(2):
            run()
        torch.cuda.synchronize()
        device_ms = [events_ms(run, a.reps) for _ in range(3)]
        st = np.median(np.array([core.align_batch(xs, ys, method, stage_ms=True).stage_ms for _ in range(a.reps)]), axis=0)
        r = core.align_batch(xs, ys, method).split()
        t0 = time.perf_counter()
        for p in range(a.oracle_pairs):
            xp, yp = xs[p].cpu(), ys[p].cpu()
            O.align(method, xp[:, None] if method == 'NaiveDTW' and xp.dim() == 1 else xp,
                    yp[:, None] if method == 'NaiveDTW' and yp.dim() == 1 else yp)
        oracle_s = (time.perf_counter() - t0) / a.oracle_pairs
        m = {'device_ms_per_batch': [round(x, 3) for x in device_ms],
             'stage_ms': {'features': round(st[0], 4), 'cost': round(st[1], 4), 'dtw': round(st[2], 4), 'backtrack': round(st[3], 4)},
             'cpu_baseline': {'impl': 'oracle (oracle/dtw_baselines.py: torch.cdist on the CPU, vectorised numpy DTW)',
                              'host_cores': os.cpu_count(), 's_per_pair': round(oracle_s, 3),
                              's_per_batch_serial': round(oracle_s * a.pairs, 1)}}
        assert [len(x) for x in r] == [t for _, t in lens]
        if method != 'NInterpo':
            flop, nbytes = cost_work(method, K, cells, frames, 4)
            cost_s = st[1] / 1e3
            m.update({'cost_flop': flop, 'cost_bytes': nbytes, 'cost_flop_per_s': flop / cost_s,
                      'cost_flop_share_of_fp32_peak': flop / cost_s / FP32_FLOP_PER_S,
                      'cost_bytes_per_s': nbytes / cost_s, 'cost_bytes_share_of_hbm': nbytes / cost_s / HBM_BYTES_PER_S,
                      'cost_bound': 'compute' if flop / FP32_FLOP_PER_S > nbytes / HBM_BYTES_PER_S else 'memory'})
        methods[key] = m
    res = {'metric': 'dtw_baselines_batch', 'card': name, 'power_limit_and_max_sm_clock': power, 'pairs': a.pairs,
           'frames_mean': a.frames, 'cells': cells, 'dtype': 'float32', 'methods': methods}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()

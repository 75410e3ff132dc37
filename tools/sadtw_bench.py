"""Shape-aware DTW pitch alignment on the GPU (csrc/sadtw.cu): prints one JSON line.

    python tools/sadtw_bench.py [--pairs 256] [--frames 1378] [--reps 10] [--oracle-pairs 4] [--out result.json]

EHSADTW on `pairs` pairs of about 8 s (frames +- 15 %, float64 f0 as a pitch extractor returns it):
  * device_ms_per_batch: align_batch on f0 already on the device, CUDA events around the call (metadata upload included);
  * e2e_ms_per_batch: align_pitch from host numpy f0 to host int64 alignments, host clock;
  * per-kernel times from CUDA events (stage_ms of svb_sadtw_align) with the bound each kernel hits;
  * one 5000 x 5000 pair's latency;
  * the CPU baseline is the oracle (oracle/sadtw.py, vectorised numpy) on this host's cores, per pair and scaled to the batch.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=256)
    ap.add_argument('--frames', type=int, default=1378)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--oracle-pairs', type=int, default=4)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('sadtw_bench needs a CUDA device')
    name, power = card()
    rs = np.random.RandomState(2026)
    lens = [(int(a.frames * rs.uniform(0.85, 1.15)), int(a.frames * rs.uniform(0.85, 1.15))) for _ in range(a.pairs)]
    host = [S.make_f0_pair(1000 + p, s, t) for p, (s, t) in enumerate(lens)]
    dev_src = [torch.from_numpy(x).cuda() for x, _ in host]
    dev_tgt = [torch.from_numpy(y).cuda() for _, y in host]
    cells = sum(s * t for s, t in lens)
    frames = sum(s + t for s, t in lens)

    run = lambda: core.align_batch(dev_src, dev_tgt, 'EHSADTW')
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    device_ms = [events_ms(run, a.reps) for _ in range(3)]

    stages = []
    for _ in range(a.reps):
        stages.append(core.align_batch(dev_src, dev_tgt, 'EHSADTW', stage_ms=True).stage_ms)
    st = np.median(np.array(stages), axis=0)

    srcs, tgts = [x for x, _ in host], [y for _, y in host]
    align_pitch_out = core.align_pitch(srcs, tgts)
    e2e = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        align_pitch_out = core.align_pitch(srcs, tgts)
        e2e.append((time.perf_counter() - t0) * 1e3)
    assert [len(x) for x in align_pitch_out] == [t for _, t in lens]

    big = S.make_f0_pair(5000, 5000, 5000)
    bs, bt = [torch.from_numpy(big[0]).cuda()], [torch.from_numpy(big[1]).cuda()]
    rb = lambda: core.align_batch(bs, bt, 'EHSADTW')
    rb()
    big_ms = events_ms(rb, 3)
    big_st = core.align_batch(bs, bt, 'EHSADTW', stage_ms=True).stage_ms

    from oracle import sadtw as O
    t0 = time.perf_counter()
    for p in range(a.oracle_pairs):
        al, _ = O.shape_aware_align(srcs[p], tgts[p], 'EHSADTW')
        assert np.array_equal(al, align_pitch_out[p]), f'pair {p}: GPU alignment differs from the oracle'
    oracle_s = (time.perf_counter() - t0) / a.oracle_pairs

    # bounds: histogram and cost are arithmetic (IEEE divisions), the DTW wavefront is barrier / latency bound (S + T - 1 steps
    # per CTA), the backtrack is a chain of dependent byte loads (about S + T per pair)
    hist_s, cost_s, dtw_s, bt_s = (x / 1e3 for x in st)
    neighbours = 128                                       # slope windows cover about 128 frames per frame at scale ~1
    res = {
        'metric': 'sadtw_ehsadtw_batch', 'card': name, 'power_limit_and_max_sm_clock': power,
        'pairs': a.pairs, 'frames_mean': a.frames, 'cells': cells, 'f0_dtype': 'float64',
        'device_ms_per_batch': [round(x, 3) for x in device_ms],
        'e2e_ms_per_batch_host_numpy_to_host_alignments': [round(x, 2) for x in e2e],
        'stage_ms': {'histogram': round(st[0], 4), 'cost': round(st[1], 4), 'dtw': round(st[2], 4), 'backtrack': round(st[3], 4)},
        'histogram_slopes_per_s': frames * neighbours / hist_s,
        'cost_cells_per_s': cells / cost_s, 'cost_bin_terms_per_s': cells * 48 / cost_s,
        'cost_write_bytes_share_of_hbm': cells * 4 / cost_s / HBM_BYTES_PER_S,
        'dtw_cells_per_s': cells / dtw_s,
        'dtw_bytes_share_of_hbm': cells * 5 / dtw_s / HBM_BYTES_PER_S,
        'dtw_us_per_wavefront_step': dtw_s / max(s + t - 1 for s, t in lens) * 1e6,
        'backtrack_us_per_step': bt_s / max(s + t for s, t in lens) * 1e6,
        'pair_5000x5000_ms': round(big_ms, 3),
        'pair_5000x5000_stage_ms': [round(x, 3) for x in big_st],
        'cpu_baseline': {'impl': 'oracle (oracle/sadtw.py, vectorised numpy; the reference is not part of this repository)',
                         'host_cores': os.cpu_count(), 's_per_pair': round(oracle_s, 3),
                         's_per_batch_serial': round(oracle_s * a.pairs, 1)},
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()

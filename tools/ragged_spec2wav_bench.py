"""Vocode a test set of clips of different lengths three ways, alternating in one run:

  per-clip   ``HifiGAN.spec2wav`` once per clip (what the batch-1 test loops do)
  padded     one ``spec2wav_batch`` over [B, T_max, n_mel], every clip padded to the longest
  ragged     one ``spec2wav_batch`` over the list of [T_b, n_mel] mels (svb_gen_spec2wav_ragged_host)

32 clips, lengths uniform in [2, 15] s from a fixed seed, NSF f0 given, on the config-2 architecture (hop 256) and the hop-128
singing architecture, at bf16x3.  Each arm runs on its own generator handle; the clip order is shuffled every round, so the
ragged arm pays for re-zeroing the rows a previous, longer clip left behind.  Per arm: audio seconds per second, ms per batch
(host clock around the whole call: staging, H2D, forward, D2H, synchronisation), kernel launches and algorithmic FLOPs of the
generator forwards of one batch.  Also the useful-work ratio sum(T_b) / (B * T_max) and the GPU's name, power limit and maximum
SM clock, read in the same run.  Prints one JSON line per architecture.

    python tools/ragged_spec2wav_bench.py [--clips 32] [--rounds 5] [--precision bf16x3]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from neuralsvb_b200 import _native  # noqa: E402
from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator  # noqa: E402
from neuralsvb_b200.utils import synthetic as S  # noqa: E402
from neuralsvb_b200.vocoders.hifigan import HifiGAN  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(', ')
        return {'gpu': out[0], 'power_limit_w': float(out[1]), 'sm_max_mhz': float(out[2])}
    except Exception as e:                                              # noqa: BLE001
        return {'gpu': torch.cuda.get_device_name(0), 'power_limit_w': None, 'sm_max_mhz': None, 'query_error': str(e)}


def vocoder(h, precision, seed):
    m = HifiGanGenerator(h, precision=precision)
    m.load_state_dict(S.make_generator_state_dict(h, seed), strict=True)
    with contextlib.redirect_stdout(io.StringIO()):
        m.remove_weight_norm()
    return HifiGAN.from_model(m.eval().cuda(), h)


def counters(voc):
    lib = _native.lib()
    g = voc.model.native_handle(voc.device)
    return int(lib.svb_gen_last_launches(g)), float(lib.svb_gen_last_flops(g))


def run_arm(arm, voc, mels, f0s):
    """one batch of the arm -> (seconds, launches, flops, total samples)"""
    torch.cuda.synchronize()
    launches, flops, n = 0, 0.0, 0
    t0 = time.perf_counter()
    if arm == 'per_clip':
        for m, f in zip(mels, f0s):
            n += len(voc.spec2wav(m, f0=f, seed=1))
            la, fl = counters(voc)
            launches, flops = launches + la, flops + fl
    elif arm == 'padded':
        T = max(len(m) for m in mels)
        mp = np.stack([np.pad(m, ((0, T - len(m)), (0, 0)), mode='edge') for m in mels])
        fp = np.stack([np.pad(f, (0, T - len(f)), mode='edge') for f in f0s])
        out = voc.spec2wav_batch(mp, fp, seed=1)
        n = out.size
        launches, flops = counters(voc)
    else:
        out = voc.spec2wav_batch(mels, f0s, seed=1)
        n = sum(len(o) for o in out)
        launches, flops = counters(voc)
    return time.perf_counter() - t0, launches, flops, n


def bench(name, h, args, info):
    sr, hop = h['audio_sample_rate'], h['hop_size']
    rs = np.random.RandomState(args.seed)
    secs = rs.uniform(2.0, 15.0, args.clips)
    lengths = [max(1, int(round(s * sr / hop))) for s in secs]
    T_max = max(lengths)
    mel, f0 = S.make_mel_f0(args.clips, T_max, args.seed)
    mels = [np.ascontiguousarray(mel[b, :, :L].T.numpy()) for b, L in enumerate(lengths)]
    f0s = [np.ascontiguousarray(f0[b, :L].numpy()) for b, L in enumerate(lengths)]
    audio_s = sum(lengths) * hop / sr
    arms = ['per_clip', 'padded', 'ragged']
    vocs = {a: vocoder(h, args.precision, args.seed) for a in arms}
    times = {a: [] for a in arms}
    stats = {}
    order = np.arange(args.clips)
    for r in range(args.rounds + 1):                                    # round 0 warms every arm up
        for a in arms:
            t, la, fl, n = run_arm(a, vocs[a], [mels[i] for i in order], [f0s[i] for i in order])
            if r > 0:
                times[a].append(t)
            stats[a] = (la, fl, n)
        order = rs.permutation(args.clips)
    res = {'arch': name, 'precision': args.precision, 'clips': args.clips, 'hop': hop, 'T_max_frames': T_max,
           'audio_s': round(audio_s, 2), 'useful_work_ratio': round(sum(lengths) / (args.clips * T_max), 4), **info}
    for a in arms:
        ms = 1e3 * float(np.median(times[a]))
        res[a] = {'ms_per_batch': round(ms, 2), 'ms_min': round(1e3 * min(times[a]), 2), 'audio_s_per_s': round(audio_s / (ms / 1e3), 1),
                  'launches': stats[a][0], 'gflops': round(stats[a][1] / 1e9, 1)}
    res['ragged_over_padded_time'] = round(res['ragged']['ms_per_batch'] / res['padded']['ms_per_batch'], 4)
    res['ragged_over_per_clip_time'] = round(res['ragged']['ms_per_batch'] / res['per_clip']['ms_per_batch'], 4)
    del vocs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clips', type=int, default=32)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--precision', default='bf16x3')
    ap.add_argument('--seed', type=int, default=1234)
    ap.add_argument('--arch', choices=['hop256', 'hop128', 'both'], default='both')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ragged_spec2wav_bench needs a CUDA device')
    torch.cuda.set_device(0)
    info = gpu_info()
    archs = [('hop256', 256), ('hop128', 128)]
    for name, hop in archs:
        if args.arch in (name, 'both'):
            print(json.dumps(bench(name, S.hifigan_config(True, hop=hop), args, info)), flush=True)


if __name__ == '__main__':
    main()

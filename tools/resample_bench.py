"""Measure the GPU resampler (csrc/resample.cu) and the paired binarizer on off-rate input.

    python tools/resample_bench.py [--clips 256] [--seconds 8] [--repeats 10] [--oracle-clips 4] [--out result.json]

* per source rate (44.1 kHz and 48 kHz -> 22.05 kHz), --clips clips of --seconds s +- 15 %: per-kernel CUDA-event medians over
  --repeats after a warm-up (time register, filter), seconds of audio per second, and the work counted from the shapes: taps (each
  4 FP64 operations -- two multiplies, two adds, none fused -- and two float32 <-> float64 conversions), {win, delta} table bytes
  read through L1 / L2 (16 per tap), and HBM bytes (samples in and out, the time register written and read, the tables);
  shares of the 34 TFLOP/s FP64 and 3.35 TB/s data-sheet figures;
* the oracle (numpy, one process per core of this host) as the CPU baseline, in seconds of audio per second;
* the paired binarizer end to end on the same write_svb_raw set written at 44.1 kHz stereo and at 22.05 kHz mono;
* the card's name, power limit and maximum SM clock, read in the same run.
Prints one JSON line (and writes it to --out when given)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
TARGET = 22050


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [x.strip() for x in q.split(',')]
        return {'gpu': name, 'power_limit': pl, 'max_sm_clock': clk}
    except Exception as e:                       # the measurement still stands; say what is missing
        return {'gpu': None, 'error': str(e)}


def taps(n_in, sr):
    """Taps of one clip (left + right wings over every output), from the oracle's index arithmetic."""
    from oracle import resample as R
    ratio = float(TARGET) / sr
    n_res, _ = R.lengths(n_in, sr, TARGET)
    scale, nwin = min(1.0, ratio), 32769
    step = int(scale * 512)
    tr = R.time_register(n_res, 1.0 / ratio)
    n = tr.astype(np.int64)
    frac = scale * (tr - n)
    off = (frac * 512).astype(np.int64)
    left = np.minimum(n + 1, (nwin - off) // step)
    off = ((scale - frac) * 512).astype(np.int64)
    right = np.maximum(np.minimum(n_in - n - 1, (nwin - off) // step), 0)
    return int(left.sum() + right.sum())


def _oracle(args):
    from oracle import resample as R
    x, sr = args
    R.resample(x, sr, TARGET)
    return len(x) / sr


def run_device(wavs, sr, repeats):
    import torch

    from neuralsvb_b200 import _native
    from neuralsvb_b200.utils import audio
    lib = _native.lib()
    win, num_table = audio.kaiser_best_window()
    srs = np.full(len(wavs), sr, np.int32)
    lens = np.array([len(w) for w in wavs], np.int64)
    _, out_lens = audio.resample_lengths(lens, srs, TARGET)
    ws_bytes = lib.svb_resample_plan(TARGET, srs.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p), len(wavs),
                                     len(win), num_table, None, None)
    x = torch.from_numpy(np.concatenate(wavs)).cuda()
    y = torch.empty(int(out_lens.sum()), device='cuda')
    ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device='cuda')
    ms = np.zeros(2, np.float32)

    def call():
        _native.check(lib.svb_resample_batch(TARGET, srs.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                                             len(wavs), win.ctypes.data_as(ctypes.c_void_p), len(win), num_table,
                                             ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(y.data_ptr()),
                                             ctypes.c_void_p(ws.data_ptr()), int(ws_bytes), ms.ctypes.data_as(ctypes.c_void_p),
                                             _native.current_stream_ptr()), 'resample')
        return ms.astype(np.float64).copy()

    call()
    med = np.median(np.array([call() for _ in range(repeats)]), axis=0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(repeats):
        audio.resample_batch(wavs, srs, TARGET)
    host_ms = (time.perf_counter() - t0) / repeats * 1e3
    n_in, n_out = int(lens.sum()), int(out_lens.sum())
    n_taps = sum(taps(len(w), sr) for w in wavs)
    seconds = n_in / sr
    fp64 = 4.0 * n_taps
    hbm = 4.0 * n_in + 4.0 * n_out + 2 * 8.0 * out_lens.max() + 8.0 * n_out + 16.0 * 32769
    filt_s = med[1] / 1e3
    return {
        'sr': sr, 'clips': len(wavs), 'audio_s': seconds, 'outputs': n_out, 'taps': n_taps, 'taps_per_output': n_taps / n_out,
        'time_register_ms': float(med[0]), 'filter_ms': float(med[1]),
        'audio_s_per_s_kernels': seconds / (med.sum() / 1e3), 'host_call_ms': host_ms, 'audio_s_per_s_host_call': seconds / (host_ms / 1e3),
        'fp64_ops': fp64, 'fp64_tops': fp64 / filt_s / 1e12, 'fp64_share_of_34tflops': fp64 / filt_s / 34e12,
        'table_bytes_l1_l2': 16.0 * n_taps, 'table_tb_per_s': 16.0 * n_taps / filt_s / 1e12,
        'hbm_bytes': hbm, 'hbm_share_of_3_35tbs': hbm / filt_s / 3.35e12,
        'f2f_conversions': 2.0 * n_taps,
    }


def binarize(raw, binary):
    from neuralsvb_b200.data_gen.singing.binarize_para import PopBuTFyENSpkEMBinarizer
    from neuralsvb_b200.utils.hparams import set_hparams
    set_hparams(os.path.join(ROOT, 'egs', 'svb_binarize_synthetic.yaml'), '',
                f'processed_data_dir={raw},binary_data_dir={binary},spk_emb_data_dir={raw}/spk_emb,max_mel_tech_gap=2000',
                print_hparams=False)
    PopBuTFyENSpkEMBinarizer().process()        # warm-up: module loads, allocator
    t0 = time.perf_counter()
    PopBuTFyENSpkEMBinarizer().process()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clips', type=int, default=256)
    ap.add_argument('--seconds', type=float, default=8.0)
    ap.add_argument('--repeats', type=int, default=10)
    ap.add_argument('--oracle-clips', type=int, default=4)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    a = ap.parse_args()
    import torch

    from neuralsvb_b200.utils import audio, synthetic as S
    if not torch.cuda.is_available():
        raise SystemExit('resample_bench measures the GPU resampler: no CUDA device')
    res = {'target_sr': TARGET, **card()}
    for sr in (44100, 48000):
        rs = np.random.RandomState(sr)
        base = [S.make_clip(int(a.seconds * 1.15 * sr) + 1, sr, seed=i) for i in range(16)]
        wavs = [base[i % 16][:int(a.seconds * rs.uniform(0.85, 1.15) * sr)] for i in range(a.clips)]
        res[f'gpu_{sr}'] = run_device(wavs, sr, a.repeats)
        jobs = [(wavs[i], sr) for i in range(a.oracle_clips * (os.cpu_count() or 1))]
        t0 = time.perf_counter()
        with ProcessPoolExecutor(os.cpu_count()) as ex:
            secs = sum(ex.map(_oracle, jobs))
        res[f'cpu_oracle_{sr}'] = {'processes': os.cpu_count(), 'audio_s': secs,
                                   'audio_s_per_s': secs / (time.perf_counter() - t0)}
    with tempfile.TemporaryDirectory() as d:
        for name, kw in (('binarizer_22050_mono', {}), ('binarizer_44100_stereo', {'file_sr': 44100, 'channels': 2})):
            raw, binary = os.path.join(d, name, 'raw'), os.path.join(d, name, 'bin')
            S.write_svb_raw(raw, binary, seconds=(6.0, 10.0), **kw)
            secs = 0.0
            for root, _, files in os.walk(os.path.join(raw, 'data')):
                for f in files:
                    if '#singing#' in f:
                        secs += audio.wav_seconds(os.path.join(root, f))
            wall = binarize(raw, binary)
            res[name] = {'audio_s': secs, 'wall_s': wall, 'audio_s_per_s': secs / wall}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()

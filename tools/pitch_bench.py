"""Measure the GPU pitch tracker (csrc/pitch_ac.cu) and the paired binarizer.

    python tools/pitch_bench.py [--clips 256] [--seconds 8] [--repeats 20] [--oracle-clips 8] [--out result.json]

* the tracker on --clips clips of --seconds s +- 15 % (sung takes of utils/synthetic): per-stage times from CUDA events (median over
  --repeats after a warm-up), analysis frames per second, and the candidate kernel's FLOP rate (2 L (tau_max + 2) FMA-FLOP per frame,
  the direct autocorrelation it computes) against the 67 TFLOP/s FP32 data-sheet figure;
* the float64 oracle's seconds per clip on this host's cores (the CPU baseline);
* the binarizer end to end on a write_svb_raw set, in seconds of audio per second;
* the card's name and power limit, read in the same run.
Prints one JSON line (and writes it to --out when given)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [x.strip() for x in q.split(',')]
        return {'gpu': name, 'power_limit': pl, 'max_sm_clock': clk}
    except Exception as e:                       # the measurement still stands; say what is missing
        return {'gpu': None, 'error': str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clips', type=int, default=256)
    ap.add_argument('--seconds', type=float, default=8.0)
    ap.add_argument('--repeats', type=int, default=20)
    ap.add_argument('--oracle-clips', type=int, default=8)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    a = ap.parse_args()
    import torch

    from neuralsvb_b200.data_gen.tts import data_gen_utils as DG
    from neuralsvb_b200.utils import synthetic as S
    from oracle import pitch_ac as P
    if not torch.cuda.is_available():
        raise SystemExit('pitch_bench measures the GPU tracker: no CUDA device')
    sr, hop = 22050, 128
    fps = sr / hop
    hp = {'audio_sample_rate': sr, 'hop_size': hop}
    rs = np.random.RandomState(0)
    base = []
    for i in range(16):                          # 16 distinct takes, reused round-robin at varied lengths
        n = int(a.seconds * 1.15 * fps) + 1
        fa, _ = S.make_f0_pair(i, n, n, fps)
        base.append(S.make_sung_take(fa, i, sr, hop)[0])
    ws = [base[i % 16][:int(a.seconds * rs.uniform(0.85, 1.15) * sr)] for i in range(a.clips)]
    lens = np.array([len(w) for w in ws])
    n_mel = lens // hop + 1
    cat = torch.from_numpy(np.concatenate(ws)).cuda()
    DG.pitch_ac_device(cat, lens, n_mel, hp, stage_ms=True)
    ms = np.array([DG.pitch_ac_device(cat, lens, n_mel, hp, stage_ms=True).stage_ms for _ in range(a.repeats)])
    med = np.median(ms, axis=0).astype(np.float64)
    tr = DG.pitch_ac_device(cat, lens, n_mel, hp)
    frames = int(tr.frames.sum())
    L, nlag = 827, 278
    flop = 2.0 * L * nlag * frames
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.repeats):
        DG.pitch_ac_device(cat, lens, n_mel, hp)
    torch.cuda.synchronize()
    call_ms = (time.perf_counter() - t0) / a.repeats * 1e3
    # CPU baseline: the float64 oracle
    t0 = time.perf_counter()
    for w in ws[:a.oracle_clips]:
        P.track(w, sr, hop)
    oracle_s = (time.perf_counter() - t0) / a.oracle_clips
    # binarizer end to end
    with tempfile.TemporaryDirectory() as d:
        raw, binary = os.path.join(d, 'raw'), os.path.join(d, 'bin')
        S.write_svb_raw(raw, binary, seconds=(6.0, 10.0))
        audio = 0.0
        from scipy.io import wavfile
        for root, _, files in os.walk(os.path.join(raw, 'data')):
            for f in files:
                if '#singing#' in f:
                    r, x = wavfile.read(os.path.join(root, f))
                    audio += len(x) / r
        from neuralsvb_b200.data_gen.singing.binarize_para import PopBuTFyENSpkEMBinarizer
        from neuralsvb_b200.utils.hparams import set_hparams
        set_hparams(os.path.join(ROOT, 'egs', 'svb_binarize_synthetic.yaml'), '',
                    f'processed_data_dir={raw},binary_data_dir={binary},spk_emb_data_dir={raw}/spk_emb,max_mel_tech_gap=2000',
                    print_hparams=False)
        PopBuTFyENSpkEMBinarizer().process()        # warm-up: module loads, allocator
        t0 = time.perf_counter()
        PopBuTFyENSpkEMBinarizer().process()
        bin_s = time.perf_counter() - t0
    res = {
        'clips': a.clips, 'seconds_mean': float(lens.mean() / sr), 'frames': frames,
        'stage_ms': {'clip_stats': float(med[0]), 'candidates': float(med[1]), 'path': float(med[2])},
        'call_ms_device_tensors': call_ms,
        'frames_per_s': frames / (med.sum() / 1e3),
        'candidate_tflops': flop / (med[1] / 1e3) / 1e12,
        'candidate_share_of_fp32_67tflops': flop / (med[1] / 1e3) / 67e12,
        'oracle_s_per_clip': float(oracle_s), 'oracle_threads': os.cpu_count(),
        'binarizer_audio_s': audio, 'binarizer_wall_s': bin_s, 'binarizer_audio_s_per_s': audio / bin_s,
        **card(),
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()

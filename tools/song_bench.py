"""Beautify whole songs (SVBBeautifier.beautify_songs) and time the cluster DTW that aligns them.

Workload: 4 synthetic songs of 3-4 min (make_f0_pair / make_sung_take at 22050 Hz, hop 128): the amateur take is the professional
one time-warped by 0.85-1.15 and detuned (make_f0_pair's amateur contour); song 0 is a pair of 44.1 kHz WAV files, so the
resampler runs, the others are float32 arrays.  Weights are random draws of the reference architectures, as in
tools/beautify_bench.py: the timings do not depend on what the weights have learnt.

Reports, with the card's name and power limit read in the same run:
  * CUDA-event times per stage of one call (h2d, resample, front_end, pitch, alignment = align_songs' histogram + forward +
    backward + backtrack with their own event times, plan_conditioning = host planning and conditioning, acoustic_model, stitch, vocoder, d2h);
  * DTW microseconds per anti-diagonal step: the cluster kernel on each song aligned alone, and on a 5000 x 5000 pair the cluster
    kernel forced by SVB_DTW_CTA_CELLS (2 and 8 CTAs) against the one-CTA kernel, alternated in this process;
  * peak device memory of one call (torch.cuda.max_memory_allocated) and the alignment workspace of each song;
  * input audio seconds per second of the whole call (host clock around beautify_songs, which returns host arrays).

    python tools/song_bench.py [--songs 4] [--repeats 2] [--out result.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from beautify_bench import card, make_experiment  # noqa: E402
from neuralsvb_b200.inference import beautify as BF  # noqa: E402
from neuralsvb_b200.modules.voice_conversion.dtw import core  # noqa: E402
from neuralsvb_b200.utils import synthetic as S  # noqa: E402

SR, HOP, FILE_SR = 22050, 128, 44100


def make_songs(root, n, seed=4321):
    from scipy.io import wavfile
    rs = np.random.RandomState(seed)
    fps = SR / HOP
    ama, prof, emb, seconds = [], [], [], 0.0
    for i in range(n):
        Tf = int(rs.uniform(180.0, 240.0) * fps)
        Sf = int(Tf * rs.uniform(0.85, 1.15))
        fa, fp = S.make_f0_pair(int(rs.randint(0, 2 ** 31 - 1)), Sf, Tf, fps)
        off = i == 0
        sr, hop = (FILE_SR, 2 * HOP) if off else (SR, HOP)
        takes = []
        for k, f in enumerate((fa, fp)):
            w, _ = S.make_sung_take(f, int(rs.randint(0, 2 ** 31 - 1)), sr, hop)
            if off:
                fn = os.path.join(root, f'song{i}_{k}.wav')
                wavfile.write(fn, sr, np.round(w * 32767).astype(np.int16))
                takes.append(fn)
            else:
                takes.append(w)
            seconds += len(w) / sr
        ama.append(takes[0])
        prof.append(takes[1])
        emb.append(rs.normal(0, 0.5, 256).astype(np.float32))
    return ama, prof, emb, seconds


def dtw_us_per_step(srcs, tgts, cells=None):
    """(histogram, cost, DTW, backtrack) ms of one align_long call, and DTW us per anti-diagonal step of its longest pair."""
    if cells is None:
        os.environ.pop('SVB_DTW_CTA_CELLS', None)
    else:
        os.environ['SVB_DTW_CTA_CELLS'] = str(cells)
    try:
        r = core.align_long(srcs, tgts, stage_ms=True) if cells is not None else core.align_batch(srcs, tgts, stage_ms=True)
    finally:
        os.environ.pop('SVB_DTW_CTA_CELLS', None)
    steps = max(len(a) + len(b) - 1 for a, b in zip(srcs, tgts))
    return r.stage_ms, 1e3 * r.stage_ms[2] / steps


def time_modes(b, run, repeats):
    """The acoustic_model stage (device ms) and the whole call (s) of ``run(batch_invariant)``, default and length-aware
    alternated, after one warm-up call of each."""
    out = {'default': {'acoustic_model_ms': [], 'call_s': []}, 'batch_invariant': {'acoustic_model_ms': [], 'call_s': []}}
    b.timing = True
    for mode in (False, True):
        run(mode)
    for _ in range(repeats):
        for mode, key in ((False, 'default'), (True, 'batch_invariant')):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(mode)
            out[key]['call_s'].append(round(time.perf_counter() - t0, 3))
            out[key]['acoustic_model_ms'].append(round(b.stage_ms['acoustic_model'], 2))
    b.timing = False
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--songs', type=int, default=4)
    ap.add_argument('--repeats', type=int, default=2)
    ap.add_argument('--out', type=str, default='')
    ap.add_argument('--modes', action='store_true',
                    help='also time the acoustic model in both modes (batch_invariant False / True), alternated in this process')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('song_bench measures on a CUDA device; none is visible')
    res = {'card': card()}
    with tempfile.TemporaryDirectory() as root:
        ama, prof, emb, audio_s = make_songs(root, args.songs)
        b = BF.SVBBeautifier(make_experiment(root))
        N = args.songs
        eps = torch.randn(N, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(0))
        call = (ama, prof, emb)
        b.beautify_songs(*call, seed=1, eps=eps)                    # warm-up
        walls = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            wavs = b.beautify_songs(*call, seed=1, eps=eps)
            walls.append(time.perf_counter() - t0)
        peak = torch.cuda.max_memory_allocated()
        b.timing = True
        b.beautify_songs(*call, seed=1, eps=eps)
        stages, align_ms, plans = b.stage_ms, b.align_ms, b.song_plans
        b.timing = False
        if args.modes:
            res['modes'] = time_modes(b, lambda m: b.beautify_songs(*call, seed=1, eps=eps, batch_invariant=m), args.repeats)
            for k, v in res['modes'].items():
                print(f"  acoustic model, {k:15s}: {v['acoustic_model_ms']} ms (calls {v['call_s']} s)")
        # the songs' f0 as the call aligns it: each song alone on the cluster kernel
        f0_dev, f0s = b._pitch(*_front(b, call))
        frames = [len(f) for f in f0s]
        t = torch.split(f0_dev.double(), frames)
        per_song = []
        for i in range(N):
            ms, us = dtw_us_per_step([t[i]], [t[N + i]], cells=8192)
            per_song.append({'frames': [frames[i], frames[N + i]], 'ctas': -(-min(frames[i], frames[N + i]) // 8192),
                             'workspace_GB': round(core.long_workspace_bytes([frames[i]], [frames[N + i]]) / 1e9, 2),
                             'stage_ms': [round(x, 2) for x in ms], 'dtw_us_per_step': round(us, 3), 'segments': len(plans[i])})
        # 5000 x 5000: one-CTA kernel against the cluster kernel forced onto 2 and 8 CTAs, alternated
        a, p = S.make_f0_pair(5, 5000, 5000)
        a, p = torch.from_numpy(a).cuda(), torch.from_numpy(p).cuda()
        short = {'one_cta': [], 'cluster_2': [], 'cluster_8': []}
        for _ in range(2):                                          # warm-up
            dtw_us_per_step([a], [p]), dtw_us_per_step([a], [p], 2500), dtw_us_per_step([a], [p], 625)
        for _ in range(5):
            short['one_cta'].append(dtw_us_per_step([a], [p])[1])
            short['cluster_2'].append(dtw_us_per_step([a], [p], 2500)[1])
            short['cluster_8'].append(dtw_us_per_step([a], [p], 625)[1])
    wall = float(np.median(walls))
    res.update({'songs': N, 'input_audio_s': round(audio_s, 1), 'output_audio_s': round(sum(len(w) for w in wavs) / SR, 1),
                'call_s': [round(x, 3) for x in walls], 'audio_s_per_s': round(audio_s / wall, 1),
                'peak_memory_GB': round(peak / 1e9, 2), 'stage_ms': {k: round(v, 2) for k, v in stages.items()},
                'align_groups_ms': [[round(x, 2) for x in g] for g in align_ms], 'per_song': per_song,
                'dtw_5000x5000_us_per_step': {k: [round(x, 3) for x in v] for k, v in short.items()}})
    print(f"card: {res['card']}")
    print(f"{N} songs, {audio_s:.1f} s of input audio (both takes); call {wall:.3f} s (median of {args.repeats}), "
          f"{audio_s / wall:.1f} audio-s/s, peak device memory {peak / 1e9:.2f} GB")
    print('  stage (device time, ms): ' + ', '.join(f'{k} {v:.1f}' for k, v in res['stage_ms'].items()))
    print('  alignment (histogram, forward, backward, backtrack ms): ' + str(res['align_groups_ms']))
    for i, s in enumerate(per_song):
        print(f"  song {i}: {s['frames']} frames, {s['ctas']} CTAs, {s['workspace_GB']} GB workspace, {s['segments']} segments, "
              f"DTW {s['dtw_us_per_step']:.3f} us/step (stages {s['stage_ms']} ms)")
    for k, v in short.items():
        print(f"  5000 x 5000 {k}: median {np.median(v):.3f} us/step ({v})")
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


def _front(b, call):
    """(padded waveforms, frame counts) of the call's takes, through the beautifier's own front end."""
    dec, rates, lens, frames, _ = b._takes(*call, songs=True)
    _, wav = b._front_end(dec, rates, lens, BF._Stages(False))
    return wav, frames


if __name__ == '__main__':
    main()

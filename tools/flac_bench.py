"""FLAC input on the GPU: the decoder alone and the beautifier on FLAC takes against the same takes as WAV.

Workload 1: the 64-pair workload of tools/beautify_bench.py (8 s takes, a quarter of them 44.1 kHz files), every take stored as a
file.  Workload 2: the 4 songs of 3-4 min of tools/song_bench.py, the same way.  Each take is written twice with the same int16 PCM:
as WAV, and as FLAC by the project's test encoder (oracle/flac.py: FIXED order-2 subframes, Rice partitions of order 4, 4096-sample
blocks).  No FLAC encoder of FFmpeg's levels is available where the benchmark runs, so the streams are not FFmpeg's level 5; they
hold the same subframe and residual coding a level-5 file mostly does.

Reports, with the card's name and power limit read in the same run:
  * the decode launches' CUDA-event time for all takes of a workload in one call, decoded samples per second, the bytes copied to
    the device (compressed FLAC against the float32 samples of the WAV route);
  * the whole beautify_batch / beautify_songs call on the FLAC files against the WAV files, alternated in one process, and whether
    the outputs are equal.

    python tools/flac_bench.py [--pairs 64] [--songs 4] [--repeats 3] [--out result.json]"""
import argparse
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from beautify_bench import card, make_experiment, make_pairs  # noqa: E402
from song_bench import make_songs  # noqa: E402

from neuralsvb_b200.inference import beautify as BF  # noqa: E402
from neuralsvb_b200.utils import audio  # noqa: E402
from oracle import flac as F  # noqa: E402

SR = 22050


def _encode(args):
    wav_fn, pcm, sr = args
    from scipy.io import wavfile
    wavfile.write(wav_fn, sr, pcm.astype(np.int16))
    with open(wav_fn[:-4] + '.flac', 'wb') as f:
        f.write(F.encode(pcm.astype(np.int64), sr, 16, block_size=4096, subframe=dict(type='fixed', order=2, partition_order=4)))
    return wav_fn, wav_fn[:-4] + '.flac'


def as_files(root, takes, tag):
    """Every take (an array at SR or a WAV path) -> (WAV path, FLAC path) of the same int16 PCM."""
    from scipy.io import wavfile
    jobs = []
    for k, t in enumerate(takes):
        if isinstance(t, str):
            sr, pcm = wavfile.read(t)
        else:
            sr, pcm = SR, np.round(np.asarray(t) * 32767).astype(np.int16)
        jobs.append((os.path.join(root, f'{tag}{k}.wav'), pcm, sr))
    with ProcessPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        return list(ex.map(_encode, jobs))


def decode_stats(flacs, repeats):
    blobs = [open(f, 'rb').read() for f in flacs]
    audio.flac_decode_device(blobs)                                  # warm-up
    ms = []
    for _ in range(repeats):
        audio.flac_decode_device(blobs, stage_ms=ms)
    y, lens, _ = audio.flac_decode_device(blobs)
    samples = int(sum(audio.flac_info(b)['total_samples'] * audio.flac_info(b)['channels'] for b in blobs))
    return dict(streams=len(blobs), compressed_bytes=sum(len(b) for b in blobs), float32_bytes=int(lens.sum()) * 4,
                decode_ms=[round(m, 3) for m in ms], decoded_samples_per_s=samples / (min(ms) / 1e3))


def alternate(call, wav_args, flac_args, repeats, **kw):
    call(*wav_args, **kw), call(*flac_args, **kw)                   # warm-up, both
    tw, tf = [], []
    for _ in range(repeats):
        for args, ts in ((wav_args, tw), (flac_args, tf)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = call(*args, **kw)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
    same = all(np.array_equal(a, b) for a, b in zip(call(*wav_args, **kw), call(*flac_args, **kw)))
    return dict(wav_s=[round(t, 4) for t in tw], flac_s=[round(t, 4) for t in tf], outputs_equal=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=64)
    ap.add_argument('--songs', type=int, default=4)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', type=str, default='')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('flac_bench measures on a CUDA device; none is visible')
    res = {'card': card()}
    with tempfile.TemporaryDirectory() as root:
        b = BF.SVBBeautifier(make_experiment(root))
        for name, make, call, n in (('pairs', make_pairs, b.beautify_batch, args.pairs), ('songs', make_songs, b.beautify_songs, args.songs)):
            if n <= 0:
                continue
            t0 = time.perf_counter()
            ama, prof, emb, seconds = make(root, n)
            files = as_files(root, list(ama) + list(prof), name)
            wavs, flacs = [w for w, _ in files], [f for _, f in files]
            r = dict(audio_seconds=seconds, encode_s=round(time.perf_counter() - t0, 1))
            r.update(decode_stats(flacs, args.repeats))
            eps = torch.randn(n, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(0))
            r.update(alternate(call, (wavs[:n], wavs[n:], emb), (flacs[:n], flacs[n:], emb), args.repeats, seed=1, eps=eps))
            res[name] = r
            print(name, json.dumps(r), flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()

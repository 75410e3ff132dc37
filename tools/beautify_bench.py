"""Beautify N raw pairs in one call (neuralsvb_b200.inference.beautify) and through the existing per-pair route, in one process.

Workload: N pairs (default 64) of sung takes of 8 s +- 15 % (make_f0_pair / make_sung_take at the singing configuration, 22050 Hz,
hop 128); the professional take is 0.85-1.15 x the amateur one.  Every fourth pair is a pair of 44.1 kHz WAV files, so the
resampler runs; the other takes are in-memory float32 arrays at 22050 Hz.  Weights are random draws of the reference
architectures (write_svb_checkpoints, make_svb_state_dict): the timings do not depend on what the weights have learnt.

Reports:
  * per-stage device time of one call (CUDA events; 'conditioning' is the host code between the alignment and the model);
  * end-to-end pairs/s and audio-s/s of the one-call path: host clock around beautify_batch (which returns host arrays);
  * the H2D / D2H copies of one call, from a torch.profiler run of its own;
  * the same pairs through the existing route, timed alternately with the one-call path: PopBuTFyENBinarizer.process_batch over
    groups of binarize_batch_seconds, then per pair a batch-1 MleSVBVAE call on the dataset's collated sample and a spec2wav, as
    tasks/run.py --infer runs them;
  * the card's name and power limit.

    python tools/beautify_bench.py [--pairs 64] [--repeats 3] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import yaml

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from neuralsvb_b200.inference import beautify as BF  # noqa: E402
from neuralsvb_b200.utils import synthetic as S  # noqa: E402

SR, HOP, FILE_SR = 22050, 128, 44100
CONFIG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'egs', 'svb_vae_train_synthetic.yaml')


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except (OSError, IndexError, subprocess.SubprocessError):
        return f'{torch.cuda.get_device_name()}, power limit not read'


def make_pairs(root, n, seed=1234):
    from scipy.io import wavfile
    rs = np.random.RandomState(seed)
    fps = SR / HOP
    ama, prof, emb, seconds = [], [], [], 0.0
    for i in range(n):
        Sf = int(8.0 * rs.uniform(0.85, 1.15) * fps)
        Tf = int(Sf * rs.uniform(0.85, 1.15))
        fa, fp = S.make_f0_pair(int(rs.randint(0, 2 ** 31 - 1)), Sf, Tf, fps)
        off = i % 4 == 0
        sr, hop = (FILE_SR, 2 * HOP) if off else (SR, HOP)
        takes = []
        for k, f in enumerate((fa, fp)):
            w, _ = S.make_sung_take(f, int(rs.randint(0, 2 ** 31 - 1)), sr, hop)
            if off:
                fn = os.path.join(root, f'pair{i}_{k}.wav')
                wavfile.write(fn, sr, np.round(w * 32767).astype(np.int16))
                takes.append(fn)
            else:
                takes.append(w)
            seconds += len(w) / sr
        ama.append(takes[0])
        prof.append(takes[1])
        emb.append(rs.normal(0, 0.5, 256).astype(np.float32))
    return ama, prof, emb, seconds


def make_experiment(root):
    binary = os.path.join(root, 'binary')
    S.write_svb_checkpoints(binary, 1234)
    np.save(os.path.join(binary, 'train_f0s_mean_std.npy'), [300.0, 80.0])
    with open(CONFIG) as f:
        cfg = yaml.safe_load(f)
    cfg.update(binary_data_dir=binary, vocoder_ckpt=os.path.join(binary, 'hifigan'), pretrain_asr_ckpt=os.path.join(binary, 'asr'),
               binarize_batch_seconds=600.0)
    work = os.path.join(root, 'work')
    os.makedirs(work)
    with open(os.path.join(work, 'config.yaml'), 'w') as f:
        yaml.safe_dump(cfg, f)
    torch.save({'state_dict': {'model': S.make_svb_state_dict(1234)}, 'global_step': 1}, os.path.join(work, 'model_ckpt_steps_1.ckpt'))
    return work


def existing_route(b, ama, prof, emb, eps, seed):
    """process_batch over groups of binarize_batch_seconds, then per pair a batch-1 model call and a spec2wav."""
    from neuralsvb_b200.data_gen.singing.binarize_para import PopBuTFyENBinarizer
    from neuralsvb_b200.tasks.singing.dataset_utils import MultiSpkEmbDataset
    from neuralsvb_b200.utils import audio, move_to_cuda
    from neuralsvb_b200.utils.pitch_utils import denorm_f0
    from neuralsvb_b200.vocoders.hifigan import HifiGAN
    hp = b.hp
    binz = PopBuTFyENBinarizer.__new__(PopBuTFyENBinarizer)
    metas = [(f'pair{i}', a, 0, p) for i, (a, p) in enumerate(zip(ama, prof))]
    secs = lambda w: audio.wav_seconds(w) if isinstance(w, str) else len(w) / SR
    items, cur, sec = [], [], 0.0
    for m in metas + [None]:
        s = 0.0 if m is None else secs(m[1]) + secs(m[3])
        if cur and (m is None or sec + s > hp['binarize_batch_seconds']):
            items += binz.process_batch(HifiGAN, cur)
            cur, sec = [], 0.0
        if m is not None:
            cur.append(m)
            sec += s
    ds = MultiSpkEmbDataset.__new__(MultiSpkEmbDataset)
    ds.hparams = hp
    out = []
    for i, it in enumerate(items):
        it['multi_spk_emb'] = emb[i][None]
        ds._get_item, ds.sizes = (lambda _, it=it: it), [max(len(it['mel']), len(it['prof_mel']))]
        sample = move_to_cuda(ds.collater([ds[0]]))
        spk = sample['multi_spk_emb'][:, 0, :]
        with torch.no_grad():
            o = b.model(amateur_mel=sample['mels'], prof_mel=sample['prof_mels'], amateur_pitch=sample['pitch'],
                        prof_pitch=sample['prof_pitch'], amateur_spk_id=spk, prof_spk_id=spk, a2p_alignment=sample['a2p_f0_alignment'],
                        infer=False, concurrent_ways=['a2a', 'p2p', 'a2p'], disable_map=hp['disable_map'], eps=eps[i:i + 1].cuda())
        f0 = denorm_f0(sample['prof_f0'], sample['prof_uv'], hp)
        out.append(b.vocoder.spec2wav(o['a2p']['mel_out'][0].float().cpu().numpy(), f0=f0[0].cpu().numpy(), seed=seed))
    return out


def copies(b, args):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        b.beautify_batch(*args, seed=3)
        torch.cuda.synchronize()
    fd, fn = tempfile.mkstemp(suffix='.json')
    os.close(fd)
    prof.export_chrome_trace(fn)
    with open(fn) as f:
        trace = json.load(f)
    os.unlink(fn)
    res = {'HtoD': [], 'DtoH': []}
    for e in trace.get('traceEvents', []):
        if e.get('cat') == 'gpu_memcpy':
            for d in res:
                if d in e.get('name', ''):
                    res[d].append(int(e.get('args', {}).get('bytes', 0)))
    return {d: {'count': len(v), 'bytes': int(sum(v)), 'largest': int(max(v, default=0)),
                'small': int(sum(1 for x in v if x < 1 << 20))} for d, v in res.items()}


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
    ap.add_argument('--pairs', type=int, default=64)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', type=str, default='')
    ap.add_argument('--modes', action='store_true',
                    help='also time the acoustic model in both modes (batch_invariant False / True), alternated in this process')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('beautify_bench measures on a CUDA device; none is visible')
    with tempfile.TemporaryDirectory() as root:
        ama, prof, emb, audio_s = make_pairs(root, args.pairs)
        b = BF.SVBBeautifier(make_experiment(root))
        N = args.pairs
        eps = torch.randn(N, b.hp['latent_size'], 1, generator=torch.Generator().manual_seed(0))
        call = (ama, prof, emb)
        b.beautify_batch(*call, seed=1, eps=eps)                    # warm-up: every shape of the timed calls
        existing_route(b, ama, prof, emb, eps, 1)
        one, old = [], []
        for _ in range(args.repeats):                               # alternating, same process
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b.beautify_batch(*call, seed=1, eps=eps)
            one.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            existing_route(b, ama, prof, emb, eps, 1)
            torch.cuda.synchronize()
            old.append(time.perf_counter() - t0)
        b.timing = True
        b.beautify_batch(*call, seed=1, eps=eps)
        stages = b.stage_ms
        b.timing = False
        cp = copies(b, call)
        modes = time_modes(b, lambda m: b.beautify_batch(*call, seed=1, eps=eps, batch_invariant=m), args.repeats) if args.modes else None
    t1, t0 = float(np.median(one)), float(np.median(old))
    res = {'card': card(), 'pairs': N, 'input_audio_s': round(audio_s, 1), 'repeats': args.repeats,
           'one_call_s': [round(x, 3) for x in one], 'existing_route_s': [round(x, 3) for x in old],
           'one_call_pairs_per_s': round(N / t1, 2), 'one_call_audio_s_per_s': round(audio_s / t1, 1),
           'existing_pairs_per_s': round(N / t0, 2), 'existing_audio_s_per_s': round(audio_s / t0, 1),
           'stage_ms': {k: round(v, 2) for k, v in stages.items()}, 'copies': cp}
    if modes:
        res['modes'] = modes
        for k, v in modes.items():
            print(f"  acoustic model, {k:15s}: {v['acoustic_model_ms']} ms (calls {v['call_s']} s)")
    print(f"card: {res['card']}")
    print(f"{N} pairs, {audio_s:.1f} s of input audio (both takes), median of {args.repeats}")
    print(f"  one call      {t1:8.3f} s   {N / t1:7.2f} pairs/s   {audio_s / t1:8.1f} audio-s/s")
    print(f"  existing route{t0:8.3f} s   {N / t0:7.2f} pairs/s   {audio_s / t0:8.1f} audio-s/s")
    print('  stage (device time, ms): ' + ', '.join(f'{k} {v:.1f}' for k, v in res['stage_ms'].items()))
    for d, v in cp.items():
        print(f"  {d}: {v['count']} copies, {v['bytes'] / 1e6:.2f} MB, largest {v['largest'] / 1e6:.2f} MB, {v['small']} under 1 MB")
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()

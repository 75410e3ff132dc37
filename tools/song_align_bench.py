"""Time and size the whole-song alignment: align_long grouped as beautify_songs grouped it before align_songs (consecutive songs
up to 24 GiB of workspace), align_songs in single pass (the 24 GiB default budget) and align_songs checkpointed at a 1 GiB budget.

Workload: the 4 songs of tools/song_bench.py (3-4 min each), their f0 from the beautifier's own front end and pitch tracker, in
float64 as beautify_songs aligns them; plus one 65536 x 65536 pair (the frame limit) in single pass and at 1 GiB.  The variants
alternate in this process, each run is a host clock around the call ending in a device synchronise, and the report gives the
median and the spread, the peak device memory above what was allocated before the call (torch.cuda.max_memory_allocated), the
(histogram, cost, DTW, backtrack) or (histogram, forward, backward, backtrack) CUDA-event times of the median run, the card's name
and its power limit.  Every variant's alignments and path costs are checked equal to align_long's.

    python tools/song_align_bench.py [--repeats 5] [--out result.json]
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
from song_bench import _front, make_songs  # noqa: E402
from neuralsvb_b200.inference import beautify as BF  # noqa: E402
from neuralsvb_b200.modules.voice_conversion.dtw import core  # noqa: E402
from neuralsvb_b200.utils import synthetic as S  # noqa: E402

GiB = 1 << 30


def align_long_grouped(srcs, tgts):
    """The alignment beautify_songs ran before align_songs: align_long over consecutive songs up to 24 GiB of workspace."""
    ws = [core.long_workspace_bytes([len(a)], [len(b)]) for a, b in zip(srcs, tgts)]
    al, pc, ms = [], [], []
    for g0, g1 in BF._groups(ws, 24 * GiB):
        r = core.align_long(srcs[g0:g1], tgts[g0:g1], stage_ms=True)
        al += r.split()
        pc.append(r.path_cost)
        ms.append(r.stage_ms)
    return al, torch.cat(pc), [sum(x) for x in zip(*ms)], None


def align_songs(budget):
    def run(srcs, tgts):
        r = core.align_songs(srcs, tgts, workspace_bytes=budget, stage_ms=True)
        return r.split(), r.path_cost, list(r.stage_ms), (r.mode, r.stripe_diags, r.workspace_bytes)
    return run


def measure(variants, srcs, tgts, repeats):
    """Alternate the variants: per variant the call times, the peak memory, the stage times of the median run and its plan."""
    out = {k: {'s': [], 'peak_GB': [], 'stage_ms': []} for k in variants}
    results = {}
    for rep in range(repeats + 1):                      # the first round warms up
        for name, fn in variants.items():
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            al, pc, ms, plan = fn(srcs, tgts)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            peak = torch.cuda.max_memory_allocated() - base
            results[name] = (al, pc.cpu())
            del al, pc
            if rep == 0:
                continue
            out[name]['s'].append(round(dt, 4))
            out[name]['peak_GB'].append(round(peak / 1e9, 3))
            out[name]['stage_ms'].append([round(x, 2) for x in ms])
            out[name]['plan'] = plan
    ref_al, ref_pc = next(iter(results.values()))
    for name, (al, pc) in results.items():
        out[name]['equal_to_first'] = bool(torch.equal(pc, ref_pc) and all(np.array_equal(x, y) for x, y in zip(al, ref_al)))
        k = int(np.argsort(out[name]['s'])[len(out[name]['s']) // 2])
        out[name].update(median_s=out[name]['s'][k], median_stage_ms=out[name]['stage_ms'][k], peak_GB=max(out[name]['peak_GB']))
        del out[name]['stage_ms']
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--big_repeats', type=int, default=2)
    ap.add_argument('--out', type=str, default='')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('song_align_bench measures on a CUDA device; none is visible')
    res = {'card': card()}
    with tempfile.TemporaryDirectory() as root:
        ama, prof, emb, _ = make_songs(root, 4)
        b = BF.SVBBeautifier(make_experiment(root))
        f0_dev, f0s = b._pitch(*_front(b, (ama, prof, emb)))
        frames = [len(f) for f in f0s]
        t = [x.clone() for x in torch.split(f0_dev.double(), frames)]
        del b, f0_dev
    N = len(frames) // 2
    srcs, tgts = t[:N], t[N:]
    res['songs_frames'] = [[frames[i], frames[N + i]] for i in range(N)]
    res['songs'] = measure({'align_long_grouped': align_long_grouped, 'single_pass': align_songs(24 * GiB),
                            'checkpointed_1GiB': align_songs(GiB)}, srcs, tgts, args.repeats)
    a, p = S.make_f0_pair(3, 65536, 65536)
    res['pair_65536'] = measure({'single_pass': align_songs(24 * GiB), 'checkpointed_1GiB': align_songs(GiB)},
                                [torch.from_numpy(a).cuda()], [torch.from_numpy(p).cuda()], args.big_repeats)
    print(f"card: {res['card']}")
    for part in ('songs', 'pair_65536'):
        for name, r in res[part].items():
            print(f"  {part} {name}: median {r['median_s']:.3f} s {r['s']}, peak {r['peak_GB']:.2f} GB, plan {r.get('plan')}, "
                  f"stages {r['median_stage_ms']} ms, equal {r['equal_to_first']}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()

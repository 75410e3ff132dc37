"""The paper's comparison of pitch alignments (tasks/singing/pitch_alignment_task.py of the reference) on the GPU: every item of
a paired IndexedDataset (f0, mel2ph, prof_f0, prof_mel2ph) is aligned amateur -> professional by each requested method, in batches,
and scored by the alignment accuracy (prof_mel2ph == mel2ph[alignment]).sum() / (prof_mel2ph != 0).sum().

    python tools/pitch_align_eval.py --data DIR/train --methods EHSADTW,SADTW,LoNDTW,ZMNaiveDTW,NNaiveDTW,NInterpo [--save DIR]

The f0 fed to the alignment is the dataset's round trip: norm_interp_f0, then denorm_f0 with the padding frames (mel2ph == 0)
zeroed.  NaiveDTW runs on the [T, 1] f0 here.  Prints 'avg / max / min' accuracy per method; --save writes
{item_name}_alignment.npy per item and method under DIR/a2p_alignments_by_{method}.
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from neuralsvb_b200.modules.voice_conversion.dtw import core  # noqa: E402
from neuralsvb_b200.utils import pitch_utils as PU  # noqa: E402
from neuralsvb_b200.utils.indexed_datasets import IndexedDataset  # noqa: E402


def load_items(path, hparams):
    ds = IndexedDataset(path)
    items = []
    for i in range(len(ds)):
        it = ds[i]
        rec = {'item_name': it.get('item_name', str(i))}
        for pre in ('', 'prof_'):
            mel2ph = torch.as_tensor(np.asarray(it[f'{pre}mel2ph']), dtype=torch.int64)
            f0, uv = PU.norm_interp_f0(np.asarray(it[f'{pre}f0'])[:len(mel2ph)], hparams)
            rec[f'{pre}f0'] = PU.denorm_f0(f0, uv, hparams, pitch_padding=mel2ph == 0)
            rec[f'{pre}mel2ph'] = mel2ph
        items.append(rec)
    return items


def evaluate(items, methods, batch=64, save=None):
    """{method: float64 accuracies [n]}; with save, writes each alignment as {save}/a2p_alignments_by_{method}/{item}_alignment.npy."""
    out = {}
    for method in methods:
        accs = []
        for b0 in range(0, len(items), batch):
            chunk = items[b0:b0 + batch]
            r = core.align_batch([it['f0'] for it in chunk], [it['prof_f0'] for it in chunk], method)
            accs.append(core.alignment_accuracy(r, [it['mel2ph'] for it in chunk], [it['prof_mel2ph'] for it in chunk]))
            if save:
                d = os.path.join(save, f'a2p_alignments_by_{method}')
                os.makedirs(d, exist_ok=True)
                for it, al in zip(chunk, r.split()):
                    np.save(os.path.join(d, f"{it['item_name']}_alignment.npy"), al)
        out[method] = np.concatenate(accs)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--data', required=True, help='IndexedDataset path prefix ({path}.idx / {path}.data)')
    ap.add_argument('--methods', default=','.join(core.METHODS))
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--pitch-norm', default='log', choices=('log', 'standard'))
    ap.add_argument('--f0-mean', type=float, default=0.0)
    ap.add_argument('--f0-std', type=float, default=1.0)
    ap.add_argument('--save', default=None, help='directory for {item}_alignment.npy')
    a = ap.parse_args(argv)
    methods = a.methods.split(',')
    for m in methods:
        if m not in core.METHODS:
            ap.error(f'unknown method {m!r} (one of {", ".join(core.METHODS)})')
    hp = dict(pitch_norm=a.pitch_norm, use_uv=True, f0_mean=a.f0_mean, f0_std=a.f0_std)
    items = load_items(a.data, hp)
    res = evaluate(items, methods, a.batch, a.save)
    for m, acc in res.items():
        print(f'{m}: avg {acc.mean():.6f} max {acc.max():.6f} min {acc.min():.6f} ({len(acc)} items)')
    return res


if __name__ == '__main__':
    main()

"""Drop-in for modules/voice_conversion/dtw/local_norm_dtw.py (LoNDTW) on the GPU: the local-context features, the cdist cost, the
DTW and the backtrack run in csrc/sadtw.cu.  Names, signatures and return types are the reference's; f0 may be numpy or torch, on
the host or on a CUDA device, float32 or float64 (the cost is computed in that type, as in the reference)."""
import torch

from neuralsvb_b200.modules.voice_conversion.dtw import core as _core

METHOD = 'LoNDTW'


def get_local_context(input_f, max_window=32, scale_factor=1.):
    """[S, 2 max_window] list of lists: row t = input_f[t - max_window .. t + max_window - 1], 0 outside [0, S).  scale_factor is
    unused, as in the reference.  A host-side view for inspection; the alignment builds the contexts on the device."""
    f = _core.as_tensor(input_f).reshape(-1).cpu()
    z = torch.zeros(max_window, dtype=f.dtype)
    return torch.cat([z, f, z]).unfold(0, 2 * max_window, 1)[:f.shape[0]].tolist()


def cal_localnorm_dist(src, tgt, src_len, tgt_len):
    """[1, S, T] cdist between the mean-removed 64-frame contexts of src and tgt, in the input's type, on src's device."""
    d = _core.baseline_costs([src], [tgt], METHOD)[0]
    return d.unsqueeze(0).to(src.device if torch.is_tensor(src) else torch.device('cpu'))


def DTW_align(srcs, tgts, inputs, srcs_lens=None, tgt_lens=None):
    """Batch API: srcs [B, S] / tgts [B, T] f0, inputs [B, S, ...] -> inputs aligned to the professional frames, [B, T, ...].  Each
    pair uses its whole padded rows, as the reference does (the lengths are not used); all pairs run in one launch sequence."""
    B = len(srcs)
    r = _core.align_batch([srcs[b] for b in range(B)], [tgts[b] for b in range(B)], METHOD)
    return torch.stack([inputs[b][a.tolist()] for b, a in enumerate(r.split())], dim=0)


def LoNDTW(src, tgt, input):
    """One pair: (input[alignment], alignment), alignment a list of T amateur frame indices."""
    return _core.align_one(src, tgt, input, METHOD)


def spec_to_figure(spec, vmin=None, vmax=None, name=''):
    raise NotImplementedError('plotting is not part of neuralsvb_b200')


def f0_to_figure(f0_src, f0_aligned=None, f0_prof=None, name='f0.png'):
    raise NotImplementedError('plotting is not part of neuralsvb_b200')

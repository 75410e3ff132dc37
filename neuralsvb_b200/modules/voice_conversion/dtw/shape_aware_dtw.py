"""Drop-in for modules/voice_conversion/dtw/shape_aware_dtw.py (SADTW) on the GPU: the slope histograms, the chi-square cost,
the DTW and the backtrack all run in csrc/sadtw.cu.  Names, signatures and return types are the reference's; f0 may be numpy or
torch, on the host or on a CUDA device, float32 or float64 (the histogram arithmetic runs in that type, as in the reference)."""
from neuralsvb_b200.modules.voice_conversion.dtw import core as _core

METHOD = 'SADTW'


def cal_hist_of_f0(input_f, max_window=64, normalize_hist=False, scale_factor=1.):
    """[S, 48] slope histogram as a list of lists (ints, or k / total with normalize_hist); only max_window=64 is implemented."""
    return _core.hist_of_f0(input_f, METHOD, max_window, normalize_hist, scale_factor)


def cal_hist_dist(hist_a, hist_b):
    """[T1, T2] float32: sum over the 48 bins of 0.5 (b - a)^2 / (b + a + 1e-8)."""
    return _core.hist_dist(hist_a, hist_b)


def cal_shape_dist(src, tgt, src_len, tgt_len):
    """[1, S, T] float32 cost between the normalised histograms of src (scale 1) and tgt (scale tgt_len / src_len)."""
    return _core.shape_dist(src, tgt, src_len, tgt_len, METHOD)


def DTW_align(srcs, tgts, inputs, srcs_lens=None, tgt_lens=None):
    """Batch API: srcs [B, S, H] / tgts [B, T, H] f0, inputs [B, S, ...] -> inputs aligned to the professional frames, [B, T, ...].
    All pairs run in one launch sequence; lengths default to the padded ones."""
    return _core.dtw_align_batch(srcs, tgts, inputs, srcs_lens, tgt_lens, METHOD)


def SADTW(src, tgt, input):
    """One pair: (input[alignment], alignment), alignment a list of T amateur frame indices."""
    return _core.align_one(src, tgt, input, METHOD)


def spec_to_figure(spec, vmin=None, vmax=None, name='', dir='tmp'):
    raise NotImplementedError('plotting is not part of neuralsvb_b200')


def f0_to_figure(f0_src, f0_aligned=None, f0_prof=None, name='f0.png', dir='tmp'):
    raise NotImplementedError('plotting is not part of neuralsvb_b200')

"""Drop-in for modules/voice_conversion/dtw/enhance_sadtw.py (EHSADTW, the binarizer's default pitch alignment) on the GPU:
sixteen-frame slope windows with the slopes of the outer windows damped (x0.5 / 0.75 / 0.9), then the same cost, DTW and
backtrack as SADTW, all in csrc/sadtw.cu.  Names, signatures and return types are the reference's."""
from neuralsvb_b200.modules.voice_conversion.dtw import core as _core

METHOD = 'EHSADTW'


def cal_hist_of_f0(input_f, max_window=64, normalize_hist=False, scale_factor=1.):
    """[S, 48] slope histogram as a list of lists (ints, or k / total with normalize_hist); only max_window=64 is implemented."""
    return _core.hist_of_f0(input_f, METHOD, max_window, normalize_hist, scale_factor)


def cal_hist_dist(hist_a, hist_b, src=None, tgt=None):
    """[T1, T2] float32: sum over the 48 bins of 0.5 (b - a)^2 / (b + a + 1e-8); src / tgt are unused, as in the reference."""
    return _core.hist_dist(hist_a, hist_b)


def cal_shape_dist(src, tgt, src_len, tgt_len):
    """[1, S, T] float32 cost between the normalised histograms of src (scale 1) and tgt (scale tgt_len / src_len)."""
    return _core.shape_dist(src, tgt, src_len, tgt_len, METHOD)


def EHSADTW(src, tgt, input):
    """One pair: (input[alignment], alignment), alignment a list of T amateur frame indices."""
    return _core.align_one(src, tgt, input, METHOD)

"""Drop-in for modules/voice_conversion/dtw/align.py on the GPU: the DTW recurrence and the backtrack of csrc/sadtw.cu on an
arbitrary float32 or float64 cost matrix (numpy or torch, host or device).  The results are the reference's bit for bit: the
recurrence runs in the cost's type and both minimums keep the first operand unless a later one is strictly smaller."""
from neuralsvb_b200.modules.voice_conversion.dtw import core as _core


def time_warp(costs):
    """dtw [rows, cols] as a numpy array of the cost's type: dtw[0, 0] = 0, the rest of row 0 and column 0 inf,
    dtw[i, j] = costs[i, j] + min(dtw[i-1, j], dtw[i, j-1], dtw[i-1, j-1])."""
    _, _, full = _core.dtw(costs, alignment=False, matrix=True)
    return full.cpu().numpy()


def align_from_distances(distance_matrix, debug=False):
    """For each row of the distance matrix the column the monotonic DTW path assigns it, as a Python list."""
    if debug:
        raise NotImplementedError('align_from_distances(debug=True) plots the path; plotting is not part of neuralsvb_b200')
    al, _, _ = _core.dtw(distance_matrix)
    return al.cpu().tolist()

"""Pitch alignment on the GPU (csrc/sadtw.cu): drop-ins for the reference's modules/voice_conversion/dtw/ ``align``,
``shape_aware_dtw`` (SADTW), ``enhance_sadtw`` (EHSADTW), ``local_norm_dtw`` (LoNDTW), ``naive_dtw`` (NaiveDTW, ZMNaiveDTW,
NNaiveDTW) and ``naive_interpo`` (NInterpo), and the batched helpers ``align_pitch`` (a binarizer's a2p alignments),
``a2p_alignment_batch`` (MleSVBVAE's a2p_alignment from f0) and ``alignment_accuracy`` (the paper's mel2ph accuracy)."""
from neuralsvb_b200.modules.voice_conversion.dtw.core import a2p_alignment_batch, align_pitch, alignment_accuracy  # noqa: F401

"""Shape-aware DTW pitch alignment on the GPU (csrc/sadtw.cu): drop-ins for the reference's modules/voice_conversion/dtw/
``align``, ``shape_aware_dtw`` (SADTW) and ``enhance_sadtw`` (EHSADTW), and the batched helpers ``align_pitch`` (a binarizer's
a2p alignments) and ``a2p_alignment_batch`` (MleSVBVAE's a2p_alignment from f0)."""
from neuralsvb_b200.modules.voice_conversion.dtw.core import a2p_alignment_batch, align_pitch  # noqa: F401

"""must3r_b200: H100-native (sm_90a) implementation of the MUSt3R multi-view inference hot path.

Public surface mirrors the reference: ``must3r_b200.model`` (load_model, Dust3rEncoder, MUSt3R, ...) and
``must3r_b200.engine`` (inference_multi_ar, inference_video_multi_ar, inference, postprocess, ...).
All compute runs in hand-written CUDA kernels behind the C ABI of ``include/must3r_b200.h``
(``libm3r_b200.so``); there is no CPU or PyTorch fallback.
"""
__version__ = "0.1.0"

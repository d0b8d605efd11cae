"""GPU-native Augmented Autoencoder hot path for the NVIDIA H100 (encoder -> latent -> codebook match; decoder + training step).

Python host code over torch tensors (device memory, streams, torch.distributed) calling hand-written sm_90a
CUDA through the C ABI in include/aae_b200.h.  The class surface mirrors the reference's ``auto_pose.ae``
(Encoder / Decoder / Codebook / AE / factory) and ``auto_pose.m3_interface.AePoseEstimator``.
There is no CPU fallback: every compute entry point raises if the CUDA library or a GPU is missing.
"""
__version__ = "0.1.0"

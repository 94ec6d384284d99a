"""stp3_b200 — H100-native (sm_90a) implementation of ST-P3's camera->BEV perception hot path.

Host side: Python/PyTorch modules that keep the reference's nn.Module surfaces
(stp3.models.encoder.Encoder, stp3.layers.temporal.TemporalBlock, stp3.models.temporal_model.TemporalModel,
stp3.models.decoder.Decoder, stp3.models.stp3.STP3) and call hand-written CUDA through the C ABI declared
in include/stp3_b200.h (libstp3_b200.so, loaded with ctypes).  There is no CPU fallback: the ops raise if
the library or a CUDA device is missing.
"""
__version__ = "0.1.0"

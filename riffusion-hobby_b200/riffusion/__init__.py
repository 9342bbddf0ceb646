"""riffusion — H100-native drop-in for the two hot paths of riffusion/riffusion-hobby.

Same import paths and call signatures as the reference package
(`riffusion.spectrogram_converter.SpectrogramConverter`, ...); the arithmetic runs in
hand-written sm_90a CUDA kernels behind the C-ABI in include/rf_b200.h.
"""
__version__ = "0.1.0"

"""paddlemix_b200 — H100-native (sm_90a) implementation of PaddleMIX's denoiser-forward / ViT+LLM attention hot path.

Layout: csrc/ (hand-written CUDA kernels + C ABI -> libb200mix.so), _lib.py (ctypes binding), ops.py (tensor-level
wrappers), ppdiffusers/ (host-side mirrors of the reference's UNet2DConditionModel / schedulers / pipeline loop).
Importing the package does not touch the GPU; importing `paddlemix_b200.ops` loads libb200mix.so and fails loudly
if it has not been built.
"""
__version__ = "0.1.0"

"""jepa_b200: H100-native (sm_90a) V-JEPA pre-training hot path.

csrc/ holds the hand-written CUDA kernels behind the C ABI of include/vjepa_b200.h; the Python
modules mirror the reference's src/ and app/ API on top of it.  PyTorch provides device memory,
streams, autograd edges and torch.distributed only.
"""
__version__ = "0.1.0"

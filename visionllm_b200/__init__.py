"""visionllm_b200 -- H100-native (sm_90a) forward hot path of VisionLLM v2.

Host code is Python/PyTorch (device memory, streams, torch.distributed);
compute is hand-written CUDA behind the C-ABI library ``lib/libvllm_b200.so``
(``include/vllm_b200.h``).  There is no CPU fallback: importing an operator
without the built library raises.
"""
__version__ = "0.1"

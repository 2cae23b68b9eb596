"""bitnetmcu_b200 -- H100-native drop-in for the integer inference hot path of cpldcpu/BitNetMCU.

Package contents (only what the path needs):
  csrc/            hand-written sm_90a CUDA (fused wgmma FC chain, CUDA-core layer kernels, CNN front-end) + C ABI
  model.py         BitNetMCU_model.h parser / runtime descriptor / BNM1 blob
  pack.py          exportquant-compatible weight packer
  engine.py        host-side mirror of the reference interface over the C ABI
  dist.py          batch sharding across the GPUs of one box (torch.distributed as plumbing)
"""
from . import model, pack  # noqa: F401

__all__ = ["model", "pack"]

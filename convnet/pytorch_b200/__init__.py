"""convnet.pytorch_b200 -- a Hopper (sm_90a) native training hot path behind the public surface of
eladhoffer/convNet.pytorch: ``trainer.Trainer``, the ``models`` registry (ResNet / ResNeXt / MobileNet-v2),
``utils.optim.OptimRegime`` regimes and the ``main.py`` CLI.

Layout
  csrc/ + libb200conv.so   hand-written CUDA kernels behind the C ABI of include/b200conv.h
  lib.py, ops.py           ctypes binding / tensor-level wrappers (no fallback path)
  engine.py                parameter arenas, fused block forward/backward built on the kernels
  models/, trainer.py, data.py, main.py, utils/   host side mirroring the reference interface
"""
__version__ = "0.1.0"

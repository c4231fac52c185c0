"""fastdepth_b200 -- H100-native FastDepth forward path (MobileNetSkipAdd.forward).

Python host side of the C-ABI in include/fastdepth_b200.h:

  build     in-tree nvcc build of libfastdepth_b200.so (sm_90a)
  _lib      ctypes binding (fails loudly if the library is missing; no fallback)
  plan      BN folding + stage description + Plan wrapper around fd_plan
  engine    lazy per-shape plan cache behind models.MobileNetSkipAdd.forward
  evaluate  image-sharded evaluation with one all-reduce of the metric sums
  synthetic deterministic weights / inputs (no trained weights exist offline)

The importable package is ``fastdepth_b200`` (a hyphen cannot appear in a Python package
name, so the task's ``fast-depth_b200`` spelling maps to this directory).
"""
__version__ = '0.1.0'

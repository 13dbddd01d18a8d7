"""cotr_b200 - H100-native (sm_90a) implementation of the COTR correspondence-inference hot path.

Layout (mirrors the reference's packages for this path only):
  csrc/       hand-written CUDA kernels + the C ABI (include/cotr_b200.h)
  capi.py     ctypes binding of the C ABI
  models/     build_model(args) -> nn.Module with the reference's state_dict schema (COTR/models)
  inference/  SparseEngine / FasterSparseEngine / cotr_flow / cotr_corr_base (COTR/inference)
  utils/, options/, global_configs/   the boundary helpers the reference demos import
"""
__version__ = "0.1.0"

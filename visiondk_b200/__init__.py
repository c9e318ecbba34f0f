"""visiondk_b200 — the sm_90a (H100) implementation of DORAEMON's (wuji3/visiondk) embedding hot path.

Only what the path needs lives here:
  csrc/        hand-written CUDA (wgmma / TMA) behind the C ABI declared in include/vdk_b200.h
  _lib.py      ctypes binding of libvdk_b200.so (fails loudly when the library or an H100 is missing)
  retrieval.py FlatIPIndex / index() / search(): the faiss seam of engine/cbir/evaluation.py
  ...
"""
__version__ = "0.1.0"

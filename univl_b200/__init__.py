"""univl_b200 — H100-native (sm_90a) implementation of the UniVL data-parallel transformer hot path.

`univl_b200.modules` mirrors the reference's `modules` package (UniVL, BertModel, ... same class surface and
checkpoint layout); `univl_b200.lib` is the ctypes binding of the C-ABI kernel library (include/univl_b200.h).
"""
__version__ = "0.1.0"

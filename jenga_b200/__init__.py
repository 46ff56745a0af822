"""jenga_b200 — H100-native (sm_90a) AttenCarve hot path of dvlab-research/Jenga.

Public surface mirrors the reference's operator for this path:
  jenga_b200.attention.block_sparse_attention(...)   (hyvideo / hyvideo_i2v / wan variants)
  jenga_b200.gilbert.*                               (curve permutations, block adjacency)
The compute lives in libjenga_b200.so (C-ABI, include/jenga_b200.h); Python only moves
pointers.  There is no fallback path.
"""
__version__ = "0.1.0"

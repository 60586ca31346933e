"""gem_b200 -- H100 (sm_90a) core for GEM's HOPE and node2vec behind the StaticGraphEmbedding API.

    from gem_b200.embedding.hope import HOPE
    from gem_b200.embedding.node2vec import node2vec

Python host code -> ctypes -> libgemb200.so (hand-written CUDA).  No CPU fallback.
"""
__version__ = '0.1.0'

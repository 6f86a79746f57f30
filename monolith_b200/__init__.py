"""monolith_b200 — H100-native collisionless-embedding engine behind Monolith's MultiHashTable op surface (the package
keeps the name it was first written under).

Only the embedding hot path is here (see DESIGN.md): hand-written sm_90a CUDA in csrc/ behind the
C ABI of include/mono_emb.h, and a host-side mirror of the reference's Python interface
(monolith/native_training/{multi_hash_table_ops,distribution_ops,distributed_ps,entry}.py).
There is no CPU fallback: compute entry points raise when the CUDA library or a GPU is missing.
"""
from . import entry  # noqa: F401
from .multi_hash_table_ops import MultiHashTable, PoolPart  # noqa: F401

__all__ = ["entry", "MultiHashTable", "PoolPart"]

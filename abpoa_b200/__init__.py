"""abpoa_b200 -- H100-native adaptive-banded partial-order alignment.

The product is the C-ABI shared library ``abpoa_b200/lib/libabpoa_b200.so`` (host C behind
abPOA's ``abpoa.h`` interface + hand-written sm_90a CUDA kernels, built by
``__graft_entry__.build()`` / ``make``).  This package is the thin Python host-side mirror of
the reference's Python interface (pyabpoa) on top of that library.
"""
from .aligner import PoaConfig, PoaSession, decode, encode, msa_aligner, msa_result  # noqa: F401
from . import capi, synth  # noqa: F401

__all__ = ["PoaConfig", "PoaSession", "msa_aligner", "msa_result", "encode", "decode", "capi", "synth"]

"""reversi_zero_b200 -- H100-native self-play hot path for reversi-alpha-zero.

Host-side mirror of the reference's Python interface for the self-play path (``ReversiEnv``,
``ReversiPlayer``, ``ReversiModelAPI``, ``SelfPlayWorker``, ``lib.bitboard``) over the C ABI of
``csrc/librz_engine.so`` (include/rz_engine.h).  All compute is hand-written sm_90a CUDA; there is
no CPU fallback -- calls raise if the shared library is missing.
"""
__version__ = "0.1.0"

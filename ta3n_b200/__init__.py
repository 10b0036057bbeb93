"""ta3n_b200 -- H100 (sm_90a) implementation of the TA3N hot path.

Drop-in for the reference's ``models.VideoModel`` / ``TRNmodule.RelationModuleMultiScale`` /
``opts.parser`` on the path ``frame_aggregation='trn-m'`` (TRN-M relation aggregation +
domain-attentive pooling + gradient-reversal discriminators).  All arithmetic runs in
hand-written CUDA behind the C ABI of ``include/ta3n_b200.h``; there is no CPU fallback.
"""
from ._lib import Ta3nError, get_gemm_engine, launch_count, reset_launch_count, set_gemm_engine  # noqa: F401

__all__ = ["Ta3nError", "set_gemm_engine", "get_gemm_engine", "launch_count", "reset_launch_count"]

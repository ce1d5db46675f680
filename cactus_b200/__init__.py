"""cactus_b200 -- H100-native engine for Cactus' BAR phase (POA mode and the cPecan pair-HMM posteriors).

Python mirror of the reference's POA entry points (bar/inc/poaBarAligner.h) on top of the C ABI of
``libbarb200.so`` (include/barb200.h). The library is CUDA-only: importing works anywhere, but creating an
:class:`Engine` without a CUDA device (or without the built library) raises -- there is no CPU fallback.
"""
from .api import (Engine, Msa, BarB200Error, PoaParams, PairwiseAlignmentParameters, MumParams, load_library, library_path,
                  msa_to_base, msa_to_byte, parse_trace, first_trace_difference, parse_end_trace, first_end_trace_difference,
                  pecan_band, pecan_split_points)

__all__ = ["Engine", "Msa", "BarB200Error", "PoaParams", "PairwiseAlignmentParameters", "MumParams", "load_library", "library_path",
           "msa_to_base", "msa_to_byte", "parse_trace", "first_trace_difference", "parse_end_trace",
           "first_end_trace_difference", "pecan_band", "pecan_split_points"]

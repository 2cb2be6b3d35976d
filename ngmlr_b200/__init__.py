"""ngmlr_b200 -- H100-native (sm_90a CUDA) implementation of ngmlr's alignment hot path behind the
reference's IAlignment plugin surface. See DESIGN.md / INTEGRATION.md."""
from .aligner import (Align, B200Aligner, IntervalBatch, PackedBatch, PackedReads, select_candidates, split_read,  # noqa: F401
                      DEFAULT_SCORING)

__all__ = ["Align", "B200Aligner", "IntervalBatch", "PackedBatch", "PackedReads", "select_candidates", "split_read", "DEFAULT_SCORING"]

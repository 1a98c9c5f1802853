"""Root-level shim so that the reference's plugin seam `run.py -g gru4rec` (run.py:21,39) and pickles that
name `gru4rec.GRU4Rec` resolve to the CUDA implementation."""
from gru4rec_b200.gru4rec import GRU4Rec  # noqa: F401

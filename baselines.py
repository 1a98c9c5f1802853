"""Root-level shim: `import baselines` resolves to the device implementation of the reference's session baselines: Pop,
SessionPop, ItemKNN and BPR (BPR-MF), and session-based kNN (SessionKNN, STAN)."""
from gru4rec_b200.baselines import Pop, SessionPop, ItemKNN, BPR, SessionKNN, STAN  # noqa: F401

"""Root-level shim: `import baselines` resolves to the device implementation of the reference's session baselines: Pop,
SessionPop, ItemKNN and BPR (BPR-MF)."""
from gru4rec_b200.baselines import Pop, SessionPop, ItemKNN, BPR  # noqa: F401

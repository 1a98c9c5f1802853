"""Root-level shim: `import baselines` resolves to the device implementation of the reference's session baselines."""
from gru4rec_b200.baselines import Pop, SessionPop, ItemKNN  # noqa: F401

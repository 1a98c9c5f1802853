"""Root-level shim: `import baselines` resolves to the device implementation of the reference's session baselines: Pop,
SessionPop, ItemKNN and BPR (BPR-MF), session-based kNN (SessionKNN, STAN, VSTAN), the rule-based baselines (SR, AR) and the
neural NARM, SASRec, SR-GNN, STAMP, NextItNet and BERT4Rec."""
from gru4rec_b200.baselines import Pop, SessionPop, ItemKNN, BPR, SessionKNN, STAN, VSTAN, SR, AR, NARM, SASRec, SRGNN, STAMP, NextItNet, BERT4Rec  # noqa: F401

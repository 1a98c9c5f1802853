"""Root-level shim: `import evaluation` in run.py (run.py:40) resolves to the CUDA implementation."""
from gru4rec_b200.evaluation import evaluate_gpu, evaluate_events, evaluate_rest  # noqa: F401

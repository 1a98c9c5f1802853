"""TEST INFRASTRUCTURE ONLY.  Runs the reference's datatools.py (plain pandas / NumPy) on the frames of
tests/golden_utils.datatools_cases() and records what sort_if_needed printed, the frame it left behind and compute_offset's result
-> tests/golden/datatools/cases.npz.  tests/test_host_logic.py replays the cases through gru4rec_b200/datatools.py.

Usage: python oracle/make_datatools_golden.py <directory of the reference checkout>"""
import importlib.util
import json
import os
import sys
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from golden_utils import GOLDEN_DIR, datatools_cases, datatools_outcome  # noqa: E402

spec = importlib.util.spec_from_file_location('ref_datatools', os.path.join(sys.argv[1], 'datatools.py'))
ref = importlib.util.module_from_spec(spec); spec.loader.exec_module(ref)
lines, frames, offsets = [], [], []
for df, cols, any_order in datatools_cases():
    l, f, o = datatools_outcome(ref, df, cols, any_order)
    lines.append(l); frames.append(f); offsets.append(o)
path = os.path.join(GOLDEN_DIR, 'datatools', 'cases.npz')
np.savez_compressed(path, lines=json.dumps(lines), frame_rows=np.array([len(f) for f in frames], np.int32),
                    frames=np.concatenate(frames).astype(np.int16), offset_len=np.array([len(o) for o in offsets], np.int32),
                    offsets=np.concatenate(offsets), offset_dtype=str(offsets[0].dtype))
print('wrote', path, len(lines), 'cases')

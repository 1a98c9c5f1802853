"""The C ABI of per-event evaluation from a C99 caller, without a device: an evaluation schedule's positions (g4r_schedule_positions)
and g4r_eval_events' argument checks."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r'''
#include <stdio.h>
#include "g4r.h"

int main(void) {
  /* sessions [10 11 12] [13] [14 15]: the single-event session yields no event */
  const int64_t items[6] = {10, 11, 12, 13, 14, 15};
  const int32_t off[4] = {0, 3, 4, 6};
  g4r_schedule* s = NULL;
  int64_t pos[16];
  int32_t cut = 20, counts[8];
  double rec = 0.0, mrr = 0.0;
  int64_t i, n, steps;
  if (g4r_schedule_build(items, 6, off, 3, NULL, 2, 0, 1 | G4R_SCHED_POSITIONS, &s) != G4R_OK) return 1;
  steps = g4r_schedule_steps(s);
  n = g4r_schedule_events(s);
  if (steps * 2 > 16 || g4r_schedule_positions(s, pos) != G4R_OK) return 2;
  for (i = 0; i < steps * 2; i++) printf("%lld ", (long long)pos[i]);
  printf("| %lld\n", (long long)n);
  if (g4r_eval_events(NULL, s, &cut, 1, 0, 0, &rec, &mrr, &n, counts, NULL, NULL) != G4R_ERR_INVALID) return 3;
  g4r_schedule_free(s);
  for (i = 0; i < 2; i++) {       /* training and plain evaluation schedules record no positions */
    if (g4r_schedule_build(items, 6, off, 3, NULL, 2, 0, (int32_t)i, &s) != G4R_OK) return 4;
    if (g4r_schedule_positions(s, pos) != G4R_ERR_STATE) return 5;
    g4r_schedule_free(s);
  }
  return 0;
}
'''


def test_c99_caller_of_eval_events(tmp_path):
    gcc = shutil.which('gcc') or shutil.which('cc')
    if gcc is None:
        pytest.skip('no C compiler')
    inc, libdir = os.path.join(ROOT, 'include'), os.path.join(ROOT, 'gru4rec_b200')
    src = tmp_path / 'caller.c'
    src.write_text(SRC)
    exe = str(tmp_path / 'caller')
    cuda_lib = '/usr/local/cuda/lib64'
    r = subprocess.run([gcc, '-std=c99', '-Wall', '-Wextra', '-pedantic', '-Werror', '-I' + inc, str(src), '-L' + libdir, '-lg4r',
                        '-Wl,-rpath,' + libdir, '-L' + cuda_lib, '-Wl,-rpath,' + cuda_lib, '-o', exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    # two lanes: session 0 runs two steps in lane 0 while session 2 takes lane 1; the schedule then ends with one lane
    pos = [int(x) for x in r.stdout.split('|')[0].split()]
    assert sorted(p for p in pos if p >= 0) == [0, 1, 4]
    assert int(r.stdout.split('|')[1]) == 3

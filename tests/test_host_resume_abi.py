"""The C ABI of training-state export / import and catalogue growth from a C99 caller, without a device: the symbols link with
the prototypes of include/g4r.h and refuse null handles before touching anything."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r'''
#include <stdio.h>
#include "g4r.h"

int main(void) {
  size_t n = 7;
  char blob[128] = {0};
  float rows[4] = {0.f, 0.f, 0.f, 0.f};
  int (*bytes)(g4r_handle*, size_t*) = g4r_train_state_bytes;
  int (*exp_)(g4r_handle*, void*, size_t) = g4r_train_state_export;
  int (*imp)(g4r_handle*, const void*, size_t) = g4r_train_state_import;
  int (*grow)(g4r_handle*, g4r_handle*, const float*, const float*, const float*) = g4r_copy_item_tables;
  if (bytes(NULL, &n) != G4R_ERR_INVALID || n != 7) return 1;
  if (exp_(NULL, blob, sizeof blob) != G4R_ERR_INVALID) return 2;
  if (imp(NULL, blob, sizeof blob) != G4R_ERR_INVALID) return 3;
  if (grow(NULL, NULL, rows, rows, NULL) != G4R_ERR_INVALID) return 4;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_train_state_and_growth(tmp_path):
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
    assert r.stdout.startswith('ok ')

"""The ctypes mirror of rvb_wavlm_seg_config has the size gcc gives the C struct (no GPU)."""
import ctypes
import os
import shutil
import subprocess

import pytest

from reverb_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_wavlm_seg_config_mirror_matches_the_c_header(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    src = tmp_path / "size.c"
    src.write_text('#include <stdio.h>\n#include "rvb_diar.h"\n'
                   'int main(void) { printf("%zu\\n", sizeof(rvb_wavlm_seg_config)); return 0; }\n')
    exe = tmp_path / "size"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                   check=True)
    size = int(subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout)
    assert size == ctypes.sizeof(_lib.WavlmSegConfig)

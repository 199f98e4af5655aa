"""The resident-state entry points of libcookgpu.so are exported, and abi.py's StateDelta has the layout of
include/cook_gpu.h's cook_state_delta (checked against the C compiler; no GPU needed)."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from cook_b200 import abi, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_state_symbols_exported():
    if not os.path.exists(engine.LIB_PATH):
        pytest.skip("libcookgpu.so not built")
    lib = engine.load_library()
    for name in ("cook_state_apply", "cook_state_rank", "cook_state_match"):
        assert hasattr(lib, name), name


def test_state_delta_layout(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    fields = [n for n, _ in abi.StateDelta._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "cook_gpu.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(cook_state_delta));\n' +
                   "".join(f'  printf("%zu\\n", offsetof(cook_state_delta, {n}));\n' for n in fields) +
                   '  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(abi.StateDelta)
    assert got[1:] == [getattr(abi.StateDelta, n).offset for n in fields]
    assert abi.PHASE_STATE == 4

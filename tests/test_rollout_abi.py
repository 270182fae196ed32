"""CPU-side checks of the closed-loop rollout's C ABI: tinympc_rollout_t's ctypes mirror matches the header, and the entry point
refuses bad arguments before it touches a device."""
import ctypes as C
import os
import subprocess
import tempfile

from tinympc_b200 import _lib, abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = [n for n, _ in abi.Rollout._fields_]


def test_rollout_layout_matches_header():
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"tinympc_b200.h\"\nint main(void){\n"
    src += '  printf("%zu\\n", sizeof(tinympc_rollout_t));\n'
    src += "".join(f'  printf("%zu\\n", offsetof(tinympc_rollout_t, {n}));\n' for n in FIELDS)
    src += "  return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "probe.c")
        open(c, "w").write(src)
        exe = os.path.join(td, "probe")
        subprocess.check_call(["/usr/bin/gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe], text=True).split()))
    assert out[0] == C.sizeof(abi.Rollout)
    assert out[1:] == [getattr(abi.Rollout, n).offset for n in FIELDS]


def test_rollout_null_arguments():
    lib = _lib.load()
    assert lib.tinympc_b200_rollout(None, None, None, None) == abi.ERR_ARG
    assert b"null" in lib.tinympc_b200_last_error()

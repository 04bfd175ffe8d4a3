"""CPU: the C-ABI library builds/loads and exports every symbol include/avc_b200.h declares
(no compute calls -- there is no GPU here)."""
import os
import re

from conftest import ROOT


def header_functions():
    src = open(os.path.join(ROOT, "include", "avc_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(avc_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    from adaptive_voice_conversion_b200 import _lib as L
    assert header_functions() == sorted(L.PROTOTYPES)


def test_library_exports_every_declared_symbol():
    from adaptive_voice_conversion_b200 import _lib as L
    lib = L.load()
    for name in header_functions():
        assert getattr(lib, name) is not None
    assert b"sm_90a" in lib.avc_build_info()
    assert lib.avc_launch_count() == 0


def test_struct_layouts_match_header_sizes():
    """ctypes mirrors of the descriptor structs have the size the C compiler gives them."""
    import ctypes, subprocess, tempfile
    from adaptive_voice_conversion_b200 import _lib as L
    prog = '#include <stdio.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(avc_conv_desc), sizeof(avc_wgrad_desc), sizeof(avc_fold_desc), sizeof(avc_linear_desc), sizeof(avc_dense_stack_desc), sizeof(avc_linear_batch_desc));return 0;}\n'
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write(prog)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(L.ConvDesc), ctypes.sizeof(L.WgradDesc), ctypes.sizeof(L.FoldDesc), ctypes.sizeof(L.LinearDesc),
                     ctypes.sizeof(L.DenseStackDesc), ctypes.sizeof(L.LinearBatchDesc)]


def test_sass_is_sm90a():
    import subprocess
    from adaptive_voice_conversion_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-lelf", L.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out

"""CPU checks of the C-ABI boundary: libt2h.so loads and exports every symbol
include/t2h.h declares, the ctypes struct mirrors the C struct, and argument
validation fails loudly (no compute calls — there is no GPU here)."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest

from text2human_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "t2h.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(t2h_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    names = declared_symbols()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f"libt2h.so does not export {n}"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in text2human_b200/_lib.py"
    assert sorted(_lib.SIGNATURES) == names


def test_abi_version_matches_header_and_error_string():
    """the library, the header's T2H_VERSION and the ctypes mirrors' ABI_VERSION agree"""
    lib = _lib.load()
    assert lib.t2h_version() == _lib.ABI_VERSION
    assert re.search(r"#define T2H_VERSION (\d+)", open(HEADER).read()).group(1) == str(_lib.ABI_VERSION)
    assert isinstance(lib.t2h_last_error(), bytes)


def test_struct_layout_matches_header():
    """sizeof and the offset of every field of both ctypes mirrors, against the C compiler's view of the header"""
    structs = {"t2h_tapgemm_params": _lib.TapGemmParams, "t2h_conv_wgrad_params": _lib.ConvWgradParams}
    prints, want = [], []
    for cname, py in structs.items():
        prints.append(f'printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        want.append(f"{cname} sizeof {ctypes.sizeof(py)}")
        for field in (f[0] for f in py._fields_):
            prints.append(f'printf("{cname} {field} %zu\\n", offsetof({cname}, {field}));')
            want.append(f"{cname} {field} {getattr(py, field).offset}")
    code = "#include \"t2h.h\"\n#include <stdio.h>\n#include <stddef.h>\nint main(void) {\n" + "\n".join(prints) + \
        "\nreturn 0;\n}\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write(code)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = subprocess.check_output([exe]).decode().splitlines()
    assert got == want


def test_argument_validation_reports_errors():
    lib = _lib.load()
    p = _lib.TapGemmParams()  # all zero: null operands
    rc = lib.t2h_tapgemm(ctypes.byref(p), None)
    assert rc == -1
    assert b"null operand" in lib.t2h_last_error()
    with pytest.raises(_lib.T2HError):
        _lib.check(rc)
    assert lib.t2h_gn_stats(None, None, 1, 1, 32, 32, None) == -1
    assert lib.t2h_vq_search(None, None, None, 1, 1, 1, 4, 1, 1, 1, 1, None, None, None, None, None, None,
                             None, 0, None) == -1


def test_ops_refuse_cpu_tensors():
    import torch
    from text2human_b200 import ops
    with pytest.raises(_lib.T2HError):
        ops.nchw_to_nhwc(torch.zeros(1, 8, 4, 4))

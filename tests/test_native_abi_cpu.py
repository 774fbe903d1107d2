"""The ctypes declarations of libmvb200.so (multiverso_b200/_native.py) against its C header, without a GPU:
every declared signature and every struct mirror must match csrc/cuda/mvb200.h, and every kernel-library
function the Python code calls must be declared."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from multiverso_b200 import _native as N
from test_bindings_abi import _parse_c_decls

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "csrc" / "cuda" / "mvb200.h"

_CT_KIND = {C.c_int: "i32", C.c_int64: "i64", C.c_uint32: "u32", C.c_uint64: "u64", C.c_float: "f32",
            C.c_double: "f64"}


def _ct_kind(t) -> str:
    if t is N.Ptr or t is C.c_char_p or issubclass(t, C._Pointer):
        return "ptr"
    return _CT_KIND[t]


def test_declarations_match_the_header():
    hdr = _parse_c_decls(HEADER.read_text(), prefix="mvb_")
    assert len(hdr) >= 90
    for name, (restype, argtypes, _) in N._CUDA_FUNCS.items():
        assert name in hdr, name
        assert (_ct_kind(restype), [_ct_kind(t) for t in argtypes]) == hdr[name], name


def test_every_called_function_is_declared():
    called = set()
    for path in ROOT.rglob("*.py"):
        rel = path.relative_to(ROOT).parts
        if any(p.startswith(".") or p in ("build", "_ref") for p in rel):
            continue
        called |= set(re.findall(r"\.(mvb_\w+)\b", path.read_text(errors="replace")))
    assert "mvb_ftrl_delta" in called
    assert not called - set(N._CUDA_FUNCS), sorted(called - set(N._CUDA_FUNCS))


def _mirrors():
    return [v for v in vars(N).values() if isinstance(v, type) and issubclass(v, C.Structure)]


def test_struct_mirrors_match_the_c_layout(tmp_path):
    cc = shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler on PATH")
    lines, want = [], []
    for s in _mirrors():
        cname = "Mvb" + s.__name__
        lines.append(f'printf("%zu\\n", sizeof({cname}));')
        want.append((s.__name__, "sizeof", C.sizeof(s)))
        for field, _ in s._fields_:
            cfield = "lambda" if field == "lam" else field
            lines.append(f'printf("%zu\\n", offsetof({cname}, {cfield}));')
            want.append((s.__name__, field, getattr(s, field).offset))
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "mvb200.h"\nint main(void) {\n'
                   + "\n".join(lines) + "\nreturn 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", str(HEADER.parent), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert len(_mirrors()) >= 15 and len(got) == len(want)
    for (struct, field, value), c_value in zip(want, got):
        assert value == int(c_value), (struct, field, value, int(c_value))


def test_loaded_library_behaves_as_declared():
    lib = N.cuda_lib()
    for name in N._CUDA_FUNCS:
        assert hasattr(lib, name), name
    assert lib.mvb_embedding_bag_scratch_bytes(10**9, 300) == 9_406_250_176      # needs the int64_t return
    with pytest.raises(N.NativeError, match=r"^mvb_set_device failed rc=\d+: \S"):
        lib.mvb_set_device(-1)
    with pytest.raises(C.ArgumentError, match="expected a tensor, an int address, a c_void_p or None"):
        lib.mvb_symm_free(1.5)
    assert N.Ptr.from_param(C.c_void_p(4096)).value == 4096          # hand-wrapped pointers still pass

"""Static ABI test of the language bindings that cannot be executed here (no luajit, no dotnet):
every C symbol the Lua FFI cdef and the C# P/Invoke declarations reference must be exported by
libmultiverso.so with the reference's C API names (include/multiverso/c_api.h:16-54)."""
import ctypes
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REFERENCE_C_API = [
    "MV_Init", "MV_ShutDown", "MV_Barrier", "MV_NumWorkers", "MV_WorkerId", "MV_ServerId",
    "MV_NewArrayTable", "MV_GetArrayTable", "MV_AddArrayTable", "MV_AddAsyncArrayTable",
    "MV_NewMatrixTable", "MV_GetMatrixTableAll", "MV_AddMatrixTableAll", "MV_AddAsyncMatrixTableAll",
    "MV_GetMatrixTableByRows", "MV_AddMatrixTableByRows", "MV_AddAsyncMatrixTableByRows",
]


def _lib():
    from multiverso_b200 import _native
    return _native.host_lib()


def test_reference_c_api_symbols_exported():
    lib = _lib()
    for name in REFERENCE_C_API:
        assert hasattr(lib, name), name


def test_lua_cdef_symbols_exported():
    src = open(os.path.join(ROOT, "binding", "lua", "init.lua")).read()
    cdef = src[src.index("ffi.cdef[["):src.index("]]")]
    names = re.findall(r"\b(MV_\w+)\s*\(", cdef)
    assert set(REFERENCE_C_API) <= set(names)
    lib = _lib()
    for n in names:
        assert hasattr(lib, n), n


def test_csharp_pinvoke_symbols_exported():
    src = open(os.path.join(ROOT, "binding", "csharp", "MultiversoWrapper.cs")).read()
    names = re.findall(r"static extern \w+ (MV_\w+)\(", src)
    assert len(names) >= 15
    lib = _lib()
    for n in names:
        assert hasattr(lib, n), n


def test_c_api_roundtrip_through_ctypes():
    """The float-only reference entry points, driven exactly like the reference's Python binding."""
    import numpy as np
    lib = _lib()
    lib.MV_Init(None, None)
    h = ctypes.c_void_p()
    lib.MV_NewArrayTable(100, ctypes.byref(h))
    d = np.arange(100, dtype=np.float32)
    lib.MV_AddArrayTable(h, d.ctypes.data_as(ctypes.c_void_p), 100)
    out = np.zeros(100, np.float32)
    lib.MV_GetArrayTable(h, out.ctypes.data_as(ctypes.c_void_p), 100)
    assert np.array_equal(out, d)
    m = ctypes.c_void_p()
    lib.MV_NewMatrixTable(4, 3, ctypes.byref(m))
    rows = (ctypes.c_int * 2)(1, 3)
    v = np.ones(6, np.float32)
    lib.MV_AddMatrixTableByRows(m, v.ctypes.data_as(ctypes.c_void_p), 6, rows, 2)
    full = np.zeros(12, np.float32)
    lib.MV_GetMatrixTableAll(m, full.ctypes.data_as(ctypes.c_void_p), 12)
    assert full.reshape(4, 3)[[1, 3]].sum() == 6 and full.sum() == 6
    lib.MV_ShutDownEx(0)


def test_gpu_c_api_library_exports_the_reference_abi():
    """libmultiverso_gpu.so (the reference's C API served by the device plane) must export exactly the
    entry points the bindings bind to, unmangled, so that it can be loaded in place of libmultiverso.so."""
    import subprocess
    from multiverso_b200 import _build
    _build.build_device_rt()
    lib = os.path.join(ROOT, "multiverso_b200", "_lib", "libmultiverso_gpu.so")
    assert os.path.exists(lib)
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert set(REFERENCE_C_API) <= exported, set(REFERENCE_C_API) - exported
    assert not [n for n in exported if n.startswith("MV_") and n not in REFERENCE_C_API]


# ---- signature-level checks (parameter count, widths and pointer-ness), still without a Lua / .NET runtime ----
def _c_kind(t: str) -> str:
    t = t.replace("const", " ").strip()
    if "*" in t or "[" in t or t.split()[0] == "TableHandler":
        return "ptr"
    base = t.split()[0]
    return {"int": "i32", "int64_t": "i64", "uint32_t": "u32", "uint64_t": "u64", "float": "f32", "double": "f64",
            "void": "void", "char": "i8"}[base]


def _parse_c_decls(text: str, prefix: str = "MV_"):
    """name -> (return kind, [parameter kinds]) for every ``prefix``* prototype in a C declaration block."""
    out = {}
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"//[^\n]*", " ", text)
    for m in re.finditer(r"(?:DllExport\s+)?((?:const\s+)?\w+\s*\*?)\s*(" + prefix + r"\w+)\s*\(([^)]*)\)\s*;", text):
        ret, name, params = m.group(1), m.group(2), m.group(3).strip()
        kinds = []
        if params and params != "void":
            for p in params.split(","):
                p = " ".join(p.split())
                # drop the parameter name (last identifier) unless the declarator is only a type
                mm = re.match(r"(.*?)(\w+)(\s*\[\s*\])?$", p)
                typ = (mm.group(1) + (mm.group(3) or "")) if mm and mm.group(1).strip() else p
                kinds.append(_c_kind(typ))
        out[name] = (_c_kind(ret), kinds)
    return out


def _header_decls():
    return _parse_c_decls(open(os.path.join(ROOT, "include", "multiverso", "c_api.h")).read())


def test_lua_cdef_signatures_match_the_header():
    src = open(os.path.join(ROOT, "binding", "lua", "init.lua")).read()
    cdef = src[src.index("ffi.cdef[[") + len("ffi.cdef[["):src.index("]]")]
    lua, hdr = _parse_c_decls(cdef), _header_decls()
    assert len(lua) >= len(REFERENCE_C_API)
    for name, sig in lua.items():
        assert hdr[name] == sig, (name, hdr[name], sig)


_CS_KIND = {"int": "i32", "long": "i64", "float": "f32", "double": "f64", "string": "ptr", "IntPtr": "ptr",
            "void": "void"}


def test_csharp_pinvoke_signatures_match_the_header():
    src = open(os.path.join(ROOT, "binding", "csharp", "MultiversoWrapper.cs")).read()
    hdr = _header_decls()
    decls = re.findall(r"static extern (\w+) (MV_\w+)\(([^)]*)\)", src)
    assert len(decls) >= 15
    for ret, name, params in decls:
        kinds = []
        for p in [q for q in (" ".join(x.split()) for x in params.split(",")) if q]:
            toks = p.split()
            typ = toks[-2]                                   # [out|ref] type name
            by_ref = toks[0] in ("out", "ref")
            kinds.append("ptr" if (by_ref or typ.endswith("[]")) else _CS_KIND[typ])
        want_ret, want = hdr[name]
        # the C string return of MV_Version is marshalled as IntPtr
        assert _CS_KIND[ret] == want_ret, (name, ret, want_ret)
        assert kinds == want, (name, kinds, want)

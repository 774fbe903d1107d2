"""In-tree native build of multiverso-b200.

Two artefacts, both built with explicit compiler invocations (no JIT cache, so the
``.so`` files travel with the repo snapshot to the GPU box):

* ``multiverso_b200/_lib/libmvb200.so``      -- sm_90a data-plane kernels (nvcc,
  ``-gencode arch=compute_90a,code=sm_90a -lineinfo``), sources ``csrc/cuda/*.cu``
* ``multiverso_b200/_lib/libmultiverso.so``  -- C++17 host runtime + C API (g++),
  sources ``csrc/host/**/*.cpp``; plus the native tools/apps under ``build/bin``.

Objects are cached under ``build/`` and rebuilt only when a source or header is newer.
"""
from __future__ import annotations

import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
LIBDIR = Path(__file__).resolve().parent / "_lib"
BUILD = ROOT / "build"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]
CXX_FLAGS = ["-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-pthread", "-fopenmp"]


def _newer(src_list, target: Path) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(s).stat().st_mtime > t for s in src_list)


def _run(cmd, what):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"{what} failed:\n{' '.join(map(str, cmd))}\n{r.stdout}\n{r.stderr}")
    return r


def _find(tool, fallback):
    p = shutil.which(tool)
    if p:
        return p
    return fallback if Path(fallback).exists() else None


def build_cuda(verbose: bool = False) -> Path:
    """Compile csrc/cuda/*.cu for sm_90a and link libmvb200.so."""
    nvcc = _find("nvcc", "/usr/local/cuda/bin/nvcc")
    out = LIBDIR / "libmvb200.so"
    srcs = sorted((ROOT / "csrc" / "cuda").glob("*.cu"))
    hdrs = sorted((ROOT / "csrc" / "cuda").glob("*.h")) + sorted((ROOT / "csrc" / "cuda").glob("*.cuh"))
    if nvcc is None:
        if out.exists():
            return out
        raise RuntimeError("nvcc not found and libmvb200.so not prebuilt")
    objdir = BUILD / "cuda"
    objdir.mkdir(parents=True, exist_ok=True)
    LIBDIR.mkdir(parents=True, exist_ok=True)
    inc = []
    cutlass = _cutlass_include()
    if cutlass:
        inc = ["-I", str(cutlass)]

    def one(src: Path):
        obj = objdir / (src.stem + ".o")
        if _newer([src] + hdrs, obj):
            if verbose:
                print(f"[build] nvcc {src.name}", flush=True)
            _run([nvcc, *NVCC_FLAGS, *inc, "-c", str(src), "-o", str(obj)], f"nvcc {src.name}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs) or 1)) as ex:
        objs = list(ex.map(one, srcs))
    if _newer(objs, out):
        _run([nvcc, "-shared", "-o", str(out), *map(str, objs), "-lcuda"], "link libmvb200.so")
    return out


def _cutlass_include():
    try:
        import flashinfer  # noqa: F401
        p = Path(flashinfer.__file__).parent / "data" / "cutlass" / "include"
        if p.exists():
            return p
    except Exception:
        pass
    return None


def build_host(verbose: bool = False) -> Path:
    """Compile the C++17 host runtime (csrc/host) into libmultiverso.so and build the
    native test / app executables under build/bin."""
    cxx = _find("g++", "/usr/bin/g++")
    out = LIBDIR / "libmultiverso.so"
    srcdir = ROOT / "csrc" / "host"
    srcs = sorted(p for p in srcdir.rglob("*.cpp") if "apps" not in p.parts and "tools" not in p.parts)
    if not srcs:
        return out
    hdrs = sorted((ROOT / "include").rglob("*.h")) + sorted(srcdir.rglob("*.h"))
    if cxx is None:
        if out.exists():
            return out
        raise RuntimeError("g++ not found and libmultiverso.so not prebuilt")
    objdir = BUILD / "host"
    objdir.mkdir(parents=True, exist_ok=True)
    LIBDIR.mkdir(parents=True, exist_ok=True)
    inc = ["-I", str(ROOT / "include"), "-I", str(srcdir)]

    def one(src: Path):
        rel = src.relative_to(srcdir)
        obj = objdir / ("_".join(rel.with_suffix("").parts) + ".o")
        if _newer([src] + hdrs, obj):
            if verbose:
                print(f"[build] g++ {rel}", flush=True)
            _run([cxx, *CXX_FLAGS, *inc, "-c", str(src), "-o", str(obj)], f"g++ {rel}")
        return obj

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(one, srcs))
    if _newer(objs, out):
        _run([cxx, "-shared", "-o", str(out), *map(str, objs), "-pthread", "-fopenmp", "-ldl"],
             "link libmultiverso.so")
    # executables: each csrc/host/{apps,tools}/<name>/*.cpp -> build/bin/<name>
    bindir = BUILD / "bin"
    bindir.mkdir(parents=True, exist_ok=True)
    for group in ("apps", "tools"):
        gdir = srcdir / group
        if not gdir.exists():
            continue
        for appdir in sorted(p for p in gdir.iterdir() if p.is_dir()):
            asrcs = sorted(appdir.glob("*.cpp"))
            if not asrcs:
                continue
            exe = bindir / appdir.name
            if _newer(asrcs + hdrs + [out], exe):
                if verbose:
                    print(f"[build] link {exe.name}", flush=True)
                _run([cxx, *CXX_FLAGS, *inc, "-I", str(appdir), *map(str, asrcs), "-o", str(exe),
                      f"-L{LIBDIR}", "-lmultiverso", f"-Wl,-rpath,{LIBDIR}", "-pthread", "-fopenmp"],
                     f"link {exe.name}")
    return out


def build_device_rt(verbose: bool = False) -> Path:
    """Compile the native C++ device runtime (csrc/device_rt -> libmvdevice.so: C++ tables over
    libmvb200.so + the host control plane of libmultiverso.so) and its tools under build/bin."""
    cxx = _find("g++", "/usr/bin/g++")
    out = LIBDIR / "libmvdevice.so"
    srcdir = ROOT / "csrc" / "device_rt"
    srcs = sorted(srcdir.glob("*.cpp"))
    if cxx is None or not srcs:
        return out
    hdrs = sorted((ROOT / "include").rglob("*.h")) + [ROOT / "csrc" / "cuda" / "mvb200.h"] + sorted(srcdir.glob("*.h"))
    inc = ["-I", str(ROOT / "include")]
    # vmm.cpp uses the TYPES of the driver API (cuda.h); the entry points are resolved with dlopen at run time
    nvcc = _find("nvcc", "/usr/local/cuda/bin/nvcc")
    cuda_inc = (Path(nvcc).resolve().parent.parent / "include") if nvcc else Path("/usr/local/cuda/include")
    lib_inc = inc + ["-I", str(cuda_inc)]
    deps = [LIBDIR / "libmultiverso.so", LIBDIR / "libmvb200.so"]
    if _newer(srcs + hdrs + deps, out):
        if verbose:
            print("[build] g++ device_rt -> libmvdevice.so", flush=True)
        _run([cxx, *CXX_FLAGS, *lib_inc, "-shared", *map(str, srcs), "-o", str(out), f"-L{LIBDIR}", "-lmultiverso",
              "-lmvb200", "-ldl", "-Wl,-rpath,$ORIGIN"], "link libmvdevice.so")
    # the reference's C API served by the device plane (what a Lua / C# / ctypes binding can load
    # instead of libmultiverso.so to get HBM-resident tables)
    capi = sorted((srcdir / "c_api_gpu").glob("*.cpp"))
    capi_out = LIBDIR / "libmultiverso_gpu.so"
    if capi and _newer(capi + hdrs + [out], capi_out):
        if verbose:
            print("[build] g++ c_api_gpu -> libmultiverso_gpu.so", flush=True)
        _run([cxx, *CXX_FLAGS, *inc, "-shared", *map(str, capi), "-o", str(capi_out), f"-L{LIBDIR}", "-lmvdevice",
              "-lmultiverso", "-lmvb200", "-Wl,-rpath,$ORIGIN"], "link libmultiverso_gpu.so")
    bindir = BUILD / "bin"
    bindir.mkdir(parents=True, exist_ok=True)
    # executables: csrc/device_rt/{tools,apps}/<name>/*.cpp -> build/bin/<name>; an optional SOURCES
    # file lists extra repository sources and -I include directories shared with the CPU applications
    appdirs = [p for group in ("tools", "apps") if (srcdir / group).exists()
               for p in sorted((srcdir / group).iterdir()) if p.is_dir()]
    for appdir in appdirs:
        asrcs = sorted(appdir.glob("*.cpp"))
        extra_inc = []
        listing = appdir / "SOURCES"
        if listing.exists():
            for line in listing.read_text().splitlines():
                line = line.split("#", 1)[0].strip()
                if line.startswith("-I"):
                    extra_inc += ["-I", str(ROOT / line[2:])]
                elif line:
                    asrcs.append(ROOT / line)
        exe = bindir / appdir.name
        app_hdrs = hdrs + sorted((srcdir.parent / "host" / "apps").rglob("*.h"))
        if asrcs and _newer(asrcs + app_hdrs + [out], exe):
            if verbose:
                print(f"[build] link {exe.name}", flush=True)
            _run([cxx, *CXX_FLAGS, *inc, *extra_inc, *map(str, asrcs), "-o", str(exe), f"-L{LIBDIR}", "-lmvdevice",
                  "-lmultiverso", "-lmvb200", f"-Wl,-rpath,{LIBDIR}"], f"link {exe.name}")
    return out


def build_all(verbose: bool = False):
    build_host(verbose)
    build_cuda(verbose)
    build_device_rt(verbose)


if __name__ == "__main__":
    build_all(verbose=True)
    print("ok")

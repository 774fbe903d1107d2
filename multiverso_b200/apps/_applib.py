"""ctypes signatures of the native application support library (include/multiverso/apps/app_api.h)."""
from __future__ import annotations

import ctypes as C

from .. import _native as N

_lib = None


def run_native(app: str, argv) -> dict:
    """Run the native build/bin/<app> (CPU workers / servers on the host runtime) with `argv`
    and return the JSON result line it prints -- what the Python app drivers fall back to
    when there is no GPU.  Under a rank launcher (tools/mvrun.py, torchrun) every rank execs
    its own copy; the host runtime bootstraps from the inherited MV_RANK / MV_SIZE / MV_PORT
    (or RANK / WORLD_SIZE / MASTER_PORT) environment."""
    import json
    import subprocess
    from .. import _build
    _build.build_host()
    exe = _build.BUILD / "bin" / app
    p = subprocess.run([str(exe), *map(str, argv)], stdout=subprocess.PIPE, text=True)
    stats = {}
    for line in p.stdout.splitlines():
        if line.startswith("{"):
            stats = json.loads(line)
        else:
            print(line)
    if p.returncode != 0:
        raise RuntimeError(f"{exe} exited with {p.returncode}")
    return stats


def lib():
    global _lib
    if _lib is None:
        L = N.host_lib()
        vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int
        L.MVA_DictLoad.restype = vp
        L.MVA_DictLoad.argtypes = [C.c_char_p, i32]
        L.MVA_DictFromCorpus.restype = vp
        L.MVA_DictFromCorpus.argtypes = [C.c_char_p, i32]
        L.MVA_DictSize.argtypes = [vp]
        L.MVA_DictTotalWords.restype = i64
        L.MVA_DictTotalWords.argtypes = [vp]
        L.MVA_DictCounts.argtypes = [vp, vp]
        L.MVA_DictWord.restype = C.c_char_p
        L.MVA_DictWord.argtypes = [vp, i32]
        L.MVA_DictIndex.argtypes = [vp, C.c_char_p]
        L.MVA_DictFree.argtypes = [vp]
        L.MVA_WordCount.restype = i64
        L.MVA_WordCount.argtypes = [C.c_char_p, C.c_char_p, i32]
        L.MVA_CorpusOpen.restype = vp
        L.MVA_CorpusOpen.argtypes = [vp, C.c_char_p, C.c_char_p, C.c_double, C.c_uint64]
        L.MVA_CorpusNextBlock.restype = i64
        L.MVA_CorpusNextBlock.argtypes = [vp, vp, i64, vp]
        L.MVA_CorpusReset.argtypes = [vp]
        L.MVA_CorpusClose.argtypes = [vp]
        L.MVA_HuffmanBuild.argtypes = [vp, i32, i32, vp, vp, vp]
        L.MVA_EdgeListOpen.restype = vp
        L.MVA_EdgeListOpen.argtypes = [C.c_char_p, i32]
        L.MVA_EdgeListError.restype = C.c_char_p
        L.MVA_EdgeListError.argtypes = [vp]
        L.MVA_EdgeListSize.restype = i64
        L.MVA_EdgeListSize.argtypes = [vp]
        L.MVA_EdgeListCopy.argtypes = [vp, vp, vp, vp]
        L.MVA_EdgeListClose.argtypes = [vp]
        L.MVA_LRReaderOpen.restype = vp
        L.MVA_LRReaderOpen.argtypes = [C.c_char_p, C.c_char_p, i32, i64, i32]
        L.MVA_LRReaderNext.restype = i64
        L.MVA_LRReaderNext.argtypes = [vp, i64, i64, vp, vp, vp, vp, vp]
        L.MVA_LRReaderReset.argtypes = [vp]
        L.MVA_LRReaderClose.argtypes = [vp]
        _lib = L
    return _lib

"""CPU-only check of the ctypes binding against include/hs_gpu.h: every entry point's argtypes has one entry per parameter
of its prototype, so that a binding list that drifts from the header fails here rather than passing wrong arguments."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _prototypes():
    """{symbol: parameter count} of every function include/hs_gpu.h declares, comments stripped."""
    text = open(os.path.join(ROOT, "include", "hs_gpu.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    protos = {}
    for m in re.finditer(r"\b(hs_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", text):
        params = m.group(2).strip()
        protos[m.group(1)] = 0 if params in ("", "void") else params.count(",") + 1
    return protos


def test_argtypes_match_the_header():
    from hyperspace_b200 import _native

    assert os.path.exists(_native.LIB_PATH), "libhs_gpu.so not built: run __graft_entry__.build()"
    lib = _native.load_library()
    protos = _prototypes()
    assert sorted(protos) == sorted(_native.EXPORTED_SYMBOLS)
    assert protos["hs_bucket_join_exists"] == 22 and protos["hs_filter_scan_cmp"] == 14
    for sym, n_params in protos.items():
        argtypes = getattr(lib, sym).argtypes or []
        assert len(argtypes) == n_params, f"{sym}: {len(argtypes)} argtypes, {n_params} parameters in hs_gpu.h"

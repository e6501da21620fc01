"""The C-ABI library loads on a box without a GPU and exports every symbol the header declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = set()
    for header in ("gandiva_b200.h", "gandiva_b200_arrow.h"):
        text = open(os.path.join(ROOT, "include", header)).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        names |= set(re.findall(r"\b(gdv_[a-z0-9_]+)\s*\(", text))
    return sorted(names)


def test_header_symbols_exported():
    lib = ctypes.CDLL(os.path.join(ROOT, "gandiva_b200", "libgandiva_b200.so"))
    names = declared_symbols()
    assert len(names) > 45
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, "declared in include/*.h but not exported: %s" % missing


def test_library_loads_without_gpu(gandiva):
    assert gandiva.lib.gdv_version().startswith(b"gandiva_b200")
    # never raises; 0 on this CPU-only container, 1 on a GPU machine
    assert gandiva.lib.gdv_cuda_available() in (0, 1)


def test_no_oracle_in_product():
    """The product package must not import, link, dlopen or call anything under oracle/
    (gandiva_b200/build.py only *builds* the checker next to the product)."""
    pkg = os.path.join(ROOT, "gandiva_b200")
    for dirpath, _, files in os.walk(pkg):
        if "_build" in dirpath or "__pycache__" in dirpath:
            continue
        for f in files:
            if f == "build.py" or not f.endswith((".py", ".cc", ".h", ".cu", ".cuh")):
                continue
            text = open(os.path.join(dirpath, f), errors="replace").read()
            assert "libgdv_oracle" not in text, f
            assert not re.search(r"^\s*(import|from)\s+oracle", text, flags=re.M), f
            assert not re.search(r"#include\s+[\"<][^\">]*(oracle|lineitem\.h)", text), f
            assert "orc_" not in text, f

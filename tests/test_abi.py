"""CPU: the C-ABI shared library loads and exports every symbol include/dph_b200.h declares (no compute calls)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "dph_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dph_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from densephrases_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "run `make` / __graft_entry__.build() first"
    L = ctypes.CDLL(_lib.LIB_PATH)
    names = header_functions()
    assert len(names) >= 30
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, f"declared in include/dph_b200.h but not exported: {missing}"
    assert sorted(_lib.EXPORTS) == names, "densephrases_b200/_lib.py signature table is out of sync with the header"
    assert L.dph_version() >= 100


def test_no_cpu_fallback_without_gpu():
    """The product path must fail loudly when there is no H100 (no silent CPU fallback)."""
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from densephrases_b200 import IvfPqIndex
    with pytest.raises(RuntimeError):
        IvfPqIndex(16)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "densephrases_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "from oracle" not in txt and "import oracle" not in txt and "ivfpq_ref" not in txt.replace("oracle/ivfpq_ref.c", ""), f

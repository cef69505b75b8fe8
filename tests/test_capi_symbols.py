"""CPU-side checks of the drop-in boundary: the shared library loads, exports every symbol declared in
include/dmvio_b200.h, and fails loudly (no CPU fallback) when there is no CUDA device."""
import os
import re

import pytest


def _header_symbols():
    """every entry point declared in include/*.h: the drop-in surface (dmvio_b200.h) and the measurement-only one (dmvio_b200_bench.h)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    syms = set()
    for h in ("dmvio_b200.h", "dmvio_b200_bench.h"):
        txt = open(os.path.join(root, "include", h)).read()
        syms |= set(re.findall(r"\b(dmv_[A-Za-z0-9_]+)\s*\(", txt))
    return sorted(syms)


def test_library_exports_every_declared_symbol():
    import dmvio_b200.capi as c
    L = c.lib()
    syms = _header_symbols()
    assert len(syms) >= 35
    for s in syms:
        assert hasattr(L, s), f"libdmvio_b200.so lacks {s}"
    assert sorted(c.SYMBOLS) == syms
    assert b"sm_90a" in L.dmv_version()


def test_no_cpu_fallback():
    import dmvio_b200.capi as c
    if c.lib().dmv_device_count() > 0:
        pytest.skip("a GPU is visible; the failure path is exercised on the CPU-only box")
    with pytest.raises(c.DmvError, match="no CUDA device"):
        c.BA(640, 480)
    with pytest.raises(c.DmvError, match="no CUDA device"):
        c.CT(640, 480, 4)


def test_product_never_imports_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "dm-vio_b200")
    for dp, _, fns in os.walk(pkg):
        for fn in fns:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dp, fn), errors="ignore").read()
                assert "liborc" not in txt and "from oracle" not in txt and "import oracle" not in txt and "orc_" not in txt, fn


def test_integration_doc_maps_every_symbol():
    """INTEGRATION.md's symbol map names every entry point of the header (full name, or the `_suffix` shorthand used for families like
    `dmv_ba_create / _destroy`)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    doc = open(os.path.join(root, "INTEGRATION.md")).read()
    for s in _header_symbols():
        parts = s.split("_", 2)
        suffix = "_" + parts[2] if len(parts) > 2 else s
        assert s in doc or suffix in doc, f"{s} is not mapped in INTEGRATION.md"

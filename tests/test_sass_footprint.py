"""CPU-side guard on the code size of the single-window BA launch (tools/sass_phases.py): every instruction of
ba_fused_kernel<16, false, false, false> runs once per CTA from a cold instruction cache, so growth costs time directly.
Fails when the single-GPU kernel carries peer-exchange code or grows past its budget."""
import importlib.util
import os
import shutil

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dm-vio_b200", "libdmvio_b200.so")
SRC = os.path.join(ROOT, "dm-vio_b200", "csrc", "ba_fused.cu")
HEADLINE = "ba_fused_kernel<16, false, false, false>"
TOTAL_BUDGET = 3300        # whole kernel (3984 before the exchange code left and phase D was rewritten)
AFTER_BARRIER_BUDGET = 820  # phases D + E (1126 + 317 of inlined exchange code before)


def _tool():
    spec = importlib.util.spec_from_file_location("sass_phases", os.path.join(ROOT, "tools", "sass_phases.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _attribution(kernel):
    cuda_bin = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
    if not all(shutil.which(t) or os.path.exists(os.path.join(cuda_bin, t)) for t in ("cuobjdump", "nvdisasm")):
        pytest.skip("cuobjdump / nvdisasm not available")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    m = _tool()
    prefix = m.mangle(kernel)
    return m.attribute(m.disassemble(LIB, prefix), prefix, m.region_lines(SRC), os.path.basename(SRC))


def test_headline_kernel_has_no_exchange_code():
    rows, _, _ = _attribution(HEADLINE)
    assert rows.get("peer exchange (xchg_*)", 0) == 0, rows


def test_headline_kernel_within_budget():
    rows, total, after = _attribution(HEADLINE)
    assert total <= TOTAL_BUDGET, (total, rows)
    assert after <= AFTER_BARRIER_BUDGET, (after, rows)


def test_sharded_kernel_keeps_the_exchange():
    rows, _, _ = _attribution("ba_fused_kernel<16, false, false, true>")
    assert rows.get("peer exchange (xchg_*)", 0) > 0, rows

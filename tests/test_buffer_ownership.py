"""CPU-side guard on how the library's handles own CUDA memory: every device and pinned host buffer is held by one of the owner types
in csrc/common_host.h, which alone allocate and free, and the dmv_*_destroy functions release nothing by hand (the owners do, when the
handle is deleted).  A hand-written allocation or free list elsewhere is the pattern that leaked and reused freed buffers on
allocation-failure paths."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dm-vio_b200", "csrc")
OWNERS_FILE = "common_host.h"
OWNER_CLASSES = ("CudaBuf", "CudaObj")
MEMORY_CALL = re.compile(r"\bcuda(?:Malloc\w*|HostAlloc|Free\w*)\b")
RELEASE_CALL = re.compile(r"\bcuda(?:Free\w*|EventDestroy|StreamDestroy)\b|\b\w+_(?:free|release)\s*\(")


def _code(text):
    """text with comments blanked out (string and character literals are kept; newlines are kept so line numbers stay)"""
    out, i, n = [], 0, len(text)
    while i < n:
        c = text[i]
        if text.startswith("//", i):
            j = text.find("\n", i)
            i = n if j < 0 else j
        elif text.startswith("/*", i):
            j = text.find("*/", i + 2)
            j = n if j < 0 else j + 2
            out.append("\n" * text.count("\n", i, j))
            i = j
        elif c in "\"'":
            j = i + 1
            while j < n and text[j] != c:
                j += 2 if text[j] == "\\" else 1
            out.append(text[i:j + 1])
            i = j + 1
        else:
            out.append(c)
            i += 1
    return "".join(out)


def _block(code, start):
    """[start, end) of the brace-balanced block whose '{' is the first at or after start"""
    i = code.index("{", start)
    depth = 0
    for j in range(i, len(code)):
        depth += {"{": 1, "}": -1}.get(code[j], 0)
        if depth == 0:
            return i, j + 1
    raise AssertionError("unbalanced braces")


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, _code(f.read())


def test_cuda_memory_is_allocated_and_freed_only_by_the_owner_types():
    found, owners = [], []
    for name, code in _sources():
        if name == OWNERS_FILE:
            for cls in OWNER_CLASSES:
                m = re.search(r"\bclass\s+%s\b" % cls, code)
                if m:
                    owners.append(cls)
                    _, e = _block(code, m.end())
                    code = code[:m.start()] + "\n" * code.count("\n", m.start(), e) + code[e:]
        for m in MEMORY_CALL.finditer(code):
            found.append(f"{name}:{code.count(chr(10), 0, m.start()) + 1}: {m.group(0)}")
    assert not found, "CUDA memory handled outside the owner types of common_host.h:\n" + "\n".join(found)
    assert owners == list(OWNER_CLASSES), f"{OWNERS_FILE} defines {owners} of {OWNER_CLASSES}"


def test_destroy_functions_release_nothing_by_hand():
    seen = []
    for name, code in _sources():
        for m in re.finditer(r"\bint\s+(dmv_\w+_destroy)\s*\(\s*\w+\s*\*\s*(\w+)\s*\)\s*\{", code):
            fn, handle = m.group(1), m.group(2)
            b, e = _block(code, m.end() - 1)
            body = code[b:e]
            seen.append(fn)
            released = RELEASE_CALL.findall(body)
            assert not released, f"{name}: {fn} releases {released} itself"
            deletes = re.findall(r"\bdelete\b\s*(\[\s*\])?\s*([^;]*);", body)
            assert deletes == [("", handle)], f"{name}: {fn} must delete only the handle {handle!r}, found {deletes}"
    assert {"dmv_ba_destroy", "dmv_ct_destroy", "dmv_ci_destroy", "dmv_ba_batch_destroy"} <= set(seen), seen

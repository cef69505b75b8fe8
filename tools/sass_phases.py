#!/usr/bin/env python
"""SASS footprint of ba_fused_kernel, attributed to the phases of csrc/ba_fused.cu (runs on a CPU machine, no GPU needed).

Each phase of the single-window launch runs once per CTA and is fetched into a cold instruction cache (DESIGN.md §6), so its size in
instructions is what it costs.  The script extracts the sm_90a cubin of ba_fused.cu from the built library (or from csrc/ba_fused.o),
disassembles one kernel instantiation with `nvdisasm -g` and attributes every instruction to the source line it came from (the innermost
inlined line).  Lines of ba_fused.cu are grouped into regions that start at the anchor strings in REGIONS; instructions from other files
(the CUDA intrinsic headers: shuffles, __ldg, ...) get their own rows.

    python tools/sass_phases.py                                    # headline kernel ba_fused_kernel<16, false, false, false>
    python tools/sass_phases.py --kernel 'ba_fused_kernel<32, false, false, false>' --json out.json
    python tools/sass_phases.py --lib other/libdmvio_b200.so --source other/csrc/ba_fused.cu
"""
import argparse
import glob
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "dm-vio_b200")

# (region, anchor): a region runs from the first line containing its anchor to the line before the next region's anchor.  Anchors that
# a source does not contain are skipped.  "after the grid barrier" = the regions flagged True.
REGIONS = [
    ("helpers (top_entry, pair_entry, geo_jac, tables)", "compile-time helpers", False),
    ("grid barrier + phase clock", "__device__ __forceinline__ unsigned ld_acquire_u32", False),
    ("peer exchange (xchg_*)", "exchange of result entries between ranks", True),
    ("decode + adjoint staging", "__device__ __forceinline__ void fused_chunk(", False),
    ("A (LPR = 1)", "phase A (LPR = 1)", False),
    ("A: loads + fused resubstitution", "phase A (LPR = 4)", False),
    ("A: projection", "// ---- centre pixel at the FEJ point (every lane)", False),
    ("A: taps + pixel math", "// ---- the lane's 2 x 4 taps", False),
    ("A: 4-lane sums, classification, outputs, JpJdF", "{  // every sample finite", False),
    ("A: 13x13 rows + butterfly + store", "// ---- the pair's 13x13 block, rows split", False),
    ("A: counters", "{  // counters: warp sums", False),
    ("B + C", "phases B and C", False),
    ("D", "// phase D item", True),
    ("D", "void fused_reduce(", True),
    ("E", "phase E: [H_sc | b_sc]", True),
    ("kernel entry + launch", "ba_fused_kernel(const __grid_constant__", False),
]
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
FILE = re.compile(r'//## File "([^"]+)", line (\d+)')


def tool(name):
    p = shutil.which(name) or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    if not os.path.exists(p):
        sys.exit(f"{name} not found (CUDA toolkit bin/ on PATH or CUDA_HOME)")
    return p


def mangle(kernel):
    """'ba_fused_kernel<16, false, false, false>' -> Itanium name of the dmv:: template instance"""
    m = re.fullmatch(r"\s*(\w+)\s*<([^>]*)>\s*", kernel)
    if not m:
        sys.exit(f"bad --kernel {kernel!r}")
    name, args = m.group(1), [a.strip() for a in m.group(2).split(",") if a.strip()]
    enc = "".join(f"Lb{int(a == 'true')}E" if a in ("true", "false") else f"Li{int(a)}E" for a in args)
    return f"_ZN3dmv{len(name)}{name}I{enc}E"


def region_lines(source):
    """source line -> region name, from the anchors"""
    text = open(source).read()
    starts = []
    for name, anchor, after in REGIONS:
        i = text.find(anchor)
        if i >= 0:
            starts.append((text.count("\n", 0, i) + 1, name, after))
    starts.sort()
    return starts


def region_of(starts, line):
    name, after = "file header", False
    for l0, n, a in starts:
        if line >= l0:
            name, after = n, a
    return name, after


def disassemble(lib, prefix):
    with tempfile.TemporaryDirectory() as d:
        subprocess.run([tool("cuobjdump"), "-xelf", "all", os.path.abspath(lib)], cwd=d, check=True, capture_output=True)
        for cub in sorted(glob.glob(os.path.join(d, "*.cubin"))):
            r = subprocess.run([tool("nvdisasm"), "-g", "-c", cub], capture_output=True, text=True)
            if r.returncode == 0 and (".text." + prefix) in r.stdout:
                return r.stdout
    sys.exit(f"no cubin of {lib} holds a kernel {prefix}*")


def attribute(sass, prefix, starts, src_name):
    """instruction counts per region of one kernel"""
    rows, cur, in_fn, total, after = {}, None, False, 0, 0
    for ln in sass.splitlines():
        if ln.split(None, 1)[:1] == [".section"]:
            in_fn = (".text." + prefix) in ln
            continue
        if not in_fn:
            continue
        m = FILE.search(ln)
        if m:
            cur = (m.group(1), int(m.group(2)))
            continue
        m = INSN.match(ln)
        if not m:
            continue
        total += 1
        if cur is None:
            key, aft = "(no line info)", False
        elif os.path.basename(cur[0]) == src_name:
            key, aft = region_of(starts, cur[1])
        elif "/include/sm_" in cur[0] or "/targets/" in cur[0]:
            key, aft = "CUDA intrinsic headers (shuffles, __ldg, ...)", False
        else:
            key, aft = os.path.basename(cur[0]), False
        rows[key] = rows.get(key, 0) + 1
        after += aft
    if total == 0:
        sys.exit(f"kernel {prefix}* not found in the disassembly")
    return rows, total, after


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=None, help="library or object holding ba_fused.cu's cubin (default: the built libdmvio_b200.so)")
    ap.add_argument("--source", default=os.path.join(PKG, "csrc", "ba_fused.cu"), help="the ba_fused.cu the library was built from")
    ap.add_argument("--kernel", default="ba_fused_kernel<16, false, false, false>")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    lib = args.lib or os.path.join(PKG, "libdmvio_b200.so")
    if not os.path.exists(lib):
        sys.exit(f"{lib} does not exist: build first (make -C dm-vio_b200)")
    prefix = mangle(args.kernel)
    sass = disassemble(lib, prefix)
    starts = region_lines(args.source)
    rows, total, after = attribute(sass, prefix, starts, os.path.basename(args.source))
    order = [n for _, n, _ in sorted(starts)]
    keys = sorted(rows, key=lambda k: (order.index(k) if k in order else len(order), k))
    print(f"{args.kernel}: {total} SASS instructions ({total * 16 / 1024:.1f} KB); after the grid barrier (D, E, peer exchange): {after}")
    print(f"{'source region':50s} {'SASS':>6s}")
    for k in keys:
        print(f"{k:50s} {rows[k]:6d}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"kernel": args.kernel, "total": total, "after_barrier": after, "regions": rows}, f, indent=1)
    return rows, total, after


if __name__ == "__main__":
    main()

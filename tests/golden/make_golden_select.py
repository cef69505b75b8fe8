"""Writes tests/golden/golden_select.npz from the reference's compiled PixelSelector, makeImages and ImmaturePoint constructor
(oracle/_ref/libselect_ref.so, built by oracle/ref_build.sh): per case of oracle/select.py the points makeNewTraces creates, numPointsTotal and
the potential after the call, and for the keyframe sequence on one persistent selector the same per keyframe.  The keyframes are regenerated
from their seeds.
    python tests/golden/make_golden_select.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import select as S  # noqa: E402


def put(out, key, r):
    for k in S.POINT_KEYS:
        out[f"{key}/{k}"] = r["points"][k]
    out[f"{key}/numPointsTotal"] = np.int32(r["numPointsTotal"])
    out[f"{key}/potential"] = np.int32(r["potential"])


out = {}
for name, (w, h, lv, kind, seed, args) in sorted(S.CASES.items()):
    a = S.case_args(args)
    R = S.Ref(w, h)
    R.potential = a.pop("potential", 3)
    put(out, name, R.new_traces(S.image(kind, w, h, seed), S.K_of(w, h), **a))
    R.close()
w, h = S.SEQ[0][:2]
R = S.Ref(w, h)
for i, (w_, h_, lv, kind, seed) in enumerate(S.SEQ):
    put(out, f"seq{i}", R.new_traces(S.image(kind, w, h, seed), S.K_of(w, h)))
R.close()
path = os.path.join(ROOT, "tests", "golden", "golden_select.npz")
np.savez_compressed(path, **out)
print(path, os.path.getsize(path), "bytes")

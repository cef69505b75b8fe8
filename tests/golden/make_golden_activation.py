"""Regenerates tests/golden/golden_activation.npz from the REFERENCE's own CoarseDistanceMap (oracle/_ref/libactivation_ref.so, built by
oracle/ref_build.sh): per case of oracle.activation.CASES, the [KRKi | Kt] tables the reference computed, the actions, toOptimize
and the final distance map.  The inputs are regenerated from the cases' seeds.  Run from the repository root:
    python tests/golden/make_golden_activation.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import activation as A  # noqa: E402

out = {}
for name, kw in A.CASES.items():
    act, opt, m, tab = A.reference(A.make_case(**kw))
    out[f"{name}/tab"], out[f"{name}/action"], out[f"{name}/opt"], out[f"{name}/map"] = tab, act, opt, m
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "golden_activation.npz"), **out)
print(f"golden_activation.npz: {len(A.CASES)} cases")

"""Writes tests/golden/golden_undistort.npz from the reference's compiled Undistort (oracle/_ref/libundistort_ref.so, built by
oracle/ref_build.sh): the reduced-size cameras of oracle/undistort.py, their remap tables, the raw frames and the reference's output for every
photometric case.
    python tests/golden/make_golden_undistort.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import undistort as U  # noqa: E402

out = {}
for cam, (text, (wOrg, hOrg)) in sorted(U.CAMERAS_SMALL.items()):
    for bpp in (1, 2):
        out[f"{cam}/raw{bpp}"] = U.raw_frame(wOrg, hOrg, bpp, 11)
    for name, bpp, nG, mode, exposure, factor, vig in U.PHOTOMETRIC:
        ref = U.Ref(text, nG, U.vignette8(wOrg, hOrg) if vig else None, mode)
        out[f"{cam}/{name}"] = ref.undistort(out[f"{cam}/raw{bpp}"], exposure, factor)
        if not ref.passthrough:
            rx, ry, _, _ = ref.tables()
            out[f"{cam}/remapX"], out[f"{cam}/remapY"] = rx.reshape(ref.h_, ref.w), ry.reshape(ref.h_, ref.w)
        ref.close()
path = os.path.join(ROOT, "tests", "golden", "golden_undistort.npz")
np.savez_compressed(path, **out)
print(path, os.path.getsize(path), "bytes")

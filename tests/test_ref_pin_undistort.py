"""Pins the CPU restatement of Undistort::undistort<T> (oracle/orc_undistort.cpp) to the reference's own compiled Undistort.cpp bit for bit,
on every camera model and photometric branch the device ingest supports; and pins both to the golden fixture made from the reference, so
the pin also holds where the reference is absent."""
import os

import numpy as np
import pytest

from oracle import undistort as U

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_undistort.npz")
needs_ref = pytest.mark.skipif(not U.ref_available(), reason="oracle/_ref/libundistort_ref.so not built (no reference sources)")


def _ref_case(cams, cam, case, seed=3):
    name, bpp, nG, mode, exposure, factor, vig = case
    text, (wOrg, hOrg) = cams[cam]
    ref = U.Ref(text, nG, U.vignette8(wOrg, hOrg) if vig else None, mode)
    raw = U.raw_frame(wOrg, hOrg, bpp, seed)
    return ref, raw


@needs_ref
@pytest.mark.parametrize("cam", sorted(U.CAMERAS))
@pytest.mark.parametrize("case", U.PHOTOMETRIC, ids=[c[0] for c in U.PHOTOMETRIC])
def test_restatement_equals_reference(cam, case):
    name, bpp, nG, mode, exposure, factor, vig = case
    ref, raw = _ref_case(U.CAMERAS, cam, case)
    try:
        assert ref.passthrough == (cam == "pinhole") and ref.valid == vig
        rx, ry, G, vi = ref.tables()
        remap = None if ref.passthrough else (rx, ry)
        # the tables the device tests build without the reference are the reference's own
        t = U.device_tables(None, mode, nG, vig, ref.wOrg, ref.hOrg, remap)
        if vig and mode != 0:
            assert np.array_equal(t[2], G[:nG]) and (mode != 2 or np.array_equal(t[4], vi))
        out_ref = ref.undistort(raw, exposure, factor)
        out_orc = U.restate(ref.w, ref.h_, raw, *t[:3], t[4], mode, exposure, factor)
        assert out_ref.shape == (ref.h_, ref.w)
        assert np.array_equal(out_ref.view(np.uint32), out_orc.view(np.uint32)), f"{cam}/{name}: max |diff| {np.abs(out_ref - out_orc).max()}"
        if not ref.passthrough:
            assert (rx >= 0).mean() > 0.5 and ((rx < 0) | ((rx < ref.wOrg - 1) & (ry >= 0) & (ry < ref.hOrg - 1))).all()
    finally:
        ref.close()


@needs_ref
def test_golden_fixture_is_the_reference():
    g = np.load(GOLDEN)
    for cam in sorted(U.CAMERAS_SMALL):
        for case in U.PHOTOMETRIC:
            ref, raw = _ref_case(U.CAMERAS_SMALL, cam, case, seed=11)
            try:
                assert np.array_equal(raw, g[f"{cam}/raw{case[1]}"])
                assert np.array_equal(ref.undistort(raw, case[4], case[5]).view(np.uint32), g[f"{cam}/{case[0]}"].view(np.uint32))
                if not ref.passthrough:
                    rx, ry, _, _ = ref.tables()
                    assert np.array_equal(rx, g[f"{cam}/remapX"].reshape(-1)) and np.array_equal(ry, g[f"{cam}/remapY"].reshape(-1))
            finally:
                ref.close()


def golden_cases():
    g = np.load(GOLDEN)
    for cam in sorted(U.CAMERAS_SMALL):
        wOrg, hOrg = U.CAMERAS_SMALL[cam][1]
        remap = (g[f"{cam}/remapX"], g[f"{cam}/remapY"]) if f"{cam}/remapX" in g else None
        h, w = g[f"{cam}/{U.PHOTOMETRIC[0][0]}"].shape
        for case in U.PHOTOMETRIC:
            name, bpp, nG, mode, exposure, factor, vig = case
            yield cam, name, w, h, g[f"{cam}/raw{bpp}"], U.device_tables(None, mode, nG, vig, wOrg, hOrg, remap), case, g[f"{cam}/{name}"]


def test_restatement_equals_golden():
    n = 0
    for cam, name, w, h, raw, t, case, want in golden_cases():
        out = U.restate(w, h, raw, *t[:3], t[4], case[3], case[4], case[5])
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), f"{cam}/{name}"
        n += 1
    assert n == len(U.CAMERAS_SMALL) * len(U.PHOTOMETRIC)

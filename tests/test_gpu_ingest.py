"""Raw-frame ingest on the device (dmv_ct_set_undistort / dmv_ct_upload_raw_image / dmv_ct_download_frame): the level-0 plane equals the CPU
restatement of Undistort::undistort<T> (oracle/orc_undistort.cpp, pinned to the reference by tests/test_ref_pin_undistort.py) and the golden
fixture bit for bit, the pyramid equals the float-upload path's, and tracking after a raw upload is bit-identical."""
import numpy as np
import pytest

from oracle import undistort as U
from test_ref_pin_undistort import golden_cases

pytestmark = pytest.mark.gpu

LEVELS = 4


def _ct(w, h, levels=LEVELS):
    import dmvio_b200.capi as capi
    if capi.lib().dmv_device_count() < 1:
        pytest.skip("needs a CUDA device")
    return capi.CT(w, h, levels, max_points=4096)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _full_cases():
    for cam in sorted(U.CAMERAS):
        (wOrg, hOrg), w, h = U.CAMERAS[cam][1], *[int(v) for v in U.CAMERAS[cam][0].split("\n")[3].split()]
        remap = None if cam == "pinhole" else U.synthetic_remap(w, h, wOrg, hOrg, seed=len(cam))
        for case in U.PHOTOMETRIC:
            yield cam, w, h, wOrg, hOrg, remap, case


@pytest.mark.parametrize("cam,w,h,wOrg,hOrg,remap,case", list(_full_cases()), ids=[f"{c[0]}-{c[6][0]}" for c in _full_cases()])
def test_level0_and_pyramid_equal_oracle(cam, w, h, wOrg, hOrg, remap, case):
    name, bpp, nG, mode, exposure, factor, vig = case
    t = U.device_tables(None, mode, nG, vig, wOrg, hOrg, remap)
    raw = U.raw_frame(wOrg, hOrg, bpp, seed=5)
    want = U.restate(w, h, raw, *t[:3], t[4], mode, exposure, factor)
    ct = _ct(w, h)
    ct.set_undistort(wOrg, hOrg, t[0], t[1], t[2], t[4], mode)
    ct.upload_raw_image(raw, exposure, factor)
    got = [ct.download_frame(l, w, h) for l in range(LEVELS)]
    assert np.array_equal(_bits(got[0][..., 0]), _bits(want)), f"max |diff| {np.abs(got[0][..., 0] - want).max()}"
    # the same frame through the float upload: every level (I, dx, dy) identical
    ct.upload_new_image(want)
    for l in range(LEVELS):
        assert np.array_equal(_bits(ct.download_frame(l, w, h)), _bits(got[l])), f"level {l}"
    # a second raw upload of the same frame on the same handle
    ct.upload_raw_image(raw, exposure, factor)
    assert np.array_equal(_bits(ct.download_frame(0, w, h)), _bits(got[0]))
    ct.close()


def test_golden_fixture():
    n = 0
    for cam, name, w, h, raw, t, case, want in golden_cases():
        ct = _ct(w, h, levels=1)
        ct.set_undistort(raw.shape[1], raw.shape[0], t[0], t[1], t[2], t[4], case[3])
        ct.upload_raw_image(raw, case[4], case[5])
        assert np.array_equal(_bits(ct.download_frame(0, w, h)[..., 0]), _bits(want)), f"{cam}/{name}"
        ct.close()
        n += 1
    assert n == len(U.CAMERAS_SMALL) * len(U.PHOTOMETRIC)


def _scene():
    import dmvio_b200.synth as synth
    T = synth.make_tracking_pair(w=160, h=120, seed=77, npts=400)
    raw = np.clip(np.rint(T["img_new"]), 0, 255).astype(np.uint8)
    return T, raw


def test_track_after_raw_upload_is_bit_identical():
    import dmvio_b200.hostmath as hm  # noqa: F401
    from oracle import orc
    T, raw = _scene()
    w, h = T["w"], T["h"]
    oc = orc.CoarseTracker(w, h, T["K"], 0)
    oc.make_coarse_depth(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"], T["pyr_ref"])
    img = U.restate(w, h, raw, None, None, None, None, 0, 1.0, 1.0)
    res = []
    for use_raw in (False, True):
        ct = _ct(w, h, oc.levels)
        for l in range(oc.levels):
            k, _ = oc.K(l)
            ct.set_K(l, *[float(x) for x in k])
            p = oc.ref_points(l)
            ct.set_ref(l, p["u"], p["v"], p["idepth"], p["color"])
        if use_raw:
            ct.set_undistort(w, h)
            ct.upload_raw_image(raw)
        else:
            ct.upload_new_image(img)
        res.append(ct.track(np.eye(3), np.zeros(3), 0.0, 0.0))
        ct.close()
    a, b = res
    for k in ("R", "t", "lastResiduals", "flow"):
        assert np.array_equal(np.asarray(a[k]).view(np.uint64), np.asarray(b[k]).view(np.uint64)), k
    assert (a["a"], a["b"], a["iterations"], a["good"]) == (b["a"], b["b"], b["iterations"], b["good"])


def test_adapter_raw_path_equals_abi():
    import dmvio_b200.hostapi as hostapi
    T, raw = _scene()
    w, h = T["w"], T["h"]
    rx, ry = U.synthetic_remap(w, h, w + 20, h + 10, seed=2)
    big = U.raw_frame(w + 20, h + 10, 1, seed=9)
    G = U.G_from_file(U.response_file_values(256))[:256]
    ct = _ct(w, h)
    ct.set_undistort(w + 20, h + 10, rx, ry, G, None, 1)
    ct.upload_raw_image(big, 1.0)
    want = [ct.download_frame(l, w, h) for l in range(LEVELS)]
    ct.close()
    ht = hostapi.CoarseTracker(w, h, T["K"], LEVELS)
    ht.set_undistort(w + 20, h + 10, rx, ry, G, None, 1)
    ht.upload_raw_image(big, 1.0)
    for l in range(LEVELS):
        assert np.array_equal(_bits(ht.download_frame(l, w, h)), _bits(want[l]))
    ht.close()


def test_invalid_inputs_are_rejected():
    import ctypes as C
    import dmvio_b200.capi as capi
    w, h = 64, 48
    ct = _ct(w, h)
    L = ct.L
    raw8 = np.zeros((h, w), np.uint8)
    assert L.dmv_ct_upload_raw_image(ct.h, raw8.ctypes.data, 1, 1.0, 1.0) == -1  # before set_undistort
    assert L.dmv_ct_set_undistort(ct.h, None) == -1
    rx, ry = U.synthetic_remap(w, h, w + 8, h + 8)
    idx = np.flatnonzero(rx >= 0)[0]
    for X, Y in ((rx, None), (np.where(np.arange(rx.size).reshape(rx.shape) == idx, np.float32(w + 7), rx), ry),
                 (rx, np.where(np.arange(ry.size).reshape(ry.shape) == idx, np.float32(-0.5), ry)),
                 (np.where(np.arange(rx.size).reshape(rx.shape) == idx, np.float32(np.nan), rx), ry)):
        with pytest.raises(capi.DmvError):
            ct.set_undistort(w + 8, h + 8, X, Y)
    with pytest.raises(capi.DmvError):  # passthrough needs the level-0 size
        ct.set_undistort(w + 8, h + 8)
    with pytest.raises(capi.DmvError):  # too short a response map
        ct.set_undistort(w + 8, h + 8, rx, ry, np.arange(100, dtype=np.float32), None, 1)
    with pytest.raises(capi.DmvError):  # mode 2 without a vignette
        ct.set_undistort(w + 8, h + 8, rx, ry, np.arange(256, dtype=np.float32), None, 2)
    ct.set_undistort(w + 8, h + 8, rx, ry, np.arange(256, dtype=np.float32), None, 1)
    with pytest.raises(capi.DmvError):  # a 256-entry map does not cover 16-bit pixels
        ct.upload_raw_image(np.zeros((h + 8, w + 8), np.uint16), 1.0)
    assert L.dmv_ct_upload_raw_image(ct.h, None, 1, 1.0, 1.0) == -1
    assert L.dmv_ct_upload_raw_image(ct.h, raw8.ctypes.data, 3, 1.0, 1.0) == -1
    out = np.zeros(w * h * 3, np.float32)
    assert L.dmv_ct_download_frame(ct.h, LEVELS, out) == -1
    assert L.dmv_ct_download_frame(C.c_void_p(), 0, out) == -1
    ct.close()

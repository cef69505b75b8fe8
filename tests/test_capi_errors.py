"""Error behaviour of the C ABI that can be checked without a GPU (include/dmvio_b200.h: "no CPU fallback"):
argument validation comes first, a missing device gives DMV_ERR_NO_DEVICE with a message, never a silent CPU path."""
import ctypes as C

import pytest

from dmvio_b200.capi import DMV_ERR_INVALID, DMV_ERR_NO_DEVICE, DMV_OK


@pytest.fixture(scope="module")
def capi():
    import dmvio_b200.capi as c
    c.lib()
    return c


def test_create_validates_arguments(capi):
    L = capi.lib()
    h = C.c_void_p()
    assert L.dmv_ba_create(None, C.byref(h)) == DMV_ERR_INVALID
    cfg = capi.BAConfig(640, 480, 99, 2000, 0, 0)  # max_frames > DMV_MAX_FRAMES
    assert L.dmv_ba_create(C.byref(cfg), C.byref(h)) == DMV_ERR_INVALID
    assert b"max_frames" in L.dmv_last_error()
    cfg = capi.BAConfig(4, 4, 7, 2000, 0, 0)       # image too small
    assert L.dmv_ba_create(C.byref(cfg), C.byref(h)) == DMV_ERR_INVALID
    ct = capi.CTConfig(640, 480, 9, 1000, 0)       # levels > DMV_MAX_PYR_LEVELS
    assert L.dmv_ct_create(C.byref(ct), C.byref(h)) == DMV_ERR_INVALID
    assert L.dmv_ba_destroy(None) == DMV_OK and L.dmv_ct_destroy(None) == DMV_OK


def test_no_device_means_error_not_cpu_fallback(capi):
    L = capi.lib()
    if L.dmv_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    h = C.c_void_p()
    cfg = capi.BAConfig(640, 480, 7, 2000, 0, 0)
    assert L.dmv_ba_create(C.byref(cfg), C.byref(h)) == DMV_ERR_NO_DEVICE
    assert b"no CPU path" in L.dmv_last_error()
    assert not h.value
    ct = capi.CTConfig(640, 480, 4, 1000, 0)
    assert L.dmv_ct_create(C.byref(ct), C.byref(h)) == DMV_ERR_NO_DEVICE
    with pytest.raises(capi.DmvError):
        capi.BA(640, 480)
    # the C++ host adapters report the same condition instead of computing on the CPU
    import numpy as np
    import dmvio_b200.hostapi as hostapi
    Lh = hostapi.lib()
    w = Lh.dmvh_window_create(640, 480, 7, 2000, 0, np.array([320.0, 320.0, 319.5, 239.5]))
    assert b"no CPU path" in Lh.dmvh_window_error(w)
    Lh.dmvh_window_destroy(w)


def test_version_string(capi):
    assert b"sm_90a" in capi.lib().dmv_version()


def test_keyframe_entry_points_validate_arguments(capi):
    """null handles / null argument blocks are rejected before anything touches CUDA"""
    L = capi.lib()
    assert L.dmv_ba_reset_oob(None) == DMV_ERR_INVALID
    import numpy as np
    assert L.dmv_ba_drop_residuals(None, 0, np.zeros(1, np.int32)) == DMV_ERR_INVALID
    assert L.dmv_ba_marginalize_points(None, None) != DMV_OK
    assert L.dmv_ba_activate_points(None, None) != DMV_OK
    assert L.dmv_last_error() != b""

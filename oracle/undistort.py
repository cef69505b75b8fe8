"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the Undistort oracles and the inputs the ingest tests share.

  restate(...)   liborc.so: the CPU restatement of Undistort::undistort<T> (orc_undistort.cpp)
  Ref            _ref/libundistort_ref.so: the REFERENCE's own Undistort (ref_undistort.cpp, built by ref_build.sh)
  the calibration / response / vignette inputs of the cases, and table builders that need no reference (synthetic_remap, G_from_file,
  vignette_inv), so that the device tests run where the reference is absent."""
import ctypes as C
import functools
import os
import tempfile

import numpy as np

from . import orc, ref

REF_LIB = "libundistort_ref.so"
vp = C.c_void_p

# (calibration file text, raw size) of the cases: EuRoC-like RadTan crop, TUM-VI-like EquiDistant, FOV, Pinhole passthrough
CAMERAS = {
    "radtan": ("RadTan 458.654 457.296 367.215 248.375 -0.28340811 0.07395907 0.00019359 1.76187114e-05\n752 480\ncrop\n640 480\n", (752, 480)),
    "equi": ("EquiDistant 190.978 190.973 254.932 256.897 0.0034823894 0.000715034 -0.0020532361 0.00020293673\n512 512\ncrop\n512 512\n", (512, 512)),
    "fov": ("FOV 0.349 0.545 0.5 0.5 0.93\n640 480\ncrop\n640 480\n", (640, 480)),
    "pinhole": ("Pinhole 0.7 0.9 0.5 0.5 0\n640 480\nnone\n640 480\n", (640, 480)),
}
# the same cameras at a reduced size (the golden fixture): intrinsics in pixels scaled by 1/16
CAMERAS_SMALL = {
    "radtan": ("RadTan 28.665875 28.581 22.9509375 15.5234375 -0.28340811 0.07395907 0.00019359 1.76187114e-05\n47 30\ncrop\n40 30\n", (47, 30)),
    "equi": ("EquiDistant 11.936125 11.9358125 15.93325 16.0560625 0.0034823894 0.000715034 -0.0020532361 0.00020293673\n32 32\ncrop\n32 32\n", (32, 32)),
    "fov": ("FOV 0.349 0.545 0.5 0.5 0.93\n40 30\ncrop\n40 30\n", (40, 30)),
    "pinhole": ("Pinhole 0.7 0.9 0.5 0.5 0\n32 24\nnone\n32 24\n", (32, 24)),
}


def response_file_values(n):
    """the (strictly increasing, float32) inverse response a response file of n entries holds"""
    x = np.arange(n, dtype=np.float64) / (n - 1)
    return (100.0 * x ** 0.8 + 3.0 * x).astype(np.float32)


def G_from_file(vals):
    """PhotometricUndistorter's G from the file values (Undistort.cpp:L107-109; mode != 0), padded to the 65536 entries it holds"""
    g = np.asarray(vals, np.float32)
    mn, mx = g[0], g[-1]
    G = np.zeros(65536, np.float32)
    G[:len(g)] = (255.0 * (g - mn).astype(np.float64) / np.float64(np.float32(mx - mn))).astype(np.float32)
    return G


def vignette8(wOrg, hOrg):
    y, x = np.mgrid[0:hOrg, 0:wOrg].astype(np.float64)
    r2 = ((x - wOrg / 2) ** 2 + (y - hOrg / 2) ** 2) / (0.6 * max(wOrg, hOrg)) ** 2
    return np.clip(255 * (1 - 0.45 * r2), 20, 255).astype(np.uint8)


def vignette_inv(v8):
    """vignetteMapInv from an 8-bit vignette image (Undistort.cpp:L154-159, L173-174)"""
    vm = v8.astype(np.float32).reshape(-1) / np.float32(v8.max())
    return (np.float32(1.0) / vm).astype(np.float32)


def synthetic_remap(w, h, wOrg, hOrg, k1=-0.25, seed=0):
    """a radially distorted remap with the reference constructor's validity rule (L921-943): x, y of a valid pixel in (0, wOrg-1) x (0, hOrg-1),
    (-1, -1) elsewhere"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    cx, cy, f = (w - 1) / 2, (h - 1) / 2, 0.8 * max(w, h)
    xn, yn = (x - cx) / f, (y - cy) / f
    d = 1 + k1 * (xn * xn + yn * yn)
    ix = (xn * d * f * 1.1 + (wOrg - 1) / 2 + rng.uniform(-0.3, 0.3)).astype(np.float32)
    iy = (yn * d * f * 1.1 + (hOrg - 1) / 2 + rng.uniform(-0.3, 0.3)).astype(np.float32)
    ok = (ix > 0) & (iy > 0) & (ix < wOrg - 1) & (iy < hOrg - 1)
    return np.where(ok, ix, -1).astype(np.float32), np.where(ok, iy, -1).astype(np.float32)


def raw_frame(wOrg, hOrg, bpp, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:hOrg, 0:wOrg].astype(np.float64)
    top = 255 if bpp == 1 else 65535
    img = top * (0.5 + 0.3 * np.sin(x / 7.0) * np.cos(y / 11.0)) + rng.normal(0, 0.05 * top, (hOrg, wOrg))
    return np.clip(img, 0, top).astype(np.uint8 if bpp == 1 else np.uint16)


@functools.cache
def orc_lib():
    L = orc.lib()
    L.orc_undistort.argtypes = [C.c_int] * 4 + [vp] * 4 + [C.c_int, vp, C.c_int, C.c_float, C.c_float, vp]
    L.orc_undistort.restype = None
    return L


def _p(a):
    return None if a is None else a.ctypes.data


def restate(w, h, raw, remapX, remapY, G, vigInv, mode, exposure, factor):
    """orc_undistort: the w*h float image Undistort::undistort<T> returns (remapX None = passthrough, G None = no calibration)"""
    raw = np.ascontiguousarray(raw)
    hOrg, wOrg = raw.shape
    c = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
    keep = [c(remapX), c(remapY), c(G), c(vigInv)]
    out = np.zeros((h, w), np.float32)
    orc_lib().orc_undistort(w, h, wOrg, hOrg, *[_p(a) for a in keep], int(mode), raw.ctypes.data, raw.itemsize, float(exposure), float(factor), out.ctypes.data)
    return out


def ref_available():
    return ref.built(REF_LIB)


@functools.cache
def ref_lib():
    L = ref.open_ref(REF_LIB)
    L.refu_create.restype = vp
    L.refu_create.argtypes = [C.c_char_p, C.c_char_p, vp, C.c_int, C.c_int, C.c_int, C.c_int]
    L.refu_destroy.argtypes = [vp]
    L.refu_info.argtypes = [vp, vp, vp]
    L.refu_tables.argtypes = [vp, vp, vp, vp, vp]
    L.refu_undistort.argtypes = [vp, vp, C.c_int, C.c_float, C.c_float, C.c_int, vp]
    return L


class Ref:
    """the reference's Undistort::getUndistorterForFile on a calibration text, nG response entries and an 8-bit vignette (None: none)"""

    def __init__(self, calib_text, nG, vignette, mode):
        L = ref_lib()
        self.mode = mode
        with tempfile.TemporaryDirectory() as d:
            cf, gf = os.path.join(d, "camera.txt"), os.path.join(d, "pcalib.txt")
            open(cf, "w").write(calib_text)
            open(gf, "w").write(" ".join(repr(float(v)) for v in response_file_values(nG)) + "\n")
            self._v = None if vignette is None else np.ascontiguousarray(vignette, np.uint8)
            self.h = L.refu_create(cf.encode(), gf.encode(), _p(self._v), 1, 0 if self._v is None else self._v.shape[1],
                                   0 if self._v is None else self._v.shape[0], int(mode))
        assert self.h, "the reference rejected the calibration"
        info, vg = np.zeros(4, np.int32), np.zeros(2, np.int32)
        self.passthrough = bool(L.refu_info(self.h, info.ctypes.data, vg.ctypes.data))
        self.w, self.h_, self.wOrg, self.hOrg = (int(v) for v in info)
        self.valid, self.GDepth = bool(vg[0]), int(vg[1])

    def tables(self):
        rx, ry = np.zeros(self.w * self.h_, np.float32), np.zeros(self.w * self.h_, np.float32)
        G, vi = np.zeros(65536, np.float32), np.zeros(self.wOrg * self.hOrg, np.float32)
        ref_lib().refu_tables(self.h, rx.ctypes.data, ry.ctypes.data, G.ctypes.data, vi.ctypes.data)
        return rx, ry, G, vi

    def undistort(self, raw, exposure, factor):
        raw = np.ascontiguousarray(raw)
        out = np.zeros((self.h_, self.w), np.float32)
        ref_lib().refu_undistort(self.h, raw.ctypes.data, raw.itemsize, float(exposure), float(factor), self.mode, out.ctypes.data)
        return out

    def close(self):
        if self.h:
            ref_lib().refu_destroy(self.h)
            self.h = None


# photometric cases: (name, bytes per pixel, response entries, photometric mode, exposure, factor, vignette given)
PHOTOMETRIC = [
    ("u8_mode0", 1, 256, 0, 1.0, 1.0, True),
    ("u8_mode1", 1, 256, 1, 1.0, 1.0, True),
    ("u8_mode2", 1, 256, 2, 1.0, 1.0, True),
    ("u8_mode2_exposure0", 1, 256, 2, 0.0, 1.0, True),
    ("u8_no_vignette", 1, 256, 2, 1.0, 1.0, False),
    ("u16_factor", 2, 256, 0, 1.0, 1.0 / 256, True),
    ("u16_mode1_G65536", 2, 65536, 1, 1.0, 1.0 / 256, True),
    ("u16_mode2_G65536", 2, 65536, 2, 1.0, 1.0 / 256, True),
]


def device_tables(ref_or_none, mode, nG, vignette_given, wOrg, hOrg, remap):
    """the dmv_undistort_config inputs of a case: (remapX, remapY, G, nG, vignetteInv); remap = (rx, ry) or None (passthrough).  The response map
    and vignetteMapInv are the ones the reference builds (a valid calibration needs the vignette; mode 0 never reads them)."""
    if not vignette_given:
        return (*remap, None, 0, None) if remap else (None, None, None, 0, None)
    G = G_from_file(response_file_values(nG))[:nG]
    vi = vignette_inv(vignette8(wOrg, hOrg))
    rx, ry = remap if remap else (None, None)
    return rx, ry, G, nG, (vi if mode == 2 else None)

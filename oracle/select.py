"""TEST INFRASTRUCTURE ONLY — bindings and cases of the pixel-selection oracles (dmv_ct_make_new_traces).

  restate(...)   liborc_select.so: the CPU restatement of PixelSelector::makeMaps and makeNewTraces' loop (orc_select.cpp, built by select.mk);
                 the ImmaturePoint constructor is orc.ip_init
  Ref            _ref/libselect_ref.so: the REFERENCE's own PixelSelector / makeImages / ImmaturePoint (ref_select.cpp, ref_build_select.sh)
  CASES          seeded keyframes and arguments shared by the CPU pin, the golden fixture and the device tests"""
import ctypes as C
import os

import numpy as np

from . import orc

_HERE = os.path.dirname(os.path.abspath(__file__))
ORC_PATH = os.path.join(_HERE, "liborc_select.so")
REF_PATH = os.path.join(_HERE, "_ref", "libselect_ref.so")
vp = C.c_void_p
f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
_ORC = None
_REF = None

DEFAULTS = dict(minGradHistCut=0.5, minGradHistAdd=7.0, gradDownweightPerLevel=0.75, selectDirectionDistribution=1, gammaWeightsPixelSelect=1)
POINT_KEYS = ("u", "v", "type", "color", "weights", "gradH", "energyTH")


def orc_lib():
    global _ORC
    if _ORC is None:
        L = C.CDLL(ORC_PATH)
        L.orc_sel_random_pattern.argtypes = [C.c_uint, C.c_int, u8p]
        L.orc_sel_make_maps.restype = C.c_int
        L.orc_sel_make_maps.argtypes = [C.c_int, C.c_int, f32p, f32p, f32p, f32p, f32p, i32p, C.c_float, C.c_int, C.c_float, C.POINTER(C.c_int), f32p,
                                        C.POINTER(C.c_longlong), C.POINTER(C.c_float)]
        L.orc_sel_trace_pixels.restype = C.c_int
        L.orc_sel_trace_pixels.argtypes = [C.c_int, C.c_int, f32p, i32p, i32p, f32p]
        _ORC = L
    return _ORC


def ref_available():
    return os.path.exists(REF_PATH)


def random_pattern(n, seed=3141592):
    out = np.zeros(n, np.uint8)
    orc_lib().orc_sel_random_pattern(seed, n, out)
    return out


def identity_B():
    return np.arange(256, dtype=np.float32)


def gamma_B():
    """a non-identity CalibHessian::B as FullSystem::setGammaFunction leaves it, for an inverse response Binv[i] = 255 (i/255)^0.7"""
    Binv = (255.0 * (np.arange(256) / 255.0) ** 0.7).astype(np.float32)
    B = np.zeros(256, np.float32)
    for i in range(1, 255):
        for s in range(1, 255):
            if Binv[s] <= i and Binv[s + 1] >= i:
                B[i] = np.float32(s) + (np.float32(i) - Binv[s]) / (Binv[s + 1] - Binv[s])
                break
    B[0], B[255] = 0, 255
    return B


def _settings(s):
    s = dict(DEFAULTS, **(s or {}))
    return (np.array([s["minGradHistCut"], s["minGradHistAdd"], s["gradDownweightPerLevel"]], np.float32),
            np.array([s["selectDirectionDistribution"], s["gammaWeightsPixelSelect"]], np.int32))


def restate(pyr, B=None, settings=None, density=1500.0, recursionsLeft=1, thFactor=1.0, potential=3):
    """makeMaps + makeNewTraces on levels 0-2 of pyr ((h_l, w_l, 3) [I, dx, dy] arrays) -> dict(map, numPointsTotal, potential, n_mixed, quotia, points)"""
    L = orc_lib()
    h, w = pyr[0].shape[:2]
    c = lambda a: np.ascontiguousarray(a, np.float32).reshape(-1)
    sf, si = _settings(settings)
    pot = C.c_int(int(potential))
    mixed = C.c_longlong(0)
    quotia = C.c_float(0)
    m = np.zeros(w * h, np.float32)
    npt = L.orc_sel_make_maps(w, h, c(pyr[0]), c(pyr[1]), c(pyr[2]), c(identity_B() if B is None else B), sf, si, float(density), int(recursionsLeft),
                              float(thFactor), C.byref(pot), m, C.byref(mixed), C.byref(quotia))
    u = np.zeros(w * h, np.int32); v = np.zeros(w * h, np.int32); t = np.zeros(w * h, np.float32)
    n = L.orc_sel_trace_pixels(w, h, m, u, v, t)
    P = orc.ip_init(pyr[0], w, h, u[:n], v[:n])
    ok = P["ok"].astype(bool)
    pts = dict(u=u[:n][ok], v=v[:n][ok], type=t[:n][ok], color=P["color"][ok], weights=P["weights"][ok], gradH=P["gradH"][ok], energyTH=P["energyTH"][ok])
    return dict(map=m.reshape(h, w), numPointsTotal=int(npt), potential=pot.value, n_mixed=int(mixed.value), quotia=quotia.value, points=pts)


class Ref:
    """the reference's PixelSelector (persistent: currentPotential carries over between calls), keyframes built by its makeImages"""

    def __init__(self, w, h):
        global _REF
        if _REF is None:
            L = C.CDLL(REF_PATH)
            L.ref_sel_settings.argtypes = [C.c_float, C.c_float, C.c_float, C.c_int, C.c_int]
            L.ref_sel_frame_create.restype = vp
            L.ref_sel_frame_create.argtypes = [C.c_int, C.c_int, f64p, f32p, vp]
            L.ref_sel_frame_destroy.argtypes = [vp]
            L.ref_sel_frame_dI.argtypes = [vp, C.c_int, f32p]
            L.ref_sel_create.restype = vp
            L.ref_sel_create.argtypes = [C.c_int, C.c_int]
            L.ref_sel_destroy.argtypes = [vp]
            L.ref_sel_get_potential.argtypes = [vp]
            L.ref_sel_set_potential.argtypes = [vp, C.c_int]
            L.ref_sel_make_maps.restype = C.c_int
            L.ref_sel_make_maps.argtypes = [vp, vp, f32p, C.c_float, C.c_int, C.c_float]
            L.ref_sel_new_traces.restype = C.c_int
            L.ref_sel_new_traces.argtypes = [vp, f32p, i32p, i32p, f32p, f32p, f32p, f32p, f32p]
            _REF = L
        self.L = _REF
        self.w, self.h = w, h
        self.ps = self.L.ref_sel_create(w, h)
        self.frames = []   # kept alive until close(): makeMaps caches its histogram by FrameHessian address

    @property
    def potential(self):
        return self.L.ref_sel_get_potential(self.ps)

    @potential.setter
    def potential(self, p):
        self.L.ref_sel_set_potential(self.ps, int(p))

    def new_traces(self, img, K, B=None, settings=None, density=1500.0, recursionsLeft=1, thFactor=1.0):
        """makeImages of img, then makeNewTraces with this selector -> the same dict as restate() (without n_mixed) plus pyr (levels 0-2)"""
        s = dict(DEFAULTS, **(settings or {}))
        self.L.ref_sel_settings(s["minGradHistCut"], s["minGradHistAdd"], s["gradDownweightPerLevel"], s["selectDirectionDistribution"], s["gammaWeightsPixelSelect"])
        Bp = None if B is None else np.ascontiguousarray(B, np.float32)
        fr = self.L.ref_sel_frame_create(self.w, self.h, np.ascontiguousarray(K, np.float64), np.ascontiguousarray(img, np.float32).reshape(-1),
                                         None if Bp is None else Bp.ctypes.data)
        self.frames.append(fr)
        w, h = self.w, self.h
        m = np.zeros(w * h, np.float32)
        npt = self.L.ref_sel_make_maps(self.ps, fr, m, float(density), int(recursionsLeft), float(thFactor))
        pyr = []
        for l in range(3):
            a = np.zeros((h >> l) * (w >> l) * 3, np.float32)
            self.L.ref_sel_frame_dI(fr, l, a)
            pyr.append(a.reshape(h >> l, w >> l, 3))
        N = w * h
        u = np.zeros(N, np.int32); v = np.zeros(N, np.int32); t = np.zeros(N, np.float32)
        col = np.zeros((N, 8), np.float32); wt = np.zeros((N, 8), np.float32); gH = np.zeros((N, 4), np.float32); e = np.zeros(N, np.float32)
        n = self.L.ref_sel_new_traces(fr, m, u, v, t, col, wt, gH, e)
        pts = dict(u=u[:n], v=v[:n], type=t[:n], color=col[:n], weights=wt[:n], gradH=gH[:n], energyTH=e[:n])
        return dict(map=m.reshape(h, w), numPointsTotal=int(npt), potential=self.potential, points=pts, pyr=pyr)

    def close(self):
        for fr in self.frames:
            self.L.ref_sel_frame_destroy(fr)
        self.frames = []
        if self.ps:
            self.L.ref_sel_destroy(self.ps)
            self.ps = None


# ---- seeded keyframes
def K_of(w, h):
    return np.array([0.8 * w, 0.8 * w, w / 2 - 0.5, h / 2 - 0.5], np.float64)


def image(kind, w, h, seed):
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    if kind == "tex":        # 8-bit quantised smooth texture
        a = gaussian_filter(rng.normal(size=(h, w)), 2.5)
        a = 128 + 90 * a / np.abs(a).max()
    elif kind == "low":      # weak texture: few candidates, makeMaps lowers the potential
        a = gaussian_filter(rng.normal(size=(h, w)), 6.0)
        a = 128 + 12 * a / np.abs(a).max()
    elif kind == "high":     # strong fine texture: many candidates, makeMaps raises the potential
        a = gaussian_filter(rng.normal(size=(h, w)), 0.7)
        a = 128 + 120 * a / np.abs(a).max()
    elif kind == "flat":
        a = np.full((h, w), 128.0)
    elif kind == "stripe":   # horizontal stripes: dx == 0 everywhere, every textured pot-block is mixed
        a = 128 + 100 * np.sin(y * (0.9 + 0.3 * rng.random())) * (0.2 + 0.8 * rng.random((h, 1)))
        a = np.broadcast_to(a, (h, w))
    elif kind == "stair":    # diagonal staircase: dx == dy on the step edges
        a = 40.0 * (((x + y) // 7) % 5) + 30
    else:
        raise ValueError(kind)
    return np.clip(np.round(a), 0, 255).astype(np.float32)


# name -> (w, h, levels, image kind, seed, args of makeNewTraces); "seq" is a sequence of keyframes on one persistent selector
CASES = {
    "tex640_l5": (640, 480, 5, "tex", 1, {}),
    "tex512_l4": (512, 512, 4, "tex", 2, {}),
    "tex640_l4_rec0": (640, 480, 4, "tex", 3, dict(recursionsLeft=0)),
    "low640_l5": (640, 480, 5, "low", 4, {}),
    "low512_l5_pot1": (512, 512, 5, "low", 5, dict(potential=1)),
    "high640_l4": (640, 480, 4, "high", 6, {}),
    "high512_l4_rec0": (512, 512, 4, "high", 7, dict(recursionsLeft=0)),
    "flat640_l4": (640, 480, 4, "flat", 8, {}),
    "tex640_l5_th2": (640, 480, 5, "tex", 9, dict(thFactor=2.0)),
    "tex512_l5_nodir": (512, 512, 5, "tex", 10, dict(settings=dict(selectDirectionDistribution=0))),
    "tex640_l4_gamma": (640, 480, 4, "tex", 11, dict(B="gamma")),
    "stripe640_l4": (640, 480, 4, "stripe", 12, {}),
    "stair512_l5": (512, 512, 5, "stair", 13, {}),
}
SEQ = [(640, 480, 5, kind, 20 + i) for i, kind in enumerate(("tex", "high", "tex", "low", "stripe"))]


def case_args(args):
    a = dict(args)
    if a.get("B") == "gamma":
        a["B"] = gamma_B()
    return a

"""TEST INFRASTRUCTURE ONLY — ctypes binding of the CPU oracle (oracle/liborc.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")


def build(native=False):
    target = "native" if native else "all"
    subprocess.check_call(["make", "-s", "-C", _HERE, target])


def lib(native=False):
    global _LIB
    name = "liborc_native.so" if native else "liborc.so"
    path = os.path.join(_HERE, name)
    if native:
        if not os.path.exists(path):
            build(native=True)
        return _declare(C.CDLL(path))
    if _LIB is None:
        if not os.path.exists(path):
            build()
        _LIB = _declare(C.CDLL(path))
    return _LIB


def _declare(L):
    vp = C.c_void_p
    L.orc_win_create.restype = vp
    L.orc_win_create.argtypes = [C.c_int, C.c_int, C.c_int, f64p, C.c_int]
    L.orc_win_destroy.argtypes = [vp]
    L.orc_win_set_setting.argtypes = [vp, C.c_char_p, C.c_double]
    L.orc_win_set_frame.argtypes = [vp, C.c_int, f64p, f64p, f64p, f64p, C.c_float, C.c_float, C.c_int, f32p]
    L.orc_win_set_points.argtypes = [vp, C.c_int, i32p, f32p, f32p, f32p, f32p, f32p, f32p, u8p]
    L.orc_win_set_residuals.argtypes = [vp, C.c_int, i32p, i32p, vp, vp, vp]
    L.orc_win_set_marg_prior.argtypes = [vp, vp, vp]
    L.orc_win_prepare.argtypes = [vp]
    for n in ("orc_win_nres", "orc_win_npts", "orc_win_nf"):
        getattr(L, n).argtypes = [vp]
    L.orc_win_get_precalc.argtypes = [vp, f32p]
    L.orc_win_get_RT.argtypes = [vp, f32p]
    L.orc_win_get_adjoints.argtypes = [vp, f64p, f64p]
    L.orc_win_get_adHTdeltaF.argtypes = [vp, f32p]
    L.orc_win_get_frame_tables.argtypes = [vp, f64p, f64p, f64p, f32p]
    L.orc_win_get_calib.argtypes = [vp, f32p, f32p, f64p]
    L.orc_win_linearize_all.restype = C.c_double
    L.orc_win_linearize_all.argtypes = [vp, C.c_int, C.c_int]
    L.orc_win_apply_res.argtypes = [vp]
    L.orc_win_override_new_states.restype = C.c_double
    L.orc_win_override_new_states.argtypes = [vp, i32p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.orc_win_get_res_outputs.argtypes = [vp, i32p, f32p, f32p, f32p, vp, i32p, u8p, f32p]
    L.orc_win_accumulate.argtypes = [vp, C.c_int, f64p, f64p, f64p, f64p, f64p, f64p, C.POINTER(C.c_int)]
    L.orc_win_get_nullspaces.argtypes = [vp, f64p]
    L.orc_win_orthogonalize.argtypes = [vp, f64p]
    L.orc_win_marginalize_frame.argtypes = [vp, C.c_int, f64p, f64p, f64p, f64p]
    L.orc_win_finish_optimize.restype = C.c_double
    L.orc_win_finish_optimize.argtypes = [vp, i32p, C.c_int, C.POINTER(C.c_int)]
    L.orc_win_get_point_stats.argtypes = [vp, f32p, i32p]
    L.orc_win_marginalize.argtypes = [vp, C.c_int, i32p, C.c_int, f64p, f64p, f64p, f64p, f64p, f64p, C.POINTER(C.c_int), i32p, f32p, u8p]
    L.orc_win_get_point_outputs.argtypes = [vp, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p]
    L.orc_win_solve.argtypes = [vp, C.c_int, C.c_double, C.c_int, f64p, f64p, f64p]
    L.orc_win_resubstitute.argtypes = [vp, f64p]
    L.orc_win_calc_LEnergy.restype = C.c_double
    L.orc_win_calc_LEnergy.argtypes = [vp]
    L.orc_win_calc_MEnergy.restype = C.c_double
    L.orc_win_calc_MEnergy.argtypes = [vp]
    L.orc_win_optimize.argtypes = [vp, C.c_int, C.c_int, f64p, C.c_int]
    L.orc_win_get_frame_states.argtypes = [vp, f64p]
    L.orc_win_gn_iteration.restype = C.c_double
    L.orc_win_gn_iteration.argtypes = [vp, C.c_double, C.c_int, C.c_int]
    L.orc_win_hot_iteration.restype = C.c_double
    L.orc_win_hot_iteration.argtypes = [vp, f64p, C.c_int]
    L.orc_win_eval_raw_double.argtypes = [vp, C.c_int, f64p, f64p, C.c_double, f64p, f64p]
    L.orc_pyr_levels.argtypes = [C.c_int, C.c_int, C.c_int]
    L.orc_make_images.restype = C.c_int64
    L.orc_make_images.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, f32p, f32p, vp]
    L.orc_init_point.argtypes = [f32p, C.c_int, C.c_float, C.c_float, f32p, f32p]
    L.orc_ct_create.restype = vp
    L.orc_ct_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float]
    L.orc_ct_destroy.argtypes = [vp]
    L.orc_ct_set_setting.argtypes = [vp, C.c_char_p, C.c_double]
    L.orc_ct_set_ref_points.argtypes = [vp, C.c_int, C.c_int, f32p, f32p, f32p, f32p]
    L.orc_ct_make_coarse_depth.argtypes = [vp, C.c_int, f32p, f32p, f32p, f32p, f32p]
    L.orc_ct_get_ref_points.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    L.orc_ct_set_new_frame.argtypes = [vp, f32p, C.c_float, C.c_float, C.c_double, C.c_double]
    L.orc_ct_get_K.argtypes = [vp, C.c_int, f32p, i32p]
    L.orc_ct_calc_res.argtypes = [vp, C.c_int, f64p, f64p, C.c_double, C.c_double, C.c_float, f64p]
    L.orc_ct_get_warped.argtypes = [vp, vp]
    L.orc_ct_calc_gs.argtypes = [vp, C.c_int, C.c_double, C.c_double, C.c_int, f64p, f64p]
    L.orc_ct_track.argtypes = [vp, f64p, f64p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, f64p, C.c_int, f64p, f64p, C.POINTER(C.c_int)]
    L.orc_ip_activate.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, f32p, f32p, f32p, f32p, i32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, C.c_int,
                                  C.c_float, i32p, f32p, i32p]
    L.orc_ip_init.argtypes = [C.c_int, f32p, C.c_int, C.c_int, i32p, i32p, f32p, f32p, f32p, f32p, u8p]
    L.orc_ip_trace.argtypes = [C.c_int, f32p, C.c_int, C.c_int, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, i32p, f32p, f32p]
    L.orc_ip_trace_diag.argtypes = L.orc_ip_trace.argtypes + [i32p]
    L.orc_se3_exp.argtypes = [f64p, f64p, f64p]
    L.orc_se3_log.argtypes = [f64p, f64p, f64p]
    return L


RAWJ_FLOATS = 74
# offsets (in floats) into the 74-float RawJ dump
J_RESF, J_JPDXI, J_JPDC, J_JPDD, J_JIDX, J_JABF, J_JIDX2, J_JABJIDX, J_JAB2 = 0, 8, 20, 28, 30, 46, 62, 66, 70


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Window:
    """A sliding window loaded into the oracle from a dmvio_b200.synth.make_window() dict."""

    def __init__(self, W, nthreads=1, native=False, settings=None, _lib=None):
        self.L = _lib if _lib is not None else lib(native)
        self.W = W
        self.nf, self.npts, self.nres = W["nf"], len(W["host"]), len(W["res_point"])
        self.N = 8 * self.nf + 4
        self._keep = []
        self.h = self.L.orc_win_create(W["w"], W["h"], self.nf, np.ascontiguousarray(W["K"], np.float64), nthreads)
        for k, v in (settings or {}).items():
            self.L.orc_win_set_setting(self.h, k.encode(), float(v))
        for k in range(self.nf):
            dI = np.ascontiguousarray(W["dI"][k], np.float32)
            self._keep.append(dI)
            self.L.orc_win_set_frame(self.h, k, np.ascontiguousarray(W["R_eval"][k].reshape(-1)), np.ascontiguousarray(W["t_eval"][k]),
                                     np.ascontiguousarray(W["state"][k]), np.ascontiguousarray(W["state_zero"][k]),
                                     float(W["exposure"][k]), float(W["frameEnergyTH"][k]), int(W["frameID"][k]), dI)
        c = lambda a, t: np.ascontiguousarray(a, t)
        self.L.orc_win_set_points(self.h, self.npts, c(W["host"], np.int32), c(W["u"], np.float32), c(W["v"], np.float32),
                                  c(W["idepth"], np.float32), c(W["idepth_zero"], np.float32), c(W["color"], np.float32),
                                  c(W["weights"], np.float32), c(W["hasDepthPrior"], np.uint8))
        ss = W.get("res_state")
        se = W.get("res_energy")
        self.L.orc_win_set_residuals(self.h, self.nres, c(W["res_point"], np.int32), c(W["res_target"], np.int32),
                                     _ptr(None if ss is None else c(ss, np.int32)), _ptr(None if se is None else c(se, np.float32)), None)
        HM, bM = W.get("HM"), W.get("bM")
        if HM is not None or bM is not None or _lib is None:
            self.L.orc_win_set_marg_prior(self.h, _ptr(None if HM is None else c(HM, np.float64)), _ptr(None if bM is None else c(bM, np.float64)))
        self.L.orc_win_prepare(self.h)

    def __del__(self):
        try:
            self.L.orc_win_destroy(self.h)
        except Exception:
            pass

    # ---- tables
    def precalc(self):
        out = np.zeros((self.nf * self.nf, 32), np.float32)
        self.L.orc_win_get_precalc(self.h, out)
        return out

    def RT(self):
        """PRE_RTll | PRE_tTll per pair [h*nf+t] (current relative poses), nf*nf x 12 float32"""
        out = np.zeros((self.nf * self.nf, 12), np.float32)
        self.L.orc_win_get_RT(self.h, out)
        return out

    def adjoints(self):
        a = np.zeros((self.nf * self.nf, 8, 8)); b = np.zeros((self.nf * self.nf, 8, 8))
        self.L.orc_win_get_adjoints(self.h, a, b)
        return a, b

    def adHTdeltaF(self):
        out = np.zeros((self.nf * self.nf, 8), np.float32)
        self.L.orc_win_get_adHTdeltaF(self.h, out)
        return out

    def frame_tables(self):
        p = np.zeros((self.nf, 8)); dp = np.zeros((self.nf, 8)); d = np.zeros((self.nf, 8)); th = np.zeros(self.nf, np.float32)
        self.L.orc_win_get_frame_tables(self.h, p, dp, d, th)
        return dict(prior=p, delta_prior=dp, delta=d, frameEnergyTH=th)

    def calib(self):
        k8 = np.zeros(8, np.float32); cd = np.zeros(4, np.float32); cp = np.zeros(4)
        self.L.orc_win_get_calib(self.h, k8, cd, cp)
        return dict(k8=k8, cDeltaF=cd, cPrior=cp)

    # ---- hot path
    def linearize_all(self, fix=False, update_th=True):
        return self.L.orc_win_linearize_all(self.h, int(fix), int(update_th))

    def apply_res(self):
        self.L.orc_win_apply_res(self.h)

    def override_new_states(self, newState):
        """impose another implementation's classification on the tentative linearisation (threshold ties); returns
        (energy sum under that classification, #changed, #unfixable)"""
        ch, bad = C.c_int(0), C.c_int(0)
        E = self.L.orc_win_override_new_states(self.h, np.ascontiguousarray(newState, np.int32), C.byref(ch), C.byref(bad))
        return E, ch.value, bad.value

    def res_outputs(self, want_J=True):
        n = self.nres
        o = dict(newState=np.zeros(n, np.int32), newEnergy=np.zeros(n, np.float32), newEnergyWithOutlier=np.zeros(n, np.float32),
                 centerProjectedTo=np.zeros((n, 3), np.float32), J=np.zeros((n, RAWJ_FLOATS), np.float32) if want_J else None,
                 state=np.zeros(n, np.int32), isActive=np.zeros(n, np.uint8), JpJdF=np.zeros((n, 8), np.float32))
        self.L.orc_win_get_res_outputs(self.h, o["newState"], o["newEnergy"], o["newEnergyWithOutlier"], o["centerProjectedTo"],
                                       _ptr(o["J"]), o["state"], o["isActive"], o["JpJdF"])
        return o

    def accumulate(self, precision=1):
        N = self.N
        o = dict(HA=np.zeros((N, N)), bA=np.zeros(N), HL=np.zeros((N, N)), bL=np.zeros(N), Hsc=np.zeros((N, N)), bsc=np.zeros(N))
        n = C.c_int(0)
        self.L.orc_win_accumulate(self.h, precision, o["HA"], o["bA"], o["HL"], o["bL"], o["Hsc"], o["bsc"], C.byref(n))
        o["resInA"] = n.value
        return o

    def marginalize(self, pts, precision=1):
        """flagPointsForRemoval's linearize/applyRes/fixLinearizationF loop + marginalizePointsF on the listed points
        (FullSystem.cpp:L826-838, EnergyFunctional.cpp:L678-742).  H = M - Msc, b = Mb - Mbsc (before margWeightFac); HM, bM after the update."""
        N, nres = self.N, self.L.orc_win_nres(self.h)
        pts = np.ascontiguousarray(pts, np.int32)
        o = dict(M=np.zeros((N, N)), Mb=np.zeros(N), Msc=np.zeros((N, N)), Mbsc=np.zeros(N), HM=np.zeros((N, N)), bM=np.zeros(N),
                 ngood=np.zeros(len(pts), np.int32), rtz=np.zeros((nres, 8), np.float32), isLinearized=np.zeros(nres, np.uint8))
        n = C.c_int(0)
        self.L.orc_win_marginalize(self.h, len(pts), pts, precision, o["M"], o["Mb"], o["Msc"], o["Mbsc"], o["HM"], o["bM"], C.byref(n),
                                   o["ngood"], o["rtz"], o["isLinearized"])
        o["resInM"] = n.value
        o["H"], o["b"] = o["M"] - o["Msc"], o["Mb"] - o["Mbsc"]
        return o

    def point_outputs(self):
        n = self.npts
        o = dict(Hdd=np.zeros(n, np.float32), bd=np.zeros(n, np.float32), Hcd=np.zeros((n, 4), np.float32), HdiF=np.zeros(n, np.float32),
                 bdSumF=np.zeros(n, np.float32), step=np.zeros(n, np.float32), idepth=np.zeros(n, np.float32), maxRelBaseline=np.zeros(n, np.float32))
        self.L.orc_win_get_point_outputs(self.h, o["Hdd"], o["bd"], o["Hcd"], o["HdiF"], o["bdSumF"], o["step"], o["idepth"], o["maxRelBaseline"])
        return o

    def solve(self, iteration=0, lam=1e-5, precision=1):
        N = self.N
        x = np.zeros(N); HF = np.zeros((N, N)); bF = np.zeros(N)
        self.L.orc_win_solve(self.h, iteration, lam, precision, x, HF, bF)
        return x, HF, bF

    def resubstitute(self, x):
        self.L.orc_win_resubstitute(self.h, np.ascontiguousarray(x, np.float64))

    def optimize(self, its=6, precision=1):
        log = np.zeros(64)
        n = self.L.orc_win_optimize(self.h, its, precision, log, 64)
        return n, log[log >= 0]

    def nullspaces(self):
        """FullSystem::getNullspaces: (7, N) = 6 pose + 1 scale gauge directions at the frames' evaluation points"""
        out = np.zeros((7, self.N))
        self.L.orc_win_get_nullspaces(self.h, out.reshape(-1))
        return out

    def orthogonalize(self, x):
        """EnergyFunctional::orthogonalize(&x, 0)"""
        v = np.ascontiguousarray(x, np.float64).copy()
        self.L.orc_win_orthogonalize(self.h, v)
        return v

    def marginalize_frame(self, idx, HM, bM):
        """EnergyFunctional::marginalizeFrame (EnergyFunctional.cpp:L522-675) of frame idx on the prior (HM, bM); the frame leaves the window"""
        odim = 8 * self.nf + 4
        HM = np.ascontiguousarray(HM, np.float64).reshape(odim * odim); bM = np.ascontiguousarray(bM, np.float64)
        Ho = np.zeros((odim - 8) * (odim - 8)); bo = np.zeros(odim - 8)
        self.L.orc_win_marginalize_frame(self.h, int(idx), HM, bM, Ho, bo)
        self.nf -= 1; self.N -= 8
        return Ho.reshape(odim - 8, odim - 8), bo

    def finish_optimize(self):
        """tail of FullSystem::optimize (FullSystemOptimize.cpp:L591-609): setEvalPT of the newest frame, adjoints, precalc, linearizeAll(true).
        Returns (energy, removed residual indices)."""
        rem = np.zeros(self.L.orc_win_nres(self.h), np.int32)
        n = C.c_int(0)
        E = self.L.orc_win_finish_optimize(self.h, rem, len(rem), C.byref(n))
        return E, rem[:n.value].copy()

    def point_stats(self):
        mrb = np.zeros(self.npts, np.float32); ng = np.zeros(self.npts, np.int32)
        self.L.orc_win_get_point_stats(self.h, mrb, ng)
        return dict(maxRelBaseline=mrb, numGoodResiduals=ng)

    def frame_states(self):
        s = np.zeros((self.nf, 10))
        self.L.orc_win_get_frame_states(self.h, s)
        return s

    def gn_iteration(self, lam=1e-5, precision=0, do_step=True):
        return self.L.orc_win_gn_iteration(self.h, lam, precision, int(do_step))

    def hot_iteration(self, x, precision=0):
        return self.L.orc_win_hot_iteration(self.h, np.ascontiguousarray(x, np.float64), precision)

    def eval_raw(self, ri, dsh=None, dst=None, didepth=0.0, dcalib=None):
        z8 = np.zeros(8)
        r = np.zeros(8)
        ok = self.L.orc_win_eval_raw_double(self.h, ri, z8 if dsh is None else np.ascontiguousarray(dsh, np.float64),
                                            z8 if dst is None else np.ascontiguousarray(dst, np.float64), float(didepth),
                                            np.zeros(4) if dcalib is None else np.ascontiguousarray(dcalib, np.float64), r)
        return (r if ok else None)


def make_images(img, K, levels=0):
    L = lib()
    h, w = img.shape
    lv = L.orc_pyr_levels(w, h, levels)
    tot = sum((w >> l) * (h >> l) * 3 for l in range(lv))
    out = np.zeros(tot, np.float32)
    n = L.orc_make_images(w, h, levels, float(K[0]), float(K[1]), float(K[2]), float(K[3]), np.ascontiguousarray(img, np.float32).reshape(-1), out, None)
    assert n == tot
    res, off = [], 0
    for l in range(lv):
        sz = (w >> l) * (h >> l) * 3
        res.append(out[off:off + sz].reshape(h >> l, w >> l, 3))
        off += sz
    return res


class CoarseTracker:
    def __init__(self, w, h, K, levels=0, settings=None):
        self.L = lib()
        self.levels = self.L.orc_pyr_levels(w, h, levels)
        self.w, self.h = w, h
        self.hd = self.L.orc_ct_create(w, h, levels, float(K[0]), float(K[1]), float(K[2]), float(K[3]))
        for k, v in (settings or {}).items():
            self.L.orc_ct_set_setting(self.hd, k.encode(), float(v))
        self._keep = []

    def __del__(self):
        try:
            self.L.orc_ct_destroy(self.hd)
        except Exception:
            pass

    @staticmethod
    def _concat(pyr):
        return np.ascontiguousarray(np.concatenate([p.reshape(-1) for p in pyr]), np.float32)

    def make_coarse_depth(self, Ku, Kv, nid, HdiF, pyr_ref):
        ref = self._concat(pyr_ref)
        c = lambda a: np.ascontiguousarray(a, np.float32)
        return self.L.orc_ct_make_coarse_depth(self.hd, len(Ku), c(Ku), c(Kv), c(nid), c(HdiF), ref)

    def set_ref_points(self, lvl, u, v, idepth, color):
        c = lambda a: np.ascontiguousarray(a, np.float32)
        self.L.orc_ct_set_ref_points(self.hd, lvl, len(u), c(u), c(v), c(idepth), c(color))

    def ref_points(self, lvl):
        n = self.L.orc_ct_get_ref_points(self.hd, lvl, None, None, None, None)
        a = [np.zeros(n, np.float32) for _ in range(4)]
        self.L.orc_ct_get_ref_points(self.hd, lvl, *[_ptr(x) for x in a])
        return dict(u=a[0], v=a[1], idepth=a[2], color=a[3])

    def set_new_frame(self, pyr_new, ref_exposure=1.0, new_exposure=1.0, ref_a=0.0, ref_b=0.0):
        buf = self._concat(pyr_new)
        self._keep = [buf]
        self.L.orc_ct_set_new_frame(self.hd, buf, ref_exposure, new_exposure, ref_a, ref_b)

    def K(self, lvl):
        k = np.zeros(4, np.float32); wh = np.zeros(2, np.int32)
        self.L.orc_ct_get_K(self.hd, lvl, k, wh)
        return k, wh

    def calc_res(self, lvl, R, t, a, b, cutoff=20.0):
        out = np.zeros(6)
        self.L.orc_ct_calc_res(self.hd, lvl, np.ascontiguousarray(R, np.float64).reshape(-1), np.ascontiguousarray(t, np.float64), a, b, cutoff, out)
        return out

    def warped(self):
        n = self.L.orc_ct_get_warped(self.hd, None)
        buf = np.zeros((8, n), np.float32)
        self.L.orc_ct_get_warped(self.hd, _ptr(buf))
        return buf

    def calc_gs(self, lvl, a, b, precision=1):
        H = np.zeros((8, 8)); bb = np.zeros(8)
        self.L.orc_ct_calc_gs(self.hd, lvl, a, b, precision, H.reshape(-1), bb)
        return H, bb

    def track(self, R, t, a, b, coarsest=None, minRes=None, precision=1):
        R = np.ascontiguousarray(R, np.float64).reshape(-1).copy(); t = np.ascontiguousarray(t, np.float64).copy()
        ca, cb = C.c_double(a), C.c_double(b)
        its = C.c_int(0)
        lastRes = np.zeros(5); flow = np.zeros(3)
        mr = np.full(5, np.nan) if minRes is None else np.ascontiguousarray(minRes, np.float64)
        good = self.L.orc_ct_track(self.hd, R, t, C.byref(ca), C.byref(cb), self.levels - 1 if coarsest is None else coarsest, mr, precision,
                                   lastRes, flow, C.byref(its))
        return dict(good=bool(good), R=R.reshape(3, 3), t=t, a=ca.value, b=cb.value, lastResiduals=lastRes, flow=flow, iterations=its.value)


# ---- immature points (SURVEY.md 8f-2): ImmaturePoint constructor + traceOn
IP_STATE_KEYS = ("idepth_min", "idepth_max", "quality", "status", "lastTraceUV", "lastTracePixelInterval")


def ip_init(dI_host, w, h, u, v, _fn=None):
    """ImmaturePoint constructor for integer pixels (u, v) of the host frame -> dict of per-point arrays (fresh trace state included)."""
    n = len(u)
    c = lambda a, t: np.ascontiguousarray(a, t)
    P = dict(u=c(u, np.float32), v=c(v, np.float32), color=np.zeros((n, 8), np.float32), weights=np.zeros((n, 8), np.float32),
             gradH=np.zeros((n, 4), np.float32), energyTH=np.zeros(n, np.float32), ok=np.zeros(n, np.uint8))
    fn = _fn or (lambda *a: lib().orc_ip_init(*a))
    fn(n, c(dI_host, np.float32).reshape(-1), w, h, c(u, np.int32), c(v, np.int32), P["color"], P["weights"], P["gradH"], P["energyTH"], P["ok"])
    P.update(idepth_min=np.zeros(n, np.float32), idepth_max=np.full(n, np.nan, np.float32), quality=np.full(n, 10000, np.float32),
             status=np.full(n, 5, np.int32), lastTraceUV=np.zeros((n, 2), np.float32), lastTracePixelInterval=np.zeros(n, np.float32))
    return P


# per-point columns of ip_trace(..., diag=True)["diag"] (oracle/orc_trace.h IPD_*): what each traceOn call went through
IP_DIAG_KEYS = ("numSteps", "bestIdx", "nTied", "maxTiedIdx", "gnIts", "gnBreak", "nonfiniteSearch", "nonfiniteGN", "exit")
# values of the "exit" column (oracle/orc_trace.h IPX_*): the return traceOn took
IPX = dict(STICKY_OOB=0, UMIN_OOB=1, UMAX_OOB=2, DEPTH_RANGE=3, SKIPPED=4, BADCONDITION=5, NONFINITE_DIR=6, GN_OOB=7, OUTLIER=8, OUTLIER_TWICE=9,
           BAD_INTERVAL=10, GOOD=11)


def ip_trace(P, dI, w, h, KRKi, Kt, aff, _fn=None, diag=False):
    """ImmaturePoint::traceOn for every point of P against the frame dI; returns the updated state (P is not modified).
    diag=True also returns Q["diag"], (n, len(IP_DIAG_KEYS)) int32: the search's step count, best step and ties, the GN iterations, the
    non-finite samples met and the return taken, per point (same arithmetic: the state fields are those of diag=False)."""
    c = lambda a, t: np.ascontiguousarray(a, t)
    out = {k: np.array(P[k], copy=True) for k in IP_STATE_KEYS}
    n = len(P["u"])
    dg = np.zeros((n, len(IP_DIAG_KEYS)), np.int32)
    if diag:
        assert _fn is None, "diagnostics come from the oracle's own traceOn"
        fn = lambda *a: lib().orc_ip_trace_diag(*a, dg.reshape(-1))
    else:
        fn = _fn or (lambda *a: lib().orc_ip_trace(*a))
    fn(n, c(dI, np.float32).reshape(-1), w, h, c(KRKi, np.float32).reshape(-1), c(Kt, np.float32), c(aff, np.float32), P["u"], P["v"],
       P["color"], P["weights"], P["gradH"], P["energyTH"], out["idepth_min"], out["idepth_max"], out["quality"], out["status"], out["lastTraceUV"],
       out["lastTracePixelInterval"])
    Q = dict(P)
    Q.pop("diag", None)
    Q.update(out)
    if diag:
        Q["diag"] = dg
    return Q


def ip_activate(W, RT, aff, calib6, host, P, minObs=1, huberTH=9.0):
    """FullSystem::optimizeImmaturePoint for the immature points P (dict as ip_init / ip_trace) hosted in frames `host` of the window W.
    RT: (nf*nf, 12), aff: (nf*nf, 2), calib6 = fxl fyl cxl cyl fxli fyli, huberTH = setting_huberTH.  Returns status (1/0/-1), idepth, res_state (n, nf)."""
    nf, w, h = W["nf"], W["w"], W["h"]
    n = len(P["u"])
    c = lambda a, t: np.ascontiguousarray(a, t)
    dI_all = c(np.stack([np.asarray(d, np.float32).reshape(-1) for d in W["dI"]]), np.float32)
    status = np.zeros(n, np.int32); idepth = np.zeros(n, np.float32); rs = np.zeros((n, nf), np.int32)
    lib().orc_ip_activate(n, nf, w, h, c(calib6, np.float32), dI_all.reshape(-1), c(RT, np.float32).reshape(-1), c(aff, np.float32).reshape(-1),
                          c(host, np.int32), P["u"], P["v"], P["color"], P["weights"], P["energyTH"], c(P["idepth_min"], np.float32),
                          c(P["idepth_max"], np.float32), int(minObs), float(huberTH), status, idepth, rs.reshape(-1))
    return status, idepth, rs


class CoarseInit:
    """CoarseInitializer (FullSystem/CoarseInitializer.cpp) restated (orc_init.h), or — through oracle/ref.py — the reference's compiled one.
    Points (all levels), parents and neighbour lists are inputs: the pixel selector and the kd-tree are not part of the restated path."""

    _PREFIX = "orc_ci_"

    def __init__(self, w, h, K, _lib=None):
        self.L = _lib if _lib is not None else lib()
        self._bind(self.L)
        self.w, self.h = w, h
        self.hd = self._f("create")(w, h, np.ascontiguousarray(K, np.float64))
        self.levels = self._f("levels")(self.hd)
        self.n = None

    def _f(self, name):
        return getattr(self.L, self._PREFIX + name)

    @classmethod
    def _bind(cls, L):
        vp = C.c_void_p
        f = lambda n: getattr(L, cls._PREFIX + n)
        f("create").restype = vp
        f("create").argtypes = [C.c_int, C.c_int, f64p]
        f("destroy").argtypes = [vp]
        f("levels").argtypes = [vp]
        f("set_first").argtypes = [vp, f32p, C.c_float, i32p, f32p, f32p, f32p, i32p, i32p]
        f("set_new").argtypes = [vp, f32p, C.c_float]
        f("calc").argtypes = [vp, C.c_int, f64p, f64p, C.c_double, C.c_double, f32p, f32p, f32p, f32p, f32p]
        for n in ("apply_step", "opt_reg", "propagate_up", "propagate_down", "reset_points", "set_snapped", "npts"):
            f(n).argtypes = [vp, C.c_int]
        f("do_step").argtypes = [vp, C.c_int, C.c_float, f32p]
        f("calc_ec").argtypes = [vp, C.c_int, f32p]
        f("get_points").argtypes = [vp, C.c_int, f32p]
        f("set_points").argtypes = [vp, C.c_int, f32p]
        f("track").argtypes = [vp, f32p, C.c_float, f64p, f64p, f64p, i32p]

    def __del__(self):
        try:
            self._f("destroy")(self.hd)
        except Exception:
            pass

    @staticmethod
    def _concat(pyr):
        return np.ascontiguousarray(np.concatenate([np.asarray(p, np.float32).reshape(-1) for p in pyr]))

    def set_first(self, pyr, exposure, pts):
        """pts: list per level of dict(u, v, type, parent, neighbours (n, 10))"""
        self.n = np.array([len(p["u"]) for p in pts], np.int32)
        cat = lambda k, t: np.ascontiguousarray(np.concatenate([np.asarray(p[k], t).reshape(-1) for p in pts]))
        self._keep = (self._concat(pyr[:self.levels]),)
        self._f("set_first")(self.hd, self._keep[0], float(exposure), self.n, cat("u", np.float32), cat("v", np.float32), cat("type", np.float32),
                             cat("parent", np.int32), cat("neighbours", np.int32))

    def set_new(self, pyr, exposure):
        self._f("set_new")(self.hd, self._concat(pyr[:self.levels]), float(exposure))

    def calc(self, lvl, R, t, a, b):
        H, bb, Hsc, bsc, res = np.zeros(64, np.float32), np.zeros(8, np.float32), np.zeros(64, np.float32), np.zeros(8, np.float32), np.zeros(3, np.float32)
        self._f("calc")(self.hd, lvl, np.ascontiguousarray(R, np.float64).reshape(-1), np.ascontiguousarray(t, np.float64), float(a), float(b), H, bb, Hsc, bsc, res)
        return dict(H=H.reshape(8, 8), b=bb, Hsc=Hsc.reshape(8, 8), bsc=bsc, res=res)

    def static_fields(self, lvl):
        """u, v, outlierTH of points[lvl] (restatement only)"""
        n = self._f("npts")(self.hd, lvl)
        u, v, th = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
        f = self.L.orc_ci_get_static
        f.argtypes = [C.c_void_p, C.c_int, f32p, f32p, f32p]
        f(self.hd, lvl, u, v, th)
        return u, v, th

    def jb(self, lvl):
        """JbBuffer_new rows of the last calc() on this level (restatement only)"""
        n = self._f("npts")(self.hd, lvl)
        o = np.zeros((n, 10), np.float32)
        f = self.L.orc_ci_get_jb
        f.argtypes = [C.c_void_p, C.c_int, f32p]
        f(self.hd, lvl, o.reshape(-1))
        return o

    def K(self, lvl):
        k4, wh = np.zeros(4), np.zeros(2, np.int32)
        f = self.L.orc_ci_get_K
        f.argtypes = [C.c_void_p, C.c_int, f64p, i32p]
        f(self.hd, lvl, k4, wh)
        return k4, wh

    def points(self, lvl):
        n = self._f("npts")(self.hd, lvl)
        o = np.zeros((n, 12), np.float32)
        self._f("get_points")(self.hd, lvl, o.reshape(-1))
        keys = ("idepth", "idepth_new", "iR", "energy0", "energy1", "energy_new0", "energy_new1", "lastHessian", "lastHessian_new", "maxstep", "isGood", "isGood_new")
        return {k: o[:, i].copy() for i, k in enumerate(keys)}

    def set_points(self, lvl, idepth, idepth_new, iR, lastHessian, isGood):
        a = np.ascontiguousarray(np.stack([idepth, idepth_new, iR, lastHessian, np.asarray(isGood, np.float32)], axis=1), np.float32)
        self._f("set_points")(self.hd, lvl, a.reshape(-1))

    def apply_step(self, lvl): self._f("apply_step")(self.hd, lvl)
    def opt_reg(self, lvl): self._f("opt_reg")(self.hd, lvl)
    def propagate_up(self, lvl): self._f("propagate_up")(self.hd, lvl)
    def propagate_down(self, lvl): self._f("propagate_down")(self.hd, lvl)
    def reset_points(self, lvl): self._f("reset_points")(self.hd, lvl)
    def set_snapped(self, s): self._f("set_snapped")(self.hd, int(s))

    def do_step(self, lvl, lam, inc):
        self._f("do_step")(self.hd, lvl, float(lam), np.ascontiguousarray(inc, np.float32))

    def calc_ec(self, lvl):
        o = np.zeros(3, np.float32)
        self._f("calc_ec")(self.hd, lvl, o)
        return o

    def track(self, pyr, exposure):
        R, t, ab, st = np.zeros(9), np.zeros(3), np.zeros(2), np.zeros(3, np.int32)
        ok = self._f("track")(self.hd, self._concat(pyr[:self.levels]), float(exposure), R, t, ab, st)
        return dict(ok=bool(ok), R=R.reshape(3, 3), t=t, a=ab[0], b=ab[1], snapped=bool(st[0]), snappedAt=int(st[1]), frameID=int(st[2]))

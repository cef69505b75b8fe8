"""ctypes binding of the C glue (host/host_capi.h) over the C++ host adapters WindowBA / CoarseTracker — the classes a
DM-VIO checkout would link directly.  Python only marshals arrays here; all logic is C++ + CUDA."""
import ctypes as C

import numpy as np

from . import capi

f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
vp = C.c_void_p
_L = None


def lib():
    global _L
    if _L is None:
        _L = _bind(capi.lib())
    return _L


def _bind(L):
    """declares the signatures of the C glue on a loaded library (the product's libdmvio_b200.so; tests/test_host_on_oracle.py binds the
    host-logic test build the same way)"""
    if True:
        L.dmvh_window_create.restype = vp
        L.dmvh_window_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, f64p]
        L.dmvh_window_set_setting.argtypes = [vp, C.c_char_p, C.c_double]
        L.dmvh_window_destroy.argtypes = [vp]
        L.dmvh_window_error.restype = C.c_char_p
        L.dmvh_window_error.argtypes = [vp]
        L.dmvh_window_add_frame.argtypes = [vp, f32p, C.c_int, f64p, f64p, f64p, f64p, C.c_float, C.c_int]
        L.dmvh_window_drop_frame.argtypes = [vp, C.c_int]
        L.dmvh_window_marginalize_frame.argtypes = [vp, C.c_int, vp, vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.dmvh_marginalize_frame_hm.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp]
        L.dmvh_marginalize_frame_hm.restype = None
        L.dmvh_nullspaces_orthogonalize.argtypes = [C.c_int, vp, vp, vp, C.c_double]
        L.dmvh_nullspaces_orthogonalize.restype = None
        L.dmvh_window_finish_optimize.restype = C.c_double
        L.dmvh_window_finish_optimize.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.dmvh_window_get_point_stats.argtypes = [vp, vp, vp]
        L.dmvh_window_set_last_residuals.argtypes = [vp, vp, vp]
        L.dmvh_window_flag_points.argtypes = [vp, C.c_int, vp, vp, C.POINTER(C.c_int), vp, C.POINTER(C.c_int)]
        L.dmvh_window_marginalize_points.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.dmvh_window_set_points.argtypes = [vp, C.c_int, i32p, f32p, f32p, f32p, f32p, f32p, f32p, vp]
        L.dmvh_window_set_points_carry.argtypes = [vp, C.c_int, i32p, f32p, f32p, f32p, f32p, f32p, f32p, vp, i32p]
        L.dmvh_window_set_residuals.argtypes = [vp, C.c_int, i32p, i32p]
        L.dmvh_window_prepare.argtypes = [vp]
        L.dmvh_window_profile.argtypes = [vp, f64p, C.c_int]
        L.dmvh_window_profile.restype = None
        L.dmvh_window_set_sharding.argtypes = [vp, C.c_int, C.c_int, vp, vp]
        L.dmvh_window_p2p_setup.argtypes = [vp]
        L.dmvh_window_comm_init.argtypes = [vp, vp]
        L.dmvh_window_linearize.restype = C.c_double
        L.dmvh_window_linearize.argtypes = [vp, C.c_int]
        L.dmvh_window_apply.argtypes = [vp]
        L.dmvh_window_solve.argtypes = [vp, C.c_int, C.c_double, f64p]
        L.dmvh_window_optimize.argtypes = [vp, C.c_int, f64p, C.c_int]
        L.dmvh_window_get_tables.argtypes = [vp, f32p, f64p, f64p]
        L.dmvh_window_get_system.argtypes = [vp, f64p, f64p, f64p, f64p, f64p, f64p]
        L.dmvh_window_get_states.argtypes = [vp, f64p, f32p, f32p]
        L.dmvh_window_energy_L.restype = C.c_double
        L.dmvh_window_energy_L.argtypes = [vp]
        L.dmvh_window_energy_M.restype = C.c_double
        L.dmvh_window_energy_M.argtypes = [vp]
        L.dmvh_ci_create.restype = vp
        L.dmvh_ci_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, f64p]
        L.dmvh_ci_destroy.argtypes = [vp]
        L.dmvh_ci_error.restype = C.c_char_p
        L.dmvh_ci_error.argtypes = [vp]
        L.dmvh_ci_set_first.argtypes = [vp, f32p, C.c_float, i32p, f32p, f32p, f32p, i32p, i32p]
        L.dmvh_ci_track.argtypes = [vp, f32p, C.c_float, f64p, f64p, f64p, i32p]
        L.dmvh_ci_npts.argtypes = [vp, C.c_int]
        L.dmvh_ci_get_points.argtypes = [vp, C.c_int, f32p]
        L.dmvh_ci_evaluations.restype = C.c_longlong
        L.dmvh_ci_evaluations.argtypes = [vp]
        L.dmvh_ct_create.restype = vp
        L.dmvh_ct_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, f64p]
        L.dmvh_ct_destroy.argtypes = [vp]
        L.dmvh_ct_set_ref.argtypes = [vp, C.c_int, f32p, f32p, f32p, f32p, f32p, C.c_double, C.c_double, C.c_float]
        L.dmvh_ct_pc_n.argtypes = [vp, C.c_int]
        L.dmvh_ct_set_new_image.argtypes = [vp, f32p, C.c_float]
        L.dmvh_ct_set_ref_device.argtypes = [vp, C.c_int, f32p, f32p, f32p, f32p, f32p, C.c_double, C.c_double, C.c_float]
        L.dmvh_ct_set_device_lm.argtypes = [vp, C.c_int]
        L.dmvh_ct_track.argtypes = [vp, f64p, f64p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, f64p, f64p, f64p, C.POINTER(C.c_int),
                                    C.POINTER(C.c_longlong)]
    return L


def _c(a, t):
    return np.ascontiguousarray(a, t)


def nullspaces_orthogonalize(R_eval, t_eval, x=None, delta=1e-5):
    """host/nullspace.h on plain arrays: returns (nullspaces (7, N), x projected off them or None) — host-only, usable without a GPU"""
    nf = len(R_eval)
    N = 8 * nf + 4
    T = np.concatenate([np.asarray(R_eval, np.float64).reshape(nf, 9), np.asarray(t_eval, np.float64).reshape(nf, 3)], axis=1).copy()
    ns = np.zeros((7, N))
    xv = None if x is None else np.array(x, np.float64).copy()
    lib().dmvh_nullspaces_orthogonalize(nf, T.ctypes.data, ns.ctypes.data, None if xv is None else xv.ctypes.data, float(delta))
    return ns, xv


def marginalize_frame_hm(HM, bM, nframes, idx, prior8, delta_prior8):
    """host/marg_frame.h (EnergyFunctional::marginalizeFrame, visual branch) on plain arrays — host-only, usable without a GPU"""
    odim = 8 * nframes + 4
    H = np.array(HM, np.float64).reshape(odim * odim).copy(); b = np.array(bM, np.float64).copy()
    p, d = _c(prior8, np.float64), _c(delta_prior8, np.float64)
    lib().dmvh_marginalize_frame_hm(H.ctypes.data, b.ctypes.data, int(nframes), int(idx), p.ctypes.data, d.ctypes.data)
    n = odim - 8
    return H[:n * n].reshape(n, n).copy(), b[:n].copy()


ALLGATHER_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p)


class WindowBA:
    """dmvio_b200::WindowBA loaded from a synth.make_window() dict."""

    def __init__(self, W, device=0, use_device_pyramid=False, shard=None):
        """shard (multi-GPU, one WindowBA per rank): dict(rank, nranks, allgather=f(bytes) -> bytes of all ranks in rank order,
        exchange="p2p" | "nccl", uid=NCCL unique id for "nccl").  Every rank passes the SAME window."""
        self.L = lib()
        self.nf, self.npts, self.nres = W["nf"], len(W["host"]), len(W["res_point"])
        self.N = 8 * self.nf + 4
        self.h = self.L.dmvh_window_create(W["w"], W["h"], max(2, self.nf), self.npts, device, _c(W["K"], np.float64))
        for k in range(self.nf):
            data = _c(W["images"][k], np.float32).reshape(-1) if use_device_pyramid else _c(W["dI"][k], np.float32).reshape(-1)
            rc = self.L.dmvh_window_add_frame(self.h, data, int(use_device_pyramid), _c(W["R_eval"][k], np.float64).reshape(-1), _c(W["t_eval"][k], np.float64),
                                              _c(W["state"][k], np.float64), _c(W["state_zero"][k], np.float64), float(W["exposure"][k]), int(W["frameID"][k]))
            if rc < 0:
                raise capi.DmvError(self.L.dmvh_window_error(self.h).decode())
        self.L.dmvh_window_set_points(self.h, self.npts, _c(W["host"], np.int32), _c(W["u"], np.float32), _c(W["v"], np.float32), _c(W["idepth"], np.float32),
                                      _c(W["idepth_zero"], np.float32), _c(W["color"], np.float32).reshape(-1), _c(W["weights"], np.float32).reshape(-1), None)
        self.L.dmvh_window_set_residuals(self.h, len(W["res_point"]), _c(W["res_point"], np.int32), _c(W["res_target"], np.int32))
        if shard is not None:
            ag = shard["allgather"]

            def _cb(send, recv, nbytes, user):
                allb = ag(C.string_at(send, nbytes))
                C.memmove(recv, allb, len(allb))
            self._ag_cb = ALLGATHER_CB(_cb)   # keep alive as long as the window
            if self.L.dmvh_window_set_sharding(self.h, int(shard["rank"]), int(shard["nranks"]), C.cast(self._ag_cb, vp), None) != 0:
                raise capi.DmvError(self.L.dmvh_window_error(self.h).decode())
            rc = self.L.dmvh_window_comm_init(self.h, shard["uid"]) if shard.get("exchange", "p2p") == "nccl" else self.L.dmvh_window_p2p_setup(self.h)
            if rc != 0:
                raise capi.DmvError(self.L.dmvh_window_error(self.h).decode())
        if self.L.dmvh_window_prepare(self.h) != 0:
            raise capi.DmvError(self.L.dmvh_window_error(self.h).decode())

    def close(self):
        if self.h:
            self.L.dmvh_window_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def profile(self, reset=True):
        """per-iteration wall-clock split of optimize()'s LM loop, microseconds: dict(solve, step, linearize, energies, iterations)"""
        o = np.zeros(5)
        self.L.dmvh_window_profile(self.h, o, int(reset))
        n = max(1.0, o[4])
        return dict(solve=o[0] / n, step_and_tables=o[1] / n, linearize=o[2] / n, prior_energies=o[3] / n, iterations=int(o[4]))

    def tables(self):
        pc = np.zeros((self.nf * self.nf, 32), np.float32); a = np.zeros((self.nf * self.nf, 8, 8)); b = np.zeros((self.nf * self.nf, 8, 8))
        self.L.dmvh_window_get_tables(self.h, pc.reshape(-1), a.reshape(-1), b.reshape(-1))
        return pc, a, b

    def linearize(self, fix=False):
        return self.L.dmvh_window_linearize(self.h, int(fix))

    def apply(self):
        self.L.dmvh_window_apply(self.h)

    def solve(self, iteration=0, lam=1e-5):
        x = np.zeros(self.N)
        self.L.dmvh_window_solve(self.h, iteration, lam, x)
        return x

    def system(self):
        N = self.N
        o = [np.zeros(N * N), np.zeros(N), np.zeros(N * N), np.zeros(N), np.zeros(N * N), np.zeros(N)]
        self.L.dmvh_window_get_system(self.h, *o)
        return dict(HA=o[0].reshape(N, N), bA=o[1], Hsc=o[2].reshape(N, N), bsc=o[3], lastHS=o[4].reshape(N, N), lastbS=o[5])

    def optimize(self, its=6):
        log = np.zeros(64)
        n = self.L.dmvh_window_optimize(self.h, its, log, 64)
        return n, log[log >= 0]

    def finish_optimize(self):
        """WindowBA::finishOptimize — tail of FullSystem::optimize (setEvalPT of the newest frame, adjoints, precalc, linearizeAll(true)).
        Returns (energy, indices of the residuals that were deleted, residuals left)."""
        rem = np.zeros(max(1, self.nres), np.int32)
        n, left = C.c_int(0), C.c_int(0)
        E = self.L.dmvh_window_finish_optimize(self.h, rem.ctypes.data, len(rem), C.byref(n), C.byref(left))
        if not np.isfinite(E):
            raise capi.DmvError(self.L.dmvh_window_error(self.h).decode())
        self.nres = left.value
        return E, rem[:n.value].copy()

    def point_stats(self):
        mrb = np.zeros(self.npts, np.float32); ng = np.zeros(self.npts, np.int32)
        self.L.dmvh_window_get_point_stats(self.h, mrb.ctypes.data, ng.ctypes.data)
        return dict(maxRelBaseline=mrb, numGoodResiduals=ng)

    def set_last_residuals(self, target_frameID, state):
        t, s = _c(target_frameID, np.int32), _c(state, np.int32)
        assert t.shape == (self.npts, 2) and s.shape == (self.npts, 2)
        self.L.dmvh_window_set_last_residuals(self.h, t.ctypes.data, s.ctypes.data)

    def flag_points(self, flagged_frames):
        """WindowBA::flagPointsForRemoval: (toMarg, toDrop) point indices"""
        f = _c(np.asarray(flagged_frames, np.int32), np.int32)
        m = np.zeros(max(1, self.npts), np.int32); d = np.zeros(max(1, self.npts), np.int32)
        nm, nd = C.c_int(0), C.c_int(0)
        self.L.dmvh_window_flag_points(self.h, len(f), f.ctypes.data, m.ctypes.data, C.byref(nm), d.ctypes.data, C.byref(nd))
        return m[:nm.value].copy(), d[:nd.value].copy()

    def energies_LM(self):
        """(calcLEnergyF_MT, calcMEnergyF) at the current state"""
        return self.L.dmvh_window_energy_L(self.h), self.L.dmvh_window_energy_M(self.h)

    def marginalize_frame(self, idx):
        """WindowBA::marginalizeFrame: returns dict(HM, bM, nf, nres) of the smaller window"""
        nfl, nrl = C.c_int(0), C.c_int(0)
        N = self.N - 8
        HM, bM = np.zeros(self.N * self.N), np.zeros(self.N)
        rc = self.L.dmvh_window_marginalize_frame(self.h, int(idx), HM.ctypes.data, bM.ctypes.data, C.byref(nfl), C.byref(nrl))
        if rc != 0:
            raise capi.DmvError(self.L.dmvh_window_error(self.h).decode())
        self.nf, self.nres, self.N = nfl.value, nrl.value, N
        return dict(HM=HM[:N * N].reshape(N, N).copy(), bM=bM[:N].copy(), nf=self.nf, nres=self.nres)

    def marginalize_points(self, marg, drop=()):
        """WindowBA::marginalizePointsF: marginalises `marg` into HM/bM (badly constrained ones are dropped), drops `drop`, erases all of them
        and re-uploads the window.  Returns dict(resInM, HM, bM, npts, nres)."""
        N = self.N
        m, d = _c(np.asarray(marg, np.int32), np.int32), _c(np.asarray(drop, np.int32), np.int32)
        HM, bM = np.zeros((N, N)), np.zeros(N)
        npl, nrl = C.c_int(0), C.c_int(0)
        rc = self.L.dmvh_window_marginalize_points(self.h, len(m), m.ctypes.data, len(d), d.ctypes.data, HM.ctypes.data, bM.ctypes.data, C.byref(npl), C.byref(nrl))
        if rc < 0:
            raise capi.DmvError(self.L.dmvh_window_error(self.h).decode())
        self.npts, self.nres = npl.value, nrl.value
        return dict(resInM=rc, HM=HM, bM=bM, npts=npl.value, nres=nrl.value)

    def _window_ref(self):
        # bound here rather than in _bind: the CPU build of the adapters over the oracle stand-in has no device hand-off
        L = self.L
        L.dmvh_window_ba_handle.restype = vp
        L.dmvh_window_ba_handle.argtypes = [vp]
        L.dmvh_window_coarse_ref_inputs.argtypes = [vp, f32p, f32p, f32p, f32p, i32p, C.c_int]
        L.dmvh_window_get_last_residuals.argtypes = [vp, i32p, i32p]
        return L

    def ba_handle(self):
        """the window's dmv_ba* (for capi.CT.set_ref_from_ba)"""
        return self._window_ref().dmvh_window_ba_handle(self.h)

    def coarse_ref_inputs(self, with_points=False):
        """WindowBA::coarseTrackingRefInputs: (Ku, Kv, new_idepth, HdiF) of the points whose lastResiduals[0] is IN in the newest frame, in
        makeCoarseDepthL0's order (after removeOutliers' swap-with-back), as the host path downloads them for dmv_ct_make_coarse_depth;
        with_points: the points' indices as a fifth array"""
        a = [np.zeros(max(1, self.npts), np.float32) for _ in range(4)]
        pt = np.zeros(max(1, self.npts), np.int32)
        n = self._window_ref().dmvh_window_coarse_ref_inputs(self.h, *a, pt, len(pt))
        if n < 0:
            raise capi.DmvError(self.L.dmvh_window_error(self.h).decode())
        out = tuple(x[:n].copy() for x in a)
        return out + (pt[:n].copy(),) if with_points else out

    def last_residuals(self):
        """per point (target frameID, state) of lastResiduals[0..1], each (npts, 2)"""
        t, s = np.zeros((self.npts, 2), np.int32), np.zeros((self.npts, 2), np.int32)
        self._window_ref().dmvh_window_get_last_residuals(self.h, t.reshape(-1), s.reshape(-1))
        return t, s

    def states(self):
        st = np.zeros((self.nf, 10)); idd = np.zeros(self.npts, np.float32); th = np.zeros(self.nf, np.float32)
        self.L.dmvh_window_get_states(self.h, st.reshape(-1), idd, th)
        return st, idd, th


class CoarseTracker:
    def __init__(self, w, h, K, levels, max_points=65536, device=0):
        self.L = lib()
        self.levels = levels
        self.size = (w, h)
        self.h = self.L.dmvh_ct_create(w, h, levels, max_points, device, _c(K, np.float64))

    def close(self):
        if self.h:
            self.L.dmvh_ct_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_ref(self, Ku, Kv, nid, HdiF, pyr_ref, ref_a=0.0, ref_b=0.0, ref_exposure=1.0):
        ref = _c(np.concatenate([p.reshape(-1) for p in pyr_ref]), np.float32)
        rc = self.L.dmvh_ct_set_ref(self.h, len(Ku), _c(Ku, np.float32), _c(Kv, np.float32), _c(nid, np.float32), _c(HdiF, np.float32), ref, ref_a, ref_b, ref_exposure)
        if rc != 0:
            raise capi.DmvError("dmvh_ct_set_ref failed")
        return [self.L.dmvh_ct_pc_n(self.h, l) for l in range(self.levels)]

    def set_ref_device(self, Ku, Kv, nid, HdiF, img_ref, ref_a=0.0, ref_b=0.0, ref_exposure=1.0):
        """setCoarseTrackingRef with makeCoarseDepthL0 on the device (the reference keyframe arrives as a raw image)"""
        rc = self.L.dmvh_ct_set_ref_device(self.h, len(Ku), _c(Ku, np.float32), _c(Kv, np.float32), _c(nid, np.float32), _c(HdiF, np.float32),
                                           _c(img_ref, np.float32).reshape(-1), ref_a, ref_b, ref_exposure)
        if rc != 0:
            raise capi.DmvError("dmvh_ct_set_ref_device failed")
        return [self.L.dmvh_ct_pc_n(self.h, l) for l in range(self.levels)]

    def set_ref_from_ba(self, ba, ref_a=0.0, ref_b=0.0, ref_exposure=1.0):
        """CoarseTracker::setCoarseTrackingRefFromWindow: the reference is the newest keyframe of the WindowBA `ba`, built on the device from
        the window's committed residuals, last-solve HdiF and level-0 plane.  Returns pc_n per level."""
        L = self.L
        L.dmvh_ct_set_ref_from_window.argtypes = [vp, vp, C.c_double, C.c_double, C.c_float]
        if L.dmvh_ct_set_ref_from_window(self.h, ba.h, float(ref_a), float(ref_b), float(ref_exposure)) != 0:
            L.dmvh_ct_error.restype = C.c_char_p
            L.dmvh_ct_error.argtypes = [vp]
            raise capi.DmvError(L.dmvh_ct_error(self.h).decode())
        return [L.dmvh_ct_pc_n(self.h, l) for l in range(self.levels)]

    def set_new_image(self, img, exposure=1.0):
        if self.L.dmvh_ct_set_new_image(self.h, _c(img, np.float32).reshape(-1), exposure) != 0:
            raise capi.DmvError("dmvh_ct_set_new_image failed")

    def _ingest(self):
        # bound here rather than in _bind: the CPU build of the adapters over the oracle stand-in has no ingest path
        L = self.L
        L.dmvh_ct_set_undistort.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, C.c_int]
        L.dmvh_ct_upload_raw_image.argtypes = [vp, vp, C.c_int, C.c_float, C.c_float, C.c_float]
        L.dmvh_ct_download_frame.argtypes = [vp, C.c_int, f32p]
        return L

    def set_undistort(self, wOrg, hOrg, remapX=None, remapY=None, G=None, vignetteInv=None, photometric_mode=0):
        """CoarseTracker::setUndistort (dmv_ct_set_undistort)"""
        keep = [None if a is None else _c(a, np.float32).reshape(-1) for a in (remapX, remapY, G, vignetteInv)]
        p = [None if a is None else a.ctypes.data for a in keep]
        if self._ingest().dmvh_ct_set_undistort(self.h, int(wOrg), int(hOrg), p[0], p[1], p[2], 0 if G is None else len(keep[2]), p[3],
                                                int(photometric_mode)) != 0:
            raise capi.DmvError("dmvh_ct_set_undistort failed")

    def upload_raw_image(self, raw, exposure=1.0, factor=None, ab_exposure=1.0):
        """CoarseTracker::uploadRawImage: the new frame from the camera's raw bytes"""
        raw = np.ascontiguousarray(raw)
        factor = (1.0 if raw.itemsize == 1 else 1.0 / 256) if factor is None else factor
        if self._ingest().dmvh_ct_upload_raw_image(self.h, raw.ctypes.data, raw.itemsize, float(exposure), float(factor), float(ab_exposure)) != 0:
            raise capi.DmvError("dmvh_ct_upload_raw_image failed")

    def download_frame(self, lvl, w, h):
        out = np.zeros((h >> lvl) * (w >> lvl) * 3, np.float32)
        if self._ingest().dmvh_ct_download_frame(self.h, lvl, out) != 0:
            raise capi.DmvError("dmvh_ct_download_frame failed")
        return out.reshape(h >> lvl, w >> lvl, 3)

    def make_new_traces(self, potential, density=1500.0, recursionsLeft=1, thFactor=1.0, B=None, cap=16384):
        """CoarseTracker::makeNewTraces on the resident keyframe -> dict(points, numPointsTotal, potential) as capi.CT.make_new_traces
        (cap: point capacity, ten times the default density by default)"""
        L = self.L
        # bound here rather than in _bind: the CPU build of the adapters over the oracle stand-in has no pixel-selection path
        L.dmvh_ct_make_new_traces.argtypes = [vp, C.POINTER(C.c_int), C.c_float, C.c_int, C.c_float, vp, vp, C.c_int, C.POINTER(C.c_int),
                                              C.POINTER(C.c_int)] + [vp] * 8
        cap = int(cap)
        m = max(cap, 1)
        P = dict(u=np.zeros(m, np.int32), v=np.zeros(m, np.int32), type=np.zeros(m, np.float32), color=np.zeros((m, 8), np.float32),
                 weights=np.zeros((m, 8), np.float32), gradH=np.zeros((m, 4), np.float32), energyTH=np.zeros(m, np.float32))
        pot, n, npt = C.c_int(int(potential)), C.c_int(0), C.c_int(0)
        Bk = None if B is None else _c(B, np.float32)
        if L.dmvh_ct_make_new_traces(self.h, C.byref(pot), float(density), int(recursionsLeft), float(thFactor), None if Bk is None else Bk.ctypes.data, None,
                                     cap, C.byref(n), C.byref(npt), *[P[k].ctypes.data for k in ("u", "v", "type", "color", "weights", "gradH", "energyTH")],
                                     None) != 0:
            raise capi.DmvError("dmvh_ct_make_new_traces failed")
        return dict(points={k: P[k][:n.value] for k in P}, numPointsTotal=npt.value, potential=pot.value)

    def track(self, R, t, a, b, coarsest=None, minRes=None, device_lm=True):
        self.L.dmvh_ct_set_device_lm(self.h, int(device_lm))
        R = _c(R, np.float64).reshape(-1).copy(); t = _c(t, np.float64).copy()
        ca, cb = C.c_double(a), C.c_double(b)
        its, ev = C.c_int(0), C.c_longlong(0)
        lastRes, flow = np.zeros(5), np.zeros(3)
        mr = np.full(5, np.nan) if minRes is None else _c(minRes, np.float64)
        good = self.L.dmvh_ct_track(self.h, R, t, C.byref(ca), C.byref(cb), self.levels - 1 if coarsest is None else coarsest, mr, lastRes, flow,
                                    C.byref(its), C.byref(ev))
        self.L.dmvh_ct_point_evaluations.restype = C.c_double
        self.L.dmvh_ct_point_evaluations.argtypes = [C.c_void_p]
        return dict(good=bool(good), R=R.reshape(3, 3), t=t, a=ca.value, b=cb.value, lastResiduals=lastRes, flow=flow, iterations=its.value,
                    evaluations=ev.value, point_evaluations=self.L.dmvh_ct_point_evaluations(self.h))


class CoarseInit:
    """dmvio_b200::CoarseInitializer (host/coarse_initializer.h): trackFrame on the host, calcResAndGS on the device.  Points of all levels,
    parents and neighbour lists are inputs (the pixel selector and the kd-tree are not part of the path)."""

    def __init__(self, w, h, K, levels, max_points=16384, device=0):
        self.L = lib()
        self.levels = levels
        self.h = self.L.dmvh_ci_create(w, h, levels, max_points, device, _c(K, np.float64))

    def close(self):
        if self.h:
            self.L.dmvh_ci_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _concat(pyr):
        return np.ascontiguousarray(np.concatenate([np.asarray(p, np.float32).reshape(-1) for p in pyr]))

    def set_first(self, pyr, exposure, pts):
        """pts: list per level of dict(u, v, type, parent, neighbours (n, 10))"""
        n = np.array([len(p["u"]) for p in pts], np.int32)
        cat = lambda k, t: np.ascontiguousarray(np.concatenate([np.asarray(p[k], t).reshape(-1) for p in pts]))
        rc = self.L.dmvh_ci_set_first(self.h, self._concat(pyr[:self.levels]), float(exposure), n, cat("u", np.float32), cat("v", np.float32),
                                      cat("type", np.float32), cat("parent", np.int32), cat("neighbours", np.int32))
        if rc != 0:
            raise capi.DmvError(self.L.dmvh_ci_error(self.h).decode())

    def track(self, pyr, exposure):
        R, t, ab, st = np.zeros(9), np.zeros(3), np.zeros(2), np.zeros(3, np.int32)
        ok = self.L.dmvh_ci_track(self.h, self._concat(pyr[:self.levels]), float(exposure), R, t, ab, st)
        if ok < 0:
            raise capi.DmvError(self.L.dmvh_ci_error(self.h).decode())
        return dict(ok=bool(ok), R=R.reshape(3, 3), t=t, a=ab[0], b=ab[1], snapped=bool(st[0]), snappedAt=int(st[1]), frameID=int(st[2]),
                    evaluations=int(self.L.dmvh_ci_evaluations(self.h)))

    def points(self, lvl):
        n = self.L.dmvh_ci_npts(self.h, lvl)
        o = np.zeros((n, 12), np.float32)
        self.L.dmvh_ci_get_points(self.h, lvl, o.reshape(-1))
        keys = ("idepth", "idepth_new", "iR", "energy0", "energy1", "energy_new0", "energy_new1", "lastHessian", "lastHessian_new", "maxstep", "isGood", "isGood_new")
        return {k: o[:, i].copy() for i, k in enumerate(keys)}

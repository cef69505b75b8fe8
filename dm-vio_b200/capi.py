"""ctypes binding of the C ABI in include/dmvio_b200.h (libdmvio_b200.so).

This is the only way Python (tests, bench.py, __graft_entry__) reaches the product: there is no Python/torch
re-implementation of the path and no CPU fallback — loading fails loudly if the CUDA library is missing.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DMVIO_B200_LIB") or os.path.join(_HERE, "libdmvio_b200.so")   # override: A/B runs of differently built libraries
_LIB = None

f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
vp = C.c_void_p

MAX_FRAMES = 8
PRECALC_FLOATS = 32
# dmv_status (include/dmvio_b200.h)
DMV_OK, DMV_ERR_INVALID, DMV_ERR_NO_DEVICE, DMV_ERR_CUDA, DMV_ERR_STATE, DMV_ERR_NCCL, DMV_ERR_TIMEOUT = 0, -1, -2, -3, -4, -5, -6


class DmvError(RuntimeError):
    pass


class BAConfig(C.Structure):
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("max_frames", C.c_int), ("max_points", C.c_int), ("device", C.c_int), ("chunk_points", C.c_int)]


class BAParams(C.Structure):
    _fields_ = [("huberTH", C.c_float), ("outlierTHSumComponent", C.c_float), ("affineOptModeA", C.c_float), ("affineOptModeB", C.c_float)]


class BAState(C.Structure):
    _fields_ = [("calib", C.c_float * 8), ("precalc", vp), ("frameEnergyTH", vp), ("idepth", vp), ("idepth_zero", vp)]


class BALinResult(C.Structure):
    _fields_ = [("energy", C.c_double), ("n_in", C.c_int), ("n_oob", C.c_int), ("n_outlier", C.c_int)]


class BAActivateArgs(C.Structure):
    _fields_ = [("n", C.c_int)] + [(k, C.c_void_p) for k in ("host", "u", "v", "color8", "weights8", "energyTH", "idepth_min", "idepth_max", "RT")] + \
               [("minObs", C.c_int)] + [(k, C.c_void_p) for k in ("status", "idepth", "res_state")]


class BASelectArgs(C.Structure):
    _fields_ = [("nf", C.c_int), ("newest", C.c_int), ("tables12", vp), ("flagged", vp), ("n_active", C.c_int)] + \
               [(k, vp) for k in ("act_u", "act_v", "act_idepth_scaled", "act_host", "imm_offset", "u", "v", "idepth_min", "idepth_max", "lastTraceStatus",
                                  "lastTracePixelInterval", "quality", "my_type")] + \
               [("currentMinActDist", C.c_float), ("minTraceQuality", C.c_float), ("cap", C.c_int)] + [(k, vp) for k in ("n_opt", "action", "opt_idx", "map", "stats")]


class BAActivateStoreArgs(C.Structure):
    _fields_ = [("nf", C.c_int), ("newest", C.c_int), ("tables12", vp), ("flagged", vp), ("n_active", C.c_int)] + \
               [(k, vp) for k in ("act_u", "act_v", "act_idepth_scaled", "act_host", "slot", "my_type")] + \
               [("currentMinActDist", C.c_float), ("minTraceQuality", C.c_float), ("RT", vp), ("minObs", C.c_int), ("cap", C.c_int)] + \
               [(k, vp) for k in ("n_opt", "opt_frame", "opt_index", "status", "idepth", "res_state", "order_out", "n_kept", "action", "map", "stats")]


class BAEditArgs(C.Structure):
    _fields_ = [("nf", C.c_int), ("slots", vp), ("frame_src", vp), ("npts", C.c_int), ("point_src", vp), ("new_res_target", C.c_int)]


class BAMargArgs(C.Structure):
    _fields_ = [("n", C.c_int32), ("point", C.c_void_p), ("adHTdeltaF", C.c_void_p), ("cDeltaF", C.c_float * 4), ("idepthFixPriorMargFac", C.c_float)] + \
               [(k, C.c_void_p) for k in ("M", "Mb", "Msc", "Mbsc", "resInM", "ngoodRes", "res_toZeroF", "isLinearized")]


class IPPoints(C.Structure):
    _fields_ = [("n", C.c_int)] + [(k, C.c_void_p) for k in ("u", "v", "color8", "weights8", "gradH4", "energyTH", "idepth_min", "idepth_max", "quality",
                                                              "lastTraceStatus", "lastTraceUV2", "lastTracePixelInterval")]


class TraceJob(C.Structure):
    """dmv_ct_trace_job: one handle's arguments of dmv_ct_trace_many"""
    _fields_ = [("nsets", C.c_int), ("sets", vp), ("tables14", vp)]


class TraceStoreJob(C.Structure):
    """dmv_ct_trace_store_job: one handle's arguments of dmv_ct_trace_store_many"""
    _fields_ = [("store", vp), ("nslots", C.c_int), ("tables14", vp)]


class IPSettings(C.Structure):
    """dmv_ip_settings (include/dmvio_b200.h); ip_default_settings() fills it as dmv_ip_default_settings does"""
    _fields_ = [(k, C.c_float) for k in ("maxPixSearch", "trace_stepsize", "trace_GNThreshold", "trace_extraSlackOnTH", "trace_slackInterval",
                                          "trace_minImprovementFactor", "huberTH")] + [("trace_GNIterations", C.c_int), ("minTraceTestRadius", C.c_int)]


class BABatch:
    """dmv_ba_batch: B independent windows (BA handles on one device) linearised by ONE launch (include/dmvio_b200.h)."""

    def __init__(self, bas):
        self.L = lib()
        self.bas = list(bas)
        n = len(self.bas)
        self._harr = (C.c_void_p * n)(*[b.h for b in self.bas])
        h = C.c_void_p()
        check(self.L.dmv_ba_batch_create(self._harr, n, C.byref(h)))
        self.h = h

    def _args(self, xs, states):
        n = len(self.bas)
        self._xs = [None if x is None else _c(x, np.float64) for x in (xs or [None] * n)]
        self._sts = [b._state(*st) for b, st in zip(self.bas, states)]
        xarr = (C.c_void_p * n)(*[None if x is None else x.ctypes.data for x in self._xs])
        sarr = (C.c_void_p * n)(*[C.addressof(st) for st in self._sts])
        return xarr, sarr

    def gn_step(self, xs, states):
        """states[i] = (calib8, precalc, TH); xs[i] = x or None.  Returns one result dict per window."""
        n = len(self.bas)
        xarr, sarr = self._args(xs, states)
        res = (BALinResult * n)()
        sums = np.zeros(3 * n)
        check(self.L.dmv_ba_batch_gn_step(self.h, xarr, sarr, res, sums.ctypes.data))
        return [dict(energy=r.energy, n_in=r.n_in, n_oob=r.n_oob, n_outlier=r.n_outlier, sums=sums[3 * i:3 * i + 3]) for i, r in enumerate(res)]

    def bench(self, xs, states, iters=100, warmup=5):
        """returns (kernel ms per launch [CUDA events], e2e ms per batched call [wall clock, issued from C], None)"""
        n = len(self.bas)
        xarr, sarr = self._args(xs, states)
        e2e, ker = C.c_double(0), C.c_double(0)
        check(self.L.dmv_ba_batch_bench(self.h, self._harr, n, xarr, sarr, max(1, warmup), C.byref(e2e), C.byref(ker)))
        check(self.L.dmv_ba_batch_bench(self.h, self._harr, n, xarr, sarr, iters, C.byref(e2e), C.byref(ker)))
        return ker.value, e2e.value, None

    def close(self):
        if self.h:
            self.L.dmv_ba_batch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CTConfig(C.Structure):
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("levels", C.c_int), ("max_points", C.c_int), ("device", C.c_int)]


class PSSettings(C.Structure):
    _fields_ = [("minGradHistCut", C.c_float), ("minGradHistAdd", C.c_float), ("gradDownweightPerLevel", C.c_float),
                ("selectDirectionDistribution", C.c_int), ("gammaWeightsPixelSelect", C.c_int)]


class NewTracesArgs(C.Structure):
    _fields_ = [("density", C.c_float), ("recursionsLeft", C.c_int), ("thFactor", C.c_float), ("B", C.c_void_p), ("settings", C.c_void_p),
                ("potential", C.POINTER(C.c_int)), ("cap", C.c_int), ("n", C.POINTER(C.c_int)), ("numPointsTotal", C.POINTER(C.c_int)),
                ("u", C.c_void_p), ("v", C.c_void_p), ("type", C.c_void_p), ("color8", C.c_void_p), ("weights8", C.c_void_p), ("gradH4", C.c_void_p),
                ("energyTH", C.c_void_p), ("map", C.c_void_p)]


class CTTrackArgs(C.Structure):
    _fields_ = [("R", C.c_double * 9), ("t", C.c_double * 3), ("a", C.c_double), ("b", C.c_double), ("ref_a", C.c_double), ("ref_b", C.c_double),
                ("ref_exposure", C.c_float), ("new_exposure", C.c_float), ("coarseCutoffTH", C.c_float), ("affineOptModeA", C.c_float),
                ("affineOptModeB", C.c_float), ("coarsestLvl", C.c_int), ("minResForAbort", C.c_double * 5)]


class CTTrackResult(C.Structure):
    _fields_ = [("R", C.c_double * 9), ("t", C.c_double * 3), ("a", C.c_double), ("b", C.c_double), ("lastResiduals", C.c_double * 5),
                ("flowIndicators", C.c_double * 3), ("trackingGood", C.c_int), ("iterations", C.c_int), ("evaluations", C.c_int), ("status", C.c_int)]


class CTTriesArgs(C.Structure):
    _fields_ = [("n", C.c_int), ("R", vp), ("t", vp), ("a", C.c_double), ("b", C.c_double), ("ref_a", C.c_double), ("ref_b", C.c_double),
                ("ref_exposure", C.c_float), ("new_exposure", C.c_float), ("coarseCutoffTH", C.c_float), ("affineOptModeA", C.c_float),
                ("affineOptModeB", C.c_float), ("coarsestLvl", C.c_int), ("lastCoarseRMSE0", C.c_double), ("reTrackThreshold", C.c_float)]


class CTTriesResult(C.Structure):
    _fields_ = [("R", C.c_double * 9), ("t", C.c_double * 3), ("a", C.c_double), ("b", C.c_double), ("achievedRes", C.c_double * 5),
                ("flowVecs", C.c_double * 3), ("lastResiduals", C.c_double * 5), ("flowIndicators", C.c_double * 3), ("trackingGood", C.c_int),
                ("haveOneGood", C.c_int), ("winner", C.c_int), ("tries", C.c_int), ("tries_started", C.c_int)]


class UndistortConfig(C.Structure):
    _fields_ = [("wOrg", C.c_int), ("hOrg", C.c_int), ("remapX", vp), ("remapY", vp), ("G", vp), ("nG", C.c_int), ("vignetteInv", vp),
                ("photometric_mode", C.c_int)]


class CIEvalArgs(C.Structure):
    _fields_ = [("level", C.c_int), ("RKi", C.c_float * 9), ("t_d", C.c_double * 3), ("t_log", C.c_double * 3), ("r2new_aff", C.c_float * 2),
                ("huberTH", C.c_float), ("alphaK", C.c_float), ("alphaW", C.c_float), ("couplingWeight", C.c_float),
                ("weightZeroPriorX", C.c_double), ("weightZeroPriorY", C.c_double),
                ("idepth_new", C.c_void_p), ("isGood", C.c_void_p), ("energy2", C.c_void_p), ("iR", C.c_void_p),
                ("isGood_new", C.c_void_p), ("energy_new2", C.c_void_p), ("maxstep", C.c_void_p), ("lastHessian_new", C.c_void_p),
                ("JbBuffer_new10", C.c_void_p)]


class CIEvalResult(C.Structure):
    _fields_ = [("H", C.c_float * 64), ("b", C.c_float * 8), ("Hsc", C.c_float * 64), ("bsc", C.c_float * 8), ("res3", C.c_float * 3),
                ("alphaOpt", C.c_float), ("n_good_new", C.c_int)]


# every symbol declared in include/dmvio_b200.h (checked by tests/test_capi_symbols.py)
SYMBOLS = [
    "dmv_last_error", "dmv_version", "dmv_device_count",
    "dmv_ba_create", "dmv_ba_destroy", "dmv_ba_set_params", "dmv_ba_default_params", "dmv_ba_upload_frame", "dmv_ba_upload_image", "dmv_ba_adopt_frame",
    "dmv_ba_set_window", "dmv_ba_set_points", "dmv_ba_set_residuals", "dmv_ba_set_adjoints", "dmv_ba_set_state", "dmv_ba_linearize",
    "dmv_ba_get_residual_outputs", "dmv_ba_get_target_energies", "dmv_ba_apply_res", "dmv_ba_accumulate", "dmv_ba_get_point_outputs", "dmv_ba_get_solve_HdiF",
    "dmv_ba_resubstitute", "dmv_ba_backup_points", "dmv_ba_restore_points", "dmv_ba_get_idepth", "dmv_ba_gn_step", "dmv_nccl_unique_id",
    "dmv_ba_comm_init", "dmv_ba_activate_points", "dmv_ba_select_activation", "dmv_ba_activate_store", "dmv_ba_edit_window", "dmv_ba_marginalize_points", "dmv_ba_drop_residuals", "dmv_ba_reset_oob", "dmv_ba_p2p_export", "dmv_ba_p2p_import", "dmv_ba_last_timing", "dmv_ba_bench_device", "dmv_ba_bench_phases", "dmv_ba_kernel_launch_count", "dmv_ba_io_bytes", "dmv_ba_set_timing", "dmv_ba_bench_e2e",
    "dmv_ba_batch_create", "dmv_ba_batch_destroy", "dmv_ba_batch_gn_step", "dmv_ba_batch_set_timing", "dmv_ba_batch_last_kernel_ms", "dmv_ba_batch_bench",
    "dmv_ct_create", "dmv_ct_destroy", "dmv_ct_set_K", "dmv_ct_set_ref", "dmv_ct_make_coarse_depth", "dmv_ct_set_ref_from_ba", "dmv_ct_get_ref", "dmv_ct_upload_new", "dmv_ct_upload_new_image", "dmv_ct_set_huber",
    "dmv_ci_create", "dmv_ci_destroy", "dmv_ci_set_K", "dmv_ci_upload_first", "dmv_ci_upload_new", "dmv_ci_set_points", "dmv_ci_calc_res_and_gs", "dmv_ci_kernel_launch_count",
    "dmv_ct_calc_res_gs", "dmv_ct_track", "dmv_ct_track_many", "dmv_ct_track_tries", "dmv_ct_track_tries_many", "dmv_ip_default_settings", "dmv_ct_init_points", "dmv_ct_trace_points", "dmv_ct_trace_points_multi", "dmv_ct_trace_many", "dmv_ip_store_create", "dmv_ip_store_destroy", "dmv_ip_store_put", "dmv_ip_store_get", "dmv_ip_store_remove", "dmv_ct_trace_store", "dmv_ct_trace_store_many", "dmv_ct_set_timing", "dmv_ct_last_timing", "dmv_ct_kernel_launch_count", "dmv_ct_last_point_evaluations",
    "dmv_ct_set_undistort", "dmv_ct_upload_raw_image", "dmv_ct_download_frame", "dmv_ps_default_settings", "dmv_ct_make_new_traces", "dmv_ct_make_new_traces_store",
]


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise DmvError(f"{LIB_PATH} is missing: build it with `make -C dm-vio_b200` (python -c 'import __graft_entry__ as g; g.build()')")
        _LIB = _bind(C.CDLL(LIB_PATH))
    return _LIB


def load(path):
    """another build of libdmvio_b200.so (e.g. the parent commit's, for an A/B in one process), bound as lib() is"""
    return _bind(C.CDLL(os.path.abspath(path)))


def _bind(L):
    """declares the signatures of include/dmvio_b200.h on a loaded library.  An entry point that an older build lacks stays undeclared, so
    calling it raises AttributeError."""
    for name, t in _RESTYPES.items():
        if hasattr(L, name):
            getattr(L, name).restype = t
    for name, t in _ARGTYPES.items():
        if hasattr(L, name):
            getattr(L, name).argtypes = t
    return L


_RESTYPES = {
    "dmv_last_error": C.c_char_p,
    "dmv_version": C.c_char_p,
    "dmv_ps_default_settings": None,
    "dmv_ip_default_settings": None,
}
_ARGTYPES = {
    "dmv_ba_create": [C.POINTER(BAConfig), C.POINTER(vp)],
    "dmv_ba_destroy": [vp],
    "dmv_ba_set_params": [vp, C.POINTER(BAParams)],
    "dmv_ba_default_params": [C.POINTER(BAParams)],
    "dmv_ba_upload_frame": [vp, C.c_int, f32p],
    "dmv_ba_upload_image": [vp, C.c_int, f32p],
    "dmv_ba_set_window": [vp, C.c_int, vp],
    "dmv_ba_set_points": [vp, C.c_int, i32p, f32p, f32p, f32p, vp, f32p, f32p, vp],
    "dmv_ba_set_residuals": [vp, C.c_int, i32p, i32p, vp, vp],
    "dmv_ba_set_adjoints": [vp, f64p, f64p],
    "dmv_ba_set_state": [vp, C.POINTER(BAState)],
    "dmv_ba_linearize": [vp, C.POINTER(BALinResult)],
    "dmv_ba_get_residual_outputs": [vp, vp, vp, vp, vp, vp],
    "dmv_ba_get_target_energies": [vp, C.c_int, f32p, C.c_int, C.POINTER(C.c_int)],
    "dmv_ba_apply_res": [vp],
    "dmv_ba_accumulate": [vp, f64p, f64p, f64p, f64p, C.POINTER(C.c_int)],
    "dmv_ba_get_point_outputs": [vp, vp, vp, vp, vp, vp],
    "dmv_ba_resubstitute": [vp, f64p, vp, C.c_int, f64p],
    "dmv_ba_backup_points": [vp],
    "dmv_ba_restore_points": [vp],
    "dmv_ba_get_idepth": [vp, vp, vp],
    "dmv_ba_gn_step": [vp, vp, C.POINTER(BAState), C.POINTER(BALinResult), f64p],
    "dmv_nccl_unique_id": [vp],
    "dmv_ba_comm_init": [vp, C.c_int, C.c_int, vp],
    "dmv_ba_activate_points": [vp, C.POINTER(BAActivateArgs)],
    "dmv_ba_select_activation": [vp, C.POINTER(BASelectArgs)],
    "dmv_ba_activate_store": [vp, vp, C.POINTER(BAActivateStoreArgs)],
    "dmv_ba_edit_window": [vp, C.POINTER(BAEditArgs)],
    "dmv_ba_marginalize_points": [vp, C.POINTER(BAMargArgs)],
    "dmv_ba_drop_residuals": [vp, C.c_int, i32p],
    "dmv_ba_reset_oob": [vp],
    "dmv_ba_p2p_export": [vp, vp],
    "dmv_ba_p2p_import": [vp, C.c_int, C.c_int, vp],
    "dmv_ba_last_timing": [vp, f32p],
    "dmv_ba_bench_device": [vp, vp, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float)],
    "dmv_ba_bench_phases": [vp, vp, C.c_int, C.c_int, C.c_int, vp, C.POINTER(C.c_int), f32p],
    "dmv_ba_kernel_launch_count": [vp, C.POINTER(C.c_longlong)],
    "dmv_ba_set_timing": [vp, C.c_int],
    "dmv_ba_bench_e2e": [vp, vp, C.POINTER(BAState), C.c_int, C.POINTER(C.c_double)],
    "dmv_ba_io_bytes": [vp, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)],
    "dmv_ba_get_solve_HdiF": [vp, f32p],
    "dmv_ba_adopt_frame": [vp, C.c_int, vp],
    "dmv_ba_batch_create": [vp, C.c_int, C.POINTER(vp)],
    "dmv_ba_batch_destroy": [vp],
    "dmv_ba_batch_gn_step": [vp, vp, vp, vp, vp],
    "dmv_ba_batch_set_timing": [vp, C.c_int],
    "dmv_ba_batch_last_kernel_ms": [vp, C.POINTER(C.c_float)],
    "dmv_ba_batch_bench": [vp, vp, C.c_int, vp, vp, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)],
    "dmv_ct_create": [C.POINTER(CTConfig), C.POINTER(vp)],
    "dmv_ct_destroy": [vp],
    "dmv_ct_set_K": [vp, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float],
    "dmv_ct_set_ref": [vp, C.c_int, C.c_int, f32p, f32p, f32p, f32p],
    "dmv_ct_make_coarse_depth": [vp, C.c_int, f32p, f32p, f32p, f32p, i32p],
    "dmv_ct_set_ref_from_ba": [vp, vp, i32p],
    "dmv_ct_get_ref": [vp, C.c_int, C.POINTER(C.c_int), vp, vp, vp, vp],
    "dmv_ct_upload_new": [vp, C.c_int, f32p],
    "dmv_ct_upload_new_image": [vp, f32p],
    "dmv_ct_set_huber": [vp, C.c_float],
    "dmv_ct_calc_res_gs": [vp, C.c_int, f32p, f32p, f32p, C.c_float, C.c_float, C.c_int, f64p, f64p, f64p, C.POINTER(C.c_int)],
    "dmv_ct_track": [vp, C.POINTER(CTTrackArgs), C.POINTER(CTTrackResult)],
    "dmv_ct_track_many": [C.POINTER(vp), C.c_int, C.POINTER(CTTrackArgs), C.POINTER(CTTrackResult)],
    "dmv_ct_track_tries": [vp, C.POINTER(CTTriesArgs), C.POINTER(CTTriesResult)],
    "dmv_ct_track_tries_many": [C.POINTER(vp), C.c_int, C.POINTER(CTTriesArgs), C.POINTER(CTTriesResult)],
    "dmv_ct_init_points": [vp, C.c_int, i32p, i32p, f32p, f32p, f32p, f32p, i32p],
    "dmv_ct_trace_points": [vp, C.POINTER(IPPoints), f32p, f32p, f32p, vp],
    "dmv_ct_trace_points_multi": [vp, C.c_int, vp, vp, vp],
    "dmv_ct_trace_many": [C.POINTER(vp), C.c_int, C.POINTER(TraceJob), vp],
    "dmv_ip_store_create": [C.c_int, C.POINTER(vp)],
    "dmv_ip_store_destroy": [vp],
    "dmv_ip_store_put": [vp, C.c_int, C.POINTER(IPPoints)],
    "dmv_ip_store_get": [vp, C.c_int, C.POINTER(IPPoints)],
    "dmv_ip_store_remove": [vp, C.c_int, C.c_int, vp, vp],
    "dmv_ct_trace_store": [vp, vp, C.c_int, vp, vp],
    "dmv_ct_trace_store_many": [C.POINTER(vp), C.c_int, C.POINTER(TraceStoreJob), vp],
    "dmv_ct_set_timing": [vp, C.c_int],
    "dmv_ct_last_timing": [vp, f32p],
    "dmv_ct_kernel_launch_count": [vp, C.POINTER(C.c_longlong)],
    "dmv_ct_last_point_evaluations": [vp, C.POINTER(C.c_double)],
    "dmv_ct_set_undistort": [vp, C.POINTER(UndistortConfig)],
    "dmv_ct_upload_raw_image": [vp, vp, C.c_int, C.c_float, C.c_float],
    "dmv_ct_download_frame": [vp, C.c_int, f32p],
    "dmv_ps_default_settings": [C.POINTER(PSSettings)],
    "dmv_ip_default_settings": [C.POINTER(IPSettings)],
    "dmv_ct_make_new_traces": [vp, C.POINTER(NewTracesArgs)],
    "dmv_ct_make_new_traces_store": [vp, vp, C.c_int, C.POINTER(NewTracesArgs)],
    "dmv_ci_create": [C.POINTER(CTConfig), C.POINTER(vp)],
    "dmv_ci_destroy": [vp],
    "dmv_ci_set_K": [vp, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float],
    "dmv_ci_upload_first": [vp, C.c_int, vp],
    "dmv_ci_upload_new": [vp, C.c_int, vp],
    "dmv_ci_set_points": [vp, C.c_int, C.c_int, vp, vp, vp],
    "dmv_ci_calc_res_and_gs": [vp, C.POINTER(CIEvalArgs), C.POINTER(CIEvalResult)],
    "dmv_ci_kernel_launch_count": [vp, C.POINTER(C.c_longlong)],
}


def check(rc, L=None):
    """raises DmvError with the message of the library L (default lib()) for a non-zero dmv_status"""
    if rc != 0:
        raise DmvError(f"dmvio_b200 error {rc}: {(L or lib()).dmv_last_error().decode()}")


def _p(a):
    return None if a is None else a.ctypes.data_as(vp)


def _c(a, t):
    return None if a is None else np.ascontiguousarray(a, t)


class BA:
    """Thin RAII wrapper over a dmv_ba handle; argument names follow include/dmvio_b200.h."""

    def __init__(self, w, h, max_frames=8, max_points=8192, device=0, chunk_points=0):
        self.L = lib()
        cfg = BAConfig(w, h, max_frames, max_points, device, chunk_points)
        self.h = vp()
        check(self.L.dmv_ba_create(C.byref(cfg), C.byref(self.h)))
        self.w, self.hh = w, h
        self.nf = self.npts = self.nres = 0
        self._keep = {}

    def close(self):
        if self.h:
            self.L.dmv_ba_destroy(self.h)
            self.h = vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_params(self, huberTH=9.0, outlierTHSumComponent=2500.0, affineOptModeA=1e12, affineOptModeB=1e8):
        p = BAParams(huberTH, outlierTHSumComponent, affineOptModeA, affineOptModeB)
        check(self.L.dmv_ba_set_params(self.h, C.byref(p)))

    def upload_frame(self, slot, dI):
        check(self.L.dmv_ba_upload_frame(self.h, slot, _c(dI, np.float32).reshape(-1)))

    def upload_image(self, slot, img):
        check(self.L.dmv_ba_upload_image(self.h, slot, _c(img, np.float32).reshape(-1)))

    def adopt_frame(self, slot, ct):
        """level-0 plane of the frame resident in the coarse-tracker handle `ct` (capi.CT), device to device"""
        check(self.L.dmv_ba_adopt_frame(self.h, slot, ct.h))

    def set_window(self, nf, slots=None):
        s = _c(slots, np.int32)
        check(self.L.dmv_ba_set_window(self.h, nf, _p(s)))
        self.nf = nf
        self.N = 8 * nf + 4

    def set_points(self, host, u, v, idepth, idepth_zero, color, weights, priorF=None):
        self.npts = len(host)
        iz, pf = _c(idepth_zero, np.float32), _c(priorF, np.float32)
        check(self.L.dmv_ba_set_points(self.h, self.npts, _c(host, np.int32), _c(u, np.float32), _c(v, np.float32), _c(idepth, np.float32),
                                       _p(iz), _c(color, np.float32).reshape(-1), _c(weights, np.float32).reshape(-1), _p(pf)))

    def set_residuals(self, point, target, state=None, energy=None):
        self.nres = len(point)
        s, e = _c(state, np.int32), _c(energy, np.float32)
        check(self.L.dmv_ba_set_residuals(self.h, self.nres, _c(point, np.int32), _c(target, np.int32), _p(s), _p(e)))

    def set_adjoints(self, adHost, adTarget):
        check(self.L.dmv_ba_set_adjoints(self.h, _c(adHost, np.float64).reshape(-1), _c(adTarget, np.float64).reshape(-1)))

    def _state(self, calib8, precalc, TH, idepth=None, idepth_zero=None):
        st = BAState()
        k = _c(calib8, np.float32)
        for i in range(8):
            st.calib[i] = float(k[i])
        pc, th, idd, idz = _c(precalc, np.float32), _c(TH, np.float32), _c(idepth, np.float32), _c(idepth_zero, np.float32)
        self._keep = dict(pc=pc, th=th, idd=idd, idz=idz)
        st.precalc, st.frameEnergyTH, st.idepth, st.idepth_zero = _p(pc), _p(th), _p(idd), _p(idz)
        return st

    def set_state(self, calib8, precalc, TH, idepth=None, idepth_zero=None):
        st = self._state(calib8, precalc, TH, idepth, idepth_zero)
        check(self.L.dmv_ba_set_state(self.h, C.byref(st)))

    def linearize(self):
        r = BALinResult()
        check(self.L.dmv_ba_linearize(self.h, C.byref(r)))
        return dict(energy=r.energy, n_in=r.n_in, n_oob=r.n_oob, n_outlier=r.n_outlier)

    def gn_step(self, x, calib8, precalc, TH, idepth=None, idepth_zero=None):
        st = self._state(calib8, precalc, TH, idepth, idepth_zero)
        r = BALinResult()
        sums = np.zeros(3)
        xx = _c(x, np.float64)
        check(self.L.dmv_ba_gn_step(self.h, _p(xx), C.byref(st), C.byref(r), sums))
        return dict(energy=r.energy, n_in=r.n_in, n_oob=r.n_oob, n_outlier=r.n_outlier, sums=sums)

    def residual_outputs(self):
        n = self.nres
        o = dict(newState=np.zeros(n, np.int32), newEnergy=np.zeros(n, np.float32), newEnergyWithOutlier=np.zeros(n, np.float32),
                 centerProjectedTo=np.zeros((n, 3), np.float32), JpJdF=np.zeros((n, 8), np.float32))
        check(self.L.dmv_ba_get_residual_outputs(self.h, _p(o["newState"]), _p(o["newEnergy"]), _p(o["newEnergyWithOutlier"]),
                                                 _p(o["centerProjectedTo"]), _p(o["JpJdF"])))
        return o

    def target_energies(self, target):
        out = np.zeros(max(self.npts, 1), np.float32)
        n = C.c_int(0)
        check(self.L.dmv_ba_get_target_energies(self.h, target, out, len(out), C.byref(n)))
        return out[:n.value]

    def apply_res(self):
        check(self.L.dmv_ba_apply_res(self.h))

    def accumulate(self):
        N = self.N
        o = dict(HA=np.zeros((N, N)), bA=np.zeros(N), Hsc=np.zeros((N, N)), bsc=np.zeros(N))
        n = C.c_int(0)
        check(self.L.dmv_ba_accumulate(self.h, o["HA"].reshape(-1), o["bA"], o["Hsc"].reshape(-1), o["bsc"], C.byref(n)))
        o["resInA"] = n.value
        return o

    def point_outputs(self):
        n = self.npts
        o = dict(Hdd=np.zeros(n, np.float32), bd=np.zeros(n, np.float32), Hcd=np.zeros((n, 4), np.float32), HdiF=np.zeros(n, np.float32),
                 bdSumF=np.zeros(n, np.float32))
        check(self.L.dmv_ba_get_point_outputs(self.h, _p(o["Hdd"]), _p(o["bd"]), _p(o["Hcd"]), _p(o["HdiF"]), _p(o["bdSumF"])))
        return o

    def resubstitute(self, x, apply=False):
        step = np.zeros(self.npts, np.float32)
        sums = np.zeros(3)
        check(self.L.dmv_ba_resubstitute(self.h, _c(x, np.float64), _p(step), int(apply), sums))
        return step, sums

    def backup_points(self):
        check(self.L.dmv_ba_backup_points(self.h))

    def restore_points(self):
        check(self.L.dmv_ba_restore_points(self.h))

    def get_idepth(self):
        a, b = np.zeros(self.npts, np.float32), np.zeros(self.npts, np.float32)
        check(self.L.dmv_ba_get_idepth(self.h, _p(a), _p(b)))
        return a, b

    def last_timing(self):
        ms = np.zeros(4, np.float32)
        check(self.L.dmv_ba_last_timing(self.h, ms))
        return ms

    def bench_device(self, x=None, iters=100, flush_l2=True):
        a, b = C.c_float(0), C.c_float(0)
        xx = _c(x, np.float64)
        check(self.L.dmv_ba_bench_device(self.h, _p(xx), iters, int(flush_l2), C.byref(a), C.byref(b)))
        return a.value, b.value

    def bench_phases(self, x=None, iters=100, flush_l2=True, max_ctas=1024):
        """phase clock of `iters` launches: (stamps [iters, n_ctas, 9] uint64 ns, CUDA-event ms per launch [iters])"""
        st = np.zeros((iters, max_ctas, 9), np.uint64)
        ms = np.zeros(iters, np.float32)
        n = C.c_int(0)
        xx = _c(x, np.float64)
        check(self.L.dmv_ba_bench_phases(self.h, _p(xx), iters, int(flush_l2), max_ctas, st.ctypes.data, C.byref(n), ms))
        return st[:, :n.value], ms

    def launch_count(self):
        n = C.c_longlong(0)
        check(self.L.dmv_ba_kernel_launch_count(self.h, C.byref(n)))
        return n.value

    def set_timing(self, enable=True):
        check(self.L.dmv_ba_set_timing(self.h, int(enable)))

    def bench_e2e(self, x, calib8, precalc, TH, iters=100):
        st = self._state(calib8, precalc, TH)
        ms = C.c_double(0)
        xx = _c(x, np.float64)
        check(self.L.dmv_ba_bench_e2e(self.h, _p(xx), C.byref(st), iters, C.byref(ms)))
        return ms.value

    def io_bytes(self):
        a, b = C.c_longlong(0), C.c_longlong(0)
        check(self.L.dmv_ba_io_bytes(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def comm_init(self, nranks, rank, uid_bytes):
        buf = C.create_string_buffer(bytes(uid_bytes), 128)
        check(self.L.dmv_ba_comm_init(self.h, nranks, rank, C.cast(buf, vp)))


    def activate_points(self, host, P, RT, minObs=1):
        """FullSystem::optimizeImmaturePoint for the immature points P (dict as oracle.orc.ip_init) hosted in window frames `host`;
        returns status (1 activate / 0 keep / -1 delete), idepth, res_state (n, nf)."""
        n = len(P["u"])
        keep = [_c(host, np.int32)] + [_c(P[k], np.float32) for k in ("u", "v", "color", "weights", "energyTH", "idepth_min", "idepth_max")] + [_c(RT, np.float32)]
        status = np.zeros(n, np.int32); idepth = np.zeros(n, np.float32); rs = np.zeros((n, self.nf), np.int32)
        args = BAActivateArgs(n, *[a.ctypes.data for a in keep], int(minObs), status.ctypes.data, idepth.ctypes.data, rs.ctypes.data)
        check(self.L.dmv_ba_activate_points(self.h, C.byref(args)))
        return status, idepth, rs

    def select_activation(self, nf, newest, tables12, flagged, act_u, act_v, act_idepth_scaled, act_host, imm_offset, imm, min_act_dist,
                          min_trace_quality=3.0, cap=None, want_map=True):
        """FullSystem::activatePointsMT up to activatePointsMT_Reductor (dmv_ba_select_activation): imm = dict of the immature points' u, v,
        idepth_min, idepth_max, status, interval, quality, type, grouped by host as imm_offset says.  Returns (action: 0 keep / 1 delete /
        2 optimise, toOptimize indexes, level-1 map (h/2, w/2) or None, stats dict: undecided candidates, floods run, rounds of the chain)."""
        off = _c(imm_offset, np.int32)
        n = int(off[-1])
        keep = [_c(tables12, np.float32), _c(flagged, np.uint8), _c(act_u, np.float32), _c(act_v, np.float32), _c(act_idepth_scaled, np.float32),
                _c(act_host, np.int32), off] + [_c(imm[k], t) for k, t in (("u", np.float32), ("v", np.float32), ("idepth_min", np.float32),
                ("idepth_max", np.float32), ("status", np.int32), ("interval", np.float32), ("quality", np.float32), ("type", np.float32))]
        cap = n if cap is None else int(cap)
        action, opt = np.zeros(max(n, 1), np.int32), np.zeros(max(cap, 1), np.int32)
        m = np.zeros((self.hh // 2, self.w // 2), np.float32) if want_map else None
        n_opt, stats = C.c_int(0), np.zeros(3, np.int32)
        a = BASelectArgs(int(nf), int(newest), keep[0].ctypes.data, keep[1].ctypes.data, len(keep[2]), *[k.ctypes.data for k in keep[2:]],
                         float(min_act_dist), float(min_trace_quality), cap, C.addressof(n_opt), action.ctypes.data, opt.ctypes.data,
                         m.ctypes.data if want_map else None, stats.ctypes.data)
        rc = self.L.dmv_ba_select_activation(self.h, C.byref(a))
        if rc != 0:
            raise DmvError(f"dmvio_b200 error {rc}: {lib().dmv_last_error().decode()}", n_opt.value)
        return action[:n], opt[:n_opt.value].copy(), m, dict(undecided=int(stats[0]), floods=int(stats[1]), rounds=int(stats[2]))

    def activate_store(self, store, newest, tables12, flagged, act_u, act_v, act_idepth_scaled, act_host, slot, my_type, min_act_dist, RT,
                       min_trace_quality=3.0, minObs=1, cap=None, want_map=False):
        """FullSystem::activatePointsMT on the immature points of an IPStore (dmv_ba_activate_store): frame f's points are slot slot[f]
        (-1: none), my_type[f] their types (None for a frame without points).  Updates store.counts.  Returns a dict: opt_frame,
        opt_index (toOptimize as (frame, index in its slot before the call)), status, idepth, res_state (n_opt, nf), order (one segment
        per frame), n_kept [nf], action, map ((h/2, w/2) or None), stats (undecided, floods, rounds).  On cap overflow DmvError carries
        the count needed."""
        nf = self.nf
        slot = _c(slot, np.int32)
        counts = [store.counts[k] if k >= 0 else 0 for k in slot]
        n = int(sum(counts))
        types = [None if t is None else _c(t, np.float32) for t in my_type]
        tptr = (vp * max(nf, 1))(*[None if t is None else t.ctypes.data for t in types])
        keep = [_c(tables12, np.float32), _c(flagged, np.uint8), _c(act_u, np.float32), _c(act_v, np.float32), _c(act_idepth_scaled, np.float32),
                _c(act_host, np.int32), _c(RT, np.float32)]
        cap = n if cap is None else int(cap)
        ofr, oix, st, idp = (np.zeros(max(cap, 1), t) for t in (np.int32, np.int32, np.int32, np.float32))
        rs = np.zeros((max(cap, 1), nf), np.int32)
        order, n_kept, action = np.zeros(max(n, 1), np.int32), np.zeros(nf, np.int32), np.zeros(max(n, 1), np.int32)
        m = np.zeros((self.hh // 2, self.w // 2), np.float32) if want_map else None
        n_opt, stats = C.c_int(0), np.zeros(3, np.int32)
        a = BAActivateStoreArgs(nf, int(newest), keep[0].ctypes.data, keep[1].ctypes.data, len(keep[2]), *[k.ctypes.data for k in keep[2:6]],
                                slot.ctypes.data, C.cast(tptr, vp), float(min_act_dist), float(min_trace_quality), keep[6].ctypes.data, int(minObs), cap,
                                C.addressof(n_opt), *[x.ctypes.data for x in (ofr, oix, st, idp, rs, order, n_kept, action)],
                                m.ctypes.data if want_map else None, stats.ctypes.data)
        rc = self.L.dmv_ba_activate_store(self.h, store.h, C.byref(a))
        if rc != 0:
            raise DmvError(f"dmvio_b200 error {rc}: {lib().dmv_last_error().decode()}", n_opt.value)
        for k, kept in zip(slot, n_kept):
            if k >= 0:
                store.counts[k] = int(kept)
        k = n_opt.value
        return dict(opt_frame=ofr[:k].copy(), opt_index=oix[:k].copy(), status=st[:k].copy(), idepth=idp[:k].copy(), res_state=rs[:k].copy(),
                    order=order[:int(n_kept.sum())].copy(), n_kept=n_kept, action=action[:n].copy(), map=m,
                    stats=dict(undecided=int(stats[0]), floods=int(stats[1]), rounds=int(stats[2])))

    def edit_window(self, nf, slots, frame_src, point_src, new_res_target=-1, *, nres):
        """dmv_ba_edit_window: the window becomes nf frames (image slots `slots`, None = 0..nf-1; frame_src[f] = the frame's current index or
        -1) and the points point_src (a current index, or -1 - k for entry k of the last activation).  nres is the new window's residual count
        by the header's rules (the caller replays them, as it keeps the lists the per-residual read-backs are ordered by); it sizes
        residual_outputs and the other per-residual read-backs."""
        s, fs, ps = _c(slots, np.int32), _c(frame_src, np.int32), _c(point_src, np.int32)
        a = BAEditArgs(int(nf), None if s is None else s.ctypes.data, fs.ctypes.data, len(ps), ps.ctypes.data, int(new_res_target))
        check(self.L.dmv_ba_edit_window(self.h, C.byref(a)))
        self.nf, self.N, self.npts, self.nres = int(nf), 8 * int(nf) + 4, len(ps), int(nres)

    def reset_oob(self):
        check(self.L.dmv_ba_reset_oob(self.h))

    def drop_residuals(self, idx):
        """residuals leave the window (FullSystemOptimize.cpp:L196-214); the remaining ones keep their order"""
        idx = _c(idx, np.int32)
        check(self.L.dmv_ba_drop_residuals(self.h, len(idx), idx))
        self.nres -= len(np.unique(idx))

    def marginalize_points(self, pts, adHTdeltaF, cDeltaF, prior_fac=600.0 * 600.0):
        """flagPointsForRemoval's linearize / fixLinearizationF loop + marginalizePointsF for the listed points (dmv_ba_marginalize_points).
        Returns dict: M, Mb, Msc, Mbsc, H = M - Msc, b = Mb - Mbsc, resInM, ngood [n], rtz [nres, 8], isLinearized [nres]."""
        N = 8 * self.nf + 4
        pts = _c(pts, np.int32)
        ad = _c(adHTdeltaF, np.float32)
        assert ad.size == self.nf * self.nf * 8
        o = dict(M=np.zeros((N, N)), Mb=np.zeros(N), Msc=np.zeros((N, N)), Mbsc=np.zeros(N), ngood=np.zeros(len(pts), np.int32),
                 rtz=np.zeros((self.nres, 8), np.float32), isLinearized=np.zeros(self.nres, np.uint8))
        n = C.c_int32(0)
        args = BAMargArgs(len(pts), pts.ctypes.data, ad.ctypes.data, (C.c_float * 4)(*[float(x) for x in cDeltaF]), float(prior_fac),
                          o["M"].ctypes.data, o["Mb"].ctypes.data, o["Msc"].ctypes.data, o["Mbsc"].ctypes.data, C.addressof(n),
                          o["ngood"].ctypes.data, o["rtz"].ctypes.data, o["isLinearized"].ctypes.data)
        check(self.L.dmv_ba_marginalize_points(self.h, C.byref(args)))
        o["resInM"] = n.value
        o["H"], o["b"] = o["M"] - o["Msc"], o["Mb"] - o["Mbsc"]
        return o

    def p2p_export(self):
        """64-byte CUDA IPC handle of this rank's exchange inbox (all-gather it, then p2p_import)."""
        buf = C.create_string_buffer(64)
        check(self.L.dmv_ba_p2p_export(self.h, C.cast(buf, vp)))
        return bytes(buf.raw)

    def p2p_import(self, nranks, rank, handles):
        blob = b"".join(bytes(h) for h in handles)
        assert len(blob) == 64 * nranks
        buf = C.create_string_buffer(blob, len(blob))
        check(self.L.dmv_ba_p2p_import(self.h, nranks, rank, C.cast(buf, vp)))


def ip_default_settings():
    """an IPSettings filled by dmv_ip_default_settings"""
    S = IPSettings()
    lib().dmv_ip_default_settings(C.byref(S))
    return S


def nccl_unique_id():
    buf = C.create_string_buffer(128)
    check(lib().dmv_nccl_unique_id(C.cast(buf, vp)))
    return bytes(buf.raw)


def _track_args(levels, R, t, a, b, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0, cutoff=20.0, affA=1e12, affB=1e8, coarsest=None,
                minRes=None):
    """the dmv_ct_track_args of CT.track's arguments for a handle of `levels` levels"""
    A = CTTrackArgs()
    A.R[:] = [float(x) for x in np.asarray(R, np.float64).reshape(-1)]
    A.t[:] = [float(x) for x in np.asarray(t, np.float64).reshape(-1)]
    A.a, A.b, A.ref_a, A.ref_b = float(a), float(b), float(ref_a), float(ref_b)
    A.ref_exposure, A.new_exposure, A.coarseCutoffTH, A.affineOptModeA, A.affineOptModeB = ref_exposure, new_exposure, cutoff, affA, affB
    A.coarsestLvl = levels - 1 if coarsest is None else int(coarsest)
    A.minResForAbort[:] = [float(x) for x in (np.full(5, np.nan) if minRes is None else np.asarray(minRes, np.float64))]
    return A


def _track_result(r):
    return dict(R=np.array(r.R).reshape(3, 3), t=np.array(r.t), a=r.a, b=r.b, lastResiduals=np.array(r.lastResiduals), flow=np.array(r.flowIndicators),
                good=r.trackingGood, iterations=r.iterations, evaluations=r.evaluations, status=r.status)


def _tries_args(levels, R, t, a, b, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0, cutoff=20.0, affA=1e12, affB=1e8, coarsest=None,
                lastCoarseRMSE0=100.0, reTrackThreshold=1.5):
    """the dmv_ct_tries_args of CT.track_tries's arguments (R: n 3x3 matrices, t: n 3-vectors) and the arrays it points to; the fields it
    shares with dmv_ct_track_args go through _track_args"""
    Rs = np.ascontiguousarray(np.asarray(R, np.float64).reshape(-1, 9))
    ts = np.ascontiguousarray(np.asarray(t, np.float64).reshape(-1, 3))
    if len(Rs) != len(ts):
        raise ValueError(f"{len(Rs)} rotations but {len(ts)} translations")
    T = _track_args(levels, Rs[0] if len(Rs) else np.eye(3), ts[0] if len(ts) else np.zeros(3), a, b, ref_a, ref_b, ref_exposure, new_exposure,
                    cutoff, affA, affB, coarsest)
    A = CTTriesArgs(len(Rs), Rs.ctypes.data, ts.ctypes.data, T.a, T.b, T.ref_a, T.ref_b, T.ref_exposure, T.new_exposure, T.coarseCutoffTH,
                    T.affineOptModeA, T.affineOptModeB, T.coarsestLvl, float(lastCoarseRMSE0), float(reTrackThreshold))
    return A, (Rs, ts)


def _tries_result(r):
    return dict(R=np.array(r.R).reshape(3, 3), t=np.array(r.t), a=r.a, b=r.b, achievedRes=np.array(r.achievedRes), flowVecs=np.array(r.flowVecs),
                lastResiduals=np.array(r.lastResiduals), flow=np.array(r.flowIndicators), good=r.trackingGood, haveOneGood=r.haveOneGood,
                winner=r.winner, tries=r.tries, tries_started=r.tries_started)


def ct_track_many(handles, args):
    """dmv_ct_track_many: handles[i] (a CT) tracked with args[i] (a dict of CT.track's keywords), all in one launch.  Returns the list of
    CT.track's result dicts, each bit-identical to handles[i].track(**args[i])."""
    if len(handles) != len(args):
        raise ValueError(f"{len(handles)} handles but {len(args)} argument sets")
    n = len(handles)
    H = (vp * n)(*[g.h.value for g in handles])
    A = (CTTrackArgs * n)(*[_track_args(g.levels, **a) for g, a in zip(handles, args)])
    r = (CTTrackResult * n)()
    check(lib().dmv_ct_track_many(H, n, A, r))
    return [_track_result(x) for x in r]


def ct_track_tries_many(handles, args):
    """dmv_ct_track_tries_many: handles[i] (a CT) runs trackNewCoarse's try loop with args[i] (a dict of CT.track_tries's keywords, R and t
    included), all in one launch.  Returns the list of CT.track_tries's result dicts, each bit-identical to handles[i].track_tries(**args[i])."""
    if len(handles) != len(args):
        raise ValueError(f"{len(handles)} handles but {len(args)} argument sets")
    n = len(handles)
    H = (vp * n)(*[g.h.value for g in handles])
    made = [_tries_args(g.levels, **a) for g, a in zip(handles, args)]
    A = (CTTriesArgs * n)(*[m[0] for m in made])
    r = (CTTriesResult * n)()
    check(lib().dmv_ct_track_tries_many(H, n, A, r))
    return [_tries_result(x) for x in r]


class _TraceSets:
    """the marshalling shared by CT.trace_points_multi and ct_trace_many: sets = [(P, KRKi, Kt, aff), ...] (P a dict of arrays as
    oracle.orc.ip_init returns) as one dmv_ct_trace_job.  The in/out fields are copies (P itself is not modified); results() returns the
    updated dicts."""

    def __init__(self, sets):
        self.sets = list(sets)
        ns = len(self.sets)
        self.arr = (IPPoints * max(ns, 1))()
        self.tab = np.zeros((max(ns, 1), 14), np.float32)
        self.keeps, self.outs = [], []
        for k, (P, KRKi, Kt, aff) in enumerate(self.sets):
            keep = {q: _c(P[q], np.float32) for q in ("u", "v", "color", "weights", "gradH", "energyTH")}
            out = {"idepth_min": np.array(P["idepth_min"], np.float32, copy=True), "idepth_max": np.array(P["idepth_max"], np.float32, copy=True),
                   "quality": np.array(P["quality"], np.float32, copy=True), "status": np.array(P["status"], np.int32, copy=True),
                   "lastTraceUV": np.array(P["lastTraceUV"], np.float32, copy=True), "lastTracePixelInterval": np.array(P["lastTracePixelInterval"], np.float32, copy=True)}
            self.arr[k] = IPPoints(len(P["u"]), *[x.ctypes.data for x in (keep["u"], keep["v"], keep["color"], keep["weights"], keep["gradH"], keep["energyTH"],
                                                                           out["idepth_min"], out["idepth_max"], out["quality"], out["status"], out["lastTraceUV"],
                                                                           out["lastTracePixelInterval"])])
            self.tab[k, :9] = np.asarray(KRKi, np.float32).reshape(-1); self.tab[k, 9:12] = Kt; self.tab[k, 12:14] = aff
            self.keeps.append(keep); self.outs.append(out)
        self.job = TraceJob(ns, C.addressof(self.arr), self.tab.ctypes.data)

    def results(self):
        res = []
        for (P, _, _, _), out in zip(self.sets, self.outs):
            Q = dict(P); Q.update(out); res.append(Q)
        return res


def ct_trace_many(handles, jobs, settings=None):
    """dmv_ct_trace_many: jobs[i] (the sets list CT.trace_points_multi takes) traced on handles[i] (a CT), all in one launch.  Returns the
    list of per-member lists of updated dicts, each bit-identical to handles[i].trace_points_multi(jobs[i], settings).  settings: an
    IPSettings, or None (NULL: defaults)."""
    if len(handles) != len(jobs):
        raise ValueError(f"{len(handles)} handles but {len(jobs)} jobs")
    n = len(handles)
    T = [_TraceSets(j) for j in jobs]
    H = (vp * max(n, 1))(*[g.h.value for g in handles])
    J = (TraceJob * max(n, 1))(*[t.job for t in T])
    check(lib().dmv_ct_trace_many(H, n, J, None if settings is None else C.byref(settings)))
    return [t.results() for t in T]


def _tables14(tables):
    """the tables14 array of a store trace: an (nslots, 14) array as it is, or one row per slot from (KRKi, Kt, aff), None for a slot
    without points (zeros)"""
    if isinstance(tables, np.ndarray):
        return np.ascontiguousarray(tables, np.float32).reshape(-1, 14)
    tab = np.zeros((len(tables), 14), np.float32)
    for k, t in enumerate(tables):
        if t is not None:
            KRKi, Kt, aff = t
            tab[k, :9] = np.asarray(KRKi, np.float32).reshape(-1); tab[k, 9:12] = Kt; tab[k, 12:14] = aff
    return tab


# the per-point outputs of dmv_new_traces_args: per-point shape and dtype
_NT_SHAPES = {"u": ((), np.int32), "v": ((), np.int32), "type": ((), np.float32), "color": ((8,), np.float32), "weights": ((8,), np.float32),
              "gradH": ((4,), np.float32), "energyTH": ((), np.float32)}

IP_OUT_KEYS = ("idepth_min", "idepth_max", "quality", "status", "lastTraceUV", "lastTracePixelInterval")


class IPStore:
    """a dmv_ip_store: the immature points of up to 64 host keyframes (slot k = one keyframe's list) kept on one device between frames.
    counts mirrors the store's points per slot.  L: the library, as CT takes it."""

    SLOTS = 64

    def __init__(self, device=0, L=None):
        self.L = L or lib()
        self.h = vp()
        check(self.L.dmv_ip_store_create(device, C.byref(self.h)), self.L)
        self.counts = [0] * self.SLOTS

    def _check(self, rc):
        check(rc, self.L)

    def close(self):
        if self.h:
            self.L.dmv_ip_store_destroy(self.h)
            self.h = vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def put(self, slot, P):
        """the slot's points become P (a dict of arrays as oracle.orc.ip_init returns, in/out fields included); an empty P empties it"""
        T = _TraceSets([(P, np.zeros(9), np.zeros(3), np.zeros(2))])
        self._check(self.L.dmv_ip_store_put(self.h, slot, C.byref(T.arr[0])))
        self.counts[slot] = len(P["u"])

    def get(self, slot, P=None):
        """the slot's in/out fields (IP_OUT_KEYS): a dict of them, or dict(P) updated with them"""
        n = self.counts[slot]
        out = {"idepth_min": np.zeros(n, np.float32), "idepth_max": np.zeros(n, np.float32), "quality": np.zeros(n, np.float32),
               "status": np.zeros(n, np.int32), "lastTraceUV": np.zeros((n, 2), np.float32), "lastTracePixelInterval": np.zeros(n, np.float32)}
        pts = IPPoints(n, *([None] * 6), *[out[k].ctypes.data for k in IP_OUT_KEYS])
        self._check(self.L.dmv_ip_store_get(self.h, slot, C.byref(pts)))
        Q = dict(P) if P is not None else {}
        Q.update(out)
        return Q

    def remove(self, slot, idx):
        """activatePointsMT's removal of the slot's points idx (FullSystem.cpp:L761-769); returns each survivor's index before the call, in
        the slot's new order"""
        idx = np.ascontiguousarray(idx, np.int32)
        order = np.zeros(max(self.counts[slot] - len(idx), 0), np.int32)
        self._check(self.L.dmv_ip_store_remove(self.h, slot, len(idx), idx.ctypes.data if len(idx) else None, order.ctypes.data))
        self.counts[slot] -= len(idx)
        return order


def trace_store_many(handles, jobs, settings=None):
    """dmv_ct_trace_store_many: jobs[i] = (store, tables) (an IPStore, and tables as CT.trace_store takes them, nslots = len(tables)) traced
    against handles[i]'s frame, all in one launch"""
    if len(handles) != len(jobs):
        raise ValueError(f"{len(handles)} handles but {len(jobs)} jobs")
    n = len(handles)
    L = handles[0].L if handles else lib()
    tabs = [_tables14(t) for _, t in jobs]
    H = (vp * max(n, 1))(*[g.h.value for g in handles])
    J = (TraceStoreJob * max(n, 1))(*[TraceStoreJob(st.h.value, len(tb), tb.ctypes.data if len(tb) else None) for (st, _), tb in zip(jobs, tabs)])
    check(L.dmv_ct_trace_store_many(H, n, J, None if settings is None else C.byref(settings)), L)


class CT:
    """a dmv_ct handle.  L: the library it lives in, lib() by default or another build from load()"""

    def __init__(self, w, h, levels, max_points=65536, device=0, L=None):
        self.L = L or lib()
        cfg = CTConfig(w, h, levels, max_points, device)
        self.h = vp()
        self._check(self.L.dmv_ct_create(C.byref(cfg), C.byref(self.h)))
        self.levels = levels
        self.size = (w, h)

    def _check(self, rc):
        check(rc, self.L)

    def close(self):
        if self.h:
            self.L.dmv_ct_destroy(self.h)
            self.h = vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_K(self, lvl, fx, fy, cx, cy):
        self._check(self.L.dmv_ct_set_K(self.h, lvl, fx, fy, cx, cy))

    def set_ref(self, lvl, u, v, idepth, color):
        self._check(self.L.dmv_ct_set_ref(self.h, lvl, len(u), _c(u, np.float32), _c(v, np.float32), _c(idepth, np.float32), _c(color, np.float32)))

    def upload_new(self, lvl, dIp):
        self._check(self.L.dmv_ct_upload_new(self.h, lvl, _c(dIp, np.float32).reshape(-1)))

    def upload_new_image(self, img):
        self._check(self.L.dmv_ct_upload_new_image(self.h, _c(img, np.float32).reshape(-1)))

    def set_huber(self, th):
        self._check(self.L.dmv_ct_set_huber(self.h, th))

    def set_undistort(self, wOrg, hOrg, remapX=None, remapY=None, G=None, vignetteInv=None, photometric_mode=0):
        """dmv_ct_set_undistort: the per-sequence tables of Undistort (remapX/remapY None = passthrough, G None = no photometric calibration)"""
        keep = [None if a is None else _c(a, np.float32).reshape(-1) for a in (remapX, remapY, G, vignetteInv)]
        p = [None if a is None else a.ctypes.data for a in keep]
        cfg = UndistortConfig(int(wOrg), int(hOrg), p[0], p[1], p[2], 0 if G is None else len(keep[2]), p[3], int(photometric_mode))
        self._check(self.L.dmv_ct_set_undistort(self.h, C.byref(cfg)))

    def upload_raw_image(self, raw, exposure=1.0, factor=None):
        """dmv_ct_upload_raw_image: a uint8 or uint16 frame of the raw size; factor defaults to the reference's readers' (1, or 1/256 for 16 bit)"""
        raw = np.ascontiguousarray(raw)
        if raw.dtype not in (np.uint8, np.uint16):
            raise DmvError("raw frames are uint8 or uint16")
        if factor is None:
            factor = 1.0 if raw.itemsize == 1 else 1.0 / 256
        self._check(self.L.dmv_ct_upload_raw_image(self.h, raw.ctypes.data, raw.itemsize, float(exposure), float(factor)))

    def download_frame(self, lvl, w, h):
        """dmv_ct_download_frame: dIp[lvl] as an (h_l, w_l, 3) array (w, h = level-0 size)"""
        out = np.zeros(((h >> lvl) * (w >> lvl) * 3), np.float32)
        self._check(self.L.dmv_ct_download_frame(self.h, lvl, out))
        return out.reshape(h >> lvl, w >> lvl, 3)

    def calc_res_gs(self, lvl, RKi, t, affLL, b0, cutoff, want_gs=True):
        res6 = np.zeros(6); H = np.zeros(64); b = np.zeros(8); n = C.c_int(0)
        self._check(self.L.dmv_ct_calc_res_gs(self.h, lvl, _c(RKi, np.float32).reshape(-1), _c(t, np.float32), _c(affLL, np.float32), b0, cutoff,
                                        int(want_gs), res6, H, b, C.byref(n)))
        return res6, H.reshape(8, 8), b, n.value

    def track(self, R, t, a, b, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0, cutoff=20.0, affA=1e12, affB=1e8, coarsest=None,
              minRes=None):
        """dmv_ct_track (trackNewestCoarse in one launch): every field of dmv_ct_track_result as a dict, status and evaluations included.
        minRes = minResForAbort (None: NaN, never abort); coarsest defaults to the handle's top level."""
        A = _track_args(self.levels, R, t, a, b, ref_a, ref_b, ref_exposure, new_exposure, cutoff, affA, affB, coarsest, minRes)
        r = CTTrackResult()
        self._check(self.L.dmv_ct_track(self.h, C.byref(A), C.byref(r)))
        return _track_result(r)

    def track_tries(self, R, t, a, b, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0, cutoff=20.0, affA=1e12, affB=1e8, coarsest=None,
                    lastCoarseRMSE0=100.0, reTrackThreshold=1.5):
        """dmv_ct_track_tries (FullSystem::trackNewCoarse's loop over the tries R[i], t[i] in one launch): every field of
        dmv_ct_tries_result as a dict (flowIndicators as "flow" and trackingGood as "good", as CT.track names them).  a, b = aff_last_2_l."""
        A, keep = _tries_args(self.levels, R, t, a, b, ref_a, ref_b, ref_exposure, new_exposure, cutoff, affA, affB, coarsest, lastCoarseRMSE0,
                              reTrackThreshold)
        r = CTTriesResult()
        self._check(self.L.dmv_ct_track_tries(self.h, C.byref(A), C.byref(r)))
        return _tries_result(r)

    def point_evaluations(self):
        """reference points evaluated by the last track, summed over its evaluations (dmv_ct_last_point_evaluations)"""
        n = C.c_double(0)
        self._check(self.L.dmv_ct_last_point_evaluations(self.h, C.byref(n)))
        return n.value

    def make_coarse_depth(self, Ku, Kv, new_idepth, HdiF):
        """makeCoarseDepthL0 on the device with the resident frame as the reference; returns pc_n per level"""
        pc_n = np.zeros(8, np.int32)
        self._check(self.L.dmv_ct_make_coarse_depth(self.h, len(Ku), _c(Ku, np.float32), _c(Kv, np.float32), _c(new_idepth, np.float32), _c(HdiF, np.float32), pc_n))
        return pc_n

    def set_ref_from_ba(self, ba):
        """setCoarseTrackingRef + makeCoarseDepthL0 from a BA handle on the same device (dmv_ct_set_ref_from_ba): the window's newest frame becomes
        the reference.  ba: a BA, or a raw dmv_ba* (e.g. hostapi.WindowBA.ba_handle()).  Returns pc_n per level."""
        pc_n = np.zeros(8, np.int32)
        self._check(self.L.dmv_ct_set_ref_from_ba(self.h, ba.h if isinstance(ba, BA) else ba, pc_n))
        return pc_n

    def get_ref(self, lvl):
        n = C.c_int(0)
        self._check(self.L.dmv_ct_get_ref(self.h, lvl, C.byref(n), None, None, None, None))
        a = [np.zeros(n.value, np.float32) for _ in range(4)]
        self._check(self.L.dmv_ct_get_ref(self.h, lvl, C.byref(n), *[x.ctypes.data for x in a]))
        return dict(u=a[0], v=a[1], idepth=a[2], color=a[3])

    def _ps_settings(self, settings):
        if settings is None:
            return None
        S = PSSettings()
        self.L.dmv_ps_default_settings(C.byref(S))
        for k, val in settings.items():
            setattr(S, k, val)
        return S

    def make_new_traces_store(self, store, slot, potential, density=1500.0, recursionsLeft=1, thFactor=1.0, B=None, settings=None, want=("type",),
                              cap=16384, want_map=False):
        """FullSystem::makeNewTraces with the new points put straight into slot `slot` of store, an IPStore (dmv_ct_make_new_traces_store);
        store.counts follows.  want: the per-point outputs to read back from the slot, keys of make_new_traces' points (u, v, type, color,
        weights, gradH, energyTH); with none, cap does not apply.  Returns dict(points (the wanted ones), n, numPointsTotal, potential (after),
        map (if want_map)); an overflow raises DmvError and sets last_needed, as make_new_traces does."""
        W, H = self.size
        want = tuple(want)
        bad = [k for k in want if k not in _NT_SHAPES]
        if bad:
            raise ValueError(f"unknown outputs {bad}")
        cap = int(cap) if want else 0
        pot, n, npt = C.c_int(int(potential)), C.c_int(0), C.c_int(0)
        P = {k: np.zeros((max(cap, 1),) + _NT_SHAPES[k][0], _NT_SHAPES[k][1]) for k in want}
        m = np.zeros(W * H, np.float32) if want_map else None
        Bk = None if B is None else _c(B, np.float32)
        S = self._ps_settings(settings)
        ptr = lambda k: P[k].ctypes.data if k in P else None  # noqa: E731
        a = NewTracesArgs(float(density), int(recursionsLeft), float(thFactor), None if Bk is None else Bk.ctypes.data,
                          None if S is None else C.addressof(S), C.pointer(pot), cap, C.pointer(n), C.pointer(npt), ptr("u"), ptr("v"), ptr("type"),
                          ptr("color"), ptr("weights"), ptr("gradH"), ptr("energyTH"), None if m is None else m.ctypes.data)
        rc = self.L.dmv_ct_make_new_traces_store(self.h, store.h, int(slot), C.byref(a))
        self.last_needed, self.last_potential = n.value, pot.value
        self._check(rc)
        store.counts[slot] = n.value
        out = dict(points={k: P[k][:n.value] for k in P}, n=n.value, numPointsTotal=npt.value, potential=pot.value)
        if want_map:
            out["map"] = m.reshape(H, W)
        return out

    def make_new_traces(self, potential, density=1500.0, recursionsLeft=1, thFactor=1.0, B=None, settings=None, cap=16384, want_map=False):
        """FullSystem::makeNewTraces on the resident frame (dmv_ct_make_new_traces).  potential: the selector's currentPotential before the call.
        cap: point capacity (the default is ten times the default density; an overflow raises DmvError and sets last_needed).
        Returns dict(points (u, v, type, color, weights, gradH, energyTH), numPointsTotal, potential (after), map (if want_map))."""
        W, H = self.size
        cap = int(cap)
        pot, n, npt = C.c_int(int(potential)), C.c_int(0), C.c_int(0)
        P = dict(u=np.zeros(max(cap, 1), np.int32), v=np.zeros(max(cap, 1), np.int32), type=np.zeros(max(cap, 1), np.float32),
                 color=np.zeros((max(cap, 1), 8), np.float32), weights=np.zeros((max(cap, 1), 8), np.float32), gradH=np.zeros((max(cap, 1), 4), np.float32),
                 energyTH=np.zeros(max(cap, 1), np.float32))
        m = np.zeros(W * H, np.float32) if want_map else None
        Bk = None if B is None else _c(B, np.float32)
        S = self._ps_settings(settings)
        a = NewTracesArgs(float(density), int(recursionsLeft), float(thFactor), None if Bk is None else Bk.ctypes.data,
                          None if S is None else C.addressof(S), C.pointer(pot), cap, C.pointer(n), C.pointer(npt), P["u"].ctypes.data, P["v"].ctypes.data,
                          P["type"].ctypes.data, P["color"].ctypes.data, P["weights"].ctypes.data, P["gradH"].ctypes.data, P["energyTH"].ctypes.data,
                          None if m is None else m.ctypes.data)
        rc = self.L.dmv_ct_make_new_traces(self.h, C.byref(a))
        self.last_needed, self.last_potential = n.value, pot.value
        self._check(rc)
        out = dict(points={k: P[k][:n.value] for k in P}, numPointsTotal=npt.value, potential=pot.value)
        if want_map:
            out["map"] = m.reshape(H, W)
        return out

    def init_points(self, u, v):
        """ImmaturePoint constructor on the resident frame; same dict layout as oracle.orc.ip_init."""
        n = len(u)
        P = dict(u=_c(u, np.float32), v=_c(v, np.float32), color=np.zeros((n, 8), np.float32), weights=np.zeros((n, 8), np.float32),
                 gradH=np.zeros((n, 4), np.float32), energyTH=np.zeros(n, np.float32))
        ok = np.zeros(n, np.int32)
        self._check(self.L.dmv_ct_init_points(self.h, n, _c(u, np.int32), _c(v, np.int32), P["color"].reshape(-1), P["weights"].reshape(-1), P["gradH"].reshape(-1),
                                        P["energyTH"], ok))
        P["ok"] = ok.astype(np.uint8)
        P.update(idepth_min=np.zeros(n, np.float32), idepth_max=np.full(n, np.nan, np.float32), quality=np.full(n, 10000, np.float32),
                 status=np.full(n, 5, np.int32), lastTraceUV=np.zeros((n, 2), np.float32), lastTracePixelInterval=np.zeros(n, np.float32))
        return P

    def trace_points(self, P, KRKi, Kt, aff, settings=None):
        """ImmaturePoint::traceOn for the points of one host frame (dict of arrays as oracle.orc.ip_init returns) against the resident newest
        frame; returns a dict with the updated in/out fields (P itself is not modified).  settings: an IPSettings, or None (NULL: defaults)."""
        n = len(P["u"])
        keep = {k: _c(P[k], np.float32) for k in ("u", "v", "color", "weights", "gradH", "energyTH")}
        out = {"idepth_min": np.array(P["idepth_min"], np.float32, copy=True), "idepth_max": np.array(P["idepth_max"], np.float32, copy=True),
               "quality": np.array(P["quality"], np.float32, copy=True), "status": np.array(P["status"], np.int32, copy=True),
               "lastTraceUV": np.array(P["lastTraceUV"], np.float32, copy=True), "lastTracePixelInterval": np.array(P["lastTracePixelInterval"], np.float32, copy=True)}
        pts = IPPoints(n, *[a.ctypes.data for a in (keep["u"], keep["v"], keep["color"], keep["weights"], keep["gradH"], keep["energyTH"], out["idepth_min"],
                                                     out["idepth_max"], out["quality"], out["status"], out["lastTraceUV"], out["lastTracePixelInterval"])])
        self._check(self.L.dmv_ct_trace_points(self.h, C.byref(pts), _c(KRKi, np.float32).reshape(-1), _c(Kt, np.float32), _c(aff, np.float32),
                                              None if settings is None else C.byref(settings)))
        Q = dict(P)
        Q.update(out)
        return Q

    def trace_points_multi(self, sets, settings=None):
        """sets = [(P, KRKi, Kt, aff), ...]: the immature points of several host keyframes in ONE launch (dmv_ct_trace_points_multi);
        returns the list of updated dicts.  settings: an IPSettings, or None (NULL: defaults)."""
        T = _TraceSets(sets)
        self._check(self.L.dmv_ct_trace_points_multi(self.h, T.job.nsets, T.job.sets, T.job.tables14, None if settings is None else C.byref(settings)))
        return T.results()

    def trace_store(self, store, tables, settings=None):
        """dmv_ct_trace_store: the points of store (an IPStore) traced against the resident newest frame, slot k with tables[k] (an
        (nslots, 14) array, or (KRKi, Kt, aff) per slot with None for an empty slot; nslots = len(tables))"""
        tab = _tables14(tables)
        self._check(self.L.dmv_ct_trace_store(self.h, store.h, len(tab), tab.ctypes.data if len(tab) else None, None if settings is None else C.byref(settings)))

    def set_timing(self, enable=True):
        self._check(self.L.dmv_ct_set_timing(self.h, int(enable)))

    def last_timing(self):
        ms = np.zeros(4, np.float32)
        self._check(self.L.dmv_ct_last_timing(self.h, ms))
        return ms

    def launch_count(self):
        n = C.c_longlong(0)
        self._check(self.L.dmv_ct_kernel_launch_count(self.h, C.byref(n)))
        return n.value


class CI:
    """CoarseInitializer::calcResAndGS on the device (include/dmvio_b200.h, dmv_ci_*)"""

    def __init__(self, w, h, levels, max_points=16384, device=0):
        self.L = lib()
        cfg = CTConfig(w, h, levels, max_points, device)   # dmv_ci_config has the same layout
        self.h = vp()
        check(self.L.dmv_ci_create(C.byref(cfg), C.byref(self.h)))
        self.levels = levels

    def close(self):
        if self.h:
            self.L.dmv_ci_destroy(self.h)
            self.h = vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_K(self, lvl, fx, fy, cx, cy):
        check(self.L.dmv_ci_set_K(self.h, lvl, C.c_float(fx), C.c_float(fy), C.c_float(cx), C.c_float(cy)))

    def upload_first(self, lvl, dIp):
        check(self.L.dmv_ci_upload_first(self.h, lvl, _p(_c(dIp, np.float32).reshape(-1))))

    def upload_new(self, lvl, dIp):
        check(self.L.dmv_ci_upload_new(self.h, lvl, _p(_c(dIp, np.float32).reshape(-1))))

    def set_points(self, lvl, u, v, outlierTH):
        check(self.L.dmv_ci_set_points(self.h, lvl, len(u), _p(_c(u, np.float32)), _p(_c(v, np.float32)), _p(_c(outlierTH, np.float32))))
        self._n = getattr(self, "_n", {})
        self._n[lvl] = len(u)

    def calc_res_and_gs(self, lvl, RKi, t, t_log, r2new_aff, idepth_new, isGood, energy2, iR, huberTH=9.0, alphaK=2.5 * 2.5, alphaW=150.0 * 150.0,
                        couplingWeight=1.0, wzpx=0.0, wzpy=0.0):
        n = self._n[lvl]
        a = CIEvalArgs()
        a.level = lvl
        a.RKi[:] = [float(x) for x in np.asarray(RKi, np.float32).reshape(-1)]
        a.t_d[:] = [float(x) for x in t]
        a.t_log[:] = [float(x) for x in t_log]
        a.r2new_aff[:] = [float(np.float32(x)) for x in r2new_aff]
        a.huberTH, a.alphaK, a.alphaW, a.couplingWeight, a.weightZeroPriorX, a.weightZeroPriorY = huberTH, alphaK, alphaW, couplingWeight, wzpx, wzpy
        ins = [_c(idepth_new, np.float32), _c(isGood, np.uint8), _c(energy2, np.float32).reshape(-1), _c(iR, np.float32)]
        a.idepth_new, a.isGood, a.energy2, a.iR = [x.ctypes.data for x in ins]
        o = dict(isGood_new=np.zeros(n, np.uint8), energy_new=np.zeros((n, 2), np.float32), maxstep=np.zeros(n, np.float32),
                 lastHessian_new=np.zeros(n, np.float32), Jb=np.zeros((n, 10), np.float32))
        a.isGood_new, a.energy_new2, a.maxstep, a.lastHessian_new, a.JbBuffer_new10 = [o[k].ctypes.data for k in ("isGood_new", "energy_new", "maxstep", "lastHessian_new", "Jb")]
        r = CIEvalResult()
        check(self.L.dmv_ci_calc_res_and_gs(self.h, C.byref(a), C.byref(r)))
        o.update(H=np.array(r.H, np.float32).reshape(8, 8), b=np.array(r.b, np.float32), Hsc=np.array(r.Hsc, np.float32).reshape(8, 8),
                 bsc=np.array(r.bsc, np.float32), res=np.array(r.res3, np.float32), alphaOpt=float(r.alphaOpt), n_good_new=int(r.n_good_new))
        return o

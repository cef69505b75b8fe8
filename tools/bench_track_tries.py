#!/usr/bin/env python
"""Latency of FullSystem::trackNewCoarse's try loop (FullSystem.cpp:L412-506, visual-only) on the config-2 scene (640x480, 5 levels, seed
4321: helpers.ct_scene("bench")) with the reference's 31 tries (L364-402), three workloads:
  easy      lastF_2_slast = the true motion, fh_2_slast = identity: try 0 starts at the truth and meets the break test (lastCoarseRMSE0 100)
  recovery  fh_2_slast a 0.1 rad / 0.1 rotation and translation: the constant-motion tries start far off; lastCoarseRMSE0 is set from a
            loop that never breaks so that the loop breaks at the first later try that lowers achievedRes[0] (the first candidate try list
            of test_gpu_track_tries.test_later_winner that has one)
  lost      the recovery tries with ref_b = 250 and aff_last_2_l b = 252: every try converges with |b| > 200, so none is good, nothing aborts
            and all 31 run the whole pyramid (lastCoarseRMSE0 0)
and two arms, each on its own handle loaded the same way:
  host      the loop in Python over dmv_ct_track (one launch and one synchronisation per try; ctypes arguments built once)
  device    one dmv_ct_track_tries
On the easy workload a single dmv_ct_track from try 0 is timed as well (the bar for the call).  The arms alternate within each repetition, in a rotating
order; wall time per call, each ending in a synchronisation.  Outside the timed loop every arm's result must be bit-identical to the host
loop's, or the run exits non-zero.  Reported per arm: median / p10 / p90, tries and point evaluations.
--parent-lib PATH adds an A/B of dmv_ct_track (easy workload, try 0) between this library and another build of it, e.g. the parent commit's,
loaded side by side and alternated call by call; their results must be bit-identical too.  The card's name, power limit and maximum SM clock
are read in the same run (read-only nvidia-smi query).  Prints one JSON line and writes it to --out.
    python tools/bench_track_tries.py [--warmup 30] [--reps 300] [--parent-lib PATH] [--out records/h100_track_tries.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def f32_finite(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return bool(np.isfinite(np.float32(x)))


class HostLoop:
    """L412-506 over dmv_ct_track with prebuilt ctypes arguments; result() is a dmv_ct_tries_result"""

    def __init__(self, capi, L, g, Rs, ts, k, lastCoarseRMSE0, reTrackThreshold=1.5):
        self.L, self.h = L, g.h
        self.A = [capi._track_args(g.levels, R, t, **k) for R, t in zip(Rs, ts)]
        self.out = capi.CTTrackResult()
        self.res = capi.CTTriesResult()
        self.R0, self.t0, self.a0, self.b0 = np.asarray(Rs[0]).reshape(-1), np.asarray(ts[0]), float(k["a"]), float(k["b"])
        self.bound = float(lastCoarseRMSE0) * float(np.float32(reTrackThreshold))
        self.pe = 0.0
        self.pe_c = C.c_double(0)

    def __call__(self):
        L, o = self.L, self.out
        achieved = [float("nan")] * 5
        best = None
        good_ret, tries, self.pe = 0, 0, 0.0
        for i, A in enumerate(self.A):
            A.minResForAbort[:] = achieved
            rc = L.dmv_ct_track(self.h, C.byref(A), C.byref(o))
            if rc != 0:
                return rc
            L.dmv_ct_last_point_evaluations(self.h, C.byref(self.pe_c))
            self.pe += self.pe_c.value
            tries += 1
            good = o.trackingGood != 0
            good_ret |= good
            lr = list(o.lastResiduals)
            if good and f32_finite(lr[0]) and not (lr[0] >= achieved[0]):
                best = (list(o.R), list(o.t), o.a, o.b, list(o.flowIndicators), i)
            if best is not None:
                for q in range(5):
                    if not f32_finite(achieved[q]) or achieved[q] > lr[q]:
                        achieved[q] = lr[q]
                if achieved[0] < self.bound:
                    break
        r = self.res
        if best is None:
            r.R[:], r.t[:], r.a, r.b, r.flowVecs[:], r.winner = list(self.R0), list(self.t0), self.a0, self.b0, [0.0] * 3, -1
        else:
            r.R[:], r.t[:], r.a, r.b, r.flowVecs[:], r.winner = best
        r.achievedRes[:], r.lastResiduals[:], r.flowIndicators[:] = achieved, list(o.lastResiduals), list(o.flowIndicators)
        r.trackingGood, r.haveOneGood, r.tries, r.tries_started = int(good_ret), int(best is not None), tries, tries
        return 0


def stats(ts):
    ms = 1e3 * np.asarray(ts)
    return dict(median_ms=float(np.median(ms)), p10_ms=float(np.percentile(ms, 10)), p90_ms=float(np.percentile(ms, 90)))


def workloads(capi, T, sc, g):
    """(name, Rs, ts, track keywords, lastCoarseRMSE0)"""
    k = T.kw(sc)
    Rs, ts = T.near_truth_tries(sc)
    out = [("easy", Rs, ts, k, 100.0)]
    twin = T.handle(capi, sc)
    for Rs, ts in [T.far_tries(sc, 0.1), T.near_truth_tries(sc), T.far_tries(sc, 0.05)]:
        _, _, hist = T.loop_reference(twin, Rs, ts, k, lastCoarseRMSE0=0.0)
        found = T.later_winner_L(hist)
        if found is not None:
            out.append(("recovery", Rs, ts, k, found[0]))
            break
    twin.close()
    Rs, ts = T.far_tries(sc, 0.1)
    out.append(("lost", Rs, ts, T.kw(sc, ref_b=250.0, b=252.0), 0.0))
    return out


def parent_ab(capi, T, sc, path, warmup, reps):
    """dmv_ct_track from try 0 of the easy workload through this library and through `path`, alternated call by call"""
    libs = {"this": C.CDLL(capi.LIB_PATH), "parent": C.CDLL(os.path.abspath(path))}
    for P in libs.values():
        P.dmv_ct_create.argtypes = [C.POINTER(capi.CTConfig), C.POINTER(C.c_void_p)]
        P.dmv_ct_set_K.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float]
        P.dmv_ct_set_ref.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        P.dmv_ct_upload_new.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        P.dmv_ct_track.argtypes = [C.c_void_p, C.POINTER(capi.CTTrackArgs), C.POINTER(capi.CTTrackResult)]
        P.dmv_ct_destroy.argtypes = [C.c_void_p]
    hs = {}
    keep = []
    for name, L in libs.items():
        h = C.c_void_p()
        assert L.dmv_ct_create(C.byref(capi.CTConfig(sc["w"], sc["h"], sc["levels"], 65536, 0)), C.byref(h)) == 0
        for l in range(sc["levels"]):
            assert L.dmv_ct_set_K(h, l, *[float(x) for x in sc["k4"][l]]) == 0
            p = {q: np.ascontiguousarray(sc["pts"][l][q], np.float32) for q in ("u", "v", "idepth", "color")}
            plane = np.ascontiguousarray(sc["planes"][l], np.float32).reshape(-1)
            keep += list(p.values()) + [plane]
            assert L.dmv_ct_set_ref(h, l, len(p["u"]), p["u"].ctypes.data, p["v"].ctypes.data, p["idepth"].ctypes.data, p["color"].ctypes.data) == 0
            assert L.dmv_ct_upload_new(h, l, plane.ctypes.data) == 0
        hs[name] = h
    Rs, ts = T.near_truth_tries(sc)
    A = capi._track_args(sc["levels"], Rs[0], ts[0], **T.kw(sc))
    outs = {k: capi.CTTrackResult() for k in libs}
    t = {k: [] for k in libs}
    names = list(libs)
    for rep in range(warmup + reps):
        for j in range(2):
            k = names[(rep + j) % 2]
            t0 = time.perf_counter()
            rc = libs[k].dmv_ct_track(hs[k], C.byref(A), C.byref(outs[k]))
            dt = time.perf_counter() - t0
            if rc != 0:
                raise SystemExit(f"dmv_ct_track through {k}: error {rc}")
            if rep >= warmup:
                t[k].append(dt)
    same = bytes(outs["this"]) == bytes(outs["parent"])
    for k, L in libs.items():
        L.dmv_ct_destroy(hs[k])
    return dict(parent_lib=os.path.basename(path), bit_identical=same, **{k: stats(t[k]) for k in libs}), same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--parent-lib", default=None, help="another build of libdmvio_b200.so for the dmv_ct_track A/B")
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_track_tries.json"))
    a = ap.parse_args()
    os.environ.pop("DMV_CT_CLUSTER", None)
    import dmvio_b200.capi as capi
    import dmvio_b200.synth as synth
    import helpers as H
    import test_gpu_track_tries as T
    from oracle import orc
    L = capi.lib()
    if L.dmv_device_count() < 1:
        raise SystemExit("bench_track_tries needs a CUDA device")
    sc = H.ct_scene(orc, synth, "bench")
    gs = {arm: T.handle(capi, sc) for arm in ("host", "device")}
    res = dict(card=card(), shape=[sc["w"], sc["h"]], levels=sc["levels"], tries=31, warmup=a.warmup, reps=a.reps,
               timing="wall clock per call, each call ending in a synchronisation; ctypes argument blocks built once", workloads={})
    identical = True
    for name, Rs, ts, k, Lc in workloads(capi, T, sc, gs["host"]):
        host = HostLoop(capi, L, gs["host"], Rs, ts, k, Lc)
        targs, keep = capi._tries_args(sc["levels"], Rs, ts, lastCoarseRMSE0=Lc, **k)
        out = capi.CTTriesResult()
        arms = dict(host=host, device=lambda: L.dmv_ct_track_tries(gs["device"].h, C.byref(targs), C.byref(out)))
        if name == "easy":
            A0, o0 = capi._track_args(sc["levels"], Rs[0], ts[0], **k), capi.CTTrackResult()
            arms["single"] = lambda: L.dmv_ct_track(gs["host"].h, C.byref(A0), C.byref(o0))
        names = list(arms)
        t = {q: [] for q in names}
        for rep in range(a.warmup + a.reps):
            for j in range(len(names)):
                q = names[(rep + j) % len(names)]
                t0 = time.perf_counter()
                rc = arms[q]()
                dt = time.perf_counter() - t0
                if rc != 0:
                    raise SystemExit(f"{q} on {name}: dmvio_b200 error {rc}: {L.dmv_last_error().decode()}")
                if rep >= a.warmup:
                    t[q].append(dt)
        # identity and counts, outside the timed loop: one more call of each arm
        row = dict(lastCoarseRMSE0=Lc)
        for q in ("host", "device"):
            arms[q]()
            r = host.res if q == "host" else out
            row[q] = dict(stats(t[q]), tries=r.tries, point_evaluations=host.pe if q == "host" else gs[q].point_evaluations())
        row.update(winner=host.res.winner, haveOneGood=host.res.haveOneGood)
        same = bytes(out) == bytes(host.res) and row["device"]["point_evaluations"] == row["host"]["point_evaluations"]
        row["bit_identical"] = same
        identical = identical and same
        if name == "easy":
            row["single"] = stats(t["single"])
            row["device_over_single"] = row["device"]["median_ms"] / row["single"]["median_ms"]
        row["device_over_host"] = row["device"]["median_ms"] / row["host"]["median_ms"]
        res["workloads"][name] = row
    if a.parent_lib:
        res["track_vs_parent"], same = parent_ab(capi, T, sc, a.parent_lib, a.warmup, a.reps)
        identical = identical and same
    res["bit_identical"] = identical
    for g in gs.values():
        g.close()
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    open(a.out, "w").write(line + "\n")
    if not identical:
        raise SystemExit("the arms returned different results")


if __name__ == "__main__":
    main()

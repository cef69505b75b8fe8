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

import numpy as np

import benchkit as K
import gpu_harness as G


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
            if good and G.f32_finite(lr[0]) and not (lr[0] >= achieved[0]):
                best = (list(o.R), list(o.t), o.a, o.b, list(o.flowIndicators), i)
            if best is not None:
                for q in range(5):
                    if not G.f32_finite(achieved[q]) or achieved[q] > lr[q]:
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


def workloads(capi, sc, g):
    """(name, Rs, ts, track keywords, lastCoarseRMSE0)"""
    k = G.tries_kw(sc)
    Rs, ts = G.near_truth_tries(sc)
    out = [("easy", Rs, ts, k, 100.0)]
    twin = G.ct_handle(capi, sc)
    for Rs, ts in [G.far_tries(sc, 0.1), G.near_truth_tries(sc), G.far_tries(sc, 0.05)]:
        _, _, hist = G.loop_reference(twin, Rs, ts, k, lastCoarseRMSE0=0.0)
        found = G.later_winner_L(hist)
        if found is not None:
            out.append(("recovery", Rs, ts, k, found[0]))
            break
    twin.close()
    Rs, ts = G.far_tries(sc, 0.1)
    out.append(("lost", Rs, ts, G.tries_kw(sc, ref_b=250.0, b=252.0), 0.0))
    return out


def parent_ab(capi, sc, path, warmup, reps):
    """dmv_ct_track from try 0 of the easy workload through this library and through `path`, alternated call by call"""
    libs = K.this_and_parent(path)
    gs = {k: G.ct_handle(capi, sc, L=L) for k, L in libs.items()}
    Rs, ts = G.near_truth_tries(sc)
    A = capi._track_args(sc["levels"], Rs[0], ts[0], **G.tries_kw(sc))
    outs = {k: capi.CTTrackResult() for k in libs}
    arms = {k: (lambda k=k: libs[k].dmv_ct_track(gs[k].h, C.byref(A), C.byref(outs[k]))) for k in libs}
    t = K.alternate(arms, warmup, reps, "dmv_ct_track A/B", libs)
    same = bytes(outs["this"]) == bytes(outs["parent"])
    G.close(*gs.values())
    return dict(parent_lib=os.path.basename(path), bit_identical=same, **{k: K.stats(t[k]) for k in libs}), same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--parent-lib", default=None, help="another build of libdmvio_b200.so for the dmv_ct_track A/B")
    ap.add_argument("--out", default=os.path.join(K.ROOT, "records", "h100_track_tries.json"))
    a = ap.parse_args()
    os.environ.pop("DMV_CT_CLUSTER", None)
    import dmvio_b200.capi as capi
    import dmvio_b200.synth as synth
    from oracle import orc
    L = K.device_lib("bench_track_tries")
    sc = G.ct_scene(orc, synth, "bench")
    gs = {arm: G.ct_handle(capi, sc) for arm in ("host", "device")}
    res = dict(card=K.card(), shape=[sc["w"], sc["h"]], levels=sc["levels"], tries=31, warmup=a.warmup, reps=a.reps,
               timing="wall clock per call, each call ending in a synchronisation; ctypes argument blocks built once", workloads={})
    identical = True
    for name, Rs, ts, k, Lc in workloads(capi, sc, gs["host"]):
        host = HostLoop(capi, L, gs["host"], Rs, ts, k, Lc)
        targs, keep = capi._tries_args(sc["levels"], Rs, ts, lastCoarseRMSE0=Lc, **k)
        out = capi.CTTriesResult()
        arms = dict(host=host, device=lambda: L.dmv_ct_track_tries(gs["device"].h, C.byref(targs), C.byref(out)))
        if name == "easy":
            A0, o0 = capi._track_args(sc["levels"], Rs[0], ts[0], **k), capi.CTTrackResult()
            arms["single"] = lambda: L.dmv_ct_track(gs["host"].h, C.byref(A0), C.byref(o0))
        t = K.alternate(arms, a.warmup, a.reps, f"on {name}", dict.fromkeys(arms, L))
        # identity and counts, outside the timed loop: one more call of each arm
        row = dict(lastCoarseRMSE0=Lc)
        for q in ("host", "device"):
            arms[q]()
            r = host.res if q == "host" else out
            row[q] = dict(K.stats(t[q]), tries=r.tries, point_evaluations=host.pe if q == "host" else gs[q].point_evaluations())
        row.update(winner=host.res.winner, haveOneGood=host.res.haveOneGood)
        same = bytes(out) == bytes(host.res) and row["device"]["point_evaluations"] == row["host"]["point_evaluations"]
        row["bit_identical"] = same
        identical = identical and same
        if name == "easy":
            row["single"] = K.stats(t["single"])
            row["device_over_single"] = row["device"]["median_ms"] / row["single"]["median_ms"]
        row["device_over_host"] = row["device"]["median_ms"] / row["host"]["median_ms"]
        res["workloads"][name] = row
    if a.parent_lib:
        res["track_vs_parent"], same = parent_ab(capi, sc, a.parent_lib, a.warmup, a.reps)
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

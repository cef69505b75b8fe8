#!/usr/bin/env python
"""Immature-point tracing with the points resident on the device (dmv_ip_store, dmv_ct_trace_store, dmv_ct_trace_store_many) against
tracing from host arrays, for one host thread that serves B camera streams.  Every stream has bench_trace_many.py's scene: 640x480, 6 host
keyframes x 1500 immature points.

  tracing     B in {1, 2, 4, 8, 16}: B Python threads each calling dmv_ct_trace_points_multi, one dmv_ct_trace_many, one
              dmv_ct_trace_store_many; at B = 1 also dmv_ct_trace_points_multi and dmv_ct_trace_store.  Every arm starts each round from
              the same fresh points, reset outside the timed call (the stores by dmv_ip_store_put of every slot).
  cycle       B in {1, 4, 16}: the visual-only frame cycle per round: B asynchronous dmv_ct_upload_raw_image, one dmv_ct_track_tries_many
              (bench_track_tries_many.py's easy workload), then one dmv_ct_trace_many or one dmv_ct_trace_store_many.
  turnover    one stream's keyframe turnover on the store: dmv_ip_store_get of the 6 slots, dmv_ip_store_remove of 10 % of each slot's
              points, dmv_ip_store_put of one new slot of 1500 points; beside it the dmv_ct_trace_many (B = 1) of one frame that the store
              saves, and dmv_ct_trace_store of one frame.
  parent      with --parent-lib PATH: dmv_ct_trace_points_multi (B = 1) and dmv_ct_trace_many (B = 4) through this library and through
              another build (e.g. the parent commit's), loaded side by side and alternated call by call.

Every round ends in a synchronisation (each call returns after one).  Arms alternate within each repetition, in a rotating order
(benchkit.alternate); reported per arm: median / p10 / p90 wall time per round.  Outside the timed loops the arms' results must be
bit-identical, or the run exits non-zero.  The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line
and writes it to --out.
    python tools/bench_trace_store.py [--warmup 30] [--reps 300] [--parent-lib PATH] [--out records/h100_trace_store.json]"""
import argparse
import ctypes as C
import json
import os

import numpy as np

import bench_trace_many as TM
import bench_track_tries_many as TT
import benchkit as K

BS = [1, 2, 4, 8, 16]
CYCLE_BS = [1, 4, 16]
HOSTS = TM.HOSTS


class Stores:
    """one IPStore per scene, the ctypes jobs of dmv_ct_trace_store_many, and the reset that puts every slot's fresh points back"""

    def __init__(self, capi, scenes):
        self.fresh = [[P for P, *_ in sets] for _, sets in scenes]
        self.st = [capi.IPStore() for _ in scenes]
        self.tabs = [capi._tables14([tuple(t) for _, *t in sets]) for _, sets in scenes]
        self.J = (capi.TraceStoreJob * len(scenes))(*[capi.TraceStoreJob(s.h.value, HOSTS, t.ctypes.data) for s, t in zip(self.st, self.tabs)])

    def reset(self):
        for s, Ps in zip(self.st, self.fresh):
            for k, P in enumerate(Ps):
                s.put(k, P)

    def result_bytes(self):
        return [[b"".join(s.get(k)[q].tobytes() for q in sorted(OUT_KEYS)) for k in range(HOSTS)] for s in self.st]

    def close(self):
        for s in self.st:
            s.close()


OUT_KEYS = ("idepth_min", "idepth_max", "quality", "status", "lastTraceUV", "lastTracePixelInterval")   # bench_trace_many.Arm's out keys


def row(t, B, arms):
    r = {k: dict(K.stats(t[k]), points_per_s=B * HOSTS * TM.PTS / K.stats(t[k])["median_ms"] * 1e3) for k in arms}
    return r


def tracing(capi, L, gs, scenes, warmup, reps):
    res, identical = {}, True
    for B in BS:
        hs = (C.c_void_p * B)(*[g.h.value for g in gs[:B]])
        A = {k: TM.Arm(capi, scenes[:B]) for k in ("threads", "many", "multi")}
        S = {k: Stores(capi, scenes[:B]) for k in ("store_many", "store")}
        J = (capi.TraceJob * B)(*[t.job for t in A["many"].T])
        th = TM.Threads(L, [hs[i] for i in range(B)], A["threads"].T)
        arms = dict(threads=th.run, many=lambda: L.dmv_ct_trace_many(hs, B, J, None),
                    store_many=lambda: L.dmv_ct_trace_store_many(hs, B, S["store_many"].J, None))
        if B == 1:
            j0, s0 = A["multi"].T[0].job, S["store"]
            arms["multi"] = lambda: L.dmv_ct_trace_points_multi(hs[0], j0.nsets, j0.sets, j0.tables14, None)
            arms["store"] = lambda: L.dmv_ct_trace_store(hs[0], s0.st[0].h, HOSTS, s0.tabs[0].ctypes.data, None)
        resets = {k: (A[k].reset if k in A else S[k].reset) for k in arms}
        t = K.alternate(arms, warmup, reps, f"tracing at B={B}", dict.fromkeys(arms, L), resets)
        got = {}
        for k in arms:   # one more round of each arm from the fresh points, every in/out array compared byte for byte
            resets[k]()
            arms[k]()
            got[k] = A[k].result_bytes() if k in A else S[k].result_bytes()
        same = all(got[k] == got["many"] for k in arms)
        identical = identical and same
        th.close()
        for s in S.values():
            s.close()
        r = dict(bit_identical=same, points_per_round=B * HOSTS * TM.PTS, **row(t, B, arms))
        r["store_many_over_threads"] = r["store_many"]["median_ms"] / r["threads"]["median_ms"]
        r["store_many_over_many"] = r["store_many"]["median_ms"] / r["many"]["median_ms"]
        res[str(B)] = r
    return res, identical


def cycle(capi, synth, orc, L, scenes, warmup, reps):
    """B raw uploads, dmv_ct_track_tries_many, then tracing from host arrays or from the stores"""
    res, identical = {}, True
    made = [TT.make_handle(capi, synth, orc, i) for i in range(max(CYCLE_BS))]
    for g, _ in made:
        g.set_undistort(TT.W, TT.H)
    raws = [np.clip(np.round(sc["T"]["img_new"]), 0, 255).astype(np.uint8) for _, sc in made]
    for B in CYCLE_BS:
        gs = [g for g, _ in made[:B]]
        hs = (C.c_void_p * B)(*[g.h.value for g in gs])
        tr = [capi._tries_args(TT.LEVELS, Rs, ts, lastCoarseRMSE0=Lc, **k) for Rs, ts, k, Lc in [TT.easy(sc) for _, sc in made[:B]]]
        TA = (capi.CTTriesArgs * B)(*[m[0] for m in tr])
        outs = {k: (capi.CTTriesResult * B)() for k in ("many", "store_many")}
        A = TM.Arm(capi, scenes[:B])
        S = Stores(capi, scenes[:B])
        J = (capi.TraceJob * B)(*[t.job for t in A.T])

        def frame(k, trace):
            for i in range(B):
                rc = L.dmv_ct_upload_raw_image(hs[i], raws[i].ctypes.data, 1, 1.0, 1.0)
                if rc:
                    return rc
            return L.dmv_ct_track_tries_many(hs, B, TA, outs[k]) or trace()

        arms = dict(many=lambda: frame("many", lambda: L.dmv_ct_trace_many(hs, B, J, None)),
                    store_many=lambda: frame("store_many", lambda: L.dmv_ct_trace_store_many(hs, B, S.J, None)))
        resets = dict(many=A.reset, store_many=S.reset)
        t = K.alternate(arms, warmup, reps, f"frame cycle at B={B}", dict.fromkeys(arms, L), resets)
        got = {}
        for k in arms:
            resets[k]()
            arms[k]()
            got[k] = A.result_bytes() if k == "many" else S.result_bytes()
        same = got["many"] == got["store_many"] and all(bytes(outs["many"][i]) == bytes(outs["store_many"][i]) for i in range(B))
        identical = identical and same
        S.close()
        r = dict(bit_identical=same, **{k: dict(K.stats(t[k]), frames_per_s=B / K.stats(t[k])["median_ms"] * 1e3) for k in arms})
        r["store_many_over_many"] = r["store_many"]["median_ms"] / r["many"]["median_ms"]
        res[str(B)] = r
    for g, _ in made:
        g.close()
    return res, identical


def turnover(capi, L, g, scene, warmup, reps):
    """one stream's keyframe turnover on its store, beside the per-frame calls"""
    _, sets = scene
    S = Stores(capi, [scene])
    st = S.st[0]
    rng = np.random.default_rng(7)
    idx = [np.ascontiguousarray(rng.choice(TM.PTS, TM.PTS // 10, replace=False), np.int32) for _ in range(HOSTS)]
    order = np.zeros(TM.PTS, np.int32)
    new = sets[0][0]
    newT = capi._TraceSets([(new, np.zeros(9), np.zeros(3), np.zeros(2))])
    outs = [{"idepth_min": np.zeros(TM.PTS, np.float32), "idepth_max": np.zeros(TM.PTS, np.float32), "quality": np.zeros(TM.PTS, np.float32),
             "status": np.zeros(TM.PTS, np.int32), "lastTraceUV": np.zeros((TM.PTS, 2), np.float32), "lastTracePixelInterval": np.zeros(TM.PTS, np.float32)}
            for _ in range(HOSTS)]
    gets = [capi.IPPoints(TM.PTS, *([None] * 6), *[o[k].ctypes.data for k in capi.IP_OUT_KEYS]) for o in outs]

    def turn():
        rc = 0
        for k in range(HOSTS):
            rc = rc or L.dmv_ip_store_get(st.h, k, C.byref(gets[k]))
        for k in range(HOSTS):
            rc = rc or L.dmv_ip_store_remove(st.h, k, len(idx[k]), idx[k].ctypes.data, order.ctypes.data)
        return rc or L.dmv_ip_store_put(st.h, HOSTS, C.byref(newT.arr[0]))

    def reset_turn():
        S.reset()
        L.dmv_ip_store_put(st.h, HOSTS, C.byref(capi.IPPoints()))

    A = TM.Arm(capi, [scene])
    j = A.T[0].job
    h = (C.c_void_p * 1)(g.h.value)
    J = (capi.TraceJob * 1)(j)
    arms = dict(turnover=turn, trace_many=lambda: L.dmv_ct_trace_many(h, 1, J, None),
                trace_store=lambda: L.dmv_ct_trace_store(h[0], st.h, HOSTS, S.tabs[0].ctypes.data, None))
    resets = dict(turnover=reset_turn, trace_many=A.reset, trace_store=reset_turn)
    t = K.alternate(arms, warmup, reps, "keyframe turnover", dict.fromkeys(arms, L), resets)
    S.close()
    return {k: K.stats(t[k]) for k in arms}


def parent(capi, scenes, path, warmup, reps):
    """dmv_ct_trace_points_multi (B = 1) and dmv_ct_trace_many (B = 4) through this library and through `path`, alternated call by call"""
    libs = K.this_and_parent(path)
    gs = {k: [capi.CT(TM.W, TM.H, 5, max_points=1024, L=L) for _ in range(4)] for k, L in libs.items()}
    for k in libs:
        for g, (plane, _) in zip(gs[k], scenes):
            g.upload_new(0, plane)
    res, identical = dict(parent_lib=os.path.basename(path)), True
    for what, B in (("multi", 1), ("many", 4)):
        A = {k: TM.Arm(capi, scenes[:B]) for k in libs}
        hs = {k: (C.c_void_p * B)(*[g.h.value for g in gs[k][:B]]) for k in libs}
        J = {k: (capi.TraceJob * B)(*[t.job for t in A[k].T]) for k in libs}
        if what == "multi":
            arms = {k: (lambda k=k: libs[k].dmv_ct_trace_points_multi(hs[k][0], J[k][0].nsets, J[k][0].sets, J[k][0].tables14, None)) for k in libs}
        else:
            arms = {k: (lambda k=k: libs[k].dmv_ct_trace_many(hs[k], B, J[k], None)) for k in libs}
        t = K.alternate(arms, warmup, reps, f"{what} A/B", libs, {k: A[k].reset for k in libs})
        for k in libs:
            A[k].reset()
            arms[k]()
        same = A["this"].result_bytes() == A["parent"].result_bytes()
        identical = identical and same
        res[f"{what}_B{B}"] = dict(bit_identical=same, **{k: K.stats(t[k]) for k in libs})
    for k in libs:
        for g in gs[k]:
            g.close()
    return res, identical


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--parent-lib", default=None, help="another build of libdmvio_b200.so for the A/B of the existing trace calls")
    ap.add_argument("--out", default=os.path.join(K.ROOT, "records", "h100_trace_store.json"))
    a = ap.parse_args()
    import dmvio_b200.capi as capi
    import dmvio_b200.hostmath as hm
    import dmvio_b200.synth as synth
    from oracle import orc
    L = K.device_lib("bench_trace_store")
    scenes = [TM.make_scene(synth, hm, orc, i) for i in range(max(BS))]
    gs = []
    for plane, _ in scenes:
        g = capi.CT(TM.W, TM.H, 5, max_points=1024)
        g.upload_new(0, plane)
        gs.append(g)
    res = dict(card=K.card(), shape=[TM.W, TM.H], hosts=HOSTS, points_per_host=TM.PTS, warmup=a.warmup, reps=a.reps,
               timing="wall clock per round, each round ending in a synchronisation; points reset outside the timed call")
    res["tracing"], identical = tracing(capi, L, gs, scenes, a.warmup, a.reps)
    res["cycle"], same = cycle(capi, synth, orc, L, scenes, a.warmup, a.reps)
    identical = identical and same
    res["turnover"] = turnover(capi, L, gs[0], scenes[0], a.warmup, a.reps)
    if a.parent_lib:
        res["parent"], same = parent(capi, scenes, a.parent_lib, a.warmup, a.reps)
        identical = identical and same
    res["bit_identical"] = identical
    for g in gs:
        g.close()
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    open(a.out, "w").write(line + "\n")
    if not identical:
        raise SystemExit("the arms returned different results")


if __name__ == "__main__":
    main()

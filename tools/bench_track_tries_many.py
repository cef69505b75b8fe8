#!/usr/bin/env python
"""Throughput of one host thread that serves B visual-only camera streams with FullSystem::trackNewCoarse's try loop (FullSystem.cpp:L412-506):
B coarse-tracker handles of the config-2 shape (640x480, 5 levels; synth.make_tracking_pair with seed 4321 + i, the reference built on the
device by dmv_ct_make_coarse_depth, the new frame uploaded once), each running the reference's 31 tries (L364-402) once per round.
Three workloads, named after bench_track_tries.py's:
  easy      every member easy: try 0 starts at the truth and meets the break test
  recovery  member 0 breaks at the first later try that lowers achievedRes[0] (lastCoarseRMSE0 set from a loop that never breaks), the
            others easy
  lost      member 0 lost: ref_b = 250 and aff_last_2_l b = 252, so no try is good and all 31 run the whole pyramid; the others easy
and three arms:
  seq       B dmv_ct_track_tries calls one after the other on one thread
  threads   B Python threads, one per handle, each calling dmv_ct_track_tries, released together every round (ctypes drops the GIL)
  many      one dmv_ct_track_tries_many call
Every round ends in a synchronisation (each call returns after one).  The arms alternate within each repetition, in a rotating order; the
ctypes argument blocks are built once.  Reported per arm: median / p10 / p90 wall time per round and tracked frames/s.  Outside the timed
loops the three arms must return bit-identical results and point evaluations, or the run exits non-zero.
--parent-lib PATH adds an A/B between this library and another build of it, e.g. the parent commit's, loaded side by side and alternated
call by call: dmv_ct_track (try 0 of the easy workload), dmv_ct_track_many (B = 4, the same), dmv_ct_track_tries (easy) and
dmv_ct_track_tries_many (B = 4, easy); their results must be bit-identical too.  The card's name, power limit and maximum SM clock are read
in the same run (read-only nvidia-smi query).
Prints one JSON line and writes it to --out.
    python tools/bench_track_tries_many.py [--warmup 30] [--reps 300] [--parent-lib PATH] [--out records/h100_track_tries_many.json]"""
import argparse
import ctypes as C
import json
import os
import threading

import numpy as np

import benchkit as K
import gpu_harness as G

BS = [1, 2, 4, 8, 16]
W, H, LEVELS = 640, 480, 5
ARGS = dict(R0=np.eye(3), t0=np.zeros(3), a0=0.0, b0=0.0, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0, affA=1e12, affB=1e8)


def make_handle(capi, synth, orc, i, L=None):
    """stream i's handle and the scene dict gpu_harness's try builders read (its true motion and dmv_ct_track arguments)"""
    T = synth.make_tracking_pair(w=W, h=H, seed=4321 + i, levels=LEVELS)
    oc = orc.CoarseTracker(W, H, T["K"], LEVELS)
    g = capi.CT(W, H, LEVELS, max_points=65536, L=L)
    for l in range(LEVELS):
        g.set_K(l, *[float(x) for x in oc.K(l)[0]])
    g.upload_new_image(T["img_ref"])
    g.make_coarse_depth(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"])
    g.upload_new_image(T["img_new"])
    return g, dict(T=T, args=ARGS, levels=LEVELS)


def easy(sc):
    return (*G.near_truth_tries(sc), G.tries_kw(sc), 100.0)


def recovery(g, sc):
    """bench_track_tries.py's recovery workload for this handle's scene"""
    k = G.tries_kw(sc)
    for Rs, ts in [G.far_tries(sc, 0.1), G.near_truth_tries(sc), G.far_tries(sc, 0.05)]:
        found = G.later_winner_L(G.loop_reference(g, Rs, ts, k, lastCoarseRMSE0=0.0)[2])
        if found is not None:
            return Rs, ts, k, found[0]
    raise SystemExit("no try list of stream 0 improves achievedRes[0] after a first finite try")


def lost(sc):
    return (*G.far_tries(sc, 0.1), G.tries_kw(sc, ref_b=250.0, b=252.0), 0.0)


class Threads:
    """B worker threads, each running its own handle's loop once per round; run() releases them together and returns when all are done"""

    def __init__(self, L, hs, A, R):
        self.L, self.hs, self.A, self.R = L, hs, A, R
        self.go, self.done = threading.Barrier(len(hs) + 1), threading.Barrier(len(hs) + 1)
        self.stop, self.rcs = False, [0] * len(hs)
        self.ts = [threading.Thread(target=self._work, args=(i,), daemon=True) for i in range(len(hs))]
        for t in self.ts:
            t.start()

    def _work(self, i):
        while True:
            self.go.wait()
            if self.stop:
                return
            self.rcs[i] = self.L.dmv_ct_track_tries(self.hs[i], C.byref(self.A[i]), C.byref(self.R[i]))
            self.done.wait()

    def run(self):
        self.go.wait()
        self.done.wait()
        return max(self.rcs, key=abs)

    def close(self):
        self.stop = True
        self.go.wait()
        for t in self.ts:
            t.join()


def one_workload(capi, L, gs, jobs, B, warmup, reps, what):
    """the three arms over the first B handles with jobs[i] = (Rs, ts, keywords, lastCoarseRMSE0); returns the table row"""
    hs = (C.c_void_p * B)(*[g.h.value for g in gs[:B]])
    made = [capi._tries_args(LEVELS, Rs, ts, lastCoarseRMSE0=Lc, **k) for Rs, ts, k, Lc in jobs[:B]]
    A = (capi.CTTriesArgs * B)(*[m[0] for m in made])
    outs = {k: (capi.CTTriesResult * B)() for k in ("seq", "threads", "many")}
    th = Threads(L, [hs[i] for i in range(B)], A, outs["threads"])

    def seq():
        rc = 0
        for i in range(B):
            rc = rc or L.dmv_ct_track_tries(hs[i], C.byref(A[i]), C.byref(outs["seq"][i]))
        return rc

    arms = dict(seq=seq, threads=th.run, many=lambda: L.dmv_ct_track_tries_many(hs, B, A, outs["many"]))
    t = K.alternate(arms, warmup, reps, f"{what} at B={B}", dict.fromkeys(arms, L))
    # identity, outside the timed loops: one more round of each arm, every result struct compared byte for byte, and the point evaluations
    pe = {}
    for k in arms:
        for o in outs[k]:
            C.memset(C.addressof(o), 0, C.sizeof(o))
        arms[k]()
        pe[k] = [g.point_evaluations() for g in gs[:B]]
    th.close()
    same = all(bytes(outs[k][i]) == bytes(outs["many"][i]) for k in ("seq", "threads") for i in range(B)) and pe["seq"] == pe["threads"] == pe["many"]
    row = dict(bit_identical=same, tries=[o.tries for o in outs["many"]], point_evaluations_per_round=sum(pe["many"]))
    for k in arms:
        d = K.stats(t[k])
        row[k] = dict(d, frames_per_s=B / d["median_ms"] * 1e3)
    row["many_over_threads"] = row["many"]["median_ms"] / row["threads"]["median_ms"]
    row["many_over_seq"] = row["many"]["median_ms"] / row["seq"]["median_ms"]
    return row, same


def parent_ab(capi, synth, orc, path, warmup, reps):
    """dmv_ct_track, dmv_ct_track_many (B = 4), dmv_ct_track_tries and dmv_ct_track_tries_many (B = 4) on the easy workload through this
    library and through `path`, alternated call by call"""
    libs = K.this_and_parent(path)
    res, identical = dict(parent_lib=os.path.basename(path)), True
    made = {k: [make_handle(capi, synth, orc, i, L=L) for i in range(4)] for k, L in libs.items()}
    sc = made["this"][0][1]
    Rs, ts, kw, Lc = easy(sc)
    A1 = capi._track_args(LEVELS, Rs[0], ts[0], **kw)
    easies = [easy(s) for _, s in made["this"]]
    A4 = (capi.CTTrackArgs * 4)(*[capi._track_args(LEVELS, R[0], t[0], **kw) for R, t, _, _ in easies])
    At, keep = capi._tries_args(LEVELS, Rs, ts, lastCoarseRMSE0=Lc, **kw)
    made4 = [capi._tries_args(LEVELS, R, t, lastCoarseRMSE0=L_, **k) for R, t, k, L_ in easies]
    At4 = (capi.CTTriesArgs * 4)(*[m[0] for m in made4])
    hs = {k: (C.c_void_p * 4)(*[g.h.value for g, _ in made[k]]) for k in libs}
    outs = {k: dict(track=capi.CTTrackResult(), many=(capi.CTTrackResult * 4)(), tries=capi.CTTriesResult(), tries_many=(capi.CTTriesResult * 4)())
            for k in libs}
    calls = dict(track=lambda k: libs[k].dmv_ct_track(hs[k][0], C.byref(A1), C.byref(outs[k]["track"])),
                 many=lambda k: libs[k].dmv_ct_track_many(hs[k], 4, A4, outs[k]["many"]),
                 tries=lambda k: libs[k].dmv_ct_track_tries(hs[k][0], C.byref(At), C.byref(outs[k]["tries"])),
                 tries_many=lambda k: libs[k].dmv_ct_track_tries_many(hs[k], 4, At4, outs[k]["tries_many"]))
    for name, call in calls.items():
        arms = {k: (lambda k=k, call=call: call(k)) for k in libs}
        t = K.alternate(arms, warmup, reps, f"{name} A/B", libs)
        same = bytes(outs["this"][name]) == bytes(outs["parent"][name])
        identical = identical and same
        res[name] = dict(bit_identical=same, **{k: K.stats(t[k]) for k in libs})
    for k in libs:
        G.close(*[g for g, _ in made[k]])
    return res, identical


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--parent-lib", default=None, help="another build of libdmvio_b200.so for the A/B of the existing tracking calls")
    ap.add_argument("--out", default=os.path.join(K.ROOT, "records", "h100_track_tries_many.json"))
    a = ap.parse_args()
    os.environ.pop("DMV_CT_CLUSTER", None)
    import dmvio_b200.capi as capi
    import dmvio_b200.synth as synth
    from oracle import orc
    L = K.device_lib("bench_track_tries_many")
    made = [make_handle(capi, synth, orc, i) for i in range(max(BS))]
    gs, scs = [m[0] for m in made], [m[1] for m in made]
    easies = [easy(sc) for sc in scs]
    work = dict(easy=easies, recovery=[recovery(gs[0], scs[0])] + easies[1:], lost=[lost(scs[0])] + easies[1:])
    res = dict(card=K.card(), cluster="the probe's choice (DMV_CT_CLUSTER unset)", shape=[W, H], levels=LEVELS, tries=31, warmup=a.warmup, reps=a.reps,
               timing="wall clock per round, each round ending in a synchronisation; ctypes argument blocks built once", workloads={})
    identical = True
    for name, jobs in work.items():
        res["workloads"][name] = {}
        for B in BS:
            row, same = one_workload(capi, L, gs, jobs, B, a.warmup, a.reps, name)
            identical = identical and same
            res["workloads"][name][str(B)] = row
    if a.parent_lib:
        res["vs_parent"], same = parent_ab(capi, synth, orc, a.parent_lib, a.warmup, a.reps)
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

#!/usr/bin/env python
"""Immature-point tracing throughput of one host thread that serves B camera streams: B coarse-tracker handles, each with the scene of
tools/bench_trace.py (640x480, 6 host keyframes x 1500 immature points; synth.make_window with seed 5 + i, points seeded 3 + i), traced
against the newest frame once per round (FullSystem::traceNewCoarse after every tracked frame), three ways:
  seq      B dmv_ct_trace_points_multi calls one after the other on one thread
  threads  B Python threads, one per handle, each calling dmv_ct_trace_points_multi, released together every round
  many     one dmv_ct_trace_many call
Every round ends in a synchronisation (each call returns after one).  The in/out arrays are reset to the same fresh points before every
round, outside the timed call, so each round traces the same work; the ctypes argument blocks are built once.  The arms alternate within
each repetition, in a rotating order.  Reported per arm: median / p10 / p90 wall time per round and traced points/s.  Outside the timed
loops the three arms must return bit-identical results, or the run exits non-zero.

--parent-lib PATH adds an A/B of the single-handle call (one handle, dmv_ct_trace_points_multi) between this library and another build of
it, e.g. the parent commit's, loaded side by side in the same process and alternated call by call; their results must be bit-identical too.
The card's name, power limit and maximum SM clock are read in the same run (read-only nvidia-smi query).  Prints one JSON line and writes
it to --out.
    python tools/bench_trace_many.py [--warmup 30] [--reps 300] [--parent-lib PATH] [--out records/h100_trace_many.json]"""
import argparse
import ctypes as C
import json
import os
import threading

import numpy as np

import benchkit as K

BS = [1, 2, 4, 8, 16]
W, H, HOSTS, PTS = 640, 480, 6, 1500


def make_scene(synth, hm, orc, i):
    """the new frame's level-0 plane and the sets of CT.trace_points_multi for handle i"""
    Wd = synth.make_window(nf=HOSTS + 1, npts=10, seed=5 + i, trans=0.05, rot=0.01)
    rng = np.random.default_rng(3 + i)
    sets = []
    for host in range(HOSTS):
        u, v = rng.integers(10, W - 10, PTS), rng.integers(10, H - 10, PTS)
        sets.append((orc.ip_init(Wd["dI"][host], W, H, u, v),) + tuple(hm.trace_tables(Wd, host, HOSTS)))
    return Wd["dI"][HOSTS], sets


class Arm:
    """one arm's marshalled jobs (capi._TraceSets per handle) and the fresh in/out values each round starts from"""

    def __init__(self, capi, scenes):
        self.T = [capi._TraceSets(sets) for _, sets in scenes]
        self.fresh = [[{k: a.copy() for k, a in out.items()} for out in t.outs] for t in self.T]

    def reset(self):
        for t, fr in zip(self.T, self.fresh):
            for out, f in zip(t.outs, fr):
                for k in out:
                    np.copyto(out[k], f[k])

    def result_bytes(self):
        return [[b"".join(out[k].tobytes() for k in sorted(out)) for out in t.outs] for t in self.T]


class Threads:
    """B worker threads, each tracing its own handle once per round; run() releases them together and returns when all are done"""

    def __init__(self, L, hs, T):
        self.L, self.hs, self.T = L, hs, T
        self.go, self.done = threading.Barrier(len(hs) + 1), threading.Barrier(len(hs) + 1)
        self.stop, self.rcs = False, [0] * len(hs)
        self.ts = [threading.Thread(target=self._work, args=(i,), daemon=True) for i in range(len(hs))]
        for t in self.ts:
            t.start()

    def _work(self, i):
        j = self.T[i].job
        while True:
            self.go.wait()
            if self.stop:
                return
            self.rcs[i] = self.L.dmv_ct_trace_points_multi(self.hs[i], j.nsets, j.sets, j.tables14, None)
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


def stats(t, points):
    d = K.stats(t)
    return dict(d, points_per_s=points / d["median_ms"] * 1e3)


def parent_ab(capi, plane, sets, path, warmup, reps):
    """dmv_ct_trace_points_multi on one handle of this library and one of the library at `path`, alternated call by call"""
    libs = K.this_and_parent(path)
    gs = {}
    for k, L in libs.items():
        gs[k] = capi.CT(W, H, 5, max_points=1024, L=L)
        gs[k].upload_new(0, plane)
    A = {k: Arm(capi, [(None, sets)]) for k in libs}
    arms = {k: (lambda k=k: libs[k].dmv_ct_trace_points_multi(gs[k].h, A[k].T[0].job.nsets, A[k].T[0].job.sets, A[k].T[0].job.tables14, None))
            for k in libs}
    t = K.alternate(arms, warmup, reps, "single-handle A/B", libs, {k: A[k].reset for k in libs})
    for k in libs:
        A[k].reset()
        arms[k]()
    same = A["this"].result_bytes() == A["parent"].result_bytes()
    for g in gs.values():
        g.close()
    return dict(parent_lib=os.path.basename(path), bit_identical=same, **{k: stats(t[k], HOSTS * PTS) for k in libs}), same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--parent-lib", default=None, help="another build of libdmvio_b200.so for the single-handle A/B")
    ap.add_argument("--out", default=os.path.join(K.ROOT, "records", "h100_trace_many.json"))
    a = ap.parse_args()
    import dmvio_b200.capi as capi
    import dmvio_b200.hostmath as hm
    import dmvio_b200.synth as synth
    from oracle import orc
    L = K.device_lib("bench_trace_many")
    scenes = [make_scene(synth, hm, orc, i) for i in range(max(BS))]
    gs = []
    for plane, _ in scenes:
        g = capi.CT(W, H, 5, max_points=1024)
        g.upload_new(0, plane)
        gs.append(g)
    res = dict(card=K.card(), shape=[W, H], hosts=HOSTS, points_per_host=PTS, warmup=a.warmup, reps=a.reps,
               timing="wall clock per round, each round ending in a synchronisation; in/out arrays reset outside the timed call", B={})
    identical = True
    for B in BS:
        hs = (C.c_void_p * B)(*[g.h.value for g in gs[:B]])
        A = {k: Arm(capi, scenes[:B]) for k in ("seq", "threads", "many")}
        J = (capi.TraceJob * B)(*[t.job for t in A["many"].T])
        th = Threads(L, [hs[i] for i in range(B)], A["threads"].T)

        def seq():
            rc = 0
            for i in range(B):
                j = A["seq"].T[i].job
                rc = rc or L.dmv_ct_trace_points_multi(hs[i], j.nsets, j.sets, j.tables14, None)
            return rc

        arms = dict(seq=seq, threads=th.run, many=lambda: L.dmv_ct_trace_many(hs, B, J, None))
        t = K.alternate(arms, a.warmup, a.reps, f"at B={B}", dict.fromkeys(arms, L), {k: A[k].reset for k in arms})
        # identity, outside the timed loops: one more round of each arm from the fresh points, every in/out array compared byte for byte
        for k in arms:
            A[k].reset()
            arms[k]()
        same = A["seq"].result_bytes() == A["many"].result_bytes() == A["threads"].result_bytes()
        identical = identical and same
        th.close()
        res["B"][str(B)] = dict(bit_identical=same, points_per_round=B * HOSTS * PTS, **{k: stats(t[k], B * HOSTS * PTS) for k in arms})
    if a.parent_lib:
        res["single_vs_parent"], same = parent_ab(capi, scenes[0][0], scenes[0][1], a.parent_lib, a.warmup, a.reps)
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

#!/usr/bin/env python
"""Tracking throughput of one host thread that serves B camera streams (a multi-camera rig, several robots on one server, repeated runs of a
sequence): B coarse-tracker handles of the config-2 shape (640x480, 5 levels; synth.make_tracking_pair with seed 4321 + i, the reference
built on the device by dmv_ct_make_coarse_depth, the new frame uploaded once), one frame each per round, three ways:
  seq      B dmv_ct_track calls one after the other on one thread
  threads  B Python threads, one per handle, each calling dmv_ct_track, released together every round (ctypes drops the GIL in the call)
  many     one dmv_ct_track_many call
Every round ends in a synchronisation (each call returns after one).  The arms alternate within each repetition, in a rotating order; the
ctypes argument blocks are built once, so a round times the library calls.  Reported per arm: median / p10 / p90 wall time per round,
tracked frames/s and reference-point evaluations/s (the sum of dmv_ct_last_point_evaluations over the handles).  Outside the timed loops the
three arms must return bit-identical results, or the run exits non-zero.  The card's name, power limit and maximum SM clock are read in the
same run (read-only nvidia-smi query).  Prints one JSON line and writes it to --out.
    python tools/bench_track_many.py [--cluster 16|8|4] [--warmup 30] [--reps 300] [--out records/h100_track_many.json]"""
import argparse
import ctypes as C
import json
import os
import threading

import numpy as np

import benchkit as K

BS = [1, 2, 4, 8, 16]
W, H, LEVELS = 640, 480, 5


def make_handle(capi, synth, orc, i):
    T = synth.make_tracking_pair(w=W, h=H, seed=4321 + i, levels=LEVELS)
    oc = orc.CoarseTracker(W, H, T["K"], LEVELS)
    g = capi.CT(W, H, LEVELS, max_points=65536)
    for l in range(LEVELS):
        g.set_K(l, *[float(x) for x in oc.K(l)[0]])
    g.upload_new_image(T["img_ref"])
    g.make_coarse_depth(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"])
    g.upload_new_image(T["img_new"])
    return g


class Threads:
    """B worker threads, each tracking its own handle once per round; run() releases them together and returns when all are done"""

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
            self.rcs[i] = self.L.dmv_ct_track(self.hs[i], C.byref(self.A[i]), C.byref(self.R[i]))
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cluster", type=int, default=16, choices=[16, 8, 4], help="DMV_CT_CLUSTER for the run: the cluster size every handle uses")
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--out", default=os.path.join(K.ROOT, "records", "h100_track_many.json"))
    a = ap.parse_args()
    os.environ["DMV_CT_CLUSTER"] = str(a.cluster)
    import dmvio_b200.capi as capi
    import dmvio_b200.synth as synth
    from oracle import orc
    L = K.device_lib("bench_track_many")
    gs = [make_handle(capi, synth, orc, i) for i in range(max(BS))]
    res = dict(card=K.card(), cluster=a.cluster, shape=[W, H], levels=LEVELS, warmup=a.warmup, reps=a.reps,
               timing="wall clock per round, each round ending in a synchronisation; ctypes argument blocks built once", B={})
    identical = True
    for B in BS:
        hs = (C.c_void_p * B)(*[g.h.value for g in gs[:B]])
        A = (capi.CTTrackArgs * B)(*[capi._track_args(LEVELS, np.eye(3), np.zeros(3), 0.0, 0.0) for _ in range(B)])
        outs = {k: (capi.CTTrackResult * B)() for k in ("seq", "threads", "many")}
        th = Threads(L, [hs[i] for i in range(B)], A, outs["threads"])

        def seq():
            rc = 0
            for i in range(B):
                rc = rc or L.dmv_ct_track(hs[i], C.byref(A[i]), C.byref(outs["seq"][i]))
            return rc

        arms = dict(seq=seq, threads=th.run, many=lambda: L.dmv_ct_track_many(hs, B, A, outs["many"]))
        t = K.alternate(arms, a.warmup, a.reps, f"at B={B}", dict.fromkeys(arms, L))
        # identity, outside the timed loops: one more round of each arm, every result struct compared byte for byte
        for k in arms:
            for o in outs[k]:
                C.memset(C.addressof(o), 0, C.sizeof(o))
            arms[k]()
        pe = sum(g.point_evaluations() for g in gs[:B])
        same = all(bytes(outs[k][i]) == bytes(outs["many"][i]) for k in ("seq", "threads") for i in range(B))
        identical = identical and same
        th.close()
        row = dict(bit_identical=same, point_evaluations_per_round=pe)
        for k in arms:
            d = K.stats(t[k])
            row[k] = dict(d, frames_per_s=B / d["median_ms"] * 1e3, point_evals_per_s=pe / d["median_ms"] * 1e3)
        res["B"][str(B)] = row
    res["bit_identical"] = identical
    for g in gs:
        g.close()
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    open(a.out, "w").write(line + "\n")
    if not identical:
        raise SystemExit("the three arms returned different results")


if __name__ == "__main__":
    main()

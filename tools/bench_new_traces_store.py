"""A keyframe's new immature points into the immature-point store: dmv_ct_make_new_traces followed by dmv_ip_store_put of its output (the
thinnest glue: preallocated arguments, u and v converted to float, the constructor's in/out values preallocated) against one
dmv_ct_make_new_traces_store asking for type alone.

Workload: a store pre-filled with 6 slots x 1500 points (dmv_ct_init_points on random pixels), the new keyframe's points going into slot 6,
at 640x480 and 512x512 with 5 levels.  Each arm has its own tracker handle (the same resident keyframe) and its own store; the arms
alternate call by call (benchkit.alternate), and before each call the arm's slot 6 is emptied by a put, outside the timing.  Reported per
arm: median / p10 / p90 wall time per keyframe, the bytes each way computed from the layouts, and the synchronisations per call.  After
the loop both stores are compared bit for bit (every slot's get, then again after one trace of both stores), and the run exits non-zero if
any bit differs.  The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line and writes it to --out.
    python tools/bench_new_traces_store.py [--warmup 20] [--reps 300] [--out records/h100_new_traces_store.json]"""
import argparse
import ctypes as C
import json
import os

import numpy as np

import benchkit as K
import dmvio_b200.capi as capi  # noqa: E402
from oracle import select as S  # noqa: E402

SHAPES = [(640, 480, 5), (512, 512, 5)]
SLOTS, PER_SLOT, NEW_SLOT, CAP = 6, 1500, 6, 16384
PS_STATE = 48   # bytes of ps_select.cu's PSState


def traffic(m, stored):
    """bytes up / down and synchronisations of both arms for m new points over `stored` points already in the store, from the layouts:
    make_new_traces downloads 24 words per point and the state; put uploads 31 words per point and the row map (4 bytes per point after
    the edit); the new call downloads the state, the point count (2 words) and type, and uploads the row map.  Both upload B (256 floats)."""
    total = stored + m
    pair = dict(up_bytes=4 * 256 + 4 * 31 * m + 4 * total, down_bytes=PS_STATE + 4 * 24 * m, syncs=2)
    call = dict(up_bytes=4 * 256 + 4 * total, down_bytes=PS_STATE + 8 + 4 * m, syncs=2)
    return pair, call


def fill(ct, st, w, h, rng):
    """slots 0 .. SLOTS-1 of st: PER_SLOT points each, the constructor on random pixels of ct's resident frame"""
    for k in range(SLOTS):
        u, v = rng.integers(8, w - 8, PER_SLOT), rng.integers(8, h - 8, PER_SLOT)
        P = ct.init_points(u, v)
        P.pop("ok")
        st.put(k, P)


def tables(w, h):
    """KRKi | Kt | aff for every slot: a small rotation and translation of the keyframe against itself"""
    fx, fy, cx, cy = S.K_of(w, h)
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    a = 0.01
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    t = np.array([0.02, -0.01, 0.005])
    row = np.concatenate([(Km @ R @ np.linalg.inv(Km)).reshape(-1), Km @ t, [1.0, 0.0]]).astype(np.float32)
    return np.tile(row, (SLOTS + 1, 1))


def same_stores(a, b):
    if a.counts != b.counts:
        return False
    for k in range(a.SLOTS):
        if a.counts[k]:
            P, Q = a.get(k), b.get(k)
            if not all(np.array_equal(np.ascontiguousarray(P[x]).view(np.uint32), np.ascontiguousarray(Q[x]).view(np.uint32)) for x in capi.IP_OUT_KEYS):
                return False
    return True


def shape_run(L, w, h, lv, warmup, reps):
    img = S.image("tex", w, h, 5)
    cts = {k: capi.CT(w, h, lv) for k in ("pair", "call")}
    sts = {k: capi.IPStore() for k in ("pair", "call")}
    for k in cts:
        cts[k].upload_new_image(img)
        fill(cts[k], sts[k], w, h, np.random.default_rng(w + h))   # the same points in both stores
    # the pair's preallocated arguments
    out = {k: np.zeros((CAP,) + s, t) for k, (s, t) in capi._NT_SHAPES.items()}
    uf, vf = np.zeros(CAP, np.float32), np.zeros(CAP, np.float32)
    inout = dict(idepth_min=np.zeros(CAP, np.float32), idepth_max=np.full(CAP, np.nan, np.float32), quality=np.full(CAP, 10000, np.float32),
                 status=np.full(CAP, 5, np.int32), lastTraceUV=np.zeros((CAP, 2), np.float32), lastTracePixelInterval=np.zeros(CAP, np.float32))
    pot, n, npt = C.c_int(3), C.c_int(0), C.c_int(0)
    a_pair = capi.NewTracesArgs(1500.0, 1, 1.0, None, None, C.pointer(pot), CAP, C.pointer(n), C.pointer(npt),
                                *[out[k].ctypes.data for k in ("u", "v", "type", "color", "weights", "gradH", "energyTH")], None)
    pts = capi.IPPoints(0, uf.ctypes.data, vf.ctypes.data, *[out[k].ctypes.data for k in ("color", "weights", "gradH", "energyTH")],
                        *[inout[k].ctypes.data for k in ("idepth_min", "idepth_max", "quality", "status", "lastTraceUV", "lastTracePixelInterval")])
    ctp, stp = cts["pair"].h, sts["pair"].h

    def pair():
        pot.value = 3
        rc = L.dmv_ct_make_new_traces(ctp, C.byref(a_pair))
        if rc:
            return rc
        m = n.value
        np.copyto(uf[:m], out["u"][:m], casting="unsafe")
        np.copyto(vf[:m], out["v"][:m], casting="unsafe")
        pts.n = m
        return L.dmv_ip_store_put(stp, NEW_SLOT, C.byref(pts))

    typ = np.zeros(CAP, np.float32)
    pot2, n2, npt2 = C.c_int(3), C.c_int(0), C.c_int(0)
    a_call = capi.NewTracesArgs(1500.0, 1, 1.0, None, None, C.pointer(pot2), CAP, C.pointer(n2), C.pointer(npt2), None, None, typ.ctypes.data,
                                None, None, None, None, None)
    ctc, stc = cts["call"].h, sts["call"].h

    def call():
        pot2.value = 3
        return L.dmv_ct_make_new_traces_store(ctc, stc, NEW_SLOT, C.byref(a_call))

    empty = capi.IPPoints(0)
    resets = {"pair": lambda: L.dmv_ip_store_put(stp, NEW_SLOT, C.byref(empty)), "call": lambda: L.dmv_ip_store_put(stc, NEW_SLOT, C.byref(empty))}
    t = K.alternate({"pair": pair, "call": call}, warmup, reps, f"{w}x{h}", {"pair": L, "call": L}, resets)
    # after the loop: both stores hold the last call's slot
    m = n.value
    for k in ("pair", "call"):
        sts[k].counts[NEW_SLOT] = m
    ok = (n2.value == m and pot.value == pot2.value and npt.value == npt2.value and np.array_equal(out["type"][:m].view(np.uint32), typ[:m].view(np.uint32))
          and same_stores(sts["pair"], sts["call"]))
    tab = tables(w, h)
    for k in ("pair", "call"):
        cts[k].trace_store(sts[k], tab)
    ok = ok and same_stores(sts["pair"], sts["call"])
    if not ok:
        raise SystemExit(f"{w}x{h}: the two arms' stores differ")
    p_tr, c_tr = traffic(m, SLOTS * PER_SLOT)
    res = dict(points_new=m, points_stored=SLOTS * PER_SLOT, potential_after=pot.value,
               make_new_traces_plus_put=dict(K.stats(t["pair"]), **p_tr), make_new_traces_store=dict(K.stats(t["call"]), **c_tr))
    res["ratio_of_medians"] = res["make_new_traces_store"]["median_ms"] / res["make_new_traces_plus_put"]["median_ms"]
    for k in cts:
        cts[k].close()
        sts[k].close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = K.device_lib("bench_new_traces_store")
    res = dict(card=K.card(), warmup=a.warmup, reps=a.reps,
               timing="wall clock per keyframe, each call ending in a synchronisation; arms alternate call by call; slot 6 emptied by put outside the timed call")
    for w, h, lv in SHAPES:
        res[f"{w}x{h}_l{lv}"] = shape_run(L, w, h, lv, a.warmup, a.reps)
    res["bit_identical"] = True
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

"""One keyframe's activatePointsMT on an immature-point store: the five steps on host arrays (dmv_ip_store_get of every slot,
dmv_ba_select_activation, dmv_ba_activate_points, the removal set restated in numpy, dmv_ip_store_remove per slot) against one
dmv_ba_activate_store.

Workloads: the C3-like window (7 keyframes, 6 x 1500 immature points traced over three frames, currentMinActDist 2) and the first-keyframes
window (2 keyframes, 3000 points, currentMinActDist 0), at 640x480 and 512x512.  The two arms alternate (benchkit.alternate); before each
call both stores are reset by dmv_ip_store_put to the same traced points, outside the timing.  Reported per arm: median / p10 / p90 wall time
per keyframe, the bytes each way computed from the staging layouts, and the synchronisations per call.  Outside the timed loop the arms
are compared on every output and the stores' contents (tests/test_gpu_activate_store.py's twin), and the run exits non-zero if any bit
differs.  The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line and writes it to --out."""
import argparse
import json
import os

import numpy as np

import benchkit as K

MAXF = 8
WORKLOADS = {"c3": dict(nf=7, npts=2000, per_host=1500, mad=2.0), "first_keyframes": dict(nf=2, npts=40, per_host=3000, mad=0.0)}


def traffic(n, na, nopt, per_slot, nf, removed_slots):
    """bytes up / down and synchronisations of both arms, from the staging layouts of ip_select.cu, ip_trace.cu and ip_store.cu"""
    act_cap = max(nopt, 2048)
    sel_up, sel_down = 4 * (128 + 4 * na + 8 * n), 4 * (2 * n + 8)
    act_up, act_down = 4 * (MAXF * MAXF * 14 + 22 * act_cap), 4 * (2 * act_cap + nf * nopt)
    total_after = n - sum(removed_slots.values())
    steps_remove_up = 0
    left = n
    for gone in removed_slots.values():   # each dmv_ip_store_remove uploads the store's whole row map
        left -= gone
        steps_remove_up += 4 * left
    steps = dict(up_bytes=sel_up + (act_up if nopt else 0) + steps_remove_up, down_bytes=4 * 7 * n + sel_down + (act_down if nopt else 0),
                 syncs=sum(1 for m in per_slot if m) + 1 + int(nopt > 0) + len(removed_slots))
    call = dict(up_bytes=4 * (128 + 4 * na + n) + (4 * MAXF * MAXF * 14 if nopt else 0) + (4 * total_after if removed_slots else 0),
                down_bytes=sel_down + (act_down + 4 * nopt if nopt else 0), syncs=1 + int(nopt > 0) + int(bool(removed_slots)))
    return steps, call


def workload(capi, synth, orc, Win, fill, name, shape, warmup, reps):
    cfg = WORKLOADS[name]
    nf = cfg["nf"]
    win = Win(capi, synth, orc, 7 + shape[0], *shape, nf=nf, npts=cfg["npts"])
    slot = [(3 * f + 1) % 8 if f < nf - 1 else -1 for f in range(nf)]
    fill(win, slot, cfg["per_host"])
    for t in ([nf - 1, nf - 2, nf - 1] if nf > 2 else [1, 1, 1]):
        win.trace(t)
    copies = {k: dict(win.copies[k]) for k in win.copies}
    full = {k: win.stores[0].get(k, copies[k]) for k in copies}

    def reset():
        for k, P in full.items():
            for st in win.stores:
                st.put(k, P)
        win.copies = {k: dict(P) for k, P in copies.items()}

    reset()
    r, _ = win.turnover(slot, mad=cfg["mad"], want_map=False, what=f"{name} {shape}")   # bit for bit against the five steps
    flagged = np.zeros(nf, np.uint8)
    types = win.types(slot)
    counts = [full[k]["u"].shape[0] if k >= 0 else 0 for k in slot]
    n, nopt = sum(counts), len(r["opt_frame"])
    removed = {k: counts[f] - int(r["n_kept"][f]) for f, k in enumerate(slot) if k >= 0 and counts[f] - int(r["n_kept"][f]) > 0}

    def steps():
        win.five_steps(slot, nf - 1, flagged, cfg["mad"], want_map=False, check=False)
        return 0

    def call():
        try:
            win.bas[0].activate_store(win.stores[0], nf - 1, win.tab12, flagged, *win.act, slot, types, cfg["mad"], win.RT)
        except capi.DmvError:
            return -1
        return 0

    t = K.alternate({"five_steps": steps, "activate_store": call}, warmup, reps, name, {"five_steps": capi.lib(), "activate_store": capi.lib()},
                    resets={"five_steps": reset, "activate_store": reset})
    s_steps, s_call = traffic(n, len(win.act[0]), nopt, counts, nf, removed)
    win.close()
    out = dict(points=n, active_points=len(win.act[0]), to_optimize=nopt, removed=int(sum(removed.values())),
               five_steps=dict(K.stats(t["five_steps"]), **s_steps), activate_store=dict(K.stats(t["activate_store"]), **s_call))
    out["ratio_of_medians"] = out["activate_store"]["median_ms"] / out["five_steps"]["median_ms"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(K.ROOT, "records", "h100_activate_store.json"))
    a = ap.parse_args()
    import dmvio_b200.capi as capi
    import dmvio_b200.synth as synth
    from oracle import orc
    from test_gpu_activate_store import Win, fill
    K.device_lib("bench_activate_store")
    orc.build()
    res = dict(card=K.card(), warmup=a.warmup, reps=a.reps,
               timing="wall clock per keyframe, each call ending in a synchronisation; stores reset by put outside the timed call; the five "
                      "steps are issued from Python with numpy glue, as a host adapter would issue them from C++")
    for name in WORKLOADS:
        for shape in ((640, 480), (512, 512)):
            res[f"{name}_{shape[0]}x{shape[1]}"] = workload(capi, synth, orc, Win, fill, name, shape, a.warmup, a.reps)
    res["bit_identical"] = True   # workload() raises before here on any differing bit
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

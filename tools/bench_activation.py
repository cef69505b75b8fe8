"""Wall time per keyframe of activatePointsMT's selection (makeDistanceMap + the loop up to activatePointsMT_Reductor): dmv_ba_select_activation
(device path) against the host path, the CPU restatement (oracle/orc_activation.cpp, built -O3 single-threaded with the reference's flags, the
way the reference runs this loop).  A C3-like window (7 keyframes, 2000 active points and 1500 immature points per other keyframe) and a
"first keyframes" window (2 keyframes, 40 active points, 3000 candidates, currentMinActDist 0) at 640x480 and 512x512; every timed device call
ends in a synchronise, the map not requested.  Bytes each way come from the call's staging layout; undecided = candidates the map before
the loop could not decide, floods = floods run, rounds = the serial depth of the device's chain.  Prints one JSON line, with the card's name and power limit read in the same run, and writes it to --out if given.
    python tools/bench_activation.py [--reps 50] [--out records/h100_activation.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dmvio_b200.capi as capi  # noqa: E402
from oracle import activation as A  # noqa: E402

WINDOWS = {
    "c3": dict(nf=7, n_active=2000 * 6, n_imm=1500, min_act_dist=2.0),
    "first_keyframes": dict(nf=2, n_active=40, n_imm=3000, min_act_dist=0.0, flagged=()),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    rows = []
    for w, h in ((640, 480), (512, 512)):
        ba = capi.BA(w, h, max_frames=8, max_points=64)
        for name, kw in WINDOWS.items():
            case = A.make_case(w=w, h=h, seed=w + h, **kw)
            tab = A.tables(case)
            call = lambda: ba.select_activation(case["nf"], case["newest"], tab, case["flagged"], case["act_u"], case["act_v"], case["act_id"],
                                                case["act_host"], case["off"], case["imm"], case["min_act_dist"], A.MIN_TRACE_QUALITY, want_map=False)
            act, opt, _, st = call()
            a, o, _ = A.restate(case, tab)
            assert np.array_equal(act, a) and np.array_equal(opt, o)
            for _ in range(5):
                call()
                A.restate(case, tab)
            td, th = [], []
            for _ in range(args.reps):   # alternate the two paths
                t0 = time.perf_counter(); call(); td.append(time.perf_counter() - t0)
                t0 = time.perf_counter(); A.restate(case, tab); th.append(time.perf_counter() - t0)
            n, na = int(case["off"][-1]), len(case["act_u"])
            rows.append(dict(w=w, h=h, window=name, n_immature=n, n_active=na, n_opt=len(opt), undecided=st["undecided"], floods=st["floods"], rounds=st["rounds"],
                             device_ms_median=1e3 * float(np.median(td)), device_ms_p90=1e3 * float(np.percentile(td, 90)),
                             host_ms_median=1e3 * float(np.median(th)), host_ms_p90=1e3 * float(np.percentile(th, 90)),
                             h2d_bytes=4 * (128 + 4 * na + 8 * n), d2h_bytes=4 * (2 * n + 4)))
        ba.close()
    rec = dict(tool="tools/bench_activation.py", gpu=q.strip(), reps=args.reps, rows=rows)
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

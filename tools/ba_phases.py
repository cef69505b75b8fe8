#!/usr/bin/env python
"""Phase clock of the headline BA launch: where the time of one ba_fused_kernel goes.

Builds bench.py's headline window (7 KF / 2000 points / 640x480, seed 1234) with the seeded step x, then runs the loop bench.py times
(L2 scrub, fused resubstitution + step, one linearisation launch) through dmv_ba_bench_phases, whose clocked kernel instantiation has
thread 0 of every CTA record %globaltimer at 9 points.  Prints, per segment, the mean over launches of the mean and of the max over the
CTAs, next to the CUDA-event time of the same launches.  The per-chunk stamps are exact when every CTA runs one chunk, as in the
headline window (129 chunks of 16 points).  The clock itself is a few global stores per CTA; the product kernels have none.
--no-flush skips the L2 scrub, so code and data stay warm in L2 between launches: the difference to the scrubbed run is what cold
fetches cost each phase.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import bench  # noqa: E402

STAMPS = ["entry", "chunk decoded", "first loads", "taps", "end A", "end C", "barrier released", "end D", "end E"]
SEGMENTS = [("decode", 0, 1), ("A: first loads (+ resubstitution)", 1, 2), ("A: projection + taps", 2, 3), ("A: tail + block barrier", 3, 4),
            ("B + C", 4, 5), ("grid barrier", 5, 6), ("D", 6, 7), ("E", 7, 8)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--chunk", type=int, default=0, help="points per thread block (16/32, 0 = library default)")
    ap.add_argument("--json", default=None, help="also write the table as JSON to this file")
    ap.add_argument("--no-flush", action="store_true", help="no L2 scrub between launches (warm L2)")
    args = ap.parse_args()
    C = bench.Case(bench.Dist(1, 0), 0, 1, 0, bench.NPTS, args.chunk, "none")
    for _ in range(max(3, args.warmup)):
        C.ba.gn_step(C.x, C.k8, C.precalc, C.TH)
        C.ba.apply_res()
    flush = not args.no_flush
    C.ba.bench_phases(C.x, iters=max(3, args.warmup), flush_l2=flush)
    st, ms = C.ba.bench_phases(C.x, iters=args.iters, flush_l2=flush)
    C.close()
    t = np.where(st == 0, np.nan, st.astype(np.float64))          # [launch, cta, stamp] ns; 0 = not reached
    t0 = np.nanmin(t[:, :, 0], axis=1)[:, None]                  # first CTA entry of each launch
    seg = {name: t[:, :, b] - t[:, :, a] for name, a, b in SEGMENTS}
    seg["entry skew (vs first CTA)"] = t[:, :, 0] - t0
    seg["entry -> end E"] = t[:, :, 8] - t[:, :, 0]
    rows = {k: {"mean_us": float(np.nanmean(np.nanmean(v, axis=1)) / 1e3), "max_us": float(np.nanmean(np.nanmax(v, axis=1)) / 1e3)} for k, v in seg.items()}
    first_to_last = np.nanmax(t[:, :, 8], axis=1) - t0[:, 0]
    out = {"ctas": int(st.shape[1]), "launches": int(st.shape[0]), "l2_scrubbed": flush, "segments": rows,
           "first_entry_to_last_end_us": float(np.mean(first_to_last) / 1e3),
           "event_us": {"mean": float(np.mean(ms) * 1e3), "median": float(np.median(ms) * 1e3)}}
    print(f"ba_fused_kernel phase clock: {out['launches']} launches x {out['ctas']} CTAs (headline window, {'L2 scrubbed' if flush else 'warm L2'}, resubstituting)")
    print(f"{'segment':38s} {'mean/CTA us':>12s} {'max/CTA us':>12s}")
    for k, v in rows.items():
        print(f"{k:38s} {v['mean_us']:12.2f} {v['max_us']:12.2f}")
    print(f"{'first CTA entry -> last CTA end E':38s} {out['first_entry_to_last_end_us']:12.2f}")
    print(f"{'CUDA events (mean / median)':38s} {out['event_us']['mean']:12.2f} {out['event_us']['median']:12.2f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

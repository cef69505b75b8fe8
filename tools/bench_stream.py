#!/usr/bin/env python
"""Secondary benchmark (BASELINE config 5, SURVEY.md §8d): keyframes/s of the BA back-end on a TUM-VI-shaped synthetic stream
(512x512, 7-keyframe sliding window, 2000 active points, 10 GN iterations per keyframe; IMU factors / GTSAM stubbed: the host solve is
the reference's plain LDLT branch).  Per keyframe the GPU side pays EVERYTHING a DM-VIO host would: H2D of the new raw image + device
pyramid, point / residual upload, adjoints, 10 fused GN steps with the dense solves on the host (C++ adapter WindowBA::optimize);
frames stay resident across keyframes (image slots).  The CPU side is the oracle's optimize() with 6 worker threads on the same windows
(its window construction is not timed).  Prints one JSON line.   python tools/bench_stream.py [--keyframes 40]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402


def sub_window(S, first, nfw, npts, rng):
    """frames [first, first+nfw) of the long sequence S as a window dict: points hosted by all but the newest frame."""
    fr = np.arange(first, first + nfw)
    W = dict(w=S["w"], h=S["h"], nf=nfw, K=S["K"])
    for k in ("R_eval", "t_eval", "state", "state_zero", "exposure", "frameEnergyTH", "frameID"):
        W[k] = S[k][fr].copy()
    W["frameID"] = np.arange(first, first + nfw, dtype=np.int32)
    W["dI"] = [S["dI"][f] for f in fr]
    W["images"] = [S["images"][f] for f in fr]
    cand = np.nonzero((S["host"] >= first) & (S["host"] < first + nfw - 1))[0]
    sel = np.sort(rng.choice(cand, min(npts, len(cand)), replace=False))
    sel = sel[np.argsort(S["host"][sel], kind="stable")]
    for k in ("u", "v", "idepth", "idepth_zero", "color", "weights", "hasDepthPrior"):
        W[k] = S[k][sel]
    W["host"] = (S["host"][sel] - first).astype(np.int32)
    n = len(sel)
    pt = np.repeat(np.arange(n, dtype=np.int32), nfw)
    tg = np.tile(np.arange(nfw, dtype=np.int32), n)
    keep = tg != W["host"][pt]
    W["res_point"], W["res_target"] = pt[keep], tg[keep]
    return W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=40)
    ap.add_argument("--its", type=int, default=10)
    ap.add_argument("--cpu-keyframes", type=int, default=6)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    print(json.dumps(run_stream(args.keyframes, args.its, args.cpu_keyframes, args.size, args.device)))


def run_stream(keyframes=40, its=10, cpu_keyframes=6, size=512, device=0):
    """BASELINE config 5 as written: EXACTLY `its` GN iterations per keyframe on both sides (setting_minOptIterations = setting_maxOptIterations =
    its, MainSettings.cpp:L195-196).  cpu_keyframes = 0 skips the CPU arm (replicas at N > 1)."""
    class A:
        pass
    args = A()
    args.keyframes, args.its, args.cpu_keyframes, args.size = keyframes, its, cpu_keyframes, size
    import dmvio_b200.hostapi as hostapi
    import dmvio_b200.synth as synth
    from oracle import orc
    NFW, NPTS = 7, 2000
    total = args.keyframes + NFW - 1
    rng = np.random.default_rng(7)
    S = synth.make_window(nf=total, npts=400 * total, w=args.size, h=args.size, seed=77, hosts="all", state_noise=1e-3)
    L = hostapi.lib()
    c = lambda a, t: np.ascontiguousarray(a, t)
    win = L.dmvh_window_create(S["w"], S["h"], 8, NPTS, device, c(S["K"], np.float64))
    assert L.dmvh_window_set_setting(win, b"minOptIterations", float(args.its)) == 0   # no early break: its iterations per keyframe, as the config says

    def add_frame(W, k):
        rc = L.dmvh_window_add_frame(win, c(W["images"][k], np.float32).reshape(-1), 1, c(W["R_eval"][k], np.float64).reshape(-1), c(W["t_eval"][k], np.float64),
                                     c(W["state"][k], np.float64), c(W["state_zero"][k], np.float64), float(W["exposure"][k]), int(W["frameID"][k]))
        assert rc >= 0, L.dmvh_window_error(win)

    W0 = sub_window(S, 0, NFW, NPTS, rng)
    for k in range(NFW - 1):
        add_frame(W0, k)
    log = np.zeros(64)
    gpu_t, gpu_its, energies, setup_t = [], [], [], []
    for s in range(args.keyframes):
        W = sub_window(S, s, NFW, NPTS, rng)
        t0 = time.perf_counter()
        if s > 0:
            L.dmvh_window_drop_frame(win, 0)                      # oldest keyframe leaves (marginalised on the host side)
        add_frame(W, NFW - 1)                                     # new keyframe: H2D of the raw image + device pyramid
        L.dmvh_window_set_points(win, len(W["host"]), c(W["host"], np.int32), c(W["u"], np.float32), c(W["v"], np.float32), c(W["idepth"], np.float32),
                                 c(W["idepth_zero"], np.float32), c(W["color"], np.float32).reshape(-1), c(W["weights"], np.float32).reshape(-1), None)
        L.dmvh_window_set_residuals(win, len(W["res_point"]), c(W["res_point"], np.int32), c(W["res_target"], np.int32))
        assert L.dmvh_window_prepare(win) == 0, L.dmvh_window_error(win)
        t1 = time.perf_counter()
        n = L.dmvh_window_optimize(win, args.its, log, 64)
        gpu_t.append(time.perf_counter() - t0)
        setup_t.append(t1 - t0)
        gpu_its.append(n)
        energies.append(log[log >= 0][[0, -1]].copy())
    cpu_t = []
    for s in range(min(args.cpu_keyframes, args.keyframes)):
        W = sub_window(S, s, NFW, NPTS, np.random.default_rng(7)) if s == 0 else sub_window(S, s, NFW, NPTS, rng)
        ow = orc.Window(W, nthreads=6, settings={"minOptIterations": args.its})
        t0 = time.perf_counter()
        n_o, log_o = ow.optimize(args.its, precision=0)
        cpu_t.append(time.perf_counter() - t0)
    g = float(np.median(gpu_t[2:])); cpu = float(np.median(cpu_t)) if cpu_t else float("nan")
    out = {"metric": "BA keyframes/s (7 KF window, 2000 pts, %dx%d, %d GN its/KF, IMU factors stubbed)" % (args.size, args.size, args.its),
           "gpu_ms_per_keyframe": g * 1e3, "gpu_keyframes_per_s": 1.0 / g, "gpu_gn_iterations_per_keyframe": float(np.mean(gpu_its)),
           "cpu_oracle_ms_per_keyframe": cpu * 1e3, "cpu_keyframes_per_s": 1.0 / cpu, "cpu_threads": 6, "speedup": cpu / g,
           "residuals_per_window": int(len(W["res_point"])), "energy_first_last_of_last_keyframe": [float(v) for v in energies[-1]],
           "timed_gpu": "drop oldest + H2D new image + device [I,dx,dy] + points/residuals upload + adjoints + optimize() (fused GN steps, host LDLT solves)",
           "timed_cpu": "oracle optimize() only (window construction excluded), 6 worker threads"}
    prof = np.zeros(5)
    L.dmvh_window_profile(win, prof, 1)
    nit = max(1.0, prof[4])
    out["gpu_ms_setup_per_keyframe"] = float(np.median(setup_t[2:])) * 1e3   # drop oldest + H2D + device [I,dx,dy] + point / residual upload + adjoints
    out["gpu_us_per_iteration"] = {"host_solve": prof[0] / nit, "host_state_step_and_tables": prof[1] / nit, "linearize_launch_and_sync": prof[2] / nit,
                                   "host_prior_energies": prof[3] / nit}
    L.dmvh_window_destroy(win)
    return out


if __name__ == "__main__":
    main()

"""Keyframe hand-off from the BA window to the coarse tracker: time from "the tail's linearisation returned" to "the tracker's pc_* lists
are ready", two ways:
  host    the host path of FullSystem::makeKeyFrame: download the residuals' state_NewState + centerProjectedTo (dmv_ba_get_residual_outputs)
          and the last solve's HdiF (dmv_ba_get_solve_HdiF), keep the IN residuals into the newest frame on the host in makeCoarseDepthL0's
          point order (after removeOutliers; that permutation is host bookkeeping, computed once before timing), upload the keyframe's
          raw image (dmv_ct_upload_new_image: pyramid on the device) and run dmv_ct_make_coarse_depth (collisions folded on the host)
  device  dmv_ct_set_ref_from_ba: nothing crosses PCIe but the 7 result counters
Each repetition runs both arms on the same committed window, alternating which goes first; medians over --reps repetitions after --warmup.
PCIe bytes per arm come from the shapes.  Every repetition checks that both arms give the same pc_n.  Prints one JSON line, with the card's
name and power limit read in the same run, and writes it to --out if given.
    python tools/bench_ref_handoff.py [--reps 300] [--warmup 30] [--out records/h100_ref_handoff.json]"""
import argparse
import json
import os
import time

import numpy as np

import benchkit as K  # first: it puts the repository root on sys.path
import dmvio_b200.capi as capi  # noqa: E402
import dmvio_b200.hostmath as hm  # noqa: E402
import dmvio_b200.synth as synth  # noqa: E402

WINDOWS = [("baseline_c3_7kf_2000pts_640x480", dict(nf=7, npts=2000, w=640, h=480, seed=1234), 5),
           ("7kf_2000pts_512x512", dict(nf=7, npts=2000, w=512, h=512, seed=1234), 4)]
MAXF = 8   # DMV_MAX_FRAMES: the residual slots the handle keeps per point


def committed_window(W):
    """a BA handle after the keyframe tail: linearize + commit + accumulate (solveSystemF), the non-IN residuals dropped, the tail's
    linearisation committed"""
    ba = capi.BA(W["w"], W["h"], max_frames=W["nf"], max_points=len(W["host"]))
    for k in range(W["nf"]):
        ba.upload_frame(k, W["dI"][k])
    ba.set_window(W["nf"])
    ba.set_points(W["host"], W["u"], W["v"], W["idepth"], W["idepth_zero"], W["color"], W["weights"])
    ba.set_residuals(W["res_point"], W["res_target"])
    ba.set_adjoints(*hm.adjoints(W))
    st = (hm.calib8(W["K"]), hm.precalc_table(W), W["frameEnergyTH"])
    ba.set_state(*st)
    ba.linearize(); ba.apply_res(); ba.accumulate()
    ns = ba.residual_outputs()["newState"]
    drop = np.nonzero(ns != 0)[0].astype(np.int32)
    ba.drop_residuals(drop)
    keep = np.setdiff1d(np.arange(len(ns)), drop)
    ba.gn_step(np.zeros(8 * W["nf"] + 4), *st)
    ba.apply_res()
    return ba, W["res_point"][keep], W["res_target"][keep]


def fold_order(host, rp):
    """the points in makeCoarseDepthL0's order: FullSystem::removeOutliers (FullSystemOptimize.cpp:L680-697) drops the points without
    residuals by swap-with-back"""
    alive = np.zeros(len(host), bool)
    alive[rp] = True
    out = []
    for h in np.unique(host):
        lst = list(np.nonzero(host == h)[0])
        i = 0
        while i < len(lst):
            if not alive[lst[i]]:
                lst[i] = lst[-1]
                lst.pop()
                i -= 1
            i += 1
        out += lst
    return np.asarray(out, np.int64)


def host_arm(ba, ct, rp, rt, nf, img, bufs, order):
    st, cpt, hdi = bufs
    capi.check(ba.L.dmv_ba_get_residual_outputs(ba.h, st.ctypes.data, None, None, cpt.ctypes.data, None))
    capi.check(ba.L.dmv_ba_get_solve_HdiF(ba.h, hdi))
    res_of = np.full(ba.npts, -1)
    sel = np.nonzero((rt == nf - 1) & (st == 0))[0]
    res_of[rp[sel]] = sel
    sel = res_of[order[res_of[order] >= 0]]
    c = cpt[sel]
    ct.upload_new_image(img)
    return ct.make_coarse_depth(c[:, 0], c[:, 1], c[:, 2], hdi[rp[sel]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    K.device_lib("bench_ref_handoff")
    out = dict(card=K.card(), reps=a.reps, warmup=a.warmup, windows=[])
    for name, cfg, levels in WINDOWS:
        W = synth.make_window(**cfg)
        w, h, nf = W["w"], W["h"], W["nf"]
        ba, rp, rt = committed_window(W)
        ct_h, ct_d = capi.CT(w, h, levels), capi.CT(w, h, levels)
        bufs = (np.zeros(ba.nres, np.int32), np.zeros((ba.nres, 3), np.float32), np.zeros(ba.npts, np.float32))
        img = np.ascontiguousarray(W["images"][-1], np.float32)
        order = fold_order(W["host"], rp)
        t_h, t_d = [], []
        for i in range(a.warmup + a.reps):
            arms = (0, 1) if i % 2 == 0 else (1, 0)
            res = {}
            for arm in arms:
                t0 = time.perf_counter()
                res[arm] = host_arm(ba, ct_h, rp, rt, nf, img, bufs, order) if arm == 0 else ct_d.set_ref_from_ba(ba)
                dt = (time.perf_counter() - t0) * 1e3
                if i >= a.warmup:
                    (t_h if arm == 0 else t_d).append(dt)
            if not np.array_equal(res[0], res[1]):
                raise SystemExit(f"{name}: pc_n differs between the arms: {res[0]} vs {res[1]}")
        mp = (len(W["host"]) + 31) & ~31
        ns = MAXF * mp
        n_in = int(np.count_nonzero((rt == nf - 1) & (bufs[0] == 0)))
        ip_cap = max(n_in, 2048)
        bytes_host = dict(d2h_state=ns, d2h_centerProjectedTo=3 * ns * 4, d2h_HdiF=4 * ba.npts, h2d_image=4 * w * h, h2d_splat=3 * ip_cap * 4)
        out["windows"].append(dict(
            name=name, nf=nf, npts=ba.npts, w=w, h=h, levels=levels, in_residuals_newest=n_in, pc_n=[int(x) for x in res[1][:levels]],
            host_path_ms_median=float(np.median(t_h)), device_ms_median=float(np.median(t_d)),
            host_path_ms_p10_p90=[float(np.percentile(t_h, 10)), float(np.percentile(t_h, 90))],
            device_ms_p10_p90=[float(np.percentile(t_d, 10)), float(np.percentile(t_d, 90))],
            pcie_bytes_host_path=int(sum(bytes_host.values())), pcie_bytes_host_path_parts=bytes_host,
            pcie_bytes_device=4 * (levels + 1)))
        ct_h.close(); ct_d.close(); ba.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

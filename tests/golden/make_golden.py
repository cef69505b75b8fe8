#!/usr/bin/env python
"""Generates the committed golden fixtures of the BA / coarse hot path (tests/golden/*.npz).

The reference has no golden vectors or known-answer tests for this path (SURVEY.md §4, §8c).  These vectors come from the CPU
oracle in its fp64-accumulating mode (precision=1) AFTER the oracle has been pinned bit-exact against the reference's own
compiled code (oracle/_ref, tests/test_ref_pin.py — run that first): they freeze its outputs (a) to detect drift of the oracle
or of the synthetic generator and (b) as a file-based checker for the CUDA path on a GPU machine without the reference sources.

  golden_small_ba.npz    complete inputs (96x64 images) + every intermediate of one GN iteration  -> self-contained
  golden_c1_ba.npz       BASELINE config 1 (2 KF / 200 pts / 640x480): seed + input checksum + outputs
  golden_c3_ba.npz       BASELINE config 3 (7 KF / 2000 pts / 640x480): seed + input checksum + reduced system + x
  golden_small_coarse.npz  coarse tracker on a 160x120 pair: inputs + calcRes/calcGS outputs per level + tracked pose

Run from the repo root:  python tests/golden/make_golden.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import dmvio_b200.synth as synth  # noqa: E402
from oracle import orc  # noqa: E402

INPUT_KEYS = ("K", "R_eval", "t_eval", "state", "state_zero", "exposure", "frameEnergyTH", "frameID", "host", "u", "v", "idepth", "idepth_zero",
              "color", "weights", "hasDepthPrior", "res_point", "res_target")


def window_checksum(W):
    h = hashlib.sha256()
    for k in INPUT_KEYS:
        h.update(np.ascontiguousarray(W[k]).tobytes())
    for d in W["dI"]:
        h.update(np.ascontiguousarray(d, np.float32).tobytes())
    return h.hexdigest()


def ba_outputs(W, full=True):
    ow = orc.Window(W)
    out = {}
    out["precalc"] = ow.precalc()
    adH, adT = ow.adjoints()
    out["adHost"], out["adTarget"] = adH, adT
    out["calib8"] = ow.calib()["k8"]
    out["energy"] = np.float64(ow.linearize_all(update_th=False))
    o = ow.res_outputs(True)
    out["newState"] = o["newState"]
    out["newEnergy"] = o["newEnergy"]
    out["newEnergyWithOutlier"] = o["newEnergyWithOutlier"]
    out["centerProjectedTo"] = o["centerProjectedTo"]
    if full:
        out["J"] = o["J"]
    ow.apply_res()
    o2 = ow.res_outputs(False)
    out["JpJdF"] = o2["JpJdF"]
    out["isActive"] = o2["isActive"]
    a = ow.accumulate(1)
    for k in ("HA", "bA", "HL", "bL", "Hsc", "bsc"):
        out[k] = a[k]
    out["resInA"] = np.int32(a["resInA"])
    p = ow.point_outputs()
    for k in ("Hdd", "bd", "Hcd", "HdiF", "bdSumF"):
        out["pt_" + k] = p[k]
    x, HF, bF = ow.solve(0, 1e-5, 1)
    out["x"], out["HFinal"], out["bFinal"] = x, HF, bF
    out["pt_step"] = ow.point_outputs()["step"]
    return out


def save(name, d):
    path = os.path.join(HERE, name)
    np.savez_compressed(path, **d)
    print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB, {len(d)} arrays")


def main():
    orc.build()
    # ---- small self-contained window
    cfg = dict(nf=3, npts=150, w=96, h=64, seed=11, hosts="all")
    W = synth.make_window(**cfg)
    d = {"in_" + k: np.asarray(W[k]) for k in INPUT_KEYS}
    d["in_dI"] = np.stack([np.asarray(x, np.float32) for x in W["dI"]])
    d["in_wh_nf"] = np.array([W["w"], W["h"], W["nf"]], np.int32)
    d.update(ba_outputs(W, full=True))
    save("golden_small_ba.npz", d)
    # ---- BASELINE configs 1 and 3 by seed
    for name, cfg, full in (("golden_c1_ba.npz", dict(nf=2, npts=200, seed=1234, hosts="first"), True),
                            ("golden_c3_ba.npz", dict(nf=7, npts=2000, seed=1234), False)):
        W = synth.make_window(**cfg)
        d = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
        d["input_sha256"] = np.frombuffer(window_checksum(W).encode(), np.uint8)
        o = ba_outputs(W, full=full)
        if not full:  # keep the 7-KF fixture small: reduced system, energies and states only
            for k in ("precalc", "adHost", "adTarget", "centerProjectedTo", "JpJdF", "pt_Hcd"):
                o.pop(k)
        d.update(o)
        save(name, d)
    # ---- coarse tracker, small pair
    T = synth.make_tracking_pair(w=160, h=120, seed=77, npts=400)
    ct = orc.CoarseTracker(T["w"], T["h"], T["K"], 0)
    ct.make_coarse_depth(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"], T["pyr_ref"])
    ct.set_new_frame(T["pyr_new"])
    d = dict(in_wh=np.array([T["w"], T["h"]], np.int32), in_K=T["K"], in_Ku=T["Ku"], in_Kv=T["Kv"], in_new_idepth=T["new_idepth"], in_HdiF=T["HdiF"],
             in_img_ref=T["img_ref"], in_img_new=T["img_new"], levels=np.int32(ct.levels))
    # a generic pose near the truth (not the identity: integer reference pixels would sit exactly on the bounds tests)
    R, t = synth.se3_mul(*synth.se3_exp(np.array([0.003, -0.002, 0.001, 0.001, -0.001, 0.001])), T["R_true"], T["t_true"])
    a, b = T["a_new"] + 0.01, T["b_new"] - 0.3
    d.update(pose_R=R, pose_t=t, pose_ab=np.array([a, b]))
    for l in range(ct.levels):
        rp = ct.ref_points(l)
        for k in ("u", "v", "idepth", "color"):
            d[f"ref{l}_{k}"] = rp[k]
        d[f"res6_{l}"] = ct.calc_res(l, R, t, a, b, 20.0)
        H, bb = ct.calc_gs(l, a, b, 1)
        d[f"H_{l}"], d[f"b_{l}"] = H, bb
    r = ct.track(np.eye(3), np.zeros(3), 0.0, 0.0)
    d.update(track_R=r["R"], track_t=r["t"], track_ab=np.array([r["a"], r["b"]]), track_lastRes=r["lastResiduals"], track_good=np.int32(r["good"]),
             track_iterations=np.int32(r["iterations"]))
    save("golden_small_coarse.npz", d)


if __name__ == "__main__":
    main()

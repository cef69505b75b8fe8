"""Shared helpers for the parity tests: load one synthetic window into the CPU oracle and into the CUDA product."""
import numpy as np


def calib8_from_oracle(ow):
    return ow.calib()["k8"]


def prior_f(W):
    """EFPoint::priorF of every point: setting_idepthFixPrior * SCALE_IDEPTH^2 = 50 * 50 where the point has a depth prior, else 0"""
    return np.where(np.asarray(W["hasDepthPrior"]) != 0, 50.0 * 50.0, 0.0).astype(np.float32)


def product_ba_from_oracle(capi, W, ow, chunk_points=0, device=0, max_points=None):
    """Feeds the C ABI with the host-side tables computed by the oracle (precalc, adjoints, TH)."""
    ba = capi.BA(W["w"], W["h"], max_frames=max(2, W["nf"]), max_points=max_points or len(W["host"]), device=device, chunk_points=chunk_points)
    for k in range(W["nf"]):
        ba.upload_frame(k, W["dI"][k])
    ba.set_window(W["nf"])
    ba.set_points(W["host"], W["u"], W["v"], W["idepth"], W["idepth_zero"], W["color"], W["weights"], priorF=prior_f(W))
    ba.set_residuals(W["res_point"], W["res_target"], W.get("res_state"), W.get("res_energy"))
    adH, adT = ow.adjoints()
    ba.set_adjoints(adH, adT)
    ba.set_state(calib8_from_oracle(ow), ow.precalc(), ow.frame_tables()["frameEnergyTH"])
    return ba


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


RES_IN, RES_OOB, RES_OUTLIER = 0, 1, 2


def edge_window(synth, cfg, seed_offset=101):
    """synth.make_window(**cfg) with the irregular point and residual sets of a real window:
      * ~30 % of the points carry a depth prior, and idepth_zero != idepth (the prior's shift-to-zero term is non-zero);
      * ~25 % of the residuals are missing, so the frame slots of a point have holes between its targets;
      * a few points keep only their residual into the newest frame (the last target slot of a point);
      * a few points start with every residual OOB (no good residual ever again), a few have no residual at all;
      * ~10 % of the residuals start as OUTLIER, every residual with a stored energy."""
    W = synth.make_window(**cfg)
    rng = np.random.default_rng(cfg["seed"] + seed_offset)
    npts, nf = len(W["host"]), W["nf"]
    W["idepth_zero"] = (W["idepth"] * (1 + 0.02 * rng.standard_normal(npts))).astype(np.float32)
    W["hasDepthPrior"] = (rng.random(npts) < 0.3).astype(np.uint8)
    rp, rt = W["res_point"], W["res_target"]
    keep = rng.random(len(rp)) >= 0.25
    order = rng.permutation(np.nonzero(W["host"] != nf - 1)[0])
    k = max(3, npts // 100)
    last_only, no_res, all_oob = order[:k], order[k:k + max(2, npts // 200)], order[k + max(2, npts // 200):2 * k + max(2, npts // 200)]
    m = np.isin(rp, last_only)
    keep[m] = rt[m] == nf - 1
    keep[np.isin(rp, no_res)] = False
    keep[np.isin(rp, all_oob)] = True
    W["res_point"], W["res_target"] = rp[keep].astype(np.int32), rt[keep].astype(np.int32)
    n = len(W["res_point"])
    W["res_state"] = np.where(rng.random(n) < 0.1, RES_OUTLIER, RES_IN).astype(np.int32)
    W["res_state"][np.isin(W["res_point"], all_oob)] = RES_OOB
    W["res_energy"] = rng.uniform(0, 50, n).astype(np.float32)
    W["edge_points"] = dict(last_only=np.sort(last_only), no_res=np.sort(no_res), all_oob=np.sort(all_oob))
    return W


def make_case(synth, cfg):
    """a CONFIGS entry -> window: plain synth.make_window, or edge_window when the entry carries edge=True"""
    cfg = dict(cfg)
    return edge_window(synth, cfg) if cfg.pop("edge", False) else synth.make_window(**cfg)


def points_with_in_residual(res_point, state, npts):
    """per point: does it have at least one residual in state IN (AccumulatedSCHessian::addPoint's ngoodres > 0)"""
    return np.bincount(np.asarray(res_point)[np.asarray(state) == RES_IN], minlength=npts) > 0


def ulp32(a):
    return np.spacing(np.abs(np.asarray(a, np.float32))).astype(np.float64)


def check_phase_b(pg, good, priorF, idepth, idepth_zero):
    """Phase B in closed form from the launch's own per-point sums: HdiF = 1 / max(Hdd + priorF, 1e-10) and
    bdSumF = bd + priorF * (idepth - idepth_zero) (AccumulatedSCHessian.cpp:L42-50), each within 2 ulp; exactly 0 without a good residual."""
    H = np.maximum(pg["Hdd"] + np.asarray(priorF, np.float32), np.float32(1e-10)).astype(np.float64)   # the fp32 sum, as the kernel forms it
    hdi = 1.0 / H
    assert np.all(np.abs(pg["HdiF"][good] - hdi[good]) <= 2 * ulp32(hdi[good])), "HdiF != 1 / (Hdd + priorF)"
    shift = np.asarray(priorF, np.float64) * (np.asarray(idepth, np.float32) - np.asarray(idepth_zero, np.float32)).astype(np.float64)
    bds = pg["bd"].astype(np.float64) + shift
    tol = 2 * np.maximum(ulp32(bds), ulp32(shift))
    assert np.all(np.abs(pg["bdSumF"][good] - bds[good]) <= tol[good]), "bdSumF != bd + priorF * (idepth - idepth_zero)"
    assert not pg["HdiF"][~good].any() and not pg["bdSumF"][~good].any()


def check_linearize_parity(ow, ba, r, E_o):
    """A GPU linearisation (result r, still tentative) against the oracle's (energy E_o of ow.linearize_all), then both committed and
    accumulated.  Tolerances and their reasons: tests/test_gpu_ba.py's docstring.  Returns the GPU's (residual outputs, point outputs,
    accumulated system)."""
    o = ow.res_outputs(False)
    g = ba.residual_outputs()
    # ---- states: identical except threshold ties
    mism = np.nonzero(o["newState"] != g["newState"])[0]
    for i in mism:
        eo, TH = o["newEnergyWithOutlier"][i], 512.0
        assert abs(eo - TH) < 2e-3 * TH or o["newState"][i] == 1 or g["newState"][i] == 1, (i, o["newState"][i], g["newState"][i], eo)
    assert len(mism) <= max(2, ow.nres // 500)
    assert r["n_in"] == int((g["newState"] == 0).sum())
    assert r["n_oob"] == int((g["newState"] == 1).sum())
    # ---- threshold ties: impose the GPU's classification on the oracle (its Jacobians exist on both sides of the threshold), so that every
    # comparison below runs UNCONDITIONALLY on the same residual set
    E_o, nchanged, unfixable = ow.override_new_states(g["newState"])
    assert unfixable == 0, "an OOB-boundary tie cannot be imposed on the oracle: pick another seed for this config"
    assert nchanged == len(mism)
    o = ow.res_outputs(False)
    assert np.array_equal(o["newState"], g["newState"])
    # ---- energies
    ev = o["newState"] != 1
    np.testing.assert_allclose(g["newEnergy"][ev], o["newEnergy"][ev], rtol=2e-3, atol=0.05)
    np.testing.assert_allclose(g["newEnergyWithOutlier"][ev], o["newEnergyWithOutlier"][ev], rtol=2e-3, atol=0.05)
    relerr = np.abs(g["newEnergyWithOutlier"][ev] - o["newEnergyWithOutlier"][ev]) / (np.abs(o["newEnergyWithOutlier"][ev]) + 1.0)
    assert np.median(relerr) < 2e-4
    assert abs(r["energy"] - E_o) <= 2e-5 * abs(E_o)
    np.testing.assert_allclose(g["centerProjectedTo"][ev], o["centerProjectedTo"][ev], rtol=1e-5, atol=2e-4)
    # ---- commit, then per-residual JpJdF and per-point accumulations
    ow.apply_res()
    ba.apply_res()
    o2 = ow.res_outputs(False)
    act = o2["isActive"] == 1
    scale = np.abs(o2["JpJdF"][act]).max()
    assert np.abs(g["JpJdF"][act] - o2["JpJdF"][act]).max() <= 2e-3 * scale
    assert np.median(np.abs(g["JpJdF"][act] - o2["JpJdF"][act])) <= 2e-5 * scale
    a_o = ow.accumulate(1)
    a_g = ba.accumulate()
    po, pg = ow.point_outputs(), ba.point_outputs()
    assert a_g["resInA"] == a_o["resInA"]
    for k in ("Hdd", "bd", "HdiF", "bdSumF"):
        np.testing.assert_allclose(pg[k], po[k], rtol=2e-3, atol=2e-4 * np.abs(po[k]).max())
    assert rel(a_g["HA"], a_o["HA"]) < 1e-5
    assert rel(a_g["bA"], a_o["bA"]) < 1e-4
    assert rel(a_g["Hsc"], a_o["Hsc"]) < 1e-5
    assert rel(a_g["bsc"], a_o["bsc"]) < 1e-4
    # invariants that hold regardless of ties
    assert np.abs(a_g["HA"] - a_g["HA"].T).max() <= 1e-9 * np.abs(a_g["HA"]).max()
    assert np.abs(a_g["Hsc"] - a_g["Hsc"].T).max() <= 1e-9 * np.abs(a_g["Hsc"]).max()
    return g, pg, a_g


def activation_case(synth, orc, seed=9, nf=5, n=2000, **kw):
    """A window plus immature points with depth intervals (half of them wide, half narrow) for the point-activation tests."""
    W = synth.make_window(nf=nf, npts=50, seed=seed, trans=0.06, rot=0.01, **kw)
    w, h = W["w"], W["h"]
    rng = np.random.default_rng(seed)
    host = np.sort(rng.integers(0, nf, n)).astype(np.int32)
    u, v = rng.integers(10, w - 10, n), rng.integers(10, h - 10, n)
    parts = [orc.ip_init(W["dI"][hh], w, h, u[host == hh], v[host == hh]) for hh in range(nf)]
    P = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    idt = (0.5 * (1 + 0.02 * rng.standard_normal(n))).astype(np.float32)
    wide = rng.random(n) < 0.5
    P["idepth_min"] = (idt * np.where(wide, 0.7, 0.97)).astype(np.float32)
    P["idepth_max"] = (idt * np.where(wide, 1.4, 1.03)).astype(np.float32)
    bad = rng.random(n) < 0.03            # a few hopeless intervals: far from the truth
    P["idepth_min"][bad] *= 3; P["idepth_max"][bad] *= 3
    return W, host, P


def init_points(rng, w, h, levels, counts):
    """points per level the way CoarseInitializer::setFirst lays them out (integer pixel + 0.1 inside the pattern margin, row-major order), with
    brute-force 10 nearest neighbours and the nearest parent one level up (CoarseInitializer::makeNN's outputs, without its kd-tree)"""
    pts = []
    for l in range(levels):
        wl, hl = w >> l, h >> l
        n = counts[l]
        x = rng.integers(3, wl - 4, 4 * n); y = rng.integers(3, hl - 4, 4 * n)
        xy = np.unique(np.stack([y, x], 1), axis=0)                       # row-major order, no duplicates
        xy = xy[np.sort(rng.choice(len(xy), min(n, len(xy)), replace=False))]
        pts.append(dict(u=(xy[:, 1] + 0.1).astype(np.float32), v=(xy[:, 0] + 0.1).astype(np.float32), type=np.ones(len(xy), np.float32)))
    for l in range(levels):
        p = pts[l]
        P = np.stack([p["u"], p["v"]], 1).astype(np.float64)
        d = ((P[:, None, :] - P[None, :, :]) ** 2).sum(-1)
        np.fill_diagonal(d, np.inf)
        k = min(10, len(P) - 1)
        nb = np.full((len(P), 10), -1, np.int32)
        nb[:, :k] = np.argsort(d, axis=1, kind="stable")[:, :k]
        p["neighbours"] = nb
        if l + 1 < levels:
            Q = np.stack([pts[l + 1]["u"], pts[l + 1]["v"]], 1).astype(np.float64)
            dq = ((0.5 * P[:, None, :] - Q[None, :, :]) ** 2).sum(-1)
            p["parent"] = np.argmin(dq, axis=1).astype(np.int32)
        else:
            p["parent"] = np.full(len(P), -1, np.int32)
    return pts

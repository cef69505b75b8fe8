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


# ---------------------------------------------------------------------------------------------------------------------------------
# fp64 reference of CoarseTracker::calcRes + calcGSSSE and of the visual branch of trackNewestCoarse (oracle/orc_coarse.cpp:L169-435)
# ---------------------------------------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24          # unit roundoff of fp32
CT_MAXIT = (10, 20, 50, 50, 50)
CT_SCALE = np.array([1, 1, 1, 1, 1, 1, 10.0, 1000.0])   # SCALE_XI_ROT/TRANS = 1, SCALE_A, SCALE_B


def _f32_inv3(M):
    """3x3 inverse with Eigen's fixed-size rounding: cofactors times one fp32 reciprocal of the determinant, every step rounded to fp32"""
    f = np.float32
    M = np.asarray(M, f)

    def cof(i, j):
        i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
        return f(f(M[i1, j1] * M[i2, j2]) - f(M[i1, j2] * M[i2, j1]))

    C = np.array([[cof(j, i) for j in range(3)] for i in range(3)], f)      # C[i][j] = cofactor (j, i): the adjugate
    det = f(f(f(C[0, 0] * M[0, 0]) + f(C[0, 1] * M[1, 0])) + f(C[0, 2] * M[2, 0]))
    return (C * f(f(1) / det)).astype(f)


def _f32_mm3(A, B):
    """3x3 fp32 product with Eigen's fixed-size inner-product order ((a0 b0 + a1 b1) + a2 b2), every step rounded to fp32"""
    A, B = np.asarray(A, np.float32), np.asarray(B, np.float32)
    return ((A[:, 0:1] * B[0:1, :] + A[:, 1:2] * B[1:2, :]) + A[:, 2:3] * B[2:3, :]).astype(np.float32)


def ct_Ki(k4):
    """K[lvl].inverse() in fp32 as the reference rounds it (CoarseTracker.cpp:L128)"""
    return _f32_inv3(np.array([[k4[0], 0, k4[2]], [0, k4[1], k4[3]], [0, 0, 1]], np.float32))


def ct_operands(R, t, a, b, Ki, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0):
    """the fp32 operands of calcRes (CoarseTracker.cpp:L377-379): RKi = R.cast<float>() * Ki, t.cast<float>(), affLL (fromToVecExposure)"""
    eF, eT = float(np.float32(ref_exposure)), float(np.float32(new_exposure))
    if eF == 0 or eT == 0:
        eF = eT = 1.0
    aa = np.exp(a - ref_a) * eT / eF
    return (_f32_mm3(np.asarray(R, np.float64).astype(np.float32), Ki), np.asarray(t, np.float64).astype(np.float32),
            np.array([aa, b - aa * ref_b], np.float32))


def _proj_bound(M, t, x, y, idp, fx, fy, cx, cy, form=None):
    """fp64 projection K * (M [x y 1]^T + t id) / z of fp32 operands, and a first-order bound of the fp32 evaluation's error in Ku, Kv, 1/z.
    Each term of a row passes through at most 4 roundings (one product, three adds); `form` adds the rounding of forming M itself."""
    P = M[:, 0:1] * x + M[:, 1:2] * y + M[:, 2:3] + t[:, None] * idp
    S = np.abs(M[:, 0:1] * x) + np.abs(M[:, 1:2] * y) + np.abs(M[:, 2:3]) + np.abs(t[:, None] * idp)
    dP = 4 * U32 * S
    if form is not None:
        dP = dP + U32 * (form[:, 0:1] * np.abs(x) + form[:, 1:2] * np.abs(y) + form[:, 2:3] + np.abs(t[:, None] * idp))
    z = P[2]
    uu, vv = P[0] / z, P[1] / z
    du = (dP[0] + np.abs(uu) * dP[2]) / np.abs(z) + U32 * np.abs(uu)
    dv = (dP[1] + np.abs(vv) * dP[2]) / np.abs(z) + U32 * np.abs(vv)
    Ku, Kv = fx * uu + cx, fy * vv + cy
    dKu = fx * du + 2 * U32 * (np.abs(fx * uu) + abs(cx))
    dKv = fy * dv + 2 * U32 * (np.abs(fy * vv) + abs(cy))
    return uu, vv, z, du, dv, dP[2], Ku, Kv, dKu, dKv


def calc_res_ref(pts, plane, k4, Ki, RKi, t, affLL, b0, cutoff, lvl, huber=9.0, depth=None, R=None):
    """One calcRes + calcGSSSE in fp64 from the same fp32 points, plane and operands (oracle/orc_coarse.cpp:L179-334).

    Returns E, nE, nSat, nW (unpadded), npad, res6 (the Vec6 of calcRes), H (8x8), b (8) exactly as calcGSSSE returns them, and a first-order
    bound of what an fp32 evaluation of the same formulas may differ by: dE, dH, db, dflow (for res6[2], res6[4]).  The bound sums, per point,
    the rounding of the projection (times the plane's slope in the cell) and of every later fp32 operation, plus `depth` fp32 additions per
    term for the summation order (default: the kernels' 5 butterfly adds + one per point a thread of a 4-CTA cluster takes).  Points within
    their bound of the border, cutoff or new_idepth > 0 tests are `amb`iguous and count in full in every bound.  R (fp64 rotation of the
    pose) adds the rounding of forming RKi = R.cast<float>() * Ki when RKi was formed by someone else."""
    f = np.float64
    x, y, idp, col = (np.asarray(pts[k], np.float32).astype(f) for k in ("u", "v", "idepth", "color"))
    n = len(x)
    if depth is None:
        depth = 5 + -(-n // 2048)
    hl, wl = plane.shape[:2]
    fx, fy, cx, cy = (float(np.float32(v)) for v in k4)
    M = np.asarray(RKi, np.float32).astype(f).reshape(3, 3)
    tt = np.asarray(t, np.float32).astype(f)
    form = None if R is None else 4 * (np.abs(np.asarray(R, f)) @ np.abs(np.asarray(Ki, np.float32).astype(f)))   # cast of R + 3-term fp32 sum
    uu, vv, z, du, dv, dz, Ku, Kv, dKu, dKv = _proj_bound(M, tt, x, y, idp, fx, fy, cx, cy, form)
    nid = idp / z
    dnid = np.abs(nid) * (dz / np.abs(z) + U32)
    inb = (Ku > 2) & (Kv > 2) & (Ku < wl - 3) & (Kv < hl - 3) & (nid > 0)
    amb_b = ((np.abs(Ku - 2) <= dKu) | (np.abs(Ku - (wl - 3)) <= dKu) | (np.abs(Kv - 2) <= dKv) | (np.abs(Kv - (hl - 3)) <= dKv) | (np.abs(nid) <= dnid))
    ev = inb | amb_b
    # bilinear gather (util/globalFuncs.h getInterpolatedElement33) of the 3 channels, the slope of each channel in the cell, its rounding
    ix = np.clip(np.floor(np.where(ev, Ku, 3.0)), 0, wl - 2).astype(np.int64)
    iy = np.clip(np.floor(np.where(ev, Kv, 3.0)), 0, hl - 2).astype(np.int64)
    dx, dy = np.where(ev, Ku, 3.0) - ix, np.where(ev, Kv, 3.0) - iy
    P64 = plane.astype(f)
    tl, tr, bl, br = P64[iy, ix], P64[iy, ix + 1], P64[iy + 1, ix], P64[iy + 1, ix + 1]
    w11, w10, w01 = dx * dy, dy - dx * dy, dx - dx * dy
    w00 = 1 - dx - dy + dx * dy
    hc = w11[:, None] * br + w10[:, None] * bl + w01[:, None] * tr + w00[:, None] * tl
    Gu = np.maximum(np.abs(tr - tl), np.abs(br - bl))
    Gv = np.maximum(np.abs(bl - tl), np.abs(br - tr))
    dh = Gu * dKu[:, None] + Gv * dKv[:, None] + 12 * U32 * (np.abs(tl) + np.abs(tr) + np.abs(bl) + np.abs(br))   # 4 weights (<= 4 roundings) x 4 taps
    a_, b_ = float(affLL[0]), float(affLL[1])
    r = hc[:, 0] - (a_ * col + b_)
    ar = np.abs(r)
    dr = dh[:, 0] + 2 * U32 * (np.abs(a_ * col) + abs(b_)) + U32 * ar
    cutoff = float(np.float32(cutoff))
    huber = float(np.float32(huber))
    maxE = float(np.float32(np.float32(2) * np.float32(huber) * np.float32(cutoff) - np.float32(huber) * np.float32(huber)))
    amb = ev & (amb_b | (np.abs(ar - cutoff) <= dr))
    sat = inb & (ar > cutoff)
    good = inb & ~sat
    hw = np.where(ar < huber, 1.0, huber / np.maximum(ar, 1e-30))
    e = np.where(sat, maxE, hw * r * r * (2 - hw))
    de = np.where(sat, 0.0, 2 * np.minimum(ar, huber) * dr + 5 * U32 * e)
    dhw = np.where(ar < huber, 0.0, hw * dr / np.maximum(ar, 1e-30) + U32 * hw)
    # Jacobian row of calcGSSSE (CoarseTracker.cpp:L316-336) and first-order bounds of its fp32 evaluation
    gx, gy = hc[:, 1] * fx, hc[:, 2] * fy
    dgx, dgy = fx * dh[:, 1] + U32 * np.abs(gx), fy * dh[:, 2] + U32 * np.abs(gy)
    J = np.zeros((9, n)); dJ = np.zeros((9, n))
    J[0], J[1] = nid * gx, nid * gy
    dJ[0] = np.abs(nid) * dgx + np.abs(gx) * dnid + U32 * np.abs(J[0])
    dJ[1] = np.abs(nid) * dgy + np.abs(gy) * dnid + U32 * np.abs(J[1])
    s2 = uu * gx + vv * gy
    J[2] = -nid * s2
    dJ[2] = np.abs(nid) * (np.abs(uu) * dgx + np.abs(gx) * du + np.abs(vv) * dgy + np.abs(gy) * dv + 3 * U32 * (np.abs(uu * gx) + np.abs(vv * gy))) + dnid * np.abs(s2) + U32 * np.abs(J[2])
    J[3] = -((uu * vv) * gx + gy * (1 + vv * vv))
    dJ[3] = (np.abs(vv) * du + np.abs(uu) * dv) * np.abs(gx) + np.abs(uu * vv) * dgx + (1 + vv * vv) * dgy + 2 * np.abs(gy * vv) * dv + 5 * U32 * (np.abs(uu * vv * gx) + np.abs(gy) * (1 + vv * vv))
    J[4] = (uu * vv) * gy + gx * (1 + uu * uu)
    dJ[4] = (np.abs(vv) * du + np.abs(uu) * dv) * np.abs(gy) + np.abs(uu * vv) * dgy + (1 + uu * uu) * dgx + 2 * np.abs(gx * uu) * du + 5 * U32 * (np.abs(uu * vv * gy) + np.abs(gx) * (1 + uu * uu))
    J[5] = uu * gy - vv * gx
    dJ[5] = du * np.abs(gy) + np.abs(uu) * dgy + dv * np.abs(gx) + np.abs(vv) * dgx + 3 * U32 * (np.abs(uu * gy) + np.abs(vv * gx))
    a_gs, b0 = float(np.float32(affLL[0])), float(np.float32(b0))
    J[6] = a_gs * (b0 - col)
    dJ[6] = 2 * U32 * np.abs(J[6])
    J[7] = -1.0
    J[8], dJ[8] = r, dr
    iu = np.triu_indices(9)
    Pk = J[iu[0]] * hw * J[iu[1]]                                                          # the 45 entries of the weighted outer product
    dPk = hw * (np.abs(J[iu[0]]) * dJ[iu[1]] + np.abs(J[iu[1]]) * dJ[iu[0]]) + np.abs(J[iu[0]] * J[iu[1]]) * dhw + 2 * U32 * np.abs(Pk)
    order = depth * U32 + n * 2.0 ** -53
    gm, am = good & ~amb, ev & amb & (ar <= cutoff)
    S = (Pk * good).sum(1)
    dS = (dPk * gm).sum(1) + order * (np.abs(Pk) * good).sum(1) + (np.abs(Pk) * am).sum(1)
    E = float((e * inb).sum())
    dE = float((de * (inb & ~amb)).sum() + order * (np.abs(e) * inb).sum() + (np.maximum(e, maxE) * amb).sum())
    nE, nSat, nW, namb = int(inb.sum()), int(sat.sum()), int(good.sum()), int(amb.sum())
    # flow indicators (L416-447): every 32nd point at level 0, whether it projects into the image or not
    res6 = np.zeros(6)
    dflow = np.zeros(2)
    if lvl == 0 and n > 0:
        s = np.arange(0, n, 32)
        K64 = np.asarray(Ki, np.float32).astype(f)
        xs, ys, ids = x[s], y[s], idp[s]
        pr = [_proj_bound(K64, tt, xs, ys, ids, fx, fy, cx, cy), _proj_bound(K64, -tt, xs, ys, ids, fx, fy, cx, cy),
              _proj_bound(M, tt, xs, ys, ids, fx, fy, cx, cy, form), _proj_bound(M, -tt, xs, ys, ids, fx, fy, cx, cy, form)]
        terms, dterms = [], []
        for q in pr:
            ex, ey = q[6] - xs, q[7] - ys
            terms.append(ex * ex + ey * ey)
            dterms.append(2 * np.abs(ex) * q[8] + 2 * np.abs(ey) * q[9] + 3 * U32 * (ex * ex + ey * ey))
        num = 2.0 * len(s)
        fT, fRT = terms[0] + terms[1], terms[2] + terms[3]
        res6[2], res6[4] = fT.sum() / (num + 0.1), fRT.sum() / (num + 0.1)
        ordf = (depth + 1) * U32 + len(s) * 2.0 ** -53
        dflow[0] = ((dterms[0] + dterms[1]).sum() + ordf * fT.sum()) / (num + 0.1) + 4 * U32 * res6[2]
        dflow[1] = ((dterms[2] + dterms[3]).sum() + ordf * fRT.sum()) / (num + 0.1) + 4 * U32 * res6[4]
    res6[0], res6[1] = E, nE
    res6[5] = float(np.float32(nSat) / np.float32(nE)) if nE else np.nan
    npad = (nW + 3) & ~3
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = float(np.float32(1) / np.float32(npad))
        M9, dM9 = np.zeros((9, 9)), np.zeros((9, 9))
        M9[iu], dM9[iu] = S, dS
        M9, dM9 = np.triu(M9) + np.triu(M9, 1).T, np.triu(dM9) + np.triu(dM9, 1).T
        rel_inv = 0.0 if namb == 0 else (namb + 3) / max(nW - namb, 1)
        H = M9[:8, :8] * inv * CT_SCALE[:, None] * CT_SCALE[None, :]
        b = M9[:8, 8] * inv * CT_SCALE
        dH = dM9[:8, :8] * inv * CT_SCALE[:, None] * CT_SCALE[None, :] + np.abs(H) * rel_inv
        db = dM9[:8, 8] * inv * CT_SCALE + np.abs(b) * rel_inv
    return dict(E=E, nE=nE, nSat=nSat, nW=nW, npad=npad, res6=res6, H=H, b=b, dE=dE, dH=dH, db=db, dflow=dflow, amb=namb)


def ct_mean_bound(c):
    """relative bound of E/nE from calc_res_ref's bounds"""
    if c["nE"] == 0 or c["E"] == 0:
        return np.inf
    return c["dE"] / c["E"] + c["amb"] / max(c["nE"] - c["amb"], 1)


def track_ref(sc, R0, t0, a0, b0, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0, cutoff=20.0, affA=1e12, affB=1e8, coarsest=None,
              minRes=None, depth=None):
    """CoarseTracker::trackNewestCoarse, visual branch (oracle/orc_coarse.cpp:L336-435), in fp64 on calc_res_ref; the LM system (or its 6x6 / 7x7
    sub-system when affine parameters are fixed) is solved in fp64.  sc: scene dict (pts[l], planes[l], k4[l], Ki[l]).

    Logs every evaluation (level, rep, pose, E/nE and its relative bound, saturation, accept, incNorm) and the margin of every decision;
    `decidable` is True when each margin exceeds the error bounds: accept ratio vs 1 by more than 10x the two evaluations' relative bounds,
    incNorm vs 1e-3 by more than 1 %, saturation vs 0.6 (and 0.99) by more than ambiguous/nE, the abort test by more than 1e-4 relative."""
    import dmvio_b200.synth as synth
    L = len(sc["pts"])
    coarsest = L - 1 if coarsest is None else coarsest
    minRes = np.full(5, np.nan) if minRes is None else np.asarray(minRes, np.float64)
    huber = sc.get("huber", 9.0)
    fixA, fixB = affA < 0, affB < 0
    free = [i for i in range(8) if not ((i == 6 and fixA) or (i == 7 and fixB))]
    R, t, a, b = np.asarray(R0, np.float64).reshape(3, 3).copy(), np.asarray(t0, np.float64).copy(), float(a0), float(b0)
    log, bad = [], []
    lastRes, flow = np.full(5, np.nan), np.full(3, 1000.0)
    its = evals = pevals = 0
    f32 = np.float32

    def ev(lvl, R, t, a, b, rep):
        nonlocal evals, pevals
        RKi, tf, affLL = ct_operands(R, t, a, b, sc["Ki"][lvl], ref_a, ref_b, ref_exposure, new_exposure)
        c = calc_res_ref(sc["pts"][lvl], sc["planes"][lvl], sc["k4"][lvl], sc["Ki"][lvl], RKi, tf, affLL, ref_b, f32(cutoff) * f32(rep), lvl, huber,
                         depth, R=R)
        evals += 1
        pevals += len(sc["pts"][lvl]["u"])
        with np.errstate(divide="ignore", invalid="ignore"):
            c["mean"] = c["E"] / c["nE"]
        c["rel"] = ct_mean_bound(c)
        return c

    def margin(ok, what, **kw):
        if not ok:
            bad.append(dict(what=what, **kw))

    status, haveRepeated, lvl = 0, False, coarsest
    while lvl >= 0:
        rep = f32(1)
        old = ev(lvl, R, t, a, b, rep)
        log.append(dict(kind="init", lvl=lvl, rep=float(rep), R=R.copy(), t=t.copy(), a=a, b=b, mean=old["mean"], rel=old["rel"], sat=old["res6"][5]))
        while True:
            s5, ambr = old["res6"][5], old["amb"] / max(old["nE"], 1)
            if old["nE"]:
                margin(abs(s5 - 0.6) > ambr, "saturation", lvl=lvl, sat=s5, amb=ambr)
                if rep >= 50:
                    margin(abs(s5 - 0.99) > ambr, "saturation99", lvl=lvl, sat=s5, amb=ambr)
            if s5 > 0.6 and (rep < 50 or s5 > 0.99):
                rep = f32(rep * 2)
                old = ev(lvl, R, t, a, b, rep)
                log.append(dict(kind="double", lvl=lvl, rep=float(rep), R=R.copy(), t=t.copy(), a=a, b=b, mean=old["mean"], rel=old["rel"], sat=old["res6"][5]))
            else:
                break
        H, bb = old["H"], old["b"]
        lam = f32(0.01)
        for it in range(CT_MAXIT[lvl]):
            its += 1
            Hl = H.copy()
            Hl[np.diag_indices(8)] *= float(f32(1) + lam)
            extrap = f32(1)
            if lam < f32(0.001):
                extrap = f32(np.sqrt(np.sqrt(f32(0.001) / lam, dtype=f32), dtype=f32))
            inc = np.zeros(8)
            with np.errstate(all="ignore"):
                try:
                    inc[free] = np.linalg.solve(Hl[np.ix_(free, free)], -bb[free])
                except np.linalg.LinAlgError:
                    inc[free] = np.nan
            inc *= float(extrap)
            incS = inc * CT_SCALE
            if not np.isfinite(incS.sum()):
                incS[:] = 0
            Re, te = synth.se3_exp(incS[:6])
            Rn, tn = Re @ R, Re @ t + te
            an, bn = a + incS[6], b + incS[7]
            incNorm = float(np.sqrt((inc * inc).sum()))
            new = ev(lvl, Rn, tn, an, bn, rep)
            with np.errstate(invalid="ignore"):
                ratio = new["mean"] / old["mean"]
                accept = bool(new["mean"] < old["mean"])
            if np.isfinite(ratio):
                margin(abs(ratio - 1) > 10 * (new["rel"] + old["rel"]), "accept", lvl=lvl, it=it, ratio=ratio, rel=new["rel"] + old["rel"])
            if it + 1 < CT_MAXIT[lvl] and np.isfinite(incNorm):
                margin(abs(incNorm - 1e-3) > 1e-5, "incNorm", lvl=lvl, it=it, incNorm=incNorm)
            log.append(dict(kind="lm", lvl=lvl, rep=float(rep), R=Rn, t=tn, a=an, b=bn, mean=new["mean"], rel=new["rel"], sat=new["res6"][5],
                            accept=accept, incNorm=incNorm, ratio=ratio))
            if accept:
                H, bb, old = new["H"], new["b"], new
                R, t, a, b = Rn, tn, an, bn
                lam = f32(lam * f32(0.5))
            else:
                lam = f32(lam * f32(4))
                if lam < f32(0.001):
                    lam = f32(0.001)
            if not (incNorm > 1e-3):
                break
        with np.errstate(invalid="ignore", divide="ignore"):
            lastRes[lvl] = float(np.sqrt(np.float32(old["E"] / old["nE"]), dtype=np.float32))
        flow[:] = old["res6"][2:5]
        log[-1]["end_level"] = lvl
        if np.isfinite(minRes[lvl]) and np.isfinite(lastRes[lvl]):
            margin(abs(lastRes[lvl] - 1.5 * minRes[lvl]) > 1e-4 * 1.5 * minRes[lvl], "abort", lvl=lvl, lastRes=lastRes[lvl], minRes=minRes[lvl])
        if np.isnan(lastRes[lvl]) or lastRes[lvl] > 1.5 * minRes[lvl]:
            status = 2
            break
        if rep > 1 and not haveRepeated:
            haveRepeated = True
            continue
        lvl -= 1
    good = False
    if status == 0:
        good = True
        if (affA != 0 and abs(f32(a)) > 1.2) or (affB != 0 and abs(f32(b)) > 200):
            good = False
        eF, eT = float(f32(ref_exposure)), float(f32(new_exposure))
        if eF == 0 or eT == 0:
            eF = eT = 1.0
        ra = np.exp(a - ref_a) * eT / eF
        rb = b - ra * ref_b
        if (affA == 0 and abs(np.log(f32(ra))) > 1.5) or (affB == 0 and abs(f32(rb)) > 200):
            good = False
        if fixA:
            a = 0.0
        if fixB:
            b = 0.0
    else:
        R, t, a, b = np.asarray(R0, np.float64).reshape(3, 3), np.asarray(t0, np.float64), float(a0), float(b0)
    return dict(R=R, t=t, a=a, b=b, lastResiduals=lastRes, flow=flow, good=int(good), status=status, iterations=its, evaluations=evals,
                point_evaluations=pevals, log=log, undecided=bad, decidable=not bad)


CT_AFF = dict(R0=None, a0=0.6, b0=4.5, ref_a=0.1, ref_b=3.0, ref_exposure=1.3, new_exposure=0.8)
CT_MODES = dict(free=(1e12, 1e8), fixA=(-1.0, 1e8), fixB=(1e12, -1.0), fixAB=(-1.0, -1.0))
CT_SCENES = ["bench", "aff_free", "aff_fixA", "aff_fixB", "aff_fixAB", "tma0_80x60", "tma0_160x120", "limit", "odd", "wide", "stream", "repeat"]


def _ct_random_points(T, n, seed):
    """n distinct level-0 pixels of the reference plane (depth 2 everywhere) with noisy inverse depths, row-major like makeCoarseDepthL0"""
    rng = np.random.default_rng(seed)
    w, h = T["w"], T["h"]
    sel = np.sort(rng.choice((w - 5) * (h - 5), n, replace=False))
    y, x = 2 + sel // (w - 5), 2 + sel % (w - 5)
    return dict(u=x.astype(np.float32), v=y.astype(np.float32), idepth=(0.5 * (1 + 5e-3 * rng.standard_normal(n))).astype(np.float32),
                color=T["pyr_ref"][0][y, x, 0].astype(np.float32))


def ct_scene(orc, synth, name, npts=None):
    """A coarse-tracking scene: reference points, new-frame planes and intrinsics per level plus the dmv_ct_track arguments.

    bench        640x480, 5 levels, seed 4321 (bench.py config 2): levels 0-2 gather from L2, levels 3-4 are TMA-staged
    aff_<mode>   640x480, 4 levels, start pose not identity, a0, b0, ref_a, ref_b != 0, exposures != 1; affine mode free / fixA / fixB / fixAB
    tma0_*       80x60 with 1 level (level 0 staged), 160x120 with 2 levels
    limit        256x80, 2 levels: level 1 is 128x40 = exactly 80 KiB with 2w = 256, so it is staged
    odd          752x480, 5 levels: level 4 (47x30) is staged with an odd width, level 3 (94x60, 90 240 B) is not.  Seed 20: with seed 14 a
                 level ends on an accept tie that the oracle's fp32 energy sum decides the other way (27 vs 28 iterations)
    wide         640x96, 3 levels: level 2 (160x24) fits in shared memory but not in one tensor-map box, so it is gathered from L2
    stream       640x480, 1 level, 20 001 points (npts): more than 2 register slots per thread of any cluster size
    counts_<n>   1 level with n points
    repeat       the bench scene started with b0 = -21: almost every residual saturates at the coarsest level, so the cutoff doubles and
                 the level is repeated.  Other starts were dropped: b0 = -25 ends a level on an accept tie that the oracle decides the other
                 way; with b0 = -22 the coarsest level stops where its lastResiduals differ by 1.2e-4 between the kernel's and the
                 reference's stopping poses; with b0 = -35 the saturation after the first doubling (0.63) is within its bound of 0.6; with
                 b0 = -50 the kernel decides an accept tie at the coarsest level the other way (25 vs 27 iterations)"""
    args = dict(R0=np.eye(3), t0=np.zeros(3), a0=0.0, b0=0.0, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0, affA=1e12, affB=1e8)
    geo = dict(bench=(640, 480, 5, 4321), repeat=(640, 480, 5, 4321), tma0_80x60=(80, 60, 1, 11), tma0_160x120=(160, 120, 2, 12),
               limit=(256, 80, 2, 13), odd=(752, 480, 5, 20), wide=(640, 96, 3, 15))
    if name.startswith("aff_"):
        w, h, L, seed = 640, 480, 4, 99
        args.update({k: v for k, v in CT_AFF.items() if k != "R0"})
        args["R0"], args["t0"] = synth.se3_exp(np.array([0.005, -0.004, 0.003, 0.002, -0.001, 0.002]))
        args["affA"], args["affB"] = CT_MODES[name[4:]]
    elif name in geo:
        w, h, L, seed = geo[name]
    else:
        w, h, L, seed = 640, 480, 1, 4321
    T = synth.make_tracking_pair(w=w, h=h, seed=seed, levels=L, npts=min(2000, (w - 12) * (h - 12) // 4))
    oc = orc.CoarseTracker(w, h, T["K"], L)
    assert oc.levels == L
    if name == "stream" or name.startswith("counts_") or name.startswith("points_"):
        n = npts if npts is not None else (20001 if name == "stream" else int(name.split("_")[1]))
        pts = [_ct_random_points(T, n, seed=7)]
    else:
        oc.make_coarse_depth(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"], T["pyr_ref"])
        pts = [oc.ref_points(l) for l in range(L)]
    if name == "repeat":
        args["b0"] = -21.0
    k4 = [oc.K(l)[0] for l in range(L)]
    return dict(name=name, w=w, h=h, levels=L, K=T["K"], pts=pts, planes=T["pyr_new"], k4=k4, Ki=[ct_Ki(k) for k in k4], args=args, T=T)


def ct_oracle(orc, sc):
    """the CPU oracle's CoarseTracker loaded with the scene's points, frame and settings"""
    a = sc["args"]
    oc = orc.CoarseTracker(sc["w"], sc["h"], sc["K"], sc["levels"], settings=dict(affineOptModeA=a["affA"], affineOptModeB=a["affB"]))
    for l, p in enumerate(sc["pts"]):
        oc.set_ref_points(l, p["u"], p["v"], p["idepth"], p["color"])
    oc.set_new_frame(sc["planes"], a["ref_exposure"], a["new_exposure"], a["ref_a"], a["ref_b"])
    return oc


def ct_track_ref(sc, **kw):
    a = dict(sc["args"])
    a.update(kw)
    return track_ref(sc, a["R0"], a["t0"], a["a0"], a["b0"], a["ref_a"], a["ref_b"], a["ref_exposure"], a["new_exposure"], affA=a["affA"],
                     affB=a["affB"], coarsest=a.get("coarsest"), minRes=a.get("minRes"))

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


HARD_LABELS = ("none", "nan", "flat", "border", "behind")
HARD_DESIGNED = dict(nan=RES_OOB, flat=RES_OUTLIER, border=RES_OOB, behind=RES_OOB)   # the state each exit of PointFrameResidual::linearize gives
HARD_MARGIN = 1e-3      # px: no projected coordinate of a labelled residual lies closer than this to a bound or a texel boundary


def make_images_level0(img):
    """FrameHessian::makeImages' level 0 (HessianBlocks.cpp:L169-179) of an intensity image: [I, dx, dy] with central differences on the flat
    pixel index (row ends wrap into the neighbouring rows), a non-finite gradient set to 0, the first and last rows' gradients 0"""
    import dmvio_b200.synth as synth
    with np.errstate(invalid="ignore"):
        d = synth.make_pyramid(img, 1)[0].copy()
    d[..., 1:][~np.isfinite(d[..., 1:])] = 0.0
    return d


def _plane_coords(synth, W, k, D=2.0, tex_size=1536):
    """texture coordinates (s, t) of frame k's pixels on synth.make_window's world plane Z = D, and their depths, at the pose the frame's
    state gives (exp(state[:6]) * evalPT: within 1e-3 of the pose it was rendered at)"""
    w, h = W["w"], W["h"]
    fx, fy, cx, cy = W["K"]
    R, t = synth.se3_mul(*synth.se3_exp(W["state"][k, :6]), W["R_eval"][k], W["t_eval"][k])
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    rw = np.stack([(xs - cx) / fx, (ys - cy) / fy, np.ones_like(xs)], axis=-1) @ R
    cw = -R.T @ t
    lam = (D - cw[2]) / rw[..., 2]
    tpu = fx / D
    return (cw[0] + lam * rw[..., 0]) * tpu + tex_size / 2, (cw[1] + lam * rw[..., 1]) * tpu + tex_size / 2, lam


def hard_labels(W, pc):
    """Per residual, in fp64 from the fp32 tables pc (orc.Window.precalc(), pair h * nf + t) and the window's dI, which exit of
    PointFrameResidual::linearize (Residuals.cpp:L108-273) it takes, in the reference's order:
      behind  the FEJ centre (idepth_zero) has drescale <= 0;
      border  the centre or one of the 8 pattern pixels (idepth) projects outside 1.1 < Ku < w - 3, 1.1 < Kv < h - 3;
      nan     a pattern sample's 2x2 bilinear footprint holds a non-finite intensity;
      flat    every footprint texel has zero gradient: wJI2_sum = 0 < 2;
      none    none of these.
    Returns (labels, tie, foot): tie marks residuals with a deciding coordinate within HARD_MARGIN of its bound, or a sample within
    HARD_MARGIN of a texel boundary next to a non-finite texel; foot[i, j] is sample j's top-left footprint texel (x, y)."""
    import dmvio_b200.synth as synth
    w, h, nf = W["w"], W["h"], W["nf"]
    fx, fy, cx, cy = (float(np.float32(k)) for k in W["K"])
    rp, rt = np.asarray(W["res_point"]), np.asarray(W["res_target"])
    hh = np.asarray(W["host"])[rp]
    T = np.asarray(pc, np.float32).astype(np.float64)[hh * nf + rt]
    u, v = (np.asarray(W[k], np.float32).astype(np.float64)[rp] for k in ("u", "v"))
    idp, idz = (np.asarray(W[k], np.float32).astype(np.float64)[rp] for k in ("idepth", "idepth_zero"))
    lo, hu, hv = 1.1, w - 3.0, h - 3.0
    Kl0, Kl1 = (u - cx) / fx, (v - cy) / fy
    q2 = T[:, 18] * Kl0 + T[:, 19] * Kl1 + T[:, 20] + T[:, 23] * idz
    with np.errstate(divide="ignore", invalid="ignore"):
        cKu = (T[:, 12] * Kl0 + T[:, 13] * Kl1 + T[:, 14] + T[:, 21] * idz) / q2 * fx + cx
        cKv = (T[:, 15] * Kl0 + T[:, 16] * Kl1 + T[:, 17] + T[:, 22] * idz) / q2 * fy + cy
    pu = u[:, None] + synth.PATTERN[None, :, 0]
    pv = v[:, None] + synth.PATTERN[None, :, 1]
    r2 = T[:, 6:7] * pu + T[:, 7:8] * pv + T[:, 8:9] + T[:, 11:12] * idp[:, None]
    Ku = (T[:, 0:1] * pu + T[:, 1:2] * pv + T[:, 2:3] + T[:, 9:10] * idp[:, None]) / r2
    Kv = (T[:, 3:4] * pu + T[:, 4:5] * pv + T[:, 5:6] + T[:, 10:11] * idp[:, None]) / r2

    def inside(a, b):
        return (a > lo) & (b > lo) & (a < hu) & (b < hv)

    def near(a):
        return (np.abs(a - lo) < HARD_MARGIN) | (np.abs(a - hu) < HARD_MARGIN) | (np.abs(a - hv) < HARD_MARGIN)

    behind = ~(q2 > 0)
    c_in = inside(cKu, cKv)
    p_in = inside(Ku, Kv).all(1)
    border = ~behind & ~(c_in & p_in)
    tie = np.abs(q2) < 1e-4
    tie |= ~behind & (near(cKu) | near(cKv) | near(Ku).any(1) | near(Kv).any(1))
    # footprints of the samples of the residuals that project inside
    ok = ~behind & ~border
    ix = np.where(ok[:, None], np.floor(Ku), 2).astype(np.int64)
    iy = np.where(ok[:, None], np.floor(Kv), 2).astype(np.int64)
    nan, flat = np.zeros(len(rp), bool), np.ones(len(rp), bool)
    for t in range(nf):
        m = rt == t
        if not m.any():
            continue
        dI = np.asarray(W["dI"][t], np.float32).reshape(h, w, 3)
        bad = ~np.isfinite(dI[..., 0])
        grad0 = (dI[..., 1] == 0) & (dI[..., 2] == 0)
        x, y = ix[m], iy[m]
        taps = [(y, x), (y, x + 1), (y + 1, x), (y + 1, x + 1)]
        nan[m] = np.any([bad[a, b] for a, b in taps], axis=0).any(1)
        flat[m] = np.all([grad0[a, b] for a, b in taps], axis=0).all(1)
        # a sample within HARD_MARGIN of a texel boundary next to a non-finite texel: fp32 may take the neighbouring footprint
        fu, fv = Ku[m] - x, Kv[m] - y
        edge = (np.minimum(fu, 1 - fu) < HARD_MARGIN) | (np.minimum(fv, 1 - fv) < HARD_MARGIN)
        pad = np.pad(bad, 1)
        near_bad = np.any([pad[y + 1 + a, x + 1 + b] for a in range(-1, 3) for b in range(-1, 3)], axis=0)
        tie[m] |= ok[m] & (edge & near_bad).any(1)
    labels = np.full(len(rp), "none", dtype="<U6")
    labels[ok & flat] = "flat"
    labels[ok & nan] = "nan"
    labels[border] = "border"
    labels[behind] = "behind"
    return labels, tie, np.stack([ix, iy], -1)


def hard_window(synth, orc, cfg, seed_offset=202):
    """edge_window(cfg) with what real sequences bring and synth.make_window never does (labels of every residual: hard_labels):
      * lighting: exposures in [0.6, 1.6], affine a in [-0.3, 0.3] and b in [-30, 30]; frame k is rendered as e_k exp(a_k) tex + b_k
        (AffLight::fromToVecExposure's model) and clipped to [0, 255], so that 3-7 % of the pixels saturate into flat bright areas;
      * two flat squares of the world plane (tex = 128): zero gradient wherever they are seen, in every frame;
      * in the targets 1 .. nf-1: a NaN block, a NaN row, a +inf column and single NaN texels, each in the footprint of exactly one pattern
        sample j of some residual, for every j in 0..7 (the LPR = 4 launch: one lane of the four sees it);
      * points 2-4 px from each border (half of them with idepth_zero far from idepth, so that the centre and the pattern disagree),
        points whose idepth_zero puts the FEJ centre behind the camera (inside the image, so only drescale > 0 rejects it) while idepth > 0,
        points with idepth = 0 and with idepth < 0.
    Host colours and weights come from the clean relit images; W["images"] holds the intensities (NaN, inf included) and W["dI"] their
    makeImages level 0.  A residual with a deciding coordinate within HARD_MARGIN px of its bound enters as OOB (none is expected).
    Adds W["labels"], W["single_nan"] (residual, sample j) pairs and W["hard_points"] (border, reverse, behind, zero, negative)."""
    W = edge_window(synth, cfg)
    rng = np.random.default_rng(cfg["seed"] + seed_offset)
    w, h, nf = W["w"], W["h"], W["nf"]
    npts = len(W["host"])
    # ---- lighting
    e = rng.uniform(0.6, 1.6, nf).astype(np.float32)
    A, B = rng.uniform(-0.3, 0.3, nf), rng.uniform(-30, 30, nf)
    dz = W["state_zero"][:, 6:8] - W["state"][:, 6:8]
    flat = rng.uniform(700, 836, (2, 2))      # texture coordinates of the flat squares' centres: in view of every frame
    for k in range(nf):
        a0, b0 = W["state"][k, 6] * synth.SCALE_A, W["state"][k, 7] * synth.SCALE_B
        T = (W["images"][k].astype(np.float64) - b0) / np.exp(a0)
        s, t, _ = _plane_coords(synth, W, k)
        for (sc, tc) in flat:
            T[(np.abs(s - sc) < 40) & (np.abs(t - tc) < 40)] = 128.0
        W["images"][k] = np.clip(float(e[k]) * np.exp(A[k]) * T + B[k], 0, 255).astype(np.float32)
    W["exposure"] = e
    W["state"][:, 6], W["state"][:, 7] = A / synth.SCALE_A, B / synth.SCALE_B
    W["state_zero"][:, 6:8] = W["state"][:, 6:8] + dz
    # ---- geometry: border points (and their depth on the plane), idepth = 0 and < 0
    host = W["host"]
    cand = rng.permutation(npts)
    nb = max(8, npts // 12)
    border, behind_c, zero, neg = cand[:nb], cand[nb:2 * nb], cand[2 * nb:2 * nb + npts // 100 + 2], cand[2 * nb + npts // 100 + 2:2 * nb + npts // 50 + 4]
    side = rng.integers(0, 4, nb)
    dist = rng.integers(2, 5, nb)
    u, v = W["u"], W["v"]
    u[border] = np.where(side == 0, dist, np.where(side == 1, np.minimum(w - 1 - dist, w - 4), u[border]))
    v[border] = np.where(side == 2, dist, np.where(side == 3, np.minimum(h - 1 - dist, h - 4), v[border]))
    depth = {k: _plane_coords(synth, W, k)[2] for k in np.unique(host[border])}
    for p in border:
        W["idepth"][p] = np.float32(1.0 / depth[host[p]][int(v[p]), int(u[p])] * (1 + 1e-2 * rng.standard_normal()))
    W["idepth_zero"][border] = W["idepth"][border]
    reverse = border[::2]
    W["idepth_zero"][reverse] = (W["idepth"][reverse] * rng.uniform(0.3, 1.7, len(reverse))).astype(np.float32)
    W["idepth"][zero] = 0.0
    W["idepth_zero"][zero] = 0.0
    W["idepth"][neg] = -rng.uniform(0.02, 0.2, len(neg)).astype(np.float32)
    W["idepth_zero"][neg] = W["idepth"][neg]
    # ---- host colours and weights from the clean relit images (makeImages' level 0: [I, dx, dy])
    clean = [make_images_level0(img) for img in W["images"]]
    for k in range(nf):
        m = host == k
        for j in range(8):
            c, gx, gy = synth.interp33_bilin(clean[k], u[m] + synth.PATTERN[j, 0], v[m] + synth.PATTERN[j, 1])
            W["color"][m, j] = c
            W["weights"][m, j] = np.sqrt(np.float32(2500.0) / (np.float32(2500.0) + gx * gx + gy * gy))
    W["dI"] = [d.reshape(-1).copy() for d in clean]
    pc = orc.Window(W).precalc()       # the tables depend on the frames alone: points and images may change below
    # ---- FEJ centre behind the camera: idepth_zero on the far side of q2 = 0 for one target, the centre still inside the image
    fx, fy, cx, cy = (float(k) for k in W["K"])

    def behind_idz(p):
        Kl = np.array([(u[p] - cx) / fx, (v[p] - cy) / fy, 1.0])
        for t in rng.permutation(nf):
            T = pc[host[p] * nf + t].astype(np.float64)
            a2, b2 = T[18:21] @ Kl, T[23]
            if t == host[p] or abs(b2) < 1e-3:
                continue
            for s in (0.05, 0.1, 0.2, 0.5, 1.0, 2.0, 5.0):
                z = -(a2 + s) / b2                            # q2 = -s
                cu = -(T[12:15] @ Kl + T[21] * z) / s * fx + cx
                cv = -(T[15:18] @ Kl + T[22] * z) / s * fy + cy
                if 3 < cu < w - 5 and 3 < cv < h - 5:
                    return z
        return None

    behind = []
    for p in behind_c:
        z = behind_idz(p)
        if z is not None:
            W["idepth_zero"][p] = np.float32(z)
            behind.append(p)
    behind = np.array(behind, np.int64)
    # ---- non-finite texels in the targets 1 .. nf-1
    for k in range(1, nf):
        img = W["images"][k]
        y0, x0 = rng.integers(20, h - 80), rng.integers(20, w - 100)
        img[y0:y0 + 40, x0:x0 + 60] = np.nan
        img[rng.integers(20, h - 20), :] = np.nan
        img[:, rng.integers(20, w - 20)] = np.inf
    W["dI"] = [make_images_level0(img).reshape(-1) for img in W["images"]]
    labels, tie, foot = hard_labels(W, pc)
    # single NaN texels: sample j of a residual that has no other exit, at a texel of j's footprint no other sample of it reads
    st = W["res_state"]
    single = []
    free = np.nonzero((labels == "none") & ~tie & (st != RES_OOB) & (W["res_target"] > 0))[0]
    for j in range(8):
        for i in rng.permutation(free)[:40]:
            if sum(1 for (_, jj) in single if jj == j) >= 4:
                break
            x, y = foot[i, j]
            others = {(int(a) + da, int(b) + db) for jj, (a, b) in enumerate(foot[i]) if jj != j for da in (0, 1) for db in (0, 1)}
            texels = [(int(x) + da, int(y) + db) for da in (0, 1) for db in (0, 1) if (int(x) + da, int(y) + db) not in others]
            if not texels:
                continue
            tx, ty = texels[int(rng.integers(0, len(texels)))]
            W["images"][W["res_target"][i]][ty, tx] = np.nan
            single.append((int(i), j))
            free = free[free != i]
    W["dI"] = [make_images_level0(img).reshape(-1) for img in W["images"]]
    labels, tie, foot = hard_labels(W, pc)
    st[tie] = RES_OOB
    W["labels"], W["single_nan"] = labels, np.array(single, np.int64)
    W["hard_points"] = dict(border=np.sort(border), reverse=np.sort(reverse), behind=np.sort(behind), zero=np.sort(zero), negative=np.sort(neg))
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


EPS32 = float(np.finfo(np.float32).eps)
EPS64 = float(np.finfo(np.float64).eps)
# check_system tau of the GPU-vs-oracle comparisons (check_linearize_parity, tests/test_gpu_marg.py).  The two sides differ by per-residual
# rounding (rtol <= 2e-3), so 4e-3 is a hard ceiling.  Worst ratios measured on an H100 (SXM, 80 GB) over every config of
# tests/test_gpu_ba.py and tests/test_gpu_ba_step.py at both chunk shapes: H_A 3.7e-6, b_A 1.5e-5, H_sc 5.5e-6, b_sc 1.7e-5;
# tests/test_gpu_marg.py: M 4.6e-6, Mb 4.3e-6, Msc 8.6e-6, Mbsc 3.0e-6; the oracle's own faithful-float system against its fp64 one:
# <= 7.7e-7.  tau = ~10x the worst.
SYSTEM_TAU = 2e-4
FRAME_PARAMS = ("trans x", "trans y", "trans z", "rot x", "rot y", "rot z", "a", "b")   # order of a frame's 8 parameters in the system


def system_entry_name(i):
    """row / column i of a window system [camera 4 | frame 0 (8) | frame 1 (8) | ...] in words"""
    return f"camera {i}" if i < 4 else f"frame {(i - 4) // 8} {FRAME_PARAMS[(i - 4) % 8]}"


def check_system(H, b, H_ref, b_ref, R, tau, what="system"):
    """Per-entry check of an accumulated system (H, b) against a reference (H_ref, b_ref), each entry on its own Jacobi scale.

    The systems are sums of Gram terms (sum J^T J with right-hand side sum J^T r, or sum HdiF v v^T with sum HdiF bdSum v), so by
    Cauchy-Schwarz the absolute sum behind H_ij is at most sqrt(H_ii H_jj) and that behind b_i at most sqrt(H_ii R), R a bound of the
    summed squared residuals (sum of the IN residuals' energies, sum HdiF bdSumF^2, sum res_toZeroF^2).  With d = diag(H_ref):
      |H_ij - H_ref_ij| <= tau sqrt(d_i d_j),   |b_i - b_ref_i| <= tau sqrt(d_i R),
    and where d_i = 0 the entries of row / column i are exactly 0 on both sides.  A failure names the entry (camera, or frame + parameter).
    Returns the worst ratios |error| / sqrt(...) of H and of b (what tau must exceed)."""
    H, b, Hr, br = (np.asarray(a, np.float64) for a in (H, b, H_ref, b_ref))
    d = np.diag(Hr)
    assert np.all(d >= 0), f"{what}: negative reference diagonal at {system_entry_name(int(np.argmin(d)))}"
    s = np.sqrt(d)
    ratios = []
    for name, got, ref, scale in (("H", H, Hr, np.outer(s, s)), ("b", b, br, s * np.sqrt(max(float(R), 0.0)))):
        zero = scale == 0
        nz = zero & ((got != 0) | (ref != 0))
        if nz.any():
            idx = np.unravel_index(int(np.argmax(nz)), nz.shape)
            where = ", ".join(system_entry_name(int(i)) for i in idx)
            raise AssertionError(f"{what}: {name}[{where}] = {got[idx]:.6e} / reference {ref[idx]:.6e} where the reference diagonal is 0")
        ratio = np.abs(got - ref) / np.where(zero, 1.0, scale)
        worst = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        where = ", ".join(system_entry_name(int(i)) for i in worst)
        assert ratio[worst] <= tau, (f"{what}: {name}[{where}] = {got[worst]:.9e}, reference {ref[worst]:.9e}: |error| = "
                                     f"{ratio[worst]:.3e} x its Jacobi scale {scale[worst]:.3e} > tau = {tau:.1e}")
        ratios.append(float(ratio[worst]))
    return tuple(ratios)


def energy_bound(newState, newEnergy):
    """R of check_system for a top system: the sum of newEnergy over the IN residuals.  It bounds sum resF^2: a pixel's energy is
    w^2 hw r^2 (2 - hw) and its resF^2 = w^2 hw r^2, with Huber's 2 - hw >= 1."""
    return float(np.asarray(newEnergy, np.float64)[np.asarray(newState) == RES_IN].sum())


def schur_bound(HdiF, bdSumF):
    """R of check_system for a Schur system: sum_p HdiF bdSumF^2"""
    return float((np.asarray(HdiF, np.float64) * np.asarray(bdSumF, np.float64) ** 2).sum())


def schur_vectors(W, state, JpJdF, Hcd, adH, adT):
    """The points' Schur vectors v_p in R^N (N = 8 nf + 4) from fp32 committed outputs, in fp64, and the same sums over absolute values:
      v_p[0:4] = Hcd_p;  every IN residual (host h, target t) adds adHostF[h + t nf] @ JpJdF to frame block h and
      diag(adTargetF[h + t nf]) o JpJdF to frame block t (adjoints rounded to fp32 and indexed as dmv_ba_set_adjoints reads them)."""
    nf, npts = W["nf"], len(W["host"])
    N = 8 * nf + 4
    AH = np.asarray(adH).astype(np.float32).astype(np.float64)
    AT = np.einsum("ikk->ik", np.asarray(adT)).astype(np.float32).astype(np.float64)
    V, Va = np.zeros((npts, N)), np.zeros((npts, N))
    V[:, :4] = np.asarray(Hcd, np.float32)
    Va[:, :4] = np.abs(V[:, :4])
    inn = np.asarray(state) == RES_IN
    rp, rt = np.asarray(W["res_point"])[inn], np.asarray(W["res_target"])[inn]
    J = np.asarray(JpJdF, np.float32)[inn].astype(np.float64)
    rh = np.asarray(W["host"])[rp]
    for h in range(nf):
        for t in range(nf):
            m = (rh == h) & (rt == t)
            if h == t or not m.any():
                continue
            p, Jm = rp[m], J[m]
            A, dT = AH[h + t * nf], AT[h + t * nf]
            np.add.at(V, (p[:, None], 4 + 8 * h + np.arange(8)[None, :]), Jm @ A.T)
            np.add.at(Va, (p[:, None], 4 + 8 * h + np.arange(8)[None, :]), np.abs(Jm) @ np.abs(A).T)
            np.add.at(V, (p[:, None], 4 + 8 * t + np.arange(8)[None, :]), Jm * dT)
            np.add.at(Va, (p[:, None], 4 + 8 * t + np.arange(8)[None, :]), np.abs(Jm * dT))
    return V, Va


def schur_reference(W, state, JpJdF, Hcd, HdiF, bdSumF, adH, adT):
    """H_sc = sum_p HdiF_p v_p v_p^T, b_sc = sum_p HdiF_p bdSumF_p v_p in fp64 (schur_vectors), and Habs / babs: the same sums over the
    absolute value of every product (|v_p| taken term by term).  Returns Hsc, bsc, Habs, babs."""
    V, Va = schur_vectors(W, state, JpJdF, Hcd, adH, adT)
    hd = np.asarray(HdiF, np.float32).astype(np.float64)
    bs = np.asarray(bdSumF, np.float32).astype(np.float64)
    return (V * hd[:, None]).T @ V, V.T @ (hd * bs), (Va * np.abs(hd)[:, None]).T @ Va, Va.T @ np.abs(hd * bs)


def check_linearize_parity(ow, ba, r, E_o, tau=None):
    """A GPU linearisation (result r, still tentative) against the oracle's (energy E_o of ow.linearize_all), then both committed and
    accumulated.  Tolerances and their reasons: tests/test_gpu_ba.py's docstring; the accumulated systems are compared entry by entry
    (check_system, tau = SYSTEM_TAU by default).  Returns the GPU's (residual outputs, point outputs, accumulated system); the worst
    check_system ratios are in the system's "ratios" entry."""
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
    # ---- entry by entry: whole-matrix ratios only see the largest blocks (the camera block holds ~5e-5 of ||H_A||_F)
    tau = SYSTEM_TAU if tau is None else tau
    a_g["ratios"] = (check_system(a_g["HA"], a_g["bA"], a_o["HA"], a_o["bA"], energy_bound(o["newState"], o["newEnergy"]), tau, "top system")
                     + check_system(a_g["Hsc"], a_g["bsc"], a_o["Hsc"], a_o["bsc"], schur_bound(po["HdiF"], po["bdSumF"]), tau, "Schur system"))
    print(f"check_system vs oracle: worst |error| / Jacobi scale: HA {a_g['ratios'][0]:.2e} bA {a_g['ratios'][1]:.2e} "
          f"Hsc {a_g['ratios'][2]:.2e} bsc {a_g['ratios'][3]:.2e}")
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


def ci_points(rng, w, h, levels, counts):
    """points per level the way CoarseInitializer::setFirst lays them out (integer pixel + 0.1 inside the pattern margin, row-major order),
    with no neighbours and no parent (-1): calcResAndGS reads neither, and this scales to DSO's point densities"""
    pts = []
    for l in range(levels):
        wl, hl = w >> l, h >> l
        n = counts[l]
        x = rng.integers(3, wl - 4, 4 * n); y = rng.integers(3, hl - 4, 4 * n)
        xy = np.unique(np.stack([y, x], 1), axis=0)                       # row-major order, no duplicates
        xy = xy[np.sort(rng.choice(len(xy), min(n, len(xy)), replace=False))]
        m = len(xy)
        pts.append(dict(u=(xy[:, 1] + 0.1).astype(np.float32), v=(xy[:, 0] + 0.1).astype(np.float32), type=np.ones(m, np.float32),
                        parent=np.full(m, -1, np.int32), neighbours=np.full((m, 10), -1, np.int32)))
    return pts


def init_points(rng, w, h, levels, counts):
    """ci_points with brute-force 10 nearest neighbours and the nearest parent one level up (CoarseInitializer::makeNN's outputs, without its
    kd-tree).  The neighbour search needs n^2 memory: keep it to a few thousand points per level."""
    pts = ci_points(rng, w, h, levels, counts)
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
# scenes whose new frame is lit differently from the keyframe: (gain, offset, arguments).  The new planes are intensity * gain + offset,
# gradients * gain.  aff_zeroA / aff_zeroB: the exposures (ref_b) predict the change, so a, b stay near 0 and the default modes' tests
# |a| > 1.2, |b| > 200 pass, while mode 0's |log ra| = log 5 > 1.5 and |rb| = 250 > 200 fail.  aff_bigA: gain 4 the exposures do not
# predict, so a ends near log 4 = 1.39: the default mode's |a| > 1.2 fails and mode 0's |log ra| < 1.5 passes
CT_LIGHT = dict(aff_zeroA=(5.0, 0.0, dict(new_exposure=5.0, affA=0.0)), aff_zeroB=(1.0, 250.0, dict(ref_b=-250.0, affB=0.0)),
                aff_bigA=(4.0, 0.0, dict(a0=float(np.log(4.0)) - 0.05)))


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
    if name in CT_LIGHT:
        w, h, L, seed = 640, 480, 4, 99
        args["R0"], args["t0"] = synth.se3_exp(np.array([0.005, -0.004, 0.003, 0.002, -0.001, 0.002]))
        args.update(CT_LIGHT[name][2])
    elif name.startswith("aff_"):
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
    planes = T["pyr_new"]
    if name in CT_LIGHT:
        gain, offset, _ = CT_LIGHT[name]
        planes = [np.asarray(p, np.float32) * np.float32(gain) for p in planes]
        for p in planes:
            p[..., 0] += np.float32(offset)
    return dict(name=name, w=w, h=h, levels=L, K=T["K"], pts=pts, planes=planes, k4=k4, Ki=[ct_Ki(k) for k in k4], args=args, T=T)


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


# ---------------------------------------------------------------------------------------------------------------------------------
# fp64 reference of CoarseInitializer::calcResAndGS (oracle/orc_init.cpp:L194-345)
# ---------------------------------------------------------------------------------------------------------------------------------
CI_PATTERN = np.array([[0, -2], [-1, -1], [1, -1], [-2, 0], [0, 0], [2, 0], [-1, 1], [0, 2]])   # staticPattern[8] (util/settings.h)
CI_ALPHA_K, CI_ALPHA_W = 2.5 * 2.5, 150.0 * 150.0
CI_THREADS = 256                                                                                  # ci_kernels.cu: 32 points per CTA per trip


def alpha_restatement(alphaW, alphaK, t_d, n):
    """The reference's alphaEnergy and alphaOpt (CoarseInitializer.cpp:L540-557) bit for bit: alphaW * (EAlpha.A + |t|^2 npts) with
    EAlpha.A = 0, evaluated in double and rounded to float once, then capped at float(alphaK * npts) when above it.
    Returns (res3[1], alphaOpt) as float32."""
    f = np.float32
    t = np.asarray(t_d, np.float64)
    tsq = (t[0] * t[0] + t[1] * t[1]) + t[2] * t[2]
    aE = f(float(f(alphaW)) * (0.0 + tsq * n))
    cap = f(f(alphaK) * f(n))
    return (cap, f(0)) if aE > cap else (aE, f(alphaW))


def alpha_sweep(n, alphaW=CI_ALPHA_W, alphaK=CI_ALPHA_K, count=20001, span=4e-6):
    """s around sqrt(alphaK / alphaW) (relative span), with the reference's (alphaEnergy, alphaOpt) at t = (0, 0, s) for n points and the
    product's former arithmetic, alphaW * float(|t|^2 n) in float"""
    f = np.float32
    s = np.sqrt(alphaK / alphaW) * (1 + np.linspace(-span, span, count))
    tsq = s * s
    ref = f(float(f(alphaW)) * (0.0 + tsq * n))
    old = f(alphaW) * (0.0 + tsq * n).astype(f)
    cap = f(f(alphaK) * f(n))
    return s, ref, old, cap


def alpha_cases(n):
    """values of s where the reference's rounding and the former product's disagree, one per kind where one exists:
    cap_ref_only / cap_old_only (alphaOpt), eq_ref_only / eq_old_only (the `res3[1] == alphaK n` snap test), and one where only res3[1] differs"""
    s, ref, old, cap = alpha_sweep(n)
    kinds = dict(cap_ref_only=(ref > cap) & ~(old > cap), cap_old_only=~(ref > cap) & (old > cap),
                 eq_ref_only=(ref == cap) & (old != cap), eq_old_only=(ref != cap) & (old == cap),
                 ulp=(ref != old) & (ref < cap) & (old < cap))
    return {k: float(s[np.nonzero(m)[0][0]]) for k, m in kinds.items() if m.any()}


def ci_kernel_depth(n, sms):
    """fp32 summation depth of ci_res_gs_kernel: each lane accumulates one term per trip of the grid-stride loop (grid = min(2 SMs, ceil(n/32))
    CTAs of 32 points), then a 5-level butterfly over the warp, then the rounding of the fp64 fold (warps and CTAs are folded in fp64)"""
    grid = max(1, min(2 * sms, -(-n // (CI_THREADS // 8))))
    return -(-n // (grid * (CI_THREADS // 8))) + 5 + 1


def ci_calc_ref(first, new, k4, u, v, outlierTH, idepth_new, isGood, energy, iR, RKi, t_d, t_log, aff, huber=9.0, alphaK=CI_ALPHA_K,
                alphaW=CI_ALPHA_W, coupling=1.0, wzp=(0.0, 0.0), depth=None, verdict=None, form=None):
    """One CoarseInitializer::calcResAndGS in fp64 from the same fp32 inputs (oracle/orc_init.cpp:L194-345): first / new are the level planes
    [I, dx, dy] of both frames, k4 the level's fx, fy, cx, cy (makeK, rounded to float on use), RKi the fp32 rotation times Ki, t_d the
    translation (float for the projection, double for alphaEnergy and the zero prior), t_log the first three entries of SE3::log, aff the fp32
    r2new_aff.  alphaOpt comes from alpha_restatement.

    Returns the per-point outputs (isGood_new, energy_new (n, 2), maxstep, lastHessian_new, Jb (n, 10)), H, b, Hsc, bsc (the alpha and
    zero-prior terms included), res3, alphaOpt, n_good, and a first-order bound of what an fp32 evaluation may differ by for each of them:
    dE0 (energy_new[:, 0]), dmaxstep, dlastH, dJb, dH, db, dHsc, dbsc, dres0.  The bound follows every fp32 operation of a pixel (the
    projection by _proj_bound, the gathers by the plane's slope in the cell times dKu, dKv), sums the 8 pixels of a point (Jb rows, energy)
    with 7 additions, and the points with `depth` additions per term plus n fp64 ones (default: the sequential depth n).
    A point is `amb`iguous when a test lies within its bound: Ku > 1, Kv > 1, Ku < w-2, Kv < h-2, new_idepth > 0, a gather cell whose
    neighbour holds a non-finite sample, or energy > 20 outlierTH.  With `verdict` (the device's isGood_new) given, ambiguous points take
    that verdict; they count in full in the bounds of the sums.  maxstep is comparable where every pixel passes (`allok`): the reference
    stops at the first failing pixel, and maxstep is read for good points only."""
    f, f32 = np.float64, np.float32
    n = len(u)
    depth = n if depth is None else depth
    hl, wl = new.shape[:2]
    fx, fy, cx, cy = (float(f32(x)) for x in k4)
    M = np.asarray(RKi, f32).astype(f).reshape(3, 3)
    t_d = np.asarray(t_d, f)
    tt = t_d.astype(f32).astype(f)
    X = (np.asarray(u, f32)[:, None] + CI_PATTERN[None, :, 0].astype(f32)).astype(f)     # fp32 sums, exactly as both sides form them
    Y = (np.asarray(v, f32)[:, None] + CI_PATTERN[None, :, 1].astype(f32)).astype(f)
    idp = np.asarray(idepth_new, f32).astype(f)
    ID = np.broadcast_to(idp[:, None], X.shape)
    sh = X.shape
    uu, vv, z, du, dv, dz, Ku, Kv, dKu, dKv = (q.reshape(sh) for q in _proj_bound(M, tt, X.ravel(), Y.ravel(), ID.ravel(), fx, fy, cx, cy, form))
    nid = ID / z
    dnid = np.abs(nid) * (dz / np.abs(z) + U32)
    wasGood = np.asarray(isGood) != 0
    inb = (Ku > 1) & (Kv > 1) & (Ku < wl - 2) & (Kv < hl - 2) & (nid > 0)
    amb_b = ((np.abs(Ku - 1) <= dKu) | (np.abs(Kv - 1) <= dKv) | (np.abs(Ku - (wl - 2)) <= dKu) | (np.abs(Kv - (hl - 2)) <= dKv) |
             (np.abs(nid) <= dnid))
    ev = inb | amb_b
    # bilinear gathers (util/globalFuncs.h getInterpolatedElement33 / 31): the new frame at (Ku, Kv), the first frame at the pattern pixel
    Kuc, Kvc = np.where(ev, Ku, 3.0), np.where(ev, Kv, 3.0)
    ix = np.clip(np.floor(Kuc), 0, wl - 2).astype(np.int64)
    iy = np.clip(np.floor(Kvc), 0, hl - 2).astype(np.int64)
    dx, dy = Kuc - ix, Kvc - iy
    P64 = new.astype(f)
    tl, tr, bl, br = P64[iy, ix], P64[iy, ix + 1], P64[iy + 1, ix], P64[iy + 1, ix + 1]
    w11, w10, w01, w00 = dx * dy, dy - dx * dy, dx - dx * dy, 1 - dx - dy + dx * dy
    with np.errstate(invalid="ignore"):
        hit = w11[..., None] * br + w10[..., None] * bl + w01[..., None] * tr + w00[..., None] * tl
        Gu = np.maximum(np.abs(tr - tl), np.abs(br - bl))
        Gv = np.maximum(np.abs(bl - tl), np.abs(br - tr))
        dh = Gu * dKu[..., None] + Gv * dKv[..., None] + 12 * U32 * (np.abs(tl) + np.abs(tr) + np.abs(bl) + np.abs(br))
    # a cell within dKu / dKv of its edge may be the neighbour cell on the device: ambiguous if that changes whether a tap is non-finite
    bad0 = ~np.isfinite(new[..., 0])
    cand = []
    for ox in (-1, 0, 1, 2):
        for oy in (-1, 0, 1, 2):
            cand.append(bad0[np.clip(iy + oy, 0, hl - 1), np.clip(ix + ox, 0, wl - 1)])
    near = (np.floor(Kuc - dKu) != np.floor(Kuc + dKu)) | (np.floor(Kvc - dKv) != np.floor(Kvc + dKv))
    amb_nan = ev & near & np.any(cand, axis=0) & np.isfinite(hit[..., 0])
    amb_nan |= ev & near & ~np.isfinite(hit[..., 0])
    ixr = np.clip(np.floor(X), 0, wl - 2).astype(np.int64)
    iyr = np.clip(np.floor(Y), 0, hl - 2).astype(np.int64)
    ex, ey = X - ixr, Y - iyr
    F0 = first[..., 0].astype(f)
    t00, t10, t01, t11 = F0[iyr, ixr], F0[iyr, ixr + 1], F0[iyr + 1, ixr], F0[iyr + 1, ixr + 1]
    with np.errstate(invalid="ignore"):
        rlR = ex * ey * t11 + (ey - ex * ey) * t01 + (ex - ex * ey) * t10 + (1 - ex - ey + ex * ey) * t00
        drlR = 12 * U32 * (np.abs(t00) + np.abs(t10) + np.abs(t01) + np.abs(t11))
    pix_ok = inb & np.isfinite(hit[..., 0]) & np.isfinite(rlR)
    amb_px = amb_b | amb_nan
    # pixel values where they are evaluated; zeros elsewhere, so that nothing non-finite reaches a sum
    ok_v = ev & np.isfinite(hit).all(-1) & np.isfinite(rlR)
    hit = np.where(ok_v[..., None], hit, 0.0); dh = np.where(ok_v[..., None], dh, 0.0)
    rlR = np.where(ok_v, rlR, 0.0); drlR = np.where(ok_v, drlR, 0.0)
    a0, a1 = float(f32(aff[0])), float(f32(aff[1]))
    huber = float(f32(huber))
    r = hit[..., 0] - a0 * rlR - a1
    ar = np.abs(r)
    dr = dh[..., 0] + abs(a0) * drlR + 2 * U32 * (np.abs(a0 * rlR) + abs(a1) + ar)
    hw = np.where(ar < huber, 1.0, huber / np.maximum(ar, 1e-30))
    dhw = np.where(ar < huber, 0.0, hw * dr / np.maximum(ar, 1e-30) + U32 * hw)
    e = hw * r * r * (2 - hw)
    de = 2 * np.minimum(ar, huber) * dr + 5 * U32 * e
    hs = np.sqrt(hw)                                                                  # `if (hw < 1) hw = sqrtf(hw)`
    dhs = np.where(ar < huber, 0.0, dhw / (2 * hs) + U32 * hs)
    zz = np.where(ok_v, z, 1.0)
    uu, vv = np.where(ok_v, uu, 0.0), np.where(ok_v, vv, 0.0)
    nx, ny = tt[0] - tt[2] * uu, tt[1] - tt[2] * vv
    dnx = abs(tt[2]) * du + 2 * U32 * (abs(tt[0]) + np.abs(tt[2] * uu))
    dny = abs(tt[2]) * dv + 2 * U32 * (abs(tt[1]) + np.abs(tt[2] * vv))
    rz = dz / np.abs(zz) + U32
    dxdd, dydd = nx / zz, ny / zz
    ddxdd, ddydd = dnx / np.abs(zz) + np.abs(dxdd) * rz, dny / np.abs(zz) + np.abs(dydd) * rz
    gx, gy = hs * hit[..., 1] * fx, hs * hit[..., 2] * fy
    dgx = np.abs(hit[..., 1] * fx) * dhs + hs * fx * dh[..., 1] + 2 * U32 * np.abs(gx)
    dgy = np.abs(hit[..., 2] * fy) * dhs + hs * fy * dh[..., 2] + 2 * U32 * np.abs(gy)
    nd = np.where(ok_v, nid, 0.0)
    dnd = np.where(ok_v, dnid, 0.0)
    J = np.zeros((9,) + sh); dJ = np.zeros((9,) + sh)
    J[0], J[1] = nd * gx, nd * gy
    dJ[0] = np.abs(nd) * dgx + np.abs(gx) * dnd + U32 * np.abs(J[0])
    dJ[1] = np.abs(nd) * dgy + np.abs(gy) * dnd + U32 * np.abs(J[1])
    s2 = uu * gx + vv * gy
    J[2] = -nd * s2
    dJ[2] = (np.abs(nd) * (np.abs(uu) * dgx + np.abs(gx) * du + np.abs(vv) * dgy + np.abs(gy) * dv + 3 * U32 * (np.abs(uu * gx) + np.abs(vv * gy)))
             + dnd * np.abs(s2) + U32 * np.abs(J[2]))
    J[3] = -uu * vv * gx - (1 + vv * vv) * gy
    dJ[3] = ((np.abs(vv) * du + np.abs(uu) * dv) * np.abs(gx) + np.abs(uu * vv) * dgx + (1 + vv * vv) * dgy + 2 * np.abs(gy * vv) * dv
             + 5 * U32 * (np.abs(uu * vv * gx) + np.abs(gy) * (1 + vv * vv)))
    J[4] = (1 + uu * uu) * gx + uu * vv * gy
    dJ[4] = ((np.abs(vv) * du + np.abs(uu) * dv) * np.abs(gy) + np.abs(uu * vv) * dgy + (1 + uu * uu) * dgx + 2 * np.abs(gx * uu) * du
             + 5 * U32 * (np.abs(uu * vv * gy) + np.abs(gx) * (1 + uu * uu)))
    J[5] = -vv * gx + uu * gy
    dJ[5] = du * np.abs(gy) + np.abs(uu) * dgy + dv * np.abs(gx) + np.abs(vv) * dgx + 3 * U32 * (np.abs(uu * gy) + np.abs(vv * gx))
    J[6] = -hs * a0 * rlR
    dJ[6] = np.abs(a0 * rlR) * dhs + hs * abs(a0) * drlR + 2 * U32 * np.abs(J[6])
    J[7] = -hs
    dJ[7] = dhs
    J[8] = hs * r
    dJ[8] = ar * dhs + hs * dr + U32 * np.abs(J[8])
    dd = gx * dxdd + gy * dydd
    ddd = np.abs(dxdd) * dgx + np.abs(gx) * ddxdd + np.abs(dydd) * dgy + np.abs(gy) * ddydd + 3 * U32 * (np.abs(gx * dxdd) + np.abs(gy * dydd))
    J *= ok_v; dJ *= ok_v; dd = dd * ok_v; ddd = ddd * ok_v
    e, de = e * ok_v, de * ok_v
    mx, my = dxdd * fx, dydd * fy
    m2 = mx * mx + my * my
    with np.errstate(divide="ignore"):
        ms = np.where(pix_ok & (m2 > 0), 1 / np.sqrt(m2), np.inf)
        dms = ms * ((np.abs(mx) * (fx * ddxdd + U32 * np.abs(mx)) + np.abs(my) * (fy * ddydd + U32 * np.abs(my))) / np.where(m2 > 0, m2, 1) + 4 * U32)
    # the point: its energy, outlier test and verdict
    allok = pix_ok.all(1)
    energy_pt, den = e.sum(1), de.sum(1) + 7 * U32 * np.abs(e).sum(1)
    th = (np.asarray(outlierTH, f32) * f32(20)).astype(f)
    definite_fail = (~pix_ok & ~amb_px).any(1)
    amb = wasGood & ~definite_fail & (amb_px.any(1) | (np.abs(energy_pt - th) <= den))
    good = wasGood & allok & ~(energy_pt > th)
    if verdict is not None:
        good = np.where(amb, np.asarray(verdict) != 0, good)
    amb_g = amb & good
    e0, e1 = np.asarray(energy, f32).reshape(n, 2).astype(f).T
    Jb = np.zeros((n, 10)); dJb = np.zeros((n, 10))
    for k in range(9):
        Jb[:, k] = (J[k] * dd).sum(1)
        dJb[:, k] = (np.abs(J[k]) * ddd + np.abs(dd) * dJ[k]).sum(1) + 8 * U32 * np.abs(J[k] * dd).sum(1)
    lastH = (dd * dd).sum(1)
    dlastH = (2 * np.abs(dd) * ddd).sum(1) + 8 * U32 * lastH
    # L562-586: the Schur rows with alphaOpt from the reference's arithmetic
    alphaE, alphaOpt = alpha_restatement(alphaW, alphaK, t_d, n)
    aO, c = float(alphaOpt), (float(f32(coupling)) if alphaOpt == 0 else 0.0)
    iRf = np.asarray(iR, f32).astype(f)
    idm1 = idp - 1
    Jb8 = Jb[:, 8] + aO * idm1 + c * (idp - iRf)
    dJb8 = dJb[:, 8] + 3 * U32 * (np.abs(Jb[:, 8]) + aO * np.abs(idm1) + c * np.abs(idp - iRf))
    S = lastH + aO + c
    dS = dlastH + 2 * U32 * (lastH + aO + c)
    wsc = 1 / (1 + S)
    dwsc = wsc * wsc * (dS + U32 * (1 + S)) + U32 * wsc
    Jb[:, 8], dJb[:, 8] = Jb8, dJb8
    Jb[:, 9], dJb[:, 9] = wsc, dwsc
    Jb[~good], dJb[~good] = 0, 0
    order = depth * U32 + n * 2.0 ** -53
    # Accumulator9 over the pixels of good points, and the weighted one over the Schur rows
    iu = np.triu_indices(9)
    gp = good[:, None]
    M9, dM9, S9, dS9 = np.zeros((9, 9)), np.zeros((9, 9)), np.zeros((9, 9)), np.zeros((9, 9))
    for rr, cc in zip(*iu):
        Pk = J[rr] * J[cc]
        dPk = np.abs(J[rr]) * dJ[cc] + np.abs(J[cc]) * dJ[rr] + U32 * np.abs(Pk)
        M9[rr, cc] = (Pk * gp).sum()
        dM9[rr, cc] = (dPk * gp).sum() + order * (np.abs(Pk) * gp).sum() + (np.abs(Pk) * amb_g[:, None]).sum()
        Qk = Jb[:, rr] * wsc * Jb[:, cc]
        dQk = wsc * (np.abs(Jb[:, rr]) * dJb[:, cc] + np.abs(Jb[:, cc]) * dJb[:, rr]) + np.abs(Jb[:, rr] * Jb[:, cc]) * dwsc + 2 * U32 * np.abs(Qk)
        S9[rr, cc] = (Qk * good).sum()
        dS9[rr, cc] = (dQk * good).sum() + order * (np.abs(Qk) * good).sum() + (np.abs(Qk) * amb_g).sum()
    sym = lambda A: np.triu(A) + np.triu(A, 1).T
    M9, dM9, S9, dS9 = sym(M9), sym(dM9), sym(S9), sym(dS9)
    H, b, Hsc, bsc = M9[:8, :8].copy(), M9[:8, 8].copy(), S9[:8, :8].copy(), S9[:8, 8].copy()
    dH, db = dM9[:8, :8] + U32 * np.abs(H), dM9[:8, 8] + U32 * np.abs(b)     # + the rounding to float
    dHsc, dbsc = dS9[:8, :8] + U32 * np.abs(Hsc), dS9[:8, 8] + U32 * np.abs(bsc)
    for k in range(3):   # L588-604: alpha terms in float
        tl_k = float(f32(t_log[k])) * aO * n
        dH[k, k] += 2 * U32 * (np.abs(H[k, k]) + aO * n)
        H[k, k] += aO * n
        db[k] += 3 * U32 * abs(tl_k) + U32 * (abs(b[k]) + abs(tl_k))
        b[k] += tl_k
    wx, wy = float(wzp[0]), float(wzp[1])   # L606-611: the zero prior, in double, rounded once
    H[1, 1] += wy; b[1] += wy * t_d[1]; H[0, 0] += wx; b[0] += wx * t_d[0]
    for (i, j) in ((0, 0), (1, 1)):
        dH[i, j] += U32 * abs(H[i, j])
    db[:2] += U32 * np.abs(b[:2])
    E = float(np.where(good, energy_pt, e0).sum())
    dE = float((den * (good & ~amb)).sum() + order * np.abs(np.where(good, energy_pt, e0)).sum() + ((np.abs(energy_pt) + np.abs(e0)) * amb).sum())
    idq = f32(np.asarray(idepth_new, f32) - f32(1))
    energy_new = np.stack([np.where(good, energy_pt, e0), np.where(good, (idq * idq).astype(f32).astype(f), e1)], 1)
    maxstep = np.where(wasGood, np.minimum(1e10, ms.min(1)), 1e10)
    dmaxstep = np.where(wasGood & allok & np.isfinite(ms.min(1)), np.where(np.isfinite(ms), dms, 0).max(1), 0.0)
    return dict(isGood_new=good, amb=amb, allok=allok, energy_new=energy_new, dE0=np.where(good, den, 0.0), maxstep=maxstep, dmaxstep=dmaxstep,
                lastHessian_new=np.where(good, lastH, 0.0), dlastH=np.where(good, dlastH, 0.0), Jb=Jb, dJb=dJb,
                H=H, b=b, Hsc=Hsc, bsc=bsc, dH=dH, db=db, dHsc=dHsc, dbsc=dbsc,
                res3=np.array([E, float(alphaE), 2.0 * n]), dres0=dE, alphaOpt=alphaOpt, n_good=int(good.sum()), n_amb=int(amb.sum()))


def ci_bound_ratio(got, want, bound):
    """largest |got - want| / bound (0 / 0 counts as 0, x / 0 as inf)"""
    err = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64))
    bound = np.broadcast_to(np.asarray(bound, np.float64), err.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(err == 0, 0.0, err / bound)
    return float(q.max()) if q.size else 0.0


CI_MOTION = np.array([0.004, -0.003, 0.002, 0.002, -0.001, 0.0015])   # |t| ~ 0.005: alphaW |t|^2 < alphaK, alphaOpt = alphaW
CI_SNAP = np.array([0.03, -0.02, 0.012, 0.003, -0.002, 0.001])        # |t| ~ 0.038: alphaOpt = 0, the coupling branch
CI_EDGE = np.array([0.25, -0.12, 0.05, 0.01, 0.02, -0.01])            # moves part of the points out of the image
CI_STATES = ("fresh", "motion", "snapped", "some_bad")


def ci_state(kind, n, seed):
    """the caller's point state and the pose of one calcResAndGS evaluation:
      fresh     identity pose, idepth 1 (trackFrame's first evaluation of a level)
      motion    a small motion, idepths around 1, iR = idepth
      snapped   |t| >= 0.03, iR random around idepth_new
      some_bad  the small motion with ~10 % of the points !isGood, carrying random energies
      edge      CI_EDGE, idepths in [0.5, 1.5] and a few < 0"""
    rng = np.random.default_rng(seed)
    f32 = np.float32
    st = dict(idepth_new=np.ones(n, f32), isGood=np.ones(n, np.uint8), energy=np.zeros((n, 2), f32), iR=np.ones(n, f32), xi=np.zeros(6),
              a=0.0, b=0.0)
    if kind == "fresh":
        return st
    st.update(idepth_new=(1 + 0.05 * rng.standard_normal(n)).astype(f32), xi=CI_MOTION, a=float(np.log(1.2)), b=0.3)
    st["iR"] = st["idepth_new"].copy()
    if kind == "snapped":
        st["xi"] = CI_SNAP
        st["iR"] = (st["idepth_new"] * (1 + 0.05 * rng.standard_normal(n))).astype(f32)
    elif kind == "some_bad":
        st["isGood"] = (rng.random(n) >= 0.1).astype(np.uint8)
        st["energy"] = rng.uniform(0, 500, (n, 2)).astype(f32)
    elif kind == "edge":
        st["xi"] = CI_EDGE
        st["idepth_new"] = rng.uniform(0.5, 1.5, n).astype(f32)
        st["idepth_new"][rng.choice(n, max(3, n // 500), replace=False)] *= -1
        st["iR"] = st["idepth_new"].copy()
    return st


def ci_level_K(k4):
    fx, fy, cx, cy = (float(x) for x in k4)
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])


def ci_operands(synth, k4, st):
    """R, t (double), the fp32 RKi = (R Ki).cast<float>() and SE3::log's translation part of a state's pose"""
    R, t = synth.se3_exp(np.asarray(st["xi"], np.float64))
    R, t = np.asarray(R, np.float64), np.asarray(t, np.float64)
    RKi = (R @ np.linalg.inv(ci_level_K(k4))).astype(np.float32)
    return R, t, RKi, se3_log_translation(R, t)


def se3_log_translation(R, t):
    """first three entries of Sophus::SE3::log(): V^-1 t"""
    R = np.asarray(R, np.float64); t = np.asarray(t, np.float64)
    th = np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))
    if th < 1e-10:
        return t.copy()
    w = th / (2 * np.sin(th)) * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * W + (th - np.sin(th)) / th ** 3 * (W @ W)
    return np.linalg.solve(V, t)


def ci_poison(first, new, pts0, st, k4, synth):
    """copies of the level planes with one NaN in each, at taps that some points read: the first frame at the centre pixel of point 0's
    pattern, the new frame where the centre pixel of the first point that lands well inside the image projects to (under st's pose)"""
    first, new = first.copy(), new.copy()
    u, v = pts0["u"], pts0["v"]
    first[int(v[0]), int(u[0]), 0] = np.nan
    _, _, RKi, _ = ci_operands(synth, k4, st)
    M, tt = RKi.astype(np.float64), np.asarray(synth.se3_exp(np.asarray(st["xi"]))[1], np.float32).astype(np.float64)
    idp = st["idepth_new"].astype(np.float64)
    P = M @ np.stack([u, v, np.ones_like(u)]).astype(np.float64) + tt[:, None] * idp
    Ku, Kv = k4[0] * P[0] / P[2] + k4[2], k4[1] * P[1] / P[2] + k4[3]
    hl, wl = new.shape[:2]
    inside = np.nonzero((idp > 0) & (Ku > 10) & (Kv > 10) & (Ku < wl - 10) & (Kv < hl - 10) & (np.arange(len(u)) > 0))[0]
    j = inside[len(inside) // 2]
    new[int(Kv[j]), int(Ku[j]), 0] = np.nan
    return first, new


# ---------------------------------------------------------------------------------------------------------------------------------
# Immature-point tracing scenes past one warp round of the search (tests/test_ref_pin_ip.py, tests/test_gpu_ip_edges.py)
# ---------------------------------------------------------------------------------------------------------------------------------
def ip_num_steps(w, h):
    """the discrete search's step count for a fresh point (idepth_max = NaN: dist = maxPixSearch), before the clamp at 99"""
    return int(np.float32(1.9999) + np.float32(w + h) * np.float32(0.027))


def ip_scene(synth, w, h, seed, poses, quantize=False, nan_boxes=None):
    """A textured plane at depth 2 seen by frame 0 (identity) and by one frame per pose xi (6,); the dict carries what
    hostmath.trace_tables reads (K as make_window, state 0: aff = (1, 0)) and the level-0 planes dI.

    The fresh search runs from the point at infinity (uMin = the host pixel) towards the plane; with a translation (t, 0, t) the plane's
    disparity f t (1 - x/f) / (2 + t) sweeps [0, 2 f t / (2 + t)] across the image, so choosing f t ~ numSteps puts best steps in every
    lane round.  quantize: 8-bit frames after a contrast stretch, with wide bands clipped to 0 (exact ties: a point whose pattern lies in
    such a band matches every step of the band with energy 0).  nan_boxes: {frame: [(x0, y0, x1, y1), ...]} NaN rectangles."""
    rng = np.random.default_rng(seed)
    K = (0.5 * w, 0.5 * w, 0.5 * w - 0.5, 0.5 * h - 0.5)
    tex = synth.make_texture(rng, size=1024)
    nf = 1 + len(poses)
    R_eval, t_eval = np.zeros((nf, 3, 3)), np.zeros((nf, 3))
    images, dI = [], []
    for k in range(nf):
        R, t = synth.se3_exp(np.zeros(6) if k == 0 else np.asarray(poses[k - 1], np.float64))
        R_eval[k], t_eval[k] = R, t
        img, _ = synth.render_plane(tex, K, R, t, w, h, 2.0, texel_per_unit=0.5 * K[0] / 2.0)
        if quantize:
            img = np.clip(np.round(3.0 * (img - 0.5 * 255) + 100.0), 0, 255).astype(np.float32)
        d = synth.make_pyramid(img, 1)[0]
        for (x0, y0, x1, y1) in (nan_boxes or {}).get(k, ()):
            d[y0:y1, x0:x1, :] = np.nan
        images.append(img)
        dI.append(d.reshape(-1).copy())
    return dict(w=w, h=h, nf=nf, K=np.array(K, np.float64), images=images, dI=dI, R_eval=R_eval, t_eval=t_eval, state=np.zeros((nf, 10)),
                exposure=np.ones(nf, np.float32))


def ip_points(rng, w, h, n, margin=6):
    """n distinct integer pixels at least `margin` from the border (the ImmaturePoint pattern stays inside)"""
    sel = rng.choice((w - 2 * margin) * (h - 2 * margin), n, replace=False)
    return (margin + sel % (w - 2 * margin)).astype(np.int32), (margin + sel // (w - 2 * margin)).astype(np.int32)


# shapes whose fresh search reaches lane rounds past the first: numSteps = 46, 55, 82, 99 (105 before the clamp)
IP_ROUND_SHAPES = [(848, 800, 11), (1280, 720, 12), (1920, 1080, 13), (2560, 1280, 14)]
IP_TRACE_SEQ = (1, 2, 1)   # fresh points, refinement against another frame, re-tracing (traceNewCoarse on successive frames)


def ip_poses(w, h):
    """frame 1: translation (t, 0, t) with f t = numSteps, so best steps fall in every round the search has; frame 2: a smaller motion
    (the refinement: short segments, numSteps <= 10 for most points)"""
    t = ip_num_steps(w, h) / (0.5 * w)
    return [np.array([t, 0, t, 0.002, -0.003, 0.001]), np.array([-0.3 * t, 0.2 * t, 0.2 * t, 0.001, 0.002, -0.001])]


def ip_round_case(synth, orc, w, h, seed, n=1500, quantize=False, nan_boxes=None):
    S = ip_scene(synth, w, h, seed, ip_poses(w, h), quantize=quantize, nan_boxes=nan_boxes)
    u, v = ip_points(np.random.default_rng(seed), w, h, n)
    return S, orc.ip_init(S["dI"][0], w, h, u, v)


# NaN rectangles at the same place in both traced frames: segments and GN patterns cross them (the +1e5 branches), and points that fail
# the energy test against frame 1 fail it again against frame 2 (OUTLIER, then OOB)
IP_NAN_BOXES = [(500, 250, 700, 450), (900, 0, 903, 720), (0, 600, 1280, 602)]   # a block, a column and a row


def ip_status_case(synth, orc, n=2000, seed=21):
    w, h = 1280, 720
    return ip_round_case(synth, orc, w, h, seed, n, nan_boxes={1: IP_NAN_BOXES, 2: IP_NAN_BOXES})


def ip_gn_oob_case(w=640, h=480, theta=-0.03, n=2000):
    """Points whose Gauss-Newton refinement walks a pattern sample off the left border (traceOn's OOB return inside the GN loop).

    Where it can happen: uMin > boundU = max(4, maxRotPatX + 2) and the first search position is uMin - randShift dx > uMin - 1; each GN
    iteration moves at most 0.5 px and the bound test runs before the update, so the last test is at >= uMin - randShift - 1, and a pattern
    sample at >= uMin - randShift - 1 - |rot|.  With |rot| < 2 that stays > 1: only |rot| > 2 (KRKi[0][0] > 1, a rotation about y of the
    sign of theta) and uMin within 2 - |rot| + randShift - 1 of 4 can reach posU < 0.  Here KRKi is K Ry(theta) K^-1 (|rot| = 2 KRKi[0][0]
    ~ 2.04), the search runs along +x (Kt = K (0.05, 0, 0)), the frame is a ramp I = 2 x, and the points' colours are that ramp 3 px left of
    the pattern, so the search picks step 0 and every GN step is -0.5.  The host positions u sweep uMin over [3.99, 4.05] in n steps: the oracle's diag
    tells which of them exit by GN OOB.  Returns (P, dI, w, h, KRKi, Kt, aff)."""
    f, cx, cy = 0.5 * w, 0.5 * w - 0.5, 0.5 * h - 0.5
    K = np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float64)
    c, s = np.cos(theta), np.sin(theta)
    R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    KRKi = (K @ R @ np.linalg.inv(K)).astype(np.float32)
    Kt = (K @ np.array([0.05, 0, 0])).astype(np.float32)
    xs = np.arange(w, dtype=np.float32)
    d = np.zeros((h, w, 3), np.float32)
    d[:, :, 0] = 2 * xs[None, :]
    d[:, :, 1] = 2
    v = np.full(n, 0.5 * h, np.float32)
    Ki = np.linalg.inv(KRKi.astype(np.float64))
    u = np.array([(Ki @ np.array([um, 0.5 * h, 1.0]))[0] / (Ki @ np.array([um, 0.5 * h, 1.0]))[2] for um in np.linspace(3.99, 4.05, n)], np.float32)
    pat = np.array([[0, -2], [-1, -1], [1, -1], [-2, 0], [0, 0], [2, 0], [-1, 1], [0, 2]], np.float32)
    rotx = KRKi[0, 0] * pat[:, 0] + KRKi[0, 1] * pat[:, 1]
    uMin = (KRKi[0, 0] * u + KRKi[0, 1] * v + KRKi[0, 2]) / (KRKi[2, 0] * u + KRKi[2, 1] * v + KRKi[2, 2])
    P = dict(u=u, v=v, color=(2 * (uMin[:, None] - 3 + rotx[None, :])).astype(np.float32), weights=np.ones((n, 8), np.float32),
             gradH=np.tile(np.array([32, 0, 0, 32], np.float32), (n, 1)), energyTH=np.full(n, 1152, np.float32),
             idepth_min=np.zeros(n, np.float32), idepth_max=np.full(n, np.nan, np.float32), quality=np.full(n, 10000, np.float32),
             status=np.full(n, 5, np.int32), lastTraceUV=np.zeros((n, 2), np.float32), lastTracePixelInterval=np.zeros(n, np.float32))
    return P, d.reshape(-1), w, h, KRKi, Kt, np.array([1, 0], np.float32)


def activation_edge_case(synth, orc, nf, n, seed, nan_frames=(), flat=True):
    """activation_case's window and points, with hosts in every frame (the newest included), points down to 3 px from the border (their
    patterns leave the image in some targets part-way through: the sums keep the samples before the first bad one), NaN blocks in the
    level-0 planes of nan_frames, and a flat block (I = 128, no gradient) at the same place in every frame: points there have Hdd = 0,
    below setting_minIdepthH_act (status 0)."""
    W = synth.make_window(nf=nf, npts=50, seed=seed, trans=0.06, rot=0.01, hosts="all")
    w, h = W["w"], W["h"]
    for f in range(nf):
        d = W["dI"][f].reshape(h, w, 3)
        d[200:280, 280:360] = (128.0, 0.0, 0.0)
        if f in nan_frames:
            d[60:120, 440:520] = np.nan
    rng = np.random.default_rng(seed)
    host = np.sort(np.concatenate([np.arange(nf), rng.integers(0, nf, n - nf)])).astype(np.int32)
    edge = rng.random(n) < 0.3
    u = np.where(edge, rng.choice(np.r_[3:12, w - 12:w - 4], n), rng.integers(3, w - 4, n))
    v = rng.integers(3, h - 4, n)
    flat_pts = rng.random(n) < 0.05
    u = np.where(flat_pts, rng.integers(305, 335, n), u); v = np.where(flat_pts, rng.integers(225, 255, n), v)
    parts = [orc.ip_init(W["dI"][hh], w, h, u[host == hh], v[host == hh]) for hh in range(nf)]
    P = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    idt = (0.5 * (1 + 0.02 * rng.standard_normal(n))).astype(np.float32)
    wide = rng.random(n) < 0.5
    P["idepth_min"] = (idt * np.where(wide, 0.7, 0.97)).astype(np.float32)
    P["idepth_max"] = (idt * np.where(wide, 1.4, 1.03)).astype(np.float32)
    bad = rng.random(n) < 0.03
    P["idepth_min"][bad] *= 3; P["idepth_max"][bad] *= 3
    return W, host, P


def activation_partial_oob(W, RT, calib6, host, P, status, idepth, res_state, margin=0.5):
    """(point, target) pairs of activated points whose residual is OOB with its first pattern sample inside the image and a later one
    outside, each by more than `margin` px at the point's final inverse depth (projectPoint in float64)"""
    nf, w, h = W["nf"], W["w"], W["h"]
    fx, fy, cx, cy, fxi, fyi = (float(x) for x in calib6)
    pat = np.array([[0, -2], [-1, -1], [1, -1], [-2, 0], [0, 0], [2, 0], [-1, 1], [0, 2]], np.float64)
    RT = np.asarray(RT, np.float64).reshape(nf * nf, 12)
    out = []
    for i, f in zip(*np.nonzero((np.asarray(res_state) == 1) & (np.asarray(status) == 1)[:, None])):
        M = RT[host[i] * nf + f]
        R, t = M[:9].reshape(3, 3), M[9:]
        Kp = np.stack([(P["u"][i] + pat[:, 0] - cx) * fxi, (P["v"][i] + pat[:, 1] - cy) * fyi, np.ones(8)])
        q = R @ Kp + t[:, None] * float(idepth[i])
        Ku, Kv = q[0] / q[2] * fx + cx, q[1] / q[2] * fy + cy
        inside = (Ku > 1.1 + margin) & (Kv > 1.1 + margin) & (Ku < w - 3 - margin) & (Kv < h - 3 - margin)
        outside = (Ku < 1.1 - margin) | (Kv < 1.1 - margin) | (Ku > w - 3 + margin) | (Kv > h - 3 + margin)
        if inside[0] and outside[1:].any():
            out.append((i, f))
    return out

"""dmv_ct_track_tries (FullSystem::trackNewCoarse's loop over its motion hypotheses in one launch) against the sequential loop.

The reference side of every comparison is loop_reference: FullSystem.cpp:L412-506 (visual-only) restated over CT.track on a twin handle,
each try tracked with the best residuals so far (achievedRes) as its minResForAbort.  Every field of the result must match bit for bit,
NaN payloads included, and so must the sum of the tries' point evaluations.  The tries come from reference_tries, the 31 initial poses of L364-402 built in fp64 from two
frame-to-frame motions (SE3 exp / log and Sophus's normalised quaternions).  The cluster configurations are DMV_CT_CLUSTER=16|8|4 and
unset (the probe's choice), read when a handle first probes."""
import ctypes as C

import numpy as np
import pytest

import helpers as H

DMV_ERR_INVALID, DMV_ERR_STATE = -1, -4
NAN_BITS = 0x7FF8000000000000   # Vec5::Constant(NAN)
_SC = {}


@pytest.fixture(scope="module")
def capi():
    import dmvio_b200.capi as c
    return c


@pytest.fixture
def gpu(capi):
    if capi.lib().dmv_device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on the H100")


# ---------------------------------------------------------------------------------------------------------------------------------
# the 31 tries of FullSystem::trackNewCoarse (L364-402), fp64
# ---------------------------------------------------------------------------------------------------------------------------------
def _hat(w):
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], np.float64)


def se3_exp(xi):
    """Sophus SE3::exp, xi = (upsilon, omega)"""
    ups, om = np.asarray(xi[:3], np.float64), np.asarray(xi[3:], np.float64)
    th = np.linalg.norm(om)
    W = _hat(om)
    if th < 1e-10:
        R = np.eye(3) + W + 0.5 * W @ W
        V = np.eye(3) + 0.5 * W + W @ W / 6.0
    else:
        R = np.eye(3) + np.sin(th) / th * W + (1 - np.cos(th)) / th**2 * (W @ W)
        V = np.eye(3) + (1 - np.cos(th)) / th**2 * W + (th - np.sin(th)) / th**3 * (W @ W)
    return R, V @ ups


def se3_log(R, t):
    """Sophus SE3::log: (upsilon, omega)"""
    c = np.clip((np.trace(R) - 1) / 2, -1.0, 1.0)
    th = np.arccos(c)
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    om = 0.5 * v if th < 1e-10 else th / (2 * np.sin(th)) * v
    W = _hat(om)
    if th < 1e-10:
        Vi = np.eye(3) - 0.5 * W + W @ W / 12.0
    else:
        Vi = np.eye(3) - 0.5 * W + (1 - th * np.sin(th) / (2 * (1 - np.cos(th)))) / th**2 * (W @ W)
    return np.concatenate([Vi @ t, om])


def _inv(T):
    R, t = T
    return R.T, -R.T @ t


def _mul(A, B):
    return A[0] @ B[0], A[0] @ B[1] + A[1]


def _quat(w, x, y, z):
    """SE3(Sophus::Quaterniond(w, x, y, z), 0): the quaternion is normalised"""
    q = np.array([w, x, y, z], np.float64)
    w, x, y, z = q / np.linalg.norm(q)
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return R, np.zeros(3)


def reference_tries(fh_2_slast, lastF_2_slast):
    """lastF_2_fh_tries (L364-402) from fh_2_slast (= slast_2_sprelast) and lastF_2_slast, each an (R, t) pair: 5 motion models, then the
    26 small rotations of the one rotDelta the loop visits (float 0.02)"""
    Ti = _inv(fh_2_slast)
    cm = _mul(Ti, lastF_2_slast)
    half = se3_exp(se3_log(*fh_2_slast) * 0.5)
    tries = [cm, _mul(Ti, cm), _mul(_inv(half), lastF_2_slast), lastF_2_slast, (np.eye(3), np.zeros(3))]
    d = float(np.float32(0.02))
    for x, y, z in [(d, 0, 0), (0, d, 0), (0, 0, d), (-d, 0, 0), (0, -d, 0), (0, 0, -d), (d, d, 0), (0, d, d), (d, 0, d), (-d, d, 0), (0, -d, d),
                    (-d, 0, d), (d, -d, 0), (0, d, -d), (d, 0, -d), (-d, -d, 0), (0, -d, -d), (-d, 0, -d), (-d, -d, -d), (-d, -d, d), (-d, d, -d),
                    (-d, d, d), (d, -d, -d), (d, -d, d), (d, d, -d), (d, d, d)]:
        tries.append(_mul(cm, _quat(1.0, x, y, z)))
    assert len(tries) == 31
    return np.array([R for R, _ in tries]), np.array([t for _, t in tries])


# ---------------------------------------------------------------------------------------------------------------------------------
# FullSystem.cpp:L412-506 restated over CT.track
# ---------------------------------------------------------------------------------------------------------------------------------
def _f32_finite(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return bool(np.isfinite(np.float32(x)))


def loop_reference(g, Rs, ts, kw, lastCoarseRMSE0=100.0, reTrackThreshold=1.5):
    """the sequential loop with one CT.track per try on handle g.  Returns (CT.track_tries's result dict without tries_started, the sum of
    the tries' point evaluations, the per-try history: (track result, achievedRes after the try))"""
    achieved = np.full(5, np.nan)
    flowVecs, R, t, a, b = np.full(3, 100.0), np.eye(3), np.zeros(3), 0.0, 0.0
    goodRet, haveOneGood, tries, winner = 0, 0, 0, -1
    pe, hist = 0.0, []
    lastRes, flow = None, None
    for i in range(len(Rs)):
        r = g.track(R=Rs[i], t=ts[i], minRes=achieved.copy(), **kw)
        pe += g.point_evaluations()
        tries += 1
        good = r["good"] != 0
        if good:
            goodRet = 1
        lastRes, flow = r["lastResiduals"].copy(), r["flow"].copy()
        if good and _f32_finite(lastRes[0]) and not (lastRes[0] >= achieved[0]):   # L467
            flowVecs, R, t, a, b, haveOneGood, winner = flow.copy(), r["R"], r["t"], r["a"], r["b"], 1, i
        if haveOneGood:                                                              # L476-483
            for k in range(5):
                if not _f32_finite(achieved[k]) or achieved[k] > lastRes[k]:
                    achieved[k] = lastRes[k]
        hist.append((r, achieved.copy()))
        if haveOneGood and achieved[0] < float(lastCoarseRMSE0) * float(np.float32(reTrackThreshold)):   # L486
            break
    if not haveOneGood:                                                              # L491-497
        flowVecs, a, b, R, t = np.zeros(3), float(kw["a"]), float(kw["b"]), np.asarray(Rs[0], np.float64).reshape(3, 3), np.asarray(ts[0], np.float64)
    res = dict(R=np.asarray(R, np.float64).reshape(3, 3), t=np.asarray(t, np.float64), a=a, b=b, achievedRes=achieved, flowVecs=flowVecs,
               lastResiduals=lastRes, flow=flow, good=goodRet, haveOneGood=haveOneGood, winner=winner, tries=tries)
    return res, pe, hist


# ---------------------------------------------------------------------------------------------------------------------------------
# scenes, handles, comparison
# ---------------------------------------------------------------------------------------------------------------------------------
def scene(orc, synth, name):
    if name not in _SC:
        _SC[name] = H.ct_scene(orc, synth, name)
    return _SC[name]


def set_configs(monkeypatch, cluster="default"):
    monkeypatch.delenv("DMV_CT_CLUSTER", raising=False)
    if cluster != "default":
        monkeypatch.setenv("DMV_CT_CLUSTER", str(cluster))


def handle(capi, sc, pts=None, k=True):
    pts = sc["pts"] if pts is None else pts
    g = capi.CT(sc["w"], sc["h"], sc["levels"], max_points=max(65536, max(len(p["u"]) for p in pts)))
    for l in range(sc["levels"]):
        if k:
            g.set_K(l, *[float(x) for x in sc["k4"][l]])
        p = pts[l]
        g.set_ref(l, p["u"], p["v"], p["idepth"], p["color"])
        g.upload_new(l, sc["planes"][l])
    return g


def empty_coarsest(sc):
    e = np.zeros(0, np.float32)
    pts = list(sc["pts"])
    pts[sc["levels"] - 1] = dict(u=e, v=e, idepth=e, color=e)
    return pts


def kw(sc, **over):
    """CT.track's keywords but the pose and minRes: a, b = aff_last_2_l"""
    a = dict(sc["args"])
    d = dict(a=a["a0"], b=a["b0"], ref_a=a["ref_a"], ref_b=a["ref_b"], ref_exposure=a["ref_exposure"], new_exposure=a["new_exposure"], cutoff=20.0,
             affA=a["affA"], affB=a["affB"], coarsest=a.get("coarsest"))
    d.update(over)
    return d


def truth(sc):
    return np.asarray(sc["T"]["R_true"], np.float64), np.asarray(sc["T"]["t_true"], np.float64)


def near_truth_tries(sc):
    """lastF_2_slast = the true motion, fh_2_slast = identity: try 0 starts at the truth"""
    return reference_tries((np.eye(3), np.zeros(3)), truth(sc))


def far_tries(sc, rot):
    """fh_2_slast = a rotation of `rot` rad and 0.1 translation: the constant-motion tries start far off, tries 3 and 4 near the truth"""
    return reference_tries(se3_exp(np.array([0.1, -0.05, 0.05, 0.3 * rot, rot, -0.5 * rot])), truth(sc))


def bits(x):
    return np.ascontiguousarray(np.asarray(x, np.float64)).view(np.uint64)


def assert_same(r, s, what):
    keys = [k for k in r if k != "tries_started"]
    assert sorted(keys) == sorted(s.keys()), (keys, s.keys())
    assert r["tries_started"] == r["tries"]
    for k in keys:
        assert np.array_equal(bits(r[k]), bits(s[k])), (what, k, r[k], s[k])


def run_both(g, twin, Rs, ts, k, L=100.0, thr=1.5):
    """track_tries on g and the sequential loop on twin; asserts the bits, the launch count's +1 and the point evaluations"""
    n0 = g.launch_count()
    r = g.track_tries(Rs, ts, lastCoarseRMSE0=L, reTrackThreshold=thr, **k)
    assert g.launch_count() == n0 + 1
    s, pe, hist = loop_reference(twin, Rs, ts, k, lastCoarseRMSE0=L, reTrackThreshold=thr)
    assert_same(r, s, f"L={L} n={len(Rs)}")
    assert len(Rs) >= r["tries"] >= 1
    assert g.point_evaluations() == pe
    return r, s, pe, hist


def later_winner_L(hist):
    """a lastCoarseRMSE0 under which the loop of `hist` (run with L = 0) breaks at a try j that took over a strictly smaller achievedRes[0]
    than the try before it, after an earlier finite one.  Returns (L, j, the first try with a finite achievedRes[0]) or None."""
    a0 = [h[1][0] for h in hist]
    first = next((i for i, x in enumerate(a0) if np.isfinite(x)), None)
    if first is None:
        return None
    for j in range(first + 1, len(a0)):
        if a0[j] < a0[j - 1]:
            return (a0[j] + a0[j - 1]) / 2 / 1.5, j, first
    return None


def close(*hs):
    for g in hs:
        g.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_try0_accepted(capi, gpu, orc, synth, monkeypatch):
    """try 0 starts at the truth and meets the break test at once"""
    set_configs(monkeypatch)
    sc = scene(orc, synth, "bench")
    g, twin = handle(capi, sc), handle(capi, sc)
    Rs, ts = near_truth_tries(sc)
    r, s, _, _ = run_both(g, twin, Rs, ts, kw(sc))
    assert r["tries"] == 1 and r["winner"] == 0 and r["haveOneGood"] == 1 and r["good"] == 1
    close(g, twin)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bench", "odd"])
def test_later_winner(capi, gpu, orc, synth, monkeypatch, name):
    """the loop breaks at a later try whose achievedRes[0] beat an earlier finite winner's"""
    set_configs(monkeypatch)
    sc = scene(orc, synth, name)
    g, twin = handle(capi, sc), handle(capi, sc)
    k = kw(sc)
    found = None
    for Rs, ts in [far_tries(sc, 0.1), near_truth_tries(sc), far_tries(sc, 0.05)]:
        _, _, _, hist = run_both(g, twin, Rs, ts, k, L=0.0)
        found = later_winner_L(hist)
        if found is not None:
            break
    assert found is not None, "no try list of the scene improves achievedRes[0] after a first finite try"
    L, j, first = found
    r, _, _, _ = run_both(g, twin, Rs, ts, k, L=L)
    assert r["tries"] == j + 1 and r["winner"] == j > first and r["haveOneGood"] == 1
    assert r["achievedRes"][0] < 1.5 * L
    close(g, twin)


@pytest.mark.gpu
def test_break_is_strict(capi, gpu, orc, synth, monkeypatch):
    """achievedRes[0] equal to lastCoarseRMSE0 * reTrackThreshold does not break the loop (L486 compares with <)"""
    set_configs(monkeypatch)
    sc = scene(orc, synth, "bench")
    g, twin = handle(capi, sc), handle(capi, sc)
    Rs, ts = near_truth_tries(sc)
    _, _, _, hist = run_both(g, twin, Rs, ts, kw(sc), L=0.0)
    a0 = hist[0][1][0]
    assert np.isfinite(a0)
    r, _, _, _ = run_both(g, twin, Rs, ts, kw(sc), L=a0, thr=1.0)
    assert r["tries"] > 1
    close(g, twin)


@pytest.mark.gpu
def test_nan_block_takes_the_fallback(capi, gpu, orc, synth, monkeypatch):
    """an empty coarsest level: every try aborts on a NaN residual, nothing is good, and the loop returns try 0's pose, aff_last_2_l and zero
    flow, with achievedRes still the initial NaNs"""
    set_configs(monkeypatch)
    sc = scene(orc, synth, "aff_free")
    pts = empty_coarsest(sc)
    g, twin = handle(capi, sc, pts), handle(capi, sc, pts)
    Rs, ts = far_tries(sc, 0.1)
    k = kw(sc)
    r, _, _, _ = run_both(g, twin, Rs, ts, k)
    assert r["tries"] == 31 and r["haveOneGood"] == 0 and r["winner"] == -1 and r["good"] == 0
    np.testing.assert_array_equal(r["R"], Rs[0])
    np.testing.assert_array_equal(r["t"], ts[0])
    assert r["a"] == k["a"] and r["b"] == k["b"] and not r["flowVecs"].any()
    assert (bits(r["achievedRes"]) == NAN_BITS).all()
    close(g, twin)


@pytest.mark.gpu
def test_never_breaks(capi, gpu, orc, synth, monkeypatch):
    """lastCoarseRMSE0 = 0: all 31 tries run, the later ones against the achievedRes of the earlier ones"""
    set_configs(monkeypatch)
    sc = scene(orc, synth, "bench")
    g, twin = handle(capi, sc), handle(capi, sc)
    for Rs, ts in (near_truth_tries(sc), far_tries(sc, 0.1)):
        r, _, _, _ = run_both(g, twin, Rs, ts, kw(sc), L=0.0)
        assert r["tries"] == 31 and r["haveOneGood"] == 1
    close(g, twin)


@pytest.mark.gpu
def test_one_and_32_tries(capi, gpu, orc, synth, monkeypatch):
    set_configs(monkeypatch)
    sc = scene(orc, synth, "aff_fixA")
    g, twin = handle(capi, sc), handle(capi, sc)
    Rs, ts = far_tries(sc, 0.1)
    for L in (100.0, 0.0):
        r, _, _, _ = run_both(g, twin, Rs[:1], ts[:1], kw(sc), L=L)
        assert r["tries"] == 1
    R32, t32 = np.concatenate([Rs, Rs[3:4]]), np.concatenate([ts, ts[3:4]])
    r, _, _, _ = run_both(g, twin, R32, t32, kw(sc), L=0.0)
    assert r["tries"] == 32
    close(g, twin)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bench", "odd", "aff_fixAB"])
def test_coarsest_below_top(capi, gpu, orc, synth, monkeypatch, name):
    set_configs(monkeypatch)
    sc = scene(orc, synth, name)
    g, twin = handle(capi, sc), handle(capi, sc)
    k = kw(sc, coarsest=sc["levels"] - 2)
    for L in (100.0, 0.0):
        r, _, _, _ = run_both(g, twin, *far_tries(sc, 0.05), k, L=L)
        assert np.isnan(r["lastResiduals"][sc["levels"] - 1])
    close(g, twin)


@pytest.mark.gpu
def test_level_repeat(capi, gpu, orc, synth, monkeypatch):
    """the repeat scene saturates at the coarsest level, doubles the cutoff and visits that level twice in every try"""
    set_configs(monkeypatch)
    sc = scene(orc, synth, "repeat")
    g, twin = handle(capi, sc), handle(capi, sc)
    for L in (100.0, 0.0):
        run_both(g, twin, *near_truth_tries(sc), kw(sc), L=L)
    close(g, twin)


def dependent_abort_case(g, sc, k):
    """tries (truth, far): try 0 converges; try 1 completes when tracked alone but its sequential run aborts at a level end against try 0's
    achievedRes.  Returns (Rs, ts, abort level) for the first offset that gives it, tracked on g."""
    R0, t0 = truth(sc)
    for rot in (0.3, 0.2, 0.12, 0.08, 0.05):
        R1, t1 = se3_exp(np.array([0.2, -0.1, 0.1, 0.3 * rot, rot, -0.5 * rot]))
        alone = g.track(R=R1, t=t1, **k)
        first = g.track(R=R0, t=t0, **k)
        if alone["status"] != 0 or first["good"] != 1:
            continue
        after = g.track(R=R1, t=t1, minRes=first["lastResiduals"], **k)
        if after["status"] == 2:
            fin = np.isfinite(after["lastResiduals"])
            return np.array([R0, R1]), np.array([t0, t1]), int(np.flatnonzero(fin).min())
    return None


@pytest.mark.gpu
def test_abort_depends_on_an_earlier_try(capi, gpu, orc, synth, monkeypatch):
    """try 1 completes when tracked alone but aborts against try 0's achievedRes: the result carries that abort, lastResiduals NaN below the
    abort level"""
    set_configs(monkeypatch)
    sc = scene(orc, synth, "bench")
    g, twin = handle(capi, sc), handle(capi, sc)
    k = kw(sc)
    case = dependent_abort_case(twin, sc, k)
    assert case is not None, "no offset of try 1 gives a sequential abort that depends on try 0"
    Rs, ts, lvl = case
    r, s, pe, hist = run_both(g, twin, Rs, ts, k, L=0.0)
    assert r["tries"] == 2 and r["winner"] == 0 and hist[1][0]["status"] == 2
    assert np.isfinite(r["lastResiduals"][lvl]) and np.isnan(r["lastResiduals"][:lvl]).all()
    close(g, twin)


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", ["16", "8", "4", "default"])
def test_configurations(capi, gpu, orc, synth, monkeypatch, cluster):
    """the same bits whatever the cluster size: a break at try 0, loops that never break, and a level-repeat scene"""
    set_configs(monkeypatch, cluster=cluster)
    for name, make, L in (("bench", near_truth_tries, 100.0), ("bench", lambda sc: far_tries(sc, 0.1), 0.0), ("repeat", near_truth_tries, 0.0),
                          ("tma0_160x120", lambda sc: far_tries(sc, 0.05), 0.0)):
        sc = scene(orc, synth, name)
        g, twin = handle(capi, sc), handle(capi, sc)
        run_both(g, twin, *make(sc), kw(sc), L=L)
        close(g, twin)


@pytest.mark.gpu
def test_ordering_and_state(capi, gpu, orc, synth, monkeypatch):
    """an asynchronous frame upload right before the call; the handle's frame, reference and probe stay as they were: a dmv_ct_track after
    the call equals the twin's, and a second call gives the same bits"""
    set_configs(monkeypatch)
    sc = scene(orc, synth, "bench")
    g, twin = handle(capi, sc), handle(capi, sc)
    k = kw(sc)
    Rs, ts = far_tries(sc, 0.1)
    for frame in ("img_ref", "img_new"):
        g.upload_new_image(sc["T"][frame])
        twin.upload_new_image(sc["T"][frame])
        r, _, _, _ = run_both(g, twin, Rs, ts, k, L=0.0)
        r2 = g.track_tries(Rs, ts, lastCoarseRMSE0=0.0, **k)
        assert_same(r2, {q: v for q, v in r.items() if q != "tries_started"}, f"{frame} again")
        n0 = g.launch_count()
        a = g.track(R=Rs[3], t=ts[3], **k)
        assert g.launch_count() == n0 + 1
        b = twin.track(R=Rs[3], t=ts[3], **k)
        assert all(np.array_equal(bits(a[q]), bits(b[q])) for q in a), frame
        assert g.point_evaluations() == twin.point_evaluations()
    close(g, twin)


def raw_call(capi, g, A):
    out = capi.CTTriesResult()
    out.tries, out.tries_started, out.winner, out.a = -99, -99, -99, 7.5
    rc = capi.lib().dmv_ct_track_tries(None if g is None else g.h, None if A is None else C.byref(A), C.byref(out))
    return rc, capi.lib().dmv_last_error().decode(), out


def untouched(out):
    return out.tries == -99 and out.tries_started == -99 and out.winner == -99 and out.a == 7.5


@pytest.mark.gpu
def test_refusals(capi, gpu, orc, synth, monkeypatch):
    set_configs(monkeypatch)
    sc = scene(orc, synth, "tma0_160x120")
    g = handle(capi, sc)
    Rs, ts = near_truth_tries(sc)
    k = kw(sc)
    g.track_tries(Rs, ts, **k)   # probed

    def rejected(h, A, code=DMV_ERR_INVALID, msg=None):
        n0 = h.launch_count() if h is not None else None
        rc, text, out = raw_call(capi, h, A)
        assert rc == code, (rc, text)
        assert untouched(out)
        if msg is not None:
            assert msg in text, text
        if h is not None:
            assert h.launch_count() == n0

    def args(R=Rs, t=ts, **over):
        d = dict(k)
        d.update(over)
        return capi._tries_args(g.levels, R, t, **d)

    rejected(None, args()[0], msg="null")
    rejected(g, None, msg="null")
    A, keep = args()
    A.n = 0
    rejected(g, A, msg="n = 0")
    A.n = 33
    rejected(g, A, msg="n = 33")
    A.n = 31
    A.R = None
    rejected(g, A, msg="null R")
    A, keep = args()
    A.t = None
    rejected(g, A, msg="null R / t")
    for c in (-1, g.levels):
        A, keep = args(coarsest=c)
        rejected(g, A, msg="coarsestLvl")
    rc, text, out = raw_call(capi, g, capi.CTTriesArgs())   # all zero: n = 0
    assert rc == DMV_ERR_INVALID and untouched(out)
    noK = handle(capi, sc, k=False)
    A, keep = args()
    rejected(noK, A, code=DMV_ERR_STATE)
    # the probe's refusal: a cluster size DMV_CT_CLUSTER does not allow
    set_configs(monkeypatch, cluster="5")
    h = handle(capi, sc)
    A, keep = args()
    rejected(h, A, msg="DMV_CT_CLUSTER")
    close(h)
    # after the refusals the probed handle still tracks as before
    set_configs(monkeypatch)
    twin = handle(capi, sc)
    run_both(g, twin, Rs, ts, k)
    close(g, twin, noK)


def test_symbol_and_null_handle(capi):
    """the checks that need no device"""
    L = capi.lib()
    assert hasattr(L, "dmv_ct_track_tries")
    out = capi.CTTriesResult()
    A = capi.CTTriesArgs()
    assert L.dmv_ct_track_tries(None, C.byref(A), C.byref(out)) == DMV_ERR_INVALID
    assert L.dmv_ct_track_tries(None, None, None) == DMV_ERR_INVALID
    assert b"null" in L.dmv_last_error()

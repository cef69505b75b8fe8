"""Plumbing shared by the GPU tests and the benchmark tools: the device fixtures, coarse-tracker handles loaded from helpers.ct_scene, bitwise
comparison, and trackNewCoarse's reference side (the 31 tries and the sequential loop over CT.track).

A test module imports the fixtures it uses, so pytest finds them there: `capi` and `gpu` where a module also has tests that need no device,
`device_capi` (registered as `capi`) where every test that takes `capi` needs one."""
import numpy as np
import pytest

import helpers as H

CONFIGS = ["nc16", "nc8", "nc4", "default"]   # DMV_CT_CLUSTER=16|8|4, and the hook unset (the probe's own choice)
NAN_BITS = 0x7FF8000000000000   # Vec5::Constant(NAN)
_SC = {}


# ---------------------------------------------------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------------------------------------------------
def require_device():
    """dmvio_b200.capi; fails (never skips) the calling test where no CUDA device is visible"""
    import dmvio_b200.capi as c
    if c.lib().dmv_device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on the H100")
    return c


@pytest.fixture(scope="module")
def capi():
    import dmvio_b200.capi as c
    return c


@pytest.fixture
def gpu(capi):
    require_device()


@pytest.fixture(scope="module", name="capi")
def device_capi():
    return require_device()


# ---------------------------------------------------------------------------------------------------------------------------------
# coarse-tracker scenes and handles
# ---------------------------------------------------------------------------------------------------------------------------------
def ct_scene(orc, synth, name):
    """helpers.ct_scene, built once per process"""
    if name not in _SC:
        _SC[name] = H.ct_scene(orc, synth, name)
    return _SC[name]


def set_cluster(monkeypatch, cfg="default"):
    """DMV_CT_CLUSTER for the handles that probe next: a CONFIGS entry or a bare size ("8"); "default" unsets it"""
    monkeypatch.delenv("DMV_CT_CLUSTER", raising=False)
    if cfg != "default":
        monkeypatch.setenv("DMV_CT_CLUSTER", cfg.removeprefix("nc"))


def ct_handle(capi, sc, pts=None, k=True, device=0, L=None):
    """a CT loaded with the scene: K per level (unless k is False), the reference points (pts, default the scene's) and the new frame's
    planes.  L: the library, as CT takes it."""
    pts = sc["pts"] if pts is None else pts
    g = capi.CT(sc["w"], sc["h"], sc["levels"], max_points=max(65536, max(len(p["u"]) for p in pts)), device=device, L=L)
    for l in range(sc["levels"]):
        if k:
            g.set_K(l, *[float(x) for x in sc["k4"][l]])
        p = pts[l]
        g.set_ref(l, p["u"], p["v"], p["idepth"], p["color"])
        g.upload_new(l, sc["planes"][l])
    return g


def empty_coarsest(sc):
    """the scene's reference points with none at the coarsest level"""
    e = np.zeros(0, np.float32)
    pts = list(sc["pts"])
    pts[sc["levels"] - 1] = dict(u=e, v=e, idepth=e, color=e)
    return pts


def track_kw(sc, **over):
    """CT.track's keywords for the scene's arguments; `over` replaces entries of sc["args"] (R0, b0, minRes, ...)"""
    a = dict(sc["args"])
    a.update(over)
    return dict(R=a["R0"], t=a["t0"], a=a["a0"], b=a["b0"], ref_a=a["ref_a"], ref_b=a["ref_b"], ref_exposure=a["ref_exposure"],
                new_exposure=a["new_exposure"], cutoff=20.0, affA=a["affA"], affB=a["affB"], coarsest=a.get("coarsest"), minRes=a.get("minRes"))


def tries_kw(sc, **over):
    """CT.track's keywords but the pose and minRes, as CT.track_tries and loop_reference take them (a, b = aff_last_2_l); `over` replaces
    any of them"""
    d = track_kw(sc)
    del d["R"], d["t"], d["minRes"]
    d.update(over)
    return d


def close(*hs):
    for g in hs:
        g.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# bitwise comparison
# ---------------------------------------------------------------------------------------------------------------------------------
def bits(x):
    return np.ascontiguousarray(np.asarray(x, np.float64)).view(np.uint64)


def assert_same(r, s, what):
    """two result dicts with the same keys and the same bits in every field, NaN payloads included"""
    assert r.keys() == s.keys(), (r.keys(), s.keys())
    for k in r:
        assert np.array_equal(bits(r[k]), bits(s[k])), (what, k, r[k], s[k])


# ---------------------------------------------------------------------------------------------------------------------------------
# the 31 tries of FullSystem::trackNewCoarse (L364-402), fp64.  These SE3 helpers are not synth.se3_exp: the small-angle branches differ,
# and the tries must stay bit for bit as they are.
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


def truth(sc):
    return np.asarray(sc["T"]["R_true"], np.float64), np.asarray(sc["T"]["t_true"], np.float64)


def near_truth_tries(sc):
    """lastF_2_slast = the true motion, fh_2_slast = identity: try 0 starts at the truth"""
    return reference_tries((np.eye(3), np.zeros(3)), truth(sc))


def far_tries(sc, rot):
    """fh_2_slast = a rotation of `rot` rad and 0.1 translation: the constant-motion tries start far off, tries 3 and 4 near the truth"""
    return reference_tries(se3_exp(np.array([0.1, -0.05, 0.05, 0.3 * rot, rot, -0.5 * rot])), truth(sc))


# ---------------------------------------------------------------------------------------------------------------------------------
# FullSystem.cpp:L412-506 restated over CT.track
# ---------------------------------------------------------------------------------------------------------------------------------
def f32_finite(x):
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
        if good and f32_finite(lastRes[0]) and not (lastRes[0] >= achieved[0]):    # L467
            flowVecs, R, t, a, b, haveOneGood, winner = flow.copy(), r["R"], r["t"], r["a"], r["b"], 1, i
        if haveOneGood:                                                              # L476-483
            for k in range(5):
                if not f32_finite(achieved[k]) or achieved[k] > lastRes[k]:
                    achieved[k] = lastRes[k]
        hist.append((r, achieved.copy()))
        if haveOneGood and achieved[0] < float(lastCoarseRMSE0) * float(np.float32(reTrackThreshold)):   # L486
            break
    if not haveOneGood:                                                              # L491-497
        flowVecs, a, b, R, t = np.zeros(3), float(kw["a"]), float(kw["b"]), np.asarray(Rs[0], np.float64).reshape(3, 3), np.asarray(ts[0], np.float64)
    res = dict(R=np.asarray(R, np.float64).reshape(3, 3), t=np.asarray(t, np.float64), a=a, b=b, achievedRes=achieved, flowVecs=flowVecs,
               lastResiduals=lastRes, flow=flow, good=goodRet, haveOneGood=haveOneGood, winner=winner, tries=tries)
    return res, pe, hist


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

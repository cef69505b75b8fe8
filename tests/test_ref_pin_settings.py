"""PINS THE ORACLE TO THE REFERENCE OFF DSO'S DEFAULT SETTINGS: the pins of tests/test_ref_pin.py re-run with setting_huberTH,
setting_outlierTHSumComponent and setting_affineOptModeA / B changed on both sides, so the oracle can stand as ground truth for the device
kernels at those settings (tests/test_gpu_settings.py).

Every setting set must change at least one output against the same run at the defaults: a setting the code path never reads would otherwise
pass for free.  The reference's settings are process-global; the `ref` fixture puts the defaults back after every test, so reference pins
that run later in the same process see DSO's defaults."""
import numpy as np
import pytest

from helpers import activation_case
from test_ref_pin import ba_path_bit_exact, marginalization_bit_exact

DEFAULTS = dict(huberTH=9.0, outlierTHSumComponent=2500.0, affineOptModeA=1e12, affineOptModeB=1e8)


def with_defaults(s):
    return dict(DEFAULTS, **s)


def set_ref_settings(ref, settings):
    """the reference's process-global settings (ref_win_set_setting ignores its window argument)"""
    for k, v in settings.items():
        ref.lib().ref_win_set_setting(None, k.encode(), float(v))


@pytest.fixture
def ref(request):
    from oracle import ref as _ref
    if not _ref.available():
        pytest.skip("oracle/_ref/libdso_ref.so not built and /root/reference absent")
    _ref.lib()
    request.addfinalizer(lambda: set_ref_settings(_ref, DEFAULTS))
    return _ref


def sid(s):
    return "_".join(f"{k}{v:g}" for k, v in s.items())


BA_SETS = [dict(huberTH=4.0), dict(huberTH=30.0), dict(outlierTHSumComponent=100.0), dict(outlierTHSumComponent=1e6),
           dict(affineOptModeA=-1.0), dict(affineOptModeB=-1.0), dict(affineOptModeA=-1.0, affineOptModeB=-1.0)]
BA_CFGS = [dict(nf=5, npts=500, seed=21), dict(nf=8, npts=300, seed=99, hosts="all")]   # incoming OOB / OUTLIER states, priors


def _differs(a, b, keys):
    return [k for k in keys if not np.array_equal(np.asarray(a[k]), np.asarray(b[k]))]


@pytest.mark.parametrize("cfg", BA_CFGS, ids=lambda c: f"nf{c['nf']}_n{c['npts']}")
@pytest.mark.parametrize("s", BA_SETS, ids=sid)
def test_ba_path_bit_exact_off_default(ref, orc, synth, cfg, s):
    """test_ref_pin.py::test_ba_path_bit_exact at the setting set s: linearize outputs, J and JpJdF bit-exact, the accumulated systems to
    1e-12, the solve to 1e-7"""
    E, r, a, p = ba_path_bit_exact(ref, orc, synth, cfg, with_defaults(s))
    E0, r0, a0, p0 = ba_path_bit_exact(ref, orc, synth, cfg, DEFAULTS)
    changed = _differs(r, r0, ("newState", "newEnergy", "J")) + _differs(a, a0, ("HA", "bA")) + (["energy"] if E != E0 else [])
    assert changed, f"{s} changes nothing the pin compares"
    if "affineOptModeA" in s or "affineOptModeB" in s:
        # Residuals.cpp:L229-242: JabF zeroed, JabJIdx / Jab2 kept; so H_A, the states and energies are those of the defaults and only b_A's
        # affine rows of the fixed parameter(s) become exactly 0
        assert E == E0 and not _differs(r, r0, ("newState", "newEnergy")) and not _differs(a, a0, ("HA", "Hsc", "bsc"))
        rows = [4 + 8 * f + j for f in range(cfg["nf"]) for j, k in ((6, "affineOptModeA"), (7, "affineOptModeB")) if k in s]
        assert not a["bA"][rows].any() and np.abs(a0["bA"][rows]).min() > 0
        others = np.setdiff1d(np.arange(len(a["bA"])), rows)
        np.testing.assert_array_equal(a["bA"][others], a0["bA"][others])


MARG_SETS = [dict(huberTH=4.0), dict(affineOptModeA=-1.0, affineOptModeB=-1.0)]


@pytest.mark.parametrize("s", MARG_SETS, ids=sid)
def test_marginalization_bit_exact_off_default(ref, orc, synth, s):
    """test_ref_pin.py::test_marginalization_bit_exact at the setting set s (res_toZeroF bit-exact, M - Msc and Mb - Mbsc to 1e-12)"""
    cfg = dict(nf=7, npts=2000, seed=1234)
    r = marginalization_bit_exact(ref, orc, synth, cfg, with_defaults(s))
    r0 = marginalization_bit_exact(ref, orc, synth, cfg, DEFAULTS)
    assert _differs(r, r0, ("rtz", "b")), f"{s} changes nothing the pin compares"


@pytest.mark.parametrize("huber", [4.0, 30.0])
def test_point_activation_off_default(ref, orc, synth, huber):
    """orc.ip_activate(huberTH=h) against the reference's optimizeImmaturePoint under setting_huberTH = h: status, idepth and residual
    states bit for bit, and different from h = 9"""
    W, host, P = activation_case(synth, orc)
    rw = ref.Window(W, settings=with_defaults(dict(huberTH=huber)))
    ow = orc.Window(W)
    aff = ow.precalc()[:, 24:26].copy()
    calib6 = ow.calib()["k8"][:6]
    for minObs in (1, 3):
        s_o, i_o, r_o = orc.ip_activate(W, ow.RT(), aff, calib6, host, P, minObs=minObs, huberTH=huber)
        s_r, i_r, r_r = rw.activate(host, P, minObs=minObs)
        np.testing.assert_array_equal(s_o, s_r)
        np.testing.assert_array_equal(i_o, i_r)
        np.testing.assert_array_equal(r_o, r_r)
        s_9, i_9, _ = orc.ip_activate(W, ow.RT(), aff, calib6, host, P, minObs=minObs)
        assert (i_9 != i_o).sum() > len(i_o) // 10 or (s_9 != s_o).any()
    assert (s_r == 1).sum() > 0.5 * len(s_r)
    del rw


def lit(pyr, gain, offset):
    """the frame as a camera with `gain` times the exposure and a black level `offset` higher sees it: intensity * gain + offset,
    gradients * gain"""
    out = []
    for p in pyr:
        q = np.asarray(p, np.float32) * np.float32(gain)
        q[..., 0] += np.float32(offset)
        out.append(q)
    return out


# per affine set: (gain, offset, ref_b) of the new frame.  The exposures say the gain (new_exposure = gain) and ref_b is chosen so that
# rb = b - ra ref_b = offset at b = 0: the true photometric change is what the exposures and ref_b predict, so a and b stay small (the
# 1e12 / 1e8 tests |a| > 1.2, |b| > 200 pass) while |log ra| = log 5 > 1.5 and |rb| = 250 > 200 fail the mode-0 tests
AFFINE_LIGHT = {("affineOptModeA",): (5.0, 0.0, -0.5), ("affineOptModeB",): (1.0, 250.0, -250.0), ("affineOptModeA", "affineOptModeB"): (5.0, 250.0, -50.0)}


CT_SETS = [dict(huberTH=4.0), dict(huberTH=30.0), dict(affineOptModeA=0.0), dict(affineOptModeB=0.0), dict(affineOptModeA=0.0, affineOptModeB=0.0)]


@pytest.mark.parametrize("s", CT_SETS, ids=sid)
def test_coarse_tracker_off_default(ref, orc, synth, s):
    """CoarseTracker::calcRes, calcGSSSE and trackNewestCoarse at the setting set s.  The affine-mode-0 sets track a frame lit as
    AFFINE_LIGHT says: trackNewestCoarse's mode-0 tests reject it, the default modes' tests do not.  huberTH changes the energies."""
    full = with_defaults(s)
    ct = {k: full[k] for k in ("huberTH", "affineOptModeA", "affineOptModeB")}
    T = synth.make_tracking_pair(seed=4321)
    gain, offset, ref_b = AFFINE_LIGHT.get(tuple(kk for kk in ("affineOptModeA", "affineOptModeB") if kk in s), (1.0, 0.0, -0.5))
    pyr_new = lit(T["pyr_new"], gain, offset)

    def run(settings):
        set_ref_settings(ref, settings)
        rc = ref.CoarseTracker(T["w"], T["h"], T["K"])
        oc = orc.CoarseTracker(T["w"], T["h"], T["K"], 0, settings=settings)
        for c in (rc, oc):
            c.make_coarse_depth(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"], T["pyr_ref"])
            c.set_new_frame(pyr_new, 1.0, gain, 0.01, ref_b)
        R, t = synth.se3_mul(*synth.se3_exp(np.array([0.003, -0.002, 0.001, 0.001, -0.001, 0.001])), T["R_true"], T["t_true"])
        res = []
        for l in range(rc.levels):
            for cutoff in (20.0, 5.0):
                r6 = rc.calc_res(l, R, t, 0.01, -0.3, cutoff)
                np.testing.assert_array_equal(oc.calc_res(l, R, t, 0.01, -0.3, cutoff), r6)
                np.testing.assert_array_equal(oc.warped(), rc.warped())
                H_r, b_r = rc.calc_gs(l, 0.01, -0.3, 0)
                H_o, b_o = oc.calc_gs(l, 0.01, -0.3, 0)
                np.testing.assert_array_equal(H_o, H_r)
                np.testing.assert_array_equal(b_o, b_r)
                res.append(r6)
        tr = rc.track(np.eye(3), np.zeros(3), 0.0, 0.0, precision=0)
        to = oc.track(np.eye(3), np.zeros(3), 0.0, 0.0, precision=0)
        assert tr["good"] == to["good"]
        np.testing.assert_allclose(to["R"], tr["R"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(to["t"], tr["t"], rtol=0, atol=1e-12)
        assert abs(to["a"] - tr["a"]) < 1e-12 and abs(to["b"] - tr["b"]) < 1e-10
        np.testing.assert_allclose(to["lastResiduals"][:rc.levels], tr["lastResiduals"][:rc.levels], rtol=1e-12)
        del rc
        return np.array(res), tr

    res, tr = run(ct)
    res0, tr0 = run({kk: DEFAULTS[kk] for kk in ct})
    if "huberTH" in s:
        assert not np.array_equal(res[:, 0], res0[:, 0]) and tr["good"]
    else:
        assert not tr["good"] and tr0["good"], (tr["good"], tr0["good"], tr["a"], tr["b"])

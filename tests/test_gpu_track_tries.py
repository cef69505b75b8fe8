"""dmv_ct_track_tries (FullSystem::trackNewCoarse's loop over its motion hypotheses in one launch) against the sequential loop.

The reference side of every comparison is loop_reference: FullSystem.cpp:L412-506 (visual-only) restated over CT.track on a twin handle,
each try tracked with the best residuals so far (achievedRes) as its minResForAbort.  Every field of the result must match bit for bit,
NaN payloads included, and so must the sum of the tries' point evaluations.  The tries come from reference_tries, the 31 initial poses of L364-402 built in fp64 from two
frame-to-frame motions (SE3 exp / log and Sophus's normalised quaternions).  The cluster configurations are DMV_CT_CLUSTER=16|8|4 and
unset (the probe's choice), read when a handle first probes."""
import ctypes as C

import numpy as np
import pytest

from dmvio_b200.capi import DMV_ERR_INVALID, DMV_ERR_STATE
import gpu_harness as G
from gpu_harness import (NAN_BITS, bits, capi, close, ct_handle, ct_scene, empty_coarsest, far_tries, gpu, later_winner_L,  # noqa: F401
                         loop_reference, near_truth_tries, se3_exp, set_cluster, tries_kw, truth)


def assert_same(r, s, what):
    """G.assert_same on every field but tries_started, which must equal tries"""
    assert r["tries_started"] == r["tries"]
    G.assert_same({k: v for k, v in r.items() if k != "tries_started"}, s, what)


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


# ---------------------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_try0_accepted(capi, gpu, orc, synth, monkeypatch):
    """try 0 starts at the truth and meets the break test at once"""
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "bench")
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    Rs, ts = near_truth_tries(sc)
    r, s, _, _ = run_both(g, twin, Rs, ts, tries_kw(sc))
    assert r["tries"] == 1 and r["winner"] == 0 and r["haveOneGood"] == 1 and r["good"] == 1
    close(g, twin)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bench", "odd"])
def test_later_winner(capi, gpu, orc, synth, monkeypatch, name):
    """the loop breaks at a later try whose achievedRes[0] beat an earlier finite winner's"""
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, name)
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    k = tries_kw(sc)
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
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "bench")
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    Rs, ts = near_truth_tries(sc)
    _, _, _, hist = run_both(g, twin, Rs, ts, tries_kw(sc), L=0.0)
    a0 = hist[0][1][0]
    assert np.isfinite(a0)
    r, _, _, _ = run_both(g, twin, Rs, ts, tries_kw(sc), L=a0, thr=1.0)
    assert r["tries"] > 1
    close(g, twin)


@pytest.mark.gpu
def test_nan_block_takes_the_fallback(capi, gpu, orc, synth, monkeypatch):
    """an empty coarsest level: every try aborts on a NaN residual, nothing is good, and the loop returns try 0's pose, aff_last_2_l and zero
    flow, with achievedRes still the initial NaNs"""
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "aff_free")
    pts = empty_coarsest(sc)
    g, twin = ct_handle(capi, sc, pts), ct_handle(capi, sc, pts)
    Rs, ts = far_tries(sc, 0.1)
    k = tries_kw(sc)
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
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "bench")
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    for Rs, ts in (near_truth_tries(sc), far_tries(sc, 0.1)):
        r, _, _, _ = run_both(g, twin, Rs, ts, tries_kw(sc), L=0.0)
        assert r["tries"] == 31 and r["haveOneGood"] == 1
    close(g, twin)


@pytest.mark.gpu
def test_one_and_32_tries(capi, gpu, orc, synth, monkeypatch):
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "aff_fixA")
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    Rs, ts = far_tries(sc, 0.1)
    for L in (100.0, 0.0):
        r, _, _, _ = run_both(g, twin, Rs[:1], ts[:1], tries_kw(sc), L=L)
        assert r["tries"] == 1
    R32, t32 = np.concatenate([Rs, Rs[3:4]]), np.concatenate([ts, ts[3:4]])
    r, _, _, _ = run_both(g, twin, R32, t32, tries_kw(sc), L=0.0)
    assert r["tries"] == 32
    close(g, twin)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bench", "odd", "aff_fixAB"])
def test_coarsest_below_top(capi, gpu, orc, synth, monkeypatch, name):
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, name)
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    k = tries_kw(sc, coarsest=sc["levels"] - 2)
    for L in (100.0, 0.0):
        r, _, _, _ = run_both(g, twin, *far_tries(sc, 0.05), k, L=L)
        assert np.isnan(r["lastResiduals"][sc["levels"] - 1])
    close(g, twin)


@pytest.mark.gpu
def test_level_repeat(capi, gpu, orc, synth, monkeypatch):
    """the repeat scene saturates at the coarsest level, doubles the cutoff and visits that level twice in every try"""
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "repeat")
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    for L in (100.0, 0.0):
        run_both(g, twin, *near_truth_tries(sc), tries_kw(sc), L=L)
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
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "bench")
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    k = tries_kw(sc)
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
    set_cluster(monkeypatch, cluster)
    for name, make, L in (("bench", near_truth_tries, 100.0), ("bench", lambda sc: far_tries(sc, 0.1), 0.0), ("repeat", near_truth_tries, 0.0),
                          ("tma0_160x120", lambda sc: far_tries(sc, 0.05), 0.0)):
        sc = ct_scene(orc, synth, name)
        g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
        run_both(g, twin, *make(sc), tries_kw(sc), L=L)
        close(g, twin)


@pytest.mark.gpu
def test_ordering_and_state(capi, gpu, orc, synth, monkeypatch):
    """an asynchronous frame upload right before the call; the handle's frame, reference and probe stay as they were: a dmv_ct_track after
    the call equals the twin's, and a second call gives the same bits"""
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "bench")
    g, twin = ct_handle(capi, sc), ct_handle(capi, sc)
    k = tries_kw(sc)
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
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "tma0_160x120")
    g = ct_handle(capi, sc)
    Rs, ts = near_truth_tries(sc)
    k = tries_kw(sc)
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
    noK = ct_handle(capi, sc, k=False)
    A, keep = args()
    rejected(noK, A, code=DMV_ERR_STATE)
    # the probe's refusal: a cluster size DMV_CT_CLUSTER does not allow
    set_cluster(monkeypatch, "5")
    h = ct_handle(capi, sc)
    A, keep = args()
    rejected(h, A, msg="DMV_CT_CLUSTER")
    close(h)
    # after the refusals the probed handle still tracks as before
    set_cluster(monkeypatch)
    twin = ct_handle(capi, sc)
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

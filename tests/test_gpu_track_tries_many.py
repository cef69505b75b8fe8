"""dmv_ct_track_tries_many (trackNewCoarse's try loop for several coarse-tracker handles in one launch, one thread-block cluster per handle)
against dmv_ct_track_tries and against the sequential loop.

Every member is held, bit for bit (NaN payloads included), to two things: dmv_ct_track_tries on a twin handle loaded the same way, and
loop_reference, FullSystem.cpp:L412-506 restated over CT.track on that twin.  So are its point evaluations and the +1 of its launch count.
The members of one call differ in their outcomes, scenes, level counts and arguments.  The cluster configurations are DMV_CT_CLUSTER=16|8|4
and unset (the probe's choice), read when a handle first probes."""
import ctypes as C

import numpy as np
import pytest

import gpu_harness as G
from dmvio_b200.capi import DMV_ERR_INVALID, DMV_ERR_STATE
from gpu_harness import (CONFIGS, NAN_BITS, bits, capi, close, ct_handle, ct_scene, empty_coarsest, far_tries, gpu,  # noqa: F401
                         later_winner_L, loop_reference, near_truth_tries, set_cluster, tries_kw)


class Job:
    """one member of a call: its handle, its twin and the arguments of its loop"""

    def __init__(self, capi, sc, Rs, ts, kw, L=100.0, thr=1.5, pts=None, name=""):
        self.g, self.twin = ct_handle(capi, sc, pts), ct_handle(capi, sc, pts)
        self.Rs, self.ts, self.kw, self.L, self.thr, self.name = Rs, ts, kw, L, thr, name or sc["name"]
        self.single = self.pe = None

    def args(self):
        return dict(R=self.Rs, t=self.ts, lastCoarseRMSE0=self.L, reTrackThreshold=self.thr, **self.kw)

    def expect(self):
        """dmv_ct_track_tries on the twin, checked against the sequential loop on the twin; kept for the calls that follow"""
        if self.single is None:
            self.single = self.twin.track_tries(**self.args())
            self.pe = self.twin.point_evaluations()
            s, pe, _ = loop_reference(self.twin, self.Rs, self.ts, self.kw, lastCoarseRMSE0=self.L, reTrackThreshold=self.thr)
            assert self.single["tries_started"] == self.single["tries"]
            G.assert_same({k: v for k, v in self.single.items() if k != "tries_started"}, s, f"{self.name}: track_tries vs loop")
            assert pe == self.pe, self.name
        return self.single

    def close(self):
        close(self.g, self.twin)


def run(capi, jobs, what=""):
    """one dmv_ct_track_tries_many over jobs; every member's result, point evaluations and launch count checked.  Returns the results."""
    expected = [j.expect() for j in jobs]
    before = [j.g.launch_count() for j in jobs]
    rs = capi.ct_track_tries_many([j.g for j in jobs], [j.args() for j in jobs])
    for j, r, s, b in zip(jobs, rs, expected, before):
        G.assert_same(r, s, f"{what} {j.name}")
        assert j.g.point_evaluations() == j.pe, j.name
        assert j.g.launch_count() == b + 1, j.name
    return rs


def hist_of(twin, Rs, ts, kw, L):
    return loop_reference(twin, Rs, ts, kw, lastCoarseRMSE0=L)[2]


def outcome_jobs(capi, orc, synth):
    """members whose loops end differently: try 0 accepted, a later winner, the strict break at equality, the NaN-block fallback, a loop
    that never breaks, 1 try and 32 tries"""
    sc = ct_scene(orc, synth, "bench")
    k = tries_kw(sc)
    jobs = [Job(capi, sc, *near_truth_tries(sc), k, name="try0")]
    later = None
    for Rs, ts in [far_tries(sc, 0.1), near_truth_tries(sc), far_tries(sc, 0.05)]:
        later = Job(capi, sc, Rs, ts, k, L=0.0, name="later")
        found = later_winner_L(hist_of(later.twin, Rs, ts, k, 0.0))
        if found is not None:
            later.L = found[0]
            break
        later.close()
    assert found is not None, "no try list of the scene improves achievedRes[0] after a first finite try"
    jobs.append(later)
    strict = Job(capi, sc, *near_truth_tries(sc), k, thr=1.0, name="strict")
    strict.L = hist_of(strict.twin, strict.Rs, strict.ts, k, 0.0)[0][1][0]
    assert np.isfinite(strict.L)
    jobs.append(strict)
    scn = ct_scene(orc, synth, "aff_free")
    jobs.append(Job(capi, scn, *far_tries(scn, 0.1), tries_kw(scn), pts=empty_coarsest(scn), name="nan_block"))
    jobs.append(Job(capi, sc, *far_tries(sc, 0.1), k, L=0.0, name="never"))
    sca = ct_scene(orc, synth, "aff_fixA")
    Rs, ts = far_tries(sca, 0.1)
    jobs.append(Job(capi, sca, Rs[:1], ts[:1], tries_kw(sca), L=0.0, name="one"))
    jobs.append(Job(capi, sca, np.concatenate([Rs, Rs[3:4]]), np.concatenate([ts, ts[3:4]]), tries_kw(sca), L=0.0, name="32"))
    return jobs, found


def scene_512(orc, synth, levels, seed):
    """a 512x512 scene built as helpers.ct_scene builds the bench scene, with `levels` levels"""
    T = synth.make_tracking_pair(w=512, h=512, seed=seed, levels=levels, npts=2000)
    oc = orc.CoarseTracker(512, 512, T["K"], levels)
    assert oc.levels == levels
    oc.make_coarse_depth(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"], T["pyr_ref"])
    args = dict(R0=np.eye(3), t0=np.zeros(3), a0=0.0, b0=0.0, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0, affA=1e12, affB=1e8)
    return dict(name=f"512x512_{levels}", w=512, h=512, levels=levels, K=T["K"], pts=[oc.ref_points(l) for l in range(levels)], planes=T["pyr_new"],
                k4=[oc.K(l)[0] for l in range(levels)], args=args, T=T)


# ---------------------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS)
def test_outcomes_differ_within_one_call(capi, gpu, orc, synth, monkeypatch, cfg):
    set_cluster(monkeypatch, cfg)
    jobs, found = outcome_jobs(capi, orc, synth)
    for rep in range(2):   # the members probe in the first call; the second reuses the handles
        rs = {j.name: r for j, r in zip(jobs, run(capi, jobs, f"{cfg} call {rep}"))}
        assert rs["try0"]["tries"] == 1 and rs["try0"]["winner"] == 0 and rs["try0"]["good"] == 1
        assert rs["later"]["tries"] == found[1] + 1 and rs["later"]["winner"] == found[1] > found[2]
        assert rs["strict"]["tries"] > 1
        nb = rs["nan_block"]
        assert nb["tries"] == 31 and nb["haveOneGood"] == 0 and nb["winner"] == -1 and (bits(nb["achievedRes"]) == NAN_BITS).all()
        assert rs["never"]["tries"] == 31 and rs["never"]["haveOneGood"] == 1
        assert rs["one"]["tries"] == 1 and rs["32"]["tries"] == 32
    for j in jobs:
        j.close()


@pytest.mark.gpu
def test_scenes_levels_and_coarsest_levels_mix(capi, gpu, orc, synth, monkeypatch):
    """640x480, 752x480, 512x512, 160x120 and 640x96 scenes of 5, 4, 3 and 2 levels in one call, some below their top level, with
    different exposures and affine modes"""
    set_cluster(monkeypatch)
    jobs = []
    for sc, coarsest, make, L in [(ct_scene(orc, synth, "bench"), None, near_truth_tries, 100.0),
                                  (ct_scene(orc, synth, "bench"), 3, lambda s: far_tries(s, 0.05), 0.0),
                                  (scene_512(orc, synth, 4, 16), None, near_truth_tries, 0.0),
                                  (scene_512(orc, synth, 5, 17), 2, lambda s: far_tries(s, 0.05), 100.0),
                                  (ct_scene(orc, synth, "aff_fixB"), None, lambda s: far_tries(s, 0.1), 0.0),
                                  (ct_scene(orc, synth, "odd"), 3, near_truth_tries, 0.0),
                                  (ct_scene(orc, synth, "tma0_160x120"), None, lambda s: far_tries(s, 0.05), 0.0),
                                  (ct_scene(orc, synth, "wide"), 1, near_truth_tries, 100.0)]:
        kw = tries_kw(sc, coarsest=coarsest)
        jobs.append(Job(capi, sc, *make(sc), kw, L=L, name=f"{sc['name']}/{coarsest}"))
    rs = run(capi, jobs)
    for j, r in zip(jobs, rs):
        c = j.kw["coarsest"]
        if c is not None and c < j.g.levels - 1:
            assert np.isnan(r["lastResiduals"][j.g.levels - 1]), j.name
    for j in jobs:
        j.close()


def sixteen(capi, orc, synth):
    names = ["bench", "aff_free", "aff_fixA", "odd", "tma0_160x120", "repeat", "wide", "limit"]
    jobs = []
    for i in range(16):
        sc = ct_scene(orc, synth, names[i % len(names)])
        Rs, ts = near_truth_tries(sc) if i % 3 == 0 else far_tries(sc, 0.05 if i % 2 else 0.1)
        jobs.append(Job(capi, sc, Rs[:31 - i], ts[:31 - i], tries_kw(sc), L=(100.0, 0.0, 1.0)[i % 3], name=f"{i}:{sc['name']}"))
    return jobs


@pytest.mark.gpu
def test_sixteen_members_subsets_and_order(capi, gpu, orc, synth, monkeypatch):
    """16 members, then the same handles reversed, every other one, pairs and single members (the single-member call launches
    ct_track_tries_kernel); the handles left out of a call keep their launch counts"""
    set_cluster(monkeypatch)
    jobs = sixteen(capi, orc, synth)
    n = len(jobs)
    calls = [list(range(n)), list(range(n))[::-1], list(range(0, n, 2)), list(range(1, n, 2)), [5, 0], [15, 3, 9], [0], [7], [15]]
    for idx in calls:
        before = [j.g.launch_count() for j in jobs]
        run(capi, [jobs[i] for i in idx], f"call {idx}")
        assert [j.g.launch_count() - b for j, b in zip(jobs, before)] == [int(i in idx) for i in range(n)]
    for j in jobs:
        j.close()


@pytest.mark.gpu
def test_ordered_behind_asynchronous_uploads(capi, gpu, orc, synth, monkeypatch):
    """each member's frame arrives by dmv_ct_upload_new_image or dmv_ct_upload_raw_image right before the call, with no synchronisation in
    between: the launch must wait for every member's upload; then a second frame goes through the same handles"""
    set_cluster(monkeypatch)
    jobs = []
    for i, name in enumerate(["bench", "odd", "aff_free", "tma0_160x120", "wide"]):
        sc = ct_scene(orc, synth, name)
        jobs.append(Job(capi, sc, *far_tries(sc, 0.05), tries_kw(sc), L=0.0))
        jobs[-1].sc, jobs[-1].raw = sc, i % 2 == 1
        if jobs[-1].raw:
            for x in (jobs[-1].g, jobs[-1].twin):
                x.set_undistort(sc["w"], sc["h"])

    def upload(j, x, frame):
        img = j.sc["T"][frame]
        if j.raw:
            x.upload_raw_image(np.clip(np.round(img), 0, 255).astype(np.uint8))
        else:
            x.upload_new_image(img)

    for frame in ("img_ref", "img_new"):
        for j in jobs:   # the twins first: their expectations are computed before the members' uploads are issued
            upload(j, j.twin, frame)
            j.single = None
            j.expect()
        for j in jobs:
            upload(j, j.g, frame)
        run(capi, jobs, frame)
    for j in jobs:
        j.close()


@pytest.mark.gpu
def test_state_after_the_call(capi, gpu, orc, synth, monkeypatch):
    """after the call every handle tracks as handles that never saw it: dmv_ct_track, dmv_ct_track_many and dmv_ct_track_tries"""
    set_cluster(monkeypatch)
    jobs = []
    for name in ("bench", "aff_fixAB", "odd"):
        sc = ct_scene(orc, synth, name)
        jobs.append(Job(capi, sc, *far_tries(sc, 0.1), tries_kw(sc), L=0.0))
    run(capi, jobs)
    fresh = [ct_handle(capi, ct_scene(orc, synth, n)) for n in ("bench", "aff_fixAB", "odd")]
    gs = [j.g for j in jobs]
    for j, f in zip(jobs, fresh):
        a = dict(R=j.Rs[3], t=j.ts[3], **j.kw)
        n0 = j.g.launch_count()
        G.assert_same(j.g.track(**a), f.track(**a), f"{j.name} track")
        assert j.g.point_evaluations() == f.point_evaluations() and j.g.launch_count() == n0 + 1
        G.assert_same(j.g.track_tries(**j.args()), f.track_tries(**j.args()), f"{j.name} track_tries")
        assert j.g.point_evaluations() == f.point_evaluations()
    args = [dict(R=j.Rs[0], t=j.ts[0], **j.kw) for j in jobs]
    for r, s, j in zip(capi.ct_track_many(gs, args), capi.ct_track_many(fresh, args), jobs):
        G.assert_same(r, s, f"{j.name} track_many")
    close(*fresh)
    for j in jobs:
        j.close()


def raw_call(capi, hs, As):
    """dmv_ct_track_tries_many through the raw symbol (hs may hold None, hs / As may be None); returns (rc, message, out) with out pre-filled
    with a sentinel"""
    m = max(len(hs or []), len(As or []), 1)
    H_ = None if hs is None else (C.c_void_p * m)(*[None if g is None else g.h.value for g in hs])
    A_ = None if As is None else (capi.CTTriesArgs * m)(*As)
    out = (capi.CTTriesResult * m)()
    for o in out:
        o.tries, o.tries_started, o.winner, o.a = -99, -99, -99, 7.5
    rc = capi.lib().dmv_ct_track_tries_many(H_, len(hs) if hs is not None else m, A_, out)
    return rc, capi.lib().dmv_last_error().decode(), out


def untouched(out):
    return all(o.tries == -99 and o.tries_started == -99 and o.winner == -99 and o.a == 7.5 for o in out)


@pytest.mark.gpu
def test_refusals(capi, gpu, orc, synth, monkeypatch):
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "tma0_160x120")
    gs = [ct_handle(capi, sc) for _ in range(17)]
    Rs, ts = near_truth_tries(sc)
    k = tries_kw(sc)
    gs[0].track_tries(Rs, ts, **k)   # one member has probed already, the others probe inside the call
    counts = [g.launch_count() for g in gs]
    keep = []

    def A(**over):
        d = dict(R=Rs, t=ts, **k)
        d.update(over)
        a, arrays = capi._tries_args(sc["levels"], **d)
        keep.append(arrays)
        return a

    def rejected(hs, As, code=DMV_ERR_INVALID, msg=None):
        rc, text, out = raw_call(capi, hs, As)
        assert rc == code, (rc, text)
        assert untouched(out)
        if msg is not None:
            assert msg in text, text
        assert [g.launch_count() for g in gs] == counts
        return text

    a = A()
    rejected(gs[:0], [a], msg="n = 0")
    rejected(gs, [a] * 17, msg="n = 17")
    rejected(None, [a] * 2, msg="null argument")
    rejected(gs[:2], None, msg="null argument")
    rc = capi.lib().dmv_ct_track_tries_many((C.c_void_p * 1)(gs[0].h.value), 1, (capi.CTTriesArgs * 1)(a), None)
    assert rc == DMV_ERR_INVALID and "null argument" in capi.lib().dmv_last_error().decode()
    rejected([gs[0], None, gs[2]], [a] * 3, msg="handles[1] is NULL")
    rejected([gs[0], gs[1], gs[0]], [a] * 3, msg="handles[0] and handles[2]")
    noR, noT = A(), A()
    noR.R, noT.t = None, None
    assert "handles[1]: null R / t" in rejected(gs[:3], [a, noR, a])
    assert "handles[2]: null R / t" in rejected(gs[:3], [a, a, noT])
    for n in (0, 33):
        bad = A()
        bad.n = n
        assert f"handles[2]: n = {n}" in rejected(gs[:4], [a, a, bad, a])
    text = rejected(gs[:5], [a, a, a, A(coarsest=sc["levels"]), a], msg="handles[3]")
    assert "coarsestLvl" in text
    noK = ct_handle(capi, sc, k=False)
    n_noK = noK.launch_count()
    rejected([gs[0], gs[1], noK], [a] * 3, code=DMV_ERR_STATE, msg="handles[2]")
    assert noK.launch_count() == n_noK
    close(noK)
    # cluster sizes that differ: one handle probed under DMV_CT_CLUSTER=8, another under 16
    monkeypatch.setenv("DMV_CT_CLUSTER", "8")
    g8 = ct_handle(capi, sc)
    g8.track_tries(Rs, ts, **k)
    monkeypatch.setenv("DMV_CT_CLUSTER", "16")
    g16 = ct_handle(capi, sc)
    g16.track_tries(Rs, ts, **k)
    n8, n16 = g8.launch_count(), g16.launch_count()
    text = rejected([g16, g8], [a, a], msg="handles[1]")
    assert "handles[0]" in text and "cluster" in text and g8.launch_count() == n8 and g16.launch_count() == n16
    close(g8, g16)
    # after the refusals the handles still track as before
    set_cluster(monkeypatch)
    twin = ct_handle(capi, sc)
    expected = twin.track_tries(Rs, ts, **k)
    for r in capi.ct_track_tries_many(gs[:3], [dict(R=Rs, t=ts, **k)] * 3):
        G.assert_same(r, expected, "after the refusals")
    close(twin, *gs)


@pytest.mark.gpu
def test_handles_on_two_devices_are_rejected(capi, gpu, orc, synth, monkeypatch):
    if capi.lib().dmv_device_count() < 2:
        pytest.skip("needs two visible GPUs")
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, "tma0_160x120")
    g0, g1 = ct_handle(capi, sc, device=0), ct_handle(capi, sc, device=1)
    a, keep = capi._tries_args(sc["levels"], *near_truth_tries(sc), **tries_kw(sc))
    rc, text, out = raw_call(capi, [g0, g1], [a, a])
    assert rc == DMV_ERR_INVALID and "device" in text and untouched(out)
    assert g0.launch_count() == g1.launch_count()
    close(g0, g1)


def test_symbol_and_arguments_without_handles(capi):
    """the checks that need no handle and no device"""
    L = capi.lib()
    assert hasattr(L, "dmv_ct_track_tries_many")
    out = (capi.CTTriesResult * 1)()
    A = (capi.CTTriesArgs * 1)()
    hs = (C.c_void_p * 1)(None)
    assert L.dmv_ct_track_tries_many(None, 1, A, out) == DMV_ERR_INVALID
    assert b"null argument" in L.dmv_last_error()
    assert L.dmv_ct_track_tries_many(hs, 1, None, out) == DMV_ERR_INVALID
    assert L.dmv_ct_track_tries_many(hs, 1, A, None) == DMV_ERR_INVALID
    assert L.dmv_ct_track_tries_many(hs, 0, A, out) == DMV_ERR_INVALID
    assert b"n = 0" in L.dmv_last_error()
    assert L.dmv_ct_track_tries_many(hs, 17, A, out) == DMV_ERR_INVALID
    assert b"n = 17" in L.dmv_last_error()
    assert L.dmv_ct_track_tries_many(hs, 1, A, out) == DMV_ERR_INVALID
    assert b"handles[0] is NULL" in L.dmv_last_error()
    with pytest.raises(capi.DmvError, match="n = 0"):
        capi.ct_track_tries_many([], [])

"""dmv_ct_track_many (several coarse-tracker handles tracked in one launch, one thread-block cluster per handle) against dmv_ct_track.

The single side of every comparison is a twin handle loaded the same way and tracked with dmv_ct_track; every field of the result must match
bit for bit (NaN positions and payloads included), and so must dmv_ct_last_point_evaluations and the +1 of dmv_ct_kernel_launch_count.
The cluster configurations are those of test_gpu_coarse_track.py: DMV_CT_CLUSTER=16|8|4, read when a handle first tracks, and "default"
(the hook unset, the probe's own choice).  Every error case is rejected before anything is launched."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
from dmvio_b200.capi import DMV_ERR_INVALID, DMV_ERR_STATE
from gpu_harness import CONFIGS, assert_same, capi, close, ct_handle, ct_scene, empty_coarsest, gpu, set_cluster, track_kw  # noqa: F401

# 15 members: 1-5 levels, five image shapes, all four affine modes, staged and L2-gathered levels, the 80 KiB limit, the box-limit level of
# wide, stream's more-points-than-register-slots loop and repeat's cutoff doubling.  At nc16 they need more clusters than are co-resident.
MEMBERS = H.CT_SCENES + ["counts_1", "counts_31", "counts_513"]
ABORTS = [("aff_free", w) for w in ("minRes_coarsest", "minRes_l1", "minRes_l0", "empty_coarsest")] + \
         [(n, w) for n in ("counts_1", "counts_31", "counts_513") for w in ("minRes_coarsest", "empty_coarsest")]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS)
def test_many_is_bit_identical_to_single(capi, gpu, orc, synth, monkeypatch, cfg):
    set_cluster(monkeypatch, cfg)
    scs = [ct_scene(orc, synth, n) for n in MEMBERS]
    gs = [ct_handle(capi, sc) for sc in scs]
    twins = [ct_handle(capi, sc) for sc in scs]
    args = [track_kw(sc) for sc in scs]
    singles = [t.track(**a) for t, a in zip(twins, args)]
    for rep in range(2):   # the members probe in the first call; the second reuses the handles
        before = [g.launch_count() for g in gs]
        rs = capi.ct_track_many(gs, args)
        for name, g, t, r, s, b in zip(MEMBERS, gs, twins, rs, singles, before):
            assert_same(r, s, f"{cfg} {name} call {rep}")
            assert g.point_evaluations() == t.point_evaluations() > 0, name
            assert g.launch_count() == b + 1, name
    close(*gs, *twins)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS)
def test_aborts_stay_local(capi, gpu, orc, synth, monkeypatch, cfg):
    """the abort cases of test_gpu_coarse_track.py::test_abort_contract mixed with members that track normally, in one call"""
    set_cluster(monkeypatch, cfg)
    cases = [("bench", None)] + ABORTS[:5] + [("stream", None)] + ABORTS[5:] + [("aff_fixA", None)]
    gs, twins, args = [], [], []
    for name, where in cases:
        sc = ct_scene(orc, synth, name)
        L = sc["levels"]
        pts = None
        over = {}
        if where == "empty_coarsest":
            pts = empty_coarsest(sc)
        twin = ct_handle(capi, sc, pts)
        if where is not None and where.startswith("minRes"):
            lvl = {"minRes_coarsest": L - 1, "minRes_l1": 1, "minRes_l0": 0}[where]
            full = twin.track(**track_kw(sc))
            assert full["status"] == 0 and full["lastResiduals"][lvl] > 0
            mr = np.full(5, np.nan)
            mr[lvl] = full["lastResiduals"][lvl] / 3
            over["minRes"] = mr
        gs.append(ct_handle(capi, sc, pts))
        twins.append(twin)
        args.append(track_kw(sc, **over))
    singles = [t.track(**a) for t, a in zip(twins, args)]
    rs = capi.ct_track_many(gs, args)
    for (name, where), r, s, a in zip(cases, rs, singles, args):
        assert_same(r, s, f"{cfg} {name} {where}")
        if where is None:
            assert r["status"] == 0
        else:
            assert r["status"] == 2 and r["good"] == 0
            np.testing.assert_array_equal(r["R"], np.asarray(a["R"], np.float64))
            np.testing.assert_array_equal(r["t"], np.asarray(a["t"], np.float64))
            assert r["a"] == a["a"] and r["b"] == a["b"]
    close(*gs, *twins)


@pytest.mark.gpu
def test_subsets_and_order(capi, gpu, orc, synth, monkeypatch):
    """the same handles in successive calls: every one alone, reversed, every other one and all of them"""
    set_cluster(monkeypatch, "default")
    names = ["bench", "aff_free", "tma0_80x60", "odd", "wide", "repeat"]
    scs = [ct_scene(orc, synth, n) for n in names]
    gs = [ct_handle(capi, sc) for sc in scs]
    twins = [ct_handle(capi, sc) for sc in scs]
    args = [track_kw(sc) for sc in scs]
    singles = [t.track(**a) for t, a in zip(twins, args)]
    calls = [[i] for i in range(len(gs))] + [list(range(len(gs)))[::-1], list(range(0, len(gs), 2)), list(range(1, len(gs), 2)), list(range(len(gs)))]
    for idx in calls:
        before = [g.launch_count() for g in gs]
        rs = capi.ct_track_many([gs[i] for i in idx], [args[i] for i in idx])
        for i, r in zip(idx, rs):
            assert_same(r, singles[i], f"{names[i]} in call {idx}")
            assert gs[i].point_evaluations() == twins[i].point_evaluations()
        assert [g.launch_count() - b for g, b in zip(gs, before)] == [int(i in idx) for i in range(len(gs))]
    close(*gs, *twins)


@pytest.mark.gpu
def test_ordered_behind_asynchronous_uploads(capi, gpu, orc, synth, monkeypatch):
    """dmv_ct_upload_new_image returns before its copy and pyramid have run; the launch must wait for every member's, then a second frame
    goes through the same handles"""
    set_cluster(monkeypatch, "default")
    scs = [ct_scene(orc, synth, n) for n in H.CT_SCENES]
    gs = [ct_handle(capi, sc) for sc in scs]
    twins = [ct_handle(capi, sc) for sc in scs]
    args = [track_kw(sc) for sc in scs]
    for frame in ("img_ref", "img_new"):
        for g, sc in zip(gs, scs):
            g.upload_new_image(sc["T"][frame])
        rs = capi.ct_track_many(gs, args)
        for t, sc, a, r, name in zip(twins, scs, args, rs, H.CT_SCENES):
            t.upload_new_image(sc["T"][frame])
            assert_same(r, t.track(**a), f"{name} {frame}")
    close(*gs, *twins)


def raw_call(capi, hs, args):
    """dmv_ct_track_many through the raw symbol (hs may hold None); returns (rc, message, out) with out pre-filled with a sentinel"""
    n = len(hs)
    m = max(n, 1)
    H_ = (C.c_void_p * m)(*[None if g is None else g.h.value for g in hs])
    A = (capi.CTTrackArgs * m)(*[capi._track_args(g.levels if g is not None else 1, **a) for g, a in zip(hs, args)])
    out = (capi.CTTrackResult * m)()
    for o in out:
        o.status, o.iterations, o.a = -99, -99, 7.5
    rc = capi.lib().dmv_ct_track_many(H_, n, A, out)
    return rc, capi.lib().dmv_last_error().decode(), out


def untouched(out):
    return all(o.status == -99 and o.iterations == -99 and o.a == 7.5 for o in out)


@pytest.mark.gpu
def test_errors_are_rejected_before_launch(capi, gpu, orc, synth, monkeypatch):
    set_cluster(monkeypatch, "default")
    sc = ct_scene(orc, synth, "tma0_80x60")
    gs = [ct_handle(capi, sc) for _ in range(17)]
    a = track_kw(sc)
    gs[0].track(**a)            # one member has probed already, the others probe inside the call
    counts = [g.launch_count() for g in gs]

    def rejected(hs, args, code=DMV_ERR_INVALID, msg=None):
        rc, text, out = raw_call(capi, hs, args)
        assert rc == code, (rc, text)
        assert untouched(out)
        if msg is not None:
            assert msg in text, text
        assert [g.launch_count() for g in gs] == counts
        return text

    rejected(gs[:0], [], msg="n = 0")
    rejected(gs, [a] * 17, msg="n = 17")
    rejected([gs[0], None, gs[2]], [a] * 3, msg="handles[1] is NULL")
    rejected([gs[0], gs[1], gs[0]], [a] * 3, msg="handles[0] and handles[2]")
    noK = ct_handle(capi, sc, k=False)
    n_noK = noK.launch_count()
    rejected([gs[0], gs[1], noK], [a] * 3, code=DMV_ERR_STATE, msg="handles[2]")
    assert noK.launch_count() == n_noK
    bad = [a] * 3 + [track_kw(sc, coarsest=sc["levels"])] + [a]
    text = rejected(gs[:5], bad, msg="handles[3]")
    assert "coarsestLvl" in text
    close(noK)
    # cluster sizes that differ: one handle probed under DMV_CT_CLUSTER=8, another under 16
    monkeypatch.setenv("DMV_CT_CLUSTER", "8")
    g8 = ct_handle(capi, sc)
    g8.track(**a)
    monkeypatch.setenv("DMV_CT_CLUSTER", "16")
    g16 = ct_handle(capi, sc)
    g16.track(**a)
    n8, n16 = g8.launch_count(), g16.launch_count()
    text = rejected([g16, g8], [a, a], msg="handles[1]")
    assert "handles[0]" in text and g8.launch_count() == n8 and g16.launch_count() == n16
    close(g8, g16, *gs)


@pytest.mark.gpu
def test_handles_on_two_devices_are_rejected(capi, gpu, orc, synth, monkeypatch):
    if capi.lib().dmv_device_count() < 2:
        pytest.skip("needs two visible GPUs")
    set_cluster(monkeypatch, "default")
    sc = ct_scene(orc, synth, "tma0_80x60")
    g0, g1 = ct_handle(capi, sc, device=0), ct_handle(capi, sc, device=1)
    rc, text, out = raw_call(capi, [g0, g1], [track_kw(sc)] * 2)
    assert rc == DMV_ERR_INVALID and "device" in text and untouched(out)
    assert g0.launch_count() == g1.launch_count()
    close(g0, g1)


def test_arguments_without_handles_are_rejected(capi):
    """the checks that need no handle and no device"""
    L = capi.lib()
    out = (capi.CTTrackResult * 1)()
    A = (capi.CTTrackArgs * 1)()
    assert L.dmv_ct_track_many(None, 1, A, out) == DMV_ERR_INVALID
    hs = (C.c_void_p * 1)(None)
    assert L.dmv_ct_track_many(hs, 0, A, out) == DMV_ERR_INVALID
    assert b"n = 0" in L.dmv_last_error()
    assert L.dmv_ct_track_many(hs, 17, A, out) == DMV_ERR_INVALID
    assert L.dmv_ct_track_many(hs, 1, None, out) == DMV_ERR_INVALID
    assert L.dmv_ct_track_many(hs, 1, A, None) == DMV_ERR_INVALID
    assert L.dmv_ct_track_many(hs, 1, A, out) == DMV_ERR_INVALID
    assert b"handles[0] is NULL" in L.dmv_last_error()
    with pytest.raises(capi.DmvError, match="n = 0"):
        capi.ct_track_many([], [])

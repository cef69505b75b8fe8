"""dmv_ct_trace_many (the immature points of several coarse-tracker handles traced in one launch) against dmv_ct_trace_points_multi.

Every member has a twin handle loaded the same way and traced with dmv_ct_trace_points_multi: every in/out field of every member must equal
the twin's bit for bit (NaN payloads included) and the oracle's traceOn (pinned to the reference's compiled ImmaturePoint.cpp by
tests/test_ref_pin_ip.py), and each member's launch count must move as the twin's does.  The kernel gives each member whole CTAs of 4
points, so members of 1, 3, 5 and 4k + 1 points end inside a CTA, and empty members and empty host sets sit between non-empty ones.
Every refused call leaves each member's output arrays and launch count as they were."""
import ctypes as C

import numpy as np
import pytest

import gpu_harness as G
import helpers as H
from dmvio_b200.capi import DMV_ERR_INVALID
from gpu_harness import capi, close, gpu  # noqa: F401

MANY_MAX = 16


class Member:
    """one handle's immature points: sets[k] hosted by frame hosts[k]; step t traces all of them against frames[seq[t]]"""

    def __init__(self, name, w, h, frames, sets, hosts, tabs, seq, images=None):
        self.name, self.w, self.h, self.frames, self.state, self.hosts, self.tabs, self.seq = name, w, h, frames, sets, hosts, tabs, seq
        self.images = images

    def job(self, t):
        return [(P,) + tuple(self.tabs(hst, self.seq[t])) for P, hst in zip(self.state, self.hosts)]

    def npoints(self):
        return sum(len(P["u"]) for P in self.state)


def window_member(synth, orc, name, seed, counts, w=640, h=480, nhost=None):
    """a synth.make_window scene: set k (counts[k] points) hosted by frame k % nhost, traced against the two frames after the hosts"""
    import dmvio_b200.hostmath as hm
    nhost = nhost or max(1, len(counts))
    W = synth.make_window(nf=nhost + 2, npts=10, seed=seed, trans=0.05, rot=0.01, w=w, h=h)
    rng = np.random.default_rng(seed)
    sets, hosts = [], []
    for k, n in enumerate(counts):
        hst = k % nhost
        u, v = rng.integers(10, w - 10, n), rng.integers(10, h - 10, n)
        sets.append(orc.ip_init(W["dI"][hst], w, h, u, v))
        hosts.append(hst)
    return Member(name, w, h, W["dI"], sets, hosts, lambda hst, f: hm.trace_tables(W, hst, f), (nhost, nhost + 1, nhost), W["images"])


def ip_case_member(name, S, P):
    import dmvio_b200.hostmath as hm
    return Member(name, S["w"], S["h"], S["dI"], [P], [0], lambda hst, f: hm.trace_tables(S, hst, f), H.IP_TRACE_SEQ, S["images"])


def gn_oob_member():
    P, dI, w, h, KRKi, Kt, aff = H.ip_gn_oob_case()
    return Member("gn_oob", w, h, [dI], [P], [0], lambda hst, f: (KRKi, Kt, aff), (0, 0, 0))


def empty_member(synth, orc, name, seed):
    return window_member(synth, orc, name, seed, [])


def bits(a):
    return np.ascontiguousarray(a).reshape(-1).view(np.uint32)


def handles(capi, synth, ms):
    return [capi.CT(m.w, m.h, synth.pyr_levels(m.w, m.h), max_points=1024) for m in ms]


def step(capi, orc, ms, gs, twins, t, settings=None, oracle=True, upload=None):
    """frame seq[t] into every member and twin, one dmv_ct_trace_many against one dmv_ct_trace_points_multi per twin; advances the state"""
    for m, g, tw in zip(ms, gs, twins):
        f = m.seq[t]
        for x in (g, tw):
            if upload is None:
                x.upload_new(0, m.frames[f])
            else:
                upload(m, x, f)
    jobs = [m.job(t) for m in ms]
    before = [g.launch_count() for g in gs]
    got = capi.ct_trace_many(gs, jobs, settings)
    for m, g, tw, job, r, b in zip(ms, gs, twins, jobs, got, before):
        tb = tw.launch_count()
        single = tw.trace_points_multi(job, settings)
        grew = tw.launch_count() - tb
        assert grew == int(m.npoints() > 0), m.name
        assert g.launch_count() - b == grew, f"{m.name}: launch count"
        assert len(r) == len(job)
        for k, (Q, S_, J) in enumerate(zip(r, single, job)):
            for key in H_KEYS:
                assert np.array_equal(bits(Q[key]), bits(S_[key])), f"{m.name} step {t} set {k}: {key} differs from dmv_ct_trace_points_multi"
            if oracle:
                ref = orc.ip_trace(J[0], m.frames[m.seq[t]], m.w, m.h, *J[1:])
                for key in H_KEYS:
                    np.testing.assert_array_equal(Q[key], ref[key], err_msg=f"{m.name} step {t} set {k}: {key} vs the oracle")
        m.state = r
    return got


H_KEYS = ("idepth_min", "idepth_max", "quality", "status", "lastTraceUV", "lastTracePixelInterval")


@pytest.mark.gpu
def test_mixed_members(capi, gpu, orc, synth):
    """640x480 and 512x512 windows, every lane round of the search (848x800 .. 2560x1280 with the clamp at 99), every status with NaN
    boxes, GN leaving the image, and two empty members, in one call per frame of IP_TRACE_SEQ (sticky OOB and refinement on calls 2 and 3)"""
    ms = [window_member(synth, orc, "640x480", 5, [700, 1, 1300, 257]), empty_member(synth, orc, "empty_a", 6),
          window_member(synth, orc, "512x512", 12, [300, 0, 501], w=512, h=512)]
    for w, h, seed in H.IP_ROUND_SHAPES:
        ms.append(ip_case_member(f"{w}x{h}", *H.ip_round_case(synth, orc, w, h, seed)))
    ms.append(ip_case_member("statuses", *H.ip_status_case(synth, orc)))
    ms.append(empty_member(synth, orc, "empty_b", 7))
    ms.append(gn_oob_member())
    gs, twins = handles(capi, synth, ms), handles(capi, synth, ms)
    seen = np.zeros(6, int)
    for t in range(3):
        got = step(capi, orc, ms, gs, twins, t)
        for r in got:
            for Q in r:
                seen += np.bincount(Q["status"], minlength=6)
    assert (seen[:5] > 0).all(), seen
    close(*gs, *twins)


@pytest.mark.gpu
def test_member_boundaries(capi, gpu, orc, synth):
    """DMV_CT_TRACE_MANY_MAX members with 0, 1, 3, 5, 4k + 1 points, empty sets between non-empty ones, one member past 2048 points (its
    staging area grows inside the call) and one with 64 host frames"""
    specs = [[0], [1], [3], [5], [401], [0, 7, 0, 0, 3, 0], [], [1300, 1301], [2] * 64, [0, 0], [33], [4], [2, 0, 2], [6, 1], [97], [1]]
    assert len(specs) == MANY_MAX
    ms = [window_member(synth, orc, f"m{i}:{sum(c)}", 40 + i, c, nhost=3 if len(c) == 64 else None) for i, c in enumerate(specs)]
    assert max(len(m.state) for m in ms) == 64 and max(m.npoints() for m in ms) > 2048
    gs, twins = handles(capi, synth, ms), handles(capi, synth, ms)
    for t in range(2):
        step(capi, orc, ms, gs, twins, t)
    close(*gs, *twins)


@pytest.mark.gpu
def test_counts_subsets_and_order(capi, gpu, orc, synth):
    """n = 1 and 2, subsets and permutations of the same handles, and a handle used by dmv_ct_trace_many, then dmv_ct_trace_points_multi,
    then dmv_ct_trace_many again"""
    base = [window_member(synth, orc, f"w{i}", 60 + i, c) for i, c in enumerate([[200, 31], [5], [0, 64], [129, 0, 3]])]
    gs, twins = handles(capi, synth, base), handles(capi, synth, base)
    calls = [[0], [2, 1], [3, 2, 1, 0], [1, 3], [0, 1, 2, 3]]
    for c, idx in enumerate(calls):
        t = c % 3
        sub = [base[i] for i in idx]   # the handles left out keep their frame and state
        step(capi, orc, sub, [gs[i] for i in idx], [twins[i] for i in idx], t)
        if c == 2:   # a single-handle call on a member between two batched calls
            m = base[1]
            job = m.job(t)
            a, b = gs[1].trace_points_multi(job), twins[1].trace_points_multi(job)
            for Q, S_ in zip(a, b):
                for key in H_KEYS:
                    assert np.array_equal(bits(Q[key]), bits(S_[key])), key
            m.state = a
    close(*gs, *twins)


@pytest.mark.gpu
def test_track_after_trace(capi, gpu, orc, synth):
    """dmv_ct_track on a member after the call equals its twin's: the trace leaves the tracker's state as dmv_ct_trace_points_multi does"""
    import dmvio_b200.hostmath as hm
    sc = H.ct_scene(orc, synth, "bench")
    w, h = sc["w"], sc["h"]
    W = synth.make_window(nf=3, npts=10, seed=8, trans=0.05, rot=0.01, w=w, h=h)
    rng = np.random.default_rng(8)

    def tracker():
        g = capi.CT(w, h, sc["levels"], max_points=65536)
        for l in range(sc["levels"]):
            g.set_K(l, *[float(x) for x in sc["k4"][l]])
            p = sc["pts"][l]
            g.set_ref(l, p["u"], p["v"], p["idepth"], p["color"])
            g.upload_new(l, sc["planes"][l])
        return g

    u, v = rng.integers(10, w - 10, 900), rng.integers(10, h - 10, 900)
    m = Member("bench", w, h, [sc["planes"][0]], [orc.ip_init(W["dI"][0], w, h, u, v)], [0], lambda hst, f: hm.trace_tables(W, 0, 2), (0,))
    other = window_member(synth, orc, "other", 9, [300])
    gs = [tracker(), capi.CT(640, 480, 5, max_points=1024)]
    twins = [tracker(), capi.CT(640, 480, 5, max_points=1024)]
    step(capi, orc, [m, other], gs, twins, 0, upload=lambda mm, x, f: x.upload_new(0, mm.frames[f]) if mm is other else None)
    a = dict(sc["args"])
    kw = dict(R=a["R0"], t=a["t0"], a=a["a0"], b=a["b0"], ref_a=a["ref_a"], ref_b=a["ref_b"], ref_exposure=a["ref_exposure"],
              new_exposure=a["new_exposure"], affA=a["affA"], affB=a["affB"], coarsest=a.get("coarsest"), minRes=a.get("minRes"))
    r, s_ = gs[0].track(**kw), twins[0].track(**kw)
    for k in r:
        assert np.array_equal(G.bits(r[k]), G.bits(s_[k])), k
    assert r["status"] == 0
    close(*gs, *twins)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["null", "defaults", "custom"])
def test_settings(capi, gpu, orc, synth, which):
    """one dmv_ip_settings for the whole call: NULL, the struct dmv_ip_default_settings fills, and non-default values, each against twins
    traced with the same settings (the oracle traces with the defaults)"""
    S = None
    if which != "null":
        S = capi.ip_default_settings()
    if which == "custom":
        S.trace_GNIterations, S.minTraceTestRadius = 1, 3
    ms = [ip_case_member("statuses", *H.ip_status_case(synth, orc, n=1500)), window_member(synth, orc, "640x480", 5, [400, 0, 333])]
    gs, twins = handles(capi, synth, ms), handles(capi, synth, ms)
    for t in range(3):
        step(capi, orc, ms, gs, twins, t, settings=S, oracle=which != "custom")
    close(*gs, *twins)


@pytest.mark.gpu
def test_ordered_behind_asynchronous_uploads(capi, gpu, orc, synth):
    """each member's frame arrives by dmv_ct_upload_new_image or dmv_ct_upload_raw_image immediately before the call, with no
    synchronisation in between: the launch must wait for every member's upload"""
    ms = [window_member(synth, orc, f"w{i}", 70 + i, c) for i, c in enumerate([[800, 300], [1], [0], [513, 2, 0, 77]])]
    ms.append(window_member(synth, orc, "512", 75, [600], w=512, h=512))
    raw = {id(ms[1]), id(ms[3])}

    def upload(m, x, f):
        if id(m) in raw:
            x.upload_raw_image(np.clip(np.round(m.images[f]), 0, 255).astype(np.uint8))
        else:
            x.upload_new_image(m.images[f])

    gs, twins = handles(capi, synth, ms), handles(capi, synth, ms)
    for m, x in zip(ms + ms, gs + twins):
        if id(m) in raw:
            x.set_undistort(m.w, m.h)
    for t in range(3):
        step(capi, orc, ms, gs, twins, t, oracle=False, upload=upload)
    close(*gs, *twins)


@pytest.mark.gpu
def test_all_empty_call_launches_nothing(capi, gpu, orc, synth):
    ms = [empty_member(synth, orc, "a", 1), window_member(synth, orc, "b", 2, [0, 0, 0])]
    gs = handles(capi, synth, ms)
    before = [g.launch_count() for g in gs]
    got = capi.ct_trace_many(gs, [m.job(0) for m in ms])
    assert [len(r) for r in got] == [0, 3] and all(len(Q["status"]) == 0 for Q in got[1])
    assert [g.launch_count() for g in gs] == before
    close(*gs)


def sentinel_jobs(capi, ms):
    """the members' jobs marshalled for the raw symbol, every output pre-filled with a sentinel"""
    T = [capi._TraceSets(m.job(0)) for m in ms]
    for t in T:
        for out in t.outs:
            for k, a in out.items():
                a[...] = -7 if a.dtype == np.int32 else 12345.0
    return T


def untouched(T):
    return all((a == (-7 if a.dtype == np.int32 else 12345.0)).all() for t in T for out in t.outs for a in out.values())


def raw_call(capi, hs, T, n=None):
    n = len(hs) if n is None else n
    m = max(len(hs), 1)
    H_ = (C.c_void_p * m)(*[None if g is None else g.h.value for g in hs])
    J = (capi.TraceJob * m)(*[t.job for t in T])
    rc = capi.lib().dmv_ct_trace_many(H_, n, J, None)
    return rc, capi.lib().dmv_last_error().decode()


@pytest.mark.gpu
def test_errors_are_rejected_before_anything(capi, gpu, orc, synth):
    ms = [window_member(synth, orc, f"w{i}", 80 + i, [5 + i, 3]) for i in range(MANY_MAX + 1)]
    gs = handles(capi, synth, ms)
    for m, g in zip(ms, gs):
        g.upload_new(0, m.frames[m.seq[0]])
    counts = [g.launch_count() for g in gs]

    def rejected(hs, T, msg, n=None):
        rc, text = raw_call(capi, hs, T, n)
        assert rc == DMV_ERR_INVALID, (rc, text)
        assert msg in text, text
        assert untouched(T)
        assert [g.launch_count() for g in gs] == counts
        return text

    T = sentinel_jobs(capi, ms)
    rejected(gs[:1], T[:1], "n = 0", n=0)
    rejected(gs, T, "n = 17")
    rejected([gs[0], None, gs[2]], T[:3], "handles[1] is NULL")
    rejected([gs[0], gs[1], gs[0]], T[:3], "handles[0] and handles[2]")
    # an incomplete set in member 3: its message names the member and the set
    T = sentinel_jobs(capi, ms[:5])
    T[3].arr[1].color8 = None
    text = rejected(gs[:5], T, "handles[3]: ")
    assert "incomplete dmv_ip_points (set 1)" in text
    # more than 64 host frames in member 2
    big = window_member(synth, orc, "65", 99, [1] * 65, nhost=3)
    T = sentinel_jobs(capi, ms[:2] + [big] + ms[3:4])
    text = rejected(gs[:4], T, "handles[2]: ")
    assert "at most 64 host frames" in text
    # a NULL sets pointer with nsets > 0 in member 1
    T = sentinel_jobs(capi, ms[:3])
    T[1].job.sets = None
    rejected(gs[:3], T, "handles[1]: null argument")
    # the accepted call after the refusals: every member traced, each launch count + 1
    T = sentinel_jobs(capi, ms[:MANY_MAX])
    rc, text = raw_call(capi, gs[:MANY_MAX], T)
    assert rc == 0, text
    assert [g.launch_count() - c for g, c in zip(gs, counts)] == [1] * MANY_MAX + [0]
    assert not untouched(T)
    close(*gs)


@pytest.mark.gpu
def test_handles_on_two_devices_are_rejected(capi, gpu, orc, synth):
    if capi.lib().dmv_device_count() < 2:
        pytest.skip("needs two visible GPUs")
    m = window_member(synth, orc, "w", 3, [10])
    g0, g1 = capi.CT(640, 480, 5, max_points=1024, device=0), capi.CT(640, 480, 5, max_points=1024, device=1)
    T = sentinel_jobs(capi, [m, m])
    rc, text = raw_call(capi, [g0, g1], T)
    assert rc == DMV_ERR_INVALID and "device" in text and untouched(T)
    assert g0.launch_count() == g1.launch_count() == 0
    close(g0, g1)


def test_arguments_without_handles_are_rejected(capi):
    """the checks that need no handle and no device"""
    L = capi.lib()
    J = (capi.TraceJob * 1)()
    hs = (C.c_void_p * 1)(None)
    assert L.dmv_ct_trace_many(None, 1, J, None) == DMV_ERR_INVALID
    assert L.dmv_ct_trace_many(hs, 1, None, None) == DMV_ERR_INVALID
    assert L.dmv_ct_trace_many(hs, 0, J, None) == DMV_ERR_INVALID
    assert b"n = 0" in L.dmv_last_error()
    assert L.dmv_ct_trace_many(hs, 17, J, None) == DMV_ERR_INVALID
    assert b"n = 17" in L.dmv_last_error()
    assert L.dmv_ct_trace_many(hs, 1, J, None) == DMV_ERR_INVALID
    assert b"handles[0] is NULL" in L.dmv_last_error()
    with pytest.raises(capi.DmvError, match="n = 0"):
        capi.ct_trace_many([], [])
    with pytest.raises(ValueError):
        capi.ct_trace_many([], [[]])

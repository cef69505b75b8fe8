"""The immature-point store (dmv_ip_store_*, dmv_ct_trace_store, dmv_ct_trace_store_many) against a twin on host arrays.

Every store has a twin: one list of host arrays per slot, traced with dmv_ct_trace_points_multi (or dmv_ct_trace_many) on a twin handle
that sees the same frames, with sets[k] = slot k and the same tables.  Whenever a slot is read back (dmv_ip_store_get) its in/out fields
must equal the twin's bit for bit, NaN payloads included, and each handle's launch count must move as its twin's does.  The keyframe
turnover edits the twin the way activatePointsMT edits host->immaturePoints (FullSystem.cpp:L761-769), restated here in numpy."""
import ctypes as C

import numpy as np
import pytest

import gpu_harness as G
from dmvio_b200.capi import DMV_ERR_INVALID
from gpu_harness import capi, close, gpu  # noqa: F401

KEYS = ("idepth_min", "idepth_max", "quality", "status", "lastTraceUV", "lastTracePixelInterval")


def bits(a):
    return np.ascontiguousarray(a).reshape(-1).view(np.uint32)


def empty_points():
    z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
    return dict(u=z(0), v=z(0), color=z(0, 8), weights=z(0, 8), gradH=z(0, 4), energyTH=z(0), idepth_min=z(0), idepth_max=z(0), quality=z(0),
                status=np.zeros(0, np.int32), lastTraceUV=z(0, 2), lastTracePixelInterval=z(0))


def swap_with_back(n, idx):
    """activatePointsMT's loop over host->immaturePoints (FullSystem.cpp:L761-769) on indices: the survivors' old indices in their new order"""
    gone = set(int(i) for i in idx)
    lst = list(range(n))
    i = 0
    while i < len(lst):
        if lst[i] in gone:
            lst[i] = lst[-1]
            lst.pop()
            i -= 1
        i += 1
    return np.array(lst, np.int32)


class Scene:
    """a synth.make_window scene: host frames 0 .. nhost - 1, new frames after them; points(host, n, seed) = fresh immature points"""

    def __init__(self, synth, orc, seed, w=640, h=480, nhost=6, nnew=3):
        import dmvio_b200.hostmath as hm
        self.w, self.h, self.nhost, self.orc, self.hm = w, h, nhost, orc, hm
        self.levels = synth.pyr_levels(w, h)
        self.W = synth.make_window(nf=nhost + nnew, npts=10, seed=seed, trans=0.05, rot=0.01, w=w, h=h)
        self.rng = np.random.default_rng(seed)
        self.new = list(range(nhost, nhost + nnew))

    def points(self, host, n):
        u, v = self.rng.integers(10, self.w - 10, n), self.rng.integers(10, self.h - 10, n)
        return self.orc.ip_init(self.W["dI"][host], self.w, self.h, u, v)

    def frame(self, t):
        return self.W["dI"][self.new[t % len(self.new)]]

    def image(self, t):
        return self.W["images"][self.new[t % len(self.new)]]

    def tables(self, hosts, t):
        """(KRKi, Kt, aff) of every slot's host against frame t; None for a slot without a host"""
        f = self.new[t % len(self.new)]
        return [None if hst is None else tuple(self.hm.trace_tables(self.W, hst, f)) for hst in hosts]


class Twin:
    """a store and its host-array twin: slot k holds sets[k] hosted by hosts[k]"""

    def __init__(self, capi, sc, store):
        self.capi, self.sc, self.store = capi, sc, store
        self.sets, self.hosts = [], []

    def nslots(self):
        return len(self.sets)

    def npoints(self):
        return sum(len(P["u"]) for P in self.sets)

    def put(self, slot, P, host):
        while len(self.sets) <= slot:
            self.sets.append(empty_points()); self.hosts.append(None)
        self.store.put(slot, P)
        self.sets[slot], self.hosts[slot] = dict(P), (host if len(P["u"]) else None)
        self.trim()

    def trim(self):
        while self.sets and len(self.sets[-1]["u"]) == 0:   # nslots covers the last slot with points
            self.sets.pop(); self.hosts.pop()

    def remove(self, slot, idx):
        n = len(self.sets[slot]["u"])
        order = self.store.remove(slot, idx)
        ref = swap_with_back(n, idx)
        assert np.array_equal(order, ref), (slot, order[:10], ref[:10])
        self.sets[slot] = {k: a[ref] for k, a in self.sets[slot].items()}
        if len(ref) == 0:
            self.hosts[slot] = None
        self.trim()
        return order

    def job(self, t):
        """the store's tables at frame t and the twin's sets for dmv_ct_trace_points_multi"""
        tabs = self.sc.tables(self.hosts, t)
        return tabs, [(P,) + (tb if tb is not None else (np.zeros(9), np.zeros(3), np.zeros(2))) for P, tb in zip(self.sets, tabs)]

    def absorb(self, res):
        self.sets = [dict(P, **{k: Q[k] for k in KEYS}) for P, Q in zip(self.sets, res)]

    def check(self, what):
        for k, P in enumerate(self.sets):
            Q = self.store.get(k)
            for key in KEYS:
                assert np.array_equal(bits(Q[key]), bits(P[key])), f"{what} slot {k}: {key} differs from dmv_ct_trace_points_multi"
        for k in range(len(self.sets), self.store.SLOTS):
            assert self.store.counts[k] == 0


def handle(capi, sc):
    return capi.CT(sc.w, sc.h, sc.levels, max_points=1024)


def trace_step(tw, g, twin_g, t):
    """frame t into g and twin_g, dmv_ct_trace_store on g against dmv_ct_trace_points_multi on twin_g"""
    for x in (g, twin_g):
        x.upload_new(0, tw.sc.frame(t))
    tabs, sets = tw.job(t)
    b, tb = g.launch_count(), twin_g.launch_count()
    g.trace_store(tw.store, tabs)
    res = twin_g.trace_points_multi(sets)
    assert twin_g.launch_count() - tb == int(tw.npoints() > 0)
    assert g.launch_count() - b == twin_g.launch_count() - tb, "launch count"
    tw.absorb(res)


def filled(capi, sc, counts):
    st = capi.IPStore()
    tw = Twin(capi, sc, st)
    for k, n in enumerate(counts):
        tw.put(k, sc.points(k % sc.nhost, n) if n else empty_points(), k % sc.nhost)
    return tw


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(640, 480), (512, 512)])
def test_frame_sequence(capi, gpu, orc, synth, shape):
    """9 frames over 6 slots x 1500 points, read back after frames 0, 3, 4 and 8"""
    sc = Scene(synth, orc, 11 + shape[0], *shape)
    tw = filled(capi, sc, [1500] * 6)
    g, twin_g = handle(capi, sc), handle(capi, sc)
    seen = np.zeros(6, int)
    for t in range(9):
        trace_step(tw, g, twin_g, t)
        if t in (0, 3, 4, 8):
            tw.check(f"frame {t}")
        for P in tw.sets:
            seen += np.bincount(P["status"], minlength=6)
    assert (seen[:3] > 0).all(), seen
    close(g, twin_g, tw.store)


@pytest.mark.gpu
def test_keyframe_turnovers(capi, gpu, orc, synth):
    """removals of the first point, the last, runs, all points and none, one whose back replacement is removed too (the i-- re-check);
    puts into a new slot and past an empty one, a marginalised slot emptied, and the store grown past its first capacity with every slot
    intact; frames traced between the edits"""
    sc = Scene(synth, orc, 21)
    tw = filled(capi, sc, [60])
    g, twin_g = handle(capi, sc), handle(capi, sc)
    t = 0

    def frames(k):
        nonlocal t
        for _ in range(k):
            trace_step(tw, g, twin_g, t)
            t += 1

    frames(2)
    tw.check("one small slot")
    for k in range(1, 6):   # the store grows several times, the traced slot 0 is copied along
        tw.put(k, sc.points(k, 1500), k)
    tw.check("after growing")
    frames(2)
    tw.check("six slots")
    n = [len(P["u"]) for P in tw.sets]
    tw.remove(0, [0])                                       # the first point
    tw.remove(1, [n[1] - 1])                                # the last
    tw.remove(2, list(range(10, 40)) + list(range(100, 120)) + list(range(n[2] - 25, n[2])))   # runs, one at the back
    assert len(tw.remove(3, [])) == n[3]                    # none
    tw.remove(5, [5, n[5] - 1, n[5] - 2, 7, n[5] - 3])      # the back replacements of 5 and 7 are removed too: i-- re-checks them
    tw.check("after removals")
    frames(2)
    tw.remove(4, np.random.default_rng(4).permutation(n[4]))   # all, in a random order
    tw.put(7, sc.points(0, 900), 0)                         # a new keyframe's points in slot 7: slots 4 and 6 are empty below it
    tw.check("slot 4 emptied, slot 7 put")
    frames(1)
    tw.put(1, empty_points(), None)                         # the marginalised keyframe
    tw.put(6, sc.points(3, 1), 3)
    frames(2)
    tw.check("after the second turnover")
    tw.put(0, sc.points(2, 4000), 2)                        # replace slot 0 by more points than the store held in all
    rng = np.random.default_rng(9)
    for k, P in enumerate(tw.sets):
        if len(P["u"]):
            tw.remove(k, rng.choice(len(P["u"]), len(P["u"]) // 3, replace=False))
    frames(1)
    tw.check("after the third turnover")
    for k, P in enumerate(list(tw.sets)):   # everything removed: the next frames launch nothing
        if len(P["u"]):
            tw.remove(k, np.arange(len(P["u"])))
    assert tw.nslots() == 0
    b = g.launch_count()
    g.trace_store(tw.store, [])
    assert g.launch_count() == b
    frames(1)
    tw.put(2, sc.points(1, 700), 1)
    frames(2)
    tw.check("refilled")
    close(g, twin_g, tw.store)


@pytest.mark.gpu
def test_two_handles_alternate(capi, gpu, orc, synth):
    """one store traced by two tracker handles in turn, as FullSystem's coarse trackers swap at every keyframe, with a dmv_ct_track on
    the other handle between the traces; afterwards each handle's own dmv_ct_trace_points_multi still matches its twin"""
    sc_t = G.ct_scene(orc, synth, "bench")
    sc = Scene(synth, orc, 31, sc_t["w"], sc_t["h"])
    tw = filled(capi, sc, [1500, 0, 700, 1500, 3])
    gs = [G.ct_handle(capi, sc_t), G.ct_handle(capi, sc_t)]
    twins = [G.ct_handle(capi, sc_t), G.ct_handle(capi, sc_t)]
    kw = G.track_kw(sc_t)
    for t in range(6):
        a = t % 2
        trace_step(tw, gs[a], twins[a], t)
        r, s_ = gs[1 - a].track(**kw), twins[1 - a].track(**kw)
        G.assert_same(r, s_, f"track after trace {t}")
        if t in (1, 5):
            tw.check(f"frame {t}")
    sets = [(sc.points(0, 300),) + sc.tables([0], 0)[0]]
    for g, x in zip(gs, twins):
        A, B = g.trace_points_multi(sets), x.trace_points_multi(sets)
        for key in KEYS:
            assert np.array_equal(bits(A[0][key]), bits(B[0][key])), key
    close(*gs, *twins, tw.store)


@pytest.mark.gpu
def test_many_ordered_behind_uploads(capi, gpu, orc, synth):
    """dmv_ct_trace_store_many over five handles whose frames arrive by dmv_ct_upload_new_image or dmv_ct_upload_raw_image immediately
    before the call, with no synchronisation in between: the arguments are marshalled first, the twins' frames go in first, and the call
    follows the members' uploads at once.  The last upload is member 1's 2560x1920 16-bit raw frame, remapped to 640x480, so its copy is
    still in flight when the call launches, and member 0 has one point, so member 1's points are among the kernel's first.  Against
    dmv_ct_trace_many on the twins."""
    L = capi.lib()
    shapes = [(640, 480), (640, 480), (512, 512), (640, 480), (512, 512)]
    scs = [Scene(synth, orc, 41 + i, w, h) for i, (w, h) in enumerate(shapes)]
    tws = [filled(capi, sc, c) for sc, c in zip(scs, [[1], [1500] * 6, [800, 0, 300], [2601, 5], [1500] * 3])]
    raw = {1: 4, 3: 1}   # member: raw pixels per pixel of the frame, each way
    gs, twins = [handle(capi, sc) for sc in scs], [handle(capi, sc) for sc in scs]
    for i, f in raw.items():
        w, h = scs[i].w, scs[i].h
        X, Y = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
        for x in (gs[i], twins[i]):
            if f == 1:
                x.set_undistort(w, h)
            else:
                x.set_undistort(w * f, h * f, f * X + 1.5, f * Y + 1.5)
    n = len(gs)
    H_ = (C.c_void_p * n)(*[g.h.value for g in gs])
    for t in range(6):
        frames = []
        for i, sc in enumerate(scs):
            img = np.clip(np.round(sc.image(t)), 0, 255)
            if i not in raw:
                frames.append(np.ascontiguousarray(sc.image(t), np.float32))
            elif raw[i] == 1:
                frames.append(img.astype(np.uint8))
            else:
                frames.append((np.kron(img, np.ones((raw[i], raw[i]))) * 256).astype(np.uint16))
        upload = lambda y, i: y.upload_raw_image(frames[i]) if i in raw else y.upload_new_image(frames[i])  # noqa: E731
        jobs = [tw.job(t) for tw in tws]
        tabs = [capi._tables14(tb) for tb, _ in jobs]
        J = (capi.TraceStoreJob * n)(*[capi.TraceStoreJob(tw.store.h.value, len(tb), tb.ctypes.data if len(tb) else None) for tw, tb in zip(tws, tabs)])
        b, bt = [g.launch_count() for g in gs], [x.launch_count() for x in twins]
        for i, x in enumerate(twins):
            upload(x, i)
        for i in (0, 2, 3, 4, 1):
            upload(gs[i], i)
        assert L.dmv_ct_trace_store_many(H_, n, J, None) == 0, L.dmv_last_error()
        res = capi.ct_trace_many(twins, [sets for _, sets in jobs])
        for tw, g, x, r, b0, bt0 in zip(tws, gs, twins, res, b, bt):
            assert g.launch_count() - b0 == x.launch_count() - bt0
            tw.absorb(r)
        for tw in tws:
            tw.check(f"frame {t}")
    close(*gs, *twins, *[tw.store for tw in tws])


def many_step(capi, tws, gs, twins, t, settings=None):
    jobs = [tw.job(t) for tw in tws]
    b = [g.launch_count() for g in gs]
    bt = [x.launch_count() for x in twins]
    capi.trace_store_many(gs, [(tw.store, tabs) for tw, (tabs, _) in zip(tws, jobs)], settings)
    res = capi.ct_trace_many(twins, [sets for _, sets in jobs], settings)
    for tw, g, x, r, b0, bt0 in zip(tws, gs, twins, res, b, bt):
        assert x.launch_count() - bt0 == int(tw.npoints() > 0)
        assert g.launch_count() - b0 == x.launch_count() - bt0
        tw.absorb(r)


@pytest.mark.gpu
def test_many_sixteen_members(capi, gpu, orc, synth):
    """16 members of 0, 1, 3, 33, 401 and 2601 points at their own image sizes, traced in subsets and permutations, with custom settings on
    one frame, against dmv_ct_trace_many on twins"""
    specs = [[0], [1], [3], [33], [401], [2601], [0, 0, 1], [0, 33], [401, 0, 3], [1, 1, 1], [2601], [33], [3, 0, 0, 0, 401], [], [0, 1], [401]]
    shapes = [(640, 480), (512, 512), (320, 240)]
    scs = [Scene(synth, orc, 60 + i, *shapes[i % 3], nhost=3) for i in range(16)]
    tws = [filled(capi, sc, c) for sc, c in zip(scs, specs)]
    for tw in tws:
        tw.trim()
    gs, twins = [handle(capi, sc) for sc in scs], [handle(capi, sc) for sc in scs]
    S = capi.ip_default_settings()
    S.trace_GNIterations, S.minTraceTestRadius = 1, 3
    calls = [list(range(16)), [15, 3, 7, 0], list(range(15, -1, -1)), [5], [2, 9, 5, 11, 1, 0, 14, 13]]
    for c, idx in enumerate(calls):
        for i in idx:
            for y in (gs[i], twins[i]):
                y.upload_new(0, scs[i].frame(c))
        many_step(capi, [tws[i] for i in idx], [gs[i] for i in idx], [twins[i] for i in idx], c, S if c == 1 else None)
        for i in idx:
            tws[i].check(f"call {c} member {i}")
    close(*gs, *twins, *[tw.store for tw in tws])


@pytest.mark.gpu
def test_all_empty_call_launches_nothing(capi, gpu, orc, synth):
    sc = Scene(synth, orc, 3, nhost=2)
    tws = [filled(capi, sc, []), filled(capi, sc, [0, 0])]
    gs = [handle(capi, sc), handle(capi, sc)]
    capi.trace_store_many(gs, [(tw.store, []) for tw in tws])
    gs[0].trace_store(tws[0].store, [])
    assert [g.launch_count() for g in gs] == [0, 0]
    close(*gs, *[tw.store for tw in tws])


# ---------------------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------------------
def snapshot(st):
    return [{k: bits(a).copy() for k, a in st.get(s).items()} for s in range(st.SLOTS) if st.counts[s]] + [list(st.counts)]


def same_snapshot(a, b):
    if a[-1] != b[-1]:
        return False
    return all(all(np.array_equal(x[k], y[k]) for k in KEYS) for x, y in zip(a[:-1], b[:-1]))


def sentinel_points(n):
    P = empty_points()
    P = {k: np.full((n,) + a.shape[1:], -7 if a.dtype == np.int32 else 12345.0, a.dtype) for k, a in P.items()}
    return P


def ip_points(capi, P, n=None):
    n = len(P["u"]) if n is None else n
    return capi.IPPoints(n, *[P[k].ctypes.data for k in ("u", "v", "color", "weights", "gradH", "energyTH", "idepth_min", "idepth_max", "quality", "status",
                                                          "lastTraceUV", "lastTracePixelInterval")])


@pytest.mark.gpu
def test_refusals_change_nothing(capi, gpu, orc, synth):
    """every refusal of the seven calls, each followed by a check that the stores' contents, every handle's launch count and the output
    sentinels are as they were"""
    L = capi.lib()
    scs = [Scene(synth, orc, 90 + i, nhost=3) for i in range(3)]
    tws = [filled(capi, sc, c) for sc, c in zip(scs, [[40, 0, 7], [5], [3, 3, 3]])]
    gs = [handle(capi, sc) for sc in scs] + [handle(capi, scs[0]) for _ in range(14)]
    for g, sc in zip(gs, scs + [scs[0]] * 14):
        g.upload_new(0, sc.frame(0))
    counts = [g.launch_count() for g in gs]
    snaps = [snapshot(tw.store) for tw in tws]
    st = tws[0].store
    out = sentinel_points(40)
    order = np.full(64, -7, np.int32)

    def refused(rc, msg):
        text = L.dmv_last_error().decode()
        assert rc == DMV_ERR_INVALID, (rc, text)
        assert msg in text, text
        assert [g.launch_count() for g in gs] == counts
        assert all(same_snapshot(snapshot(tw.store), s) for tw, s in zip(tws, snaps))
        assert (order == -7).all() and all((a == (-7 if a.dtype == np.int32 else 12345.0)).all() for a in out.values())
        return text

    P = scs[0].points(0, 10)
    full = ip_points(capi, P)
    # put
    refused(L.dmv_ip_store_put(st.h, -1, C.byref(full)), "slot -1")
    refused(L.dmv_ip_store_put(st.h, 64, C.byref(full)), "slot 64")
    refused(L.dmv_ip_store_put(st.h, 0, None), "null argument")
    bad = ip_points(capi, P); bad.gradH4 = None
    refused(L.dmv_ip_store_put(st.h, 0, C.byref(bad)), "incomplete dmv_ip_points")
    refused(L.dmv_ip_store_put(st.h, 0, C.byref(ip_points(capi, P, -1))), "incomplete dmv_ip_points")
    # get: the count, and the out pointers
    text = refused(L.dmv_ip_store_get(st.h, 0, C.byref(ip_points(capi, out, 39))), "slot 0 holds 40 points")
    bad = ip_points(capi, out); bad.lastTraceUV2 = None
    refused(L.dmv_ip_store_get(st.h, 0, C.byref(bad)), "incomplete dmv_ip_points")
    refused(L.dmv_ip_store_get(st.h, 65, C.byref(ip_points(capi, out))), "slot 65")
    # remove
    o = order.ctypes.data

    def rm(idx, n=None, slot=0):
        idx = np.asarray(idx, np.int32)
        return L.dmv_ip_store_remove(st.h, slot, len(idx) if n is None else n, idx.ctypes.data if len(idx) else None, o)

    refused(rm([0], n=-1), "null argument")
    refused(rm([], n=2), "null argument")
    refused(rm(list(range(41))), "n = 41: slot 0 holds 40 points")
    refused(rm([3, 40]), "idx[1] = 40")
    refused(rm([3, -1]), "idx[1] = -1")
    refused(rm([3, 9, 3]), "idx[2] = 3 appears twice")
    refused(rm([0], slot=1), "n = 1: slot 1 holds 0 points")
    refused(rm([0], slot=-3), "slot -3")
    # dmv_ct_trace_store
    tab = capi._tables14(scs[0].tables([0, 1, 2], 0))
    ts = lambda ns, t=tab, g=gs[0], s_=st: L.dmv_ct_trace_store(g.h, s_.h, ns, None if t is None else t.ctypes.data, None)  # noqa: E731
    refused(ts(-1), "nslots = -1")
    refused(ts(65), "nslots = 65")
    refused(ts(2), "slot 2 holds 7 points but nslots = 2")
    refused(ts(3, t=None), "null tables14 with 47 points")
    refused(L.dmv_ct_trace_store(gs[0].h, None, 3, tab.ctypes.data, None), "null argument")
    # dmv_ct_trace_store_many
    def many(hs, jobs, n=None):
        H_ = (C.c_void_p * max(len(hs), 1))(*[None if g is None else g.h.value for g in hs])
        J = (capi.TraceStoreJob * max(len(jobs), 1))(*[capi.TraceStoreJob(s_ and s_.h.value, ns, None if t is None else t.ctypes.data) for s_, ns, t in jobs])
        return L.dmv_ct_trace_store_many(H_, len(hs) if n is None else n, J, None)

    good = [(tw.store, 3, tab) for tw in tws]
    refused(many(gs[:3], good, n=0), "n = 0")
    refused(many(gs, good + [(None, 0, None)] * 14), "n = 17")
    refused(many([gs[0], None, gs[2]], good), "handles[1] is NULL")
    refused(many([gs[0], gs[1], gs[0]], good), "handles[0] and handles[2] are the same handle")
    refused(many(gs[:3], [good[0], good[1], good[0]]), "jobs[0] and jobs[2] name the same store")
    refused(many(gs[:3], [good[0], (None, 0, None), good[2]]), "handles[1]: null argument")
    refused(many(gs[:3], [good[0], good[1], (tws[2].store, 2, tab)]), "handles[2]: slot 2 holds 3 points but nslots = 2")
    refused(many(gs[:3], [good[0], (tws[1].store, 65, tab), good[2]]), "handles[1]: nslots = 65")
    refused(many(gs[:3], [(st, 3, None), good[1], good[2]]), "handles[0]: null tables14")
    refused(L.dmv_ct_trace_store_many(None, 1, (capi.TraceStoreJob * 1)(), None), "null argument")
    # the accepted calls after the refusals: each member traced once
    assert many(gs[:3], good) == 0, L.dmv_last_error()
    assert [g.launch_count() - c for g, c in zip(gs, counts)] == [1, 1, 1] + [0] * 14
    assert not same_snapshot(snapshot(st), snaps[0])
    close(*gs, *[tw.store for tw in tws])


@pytest.mark.gpu
def test_store_on_another_device_is_refused(capi, gpu, orc, synth):
    if capi.lib().dmv_device_count() < 2:
        pytest.skip("needs two visible GPUs")
    sc = Scene(synth, orc, 5, nhost=1)
    st = capi.IPStore(device=1)
    st.put(0, sc.points(0, 10))
    g = capi.CT(640, 480, 5, max_points=1024, device=0)
    with pytest.raises(capi.DmvError, match="the store is on device 1, the handle on device 0"):
        g.trace_store(st, sc.tables([0], 0))
    assert g.launch_count() == 0
    close(g, st)


def test_arguments_without_a_store_are_rejected(capi):
    """the checks that need no store, no handle and no device"""
    L = capi.lib()
    P = capi.IPPoints()
    idx = np.zeros(1, np.int32)
    assert L.dmv_ip_store_create(0, None) == DMV_ERR_INVALID
    assert L.dmv_ip_store_destroy(None) == 0
    assert L.dmv_ip_store_put(None, 0, C.byref(P)) == DMV_ERR_INVALID
    assert L.dmv_ip_store_get(None, 0, C.byref(P)) == DMV_ERR_INVALID
    assert L.dmv_ip_store_remove(None, 0, 1, idx.ctypes.data, None) == DMV_ERR_INVALID
    assert L.dmv_ct_trace_store(None, None, 0, None, None) == DMV_ERR_INVALID
    assert b"null argument" in L.dmv_last_error()
    J = (capi.TraceStoreJob * 1)()
    hs = (C.c_void_p * 1)(None)
    assert L.dmv_ct_trace_store_many(None, 1, J, None) == DMV_ERR_INVALID
    assert L.dmv_ct_trace_store_many(hs, 1, None, None) == DMV_ERR_INVALID
    assert L.dmv_ct_trace_store_many(hs, 0, J, None) == DMV_ERR_INVALID
    assert b"n = 0" in L.dmv_last_error()
    assert L.dmv_ct_trace_store_many(hs, 17, J, None) == DMV_ERR_INVALID
    assert b"n = 17" in L.dmv_last_error()
    assert L.dmv_ct_trace_store_many(hs, 1, J, None) == DMV_ERR_INVALID
    assert b"handles[0] is NULL" in L.dmv_last_error()
    assert np.array_equal(swap_with_back(6, [1, 5, 4]), [0, 3, 2])   # 1 <- 5 removed too, re-checked: 1 <- 4 removed, 1 <- 3

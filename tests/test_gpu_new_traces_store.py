"""dmv_ct_make_new_traces_store against a twin: a second tracker handle and a second store that see the same frames and run the pair the
call replaces, dmv_ct_make_new_traces then dmv_ip_store_put of its points with the ImmaturePoint constructor's in/out values.  Every
comparison is bit for bit, NaN payloads included: each slot's dmv_ip_store_get, the per-point outputs, potential, numPointsTotal, n, map,
the launch counts, and every trace and activation of the two stores afterwards."""
import ctypes as C

import numpy as np
import pytest

import dmvio_b200.hostmath as hm
from dmvio_b200.capi import DMV_ERR_INVALID, IP_OUT_KEYS
from gpu_harness import capi, close, gpu  # noqa: F401
from oracle import select as S
from test_gpu_activate_store import Win
from test_gpu_trace_store import bits

ALL = ("u", "v", "type", "color", "weights", "gradH", "energyTH")


def as_put(P):
    """make_new_traces' points as dmv_ip_store_put takes them: u, v as float, the constructor's in/out values (capi.CT.init_points')"""
    n = len(P["u"])
    return dict(u=P["u"].astype(np.float32), v=P["v"].astype(np.float32), color=P["color"], weights=P["weights"], gradH=P["gradH"],
                energyTH=P["energyTH"], idepth_min=np.zeros(n, np.float32), idepth_max=np.full(n, np.nan, np.float32),
                quality=np.full(n, 10000, np.float32), status=np.full(n, 5, np.int32), lastTraceUV=np.zeros((n, 2), np.float32),
                lastTracePixelInterval=np.zeros(n, np.float32))


def same_stores(a, b, what):
    assert a.counts == b.counts, what
    for k in range(a.SLOTS):
        if a.counts[k]:
            P, Q = a.get(k), b.get(k)
            for key in IP_OUT_KEYS:
                assert np.array_equal(bits(P[key]), bits(Q[key])), f"{what}: slot {k} {key}"


def snapshot(st):
    return list(st.counts), {k: st.get(k) for k in range(st.SLOTS) if st.counts[k]}


def unchanged(st, snap):
    counts, got = snap
    if st.counts != counts:
        return False
    return all(np.array_equal(bits(P[key]), bits(st.get(k)[key])) for k, P in got.items() for key in IP_OUT_KEYS)


class Pair:
    """handles g[i] with store st (the call) and their twins t[i] with store ts (make_new_traces + put); one potential for all, as
    FullSystem's one PixelSelector"""

    def __init__(self, capi, w, h, lv, handles=1, stores=None):
        self.g = [capi.CT(w, h, lv) for _ in range(handles)]
        self.t = [capi.CT(w, h, lv) for _ in range(handles)]
        self.st, self.ts = stores or (capi.IPStore(), capi.IPStore())
        self.pot = 3

    def close(self):
        close(*self.g, *self.t, self.st, self.ts)

    def upload(self, img, i=0):
        for x in (self.g[i], self.t[i]):
            x.upload_new_image(img)

    def keyframe(self, slot, want=("type",), i=0, what="", cap=16384, **kw):
        """the resident frame of handle i into slot `slot` of both stores; returns (the call's result, the twin's make_new_traces result)"""
        g, t = self.g[i], self.t[i]
        b, bt = g.launch_count(), t.launch_count()
        r = g.make_new_traces_store(self.st, slot, self.pot, want=want, cap=cap, want_map=True, **kw)
        o = t.make_new_traces(self.pot, want_map=True, **kw)
        self.ts.put(slot, as_put(o["points"]))
        assert g.launch_count() - b == t.launch_count() - bt, what
        assert (r["potential"], r["numPointsTotal"], r["n"]) == (o["potential"], o["numPointsTotal"], len(o["points"]["u"])), what
        assert np.array_equal(bits(r["map"]), bits(o["map"])), what
        assert sorted(r["points"]) == sorted(want), what
        for k in want:
            a, c = r["points"][k], o["points"][k]
            assert a.shape == c.shape and a.dtype == c.dtype and np.array_equal(bits(a), bits(c)), f"{what}: {k}"
        self.pot = r["potential"]
        same_stores(self.st, self.ts, what)
        return r, o


def oracle(img, w, h, lv, pot):
    from oracle import orc
    return S.restate(orc.make_images(img, S.K_of(w, h), lv)[:3], potential=pot)


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(640, 480, 5), (512, 512, 4)])
def test_shapes_and_keyframes(capi, gpu, orc, shape):
    """four seeded keyframes into four slots, every per-point output requested once, type alone otherwise; 640x480 also against the
    oracle restatement"""
    w, h, lv = shape
    p = Pair(capi, w, h, lv)
    for j, (kind, slot) in enumerate((("tex", 2), ("high", 0), ("low", 5), ("tex", 1))):
        img = S.image(kind, w, h, 40 + j)
        p.upload(img)
        pot = p.pot
        r, _ = p.keyframe(slot, want=ALL if j == 0 else ("type",), what=f"keyframe {j}")
        assert r["n"] > 0
        if j == 0 and w == 640:
            o = oracle(img, w, h, lv, pot)
            assert np.array_equal(r["map"], o["map"])
            assert (r["potential"], r["numPointsTotal"]) == (o["potential"], o["numPointsTotal"])
            for k in ALL:
                assert np.array_equal(bits(r["points"][k]), bits(np.ascontiguousarray(o["points"][k], r["points"][k].dtype))), k
    p.close()


@pytest.mark.gpu
def test_slot_placement(capi, gpu, orc):
    """slots filled out of order (63 past empty slots, then 0), an occupied slot replaced, the store grown past its first capacity with
    the points already in it unchanged, and a frame without points emptying its slot"""
    w, h, lv = 640, 480, 5
    p = Pair(capi, w, h, lv)
    p.upload(S.image("tex", w, h, 60))
    p.keyframe(5, what="slot 5")
    p.upload(S.image("high", w, h, 61))
    p.keyframe(63, what="slot 63 past empty slots")
    keep = p.st.get(63)
    p.upload(S.image("tex", w, h, 62))
    p.keyframe(0, want=ALL, what="slot 0 in front")
    p.upload(S.image("stripe", w, h, 63))
    p.keyframe(5, what="slot 5 replaced")
    first = sum(p.st.counts)
    for j, slot in enumerate((7, 8, 9, 30, 31, 40)):   # both buffers grow: a buffer holds at most 1.5x the points it last grew for
        p.upload(S.image("tex", w, h, 70 + j))
        p.keyframe(slot, what=f"growing: slot {slot}")
    assert sum(p.st.counts) > first + first // 2
    Q = p.st.get(63)
    assert all(np.array_equal(bits(keep[k]), bits(Q[k])) for k in IP_OUT_KEYS)
    p.upload(S.image("flat", w, h, 0))
    r, _ = p.keyframe(8, want=ALL, what="no points")
    assert r["n"] == 0 and p.st.counts[8] == 0
    p.keyframe(11, what="no points into an empty slot")
    assert p.st.counts[11] == 0
    p.close()


@pytest.mark.gpu
def test_tracing_afterwards(capi, gpu, orc, synth):
    """six keyframes of a synthetic sequence in slots that do not follow frame order, traced over three later frames with a different
    table row per slot"""
    w, h = 640, 480
    W = synth.make_window(nf=9, npts=10, seed=17, trans=0.05, rot=0.01, w=w, h=h)
    p = Pair(capi, w, h, synth.pyr_levels(w, h))
    host = {}
    for f, slot in enumerate((4, 0, 9, 2, 7, 1)):
        p.upload(W["images"][f])
        p.keyframe(slot, what=f"keyframe {f}")
        host[slot] = f
    ns = max(host) + 1
    for t in (6, 7, 8, 6):
        p.upload(W["images"][t])
        tabs = [tuple(hm.trace_tables(W, host[k], t)) if k in host else None for k in range(ns)]
        b = [x.launch_count() for x in (p.g[0], p.t[0])]
        p.g[0].trace_store(p.st, tabs)
        p.t[0].trace_store(p.ts, tabs)
        assert p.g[0].launch_count() - b[0] == p.t[0].launch_count() - b[1] == 1
        same_stores(p.st, p.ts, f"traced frame {t}")
    status = np.concatenate([p.st.get(k)["status"] for k in host])
    assert (status != 5).sum() > 0 and len(np.unique(status)) > 1
    p.close()


@pytest.mark.gpu
def test_activation_afterwards(capi, gpu, orc, synth):
    """dmv_ba_activate_store with my_type from the call's returned type, against activatePointsMT's five steps on the twin store with the
    twin's points and types"""
    win = Win(capi, synth, orc, 123, nf=5, npts=1200)
    w, h = win.w, win.h
    p = Pair(capi, w, h, synth.pyr_levels(w, h), stores=tuple(win.stores))
    slot = [3, 0, 6, 1, -1]
    types = {}
    for f, k in enumerate(slot[:-1]):
        p.upload(win.W["images"][f])
        r, o = p.keyframe(k, what=f"keyframe {f}")
        types[k] = r["points"]["type"]
        win.copies[k] = dict(as_put(o["points"]), type=o["points"]["type"])
        win.frame_of[k] = f
    for t in (4, 3, 4):
        win.trace(t)
    win.check_stores("traced")
    newest, flagged, mad = win.nf - 1, np.zeros(win.nf, np.uint8), 2.0
    before = [b.launch_count() for b in win.bas]
    r = win.bas[0].activate_store(win.stores[0], newest, win.tab12, flagged, *win.act, slot, [types.get(k) for k in slot], mad, win.RT, want_map=True)
    t, br = win.five_steps(slot, newest, flagged, mad, want_map=True)
    assert win.bas[0].launch_count() - before[0] == win.bas[1].launch_count() - before[1]
    for key in ("opt_frame", "opt_index", "status", "idepth", "res_state", "order", "n_kept", "action", "map"):
        assert r[key].shape == t[key].shape and np.array_equal(bits(r[key]), bits(t[key])), key
    assert r["stats"] == t["stats"]
    assert br["delete"] + len(r["opt_frame"]) > 0, br
    win.check_stores("after the activation")
    win.trace(4)
    win.check_stores("traced after the activation")
    close(*p.g, *p.t)
    win.close()


@pytest.mark.gpu
def test_raw_upload_and_two_handles(capi, gpu, orc):
    """keyframes made resident by dmv_ct_upload_raw_image, and two handles taking turns on one store with one potential"""
    w, h, lv = S.SEQ[0][:3]
    p = Pair(capi, w, h, lv, handles=2)
    for i, (_, _, _, kind, seed) in enumerate(S.SEQ):
        x = i % 2
        img = S.image(kind, w, h, seed)
        if i == 2:
            for y in (p.g[x], p.t[x]):
                y.set_undistort(w, h)
                y.upload_raw_image(img.astype(np.uint8), exposure=0.0)
        else:
            p.upload(img, x)
        p.keyframe(i, i=x, want=ALL if i == 2 else ("type",), what=f"keyframe {i} on handle {x}")
    p.close()


@pytest.mark.gpu
def test_keyframe_made_resident_by_set_ref_from_ba(capi, gpu, orc, synth):
    W = synth.make_window(nf=4, npts=600, seed=21)
    w, h, lv = W["w"], W["h"], 5
    src = capi.CT(w, h, lv)
    src.upload_new_image(W["images"][-1])
    ba = capi.BA(w, h, max_frames=W["nf"], max_points=len(W["host"]))
    for k in range(W["nf"] - 1):
        ba.upload_frame(k, W["dI"][k])
    ba.adopt_frame(W["nf"] - 1, src)
    ba.set_window(W["nf"])
    ba.set_points(W["host"], W["u"], W["v"], W["idepth"], W["idepth_zero"], W["color"], W["weights"])
    ba.set_residuals(W["res_point"], W["res_target"])
    ba.set_adjoints(*hm.adjoints(W))
    ba.set_state(hm.calib8(W["K"]), hm.precalc_table(W), W["frameEnergyTH"])
    ba.linearize(); ba.apply_res(); ba.accumulate()
    p = Pair(capi, w, h, lv)
    p.upload(W["images"][0])   # another frame was resident before the hand-off
    for x in (p.g[0], p.t[0]):
        x.set_ref_from_ba(ba)
    r, _ = p.keyframe(3, want=ALL, what="set_ref_from_ba")
    assert r["n"] > 100
    p.close(); src.close(); ba.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# cap and refusals
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cap_overflow_and_no_cap(capi, gpu, orc):
    w, h, lv = 640, 480, 5
    p = Pair(capi, w, h, lv)
    p.upload(S.image("tex", w, h, 80))
    p.keyframe(1, what="first")
    p.upload(S.image("high", w, h, 81))
    need = len(p.t[0].make_new_traces(p.pot)["points"]["u"])
    snap = snapshot(p.st)
    for want in (("type",), ("energyTH", "u")):
        b = p.g[0].launch_count()
        with pytest.raises(capi.DmvError, match=f"{need} new points exceed cap {need - 1}"):
            p.g[0].make_new_traces_store(p.st, 4, p.pot, want=want, cap=need - 1)
        assert p.g[0].last_needed == need and p.g[0].last_potential == p.pot
        assert unchanged(p.st, snap)
        launched = p.g[0].launch_count() - b
    bt = p.t[0].launch_count()
    with pytest.raises(capi.DmvError, match="exceed cap"):
        p.t[0].make_new_traces(p.pot, cap=need - 1)
    assert launched == p.t[0].launch_count() - bt - 1   # the copy into the store is not launched
    p.keyframe(4, want=("type", "gradH"), cap=need, what="retry at the exact cap")
    p.upload(S.image("tex", w, h, 82))
    r, _ = p.keyframe(6, want=(), cap=0, what="no outputs: no cap")
    assert r["n"] > 0
    p.close()


@pytest.mark.gpu
def test_refusals_change_nothing(capi, gpu, orc):
    """every refusal with its message (dmv_ct_make_new_traces' own messages where it refuses the same arguments), leaving the store, the
    potential, n, the outputs and the launch count as they were"""
    L = capi.lib()
    w, h, lv = 640, 480, 5
    img = S.image("tex", w, h, 90)
    g = capi.CT(w, h, lv)
    g.upload_new_image(img)
    st = capi.IPStore()
    g.make_new_traces_store(st, 2, 3)
    snap = snapshot(st)
    two, odd = capi.CT(w, h, 2), capi.CT(648, 480, 4)
    two.upload_new_image(img)
    hs = (g, two, odd)
    counts = [x.launch_count() for x in hs]
    cap = 16384

    class Raw:
        def __init__(self, outputs=True):
            self.pot, self.n, self.npt = C.c_int(3), C.c_int(-7), C.c_int(-7)
            self.out = {k: np.full((cap,) + s, -7, t) for k, (s, t) in capi._NT_SHAPES.items()}
            self.map = np.full(w * h, 12345.0, np.float32)
            ptr = lambda k: self.out[k].ctypes.data if outputs else None  # noqa: E731
            self.a = capi.NewTracesArgs(1500.0, 1, 1.0, None, None, C.pointer(self.pot), cap, C.pointer(self.n), C.pointer(self.npt), ptr("u"),
                                        ptr("v"), ptr("type"), ptr("color"), ptr("weights"), ptr("gradH"), ptr("energyTH"), self.map.ctypes.data)

        def untouched(self, pot=3):
            return (self.pot.value == pot and self.n.value == -7 and self.npt.value == -7 and (self.map == 12345.0).all()
                    and all((a == -7).all() for a in self.out.values()))

    def refused(rc, msg, raw, handle=g, pot=3, same_as_make_new_traces=True):
        text = L.dmv_last_error().decode()
        assert rc == DMV_ERR_INVALID, (rc, text)
        assert text == msg, text
        assert raw.untouched(pot) and [x.launch_count() for x in hs] == counts
        assert unchanged(st, snap)
        if same_as_make_new_traces:   # dmv_ct_make_new_traces refuses the same arguments with the same message
            assert L.dmv_ct_make_new_traces(handle.h, C.byref(raw.a)) == DMV_ERR_INVALID
            assert L.dmv_last_error().decode() == msg
            assert raw.untouched(pot) and [x.launch_count() for x in hs] == counts

    r = Raw()
    refused(L.dmv_ct_make_new_traces_store(None, st.h, 0, C.byref(r.a)), "null argument", r, same_as_make_new_traces=False)
    refused(L.dmv_ct_make_new_traces_store(g.h, None, 0, C.byref(r.a)), "null argument", r, same_as_make_new_traces=False)
    refused(L.dmv_ct_make_new_traces_store(g.h, st.h, 0, None), "null argument", r, same_as_make_new_traces=False)
    call = lambda raw, slot=0, h_=g: L.dmv_ct_make_new_traces_store(h_.h, st.h, slot, C.byref(raw.a))  # noqa: E731
    refused(call(r, h_=two), "pixel selection reads levels 0-2: the handle has 2", r, handle=two)
    refused(call(r, h_=odd), "pixel selection needs w and h divisible by 16 (648 x 480)", r, handle=odd)
    for field in ("potential", "n", "numPointsTotal"):
        r = Raw(); setattr(r.a, field, None)
        refused(call(r), "null argument", r)
    r = Raw(); r.a.cap = -1
    refused(call(r), "null argument", r)
    r = Raw(); r.pot.value = 0
    refused(call(r), "potential 0 < 1", r, pot=0)
    for field, val, msg in (("density", 0.0, "density must be finite and > 0"), ("density", float("inf"), "density must be finite and > 0"),
                            ("thFactor", float("nan"), "thFactor must be finite and > 0"), ("recursionsLeft", -1, "recursionsLeft must be in 0..8"),
                            ("recursionsLeft", 9, "recursionsLeft must be in 0..8")):
        r = Raw(); setattr(r.a, field, val)
        refused(call(r), msg, r)
    bad = capi.PSSettings()
    L.dmv_ps_default_settings(C.byref(bad))
    bad.minGradHistCut = 1.0
    r = Raw(); r.a.settings = C.addressof(bad)
    refused(call(r), "bad dmv_ps_settings", r)
    for slot in (-1, 64):
        r = Raw()
        refused(call(r, slot=slot), f"slot {slot}: expected 0 to 63", r, same_as_make_new_traces=False)
    if L.dmv_device_count() >= 2:
        other = capi.IPStore(device=1)
        r = Raw()
        refused(L.dmv_ct_make_new_traces_store(g.h, other.h, 0, C.byref(r.a)), "the store is on device 1, the handle on device 0", r,
                same_as_make_new_traces=False)
        other.close()
    # NULL outputs are accepted, each on its own
    r = Raw(); r.a.gradH4 = None
    assert call(r, slot=3) == 0, L.dmv_last_error()
    assert r.n.value > 0 and (r.out["gradH"] == -7).all() and not (r.out["type"] == -7).all()
    close(g, two, odd, st)


def test_refusals_without_a_device(capi):
    L = capi.lib()
    a = capi.NewTracesArgs()
    assert L.dmv_ct_make_new_traces_store(None, None, 0, None) == DMV_ERR_INVALID
    assert L.dmv_ct_make_new_traces_store(None, None, 0, C.byref(a)) == DMV_ERR_INVALID
    assert L.dmv_last_error() == b"null argument"
    assert "dmv_ct_make_new_traces_store" in capi.SYMBOLS

"""dmv_ba_activate_store against a twin: a second store with the same contents and a second BA handle on the same window running
activatePointsMT's five steps on host arrays: dmv_ip_store_get of every slot, dmv_ba_select_activation, dmv_ba_activate_points on its
toOptimize, the choice of the points to drop (FullSystem.cpp:L732-770, restated here in numpy) and dmv_ip_store_remove per slot.  Every
output, the stores' contents and counts after get, and both handles' launch counts must agree bit for bit, as must every frame traced
over the two stores afterwards."""
import ctypes as C

import numpy as np
import pytest

import dmvio_b200.hostmath as hm
from dmvio_b200.capi import DMV_ERR_INVALID, DMV_ERR_STATE, IP_OUT_KEYS
from gpu_harness import capi, close, gpu  # noqa: F401
from helpers import product_ba_from_oracle
from test_gpu_trace_store import bits, swap_with_back

DELETE = 1
IPS_OOB = 1


def level1_tables(ow, W):
    """tables12 of dmv_ba_select_activation: host f -> newest frame, level 0 -> level 1"""
    nf = W["nf"]
    fx, fy, cx, cy = [float(v) for v in ow.calib()["k8"][:4]]
    K0 = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    K1 = np.array([[fx * 0.5, 0, (cx + 0.5) / 2 - 0.5], [0, fy * 0.5, (cy + 0.5) / 2 - 0.5], [0, 0, 1]])
    RT = ow.RT().reshape(nf, nf, 12)
    tab = np.zeros((nf, 12), np.float32)
    for f in range(nf):
        tab[f, :9] = (K1 @ RT[f, nf - 1, :9].reshape(3, 3).astype(np.float64) @ np.linalg.inv(K0)).astype(np.float32).reshape(-1)
        tab[f, 9:] = (K1 @ RT[f, nf - 1, 9:].astype(np.float64)).astype(np.float32)
    return tab


class Win:
    """one window (synth.make_window, newest frame last), two BA handles on it (bas[0] runs the call, bas[1] the five steps), two stores
    with the same contents, the host's copies of every slot's points (read-only fields and type, in the slot's order) and a tracker handle"""

    def __init__(self, capi, synth, orc, seed, w=640, h=480, nf=7, npts=2000):
        self.capi, self.orc = capi, orc
        self.W = W = synth.make_window(nf=nf, npts=npts, seed=seed, trans=0.06, rot=0.01, w=w, h=h)
        self.nf, self.w, self.h = nf, w, h
        self.ow = orc.Window(W)
        self.bas = [product_ba_from_oracle(capi, W, self.ow) for _ in range(2)]
        self.stores = [capi.IPStore(), capi.IPStore()]
        self.copies, self.frame_of = {}, {}
        self.ct = capi.CT(w, h, synth.pyr_levels(w, h), max_points=1024)
        self.RT = self.ow.RT()
        self.tab12 = level1_tables(self.ow, W)
        self.rng = np.random.default_rng(seed)
        self.act = (W["u"].astype(np.float32), W["v"].astype(np.float32), W["idepth"].astype(np.float32), W["host"].astype(np.int32))

    def close(self):
        close(self.ct, *self.bas, *self.stores)

    def points(self, f, n):
        """n fresh immature points of frame f with depth intervals around the scene's (half wide, half narrow), and a type each"""
        rng = self.rng
        u, v = rng.integers(10, self.w - 10, n), rng.integers(10, self.h - 10, n)
        P = self.orc.ip_init(self.W["dI"][f], self.w, self.h, u, v)
        P.pop("ok")
        idt = (0.5 * (1 + 0.02 * rng.standard_normal(n))).astype(np.float32)
        wide = rng.random(n) < 0.5
        P["idepth_min"] = (idt * np.where(wide, 0.7, 0.97)).astype(np.float32)
        P["idepth_max"] = (idt * np.where(wide, 1.4, 1.03)).astype(np.float32)
        P["type"] = rng.choice([1.0, 2.0], n).astype(np.float32)
        return P

    def put(self, slot, P, f):
        for st in self.stores:
            st.put(slot, P)
        self.copies[slot], self.frame_of[slot] = dict(P), f

    def trace(self, t):
        """both stores traced against frame t"""
        self.ct.upload_new(0, self.W["dI"][t])
        ns = max([k + 1 for k in self.copies if self.stores[0].counts[k]] + [0])
        tabs = [tuple(hm.trace_tables(self.W, self.frame_of[k], t)) if self.stores[0].counts[k] else None for k in range(ns)]
        for st in self.stores:
            self.ct.trace_store(st, tabs)

    def check_stores(self, what):
        a, b = self.stores
        assert a.counts == b.counts, what
        for k in range(a.SLOTS):
            if a.counts[k]:
                P, Q = a.get(k), b.get(k)
                for key in IP_OUT_KEYS:
                    assert np.array_equal(bits(P[key]), bits(Q[key])), f"{what}: slot {k} {key}"

    def types(self, slot):
        return [self.copies[k]["type"] if 0 <= k < self.stores[0].SLOTS and self.stores[0].counts[k] else None for k in slot]

    def five_steps(self, slot, newest, flagged, mad, cap=None, want_map=True, check=True):
        """steps 1-5 on stores[1] and bas[1]; returns what dmv_ba_activate_store returns, restated.  check: each slot's new order against
        swap_with_back"""
        ba, st, nf = self.bas[1], self.stores[1], self.nf
        groups = []
        for f in range(nf):
            k = slot[f]
            groups.append(st.get(k, self.copies[k]) if k >= 0 and st.counts[k] else None)
        cnt = [0 if g is None else len(g["u"]) for g in groups]
        off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
        cat = lambda key, shape, t: np.concatenate([g[key] for g in groups if g is not None] or [np.zeros(shape, t)])  # noqa: E731
        imm = dict(u=cat("u", 0, np.float32), v=cat("v", 0, np.float32), idepth_min=cat("idepth_min", 0, np.float32),
                   idepth_max=cat("idepth_max", 0, np.float32), status=cat("status", 0, np.int32), interval=cat("lastTracePixelInterval", 0, np.float32),
                   quality=cat("quality", 0, np.float32), type=cat("type", 0, np.float32))
        action, opt, m, stats = ba.select_activation(nf, newest, self.tab12, flagged, *self.act, off, imm, mad, cap=cap, want_map=want_map)
        frame = (np.searchsorted(off, opt, side="right") - 1).astype(np.int32)
        if len(opt):
            sub = {key: cat(key, (0,) + shape, np.float32)[opt] for key, shape in (("u", ()), ("v", ()), ("color", (8,)), ("weights", (8,)),
                                                                                      ("energyTH", ()), ("idepth_min", ()), ("idepth_max", ()))}
            status, idepth, rs = ba.activate_points(frame, sub, self.RT)
        else:
            status, idepth, rs = np.zeros(0, np.int32), np.zeros(0, np.float32), np.zeros((0, nf), np.int32)
        dead = action == DELETE
        drop = (status != 0) | (imm["status"][opt] == IPS_OOB)
        dead[opt[drop]] = True
        order, n_kept, branches = [], [], dict(delete=int((action == DELETE).sum()), activated=int((status == 1).sum()),
                                               outlier=int((status == -1).sum()), oob=int(((status == 0) & drop).sum()))
        for f in range(nf):
            k = slot[f]
            if k < 0:
                n_kept.append(0)
                continue
            idx = np.flatnonzero(dead[off[f]:off[f + 1]]) if f != newest else np.zeros(0, np.int64)
            o = st.remove(k, idx)
            assert not check or np.array_equal(o, swap_with_back(cnt[f], idx))
            order.append(o)
            n_kept.append(len(o))
        return dict(opt_frame=frame, opt_index=(opt - off[frame]).astype(np.int32), status=status, idepth=idepth, res_state=rs,
                    order=np.concatenate(order or [np.zeros(0, np.int32)]).astype(np.int32), n_kept=np.array(n_kept, np.int32), action=action, map=m,
                    stats=stats), branches

    def turnover(self, slot, newest=None, flagged=None, mad=2.0, cap=None, want_map=True, what=""):
        """dmv_ba_activate_store on stores[0] / bas[0] against the five steps on the twin; the host's copies follow the new order"""
        nf = self.nf
        newest = nf - 1 if newest is None else newest
        flagged = np.zeros(nf, np.uint8) if flagged is None else np.asarray(flagged, np.uint8)
        types = self.types(slot)
        before = [b.launch_count() for b in self.bas]
        r = self.bas[0].activate_store(self.stores[0], newest, self.tab12, flagged, *self.act, slot, types, mad, self.RT, cap=cap, want_map=want_map)
        t, branches = self.five_steps(slot, newest, flagged, mad, cap=cap, want_map=want_map)
        assert self.bas[0].launch_count() - before[0] == self.bas[1].launch_count() - before[1] == int(len(t["opt_frame"]) > 0), what
        for key in ("opt_frame", "opt_index", "status", "idepth", "res_state", "order", "n_kept", "action"):
            assert r[key].shape == t[key].shape and np.array_equal(bits(r[key]), bits(t[key])), f"{what}: {key}"
        assert r["stats"] == t["stats"], what
        assert (r["map"] is None) == (not want_map) and (not want_map or np.array_equal(bits(r["map"]), bits(t["map"]))), what
        self.check_stores(what)
        at = 0
        for f, k in enumerate(slot):   # the host applies order_out to its read-only copies
            if k in self.copies:
                o = r["order"][at:at + r["n_kept"][f]]
                at += len(o)
                self.copies[k] = {key: a[o] for key, a in self.copies[k].items()}
        return r, branches


def fill(win, slot, n):
    for f, k in enumerate(slot):
        if k >= 0 and f != win.nf - 1:
            win.put(k, win.points(f, n), f)


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(640, 480), (512, 512)])
def test_c3_window_turnovers(capi, gpu, orc, synth, shape):
    """a C3-like window (7 keyframes, 6 x 1500 immature points) in slots that do not follow frame order; three turnovers, each after
    frames traced over both stores, and traced frames after the last"""
    win = Win(capi, synth, orc, 100 + shape[0], *shape)
    slot = [5, 2, 9, 0, 3, 7, -1]
    fill(win, slot, 1500)
    seen = dict(delete=0, activated=0, outlier=0, oob=0)
    for turn, mad in enumerate((2.0, 4.0, 1.0)):
        for t in (6, 5, 6):
            win.trace(t)
        win.check_stores(f"turnover {turn}: traced")
        _, br = win.turnover(slot, mad=mad, what=f"turnover {turn}")
        seen = {k: seen[k] + br[k] for k in seen}
    for t in (6, 4):
        win.trace(t)
    win.check_stores("traced after the turnovers")
    assert seen["delete"] > 0 and seen["activated"] > 0, seen
    win.close()


@pytest.mark.gpu
def test_slot_edge_cases(capi, gpu, orc, synth):
    """a frame without a slot, a named empty slot, a populated slot no frame names (untouched), the newest frame holding a slot (untouched),
    and a flagged host"""
    win = Win(capi, synth, orc, 7, nf=6, npts=1200)
    slot = [4, -1, 1, 63, 0, 2]
    for f, k in ((0, 4), (2, 1), (4, 0), (5, 2)):
        win.put(k, win.points(f, 900), f)
    win.put(10, win.points(3, 300), 3)            # named by no frame
    for t in (5, 4):
        win.trace(t)
    untouched = {k: win.stores[0].get(k) for k in (10, 2)}
    r, _ = win.turnover(slot, flagged=[0, 0, 1, 0, 0, 0], mad=1.0, what="edges")
    assert r["n_kept"][1] == 0 and r["n_kept"][3] == 0 and r["n_kept"][5] == 900
    assert np.array_equal(r["order"][-900:], np.arange(900))
    for k, P in untouched.items():
        Q = win.stores[0].get(k)
        assert all(np.array_equal(bits(P[key]), bits(Q[key])) for key in IP_OUT_KEYS), k
    win.trace(5)
    win.check_stores("traced after")
    win.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(640, 480), (512, 512)])
def test_first_keyframes(capi, gpu, orc, synth, shape):
    """two keyframes, currentMinActDist 0: every candidate is decided before the loop"""
    win = Win(capi, synth, orc, 3, *shape, nf=2, npts=40)
    win.put(1, win.points(0, 3000), 0)
    win.trace(1)
    r, _ = win.turnover([1, -1], mad=0.0, what="first keyframes")
    assert r["stats"]["undecided"] == 0 and len(r["opt_frame"]) > 0
    win.trace(1)
    win.check_stores("traced after")
    win.close()


@pytest.mark.gpu
@pytest.mark.parametrize("count", [0, 1])
def test_zero_and_one_candidates(capi, gpu, orc, synth, count):
    win = Win(capi, synth, orc, 20 + count, nf=3, npts=300)
    P = win.points(0, 50)
    P["lastTracePixelInterval"][:] = 100.0            # not ready: kept
    P["status"][:] = 3
    P["lastTracePixelInterval"][:count] = 1.0
    P["idepth_max"][:count] = P["idepth_min"][:count]
    win.put(0, P, 0)
    win.put(1, {k: a[:0] for k, a in P.items()}, 1)   # a named slot without points
    r, _ = win.turnover([0, 1, -1], mad=0.0, what=f"{count} candidates")
    assert len(r["opt_frame"]) == count
    win.close()


@pytest.mark.gpu
def test_every_removal_branch(capi, gpu, orc, synth):
    """points built to reach each way out: non-finite idepth_max, IPS_OUTLIER, not ready on a flagged host, not ready and OOB, projection
    outside the map, and toOptimize entries that end activated (1), outliers (-1), and not activated but OOB"""
    win = Win(capi, synth, orc, 31, nf=4, npts=600)
    rng = np.random.default_rng(5)
    slot = [2, 0, 1, -1]
    kinds = {}
    for f, k in enumerate(slot[:3]):
        P = win.points(f, 1200)
        n = len(P["u"])
        P["status"] = rng.choice([0, 3, 4, 1], n).astype(np.int32)
        P["lastTracePixelInterval"][:] = 1.0
        P["quality"][:] = 10.0
        kind = rng.integers(0, 8, n)
        P["idepth_max"][kind == 0] = np.inf
        P["status"][kind == 1] = 2
        P["lastTracePixelInterval"][kind == 2] = 9.0            # not ready (OOB too on some)
        P["u"][kind == 3] = -3000.0                            # projects outside the map
        P["energyTH"][kind == 4] = np.nan                      # activation ends -1
        weak = kind == 5                                       # no weight: Hdd 0, activation ends 0
        P["weights"][weak] = 0.0
        P["status"][weak & (rng.random(n) < 0.5)] = IPS_OOB
        win.put(k, P, f)
        kinds[f] = kind
    off = np.concatenate([[0], np.cumsum([len(kinds[f]) for f in range(3)])])
    r, br = win.turnover(slot, flagged=[1, 0, 0, 0], mad=0.0, what="branches")
    a = r["action"]
    assert br["activated"] > 0 and br["outlier"] > 0 and br["oob"] > 0 and br["delete"] > 0, br
    cat = np.concatenate([kinds[f] for f in range(3)])
    for kind in (0, 1, 3):
        assert ((cat == kind) & (a == DELETE)).sum() > 0, kind
    assert ((cat == 2) & (a == DELETE))[:off[1]].sum() > 0                    # not ready on the flagged host
    assert ((cat == 2) & (a == DELETE))[off[1]:].sum() > 0                    # not ready and OOB elsewhere
    win.close()


@pytest.mark.gpu
def test_cap_overflow_changes_nothing(capi, gpu, orc, synth):
    win = Win(capi, synth, orc, 41, nf=4, npts=600)
    slot = [0, 1, 2, -1]
    fill(win, slot, 800)
    win.trace(3)
    counts = list(win.stores[0].counts)
    snap = {k: win.stores[0].get(k) for k in range(3)}
    launches = win.bas[0].launch_count()
    with pytest.raises(capi.DmvError) as e:
        win.bas[0].activate_store(win.stores[0], 3, win.tab12, np.zeros(4, np.uint8), *win.act, slot, win.types(slot), 0.0, win.RT, cap=1)
    need = e.value.args[1]
    assert need > 1 and "exceed cap 1" in e.value.args[0]
    assert win.stores[0].counts == counts and win.bas[0].launch_count() == launches
    for k, P in snap.items():
        Q = win.stores[0].get(k)
        assert all(np.array_equal(bits(P[key]), bits(Q[key])) for key in IP_OUT_KEYS)
    win.turnover(slot, mad=0.0, cap=need, what="exact cap")
    win.close()


@pytest.mark.gpu
def test_ba_state_untouched(capi, gpu, orc, synth):
    """a dmv_ba_gn_step after the call is bit-identical to one without it"""
    outs = []
    for call in (False, True):
        win = Win(capi, synth, orc, 3, nf=4, npts=600)
        ba = win.bas[0]
        ow, W = win.ow, win.W
        tabs = (ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"])
        ba.linearize()
        ba.apply_res()
        acc = ba.accumulate()
        x = hm.solve_reduced(acc["HA"], acc["bA"], acc["Hsc"], acc["bsc"], *hm.prior_system(W), lam=1e-5)
        if call:
            fill(win, [0, 1, 2, -1], 500)
            win.trace(3)
            r, _ = win.turnover([0, 1, 2, -1], mad=0.0)
            assert len(r["opt_frame"]) > 0
        g = ba.gn_step(x, *tabs)
        ba.apply_res()
        acc = ba.accumulate()
        outs.append((g["energy"], g["n_in"], np.array(g["sums"]), ba.get_idepth()[0].copy(), {k: np.array(acc[k]) for k in ("HA", "bA", "Hsc", "bsc")}))
        win.close()
    assert outs[0][0] == outs[1][0] and outs[0][1] == outs[1][1]
    assert np.array_equal(outs[0][2], outs[1][2]) and np.array_equal(outs[0][3], outs[1][3])
    for k in outs[0][4]:
        assert np.array_equal(outs[0][4][k], outs[1][4][k]), k


# ---------------------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------------------
class Raw:
    """the raw arguments of one dmv_ba_activate_store call, outputs filled with sentinels"""

    def __init__(self, capi, win, slot, cap=64):
        nf = len(slot)
        self.slot = np.asarray(slot, np.int32)
        self.types = [None if t is None else np.ascontiguousarray(t) for t in win.types(slot)]
        self.tptr = (C.c_void_p * max(nf, 1))(*[None if t is None else t.ctypes.data for t in self.types])
        self.flagged = np.zeros(max(nf, 1), np.uint8)
        self.n_opt = C.c_int(-7)
        self.out = dict(opt_frame=np.full(cap, -7, np.int32), opt_index=np.full(cap, -7, np.int32), status=np.full(cap, -7, np.int32),
                        idepth=np.full(cap, 12345.0, np.float32), res_state=np.full(cap * 8, -7, np.int32), order=np.full(20000, -7, np.int32),
                        n_kept=np.full(8, -7, np.int32), action=np.full(20000, -7, np.int32), map=np.full(win.w * win.h // 4, 12345.0, np.float32),
                        stats=np.full(3, -7, np.int32))
        o = self.out
        self.a = capi.BAActivateStoreArgs(nf, nf - 1, win.tab12.ctypes.data, self.flagged.ctypes.data, len(win.act[0]), *[x.ctypes.data for x in win.act],
                                          self.slot.ctypes.data, C.cast(self.tptr, C.c_void_p), 2.0, 3.0, win.RT.ctypes.data, 1, cap,
                                          C.addressof(self.n_opt), *[o[k].ctypes.data for k in ("opt_frame", "opt_index", "status", "idepth", "res_state",
                                                                                                  "order", "n_kept", "action", "map", "stats")])

    def untouched(self):
        return self.n_opt.value == -7 and all(((a == -7) | (a == 12345.0)).all() for a in self.out.values())


@pytest.mark.gpu
def test_refusals_change_nothing(capi, gpu, orc, synth):
    """every refusal, with its full message, leaving both handles' launch counts, the store and the output sentinels as they were"""
    L = capi.lib()
    win = Win(capi, synth, orc, 51, nf=4, npts=600)
    slot = [0, 3, 1, -1]
    fill(win, slot, 200)
    win.trace(3)
    st, ba = win.stores[0], win.bas[0]
    counts = list(st.counts)
    snap = {k: st.get(k) for k in (0, 1, 3)}
    launches = ba.launch_count()
    empty = capi.BA(win.w, win.h, max_frames=8, max_points=64)

    def refused(rc, msg, raw, code=DMV_ERR_INVALID):
        text = L.dmv_last_error().decode()
        assert rc == code, (rc, text)
        assert text == msg, text
        assert raw.untouched() and st.counts == counts and ba.launch_count() == launches
        for k, P in snap.items():
            Q = st.get(k)
            assert all(np.array_equal(bits(P[key]), bits(Q[key])) for key in IP_OUT_KEYS)

    def call(raw, h=ba.h, s=st.h):
        return L.dmv_ba_activate_store(h, s, C.byref(raw.a))

    r = Raw(capi, win, slot)
    refused(L.dmv_ba_activate_store(None, st.h, C.byref(r.a)), "null argument", r)
    refused(L.dmv_ba_activate_store(ba.h, None, C.byref(r.a)), "null argument", r)
    refused(L.dmv_ba_activate_store(ba.h, st.h, None), "null argument", r)
    refused(call(r, h=empty.h), "dmv_ba_set_window + dmv_ba_set_state first", r, DMV_ERR_STATE)
    r = Raw(capi, win, slot + [-1])
    refused(call(r), "nf = 5: the window has 4 frames", r)
    r = Raw(capi, win, slot); r.a.slot = None
    refused(call(r), "incomplete dmv_ba_activate_store_args", r)
    r = Raw(capi, win, slot); r.a.my_type = None
    refused(call(r), "incomplete dmv_ba_activate_store_args", r)
    r = Raw(capi, win, [0, 64, 1, -1])
    refused(call(r), "slot[1] = 64: expected -1 to 63", r)
    r = Raw(capi, win, [0, -2, 1, -1])
    refused(call(r), "slot[1] = -2: expected -1 to 63", r)
    r = Raw(capi, win, [0, 3, 0, -1])
    refused(call(r), "slot[0] and slot[2] are both 0", r)
    r = Raw(capi, win, slot); r.tptr[2] = None
    refused(call(r), "my_type[2] is NULL for 200 points", r)
    r = Raw(capi, win, slot); r.a.newest = 4
    refused(call(r), "nf 4 / newest 4 out of range", r)
    r = Raw(capi, win, slot); r.a.tables12 = None
    refused(call(r), "incomplete dmv_ba_select_args", r)
    r = Raw(capi, win, slot); r.a.n_opt = None
    refused(call(r), "incomplete dmv_ba_select_args", r)
    r = Raw(capi, win, slot); r.a.cap = -1
    refused(call(r), "incomplete dmv_ba_select_args", r)
    r = Raw(capi, win, slot); r.a.act_v = None
    refused(call(r), "incomplete active points", r)
    host = win.act[3].copy(); host[5] = 4
    r = Raw(capi, win, slot); r.a.act_host = host.ctypes.data
    refused(call(r), "active point 5: host 4 out of range", r)
    for k in ("RT", "opt_frame", "opt_index", "status", "idepth", "res_state"):
        r = Raw(capi, win, slot); setattr(r.a, k, None)
        refused(call(r), "incomplete dmv_ba_activate_store_args", r)
    if L.dmv_device_count() >= 2:
        other = capi.IPStore(device=1)
        r = Raw(capi, win, slot)
        refused(call(r, s=other.h), "the store is on device 1, the handle on device 0", r)
        other.close()
    r = Raw(capi, win, slot, cap=0)
    r.a.RT = r.a.opt_frame = r.a.opt_index = r.a.status = r.a.idepth = r.a.res_state = None   # cap 0: none of them is needed
    rc = call(r)
    assert rc == DMV_ERR_INVALID and r.n_opt.value > 0 and "exceed cap 0" in L.dmv_last_error().decode()
    assert st.counts == counts and ba.launch_count() == launches
    empty.close()
    win.close()


def test_refusals_without_a_device(capi):
    """the checks that come before any handle or store is read"""
    L = capi.lib()
    a = capi.BAActivateStoreArgs()
    assert L.dmv_ba_activate_store(None, None, None) == DMV_ERR_INVALID
    assert L.dmv_ba_activate_store(None, None, C.byref(a)) == DMV_ERR_INVALID
    assert L.dmv_last_error() == b"null argument"
    assert "dmv_ba_activate_store" in capi.SYMBOLS

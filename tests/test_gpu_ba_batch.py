"""The batched BA launch (dmv_ba_batch_gn_step, ba_fused_batch_kernel) where it differs from a window's own launch.

A batch deals (window, chunk) work items round-robin over min(items, resident CTAs) CTAs, so one CTA runs chunks of several windows in a
row in the same shared memory; it finds each item's window by a scan of the item prefix, rotates every window's phase D over the grid and
prefetches the next window's first phase D item.  On the host it stages every member, then finishes each member's linearisation.  The
contract is that every member ends bit-identical to the same window run through dmv_ba_gn_step, so each window here is loaded twice: one
handle goes through the batch, its twin through dmv_ba_gn_step with the same arguments, and everything the handles report afterwards is
compared bit for bit.  The members of the 64-window batch are also held to the fp64 Schur reference of tests/test_gpu_ba_system.py, so the
batch is anchored to a reference of its own and not only to the single launch.

Covered: B = 1 (small and config 4), batches that give every CTA one item, config-4 windows next to one-chunk windows, B = 64 with >= 8
items per SM at both chunk shapes (several rounds per CTA, window boundaries inside a CTA's item sequence); x for some members and not
others, accept / reject chains and single-window steps between batch calls; members reshaped between calls; every refused argument (a
refused call leaves every member as it was); dmv_ba_get_target_energies on single handles and batch members."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import dmvio_b200.hostmath as hm
from dmvio_b200.capi import DMV_ERR_INVALID, DMV_ERR_STATE
from helpers import RES_IN, SYSTEM_TAU, check_system, make_case, prior_f, schur_bound, schur_reference
from gpu_harness import device_capi  # noqa: F401  (the "capi" fixture: every test that takes it needs the device)

pytestmark = pytest.mark.gpu

BATCH_MAX = 64           # ba_device.cuh


@pytest.fixture(scope="module")
def sms(capi):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _items(W, P):
    """work items of a window: chunks of P consecutive points of one host frame (dmv_ba_set_points)"""
    cnt = np.bincount(np.asarray(W["host"]), minlength=W["nf"])
    return int((-(-cnt // P)).sum())


_WINDOWS = {}


def window(synth, cfg):
    """helpers.make_case, rendered once per module: both chunk shapes run the same windows (not modified by the tests)"""
    key = tuple(sorted(cfg.items()))
    if key not in _WINDOWS:
        _WINDOWS[key] = make_case(synth, cfg)
    return _WINDOWS[key]


def _fill(ba, W, ow, frames=True):
    """loads window W into handle ba as helpers.product_ba_from_oracle does, into a handle of any capacity"""
    if frames:
        for k in range(W["nf"]):
            ba.upload_frame(k, W["dI"][k])
    ba.set_window(W["nf"])
    ba.set_points(W["host"], W["u"], W["v"], W["idepth"], W["idepth_zero"], W["color"], W["weights"], priorF=prior_f(W))
    ba.set_residuals(W["res_point"], W["res_target"], W.get("res_state"), W.get("res_energy"))
    ba.set_adjoints(*ow.adjoints())


class Member:
    """one window on two handles: `bt` goes through the batch, its twin `tw` through dmv_ba_gn_step"""

    def __init__(self, capi, orc, synth, cfg, P, max_points=None, max_frames=None):
        self.capi, self.orc, self.synth, self.P = capi, orc, synth, P
        self.cfg = dict(cfg)
        W = window(synth, cfg)
        cap = dict(max_frames=max_frames or max(2, W["nf"]), max_points=max_points or len(W["host"]), chunk_points=P)
        self.bt, self.tw = (capi.BA(W["w"], W["h"], **cap) for _ in range(2))
        self.load(W)
        self.a = None       # committed system (accumulate) of the last commit
        self.steps = 0

    def load(self, W, frames=True):
        self.W, self.ow = W, self.orc.Window(W)
        self.st = (self.ow.calib()["k8"], self.ow.precalc(), self.ow.frame_tables()["frameEnergyTH"])
        for ba in (self.bt, self.tw):
            _fill(ba, W, self.ow, frames)

    def reload(self, frames=True, **kw):
        """the same member with another window: set_window and everything behind it (frames=False: set_points onwards, same frames)"""
        self.cfg.update(kw)
        W = window(self.synth, self.cfg)
        if frames:
            self.load(W)
            return
        self.W, self.ow = W, self.orc.Window(W)
        self.st = (self.ow.calib()["k8"], self.ow.precalc(), self.ow.frame_tables()["frameEnergyTH"])
        for ba in (self.bt, self.tw):
            ba.set_points(W["host"], W["u"], W["v"], W["idepth"], W["idepth_zero"], W["color"], W["weights"], priorF=prior_f(W))
            ba.set_residuals(W["res_point"], W["res_target"], W.get("res_state"), W.get("res_energy"))

    def both(self, name, *args, **kw):
        return [getattr(ba, name)(*args, **kw) for ba in (self.bt, self.tw)]

    def x(self):
        """a Gauss-Newton increment from the committed system (hostmath.solve_reduced; unit damping keeps frames without residuals solvable),
        halved per step so that a chain of steps stays near the start"""
        HL, bL = hm.prior_system(self.W)
        a = self.a
        x = hm.solve_reduced(a["HA"], a["bA"], a["Hsc"], a["bsc"], HL + np.eye(len(bL)), bL, lam=1e-5)
        assert np.all(np.isfinite(x))
        return x * 0.5 ** self.steps

    def close(self):
        self.bt.close()
        self.tw.close()


def assert_same(m, rb, rt, what):
    """everything a handle reports after a step: batched member m.bt against its twin m.tw, bit for bit"""
    for k in ("energy", "n_in", "n_oob", "n_outlier"):
        assert rb[k] == rt[k], f"{what}: {k} {rb[k]!r} != {rt[k]!r}"
    np.testing.assert_array_equal(rb["sums"], rt["sums"], err_msg=f"{what}: step sums")
    gb, gt = m.both("residual_outputs")
    for k in ("newState", "newEnergy", "newEnergyWithOutlier", "centerProjectedTo"):
        np.testing.assert_array_equal(gb[k], gt[k], err_msg=f"{what}: {k}")
    inn = gt["newState"] == RES_IN   # JpJdF is defined for IN residuals only (include/dmvio_b200.h)
    np.testing.assert_array_equal(gb["JpJdF"][inn], gt["JpJdF"][inn], err_msg=f"{what}: JpJdF")
    pb, pt = m.both("point_outputs")
    for k in ("Hdd", "bd", "Hcd", "HdiF", "bdSumF"):
        np.testing.assert_array_equal(pb[k], pt[k], err_msg=f"{what}: {k}")
    (ib, zb), (it, zt) = m.both("get_idepth")
    np.testing.assert_array_equal(ib, it, err_msg=f"{what}: idepth")
    np.testing.assert_array_equal(zb, zt, err_msg=f"{what}: idepth_zero")


def commit(m, what):
    """apply_res on both handles, then the accumulated systems bit for bit; keeps the system for the next x"""
    m.both("apply_res")
    ab, at = m.both("accumulate")
    for k in ("HA", "bA", "Hsc", "bsc"):
        np.testing.assert_array_equal(ab[k], at[k], err_msg=f"{what}: {k}")
    assert ab["resInA"] == at["resInA"], what
    m.a = at
    return ab


def batch_step(batch, members, xs, what):
    """one batched call and the same steps on the twins, compared member by member"""
    xs = xs if xs is not None else [None] * len(members)
    rb = batch.gn_step(xs, [m.st for m in members])
    for i, (m, x, r) in enumerate(zip(members, xs, rb)):
        assert_same(m, r, m.tw.gn_step(x, *m.st), f"{what}, member {i} ({m.cfg})")


def single_step(m, x, what):
    """dmv_ba_gn_step on both handles of one member"""
    rb, rt = m.both("gn_step", x, *m.st)
    assert_same(m, rb, rt, what)


def schur_ratio(m):
    """the committed Schur system of the batched handle against helpers.schur_reference (fp64 from the launch's own outputs)"""
    g, po = m.bt.residual_outputs(), m.bt.point_outputs()
    Hsc, bsc, _, _ = schur_reference(m.W, g["newState"], g["JpJdF"], po["Hcd"], po["HdiF"], po["bdSumF"], *m.ow.adjoints())
    return max(check_system(m.a["Hsc"], m.a["bsc"], Hsc, bsc, schur_bound(po["HdiF"], po["bdSumF"]), SYSTEM_TAU,
                            f"Schur system of {m.cfg}"))


def mem_used():
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2 ** 30


def b64_configs():
    """64 windows: nf 2..8, npts 1..2000 (chunk boundaries at both shapes, then seeded sizes), every `hosts` mode, a third with the edge
    cases of helpers.edge_window; 320x240 images (640x480 for every eighth) keep 128 handles near 1 GB"""
    rng = np.random.default_rng(64)
    npts = [1, 2, 15, 16, 17, 31, 32, 33, 2000, 1999, 64, 65] + [int(n) for n in rng.integers(40, 2001, 52)]
    cfgs = []
    for i in range(BATCH_MAX):
        c = dict(nf=2 + i % 7, npts=npts[i], seed=1000 + i, hosts=("all_but_newest", "first", "all")[(i // 3) % 3], w=320, h=240)
        if i % 8 == 5:
            c.update(w=640, h=480)
        if i % 3 == 0:
            c["edge"] = True
        cfgs.append(c)
    return cfgs


DEAL_CASES = {
    "B1_small": lambda P: [dict(nf=3, npts=333, seed=7)],
    "B1_config4_edge": lambda P: [dict(nf=7, npts=8000, seed=1234, edge=True)],
    "one_item_per_cta": lambda P: [dict(nf=2, npts=200, seed=3, hosts="first"), dict(nf=3, npts=333, seed=7),
                                   dict(nf=5, npts=300, seed=11, edge=True), dict(nf=8, npts=150, seed=99, hosts="all")],
    "config4_and_one_chunk": lambda P: [dict(nf=7, npts=8000, seed=1234, edge=True), dict(nf=2, npts=1, seed=5, hosts="first"),
                                        dict(nf=3, npts=P + 1, seed=6, hosts="first")],
    "B64": lambda P: b64_configs(),
}


@pytest.mark.parametrize("case", list(DEAL_CASES))
@pytest.mark.parametrize("P", [16, 32])
def test_dealing_regimes(capi, orc, synth, sms, case, P):
    """a first linearisation, then a fused GN step: every member bit-identical to its twin's dmv_ba_gn_step"""
    used0 = mem_used()
    members = [Member(capi, orc, synth, c, P) for c in DEAL_CASES[case](P)]
    B = len(members)
    items = sum(_items(m.W, P) for m in members)
    if case == "one_item_per_cta":
        assert items < sms, f"{items} items on {sms} SMs: some CTA would get two"
    if case == "B64":
        assert B == BATCH_MAX
        assert items >= 8 * sms, f"{items} items < 8 x {sms} SMs: no guarantee of several rounds per CTA"
    if case.startswith("B1"):
        assert B == 1
    batch = capi.BABatch([m.bt for m in members])
    used1 = mem_used()
    worst = 0.0
    try:
        batch_step(batch, members, None, "first linearisation")
        for m in members:
            commit(m, "first linearisation")
            if case == "B64":
                worst = max(worst, schur_ratio(m))
        xs = [m.x() for m in members]
        for m in members:
            m.both("backup_points")
        batch_step(batch, members, xs, "fused GN step")
        for m in members:
            commit(m, "fused GN step")
            if case == "B64":
                worst = max(worst, schur_ratio(m))
    finally:
        batch.close()
        for m in members:
            m.close()
    print(f"{case}: B={B} P={P} S={sms} items={items} ({items / sms:.1f} per SM); device memory {used0:.2f} -> {used1:.2f} GB "
          f"with {2 * B} handles; worst check_system ratio vs the fp64 Schur reference "
          + (f"{worst:.2e} (tau {SYSTEM_TAU:.0e})" if case == "B64" else "n/a"))


@pytest.mark.parametrize("P", [16, 32])
def test_mixed_and_chained_steps(capi, orc, synth, P):
    """x for some members and None for others in one call; three calls in which every member accepts (apply_res) or rejects
    (restore_points) on its own; a single dmv_ba_gn_step on one member between two batch calls.  The twins follow the same sequence."""
    cfgs = [dict(nf=7, npts=2000, seed=1234), dict(nf=4, npts=333, seed=5), dict(nf=8, npts=777, seed=99, hosts="all", edge=True),
            dict(nf=2, npts=200, seed=3, hosts="first"), dict(nf=5, npts=900, seed=21, edge=True), dict(nf=3, npts=40, seed=8)]
    members = [Member(capi, orc, synth, c, P) for c in cfgs]
    batch = capi.BABatch([m.bt for m in members])
    rng = np.random.default_rng(P)
    try:
        batch_step(batch, members, None, "call 0")
        for m in members:
            commit(m, "call 0")
        plans = [(lambda i: i % 2 == 0), (lambda i: i % 2 == 1), (lambda i: True)]
        for call, gets_x in enumerate(plans, 1):
            xs = [m.x() if gets_x(i) else None for i, m in enumerate(members)]
            for m, x in zip(members, xs):
                if x is not None:
                    m.both("backup_points")
            batch_step(batch, members, xs, f"call {call}")
            accept = rng.random(len(members)) < 0.5
            accept[call % len(members)] = True
            accept[(call + 1) % len(members)] = False
            for m, ok in zip(members, accept):
                if ok:
                    commit(m, f"call {call}, accepted")
                else:
                    m.both("restore_points")
                    m.steps += 1
            if call == 1:   # one member steps on its own between two batch calls
                m = members[1]
                m.both("backup_points")
                single_step(m, m.x(), "single dmv_ba_gn_step between batch calls")
                commit(m, "single step")
    finally:
        batch.close()
        for m in members:
            m.close()


@pytest.mark.parametrize("P", [16, 32])
def test_members_reshaped_between_calls(capi, orc, synth, P):
    """between two calls of one BABatch: another nf (set_window), more points past a chunk boundary and fewer points (set_points on the
    same frames), dropped residuals, reset_oob, marginalised points; one member unchanged.  The batch must not keep a stale shape."""
    cfgs = [dict(nf=4, npts=333, seed=41), dict(nf=5, npts=300, seed=42), dict(nf=5, npts=700, seed=43), dict(nf=6, npts=900, seed=44, edge=True),
            dict(nf=4, npts=500, seed=45), dict(nf=7, npts=1200, seed=46), dict(nf=3, npts=333, seed=47, edge=True)]
    members = [Member(capi, orc, synth, c, P, max_points=1500, max_frames=8) for c in cfgs]
    batch = capi.BABatch([m.bt for m in members])
    rng = np.random.default_rng(7 + P)
    try:
        batch_step(batch, members, None, "call 1")
        for m in members:
            commit(m, "call 1")
        for m in members:
            m.both("backup_points")
        batch_step(batch, members, [m.x() for m in members], "call 2")
        for m in members:
            commit(m, "call 2")
        items0 = [_items(m.W, P) for m in members]
        m0, m1, m2, m3, m4, m5, _ = members
        m0.reload(nf=6)                              # set_window: another nf
        m1.reload(frames=False, npts=1000)           # more points on the same frames
        m2.reload(frames=False, npts=250)            # fewer points
        drop = np.sort(rng.choice(m3.bt.nres, m3.bt.nres // 7, replace=False)).astype(np.int32)
        m3.both("drop_residuals", drop)
        m4.both("reset_oob")
        nf5 = m5.W["nf"]
        marg = np.sort(rng.choice(len(m5.W["host"]), 240, replace=False)).astype(np.int32)
        m5.both("marginalize_points", marg, np.zeros((nf5 * nf5, 8), np.float32), np.zeros(4, np.float32))
        items1 = [_items(m.W, P) for m in members]
        assert m0.W["nf"] == 6 and items1[1] > items0[1] and items1[2] < items0[2]
        committed = [False, False, False, True, False, True, True]
        xs = [m.x() if c else None for m, c in zip(members, committed)]
        for m, x in zip(members, xs):
            if x is not None:
                m.both("backup_points")
        batch_step(batch, members, xs, "call 3, after the reshape")
        for m in members:
            commit(m, "call 3")
        for m in members:
            m.both("backup_points")
        batch_step(batch, members, [m.x() for m in members], "call 4")
    finally:
        batch.close()
        for m in members:
            m.close()


def _raw_step(capi, batch_h, xs, states):
    """dmv_ba_batch_gn_step with arbitrary (null) arguments: xs / states = None or a list of entries (None = a null entry)"""
    L = capi.lib()
    xarr = None if xs is None else (C.c_void_p * len(xs))(*[None if x is None else x.ctypes.data for x in xs])
    sarr = None if states is None else (C.c_void_p * len(states))(*[None if s is None else C.addressof(s) for s in states])
    return L.dmv_ba_batch_gn_step(batch_h, xarr, sarr, None, None)


def _refused(capi, rc, code, pattern):
    msg = capi.lib().dmv_last_error().decode()
    assert rc == code, f"rc {rc} ({msg}), expected {code}"
    assert re.search(pattern, msg), msg


def test_refusals_leave_members_untouched(capi, orc, synth, sms):
    """every argument dmv_ba_batch_create / dmv_ba_batch_gn_step refuse.  The states of the good members carry idepth / idepth_zero
    uploads, so a call that staged members before refusing a later one would show in get_idepth; after the refusals the next call
    is bit-identical to the twins."""
    P = 16
    cfgs = [dict(nf=3, npts=333, seed=7), dict(nf=4, npts=400, seed=9, edge=True), dict(nf=5, npts=250, seed=10)]
    members = [Member(capi, orc, synth, c, P) for c in cfgs]
    extra = []

    def handle(cfg, chunk_points=P, adjoints=True, points=True, max_points=None):
        W = make_case(synth, cfg)
        ow = orc.Window(W)
        ba = capi.BA(W["w"], W["h"], max_frames=W["nf"], max_points=max_points or len(W["host"]), chunk_points=chunk_points)
        extra.append(ba)
        if points:
            _fill(ba, W, ow)
            if not adjoints:   # set_window again: the handle keeps its points, loses its adjoints
                ba.set_window(W["nf"])
                ba.set_points(W["host"], W["u"], W["v"], W["idepth"], W["idepth_zero"], W["color"], W["weights"], priorF=prior_f(W))
                ba.set_residuals(W["res_point"], W["res_target"], W.get("res_state"), W.get("res_energy"))
        else:
            ba.set_window(W["nf"])
        return ba, W, ow

    batch = capi.BABatch([m.bt for m in members])
    batches = []
    try:
        batch_step(batch, members, None, "first call")
        for m in members:
            commit(m, "first call")
        xs = [m.x() for m in members]
        before = [m.bt.get_idepth() for m in members]

        def states(ms):
            """each member's state with idepth / idepth_zero uploads that differ from its current ones"""
            out = []
            for m, (idd, _) in zip(ms, before):
                out.append(m.bt._state(*m.st, idepth=idd * np.float32(1.01), idepth_zero=idd * np.float32(0.99)))
            return out

        def untouched(what):
            for i, (m, (idd, idz)) in enumerate(zip(members, before)):
                gi, gz = m.bt.get_idepth()
                np.testing.assert_array_equal(gi, idd, err_msg=f"{what}: member {i} idepth changed by a refused call")
                np.testing.assert_array_equal(gz, idz, err_msg=f"{what}: member {i} idepth_zero changed by a refused call")

        # ---- dmv_ba_batch_gn_step on the batch of the three members
        st = states(members)
        _refused(capi, _raw_step(capi, None, xs, st), DMV_ERR_INVALID, "null argument")
        _refused(capi, _raw_step(capi, batch.h, xs, None), DMV_ERR_INVALID, "null argument")
        untouched("null batch / null states")
        st = states(members)
        _refused(capi, _raw_step(capi, batch.h, xs, st[:2] + [None]), DMV_ERR_INVALID, "state 2 is null")
        untouched("null state of member 2")
        st = states(members)
        st[2].precalc = None
        _refused(capi, _raw_step(capi, batch.h, xs, st), DMV_ERR_INVALID, "state 2: precalc")
        untouched("member 2 without precalc")

        # ---- batches with one bad member behind two good ones
        def bad_batch(ba, W, ow, xbad, code, pattern, what):
            b = capi.BABatch([members[0].bt, members[1].bt, ba])
            batches.append(b)
            st = states(members[:2]) + [ba._state(ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"])]
            _refused(capi, _raw_step(capi, b.h, xs[:2] + [xbad], st), code, pattern)
            untouched(what)

        ba, W, ow = handle(dict(nf=3, npts=200, seed=12), adjoints=False)
        bad_batch(ba, W, ow, None, DMV_ERR_STATE, "window 2: dmv_ba_set_adjoints first", "member without adjoints")
        ba, W, ow = handle(dict(nf=3, npts=200, seed=13), points=False)
        bad_batch(ba, W, ow, None, DMV_ERR_STATE, "window 2: points not set", "member without points")
        ba, W, ow = handle(dict(nf=3, npts=200, seed=14))
        bad_batch(ba, W, ow, np.zeros(8 * 3 + 4), DMV_ERR_STATE, "window 2: no committed linearisation", "x without a committed linearisation")
        # chunk_points = 0: 16-point chunks when the batch is made, 32-point chunks once the window no longer fits one wave of them
        n32 = 16 * sms + 64
        ba, W, ow = handle(dict(nf=3, npts=200, seed=15), chunk_points=0, max_points=n32)
        W32 = make_case(synth, dict(nf=3, npts=n32, seed=15))
        b = capi.BABatch([members[0].bt, members[1].bt, ba])
        batches.append(b)
        ba.set_points(W32["host"], W32["u"], W32["v"], W32["idepth"], W32["idepth_zero"], W32["color"], W32["weights"], priorF=prior_f(W32))
        ba.set_residuals(W32["res_point"], W32["res_target"])
        ow32 = orc.Window(W32)
        st = states(members[:2]) + [ba._state(ow32.calib()["k8"], ow32.precalc(), ow32.frame_tables()["frameEnergyTH"])]
        _refused(capi, _raw_step(capi, b.h, xs[:2] + [None], st), DMV_ERR_STATE, "window 2 uses 32-point chunks, window 0 16")
        untouched("chunk_points = 0 member that resolved to 32-point chunks")

        # ---- dmv_ba_batch_create
        h32, _, _ = handle(dict(nf=3, npts=200, seed=16), chunk_points=32)
        with pytest.raises(capi.DmvError, match="share the device and chunk_points"):
            capi.BABatch([members[0].bt, h32])
        with pytest.raises(capi.DmvError, match="-1: 1..64 handles"):
            capi.BABatch([])
        with pytest.raises(capi.DmvError, match="-1: 1..64 handles"):
            capi.BABatch([members[0].bt] * (BATCH_MAX + 1))
        with pytest.raises(capi.DmvError, match=r"-1: handles\[0\] and handles\[2\] are the same handle"):
            capi.BABatch([members[0].bt, members[1].bt, members[0].bt])
        L = capi.lib()
        out = C.c_void_p()
        arr = (C.c_void_p * 2)(members[0].bt.h.value, None)
        _refused(capi, L.dmv_ba_batch_create(arr, 2, C.byref(out)), DMV_ERR_INVALID, "handle 1 is null")
        _refused(capi, L.dmv_ba_batch_create(None, 1, C.byref(out)), DMV_ERR_INVALID, "1..64 handles")
        assert not out.value
        untouched("refused dmv_ba_batch_create")

        # ---- after all of that: the next call on the members is bit-identical to the twins'
        for m in members:
            m.both("backup_points")
        batch_step(batch, members, xs, "first call after the refusals")
        for m in members:
            commit(m, "first call after the refusals")
    finally:
        for b in batches + [batch]:
            b.close()
        for ba in extra:
            ba.close()
        for m in members:
            m.close()


def _target_order(rp, rt, t):
    idx = np.nonzero(rt == t)[0]
    return idx[np.argsort(rp[idx], kind="stable")]


def check_target_energies(ba, rp, rt, nf, what):
    """dmv_ba_get_target_energies(t) == get_residual_outputs()["newEnergyWithOutlier"] of the residuals into t that are >= 0, in point
    order, for every target t.  Returns the newest frame's."""
    ewo = ba.residual_outputs()["newEnergyWithOutlier"]
    for t in range(nf):
        want = ewo[_target_order(rp, rt, t)]
        want = want[want >= 0]
        got = ba.target_energies(t)
        np.testing.assert_array_equal(got, want, err_msg=f"{what}: target {t}")
    return got


@pytest.mark.parametrize("P", [16, 32])
def test_target_energies(capi, orc, synth, P):
    """dmv_ba_get_target_energies reports the linearisation dmv_ba_get_residual_outputs reports, for every target (the newest frame's come
    from the kernel's pinned host copy while it belongs to that linearisation), in every state of a handle: after linearize, apply_res,
    gn_step(x) without apply, apply_res, gn_step(x) followed by marginalize_points (the committed linearisation again), drop_residuals;
    refused after reset_oob; and on every member after a batch call.  The newest frame's values also against the oracle."""
    m = Member(capi, orc, synth, dict(nf=6, npts=1500, seed=17, edge=True), P)
    others = [Member(capi, orc, synth, c, P) for c in (dict(nf=4, npts=500, seed=18), dict(nf=8, npts=300, seed=19, hosts="all", edge=True))]
    ba, W, ow = m.bt, m.W, m.ow
    nf = W["nf"]
    rp, rt = np.asarray(W["res_point"]), np.asarray(W["res_target"])
    try:
        ow.linearize_all(update_th=False)
        ba.set_state(*m.st)
        ba.linearize()
        newest = check_target_energies(ba, rp, rt, nf, "after linearize")
        g = ba.residual_outputs()
        _, _, unfixable = ow.override_new_states(g["newState"])
        assert unfixable == 0
        o = ow.res_outputs(False)["newEnergyWithOutlier"][_target_order(rp, rt, nf - 1)]
        o = o[o >= 0]
        assert len(o) == len(newest) and len(o) > 100
        np.testing.assert_allclose(newest, o, rtol=2e-3, atol=0.05, err_msg="newest frame vs the oracle's newEnergyWithOutlier")
        ba.apply_res()
        check_target_energies(ba, rp, rt, nf, "after apply_res")
        m.a = ba.accumulate()
        ba.backup_points()
        ba.gn_step(m.x(), *m.st)
        check_target_energies(ba, rp, rt, nf, "after gn_step(x), not applied")
        ba.apply_res()
        check_target_energies(ba, rp, rt, nf, "after apply_res of the step")
        committed = ba.target_energies(nf - 1)
        m.a = ba.accumulate()
        m.steps = 1
        ba.backup_points()
        ba.gn_step(m.x(), *m.st)
        tentative = ba.target_energies(nf - 1)
        assert not np.array_equal(tentative, committed), "the step must change the newest frame's energies, or the next check is blunt"
        marg = np.sort(np.random.default_rng(P).choice(len(W["host"]), 300, replace=False)).astype(np.int32)
        ba.marginalize_points(marg, np.zeros((nf * nf, 8), np.float32), np.zeros(4, np.float32))
        newest = check_target_energies(ba, rp, rt, nf, "after gn_step(x) + marginalize_points")
        np.testing.assert_array_equal(newest, committed, err_msg="after marginalize_points: the committed linearisation")
        drop = np.sort(np.random.default_rng(P + 1).choice(len(rp), len(rp) // 5, replace=False)).astype(np.int32)
        ba.drop_residuals(drop)
        rp, rt = np.delete(rp, drop), np.delete(rt, drop)
        check_target_energies(ba, rp, rt, nf, "after drop_residuals")
        ba.reset_oob()
        for t in (0, nf - 1):
            with pytest.raises(capi.DmvError, match="linearize first"):
                ba.target_energies(t)
        # ---- batch members (the first one in the state reset_oob left)
        members = [m] + others
        batch = capi.BABatch([q.bt for q in members])
        try:
            for call in range(2):
                xs = [None] * len(members) if call == 0 else [q.x() for q in members]
                batch.gn_step(xs, [q.st for q in members])
                for i, q in enumerate(members):
                    qrp, qrt = (rp, rt) if q is m else (np.asarray(q.W["res_point"]), np.asarray(q.W["res_target"]))
                    check_target_energies(q.bt, qrp, qrt, q.W["nf"], f"batch call {call}, member {i}")
                    q.bt.apply_res()
                    q.a = q.bt.accumulate()
                    q.bt.backup_points()
        finally:
            batch.close()
    finally:
        for q in [m] + others:
            q.close()

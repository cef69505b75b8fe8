"""GPU tier of dmv_ba_select_activation: the device's actions, toOptimize order and distance map against the CPU restatement of
activatePointsMT's selection (oracle/orc_activation.cpp, itself pinned to the reference by tests/test_ref_pin_activation.py) and against the
golden fixture made from the reference.  Bit equality throughout."""
import os

import numpy as np
import pytest

import dmvio_b200.capi as capi
import dmvio_b200.synth as synth
from oracle import activation as A
from oracle import orc

from helpers import product_ba_from_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_activation.npz")


def _select(ba, case, tab, **kw):
    return ba.select_activation(case["nf"], case["newest"], tab, case["flagged"], case["act_u"], case["act_v"], case["act_id"], case["act_host"],
                                case["off"], case["imm"], case["min_act_dist"], A.MIN_TRACE_QUALITY, **kw)


def _check(case, tab=None, ba=None):
    tab = A.tables(case) if tab is None else tab
    own = ba is None
    ba = ba or capi.BA(case["w"], case["h"], max_frames=8, max_points=64)
    try:
        act, opt, m, st = _select(ba, case, tab)
        act2, opt2, _, st2 = _select(ba, case, tab, want_map=False)   # floods no decision reads are skipped: same decisions
    finally:
        if own:
            ba.close()
    a, o, mm = A.restate(case, tab)
    assert np.array_equal(act, a), np.argwhere(act != a)[:5]
    assert np.array_equal(opt, o)
    assert np.array_equal(m.reshape(-1), mm), np.argwhere(m.reshape(-1) != mm)[:5]
    assert np.array_equal(act2, a) and np.array_equal(opt2, o)
    assert st["floods"] == len(o) and st2["floods"] <= len(o) and st["undecided"] == st2["undecided"] <= len(o) + np.sum(a == A.KEEP)
    if case["min_act_dist"] == 0:   # every candidate decided before the loop, no flood needed without the map
        assert st2["undecided"] == 0 and st2["floods"] == 0
    return act, opt, m


@pytest.mark.parametrize("name", sorted(A.CASES))
def test_golden_cases(name):
    G = np.load(GOLDEN)
    act, opt, m = _check(A.make_case(**A.CASES[name]), G[f"{name}/tab"])
    assert np.array_equal(act, G[f"{name}/action"]) and np.array_equal(opt, G[f"{name}/opt"]) and np.array_equal(m.reshape(-1), G[f"{name}/map"])


@pytest.mark.parametrize("wh", [(640, 480), (512, 512), (752, 480), (1280, 720)])
@pytest.mark.parametrize("mad", [0.0, 2.0, 4.0])
def test_c3_window(wh, mad):
    _check(A.make_case(w=wh[0], h=wh[1], nf=7, n_active=2000 * 6, n_imm=1500, seed=wh[0] + int(mad), min_act_dist=mad))


@pytest.mark.parametrize("wh", [(640, 480), (1280, 720)])
def test_first_keyframes(wh):
    _check(A.make_case(w=wh[0], h=wh[1], nf=2, n_active=40, n_imm=3000, seed=5, min_act_dist=0.0, flagged=()))


@pytest.mark.parametrize("mad", [1.0, 4.0])
def test_one_small_region(mad):
    """every candidate in one small block of cells: the longest chain of dependent decisions"""
    _check(A.make_case(w=640, h=480, nf=2, n_active=100, imm_counts=(4000, 0), seed=6, min_act_dist=mad, cluster=(100, 80, 4), flagged=()))


@pytest.mark.parametrize("count", [0, 1, 31, 32, 33, 20000])
def test_candidate_counts(count):
    case = A.make_case(w=640, h=480, nf=3, n_active=500, imm_counts=(count, 0, 7), seed=count, min_act_dist=1.0, flagged=())
    for k in ("status", "interval", "quality"):   # every point of frame 0 a candidate
        case["imm"][k][:count] = {"status": 0, "interval": 1.0, "quality": 10.0}[k]
    case["imm"]["idepth_max"][:count] = case["imm"]["idepth_min"][:count]
    act, opt, _ = _check(case)
    assert np.all(act[int(case["off"][2]):] == A.KEEP)   # the newest frame's points are skipped
    assert count == 0 or len(opt) > 0


def test_capacity_arguments_and_repeat():
    case = A.make_case(w=640, h=480, seed=9, min_act_dist=2.0)
    tab = A.tables(case)
    ba = capi.BA(640, 480, max_frames=8, max_points=64)
    try:
        a1, o1, m1, _ = _select(ba, case, tab)
        a2, o2, m2, _ = _select(ba, case, tab)
        assert np.array_equal(a1, a2) and np.array_equal(o1, o2) and np.array_equal(m1, m2)
        with pytest.raises(capi.DmvError) as e:
            _select(ba, case, tab, cap=len(o1) - 1)
        assert e.value.args[1] == len(o1)
        a3, o3, _, _ = _select(ba, case, tab, cap=len(o1), want_map=False)
        assert np.array_equal(a3, a1) and np.array_equal(o3, o1)
        bad_off = case["off"].copy()
        bad_off[2] = bad_off[1] - 1
        for kw in (dict(nf=0), dict(nf=9), dict(newest=7), dict(off=bad_off)):
            c = dict(case, **{k: v for k, v in kw.items() if k in ("off",)})
            nf = kw.get("nf", case["nf"])
            with pytest.raises(capi.DmvError):
                ba.select_activation(nf, kw.get("newest", case["newest"]), np.zeros(12 * max(nf, 1), np.float32), np.zeros(max(nf, 1), np.uint8),
                                     case["act_u"], case["act_v"], case["act_id"], case["act_host"], c["off"][:max(nf, 1) + 1], case["imm"], 2.0)
        host = case["act_host"].copy()
        host[3] = 7
        with pytest.raises(capi.DmvError):
            ba.select_activation(7, 6, tab, case["flagged"], case["act_u"], case["act_v"], case["act_id"], host, case["off"], case["imm"], 2.0)
        a4, o4, m4, _ = _select(ba, case, tab)   # an error leaves nothing behind
        assert np.array_equal(a4, a1) and np.array_equal(o4, o1) and np.array_equal(m4, m1)
    finally:
        ba.close()


def test_ba_state_untouched():
    """a dmv_ba_gn_step (resubstitution, point step, linearisation) after the call is bit-identical to one without it"""
    import dmvio_b200.hostmath as hm
    W = synth.make_window(nf=4, npts=600, seed=3)
    outs = []
    for call in (False, True):
        ow = orc.Window(W)
        ba = product_ba_from_oracle(capi, W, ow)
        tabs = (ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"])
        ba.linearize()
        ba.apply_res()
        a = ba.accumulate()
        x = hm.solve_reduced(a["HA"], a["bA"], a["Hsc"], a["bsc"], *hm.prior_system(W), lam=1e-5)
        if call:
            _check(A.make_case(w=W["w"], h=W["h"], nf=4, n_active=300, n_imm=200, seed=4, min_act_dist=1.0), ba=ba)
        r = ba.gn_step(x, *tabs)
        ba.apply_res()
        acc = ba.accumulate()
        outs.append((r["energy"], r["n_in"], np.array(r["sums"]), ba.get_idepth()[0].copy(), {k: np.array(acc[k]) for k in ("HA", "bA", "Hsc", "bsc")}))
        ba.close()
    assert outs[0][0] == outs[1][0] and outs[0][1] == outs[1][1]
    assert np.array_equal(outs[0][2], outs[1][2]) and np.array_equal(outs[0][3], outs[1][3])
    for k in outs[0][4]:
        assert np.array_equal(outs[0][4][k], outs[1][4][k]), k


def test_select_then_activate_equals_the_oracle():
    """dmv_ba_select_activation's toOptimize fed to dmv_ba_activate_points equals the oracle's whole activatePointsMT: the restatement's
    selection followed by its optimizeImmaturePoint on the same points, in the same order"""
    from helpers import activation_case
    W, host, P = activation_case(synth, orc)
    nf = W["nf"]
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    fx, fy, cx, cy = [float(v) for v in ow.calib()["k8"][:4]]
    K0 = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    K1 = np.array([[fx * 0.5, 0, (cx + 0.5) / 2 - 0.5], [0, fy * 0.5, (cy + 0.5) / 2 - 0.5], [0, 0, 1]])
    RT = ow.RT().reshape(nf, nf, 12)
    tab = np.zeros((nf, 12), np.float32)
    for f in range(nf):   # host f -> newest frame, level 0 -> level 1
        tab[f, :9] = (K1 @ RT[f, nf - 1, :9].reshape(3, 3).astype(np.float64) @ np.linalg.inv(K0)).astype(np.float32).reshape(-1)
        tab[f, 9:] = (K1 @ RT[f, nf - 1, 9:].astype(np.float64)).astype(np.float32)
    n = len(host)
    rng = np.random.default_rng(2)
    imm = dict(u=P["u"].astype(np.float32), v=P["v"].astype(np.float32), idepth_min=P["idepth_min"], idepth_max=P["idepth_max"],
               status=rng.choice([0, 3, 4], n).astype(np.int32), interval=np.ones(n, np.float32), quality=np.full(n, 10, np.float32),
               type=rng.choice([1.0, 2.0], n).astype(np.float32))
    off = np.concatenate([[0], np.cumsum(np.bincount(host, minlength=nf))]).astype(np.int32)
    case = dict(w=W["w"], h=W["h"], nf=nf, newest=nf - 1, flagged=np.zeros(nf, np.uint8), act_u=W["u"].astype(np.float32), act_v=W["v"].astype(np.float32),
                act_id=W["idepth"].astype(np.float32), act_host=W["host"].astype(np.int32), off=off, imm=imm, min_act_dist=1.0)
    act, opt, _ = _check(case, tab, ba=ba)
    assert 0 < len(opt) < n
    sub = {k: P[k][opt] for k in P}
    s_g, i_g, r_g = ba.activate_points(host[opt], sub, ow.RT())
    aff = ow.precalc()[:, 24:26].copy()
    s_o, i_o, r_o = orc.ip_activate(W, ow.RT(), aff, ow.calib()["k8"][:6], host[opt], sub)
    np.testing.assert_array_equal(s_g, s_o)
    np.testing.assert_array_equal(i_g, i_o)
    np.testing.assert_array_equal(r_g, r_o)
    assert (s_o == 1).sum() > 0
    ba.close()

"""The device kernels off DSO's default settings: dmv_ba_set_params (huberTH, outlierTHSumComponent, affineOptModeA / B) in the single-window,
fused-step, marginalisation, batched and activation launches, dmv_ct_set_huber and affine mode 0 in the coarse tracker, the coarse
initialiser's huberTH, and the host adapter's settings.  Ground truth is the oracle at the same settings, pinned to the reference there by
tests/test_ref_pin_settings.py, or the fp64 references of helpers.py.

Where a setting's effect is exact it is checked exactly.  affineOptMode < 0 zeroes JabF but keeps JabJIdx and Jab2 (Residuals.cpp:L229-242),
so every output of the launch equals the default launch's bit for bit except b_A's affine row of the fixed parameter, which is exactly 0.
Every other setting must change the launch's outputs against the defaults, so a kernel that ignored it would fail."""
import ctypes as C
import inspect

import numpy as np
import pytest

import dmvio_b200.hostmath as hm
import helpers as H
from gpu_harness import CONFIGS as CT_CONFIGS, assert_same, bits, capi, close, ct_handle, ct_scene, gpu, near_truth_tries, set_cluster, \
    track_kw, tries_kw  # noqa: F401
from helpers import EPS32, check_linearize_parity, check_phase_b, make_case, points_with_in_residual, prior_f, product_ba_from_oracle, \
    schur_reference
from test_gpu_ba import CONFIGS, _batched_vs_single_launches, cfg_id
from test_gpu_ba_system import TPB, check_bound
from test_gpu_marg import _case as marg_case, marginalize_parity

AFF_SETS = dict(A=dict(affineOptModeA=-1.0), B=dict(affineOptModeB=-1.0), AB=dict(affineOptModeA=-1.0, affineOptModeB=-1.0))
TH_SETS = [dict(huberTH=4.0), dict(huberTH=30.0), dict(huberTH=1e6), dict(outlierTHSumComponent=100.0), dict(outlierTHSumComponent=1e6)]


def sid(s):
    return "_".join(f"{k}{v:g}" for k, v in s.items())


def aff_rows(nf, s):
    """the system rows of the affine parameters s fixes: a (6) and / or b (7) of every frame"""
    return np.array([4 + 8 * f + j for f in range(nf) for j, k in ((6, "affineOptModeA"), (7, "affineOptModeB")) if k in s], np.int64)


def state_of(ow):
    return ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"]


def launch(ba, x, st):
    """one fused launch (x None: the first linearisation), committed and accumulated: every output it leaves on the device"""
    r = ba.gn_step(x, *st)
    g = ba.residual_outputs()
    ba.apply_res()
    return dict(r=r, g=g, a=ba.accumulate(), p=ba.point_outputs(), idepth=ba.get_idepth()[0])


def eq(a, b, what):
    assert np.array_equal(bits(a), bits(b)), what


def check_affine_identity(o, o0, rows, what):
    """o (affine parameters fixed) against o0 (defaults): everything bit-identical but b_A's rows `rows`, which are exactly 0 (and are not 0
    at the defaults wherever the frame's affine parameter is observed)"""
    for k in ("energy", "n_in", "n_oob", "n_outlier"):
        assert o["r"][k] == o0["r"][k], (what, k)
    if "sums" in o0["r"]:
        eq(o["r"]["sums"], o0["r"]["sums"], f"{what}: resubstitution sums")
    for k in ("newState", "newEnergy", "newEnergyWithOutlier", "centerProjectedTo"):
        eq(o["g"][k], o0["g"][k], f"{what}: {k}")
    inn = o0["g"]["newState"] == H.RES_IN   # JpJdF is defined for IN residuals only
    eq(o["g"]["JpJdF"][inn], o0["g"]["JpJdF"][inn], f"{what}: JpJdF")
    for k in ("Hdd", "bd", "Hcd", "HdiF", "bdSumF"):
        eq(o["p"][k], o0["p"][k], f"{what}: {k}")
    for k in ("HA", "Hsc", "bsc"):
        eq(o["a"][k], o0["a"][k], f"{what}: {k}")
    assert o["a"]["resInA"] == o0["a"]["resInA"], what
    eq(o["idepth"], o0["idepth"], f"{what}: idepth")
    bA, bA0 = o["a"]["bA"], o0["a"]["bA"]
    others = np.setdiff1d(np.arange(len(bA)), rows)
    eq(bA[others], bA0[others], f"{what}: b_A outside the fixed affine rows")
    assert not bA[rows].any(), f"{what}: b_A's fixed affine rows are not 0"
    seen = np.diag(o0["a"]["HA"])[rows] > 0
    assert seen.any() and np.all(bA0[rows][seen] != 0), f"{what}: b_A's affine rows are 0 at the defaults too: the check is blunt"


# ---------------------------------------------------------------------------------------------------------------------------------
# (a) affine modes: exact identities
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
@pytest.mark.parametrize("P", [16, 32])
def test_affine_modes_exact(capi, gpu, orc, synth, cfg, P):
    """first linearisation and a fused GN step at the same x, affineOptModeA = -1, then B, then both, against the default launch"""
    W = make_case(synth, cfg)
    ow = orc.Window(W)
    st = state_of(ow)
    base = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    o0 = launch(base, None, st)
    HL, bL = hm.prior_system(W)
    x = hm.solve_reduced(o0["a"]["HA"], o0["a"]["bA"], o0["a"]["Hsc"], o0["a"]["bsc"], HL, bL, lam=1e-5)
    base.backup_points()
    o0x = launch(base, x, st)
    assert not np.array_equal(o0x["idepth"], W["idepth"])
    base.close()
    for name, s in AFF_SETS.items():
        rows = aff_rows(W["nf"], s)
        ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
        ba.set_params(**s)
        check_affine_identity(launch(ba, None, st), o0, rows, f"{name} first linearisation")
        ba.backup_points()
        check_affine_identity(launch(ba, x, st), o0x, rows, f"{name} fused step")
        ba.close()


MARG_CFGS = [(dict(nf=7, npts=2000, seed=1234), 0.33), (dict(nf=8, npts=777, seed=99, hosts="all"), 0.1)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,frac", MARG_CFGS, ids=lambda c: cfg_id(c) if isinstance(c, dict) else f"{c:g}")
@pytest.mark.parametrize("P", [16, 32])
def test_affine_modes_marginalization(capi, gpu, orc, synth, cfg, frac, P):
    """dmv_ba_marginalize_points with the affine modes at -1.  Deltas with affine components 0: bit-identical to the default launch but
    Mb's fixed affine rows, which are 0.  Full deltas (res_toZeroF loses jaF dp6 / jbF dp7): M and Msc bit-identical to the default, Mb and
    Mbsc against the oracle at the same settings (test_gpu_marg.py's bounds)."""
    W, pts = marg_case(synth, orc, cfg, frac)
    nf = W["nf"]
    ow = orc.Window(W)
    ad = np.asarray(ow.adHTdeltaF(), np.float32).reshape(nf * nf, 8)
    ad0 = ad.copy()
    ad0[:, 6:] = 0
    cD = ow.calib()["cDeltaF"]

    def marg(prm):
        ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
        ba.set_params(**prm)
        ba.linearize(); ba.apply_res()
        z, f = ba.marginalize_points(pts, ad0, cD), ba.marginalize_points(pts, ad, cD)
        ba.close()
        return z, f

    z0, f0 = marg({})
    for name, s in AFF_SETS.items():
        rows = aff_rows(nf, s)
        z, f = marg(s)
        for k in ("M", "Msc", "Mbsc", "ngood", "isLinearized", "rtz"):
            eq(z[k], z0[k], f"{name} zero affine deltas: {k}")
        assert z["resInM"] == z0["resInM"]
        others = np.setdiff1d(np.arange(len(z["Mb"])), rows)
        eq(z["Mb"][others], z0["Mb"][others], f"{name}: Mb outside the fixed affine rows")
        assert not z["Mb"][rows].any(), f"{name}: Mb's fixed affine rows are not 0"
        seen = np.diag(z0["M"])[rows] > 0
        assert seen.any() and np.all(z0["Mb"][rows][seen] != 0)
        for k in ("M", "Msc"):
            eq(f[k], f0[k], f"{name} full deltas: {k}")
        assert not np.array_equal(f["Mb"], f0["Mb"]), f"{name}: the affine deltas do not reach res_toZeroF"
        g = marginalize_parity(capi, orc, synth, cfg, frac, P, settings=s)
        for k in ("M", "Mb", "Msc", "Mbsc"):
            eq(g[k], f[k], f"{name}: marginalize_parity's launch != this one: {k}")


# ---------------------------------------------------------------------------------------------------------------------------------
# (b) huberTH and outlierTHSumComponent against the oracle at the same settings
# ---------------------------------------------------------------------------------------------------------------------------------
TH_CFGS = [dict(nf=7, npts=2000, seed=1234, edge=True), dict(nf=3, npts=333, seed=7)]
_DEFAULT_MARG = {}


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", TH_CFGS, ids=cfg_id)
@pytest.mark.parametrize("P", [16, 32])
@pytest.mark.parametrize("s", TH_SETS, ids=sid)
def test_thresholds_against_oracle(capi, gpu, orc, synth, cfg, P, s):
    """check_linearize_parity against orc.Window(W, settings=s), phase B in closed form, the Schur system within
    test_gpu_ba_system.py::test_schur_against_fp64's fp64 bound, and outputs that differ from the default launch's"""
    W = make_case(synth, cfg)
    ow = orc.Window(W, settings=s)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    ba.set_params(**s)
    E_o = ow.linearize_all(update_th=False)
    r = ba.linearize()
    g, pg, a = check_linearize_parity(ow, ba, r, E_o)
    npts = len(W["host"])
    check_phase_b(pg, points_with_in_residual(W["res_point"], g["newState"], npts), prior_f(W), W["idepth"], W["idepth_zero"])
    gc = ba.residual_outputs()
    adH, adT = ow.adjoints()
    Hsc, bsc, Habs, babs = schur_reference(W, gc["newState"], gc["JpJdF"], pg["Hcd"], pg["HdiF"], pg["bdSumF"], adH, adT)
    gamma = (-(-npts // TPB[P]) + 38) / 2
    check_bound(a["Hsc"], Hsc, gamma * EPS32 * Habs, "H_sc")
    check_bound(a["bsc"], bsc, gamma * EPS32 * babs, "b_sc")
    ba.close()
    d = product_ba_from_oracle(capi, W, orc.Window(W), chunk_points=P)
    r0 = d.linearize()
    g0 = d.residual_outputs()
    d.close()
    assert r0["energy"] != r["energy"] and not np.array_equal(g0["newEnergy"], g["newEnergy"]), f"{s} does not reach the launch"


@pytest.mark.gpu
@pytest.mark.parametrize("P", [16, 32])
@pytest.mark.parametrize("s", TH_SETS, ids=sid)
def test_thresholds_marginalization(capi, gpu, orc, synth, P, s):
    """dmv_ba_marginalize_points against ow.marginalize at the same settings (test_gpu_marg.py's tolerances), and a different system from
    the default launch's"""
    cfg, frac = dict(nf=7, npts=2000, seed=1234), 0.33
    g = marginalize_parity(capi, orc, synth, cfg, frac, P, settings=s)
    if P not in _DEFAULT_MARG:
        _DEFAULT_MARG[P] = marginalize_parity(capi, orc, synth, cfg, frac, P)
    g0 = _DEFAULT_MARG[P]
    assert not np.array_equal(g["Mb"], g0["Mb"]), f"{s} does not reach the marginalisation launch"


# ---------------------------------------------------------------------------------------------------------------------------------
# (c) the set_params contract
# ---------------------------------------------------------------------------------------------------------------------------------
def _run(ba, st):
    """one launch as test_gpu_ba.py::test_run_to_run_bit_reproducible repeats it: first linearisation, commit, accumulate, resetOOB"""
    o = launch(ba, None, st)
    ba.reset_oob()
    return o


def _same_run(o, o0, what):
    for k in ("energy", "n_in", "n_oob", "n_outlier"):
        assert o["r"][k] == o0["r"][k], (what, k)
    for part, keys in (("g", ("newState", "newEnergy", "newEnergyWithOutlier")), ("p", ("Hdd", "bd", "HdiF", "bdSumF")), ("a", ("HA", "bA", "Hsc", "bsc"))):
        for k in keys:
            eq(o[part][k], o0[part][k], f"{what}: {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("P", [16, 32])
def test_set_params_contract(capi, gpu, orc, synth, P):
    """a set_params between launches takes effect on the next launch without any re-upload (the same outputs as a handle that had the
    parameters before its first launch); back at the defaults the outputs are the default ones bit for bit; dmv_ba_set_params(NULL) is
    refused with DMV_ERR_INVALID and changes nothing"""
    W = synth.make_window(nf=7, npts=2000, seed=1234)
    ow = orc.Window(W)
    st = state_of(ow)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    o_def = _run(ba, st)
    for s in (dict(huberTH=4.0), dict(outlierTHSumComponent=100.0), dict(affineOptModeA=-1.0, affineOptModeB=-1.0)):
        ba.set_params(**s)
        o = _run(ba, st)
        fresh = product_ba_from_oracle(capi, W, ow, chunk_points=P)
        fresh.set_params(**s)
        _same_run(o, _run(fresh, st), f"{s}: set between launches vs before the first")
        fresh.close()
        assert not np.array_equal(o["a"]["bA"], o_def["a"]["bA"]), s
        ba.set_params()
        _same_run(_run(ba, st), o_def, f"back to the defaults after {s}")
    ba.set_params(huberTH=4.0)
    ba.set_params()
    assert capi.lib().dmv_ba_set_params(ba.h, None) == capi.DMV_ERR_INVALID
    _same_run(_run(ba, st), o_def, "after set_params(NULL)")
    ba.close()


def test_default_params(capi, orc, synth):
    """dmv_ba_default_params (the parameters a new handle starts with) = BA.set_params's defaults = the oracle's Settings"""
    p = capi.BAParams()
    capi.lib().dmv_ba_default_params(C.byref(p))
    sig = inspect.signature(capi.BA.set_params).parameters
    dflt = {k: sig[k].default for k in ("huberTH", "outlierTHSumComponent", "affineOptModeA", "affineOptModeB")}
    for k, v in dflt.items():
        assert getattr(p, k) == np.float32(v), k
    W = synth.make_window(nf=3, npts=200, seed=5)
    a, b = orc.Window(W), orc.Window(W, settings=dflt)
    assert a.linearize_all(update_th=False) == b.linearize_all(update_th=False)
    ra, rb = a.res_outputs(True), b.res_outputs(True)
    for k in ra:
        np.testing.assert_array_equal(ra[k], rb[k], err_msg=k)


# ---------------------------------------------------------------------------------------------------------------------------------
# (d) the batched launch: one descriptor per member
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("P", [16, 32])
def test_batch_members_keep_their_params(capi, gpu, orc, synth, P):
    """four members at the defaults, affineOptModeA = -1, huberTH = 4 and outlierTHSumComponent = 100 in one dmv_ba_batch_gn_step: each
    bit-identical to its own single launch, first linearisation and fused step"""
    _batched_vs_single_launches(capi, orc, synth, P, params=[{}, dict(affineOptModeA=-1.0), dict(huberTH=4.0), dict(outlierTHSumComponent=100.0)])


# ---------------------------------------------------------------------------------------------------------------------------------
# (e) point activation
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_activate_points_huber(capi, gpu, orc, synth):
    """dmv_ba_activate_points after set_params(huberTH = h) against orc.ip_activate(huberTH = h), bit for bit, and not the h = 9 result"""
    W, host, P = H.activation_case(synth, orc)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    aff, calib6 = ow.precalc()[:, 24:26].copy(), ow.calib()["k8"][:6]
    for minObs in (1, 3):
        s9, i9, _ = ba.activate_points(host, P, ow.RT(), minObs=minObs)
        for h in (4.0, 30.0):
            ba.set_params(huberTH=h)
            s_g, i_g, r_g = ba.activate_points(host, P, ow.RT(), minObs=minObs)
            s_o, i_o, r_o = orc.ip_activate(W, ow.RT(), aff, calib6, host, P, minObs=minObs, huberTH=h)
            np.testing.assert_array_equal(s_g, s_o)
            eq(i_g, i_o, f"huberTH {h} minObs {minObs}: idepth")
            np.testing.assert_array_equal(r_g, r_o)
            assert (i_g != i9).sum() > len(i9) // 10, h
            ba.set_params()
    ba.close()


@pytest.mark.gpu
def test_activate_store_huber(capi, gpu, orc, synth):
    """dmv_ba_activate_store after set_params(huberTH = h) on both handles of test_gpu_activate_store.py's twin set-up: the call against its
    five steps, and its optimised points against orc.ip_activate(huberTH = h) on the same points; h = 4 and 30 against h = 9"""
    from test_gpu_activate_store import Win
    slot = [0, 1, 2, 3, 4, 5, -1]
    out = {}
    for h in (9.0, 4.0, 30.0):
        win = Win(capi, synth, orc, 321)
        for b in win.bas:
            b.set_params(huberTH=h)
        for f, k in enumerate(slot):
            if k >= 0:
                P = win.points(f, 300)
                P["status"][:] = 0                      # GOOD, traced once: candidates for activation
                P["lastTracePixelInterval"][:] = 1.0
                P["quality"][:] = 10.0
                win.put(k, P, f)
        before = {k: dict(v) for k, v in win.copies.items()}
        r, _ = win.turnover(slot, mad=2.0, what=f"huberTH {h}")
        n = len(r["opt_frame"])
        assert n > 0
        sub = {key: np.stack([before[slot[f]][key][i] for f, i in zip(r["opt_frame"], r["opt_index"])])
               for key in ("u", "v", "color", "weights", "energyTH", "idepth_min", "idepth_max")}
        aff, calib6 = win.ow.precalc()[:, 24:26].copy(), win.ow.calib()["k8"][:6]
        s_o, i_o, r_o = orc.ip_activate(win.W, win.RT, aff, calib6, r["opt_frame"], sub, huberTH=h)
        np.testing.assert_array_equal(r["status"], s_o)
        eq(r["idepth"], i_o, f"huberTH {h}: idepth")
        np.testing.assert_array_equal(r["res_state"], r_o)
        out[h] = r
        win.close()
    for h in (4.0, 30.0):
        eq(out[h]["opt_index"], out[9.0]["opt_index"], "the selection does not read huberTH")
        assert (out[h]["idepth"] != out[9.0]["idepth"]).sum() > len(out[h]["idepth"]) // 10, h


# ---------------------------------------------------------------------------------------------------------------------------------
# (f) the coarse tracker: dmv_ct_set_huber and affine mode 0
# ---------------------------------------------------------------------------------------------------------------------------------
_CT_REF = {}


def ct_ref(sc, **kw):
    key = (sc["name"], sc.get("huber", 9.0), tuple(sorted(kw.items())))
    if key not in _CT_REF:
        _CT_REF[key] = H.ct_track_ref(sc, **kw)
    return _CT_REF[key]


def huber_scene(orc, synth, name, huber):
    return dict(ct_scene(orc, synth, name), huber=huber)


def check_final_linearisation(sc, r, rep):
    """lastResiduals[0] and flow against calc_res_ref at the kernel's own pose, the level-0 cutoff repeat rep and the scene's Huber threshold"""
    a = sc["args"]
    aa = a["a0"] if a["affA"] < 0 else r["a"]
    bb = a["b0"] if a["affB"] < 0 else r["b"]
    RKi, tf, affLL = H.ct_operands(r["R"], r["t"], aa, bb, sc["Ki"][0], a["ref_a"], a["ref_b"], a["ref_exposure"], a["new_exposure"])
    c = H.calc_res_ref(sc["pts"][0], sc["planes"][0], sc["k4"][0], sc["Ki"][0], RKi, tf, affLL, a["ref_b"], np.float32(20) * np.float32(rep), 0,
                       huber=sc["huber"],
                       R=r["R"])
    m_ref = c["E"] / c["nE"]
    err = abs(float(r["lastResiduals"][0]) ** 2 - m_ref)
    assert err <= m_ref * H.ct_mean_bound(c) + 4 * H.U32 * m_ref, (r["lastResiduals"][0] ** 2, m_ref)
    for j, k in ((0, 2), (1, 4)):
        assert abs(r["flow"][2 * j] - c["res6"][k]) <= c["dflow"][j], (j, r["flow"], c["res6"], c["dflow"])


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CT_CONFIGS)
@pytest.mark.parametrize("huber", [4.0, 30.0])
@pytest.mark.parametrize("name", ["bench", "aff_free"])
def test_ct_track_huber(capi, gpu, orc, synth, monkeypatch, cfg, huber, name):
    """dmv_ct_track after dmv_ct_set_huber(h) against track_ref at h: the final linearisation within calc_res_ref's bound at the kernel's
    pose, the decision and the pose of the fp64 loop.  The iteration counts are not compared: at h = 30 an accept tie at the end of a level
    makes the fp64 loop and the fp32 oracle stop after different counts at the same pose (1e-8 apart)."""
    sc = huber_scene(orc, synth, name, huber)
    rr = ct_ref(sc)
    set_cluster(monkeypatch, cfg)
    g = ct_handle(capi, sc)
    g.set_huber(huber)
    r = g.track(**track_kw(sc))
    check_final_linearisation(sc, r, [e["rep"] for e in rr["log"] if e["lvl"] == 0][-1])
    assert r["good"] == rr["good"] and r["status"] == rr["status"] == 0
    assert np.abs(r["R"] - rr["R"]).max() < 1e-6 and np.abs(r["t"] - rr["t"]).max() < 1e-6, (r["R"] - rr["R"], r["t"] - rr["t"])
    assert abs(r["a"] - rr["a"]) < 1e-6 and abs(r["b"] - rr["b"]) < 1e-6 * 1000
    g.set_huber(9.0)
    r9 = g.track(**track_kw(sc))
    assert r9["lastResiduals"][0] != r["lastResiduals"][0]
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("huber", [4.0, 30.0])
def test_ct_calc_res_gs_huber(capi, gpu, orc, synth, monkeypatch, huber):
    """dmv_ct_calc_res_gs after dmv_ct_set_huber(h) at every pose track_ref logs, within calc_res_ref(huber = h)'s bound"""
    sc = huber_scene(orc, synth, "bench", huber)
    rr = ct_ref(sc)
    set_cluster(monkeypatch, "nc16")
    g = ct_handle(capi, sc)
    g.set_huber(huber)
    a = sc["args"]
    changed = 0
    for e in rr["log"]:
        l = e["lvl"]
        RKi, tf, affLL = H.ct_operands(e["R"], e["t"], e["a"], e["b"], sc["Ki"][l], a["ref_a"], a["ref_b"], a["ref_exposure"], a["new_exposure"])
        cut = np.float32(20) * np.float32(e["rep"])
        c = H.calc_res_ref(sc["pts"][l], sc["planes"][l], sc["k4"][l], sc["Ki"][l], RKi, tf, affLL, a["ref_b"], cut, l, huber=huber)
        r6, Hg, bg, npad = g.calc_res_gs(l, RKi, tf, affLL, float(np.float32(a["ref_b"])), float(cut), True)
        assert abs(r6[1] - c["nE"]) <= c["amb"]
        assert abs(r6[0] - c["E"]) <= c["dE"], (l, r6[0], c["E"], c["dE"])
        assert (np.abs(Hg - c["H"]) <= c["dH"]).all() and (np.abs(bg - c["b"]) <= c["db"]).all(), l
        c9 = H.calc_res_ref(sc["pts"][l], sc["planes"][l], sc["k4"][l], sc["Ki"][l], RKi, tf, affLL, a["ref_b"], cut, l)
        changed += abs(c9["E"] - c["E"]) > c["dE"] + c9["dE"]
    assert changed > 0
    g.close()


CT_MANY = [("bench", 4.0), ("aff_free", 30.0), ("odd", 9.0), ("tma0_160x120", 4.0), ("aff_fixA", 30.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CT_CONFIGS)
def test_ct_many_members_keep_their_huber(capi, gpu, orc, synth, monkeypatch, cfg):
    """one dmv_ct_track_many and one dmv_ct_track_tries_many whose members have different Huber thresholds: each member bit-identical to its
    twin tracked alone"""
    set_cluster(monkeypatch, cfg)
    scs = [ct_scene(orc, synth, n) for n, _ in CT_MANY]
    gs, twins = [ct_handle(capi, sc) for sc in scs], [ct_handle(capi, sc) for sc in scs]
    for g, t, (_, h) in zip(gs, twins, CT_MANY):
        g.set_huber(h); t.set_huber(h)
    args = [track_kw(sc) for sc in scs]
    for (name, h), r, s in zip(CT_MANY, capi.ct_track_many(gs, args), [t.track(**a) for t, a in zip(twins, args)]):
        assert_same(r, s, f"{cfg} track_many {name} huber {h}")
    targs = [dict(tries_kw(sc), **dict(zip(("R", "t"), near_truth_tries(sc)))) for sc in scs]
    for (name, h), r, s in zip(CT_MANY, capi.ct_track_tries_many(gs, targs), [t.track_tries(**a) for t, a in zip(twins, targs)]):
        assert_same(r, s, f"{cfg} track_tries_many {name} huber {h}")
    close(*gs, *twins)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["nc4", "default"])
@pytest.mark.parametrize("name,mode,good", [("aff_zeroA", dict(affA=0.0), 0), ("aff_zeroA", dict(affA=1e12), 1),
                                            ("aff_zeroB", dict(affB=0.0), 0), ("aff_zeroB", dict(affB=1e8), 1),
                                            ("aff_bigA", dict(affA=0.0), 1), ("aff_bigA", dict(affA=1e12), 0)])
def test_ct_affine_mode_zero(capi, gpu, orc, synth, monkeypatch, cfg, name, mode, good):
    """trackNewestCoarse's final test (CoarseTracker.cpp): mode 0 rejects |log ra| > 1.5 or |rb| > 200, a mode != 0 rejects |a| > 1.2 or
    |b| > 200.  helpers.CT_LIGHT's scenes make each test decide alone; the kernel's trackingGood agrees with track_ref's"""
    sc = ct_scene(orc, synth, name)
    rr = ct_ref(sc, **mode)
    assert rr["good"] == good and rr["status"] == 0
    set_cluster(monkeypatch, cfg)
    g = ct_handle(capi, sc)
    r = g.track(**track_kw(sc, **mode))
    assert r["status"] == 0 and r["good"] == good, (r["good"], r["a"], r["b"])
    assert abs(r["a"] - rr["a"]) < 1e-5 and abs(r["b"] - rr["b"]) < 1e-3
    g.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# (g) the coarse initialiser's huberTH
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("huber", [4.0, 30.0])
def test_ci_calc_res_and_gs_huber(capi, gpu, synth, huber):
    """dmv_ci_calc_res_and_gs at huberTH = h against ci_calc_ref(huber = h) with test_gpu_init_ref.py's checks and bounds, on its
    dense_640x480 and edges scenes; the system differs from h = 9's"""
    from test_gpu_init_ref import SCENES, Level, _eval, _sms
    sms = _sms()
    w, h, counts, seed = SCENES["dense_640x480"]
    T = synth.make_tracking_pair(w=w, h=h, seed=seed, trans=0.02, rot=0.005)
    nl = T["levels"]
    pts = H.ci_points(np.random.default_rng(seed), w, h, nl, counts)
    g = capi.CI(w, h, nl, max_points=max(counts))
    levels = [Level(g, l, T["pyr_ref"][l], T["pyr_new"][l], synth.level_K(T["K"], l), pts[l]) for l in range(nl)]
    worst = {}
    for lvl in range(nl - 1, -1, -1):
        for s, kind in enumerate(H.CI_STATES):
            st = H.ci_state(kind, counts[lvl], 1000 * lvl + s)
            sg, _ = _eval(levels[lvl], st, synth, sms, worst, f"dense lvl{lvl} {kind} huber {huber}", huber=huber)
            if kind == "motion":
                s9, _ = _eval(levels[lvl], st, synth, sms, {}, f"dense lvl{lvl} {kind} huber 9")
                assert not np.array_equal(sg["H"], s9["H"]), lvl
    g.close()
    T = synth.make_tracking_pair(seed=31, trans=0.02, rot=0.005)
    p0 = H.ci_points(np.random.default_rng(8), T["w"], T["h"], 1, (4999,))[0]
    k4 = synth.level_K(T["K"], 0)
    st_edge = H.ci_state("edge", len(p0["u"]), 3)
    first, new = H.ci_poison(T["pyr_ref"][0], T["pyr_new"][0], p0, st_edge, k4, synth)
    g = capi.CI(T["w"], T["h"], 1, max_points=len(p0["u"]))
    L = Level(g, 0, first, new, k4, p0)
    _eval(L, st_edge, synth, sms, worst, f"edges huber {huber}", huber=huber)
    for s, kind in enumerate(H.CI_STATES):
        _eval(L, H.ci_state(kind, len(p0["u"]), 10 + s), synth, sms, worst, f"edges {kind} huber {huber}", huber=huber)
    print(f"\nhuber {huber}: worst |err|/bound " + " ".join(f"{k}={x:.3g}" for k, x in worst.items()))
    g.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# (h) the host adapter
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_host_adapter_huber(capi, gpu, orc, synth):
    """hostapi.WindowBA with huberTH = 4 set through dmvh_window_set_setting against the oracle's optimize at huberTH = 4, with
    test_gpu_host.py::test_optimize_matches_oracle's tolerances: the adapter's dmv_ba_set_params reaches the device"""
    import dmvio_b200.hostapi as hostapi
    W = synth.make_window(state_noise=2e-3, nf=4, npts=600, seed=13)
    s = dict(huberTH=4.0)
    ow = orc.Window(W, settings=s)
    n_o, log_o = ow.optimize(6, precision=1)
    hw = hostapi.WindowBA(W, settings=s)
    n_g, log_g = hw.optimize(6)
    assert n_g == n_o and len(log_g) == len(log_o)
    assert abs(log_g[0] - log_o[0]) <= 2e-5 * abs(log_o[0])
    np.testing.assert_allclose(log_g, log_o, rtol=3e-4)
    st_g, id_g, th_g = hw.states()
    assert np.abs(st_g - ow.frame_states()).max() < 2e-5
    np.testing.assert_allclose(id_g, ow.point_outputs()["idepth"], rtol=2e-3, atol=2e-4)
    hw.close()
    h9 = hostapi.WindowBA(W)
    _, log9 = h9.optimize(6)
    h9.close()
    assert abs(log9[0] - log_g[0]) > 1e-3 * abs(log_g[0])

"""CPU tests pinning the oracle's coarse-tracker restatement (CoarseTracker.cpp) by first principles."""
import numpy as np
import pytest

import helpers as H


def _setup(orc, synth, seed=4321, levels=0):
    T = synth.make_tracking_pair(seed=seed, levels=levels)
    ct = orc.CoarseTracker(T["w"], T["h"], T["K"], levels)
    n = ct.make_coarse_depth(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"], T["pyr_ref"])
    ct.set_new_frame(T["pyr_new"])
    return T, ct, n


def test_coarse_depth_lists(orc, synth):
    T, ct, n = _setup(orc, synth)
    assert ct.levels == 4
    counts = [len(ct.ref_points(l)["u"]) for l in range(ct.levels)]
    assert sum(counts) == n
    assert counts[0] > len(T["Ku"])          # dilation adds neighbours on level 0
    p0 = ct.ref_points(0)
    assert p0["idepth"].min() > 0
    # colours are the reference image sampled at integer pixels
    np.testing.assert_array_equal(p0["color"], T["pyr_ref"][0][p0["v"].astype(int), p0["u"].astype(int), 0])
    # 5 forced levels (BASELINE config 2)
    T5, ct5, _ = _setup(orc, synth, levels=5)
    assert ct5.levels == 5 and ct5.K(4)[1].tolist() == [40, 30]


def test_energy_minimal_at_true_pose(orc, synth):
    T, ct, _ = _setup(orc, synth)
    r_true = ct.calc_res(0, T["R_true"], T["t_true"], T["a_new"], T["b_new"])
    r_id = ct.calc_res(0, np.eye(3), np.zeros(3), 0.0, 0.0)
    assert r_true[0] / r_true[1] < 0.2 * r_id[0] / r_id[1]
    assert r_true[5] < 0.05


def test_gs_is_gradient_of_energy(orc, synth):
    """b = sum w J r / n is the gradient of 0.5*sum(huber energy)/n wrt a left pose increment, up to DSO's approximation
    (gradients come from the central-difference channel, not from the interpolant): direction within a few degrees,
    magnitude within the smoothing loss of the gradient channel."""
    T, ct, _ = _setup(orc, synth)
    R0, t0 = synth.se3_mul(*synth.se3_exp(np.array([0.004, -0.003, 0.002, 0.002, -0.001, 0.0015])), T["R_true"], T["t_true"])
    a, b = T["a_new"] + 0.01, T["b_new"] + 0.5
    for lvl, cos_min, ratio_min in ((0, 0.995, 0.85), (1, 0.98, 0.7)):
        ct.calc_res(lvl, R0, t0, a, b, cutoff=1e6)
        H, g = ct.calc_gs(lvl, a, b, 1)
        n = ct.warped().shape[1]
        assert np.allclose(H, H.T) and np.linalg.eigvalsh(H).min() > -1e-9 * np.abs(H).max()

        def energy(xi):
            Re, te = synth.se3_exp(xi)
            R1, t1 = synth.se3_mul(Re, te, R0, t0)
            return 0.5 * ct.calc_res(lvl, R1, t1, a, b, cutoff=1e6)[0]
        fd = np.zeros(6)
        for k in range(6):
            e = np.zeros(6); e[k] = 2e-4
            fd[k] = (energy(e) - energy(-e)) / 4e-4 / n
        cos = fd @ g[:6] / np.linalg.norm(fd) / np.linalg.norm(g[:6])
        ratio = np.linalg.norm(g[:6]) / np.linalg.norm(fd)
        assert cos > cos_min and ratio_min < ratio < 1.1, (lvl, cos, ratio)
    # affine part: d(0.5 E)/db = sum w r * (-1) ... in the scaled parametrisation b_out[7] = SCALE_B * sum(w*(-1)*r)/n
    lvl = 0
    ct.calc_res(lvl, R0, t0, a, b, cutoff=1e6)
    H, g = ct.calc_gs(lvl, a, b, 1)
    n = ct.warped().shape[1]
    eb = 0.5  # large step: calcRes sums the energy in fp32 (CoarseTracker.cpp:L363), the quadratic-ish b-dependence tolerates it
    fdb = (0.5 * ct.calc_res(lvl, R0, t0, a, b + eb, cutoff=1e6)[0] - 0.5 * ct.calc_res(lvl, R0, t0, a, b - eb, cutoff=1e6)[0]) / (2 * eb) / n
    assert abs(fdb * 1000.0 - g[7]) <= 0.02 * abs(g[7]) + 1e-3, (fdb * 1000.0, g[7])


def test_tracking_recovers_pose(orc, synth):
    T, ct, _ = _setup(orc, synth)
    res = ct.track(np.eye(3), np.zeros(3), 0.0, 0.0)
    assert res["good"]
    assert np.linalg.norm(res["t"] - T["t_true"]) < 0.1 * np.linalg.norm(T["t_true"]) + 2e-3
    assert np.abs(res["R"] - T["R_true"]).max() < 2e-3
    # a and b are strongly correlated (a*mean(I) + b): compare the brightness transfer at the mean intensity
    assert abs((np.exp(res["a"]) * 127 + res["b"]) - (np.exp(T["a_new"]) * 127 + T["b_new"])) < 0.5
    assert res["lastResiduals"][0] < 3.0
    # fp32-faithful accumulation takes the same path
    res32 = ct.track(np.eye(3), np.zeros(3), 0.0, 0.0, precision=0)
    assert np.abs(res32["R"] - res["R"]).max() < 1e-4


# scenes where the fp64 reference and the oracle take every decision alike (wide ends an LM level on a near tie that the oracle's
# sequential fp32 energy sum decides differently; its saturation test at level 2 is also within the bound of 0.6)
AGREE = ["bench", "aff_free", "aff_fixA", "aff_fixB", "aff_fixAB", "tma0_80x60", "tma0_160x120", "limit", "odd", "stream", "repeat"]


@pytest.mark.parametrize("name", AGREE)
def test_track_ref_matches_oracle(orc, synth, name):
    """helpers.track_ref (fp64 trackNewestCoarse) against the oracle's trackNewestCoarse: same iterations and good flag, pose within 1e-6,
    lastResiduals within rtol 1e-4 (the GPU tolerance).  Of track_ref's decisions only accept tests may be undecided by its fp32 bound:
    every saturation, incNorm and abort test is decided."""
    sc = H.ct_scene(orc, synth, name)
    r = H.ct_track_ref(sc)
    a = sc["args"]
    ro = H.ct_oracle(orc, sc).track(a["R0"], a["t0"], a["a0"], a["b0"])
    assert r["iterations"] == ro["iterations"] and bool(r["good"]) == ro["good"] and r["status"] == 0
    assert np.abs(r["R"] - ro["R"]).max() < 1e-6 and np.abs(r["t"] - ro["t"]).max() < 1e-6
    assert abs(r["a"] - ro["a"]) < 1e-6 and abs(r["b"] - ro["b"]) < 1e-3
    np.testing.assert_allclose(r["lastResiduals"], ro["lastResiduals"], rtol=1e-4)
    assert {u["what"] for u in r["undecided"]} <= {"accept"}, r["undecided"]


def test_repeat_scene_doubles_cutoff_and_repeats_level(orc, synth):
    sc = H.ct_scene(orc, synth, "repeat")
    log = H.ct_track_ref(sc)["log"]
    top = sc["levels"] - 1
    assert log[0]["sat"] > 0.6 and log[1]["kind"] == "double" and log[1]["rep"] == 2.0
    assert sum(1 for e in log if e["kind"] == "init" and e["lvl"] == top) == 2      # the coarsest level runs twice


@pytest.mark.parametrize("name", H.CT_SCENES + ["counts_31"])
def test_calc_res_ref_matches_oracle(orc, synth, name):
    """helpers.calc_res_ref against the oracle's calc_res / calc_gs at every pose track_ref logs, within its bound for the oracle's summation
    order (depth n: the oracle sums E and the flow terms sequentially in fp32)"""
    sc = H.ct_scene(orc, synth, name)
    r = H.ct_track_ref(sc)
    a = sc["args"]
    oc = H.ct_oracle(orc, sc)
    for e in r["log"]:
        l = e["lvl"]
        RKi, tf, affLL = H.ct_operands(e["R"], e["t"], e["a"], e["b"], sc["Ki"][l], a["ref_a"], a["ref_b"], a["ref_exposure"], a["new_exposure"])
        n = len(sc["pts"][l]["u"])
        cut = np.float32(20) * np.float32(e["rep"])
        c = H.calc_res_ref(sc["pts"][l], sc["planes"][l], sc["k4"][l], sc["Ki"][l], RKi, tf, affLL, a["ref_b"], cut, l, depth=n, R=e["R"])
        ro = oc.calc_res(l, e["R"], e["t"], e["a"], e["b"], cutoff=float(cut))
        Ho, bo = oc.calc_gs(l, e["a"], e["b"], 1)
        assert abs(ro[1] - c["nE"]) <= c["amb"] and abs(ro[0] - c["E"]) <= c["dE"], (l, ro[:2], c["E"], c["nE"], c["dE"])
        if l == 0:
            assert abs(ro[2] - c["res6"][2]) <= c["dflow"][0] and abs(ro[4] - c["res6"][4]) <= c["dflow"][1]
        if c["amb"] == 0:
            assert ro[1] == c["nE"] and oc.warped().shape[1] == c["npad"]
            assert (np.abs(Ho - c["H"]) <= c["dH"]).all() and (np.abs(bo - c["b"]) <= c["db"]).all()

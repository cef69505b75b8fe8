"""dmv_ct_track (trackNewestCoarse in one launch) against the fp64 reference in helpers.py (calc_res_ref / track_ref), in four
configurations of ct_track_cluster_kernel: clusters of 16, 8 and 4 CTAs forced by the DMV_CT_CLUSTER test hook, and "default", the
hook unset, where the handle probes 16, 8 and 4 as it does for a user.  The environment is read when a handle first tracks, so every test
builds a fresh handle after setting it.

Bounds: calc_res_ref's first-order fp32 bound (see its docstring).  It decides every saturation, incNorm and abort test of the scenes, but
not the accept tests at the end of an LM level (energy ratios within 1e-3 of 1 against bounds of 1e-3 to 1e-2), so no scene is decidable in
the strict sense.  The trajectory checks run on the scenes whose seed and start make the fp64 reference and the CPU oracle (fp32, another
summation order) take the same decisions (test_oracle_coarse.py::test_track_ref_matches_oracle); only wide, whose saturation test at level
2 is within the bound of 0.6, and the tiny counts scenes are left out.  The largest |error| / bound of each check is printed (pytest -s)."""
import numpy as np
import pytest

import helpers as H
from gpu_harness import CONFIGS, ct_handle, ct_scene, empty_coarsest, require_device, set_cluster, track_kw

pytestmark = pytest.mark.gpu

TRAJ = ["bench", "aff_free", "aff_fixA", "aff_fixB", "aff_fixAB", "tma0_80x60", "tma0_160x120", "limit", "odd", "stream", "repeat"]
LINEAR = TRAJ + ["wide", "counts_1", "counts_31", "counts_513"]
_REF = {}
RATIOS = {}


@pytest.fixture(scope="module")
def capi():
    """require_device()'s binding; prints the largest error/bound ratios at teardown"""
    yield require_device()
    for k in sorted(RATIOS):
        print(f"max |err|/bound {k}: {RATIOS[k]:.3g}")


def _note(key, v):
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(v))


def ref(sc):
    if sc["name"] not in _REF:
        _REF[sc["name"]] = H.ct_track_ref(sc)
    return _REF[sc["name"]]


def handle(capi, sc, cfg, monkeypatch, pts=None):
    set_cluster(monkeypatch, cfg)
    return ct_handle(capi, sc, pts)


def track(g, sc, **kw):
    return g.track(**track_kw(sc, **kw))


def check_final_linearisation(sc, r, rep, key):
    """lastResiduals[0] and flow against calc_res_ref at the kernel's own returned pose and the level-0 cutoff repeat"""
    a = sc["args"]
    aa = a["a0"] if a["affA"] < 0 else r["a"]
    bb = a["b0"] if a["affB"] < 0 else r["b"]
    RKi, tf, affLL = H.ct_operands(r["R"], r["t"], aa, bb, sc["Ki"][0], a["ref_a"], a["ref_b"], a["ref_exposure"], a["new_exposure"])
    c = H.calc_res_ref(sc["pts"][0], sc["planes"][0], sc["k4"][0], sc["Ki"][0], RKi, tf, affLL, a["ref_b"], np.float32(20) * np.float32(rep), 0, R=r["R"])
    m_ref = c["E"] / c["nE"]
    m_k = float(r["lastResiduals"][0]) ** 2
    bound = m_ref * H.ct_mean_bound(c) + 4 * H.U32 * m_ref          # + rounding of (float)(E/nE), sqrtf and the square taken here
    err = abs(m_k - m_ref)
    _note(f"check1 lastRes {key}", err / bound)
    assert err <= bound, (m_k, m_ref, bound)
    for j, k in ((0, 2), (1, 4)):
        err = abs(r["flow"][2 * j] - c["res6"][k])
        _note(f"check1 flow {key}", err / c["dflow"][j])
        assert err <= c["dflow"][j], (j, r["flow"], c["res6"], c["dflow"])


def level0_rep(log):
    return [e["rep"] for e in log if e["lvl"] == 0][-1]


@pytest.mark.parametrize("cfg", CONFIGS)
@pytest.mark.parametrize("name", LINEAR)
def test_track_against_fp64_reference(capi, orc, synth, monkeypatch, name, cfg):
    """checks 1 (final linearisation) and 4 (determinism) on every scene; check 2 (trajectory) on TRAJ scenes.

    lastResiduals[l] is compared with rtol 1e-4, not 1e-5: a level stops once a step is shorter than 1e-3, not at the minimum, so its energy
    still moves to first order with the pose, and kernel and reference stop at poses up to ~1e-7 apart (the pose tolerance is 1e-6).  On an
    H100 the coarsest level of the bench scene (935 points) differed by 2.0e-5, while check 1 at the kernel's own pose stays below 0.003 of
    its bound, so the difference is the stopping pose, not the sums."""
    sc = ct_scene(orc, synth, name)
    rr = ref(sc) if not name.startswith("counts_") else None
    g = handle(capi, sc, cfg, monkeypatch)
    r = track(g, sc)
    assert g.point_evaluations() > 0
    check_final_linearisation(sc, r, 1.0 if rr is None else level0_rep(rr["log"]), f"{cfg}")
    r2 = track(g, sc)
    for k in r:
        np.testing.assert_array_equal(r2[k], r[k], err_msg=k)
    if name in TRAJ:
        for k in ("iterations", "evaluations", "good", "status"):
            assert r[k] == rr[k], (k, r[k], rr[k])
        assert g.point_evaluations() == rr["point_evaluations"]
        assert np.abs(r["R"] - rr["R"]).max() < 1e-6 and np.abs(r["t"] - rr["t"]).max() < 1e-6, (r["R"] - rr["R"], r["t"] - rr["t"])
        assert abs(r["a"] - rr["a"]) < 1e-6 and abs(r["b"] - rr["b"]) < 1e-6 * 1000
        np.testing.assert_array_equal(np.isnan(r["lastResiduals"]), np.isnan(rr["lastResiduals"]))
        fin = ~np.isnan(rr["lastResiduals"])
        _note(f"check2 lastRes rel {cfg}", np.max(np.abs(r["lastResiduals"][fin] / rr["lastResiduals"][fin] - 1)) / 1e-4)
        np.testing.assert_allclose(r["lastResiduals"][fin], rr["lastResiduals"][fin], rtol=1e-4)
    g.close()


HOST_LOOP = ["bench", "tma0_80x60", "tma0_160x120", "limit", "odd", "repeat"]


@pytest.mark.parametrize("name", LINEAR)
def test_configurations_agree_with_each_other(capi, orc, synth, monkeypatch, name):
    """check 3: the four configurations give the same counts, and so does the host-loop adapter (hostapi.CoarseTracker, device_lm=False)
    on the HOST_LOOP scenes: those built from makeCoarseDepthL0 with the adapter's photometric and affine settings (the aff_* scenes
    change them).  The host loop evaluates with ct_res_gs_kernel, which gathers every level
    from L2, so on the tma0, limit and odd scenes this also compares the TMA-staged planes with the unstaged ones."""
    sc = ct_scene(orc, synth, name)
    rs = []
    for cfg in CONFIGS:
        g = handle(capi, sc, cfg, monkeypatch)
        rs.append(track(g, sc))
        g.close()
    for r in rs[1:]:
        for k in ("iterations", "evaluations", "good", "status"):
            assert r[k] == rs[0][k], (k, [x[k] for x in rs])
    if name in HOST_LOOP:
        import dmvio_b200.hostapi as hostapi
        T, a = sc["T"], sc["args"]
        h = hostapi.CoarseTracker(T["w"], T["h"], T["K"], sc["levels"])
        h.set_ref(T["Ku"], T["Kv"], T["new_idepth"], T["HdiF"], T["pyr_ref"])
        h.set_new_image(T["img_new"])
        rh = h.track(a["R0"], a["t0"], a["a0"], a["b0"], device_lm=False)
        assert rh["iterations"] == rs[0]["iterations"] and rh["evaluations"] == rs[0]["evaluations"] and rh["good"] == bool(rs[0]["good"])
        h.close()


@pytest.mark.parametrize("cfg", CONFIGS)
def test_handle_reuse_after_another_frame(capi, orc, synth, monkeypatch, cfg):
    """check 4: a handle that tracked a different frame in between gives a bit-identical result"""
    sc = ct_scene(orc, synth, "bench")
    g = handle(capi, sc, cfg, monkeypatch)
    r1 = track(g, sc)
    for l in range(sc["levels"]):
        g.upload_new(l, sc["T"]["pyr_ref"][l])       # the keyframe itself as the new frame
    track(g, sc, b0=3.0)
    for l in range(sc["levels"]):
        g.upload_new(l, sc["planes"][l])
    r2 = track(g, sc)
    for k in r1:
        np.testing.assert_array_equal(r2[k], r1[k], err_msg=k)
    g.close()


ABORTS = [("aff_free", w) for w in ("minRes_coarsest", "minRes_l1", "minRes_l0", "empty_coarsest")] + \
         [(n, w) for n in ("counts_1", "counts_31", "counts_513") for w in ("minRes_coarsest", "empty_coarsest")]


@pytest.mark.parametrize("cfg", CONFIGS)
@pytest.mark.parametrize("name,where", ABORTS)
def test_abort_contract(capi, orc, synth, monkeypatch, cfg, name, where):
    """check 5: status 2, good 0, R t a b bit-equal to the inputs, NaN for the unfinished levels, finished levels as the run that does not abort"""
    sc = ct_scene(orc, synth, name)
    L = sc["levels"]
    g = handle(capi, sc, cfg, monkeypatch)
    full = track(g, sc)
    if where == "empty_coarsest":
        g.close()
        g = handle(capi, sc, cfg, monkeypatch, pts=empty_coarsest(sc))
        r, lvl = track(g, sc), L - 1
    else:
        lvl = {"minRes_coarsest": L - 1, "minRes_l1": 1, "minRes_l0": 0}[where]
        mr = np.full(5, np.nan)
        assert full["status"] == 0 and full["lastResiduals"][lvl] > 0
        mr[lvl] = full["lastResiduals"][lvl] / 3
        r = track(g, sc, minRes=mr)
    a = sc["args"]
    assert r["status"] == 2 and r["good"] == 0
    np.testing.assert_array_equal(r["R"], np.asarray(a["R0"], np.float64))
    np.testing.assert_array_equal(r["t"], np.asarray(a["t0"], np.float64))
    assert r["a"] == a["a0"] and r["b"] == a["b0"]
    assert np.isnan(r["lastResiduals"][:lvl]).all()
    if where == "empty_coarsest":
        assert np.isnan(r["lastResiduals"][lvl])
    else:
        np.testing.assert_array_equal(r["lastResiduals"][lvl:], full["lastResiduals"][lvl:])
    g.close()


def test_more_points_than_one_wave_of_ctas(capi, orc, synth, monkeypatch):
    """check 6: a level of #SMs*256 + 1 points, more than one 256-point CTA per SM would cover, is tracked by a cluster of 16"""
    import torch
    n = torch.cuda.get_device_properties(0).multi_processor_count * 256 + 1
    sc = H.ct_scene(orc, synth, "points_big", npts=n)
    g = handle(capi, sc, "nc16", monkeypatch)
    r = track(g, sc)
    check_final_linearisation(sc, r, level0_rep(H.ct_track_ref(sc)["log"]), "points_big nc16")
    g.close()


@pytest.mark.parametrize("name", ["bench", "aff_fixB", "repeat", "stream"])
def test_calc_res_gs_against_fp64_reference(capi, orc, synth, monkeypatch, name):
    """check 7: dmv_ct_calc_res_gs (host-loop / IMU entry point) at every logged pose of the reference, within calc_res_ref's bound.
    The padded warped count is compared exactly wherever no point is ambiguous, and at least one such pose has a count that is not a
    multiple of 4, so a missing padding cannot hide inside the bound of H and b."""
    sc = ct_scene(orc, synth, name)
    rr = ref(sc)
    g = handle(capi, sc, "nc16", monkeypatch)
    a = sc["args"]
    exact_unpadded = 0
    for e in rr["log"]:
        l = e["lvl"]
        RKi, tf, affLL = H.ct_operands(e["R"], e["t"], e["a"], e["b"], sc["Ki"][l], a["ref_a"], a["ref_b"], a["ref_exposure"], a["new_exposure"])
        cut = np.float32(20) * np.float32(e["rep"])
        c = H.calc_res_ref(sc["pts"][l], sc["planes"][l], sc["k4"][l], sc["Ki"][l], RKi, tf, affLL, a["ref_b"], cut, l)
        r6, Hg, bg, npad = g.calc_res_gs(l, RKi, tf, affLL, float(np.float32(a["ref_b"])), float(cut), True)
        assert abs(r6[1] - c["nE"]) <= c["amb"] and abs(npad - c["npad"]) <= c["amb"] + 3
        err = abs(r6[0] - c["E"])
        _note("check7 E", err / c["dE"])
        assert err <= c["dE"], (l, r6[0], c["E"], c["dE"])
        if c["amb"] == 0:
            assert npad == c["npad"] and r6[1] == c["nE"]
            exact_unpadded += c["nW"] % 4 != 0
        if c["npad"] == 0:                   # nothing warped: H and b are 0 * (1/0) in the kernel and in the reference
            assert npad == 0 and np.isnan(Hg).all() and np.isnan(bg).all()
            continue
        _note("check7 H", np.max(np.abs(Hg - c["H"]) / np.maximum(c["dH"], 1e-300)))
        _note("check7 b", np.max(np.abs(bg - c["b"]) / np.maximum(c["db"], 1e-300)))
        assert (np.abs(Hg - c["H"]) <= c["dH"]).all(), (l, np.max(np.abs(Hg - c["H"]) - c["dH"]))
        assert (np.abs(bg - c["b"]) <= c["db"]).all(), (l, bg, c["b"], c["db"])
    assert exact_unpadded > 0
    g.close()

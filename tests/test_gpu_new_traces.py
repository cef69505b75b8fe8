"""dmv_ct_make_new_traces (PixelSelector::makeMaps + makeNewTraces on the resident frame) against the CPU restatement and the golden fixture
made from the reference, bit for bit."""
import os

import numpy as np
import pytest

import dmvio_b200.capi as capi
from oracle import orc
from oracle import select as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_select.npz")


def _same_points(g, o):
    assert g["numPointsTotal"] == o["numPointsTotal"]
    assert g["potential"] == o["potential"]
    for k in S.POINT_KEYS:
        a, b = g["points"][k], o["points"][k]
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), np.ascontiguousarray(b, a.dtype).view(np.uint8)), k


def _golden(G, key):
    return dict(points={k: G[f"{key}/{k}"] for k in S.POINT_KEYS}, numPointsTotal=int(G[f"{key}/numPointsTotal"]), potential=int(G[f"{key}/potential"]))


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_matches_oracle_and_golden(name):
    w, h, lv, kind, seed, args = S.CASES[name]
    a = S.case_args(args)
    pot = a.pop("potential", 3)
    img = S.image(kind, w, h, seed)
    o = S.restate(orc.make_images(img, S.K_of(w, h), lv)[:3], potential=pot, **a)
    ct = capi.CT(w, h, lv)
    ct.upload_new_image(img)
    g = ct.make_new_traces(pot, want_map=True, **a)
    assert np.array_equal(g["map"], o["map"])
    _same_points(g, o)
    _same_points(g, _golden(np.load(GOLDEN), name))
    # the constructor fields equal dmv_ct_init_points fed with the same pixels
    P = ct.init_points(g["points"]["u"], g["points"]["v"])
    for k in ("color", "weights", "gradH", "energyTH"):
        assert np.array_equal(P[k], g["points"][k]), k
    ct.close()


def test_two_handles_share_one_potential():
    """FullSystem's two coarse trackers swap roles while one PixelSelector keeps its potential: alternate handles, one potential variable"""
    G = np.load(GOLDEN)
    w, h, lv = S.SEQ[0][:3]
    cts = [capi.CT(w, h, lv), capi.CT(w, h, lv)]
    pot = 3
    for i, (_, _, _, kind, seed) in enumerate(S.SEQ):
        ct = cts[i % 2]
        ct.upload_new_image(S.image(kind, w, h, seed))
        g = ct.make_new_traces(pot)
        _same_points(g, _golden(G, f"seq{i}"))
        pot = g["potential"]
    for ct in cts:
        ct.close()


def test_handles_of_two_sizes_alternate():
    """the scratch and the chain kernel's launch configuration of one handle survive another handle of a different size"""
    G = np.load(GOLDEN)
    names = ("tex640_l5", "tex512_l4")
    cts = {}
    for name in names:
        w, h, lv, kind, seed, _ = S.CASES[name]
        cts[name] = capi.CT(w, h, lv)
        cts[name].upload_new_image(S.image(kind, w, h, seed))
    for _ in range(2):
        for name in names:
            _same_points(cts[name].make_new_traces(3), _golden(G, name))
    for ct in cts.values():
        ct.close()


@pytest.mark.parametrize("kind,seed", [("tex", 30), ("stair", 31)])
def test_large_frame_reads_the_pattern_from_global_memory(kind, seed):
    """above 200 KB of pattern nibbles (w*h/2) the serial chain reads them from global memory instead of shared memory"""
    w, h, lv = 1024, 512, 5
    img = S.image(kind, w, h, seed)
    o = S.restate(orc.make_images(img, S.K_of(w, h), lv)[:3])
    assert o["n_mixed"] > 0
    ct = capi.CT(w, h, lv)
    ct.upload_new_image(img)
    g = ct.make_new_traces(3, want_map=True)
    assert np.array_equal(g["map"], o["map"])
    _same_points(g, o)
    ct.close()


def test_keyframe_made_resident_by_set_ref_from_ba():
    """dmv_ct_set_ref_from_ba makes the BA window's newest frame the tracker's resident frame: its points are those of the same image
    uploaded directly, and the oracle's"""
    import dmvio_b200.hostmath as hm
    import dmvio_b200.synth as synth
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
    dst = capi.CT(w, h, lv)
    dst.upload_new_image(W["images"][0])   # another frame was resident before the hand-off
    dst.set_ref_from_ba(ba)
    o = S.restate(orc.make_images(np.asarray(W["images"][-1], np.float32), np.asarray(W["K"], np.float64), lv)[:3])
    assert len(o["points"]["u"]) > 100
    g = dst.make_new_traces(3, want_map=True)
    assert np.array_equal(g["map"], o["map"])
    _same_points(g, o)
    _same_points(src.make_new_traces(3), o)
    src.close(); dst.close(); ba.close()


def test_raw_upload_is_resident():
    w, h, lv, kind, seed, _ = S.CASES["tex640_l5"]
    img = S.image(kind, w, h, seed)
    ct = capi.CT(w, h, lv)
    ct.set_undistort(w, h)
    ct.upload_raw_image(img.astype(np.uint8), exposure=0.0)
    _same_points(ct.make_new_traces(3), _golden(np.load(GOLDEN), "tex640_l5"))
    ct.close()


def test_nan_intensities_drop_the_oracles_points():
    w, h, lv, kind, seed, _ = S.CASES["tex512_l4"]
    pyr = [p.copy() for p in orc.make_images(S.image(kind, w, h, seed), S.K_of(w, h), lv)]
    o0 = S.restate(pyr[:3])
    u, v = o0["points"]["u"], o0["points"]["v"]
    for i in range(0, len(u), 7):   # a NaN in the pattern of every 7th point (the gradients stay as they were)
        pyr[0][v[i] + 1, u[i] + 1, 0] = np.nan
    o = S.restate(pyr[:3], B=S.identity_B())
    assert len(o["points"]["u"]) < len(o0["points"]["u"])
    ct = capi.CT(w, h, lv)
    for l in range(lv):
        ct.upload_new(l, pyr[l])
    g = ct.make_new_traces(3, B=S.identity_B(), want_map=True)
    assert np.array_equal(g["map"], o["map"])
    _same_points(g, o)
    ct.close()


def test_errors():
    img = S.image("tex", 640, 480, 1)
    ct = capi.CT(640, 480, 2)
    ct.upload_new_image(img)
    with pytest.raises(capi.DmvError, match="levels 0-2"):
        ct.make_new_traces(3)
    ct.close()
    ct = capi.CT(648, 480, 4)
    with pytest.raises(capi.DmvError, match="divisible by 16"):
        ct.make_new_traces(3)
    ct.close()
    ct = capi.CT(640, 480, 4)
    ct.upload_new_image(img)
    for kw in (dict(potential=0), dict(potential=3, density=0.0), dict(potential=3, thFactor=float("nan")), dict(potential=3, recursionsLeft=-1),
               dict(potential=3, settings=dict(minGradHistCut=1.0))):
        pot = kw.pop("potential")
        with pytest.raises(capi.DmvError):
            ct.make_new_traces(pot, **kw)
    full = ct.make_new_traces(3)
    n = len(full["points"]["u"])
    assert n > 10
    with pytest.raises(capi.DmvError, match="exceed cap"):
        ct.make_new_traces(3, cap=n - 1)
    assert ct.last_needed == n
    assert ct.last_potential == 3        # the selector's state is left as it was: a retry continues from the same potential
    assert len(ct.make_new_traces(3, cap=n)["points"]["u"]) == n
    ct.close()


def test_hostapi_matches_abi():
    import dmvio_b200.hostapi as hostapi
    w, h, lv, kind, seed, _ = S.CASES["tex512_l4"]
    img = S.image(kind, w, h, seed)
    ct = capi.CT(w, h, lv)
    ct.upload_new_image(img)
    g = ct.make_new_traces(3)
    ct.close()
    K = S.K_of(w, h)
    ht = hostapi.CoarseTracker(w, h, np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]]), lv)
    ht.set_new_image(img)
    r = ht.make_new_traces(3)
    ht.close()
    _same_points(r, g)

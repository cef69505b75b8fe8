"""GPU parity of immature-point tracing (dmv_ct_trace_points == ImmaturePoint::traceOn): BIT-EXACT against the CPU oracle, which is
itself pinned bit-exact against the reference's compiled ImmaturePoint.cpp (tests/test_ref_pin.py).  No tolerance: the kernel is built
with -fmad=false and keeps the reference's operation order."""
import numpy as np
import pytest

from gpu_harness import device_capi  # noqa: F401  (the "capi" fixture: every test that takes it needs the device)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", [dict(seed=5, trans=0.05, rot=0.01, n=3000), dict(seed=12, trans=0.12, rot=0.03, n=1500, w=512, h=512)], ids=["640x480", "512x512_fast"])
def test_trace_bit_exact(capi, orc, synth, cfg):
    import dmvio_b200.hostmath as hm
    kw = {k: cfg[k] for k in ("w", "h") if k in cfg}
    W = synth.make_window(nf=3, npts=10, seed=cfg["seed"], trans=cfg["trans"], rot=cfg["rot"], **kw)
    w, h = W["w"], W["h"]
    rng = np.random.default_rng(cfg["seed"])
    n = cfg["n"]
    u, v = rng.integers(10, w - 10, n), rng.integers(10, h - 10, n)
    P = orc.ip_init(W["dI"][0], w, h, u, v)
    g = capi.CT(w, h, synth.pyr_levels(w, h), max_points=1024)
    st = P
    seen = np.zeros(6, int)
    for new in (1, 2, 1):
        KRKi, Kt, aff = hm.trace_tables(W, 0, new)
        g.upload_new(0, W["dI"][new])
        Qg = g.trace_points(st, KRKi, Kt, aff)
        Qo = orc.ip_trace(st, W["dI"][new], w, h, KRKi, Kt, aff)
        for k in orc.IP_STATE_KEYS:
            np.testing.assert_array_equal(Qg[k], Qo[k], err_msg=f"frame {new}: {k}")
        seen += np.bincount(Qo["status"], minlength=6)
        st = Qo
    assert (seen[:5] > 0).all(), seen   # GOOD, OOB, OUTLIER, SKIPPED, BADCONDITION all exercised
    g.close()


def test_trace_device_pyramid_and_edge_cases(capi, orc, synth):
    import dmvio_b200.hostmath as hm
    W = synth.make_window(nf=2, npts=10, seed=3, trans=0.05, rot=0.01)
    w, h = W["w"], W["h"]
    g = capi.CT(w, h, 4, max_points=1024)
    g.upload_new_image(W["images"][1])      # level-0 [I,dx,dy] built on the device from the raw image
    KRKi, Kt, aff = hm.trace_tables(W, 0, 1)
    # empty set
    P0 = orc.ip_init(W["dI"][0], w, h, np.zeros(0, int), np.zeros(0, int))
    assert len(g.trace_points(P0, KRKi, Kt, aff)["status"]) == 0
    # border points go OOB, OOB is sticky
    u = np.array([10, 11, 320, 629]); v = np.array([10, 470, 240, 10])
    P = orc.ip_init(W["dI"][0], w, h, u, v)
    dI1 = W["dI"][1].reshape(h, w, 3).copy()
    Qg, Qo = g.trace_points(P, KRKi, Kt, aff), orc.ip_trace(P, dI1, w, h, KRKi, Kt, aff)
    for k in orc.IP_STATE_KEYS:
        np.testing.assert_array_equal(Qg[k], Qo[k], err_msg=k)
    Q2 = g.trace_points(Qg, KRKi, Kt, aff)
    np.testing.assert_array_equal(Q2["status"][Qg["status"] == 1], 1)
    g.close()


def test_trace_multi_host_equals_per_host(capi, orc, synth):
    """dmv_ct_trace_points_multi: the points of all host keyframes in one launch == one call per host (the loop of traceNewCoarse), bit for bit"""
    import dmvio_b200.hostmath as hm
    W = synth.make_window(nf=5, npts=10, seed=6, trans=0.05, rot=0.01)
    w, h = W["w"], W["h"]
    rng = np.random.default_rng(1)
    new = 4
    sets = []
    for host, n in zip(range(4), (700, 1, 1300, 257)):
        u, v = rng.integers(10, w - 10, n), rng.integers(10, h - 10, n)
        sets.append((orc.ip_init(W["dI"][host], w, h, u, v),) + tuple(hm.trace_tables(W, host, new)))
    g = capi.CT(w, h, synth.pyr_levels(w, h), max_points=1024)
    g.upload_new(0, W["dI"][new])
    one = [g.trace_points(*s_) for s_ in sets]
    allq = g.trace_points_multi(sets)
    for a, b, s_ in zip(one, allq, sets):
        ref = orc.ip_trace(s_[0], W["dI"][new], w, h, *s_[1:])
        for k in orc.IP_STATE_KEYS:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)
            np.testing.assert_array_equal(b[k], ref[k], err_msg=k)
    g.close()


def test_init_points_bit_exact(capi, orc, synth):
    """dmv_ct_init_points == ImmaturePoint constructor: colours, weights, gradH, energyTH equal to the oracle bit for bit."""
    W = synth.make_window(nf=2, npts=10, seed=4)
    w, h = W["w"], W["h"]
    rng = np.random.default_rng(2)
    n = 2500
    u, v = rng.integers(3, w - 4, n), rng.integers(3, h - 4, n)
    g = capi.CT(w, h, 4, max_points=1024)
    g.upload_new(0, W["dI"][0])
    Pg, Po = g.init_points(u, v), orc.ip_init(W["dI"][0], w, h, u, v)
    for k in ("color", "weights", "gradH", "energyTH", "ok"):
        np.testing.assert_array_equal(Pg[k], Po[k], err_msg=k)
    with pytest.raises(capi.DmvError):
        g.init_points(np.array([0]), np.array([5]))   # pattern would leave the image
    g.close()


def test_point_activation_bit_exact(capi, orc, synth):
    """dmv_ba_activate_points == FullSystem::optimizeImmaturePoint: status, inverse depth and residual states equal to the oracle bit for bit."""
    from helpers import activation_case, product_ba_from_oracle
    W, host, P = activation_case(synth, orc)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    aff = ow.precalc()[:, 24:26].copy()
    calib6 = ow.calib()["k8"][:6]
    for minObs in (1, 3):
        s_g, i_g, r_g = ba.activate_points(host, P, ow.RT(), minObs=minObs)
        s_o, i_o, r_o = orc.ip_activate(W, ow.RT(), aff, calib6, host, P, minObs=minObs)
        np.testing.assert_array_equal(s_g, s_o)
        np.testing.assert_array_equal(i_g, i_o)
        np.testing.assert_array_equal(r_g, r_o)
    assert (s_o == 1).sum() > 0.8 * len(s_o)
    ba.close()

"""GPU parity of immature-point tracing and activation where the warp layout of the kernels matters, BIT-EXACT against the CPU oracle
(pinned to the reference's compiled ImmaturePoint.cpp on the same cases by tests/test_ref_pin_ip.py).

ip_trace_kernel deals search steps lane + 32 k (k = 0..3) to the lanes and picks the best with a warp arg-min that must keep the sequential
scan's lowest-index tie rule; ip_activate_kernel runs 8 lanes per point, 4 points per warp, with the frame loops unrolled to
DMV_MAX_FRAMES.  These tests reach: every lane round of the search (up to the clamp at 99 steps), exact energy ties within and across
lanes and rounds, non-finite samples in the search and in Gauss-Newton, every trace status and transition (GN leaving the image included),
empty host sets in one multi-host launch, the ABI's settings pointer, point counts that leave a warp part-filled, and windows of 2 and 8
frames.  The oracle's diag (oracle/orc_trace.h IPD_*) says which branches each trace took; the kernels equal the oracle bit for bit, so
that is the kernels' path too, and every coverage claim below is a hard assert."""
import numpy as np
import pytest

import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    import dmvio_b200.capi as c
    if c.lib().dmv_device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on the H100")
    return c


def _col(orc, k):
    return orc.IP_DIAG_KEYS.index(k)


def _trace_seq(capi, orc, synth, S, P, seq=H.IP_TRACE_SEQ, settings=None):
    """successive traces of P on the device and in the oracle: every IP_STATE_KEYS field equal; returns the oracle's diag and statuses"""
    import dmvio_b200.hostmath as hm
    w, h = S["w"], S["h"]
    g = capi.CT(w, h, synth.pyr_levels(w, h), max_points=1024)
    st, D, seen = P, [], np.zeros(6, int)
    for new in seq:
        tabs = hm.trace_tables(S, 0, new)
        g.upload_new(0, S["dI"][new])
        Qg = g.trace_points(st, *tabs, settings=settings)
        Qo = orc.ip_trace(st, S["dI"][new], w, h, *tabs, diag=True)
        for k in orc.IP_STATE_KEYS:
            np.testing.assert_array_equal(Qg[k], Qo[k], err_msg=f"{w}x{h} frame {new}: {k}")
        D.append(Qo["diag"])
        seen += np.bincount(Qo["status"], minlength=6)
        st = Qo
    g.close()
    return np.concatenate(D), seen


@pytest.mark.parametrize("w,h,seed", H.IP_ROUND_SHAPES, ids=[f"{w}x{h}" for w, h, _ in H.IP_ROUND_SHAPES])
def test_trace_every_lane_round(capi, orc, synth, w, h, seed):
    """fresh searches of 46, 55, 82 and 99 steps: best steps in every round the search has (lanes L + 32 k), and at 2560x1280 the
    clamp of numSteps at 99 (0.027 (w + h) + 1.9999 = 105 steps before it)"""
    S, P = H.ip_round_case(synth, orc, w, h, seed)
    D, _ = _trace_seq(capi, orc, synth, S, P)
    ns, best = D[:, _col(orc, "numSteps")], D[:, _col(orc, "bestIdx")]
    full = min(99, H.ip_num_steps(w, h))
    assert ns.max() == full
    for k in range((full - 1) // 32 + 1):
        assert ((best >= 32 * k) & (best < 32 * (k + 1))).sum() >= 10, f"round {k}"
    if H.ip_num_steps(w, h) >= 100:
        assert (ns == 99).sum() >= 100 and (best >= 96).sum() > 0


def test_trace_tied_energies(capi, orc, synth):
    """8-bit frames with wide bands clipped to 0: whole runs of steps have energy exactly 0; the warp arg-min must pick the first of
    them, also when the run spans lanes and rounds (largest tied step >= 32 while the best is < 32)"""
    S, P = H.ip_round_case(synth, orc, 1280, 720, 15, quantize=True)
    D, _ = _trace_seq(capi, orc, synth, S, P)
    tied = D[:, _col(orc, "nTied")] > 1
    best, last = D[:, _col(orc, "bestIdx")], D[:, _col(orc, "maxTiedIdx")]
    assert tied.sum() >= 50
    assert (tied & (best < 32) & (last >= 32)).sum() >= 5


def test_trace_statuses_and_nonfinite(capi, orc, synth):
    """every trace status and transition, with NaN blocks, columns and rows in the traced frames.  Reached here: GOOD, OOB (sticky, uMin,
    uMax), OUTLIER, OUTLIER followed by OUTLIER (-> OOB), SKIPPED, BADCONDITION, a non-finite new interval, numSteps <= 10 and > 10 (both
    quality branches), GN leaving by its threshold and by its iteration bound, and the +1e5 branches of the search and of GN.  GN leaving
    the image needs a pattern sample within ~0.04 px of a narrow window at the border; test_trace_gn_oob builds it."""
    S, P = H.ip_status_case(synth, orc)
    D, seen = _trace_seq(capi, orc, synth, S, P)
    assert (seen[:5] > 0).all(), seen
    ex = np.bincount(D[:, _col(orc, "exit")], minlength=len(orc.IPX))
    for k in ("STICKY_OOB", "UMIN_OOB", "UMAX_OOB", "SKIPPED", "BADCONDITION", "OUTLIER", "OUTLIER_TWICE", "BAD_INTERVAL", "GOOD"):
        assert ex[orc.IPX[k]] > 0, (k, ex)
    ns = D[:, _col(orc, "numSteps")]
    assert ((ns > 0) & (ns <= 10)).sum() > 0 and (ns > 10).sum() > 0
    brk, its = D[:, _col(orc, "gnBreak")], D[:, _col(orc, "gnIts")]
    assert (brk == 1).sum() > 0 and ((brk == 0) & (its == 3)).sum() > 0
    assert (D[:, _col(orc, "nonfiniteSearch")] > 0).sum() >= 50 and (D[:, _col(orc, "nonfiniteGN")] > 0).sum() >= 20


def test_trace_gn_oob(capi, orc):
    """Gauss-Newton walking a pattern sample off the image (traceOn's OOB return inside the GN loop): tests/helpers.py ip_gn_oob_case
    derives where that can happen and builds it"""
    P, dI, w, h, KRKi, Kt, aff = H.ip_gn_oob_case()
    g = capi.CT(w, h, 4, max_points=1024)
    g.upload_new(0, dI)
    Qg = g.trace_points(P, KRKi, Kt, aff)
    Qo = orc.ip_trace(P, dI, w, h, KRKi, Kt, aff, diag=True)
    for k in orc.IP_STATE_KEYS:
        np.testing.assert_array_equal(Qg[k], Qo[k], err_msg=k)
    assert (Qo["diag"][:, _col(orc, "exit")] == orc.IPX["GN_OOB"]).sum() >= 10
    g.close()


def test_trace_multi_empty_sets_eight_hosts(capi, orc, synth):
    """dmv_ct_trace_points_multi with 8 host frames, empty sets between non-empty ones, at 848x800 (searches of 46 steps): equal to one
    call per host and to the oracle, bit for bit"""
    import dmvio_b200.hostmath as hm
    w, h = 848, 800
    t = H.ip_num_steps(w, h) / (0.5 * w)
    rng = np.random.default_rng(16)
    poses = [np.concatenate([rng.uniform(-0.3 * t, 0.3 * t, 3), rng.uniform(-0.003, 0.003, 3)]) for _ in range(7)] + [np.array([t, 0, t, 0, 0, 0])]
    S = H.ip_scene(synth, w, h, 16, poses)
    new = 8
    sets = []
    for host, n in zip(range(8), (0, 700, 0, 0, 1, 513, 0, 258)):
        u, v = H.ip_points(rng, w, h, n) if n else (np.zeros(0, np.int32), np.zeros(0, np.int32))
        sets.append((orc.ip_init(S["dI"][host], w, h, u, v),) + tuple(hm.trace_tables(S, host, new)))
    g = capi.CT(w, h, synth.pyr_levels(w, h), max_points=1024)
    g.upload_new(0, S["dI"][new])
    one = [g.trace_points(*s_) for s_ in sets]
    allq = g.trace_points_multi(sets)
    best = []
    for a, b, s_ in zip(one, allq, sets):
        ref = orc.ip_trace(s_[0], S["dI"][new], w, h, *s_[1:], diag=True)
        assert len(b["status"]) == len(s_[0]["u"])
        for k in orc.IP_STATE_KEYS:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)
            np.testing.assert_array_equal(b[k], ref[k], err_msg=k)
        best.append(ref["diag"][:, _col(orc, "bestIdx")])
    assert (np.concatenate(best) >= 32).sum() > 0
    g.close()


def test_trace_settings_pointer(capi, orc, synth):
    """the ABI's dmv_ip_settings*: the struct dmv_ip_default_settings fills traces exactly as NULL does (single and multi-host entry)"""
    import dmvio_b200.hostmath as hm
    S, P = H.ip_status_case(synth, orc, n=1500)
    d = capi.ip_default_settings()
    assert (d.maxPixSearch, d.trace_stepsize, d.trace_GNIterations, d.minTraceTestRadius) == (np.float32(0.027), 1.0, 3, 2)
    D, _ = _trace_seq(capi, orc, synth, S, P, settings=d)
    g = capi.CT(S["w"], S["h"], synth.pyr_levels(S["w"], S["h"]), max_points=1024)
    g.upload_new(0, S["dI"][1])
    tabs = hm.trace_tables(S, 0, 1)
    a = g.trace_points_multi([(P,) + tuple(tabs)], settings=d)[0]
    b = g.trace_points(P, *tabs)
    for k in orc.IP_STATE_KEYS:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    g.close()


def _activate_both(capi, orc, W, host, P, minObs=1):
    from helpers import product_ba_from_oracle
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    aff = ow.precalc()[:, 24:26].copy()
    calib6 = ow.calib()["k8"][:6]
    g = ba.activate_points(host, P, ow.RT(), minObs=minObs)
    o = orc.ip_activate(W, ow.RT(), aff, calib6, host, P, minObs=minObs)
    for a, b, k in zip(g, o, ("status", "idepth", "res_state")):
        np.testing.assert_array_equal(a, b, err_msg=k)
    return ba, ow, calib6, o


def test_activation_point_counts(capi, orc, synth):
    """n in {1, 2, 3, 5, 4k+1, 4k+3}: the groups past the end of the list (4 points per warp, 16 per CTA) stand in for the last point and
    write nothing; each result equals the oracle and the same points' result inside the full list"""
    W, host, P = H.activation_edge_case(synth, orc, 5, 2003, 35, nan_frames=(2,))
    ba, ow, calib6, full = _activate_both(capi, orc, W, host, P)
    rng = np.random.default_rng(7)
    for n in (1, 2, 3, 5, 401):
        idx = np.sort(rng.choice(len(host), n, replace=False))
        sub = {k: np.ascontiguousarray(P[k][idx]) for k in P}
        g = ba.activate_points(host[idx], sub, ow.RT())
        for a, b, k in zip(g, full, ("status", "idepth", "res_state")):
            np.testing.assert_array_equal(a, b[idx], err_msg=f"n={n}: {k}")
    assert all((full[0] == k).any() for k in (-1, 0, 1))
    ba.close()


@pytest.mark.parametrize("nf,n,nan_frames", [(2, 1001, (1,)), (8, 2003, (0, 5, 7))], ids=["nf2", "nf8"])
def test_activation_window_sizes(capi, orc, synth, nf, n, nan_frames):
    """windows of 2 frames (the smallest) and 8 (DMV_MAX_FRAMES: every unrolled residual slot live), hosts in every frame including the
    newest, NaN blocks in target frames, a flat block (status 0 through setting_minIdepthH_act), patterns that leave the image part-way"""
    W, host, P = H.activation_edge_case(synth, orc, nf, n, 30 + nf, nan_frames=nan_frames)
    assert (np.bincount(host, minlength=nf) > 0).all()
    ba, ow, calib6, (s, i, r) = _activate_both(capi, orc, W, host, P)
    assert all((s == k).any() for k in (-1, 0, 1))
    if nf == 8:
        assert len(H.activation_partial_oob(W, ow.RT(), calib6, host, P, s, i, r)) >= 10
        assert ((r[s == 1] == 0).sum(1) == nf - 1).any()     # residuals IN in all seven targets
    ba.close()

"""PINS THE ORACLE TO THE REFERENCE on the immature-point cases of tests/test_gpu_ip_edges.py: the reference's compiled ImmaturePoint.cpp
(ImmaturePoint::traceOn, and linearizeResidual under the mirrored optimizeImmaturePoint driver) next to the oracle, bit for bit, at default
settings.  Each case the GPU test compares the kernels with is shown here first to be the reference's own behaviour: search segments past
one warp round of steps (up to the clamp at 99), exact energy ties, non-finite samples, every trace status and transition, Gauss-Newton
leaving the image, activation windows of 2 and 8 frames with NaN blocks, flat blocks and patterns leaving the image part-way."""
import numpy as np
import pytest

import helpers as H


@pytest.fixture(scope="module")
def ref():
    from oracle import ref as _ref
    if not _ref.available():
        pytest.skip("oracle/_ref/libdso_ref.so not built and /root/reference absent")
    _ref.lib()
    return _ref


def _pin_trace(ref, orc, S, P, seq=H.IP_TRACE_SEQ):
    """successive traces (P, then its result against the next frame): reference == oracle on every state field; returns the oracle's diag"""
    import dmvio_b200.hostmath as hm
    w, h = S["w"], S["h"]
    st, D = P, []
    for new in seq:
        tabs = hm.trace_tables(S, 0, new)
        Qo = orc.ip_trace(st, S["dI"][new], w, h, *tabs, diag=True)
        Qr = ref.ip_trace(st, S["dI"][new], w, h, S["K"], *tabs)
        for k in orc.IP_STATE_KEYS:
            np.testing.assert_array_equal(Qo[k], Qr[k], err_msg=f"frame {new}: {k}")
        D.append(Qo["diag"])
        st = Qr
    return np.concatenate(D)


@pytest.mark.parametrize("w,h,seed", H.IP_ROUND_SHAPES, ids=[f"{w}x{h}" for w, h, _ in H.IP_ROUND_SHAPES])
def test_trace_rounds_match_reference(ref, orc, synth, w, h, seed):
    S, P = H.ip_round_case(synth, orc, w, h, seed)
    D = _pin_trace(ref, orc, S, P)
    best = D[:, orc.IP_DIAG_KEYS.index("bestIdx")]
    assert (best >= 32 * ((H.ip_num_steps(w, h) - 1) // 32)).sum() > 0      # the last round the search has is won by some points


def test_trace_ties_match_reference(ref, orc, synth):
    S, P = H.ip_round_case(synth, orc, 1280, 720, 15, quantize=True)
    D = _pin_trace(ref, orc, S, P)
    assert (D[:, orc.IP_DIAG_KEYS.index("nTied")] > 1).sum() > 0


def test_trace_statuses_match_reference(ref, orc, synth):
    S, P = H.ip_status_case(synth, orc)
    D = _pin_trace(ref, orc, S, P)
    assert (D[:, orc.IP_DIAG_KEYS.index("exit")] == orc.IPX["OUTLIER_TWICE"]).sum() > 0


def test_trace_gn_oob_matches_reference(ref, orc):
    P, dI, w, h, KRKi, Kt, aff = H.ip_gn_oob_case()
    Qo = orc.ip_trace(P, dI, w, h, KRKi, Kt, aff, diag=True)
    K = np.array([0.5 * w, 0.5 * w, 0.5 * w - 0.5, 0.5 * h - 0.5])
    Qr = ref.ip_trace(P, dI, w, h, K, KRKi, Kt, aff)
    for k in orc.IP_STATE_KEYS:
        np.testing.assert_array_equal(Qo[k], Qr[k], err_msg=k)
    assert (Qo["diag"][:, orc.IP_DIAG_KEYS.index("exit")] == orc.IPX["GN_OOB"]).sum() > 0


def test_trace_diag_leaves_state_unchanged(orc, synth):
    """diag=True and diag=False trace the same (the diagnostic counters are the only addition)"""
    import dmvio_b200.hostmath as hm
    S, P = H.ip_status_case(synth, orc, n=500)
    tabs = hm.trace_tables(S, 0, 1)
    a = orc.ip_trace(P, S["dI"][1], S["w"], S["h"], *tabs)
    b = orc.ip_trace(P, S["dI"][1], S["w"], S["h"], *tabs, diag=True)
    for k in orc.IP_STATE_KEYS:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    assert b["diag"].shape == (500, len(orc.IP_DIAG_KEYS)) and "diag" not in a


@pytest.mark.parametrize("nf,n,nan_frames", [(2, 1001, (1,)), (5, 2003, (2,)), (8, 2003, (0, 5, 7))], ids=["nf2", "nf5", "nf8"])
def test_activation_edges_match_reference(ref, orc, synth, nf, n, nan_frames):
    W, host, P = H.activation_edge_case(synth, orc, nf, n, 30 + nf, nan_frames=nan_frames)
    rw, ow = ref.Window(W), orc.Window(W)
    aff = ow.precalc()[:, 24:26].copy()
    calib6 = ow.calib()["k8"][:6]
    s_o, i_o, r_o = orc.ip_activate(W, ow.RT(), aff, calib6, host, P, minObs=1)
    s_r, i_r, r_r = rw.activate(host, P, minObs=1)
    np.testing.assert_array_equal(s_o, s_r)
    np.testing.assert_array_equal(i_o, i_r)
    np.testing.assert_array_equal(r_o, r_r)
    assert all((s_r == k).any() for k in (-1, 0, 1))
    del rw

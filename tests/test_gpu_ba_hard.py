"""The BA launch on helpers.hard_window: non-finite and textureless pixels, saturation, exposures != 1 with large affine parameters, points
at the image margins, FEJ centres behind the camera, idepth <= 0.  The oracle equals the reference's compiled code bit for bit on these
windows (tests/test_ref_pin_hard.py); here the device is held to the oracle, at both chunk shapes (P = 32: one lane per residual; P = 16:
four lanes per residual, whose OOB decisions are combined by ballots).

The window's margins keep every projected coordinate of a labelled residual HARD_MARGIN px from its bound and from a texel boundary next to
a non-finite texel, so states must match exactly: a mismatch is a kernel bug, or a tie the seed let through."""
import copy

import numpy as np
import pytest

from helpers import (RES_IN, RES_OOB, RES_OUTLIER, check_linearize_parity, check_phase_b, hard_window, make_case, points_with_in_residual,
                     prior_f, product_ba_from_oracle)
from test_ref_pin_hard import HARD_CONFIGS, check_labels, hard_flagged, hard_id
from gpu_harness import device_capi  # noqa: F401  (the "capi" fixture: every test that takes it needs the device)

pytestmark = pytest.mark.gpu

TH = np.float32(512.0)
_WINDOWS = {}


def window(synth, orc, cfg):
    """hard_window(cfg), built once per module; every test gets its own copy"""
    key = hard_id(cfg)
    if key not in _WINDOWS:
        _WINDOWS[key] = hard_window(synth, orc, cfg)
    return copy.deepcopy(_WINDOWS[key])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _tables(ow):
    return ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"]


def check_exits(W, g):
    """the exits of one linearisation, exactly: states by label, OOB keeps the incoming energy's bits with newEnergyWithOutlier = -1,
    OUTLIER has newEnergy = TH"""
    check_labels(W, g["newState"], g["newEnergy"], g["newEnergyWithOutlier"])
    oob, outl = g["newState"] == RES_OOB, g["newState"] == RES_OUTLIER
    np.testing.assert_array_equal(_bits(g["newEnergy"][oob]), _bits(np.asarray(W["res_energy"], np.float32)[oob]))
    assert np.all(g["newEnergyWithOutlier"][oob] == -1)
    assert np.all(g["newEnergy"][outl] == TH)
    assert np.all(np.isfinite(g["newEnergy"])) and np.all(np.isfinite(g["newEnergyWithOutlier"]))


def check_finite(ba):
    """nothing non-finite in the committed linearisation: systems, per-point outputs, JpJdF of the IN residuals"""
    a, p, g = ba.accumulate(), ba.point_outputs(), ba.residual_outputs()
    for k in ("HA", "bA", "Hsc", "bsc"):
        assert np.all(np.isfinite(a[k])), k
    for k in p:
        assert np.all(np.isfinite(p[k])), k
    assert np.all(np.isfinite(g["JpJdF"][g["newState"] == RES_IN]))


@pytest.mark.parametrize("cfg", HARD_CONFIGS, ids=hard_id)
@pytest.mark.parametrize("P", [16, 32])
def test_linearize_hard(capi, orc, synth, cfg, P):
    W = window(synth, orc, cfg)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    E_o = ow.linearize_all(update_th=False)
    r = ba.linearize()
    o, g = ow.res_outputs(False), ba.residual_outputs()
    mism = np.nonzero(o["newState"] != g["newState"])[0]
    assert len(mism) == 0, (f"residuals {mism[:10]} (labels {W['labels'][mism[:10]]}): device states {g['newState'][mism[:10]]}, oracle "
                            f"{o['newState'][mism[:10]]}; the window's margins exclude ties, so either the kernel is wrong or the seed is")
    check_exits(W, g)
    g, pg, a = check_linearize_parity(ow, ba, r, E_o)
    check_phase_b(pg, points_with_in_residual(W["res_point"], g["newState"], len(W["host"])), prior_f(W), W["idepth"], W["idepth_zero"])
    check_finite(ba)
    ba.close()


@pytest.mark.parametrize("cfg", HARD_CONFIGS, ids=hard_id)
@pytest.mark.parametrize("P", [16, 32])
def test_fused_step_hard(capi, orc, synth, cfg, P):
    """a fused point step from the solved x (test_gpu_ba_step's fp64 bound), the linearisation inside the same launch against a plain
    linearisation at the new depths (bit for bit) and against the oracle: the steps move samples across the NaN texels and the borders"""
    from test_gpu_ba_step import _committed, _solve, check_step
    W = window(synth, orc, cfg)
    ow = orc.Window(W)
    adH, adT = ow.adjoints()
    tabs = _tables(ow)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    ba.linearize(); ba.apply_res()
    C, x = _committed(ba), _solve(ba, W)
    idb = W["idepth"].astype(np.float32)
    ba.backup_points()
    r = ba.gn_step(x, *tabs)
    D, Dz = ba.get_idepth()
    ratio = check_step(W, x, C, adH, adT, idb, D, r["sums"])
    np.testing.assert_array_equal(D, Dz)
    print(f"P={P} {hard_id(cfg)}: step max |err| / bound = {ratio:.3f}")
    ba2 = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    ba2.linearize(); ba2.apply_res()
    ba2.set_state(*tabs, idepth=D, idepth_zero=D)
    r2 = ba2.linearize()
    for k in ("energy", "n_in", "n_oob", "n_outlier"):
        assert r[k] == r2[k], k
    g1, g2 = ba.residual_outputs(), ba2.residual_outputs()
    for k in ("newState", "newEnergy", "newEnergyWithOutlier", "centerProjectedTo"):
        np.testing.assert_array_equal(g1[k], g2[k], err_msg=k)
    changed = (g1["newState"] != C["newState"]).sum()
    W2 = dict(W, idepth=D.copy(), idepth_zero=D.copy(), res_state=C["newState"].copy(), res_energy=C["newEnergy"].copy())
    ow2 = orc.Window(W2)
    E_o = ow2.linearize_all(update_th=False)
    check_linearize_parity(ow2, ba, r, E_o)
    check_finite(ba)
    print(f"P={P} {hard_id(cfg)}: {changed} residuals changed state in the step")
    ba.close(); ba2.close()


@pytest.mark.parametrize("cfg", HARD_CONFIGS, ids=hard_id)
@pytest.mark.parametrize("P", [16, 32])
def test_schur_against_fp64_hard(capi, orc, synth, cfg, P):
    from test_gpu_ba_system import schur_against_fp64
    schur_against_fp64(capi, orc, window(synth, orc, cfg), P, hard_id(cfg))


@pytest.mark.parametrize("cfg", HARD_CONFIGS, ids=hard_id)
@pytest.mark.parametrize("P", [16, 32])
def test_marginalize_points_hard(capi, orc, synth, cfg, P):
    """the marginalisation launch (the MARG instantiation of the same residual code) on points with residuals of every label"""
    from test_gpu_marg import marginalize_parity
    W = window(synth, orc, cfg)
    pts = hard_flagged(W, cfg["seed"])
    flagged = np.isin(W["res_point"], pts)
    assert all((flagged & (W["labels"] == L)).any() for L in ("nan", "flat", "border", "behind"))
    marginalize_parity(capi, orc, synth, cfg, None, P, W=W, pts=pts)


def _linearized(ba):
    r = ba.linearize()
    g = ba.residual_outputs()
    ba.apply_res()
    return r, g, ba.accumulate(), ba.point_outputs(), ba.residual_outputs()


@pytest.mark.parametrize("cfg", HARD_CONFIGS, ids=hard_id)
@pytest.mark.parametrize("P", [16, 32])
def test_image_upload_paths_hard(capi, orc, synth, cfg, P):
    """the intensities with NaN and inf uploaded as images (dmv_ba_upload_image: the device's make_dI_kernel) linearise bit-identically to
    orc.make_images' level 0 uploaded as [I, dx, dy]; a coarse-tracker handle's pyramid of the same image (make_dI_kernel, pyr_down_kernel)
    equals orc.make_images at every level"""
    import dmvio_b200.capi as capi_mod
    W = window(synth, orc, cfg)
    w, h, nf = W["w"], W["h"], W["nf"]
    pyr = [orc.make_images(W["images"][k], W["K"]) for k in range(nf)]
    ow = orc.Window(W)
    a = product_ba_from_oracle(capi, dict(W, dI=[p[0].reshape(-1) for p in pyr]), ow, chunk_points=P)
    b = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    for k in range(nf):
        b.upload_image(k, W["images"][k])
    ra, rb = _linearized(a), _linearized(b)
    for k in ("energy", "n_in", "n_oob", "n_outlier"):
        assert ra[0][k] == rb[0][k], k
    for k in ("newState", "newEnergy", "newEnergyWithOutlier", "centerProjectedTo"):
        np.testing.assert_array_equal(_bits(ra[1][k]), _bits(rb[1][k]), err_msg=k)
    inn = ra[4]["newState"] == RES_IN
    np.testing.assert_array_equal(_bits(ra[4]["JpJdF"][inn]), _bits(rb[4]["JpJdF"][inn]))
    for k in ("HA", "bA", "Hsc", "bsc"):
        np.testing.assert_array_equal(ra[2][k], rb[2][k], err_msg=k)
    for k in ra[3]:
        np.testing.assert_array_equal(_bits(ra[3][k]), _bits(rb[3][k]), err_msg=k)
    check_exits(W, ra[1])
    a.close(); b.close()
    if P == 32:
        return
    ct = capi_mod.CT(w, h, len(pyr[0]), max_points=4096)
    for k in (1, nf - 1):
        ct.upload_new_image(W["images"][k])
        for lvl, want in enumerate(pyr[k]):
            got = ct.download_frame(lvl, w, h)
            np.testing.assert_array_equal(got, want, err_msg=f"frame {k} level {lvl}")
            assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isinf(got), np.isinf(want))
    ct.close()


@pytest.mark.parametrize("P", [16, 32])
def test_batch_member_hard(capi, orc, synth, P):
    """the hard window as one member of a dmv_ba_batch_gn_step call among make_window windows: bit-identical to its own launch, first
    linearisation and a fused step (test_gpu_ba._batched_vs_single_launches)"""
    from test_gpu_ba import _batched_vs_single_launches
    Ws = [make_case(synth, dict(nf=7, npts=2000, seed=1234)), window(synth, orc, HARD_CONFIGS[1]), window(synth, orc, HARD_CONFIGS[0]),
          make_case(synth, dict(nf=4, npts=333, seed=5))]
    _batched_vs_single_launches(capi, orc, synth, P, Ws=Ws)


@pytest.mark.parametrize("cfg", HARD_CONFIGS, ids=hard_id)
def test_host_tables_exposure_hard(capi, orc, synth, cfg):
    """the host adapter's FrameFramePrecalc tables and adjoints with exposures != 1 and large a, b (PRE_aff_mode, PRE_b0_mode)"""
    import dmvio_b200.hostapi as hostapi
    W = window(synth, orc, cfg)
    ow = orc.Window(W)
    hw = hostapi.WindowBA(W)
    pc, adH, adT = hw.tables()
    want = ow.precalc()
    assert np.abs(want[:, 24] - 1).max() > 0.5 and np.abs(want[:, 25]).max() > 20     # the affine terms are far from the identity
    np.testing.assert_allclose(pc, want, rtol=2e-6, atol=1e-4)
    np.testing.assert_allclose(pc[:, 24:27], want[:, 24:27], rtol=1e-6, atol=0)
    a_o, t_o = ow.adjoints()
    np.testing.assert_allclose(adH, a_o, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(adT, t_o, rtol=1e-12, atol=1e-12)
    hw.close()

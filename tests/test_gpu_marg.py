"""GPU parity of the point-marginalisation launch (dmv_ba_marginalize_points) against the CPU oracle, which is itself pinned bit-exactly to
the reference's compiled fixLinearizationF / marginalizePointsF (tests/test_ref_pin.py::test_marginalization_bit_exact).

Tolerances: the same reasoning as tests/test_gpu_ba.py — per-residual vectors (res_toZeroF) rtol 2e-3 of their scale with a small median
error, the summed systems ||d||_F/||.||_F <= 1e-5 (H) and 2e-4 (b: signed sums; res_toZeroF adds one more cancellation than resF) against
the fp64-accumulating oracle, and entry by entry (helpers.check_system at SYSTEM_TAU) with R = sum res_toZeroF^2 for both systems: it
bounds sum J^T rtz by Cauchy-Schwarz, and per point HdiF bd^2 <= bd^2 / Hdd <= the point's sum rtz^2, so it bounds sum_p HdiF bd^2 too.
This window has idepth_zero != idepth: the only test of the depth-delta term of res_toZeroF."""
import numpy as np
import pytest

from helpers import SYSTEM_TAU, check_system, product_ba_from_oracle, rel
from gpu_harness import device_capi  # noqa: F401  (the "capi" fixture: every test that takes it needs the device)

pytestmark = pytest.mark.gpu


def _case(synth, orc, cfg, frac):
    W = synth.make_window(**cfg)
    rng = np.random.default_rng(cfg["seed"] + 1)
    npts, nres = len(W["host"]), len(W["res_point"])
    W["idepth_zero"] = (W["idepth"] * (1 + 0.02 * rng.standard_normal(npts))).astype(np.float32)   # EFPoint::deltaF != 0
    W["hasDepthPrior"] = (rng.random(npts) < 0.3).astype(np.uint8)
    W["res_state"] = rng.choice([0, 1, 2], nres, p=[0.8, 0.1, 0.1]).astype(np.int32)              # resetOOB must bring these back to IN
    W["res_energy"] = rng.uniform(0, 50, nres).astype(np.float32)
    pts = np.sort(rng.choice(npts, max(1, int(npts * frac)), replace=False)).astype(np.int32)
    return W, pts


@pytest.mark.parametrize("cfg,frac,P", [(dict(nf=7, npts=2000, seed=1234), 0.33, 16), (dict(nf=4, npts=400, seed=3, hosts="all"), 0.5, 32),
                                        (dict(nf=8, npts=777, seed=99, hosts="all"), 0.1, 32), (dict(nf=3, npts=333, seed=7), 1.0, 16)],
                         ids=["nf7_n2000_third", "nf4_n400_half", "nf8_n777_tenth", "nf3_n333_all"])
def test_marginalize_points_parity(capi, orc, synth, cfg, frac, P):
    marginalize_parity(capi, orc, synth, cfg, frac, P)


def marginalize_parity(capi, orc, synth, cfg, frac, P, settings=None, W=None, pts=None):
    """the launch against the oracle on _case(cfg, frac), or on the window W flagging the points pts, both at `settings` (dmv_ba_set_params
    keywords; None: the defaults).  Returns the launch's result."""
    if W is None:
        W, pts = _case(synth, orc, cfg, frac)
    ow = orc.Window(W, settings=settings)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)   # carries the points' priorF (hasDepthPrior)
    if settings:
        ba.set_params(**settings)
    # a committed linearisation exists in real use (the window has just been optimised): the marginalisation must not disturb it
    ba.linearize(); ba.apply_res()
    before = ba.accumulate()
    g = ba.marginalize_points(pts, ow.adHTdeltaF(), ow.calib()["cDeltaF"])
    after = ba.accumulate()
    for k in ("HA", "bA", "Hsc", "bsc"):
        np.testing.assert_array_equal(before[k], after[k])
    o = ow.marginalize(pts, precision=1)
    # ---- which residuals were linearised (threshold ties aside)
    mism = np.nonzero(o["isLinearized"] != g["isLinearized"])[0]
    assert len(mism) <= max(1, len(W["res_point"]) // 1000), mism
    both = (o["isLinearized"] == 1) & (g["isLinearized"] == 1)
    assert both.sum() > 0
    in_set = np.isin(W["res_point"], pts)
    assert not g["isLinearized"][~in_set].any()
    assert np.all(g["rtz"][g["isLinearized"] == 0] == 0)
    assert len(mism) == 0, "a threshold tie on a seeded case: the system comparison below must never be skipped (pick another seed)"
    np.testing.assert_array_equal(g["ngood"], o["ngood"])
    assert g["resInM"] == o["resInM"]
    # ---- res_toZeroF per residual
    scale = np.abs(o["rtz"][both]).max()
    err = np.abs(g["rtz"][both] - o["rtz"][both])
    assert err.max() <= 2e-3 * scale + 1e-4, err.max()
    assert np.median(err) <= 2e-5 * scale
    # ---- the marginalisation system
    assert rel(g["M"], o["M"]) < 1e-5 and rel(g["Msc"], o["Msc"]) < 1e-5
    assert rel(g["H"], o["H"]) < 1e-5
    assert rel(g["Mb"], o["Mb"]) < 2e-4 and rel(g["Mbsc"], o["Mbsc"]) < 2e-4 and rel(g["b"], o["b"]) < 2e-4
    R = float((o["rtz"].astype(np.float64) ** 2).sum())
    r = (check_system(g["M"], g["Mb"], o["M"], o["Mb"], R, SYSTEM_TAU, "marginalisation M, Mb")
         + check_system(g["Msc"], g["Mbsc"], o["Msc"], o["Mbsc"], R, SYSTEM_TAU, "marginalisation Msc, Mbsc"))
    print(f"check_system vs oracle: worst |error| / Jacobi scale: M {r[0]:.2e} Mb {r[1]:.2e} Msc {r[2]:.2e} Mbsc {r[3]:.2e}")
    assert np.allclose(g["M"], g["M"].T) and np.allclose(g["Msc"], g["Msc"].T, rtol=1e-12, atol=0)
    ba.close()
    return g


def test_marginalize_empty_and_errors(capi, orc, synth):
    W = synth.make_window(nf=3, npts=100, seed=2)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    g = ba.marginalize_points(np.zeros(0, np.int32), ow.adHTdeltaF(), ow.calib()["cDeltaF"])       # nothing flagged: all-zero system
    assert g["resInM"] == 0 and not g["M"].any() and not g["Msc"].any() and not g["Mb"].any()
    with pytest.raises(capi.DmvError):
        ba.marginalize_points(np.array([len(W["host"])], np.int32), ow.adHTdeltaF(), ow.calib()["cDeltaF"])   # index out of range
    ba.close()

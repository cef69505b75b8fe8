"""GPU parity tests of the BA hot path: CUDA (through the C ABI) vs the CPU oracle on the same seeded inputs.

Tolerances, and why (fp32 on both sides, different operation order / FMA contraction):
  * a projected coordinate Ku ~ 300-600 px carries ~1 ulp = 3e-5..6e-5 px of rounding; times an image gradient of up to
    ~30 intensity units/px this is ~1e-3..2e-3 intensity units on every interpolated sample, i.e. up to ~1e-3 RELATIVE on a
    per-residual energy or Jacobian entry.  Per-residual quantities are therefore checked with rtol 2e-3 (+ small atol) AND a
    median relative error < 2e-4 (no systematic bias);
  * sums over thousands of residuals average these errors out: total energy rel 2e-5, H blocks ||d||_F/||.||_F <= 1e-5,
    right-hand sides (signed sums with cancellation) <= 1e-4, all against the fp64-accumulating oracle;
  * state flags identical except residuals whose deciding energy is within 1e-3 rel of its threshold.
"""
import numpy as np
import pytest

from helpers import check_linearize_parity, check_phase_b, make_case, points_with_in_residual, prior_f, product_ba_from_oracle, rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    import dmvio_b200.capi as c
    if c.lib().dmv_device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on the H100")
    return c


CONFIGS = [
    dict(nf=2, npts=200, seed=1234, hosts="first"),   # BASELINE config 1: 2 KF / 200 pts hosted in KF0
    dict(nf=3, npts=333, seed=7),                      # ragged chunk sizes
    dict(nf=7, npts=2000, seed=1234),                  # BASELINE config 3
    dict(nf=8, npts=777, seed=99, hosts="all"),        # max window size, newest frame hosts points too
    dict(nf=7, npts=8000, seed=1234),                  # BASELINE config 4 (all 8000 points on one GPU)
    dict(nf=7, npts=2000, seed=1234, w=512, h=512),    # BASELINE config 5's image shape (TUM-VI 512x512)
    # helpers.edge_window: depth priors with idepth_zero != idepth, missing / OOB / OUTLIER residuals, points without residuals
    dict(nf=7, npts=2000, seed=1234, edge=True),
    dict(nf=7, npts=8000, seed=1234, edge=True),       # several chunks per CTA at P = 16
]


def cfg_id(c):
    return f"nf{c['nf']}_n{c['npts']}" + ("_edge" if c.get("edge") else "")


def _states_equal_up_to_threshold(o_new, g_new, o_e, th_tol=1e-4):
    bad = np.nonzero(o_new != g_new)[0]
    return bad


@pytest.mark.parametrize("cfg", CONFIGS, ids=cfg_id)
@pytest.mark.parametrize("P", [16, 32])
def test_linearize_accumulate_parity(capi, orc, synth, cfg, P):
    W = make_case(synth, cfg)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    E_o = ow.linearize_all(update_th=False)
    r = ba.linearize()
    g, pg, _ = check_linearize_parity(ow, ba, r, E_o)
    # ---- phase B in closed form from the launch's own sums (depth prior and its shift to zero included)
    check_phase_b(pg, points_with_in_residual(W["res_point"], g["newState"], len(W["host"])), prior_f(W), W["idepth"], W["idepth_zero"])
    ba.close()


def test_resubstitute_and_step(capi, orc, synth):
    W = synth.make_window(nf=5, npts=900, seed=21)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    ow.linearize_all(update_th=False); ba.linearize()
    ow.apply_res(); ba.apply_res()
    x, _, _ = ow.solve(0, 1e-5, 1)   # oracle: accumulate + solve + resubstitute
    step_g, sums = ba.resubstitute(x, apply=False)
    step_o = ow.point_outputs()["step"]
    np.testing.assert_allclose(step_g, step_o, rtol=2e-3, atol=2e-4 * np.abs(step_o).max())  # step = -HdiF * (difference of O(1) sums)
    assert abs(sums[0] - float((step_o.astype(np.float64) ** 2).sum())) <= 1e-3 * sums[0]
    assert sums[2] == ba.npts
    # apply: idepth = backup + step (and idepth_zero follows, DM-VIO)
    ba.backup_points()
    ba.resubstitute(x, apply=True)
    idd, idz = ba.get_idepth()
    np.testing.assert_allclose(idd, W["idepth"] + step_g, rtol=0, atol=1e-6)
    np.testing.assert_array_equal(idd, idz)
    ba.restore_points()
    idd, _ = ba.get_idepth()
    np.testing.assert_array_equal(idd, W["idepth"])
    ba.close()


def test_oob_and_prior_states(capi, orc, synth):
    W = synth.make_window(nf=3, npts=200, seed=5)
    rng = np.random.default_rng(0)
    n = len(W["res_point"])
    W["res_state"] = rng.choice([0, 1, 2], n, p=[0.7, 0.2, 0.1]).astype(np.int32)
    W["res_energy"] = rng.uniform(0, 50, n).astype(np.float32)
    npts = len(W["host"])
    W["hasDepthPrior"] = (rng.random(npts) < 0.3).astype(np.uint8)
    W["idepth_zero"] = (W["idepth"] * (1 + 0.02 * rng.standard_normal(npts))).astype(np.float32)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    E_o = ow.linearize_all(update_th=False)
    r = ba.linearize()
    o, g = ow.res_outputs(False), ba.residual_outputs()
    assert np.all(g["newState"][W["res_state"] == 1] == 1)     # can never go back from OOB
    same = o["newState"] == g["newState"]
    assert same.mean() > 0.99
    E_o, _, unfixable = ow.override_new_states(g["newState"])
    assert unfixable == 0
    assert abs(r["energy"] - E_o) <= 2e-5 * abs(E_o)
    # the priors enter H = Hdd + priorF and bdSumF = bd + priorF * (idepth - idepth_zero)
    ow.apply_res(); ba.apply_res()
    ow.accumulate(1); ba.accumulate()
    po, pg = ow.point_outputs(), ba.point_outputs()
    for k in ("HdiF", "bdSumF"):
        np.testing.assert_allclose(pg[k], po[k], rtol=2e-3, atol=2e-4 * np.abs(po[k]).max())
    check_phase_b(pg, points_with_in_residual(W["res_point"], g["newState"], npts), prior_f(W), W["idepth"], W["idepth_zero"])
    ba.close()


def test_full_gn_iteration_matches_oracle(capi, orc, synth):
    """linearize -> apply -> accumulate -> host solve (oracle's LDLT on the GPU's H,b) -> fused gn_step at the new state."""
    W = synth.make_window(nf=4, npts=600, seed=31)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    ow.linearize_all(update_th=False); ba.linearize(); ow.apply_res(); ba.apply_res()
    a_g = ba.accumulate()
    x_o, HF, bF = ow.solve(0, 1e-5, 1)
    # same system on both sides => same x (checks the conditioning of the 1e-5 tolerance on H)
    sys_o = ow.accumulate(1)
    lam = 1e-5
    Hg = a_g["HA"] + sys_o["HL"]
    Hg[np.diag_indices_from(Hg)] *= (1 + lam)
    Hg = Hg - a_g["Hsc"] / (1 + lam)
    bg = a_g["bA"] + sys_o["bL"] - a_g["bsc"]
    s = 1.0 / np.sqrt(np.diag(Hg) + 10)
    x_g = s * np.linalg.solve(s[:, None] * Hg * s[None, :], s * bg)
    assert rel(x_g, x_o) < 1e-3
    # the fused step with the GPU-side solution against the oracle's resubstitution of the same x (step = -HdiF * (difference of O(1) sums))
    ba.backup_points()
    ba.gn_step(x_g, ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"])
    ow.resubstitute(x_g)
    step_o = ow.point_outputs()["step"]
    idd, idz = ba.get_idepth()
    step_g = idd.astype(np.float64) - W["idepth"]
    np.testing.assert_allclose(step_g, step_o, rtol=2e-3, atol=2e-4 * np.abs(step_o).max() + np.spacing(np.abs(idd)).max())
    np.testing.assert_array_equal(idd, idz)
    ba.close()


def test_batched_windows_identical_to_single_launches(capi, orc, synth):
    """SURVEY §8d batched variant: B windows of different shapes in ONE launch (dmv_ba_batch_gn_step) give, per window, bit-identical
    results to the window's own launch — first linearisation and a fused GN step (resubstitute + point step inside the launch).
    16-point chunks (the shape the automatic rule picks for these windows); the third window carries depth priors and missing / OOB /
    OUTLIER residuals."""
    _batched_vs_single_launches(capi, orc, synth, P=16)


def test_batched_windows_identical_to_single_launches_chunk32(capi, orc, synth):
    """the same with 32-point chunks: the P = 32 batch kernel, the shape ba_fused.cu names for batches"""
    _batched_vs_single_launches(capi, orc, synth, P=32)


def _batched_vs_single_launches(capi, orc, synth, P):
    import dmvio_b200.hostmath as hm
    cfgs = [dict(nf=7, npts=2000, seed=1234), dict(nf=4, npts=333, seed=5), dict(nf=8, npts=777, seed=99, hosts="all", edge=True),
            dict(nf=2, npts=200, seed=3, hosts="first")]
    Ws = [make_case(synth, c) for c in cfgs]

    def load(W):
        ow = orc.Window(W)
        ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
        return ba, (ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"])

    singles, batched = [load(W) for W in Ws], [load(W) for W in Ws]
    batch = capi.BABatch([b for b, _ in batched])
    keys = ("HA", "bA", "Hsc", "bsc")
    # ---- first linearisation
    ref = []
    for (ba, st) in singles:
        r = ba.gn_step(None, *st); ba.apply_res()
        ref.append((r, ba.accumulate(), ba.residual_outputs(), ba.point_outputs()))
    rb = batch.gn_step(None, [st for _, st in batched])
    xs = []
    for i, (ba, st) in enumerate(batched):
        ba.apply_res()
        a, g, p = ba.accumulate(), ba.residual_outputs(), ba.point_outputs()
        assert rb[i]["energy"] == ref[i][0]["energy"] and rb[i]["n_in"] == ref[i][0]["n_in"]
        for k in keys:
            np.testing.assert_array_equal(a[k], ref[i][1][k])
        for k in ("newState", "newEnergy"):
            np.testing.assert_array_equal(g[k], ref[i][2][k])
        inn = g["newState"] == 0   # JpJdF is defined for IN residuals only (include/dmvio_b200.h)
        np.testing.assert_array_equal(g["JpJdF"][inn], ref[i][2]["JpJdF"][inn])
        np.testing.assert_array_equal(p["HdiF"], ref[i][3]["HdiF"])
        np.testing.assert_array_equal(p["bdSumF"], ref[i][3]["bdSumF"])
        HL, bL = hm.prior_system(Ws[i])
        xs.append(hm.solve_reduced(a["HA"], a["bA"], a["Hsc"], a["bsc"], HL, bL, lam=1e-5))
    # ---- a fused GN step
    for (ba, st), x in zip(singles, xs):
        ba.backup_points()
    for (ba, st) in batched:
        ba.backup_points()
    ref2 = []
    for (ba, st), x in zip(singles, xs):
        r = ba.gn_step(x, *st); ba.apply_res()
        ref2.append((r, ba.accumulate(), ba.get_idepth()[0]))
    rb2 = batch.gn_step(xs, [st for _, st in batched])
    for i, (ba, st) in enumerate(batched):
        ba.apply_res()
        a = ba.accumulate()
        assert rb2[i]["energy"] == ref2[i][0]["energy"]
        np.testing.assert_array_equal(rb2[i]["sums"], ref2[i][0]["sums"])
        for k in keys:
            np.testing.assert_array_equal(a[k], ref2[i][1][k])
        np.testing.assert_array_equal(ba.get_idepth()[0], ref2[i][2])
    batch.close()
    for ba, _ in singles + batched:
        ba.close()


def test_run_to_run_bit_reproducible(capi, orc, synth):
    """no atomics on the data path: two launches on the same inputs give the same bits"""
    W = synth.make_window(nf=7, npts=2000, seed=1234)
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow)
    st = (ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"])
    outs = []
    for _ in range(3):
        r = ba.gn_step(None, *st)
        ba.apply_res()
        a = ba.accumulate()
        outs.append((r["energy"], a["HA"].copy(), a["bA"].copy(), a["Hsc"].copy(), a["bsc"].copy()))
        ba.reset_oob()
    for o in outs[1:]:
        assert o[0] == outs[0][0]
        for x, y in zip(o[1:], outs[0][1:]):
            np.testing.assert_array_equal(x, y)
    ba.close()


def test_handles_on_two_devices_in_one_process(capi, orc, synth):
    """VERDICT r1 weak #9: kernel attributes are configured per DEVICE (single-process multi-device hosts, SURVEY §8b dmv_comm_init model)"""
    if capi.lib().dmv_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    W = synth.make_window(nf=5, npts=600, seed=8)
    ow = orc.Window(W)
    res = []
    for dev in (0, 1):
        ba = product_ba_from_oracle(capi, W, ow, device=dev)
        r = ba.linearize(); ba.apply_res()
        res.append((r["energy"], ba.accumulate()))
        ba.close()
    assert res[0][0] == res[1][0]
    for k in ("HA", "bA", "Hsc", "bsc"):
        np.testing.assert_array_equal(res[0][1][k], res[1][1][k])

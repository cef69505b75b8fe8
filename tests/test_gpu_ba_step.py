"""The point step fused into the BA launch (dmv_ba_gn_step with x: EnergyFunctional::resubstituteFPt + the point part of
doStepFromBackup in ba_fused_kernel's phase A) and the linearisation that follows it in the same launch, at both chunk shapes.

  (a) the fused step against an fp64 evaluation of the same formula on the launch's own committed fp32 inputs, with a rounding bound;
  (b) against the stand-alone ba_resub_kernel on the same committed state (bit-identical at P = 32, which sums in the same order);
  (c) the linearisation at the new depths inside the fused launch against a plain linearize at those depths, bit for bit;
  (d) that linearisation against the oracle, and one more fused step against the oracle's step for the same x;
  (e) an accept / reject / accept chain through the backup / restore ping-pong of the depth buffers.

The windows are tests/test_gpu_ba.py's CONFIGS with helpers.edge_window's irregular point and residual sets.
"""
import numpy as np
import pytest

import dmvio_b200.hostmath as hm
from helpers import (RES_IN, check_linearize_parity, check_phase_b, edge_window, points_with_in_residual, prior_f, product_ba_from_oracle,
                     ulp32)
from test_gpu_ba import CONFIGS

pytestmark = pytest.mark.gpu

EPS32 = float(np.finfo(np.float32).eps)
STEP_CONFIGS = [c for c in CONFIGS if not c.get("edge")]


@pytest.fixture(scope="module")
def capi():
    import dmvio_b200.capi as c
    if c.lib().dmv_device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on the H100")
    return c


def _window(synth, cfg):
    return edge_window(synth, dict(cfg, state_noise=3e-3))


def _max_points(W):
    n = len(W["host"])
    return 4096 if n < 1000 else None    # slot pitch mp != npts on the smaller windows


def _tables(ow):
    return ow.calib()["k8"], ow.precalc(), ow.frame_tables()["frameEnergyTH"]


def _committed(ba):
    """the committed linearisation the next fused step reads (call right after apply_res)"""
    g, p = ba.residual_outputs(), ba.point_outputs()
    return dict(newState=g["newState"].copy(), newEnergy=g["newEnergy"].copy(), JpJdF=g["JpJdF"].copy(), Hcd=p["Hcd"].copy(), HdiF=p["HdiF"].copy(),
                bdSumF=p["bdSumF"].copy())


def _solve(ba, W):
    a = ba.accumulate()
    HL, bL = hm.prior_system(W)
    return hm.solve_reduced(a["HA"], a["bA"], a["Hsc"], a["bsc"], HL, bL, lam=1e-5)


def _random_x(rng, x, nf):
    """random increment with the per-block magnitude of x (camera block: that of the frame blocks, so the Hcd term is exercised)"""
    xr = np.zeros_like(x)
    frames = [x[4 + 8 * f:12 + 8 * f] for f in range(nf)]
    for f in range(nf):
        xr[4 + 8 * f:12 + 8 * f] = rng.standard_normal(8) * (np.linalg.norm(frames[f]) / np.sqrt(8))
    xr[:4] = rng.standard_normal(4) * np.mean([np.linalg.norm(b) / np.sqrt(8) for b in frames])
    return xr


def step_reference(W, x, C, adH, adT):
    """fp64 step of every point from the fp32 committed inputs C and xF = float32(x):
    step = -HdiF * (bdSumF - xc . Hcd - sum_{t != h, IN} xAd[h,t] . JpJdF_t), xAd[h,t] = xF_h^T adHostF(h,t) + xF_t o diag adTargetF(h,t)
    (adjoint blocks indexed h + t*nf, as dmv_ba_set_adjoints reads them).  Returns (step, S, ngood) with S the sum of the absolute values of
    every product in the formula, |xF| |adjoint| inside xAd included."""
    nf, npts = W["nf"], len(W["host"])
    xF = x.astype(np.float32).astype(np.float64)
    AH = adH.astype(np.float32).astype(np.float64)                            # [h + t*nf][k][c]
    AT = np.einsum("ikk->ik", adT).astype(np.float32).astype(np.float64)     # diag
    xAd, xAd_abs = np.zeros((nf, nf, 8)), np.zeros((nf, nf, 8))
    for h in range(nf):
        xh = xF[4 + 8 * h:12 + 8 * h]
        for t in range(nf):
            xt = xF[4 + 8 * t:12 + 8 * t]
            A, d = AH[h + t * nf], AT[h + t * nf]
            xAd[h, t] = xh @ A + xt * d
            xAd_abs[h, t] = np.abs(xh) @ np.abs(A) + np.abs(xt * d)
    rp, rt = W["res_point"], W["res_target"]
    host = W["host"]
    inn = C["newState"] == RES_IN
    p, t, J = rp[inn], rt[inn], C["JpJdF"][inn].astype(np.float64)
    h = host[p]
    dots = (xAd[h, t] * J).sum(1)
    dabs = (xAd_abs[h, t] * np.abs(J)).sum(1)
    Hcd = C["Hcd"].astype(np.float64)
    xc = xF[:4]
    b = C["bdSumF"].astype(np.float64) - Hcd @ xc - np.bincount(p, dots, minlength=npts)
    S = np.abs(C["bdSumF"].astype(np.float64)) + np.abs(Hcd) @ np.abs(xc) + np.bincount(p, dabs, minlength=npts)
    ngood = np.bincount(p, minlength=npts)
    step = np.where(ngood > 0, -C["HdiF"].astype(np.float64) * b, 0.0)
    return step, S, ngood


def check_step(W, x, C, adH, adT, idb, idd, sums=None):
    """bound (a) on the depths idd = idepth_backup + step written by a step; returns max |error| / bound"""
    step, S, ngood = step_reference(W, x, C, adH, adT)
    want = idb.astype(np.float64) + step
    bound = 64 * EPS32 * np.abs(C["HdiF"].astype(np.float64)) * S + ulp32(want)
    err = np.abs(idd.astype(np.float64) - want)
    worst = int(np.argmax(err / bound))
    assert np.all(err <= bound), f"point {worst}: |err| {err[worst]:.3e} > bound {bound[worst]:.3e} (ngood {ngood[worst]})"
    np.testing.assert_array_equal(idd[ngood == 0], idb[ngood == 0])     # no good residual: no step
    if sums is not None:
        assert sums[2] == len(idb)
        assert abs(sums[1] - np.abs(idb.astype(np.float64)).sum()) <= 1e-6 * sums[1]
        s2 = float((step ** 2).sum())
        assert abs(sums[0] - s2) <= 1e-5 * s2
    return float((err / bound).max())


@pytest.mark.parametrize("cfg", STEP_CONFIGS, ids=lambda c: f"nf{c['nf']}_n{c['npts']}" + (f"_{c['w']}x{c['h']}" if "w" in c else ""))
@pytest.mark.parametrize("P", [16, 32])
def test_fused_step_and_relinearisation(capi, orc, synth, cfg, P):
    W = _window(synth, cfg)
    ow = orc.Window(W)
    adH, adT = ow.adjoints()
    tabs = _tables(ow)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P, max_points=_max_points(W))
    ba.linearize(); ba.apply_res()
    C = _committed(ba)
    x = _solve(ba, W)
    idb = W["idepth"].astype(np.float32)
    ratios = []
    # ---- (a) with a random x of the solution's per-block magnitude first (a rejected step leaves no trace: restore + same committed state)
    xr = _random_x(np.random.default_rng(cfg["seed"]), x, W["nf"])
    ba.backup_points()
    rr = ba.gn_step(xr, *tabs)
    idd, idz = ba.get_idepth()
    ratios.append(check_step(W, xr, C, adH, adT, idb, idd, rr["sums"]))
    np.testing.assert_array_equal(idd, idz)
    ba.restore_points()
    # ---- (a) with the solved x
    ba.backup_points()
    r = ba.gn_step(x, *tabs)
    D, Dz = ba.get_idepth()
    ratios.append(check_step(W, x, C, adH, adT, idb, D, r["sums"]))
    np.testing.assert_array_equal(D, Dz)                           # setIdepthZero: idepth_zero follows
    assert np.abs(D.astype(np.float64) - idb).max() > 1e-4 * np.abs(idb).max()   # the steps are not negligible
    print(f"P={P} {cfg}: max |err| / bound = {max(ratios):.3f}")
    # ---- (b) the stand-alone kernel on the same committed state (the fused launch's own linearisation is still tentative)
    step_s, _ = ba.resubstitute(x, apply=False)
    D_s = (idb + step_s).astype(np.float32)
    if P == 32:
        np.testing.assert_array_equal(D, D_s)
    else:
        check_step(W, x, C, adH, adT, idb, D_s)
    # ---- (c) the linearisation inside the fused launch == linearize at the new depths (same history), bit for bit
    ba2 = product_ba_from_oracle(capi, W, ow, chunk_points=P, max_points=_max_points(W))
    ba2.linearize(); ba2.apply_res()
    ba2.set_state(*tabs, idepth=D, idepth_zero=D)
    r2 = ba2.linearize()
    for k in ("energy", "n_in", "n_oob", "n_outlier"):
        assert r[k] == r2[k], k
    g1, g2 = ba.residual_outputs(), ba2.residual_outputs()
    for k in ("newState", "newEnergy", "newEnergyWithOutlier", "centerProjectedTo"):
        np.testing.assert_array_equal(g1[k], g2[k], err_msg=k)
    inn = g1["newState"] == RES_IN                                 # JpJdF is defined for IN residuals only (include/dmvio_b200.h)
    np.testing.assert_array_equal(g1["JpJdF"][inn], g2["JpJdF"][inn])
    p1, p2 = ba.point_outputs(), ba2.point_outputs()
    for k in p1:
        np.testing.assert_array_equal(p1[k], p2[k], err_msg=k)
    check_phase_b(p1, points_with_in_residual(W["res_point"], g1["newState"], len(D)), prior_f(W), D, D)
    # ---- (d) the same linearisation against the oracle at depths D (input states = what the committed linearisation left)
    W2 = dict(W, idepth=D.copy(), idepth_zero=D.copy(), res_state=C["newState"].copy(), res_energy=C["newEnergy"].copy())
    ow2 = orc.Window(W2)
    E_o = ow2.linearize_all(update_th=False)
    _, _, a1 = check_linearize_parity(ow2, ba, r, E_o)          # commits ba's fused linearisation
    ba2.apply_res()
    a2 = ba2.accumulate()
    for k in ("HA", "bA", "Hsc", "bsc"):
        np.testing.assert_array_equal(a1[k], a2[k], err_msg=k)
    ba2.close()
    # one more fused step, with the oracle's x on both sides (the GPU's and the oracle's solutions differ by up to 1e-3 relative)
    x_o, _, _ = ow2.solve(0, 1e-5, 1)
    step_o = ow2.point_outputs()["step"]
    ba.backup_points()
    ba.gn_step(x_o, *tabs)
    D3, _ = ba.get_idepth()
    step_g = D3.astype(np.float64) - D
    np.testing.assert_allclose(step_g, step_o, rtol=2e-3, atol=2e-4 * np.abs(step_o).max() + ulp32(D3).max())
    ba.close()


@pytest.mark.parametrize("P", [16, 32])
def test_accept_reject_chain(capi, orc, synth, P):
    """backup -> step x1 (accepted) -> backup -> step x2 (rejected: restore, relinearise at the backup) -> backup -> step x3; every step within
    bound (a) of its own stage's committed linearisation, the restore exact in idepth and idepth_zero"""
    W = _window(synth, dict(nf=8, npts=777, seed=99, hosts="all"))
    ow = orc.Window(W)
    adH, adT = ow.adjoints()
    tabs = _tables(ow)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P, max_points=_max_points(W))
    ba.linearize(); ba.apply_res()
    idb = W["idepth"].astype(np.float32)
    # accept
    C1, x1 = _committed(ba), _solve(ba, W)
    ba.backup_points()
    ba.gn_step(x1, *tabs)
    D1, _ = ba.get_idepth()
    check_step(W, x1, C1, adH, adT, idb, D1)
    ba.apply_res()
    # reject
    C2, x2 = _committed(ba), 3.0 * _solve(ba, W)
    ba.backup_points()
    ba.gn_step(x2, *tabs)
    D2, _ = ba.get_idepth()
    check_step(W, x2, C2, adH, adT, D1, D2)
    ba.restore_points()
    idd, idz = ba.get_idepth()
    np.testing.assert_array_equal(idd, D1)
    np.testing.assert_array_equal(idz, D1)
    ba.gn_step(None, *tabs)
    ba.apply_res()
    # accept again, from the restored depths
    C3, x3 = _committed(ba), _solve(ba, W)
    ba.backup_points()
    ba.gn_step(x3, *tabs)
    D3, D3z = ba.get_idepth()
    check_step(W, x3, C3, adH, adT, D1, D3)
    np.testing.assert_array_equal(D3, D3z)
    ba.close()

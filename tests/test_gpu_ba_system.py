"""The systems ba_fused_kernel accumulates, checked entry by entry without the oracle's rounding in the way:

  (a) the Schur complement [H_sc | b_sc] against an fp64 evaluation on the launch's own committed outputs (JpJdF, Hcd, HdiF, bdSumF and the
      fp32 adjoints), within a rounding bound derived from the kernel's summation depths;
  (b) the top system [H_A | b_A] is additive over whole chunks (P consecutive points of one host frame): a chunk's partial does not depend on
      any other chunk, and a chunk whose residuals all enter as OOB with energy 0 adds exact zeros.  Linearising the window once per part of
      a partition of its chunks, with every residual outside the part forced to OOB, must give parts that add up to the whole window's
      system (fp64 reassociation only), counters and energy;
  (c) the marginalisation launch (dmv_ba_marginalize_points) against the plain launch: with zero deltas it is the plain launch on the
      flagged points bit for bit; a shift delta of the linearisation point changes only the right-hand sides, by exactly -M delta and
      -M_sc delta up to fp32 rounding.

Windows: tests/test_gpu_ba.py's CONFIGS plus a EuRoC-shaped one (752x480), at both chunk shapes."""
import numpy as np
import pytest

from helpers import (EPS32, EPS64, RES_IN, RES_OOB, check_system, energy_bound, make_case, product_ba_from_oracle, schur_bound,
                     schur_reference)
from test_gpu_ba import CONFIGS, cfg_id
from gpu_harness import device_capi  # noqa: F401  (the "capi" fixture: every test that takes it needs the device)

pytestmark = pytest.mark.gpu

SYS_CONFIGS = CONFIGS + [dict(nf=7, npts=2000, seed=1234, w=752, h=480)]   # EuRoC's image shape
TPB = {16: 448, 32: 224}                                                    # threads per CTA of each chunk shape (ba_fused.cu FusedCfgOf)


def sys_id(c):
    return cfg_id(c) + (f"_{c['w']}x{c['h']}" if "w" in c else "")


def check_bound(got, want, bound, what):
    """|got - want| <= bound entry by entry (exact equality where the bound is 0); returns max |error| / bound"""
    err = np.abs(np.asarray(got, np.float64) - want)
    zero = bound == 0
    assert not np.any(zero & (err != 0)), f"{what}: non-zero where the reference is an exact 0"
    ratio = np.where(zero, 0.0, err / np.where(zero, 1.0, bound))
    worst = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    assert ratio[worst] <= 1.0, f"{what}{list(worst)}: got {got[worst]:.9e}, fp64 {want[worst]:.9e}, |error| {err[worst]:.3e} > bound {bound[worst]:.3e}"
    return float(ratio[worst])


@pytest.mark.parametrize("cfg", SYS_CONFIGS, ids=sys_id)
@pytest.mark.parametrize("P", [16, 32])
def test_schur_against_fp64(capi, orc, synth, cfg, P):
    """(a) H_sc = sum_p HdiF_p v_p v_p^T and b_sc = sum_p HdiF_p bdSumF_p v_p (helpers.schur_reference) from the launch's own outputs.

    Rounding bound, per entry: gamma eps32 Habs_ij, Habs the same sum over the absolute value of every product, u = eps32 / 2:
      * a host-block entry of v_p is an 8-term fp32 dot adHostF @ JpJdF per target (<= 8 u), summed over <= 7 targets (<= 7 u): 15 u;
        target-block entries one product (u); Hcd, HdiF and bdSumF are the launch's outputs themselves (exact);
      * phase E: HdiF * v_i (u), times v_j (u), per-thread fp32 sums over m = ceil(npts / TPB) points (m u), TPB = 448 (P = 16) or 224
        (P = 32), then the 5-step fp32 butterfly (5 u), then fp64 across warps (< u);
    so |error| <= (15 + 15 + 1 + 1 + m + 5 + 1) u Habs = (m + 38) / 2 eps32 Habs (first order)."""
    schur_against_fp64(capi, orc, make_case(synth, cfg), P, sys_id(cfg))


def schur_against_fp64(capi, orc, W, P, name):
    """test_schur_against_fp64 on the window W"""
    ow = orc.Window(W)
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    ba.linearize()
    ba.apply_res()
    g, po, a = ba.residual_outputs(), ba.point_outputs(), ba.accumulate()
    adH, adT = ow.adjoints()
    Hsc, bsc, Habs, babs = schur_reference(W, g["newState"], g["JpJdF"], po["Hcd"], po["HdiF"], po["bdSumF"], adH, adT)
    m = -(-len(W["host"]) // TPB[P])
    gamma = (m + 38) / 2
    rH = check_bound(a["Hsc"], Hsc, gamma * EPS32 * Habs, "H_sc")
    rb = check_bound(a["bsc"], bsc, gamma * EPS32 * babs, "b_sc")
    jH, jb = check_system(a["Hsc"], a["bsc"], Hsc, bsc, schur_bound(po["HdiF"], po["bdSumF"]), 1.0, "Schur system vs fp64")  # reported only
    print(f"P={P} {name}: H_sc |err|/bound {rH:.3f}  b_sc {rb:.3f}  (gamma {gamma}); Jacobi-scaled H {jH:.2e} b {jb:.2e}")
    assert np.abs(Hsc).max() > 0
    ba.close()


def _chunks(host, P):
    """global chunk index of every point (chunks: P consecutive points of one host frame, hosts ascending, as dmv_ba_set_points lays them out)"""
    host = np.asarray(host)
    assert np.all(np.diff(host) >= 0)
    ch = np.zeros(len(host), np.int64)
    c0 = 0
    for h in range(int(host.max()) + 1):
        idx = np.nonzero(host == h)[0]
        ch[idx] = c0 + np.arange(len(idx)) // P
        c0 += -(-len(idx) // P)
    return ch, c0


def _linearize(capi, W, ow, P, state, energy):
    ba = product_ba_from_oracle(capi, dict(W, res_state=state, res_energy=energy), ow, chunk_points=P)
    r = ba.linearize()
    g = ba.residual_outputs()
    ba.apply_res()
    a = ba.accumulate()
    ba.close()
    return r, g, a


@pytest.mark.parametrize("cfg", SYS_CONFIGS, ids=sys_id)
@pytest.mark.parametrize("P", [16, 32])
def test_top_system_additive_over_chunks(capi, orc, synth, cfg, P):
    """(b) partitions by host frame, alternate chunks and (on the 8000-point windows: several chunks per CTA at P = 16, hosts long enough for
    phase D's dsum_long path) a seeded random half of the chunks.  Per part: the residuals of its chunks keep their input state and energy,
    every other residual enters as OOB with energy 0.  Expected: H_A, b_A of the parts add up to the whole window's within
    2 (nchunks + K) eps64 Jacobi-scaled (fp64 reassociation of the chunk partials, whose absolute sum Cauchy-Schwarz bounds by the diagonal
    scale); n_in, n_outlier, resInA add up exactly, n_oob once the residuals each part forced to OOB are taken off; the energy within fp64
    reassociation of its per-chunk sums; and every residual's outputs in its own part equal the whole window's bit for bit."""
    W = make_case(synth, cfg)
    ow = orc.Window(W)
    nres = len(W["res_point"])
    st0 = np.asarray(W.get("res_state", np.zeros(nres)), np.int32)
    en0 = np.asarray(W.get("res_energy", np.zeros(nres)), np.float32)
    r, g, a = _linearize(capi, W, ow, P, st0, en0)
    R = energy_bound(g["newState"], g["newEnergy"])
    ch, nch = _chunks(W["host"], P)
    res_ch = ch[W["res_point"]]
    parts = dict(host=np.asarray(W["host"])[W["res_point"]], alternate=res_ch % 2)
    if cfg["npts"] == 8000:
        parts["random"] = (np.random.default_rng(cfg["seed"]).random(nch) < 0.5).astype(np.int64)[res_ch]
    worst = 0.0
    for name, part in parts.items():
        keys = np.unique(part)
        K = len(keys)
        HA, bA = np.zeros_like(a["HA"]), np.zeros_like(a["bA"])
        n_in = n_outl = n_oob = resIn = 0
        E, Eabs = 0.0, 0.0
        for k in keys:
            mine = part == k
            rk, gk, ak = _linearize(capi, W, ow, P, np.where(mine, st0, RES_OOB).astype(np.int32), np.where(mine, en0, 0).astype(np.float32))
            HA += ak["HA"]
            bA += ak["bA"]
            n_in += rk["n_in"]; n_outl += rk["n_outlier"]; n_oob += rk["n_oob"] - int((~mine).sum()); resIn += ak["resInA"]
            E += rk["energy"]; Eabs += abs(rk["energy"])
            for key in ("newState", "newEnergy", "newEnergyWithOutlier", "centerProjectedTo"):
                np.testing.assert_array_equal(gk[key][mine], g[key][mine], err_msg=f"{name} part {k}: {key}")
            inn = mine & (g["newState"] == RES_IN)
            np.testing.assert_array_equal(gk["JpJdF"][inn], g["JpJdF"][inn], err_msg=f"{name} part {k}: JpJdF")
            assert np.all(gk["newState"][~mine] == RES_OOB)
        tau = 2 * (nch + K) * EPS64
        rH, rb = check_system(HA, bA, a["HA"], a["bA"], R, tau, f"sum of the {K} '{name}' parts")
        worst = max(worst, rH / tau, rb / tau)
        assert (n_in, n_outl, n_oob, resIn) == (r["n_in"], r["n_outlier"], r["n_oob"], a["resInA"]), name
        assert abs(E - r["energy"]) <= tau * Eabs, (name, E, r["energy"])
    print(f"P={P} {sys_id(cfg)}: {nch} chunks, parts {list(parts)}: worst |error| / (2 (nchunks + K) eps64 scale) = {worst:.3f}")


def _marg_window(synth, cfg, frac=0.33):
    """depth priors on ~30 % of the points with idepth_zero == idepth (EFPoint::deltaF = 0), mixed input states, a flagged set S"""
    W = synth.make_window(**cfg)
    rng = np.random.default_rng(cfg["seed"] + 5)
    npts, nres = len(W["host"]), len(W["res_point"])
    W["idepth_zero"] = W["idepth"].copy()
    W["hasDepthPrior"] = (rng.random(npts) < 0.3).astype(np.uint8)
    W["res_state"] = rng.choice([0, 1, 2], nres, p=[0.8, 0.1, 0.1]).astype(np.int32)
    W["res_energy"] = rng.uniform(0, 50, nres).astype(np.float32)
    S = np.sort(rng.choice(npts, int(npts * frac), replace=False)).astype(np.int32)
    return W, S


MARG_CONFIGS = [dict(nf=7, npts=2000, seed=1234), dict(nf=8, npts=777, seed=99, hosts="all")]


@pytest.mark.parametrize("cfg", MARG_CONFIGS, ids=cfg_id)
@pytest.mark.parametrize("P", [16, 32])
def test_marg_launch_against_plain_launch(capi, orc, synth, cfg, P):
    """(c) zero deltas: marginalize_points(S, adHTdeltaF = 0, cDeltaF = 0, prior_fac = 1) == a plain linearize + apply_res + accumulate of the
    window whose residuals of S enter as IN with energy 0 and all others as OOB, bit for bit (res_toZeroF = resF exactly when every delta is
    0, and with idepth_zero == idepth the plain launch's shiftPriorToZero adds an exact 0).

    Non-zero deltas delta (frames: pose ~1e-3, affine ~1e-4; camera ~1e-3), adHTdeltaF[h + t nf] = fp32(delta_h^T adHostF + delta_t^T
    adTargetF) as EnergyFunctional::setDeltaF forms it: M, Msc, isLinearized, ngood are unchanged bit for bit, and
      Mb(delta) = Mb(0) - M delta~,   Mbsc(delta) = Mbsc(0) - Msc delta~     (delta~ = the fp32 delta)
    within c eps32 sqrt(M_ii) (sqrt(delta~^T M delta~) + sqrt(sum rtz_0^2) + sqrt(sum rtz_delta^2)).  c: each right-hand side is a sum of
    J rtz over the residuals' pixels (8 fp32 terms, <= 5 butterfly steps, then fp64), <= 16 u of sum |J| |rtz| <= 16 u sqrt(M_ii) |rtz|
    (Cauchy-Schwarz) per launch; rtz = resF - gx jpx - gy jpy - ja dp6 - jb dp7 takes 4 roundings and jpx, jpy an 11-term dot each, and
    adHTdeltaF rounds the shift once more (<= 16 u of |J delta| per pixel); first order: 2 x 16 + 16 = 48 u = 24 eps32, c = 32."""
    W, S = _marg_window(synth, cfg)
    ow = orc.Window(W)
    nf, nres = W["nf"], len(W["res_point"])
    N = 8 * nf + 4
    ba = product_ba_from_oracle(capi, W, ow, chunk_points=P)
    z0 = ba.marginalize_points(S, np.zeros((nf * nf, 8), np.float32), np.zeros(4, np.float32), prior_fac=1.0)
    inS = np.isin(W["res_point"], S)
    st = np.where(inS, RES_IN, RES_OOB).astype(np.int32)
    _, g, a = _linearize(capi, W, ow, P, st, np.zeros(nres, np.float32))
    for km, ka in (("M", "HA"), ("Mb", "bA"), ("Msc", "Hsc"), ("Mbsc", "bsc")):
        np.testing.assert_array_equal(z0[km], a[ka], err_msg=f"{km} != {ka} of the plain launch")
    assert z0["resInM"] == a["resInA"]
    lin = inS & (g["newState"] == RES_IN)
    np.testing.assert_array_equal(z0["isLinearized"], lin.astype(np.uint8))
    np.testing.assert_array_equal(z0["ngood"], np.bincount(W["res_point"][lin], minlength=len(W["host"]))[S])
    assert lin.sum() > 0 and np.abs(z0["Mb"]).max() > 0
    # ---- non-zero deltas
    rng = np.random.default_rng(cfg["seed"] + 6)
    dfr = np.concatenate([1e-3 * rng.standard_normal((nf, 6)), 1e-4 * rng.standard_normal((nf, 2))], 1).astype(np.float32).astype(np.float64)
    dc = (1e-3 * rng.standard_normal(4)).astype(np.float32)
    adH, adT = ow.adjoints()
    AH = adH.astype(np.float32).astype(np.float64)
    AT = np.einsum("ikk->ik", adT).astype(np.float32).astype(np.float64)
    adHT = np.zeros((nf * nf, 8), np.float32)
    for h in range(nf):
        for t in range(nf):
            adHT[h + t * nf] = dfr[h] @ AH[h + t * nf] + dfr[t] * AT[h + t * nf]
    z1 = ba.marginalize_points(S, adHT, dc, prior_fac=1.0)
    ba.close()
    for k in ("M", "Msc", "isLinearized", "ngood"):
        np.testing.assert_array_equal(z1[k], z0[k], err_msg=f"{k} depends on the deltas")
    assert z1["resInM"] == z0["resInM"]
    d = np.concatenate([dc.astype(np.float64), dfr.reshape(-1)])
    assert d.shape == (N,)
    norms = np.sqrt((z0["rtz"].astype(np.float64) ** 2).sum()) + np.sqrt((z1["rtz"].astype(np.float64) ** 2).sum())
    c = 32
    ratios = []
    for kH, kb in (("M", "Mb"), ("Msc", "Mbsc")):
        H = z0[kH]
        want = z0[kb] - H @ d
        shift = float(d @ H @ d)
        assert shift > 0
        bound = c * EPS32 * np.sqrt(np.maximum(np.diag(H), 0)) * (np.sqrt(shift) + norms)
        ratios.append(check_bound(z1[kb], want, bound, f"{kb}(delta) - ({kb}(0) - {kH} delta)"))
        moved = np.abs(z1[kb] - z0[kb])
        assert moved.max() > 100 * bound.max(), f"{kb}: the deltas hardly move the right-hand side; the check would be blunt"
    print(f"P={P} {cfg_id(cfg)}: marg vs plain bit-identical; delta identity |err|/bound Mb {ratios[0]:.3f} Mbsc {ratios[1]:.3f}")

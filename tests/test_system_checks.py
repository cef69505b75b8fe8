"""The per-entry system checks of the BA tests (helpers.check_system, helpers.schur_reference) proven on the CPU oracle: the fp64 Schur
reference reproduces the oracle's own Schur complement, and check_system accepts what it must (the oracle's faithful-float system) and
rejects the errors a whole-matrix Frobenius ratio lets through (a wrong camera block, a wrong affine right-hand side, a misplaced or dropped
frame-pair block).  No GPU."""
import numpy as np
import pytest

from helpers import RES_IN, RES_OOB, SYSTEM_TAU, check_system, energy_bound, make_case, rel, schur_bound, schur_reference

WINDOWS = [dict(nf=7, npts=2000, seed=1234), dict(nf=8, npts=777, seed=99, hosts="all", edge=True), dict(nf=2, npts=200, seed=1234, hosts="first")]


def _id(c):
    return f"nf{c['nf']}_n{c['npts']}" + ("_edge" if c.get("edge") else "")


def _oracle_system(orc, synth, cfg):
    W = make_case(synth, cfg)
    ow = orc.Window(W)
    ow.linearize_all(update_th=False)
    ow.apply_res()
    a = ow.accumulate(1)
    o, po = ow.res_outputs(False), ow.point_outputs()
    adH, adT = ow.adjoints()
    return W, ow, a, o, po, adH, adT


@pytest.mark.parametrize("cfg", WINDOWS, ids=_id)
def test_schur_reference_reproduces_oracle(orc, synth, cfg):
    """schur_reference on the oracle's committed point outputs == the oracle's fp64 H_sc, b_sc within 1e-6 Jacobi-scaled (measured <= 7e-8)"""
    W, _, a, o, po, adH, adT = _oracle_system(orc, synth, cfg)
    Hsc, bsc, _, _ = schur_reference(W, o["newState"], o["JpJdF"], po["Hcd"], po["HdiF"], po["bdSumF"], adH, adT)
    rH, rb = check_system(Hsc, bsc, a["Hsc"], a["bsc"], schur_bound(po["HdiF"], po["bdSumF"]), 1e-6, "Schur reference")
    print(f"{_id(cfg)}: Schur reference vs oracle: H {rH:.2e}  b {rb:.2e}")


@pytest.mark.parametrize("cfg", WINDOWS, ids=_id)
def test_check_system_accepts_faithful_float(orc, synth, cfg):
    """the oracle's faithful-float accumulation (the reference's fp32 accumulators) passes at SYSTEM_TAU (measured <= 8e-7)"""
    W, ow, a, o, po, _, _ = _oracle_system(orc, synth, cfg)
    a0 = ow.accumulate(0)
    check_system(a["HA"], a["bA"], a["HA"], a["bA"], 1.0, 0.0, "identical system")
    r = (check_system(a0["HA"], a0["bA"], a["HA"], a["bA"], energy_bound(o["newState"], o["newEnergy"]), SYSTEM_TAU, "float top system")
         + check_system(a0["Hsc"], a0["bsc"], a["Hsc"], a["bsc"], schur_bound(po["HdiF"], po["bdSumF"]), SYSTEM_TAU, "float Schur system"))
    print(f"{_id(cfg)}: faithful float vs fp64: " + " ".join(f"{x:.2e}" for x in r))
    assert max(r) <= 1e-6


@pytest.mark.parametrize("cfg", WINDOWS, ids=_id)
def test_check_system_rejects_perturbations(orc, synth, cfg):
    """check_system at SYSTEM_TAU rejects each perturbation and names the entry; the whole-matrix ratio accepts the camera one"""
    W, _, a, o, po, adH, adT = _oracle_system(orc, synth, cfg)
    nf = W["nf"]
    RA, RS = energy_bound(o["newState"], o["newEnergy"]), schur_bound(po["HdiF"], po["bdSumF"])

    def rejects(H, b, H_ref, b_ref, R, what, entry):
        """check_system fails, and its message names the perturbed entry (regular expression `entry`)"""
        with pytest.raises(AssertionError, match=entry):
            check_system(H, b, H_ref, b_ref, R, SYSTEM_TAU, what)

    # the camera block 10 % wrong: invisible to the whole-matrix ratio of the former check (rel < 1e-5)
    H = a["HA"].copy()
    H[:4, :4] *= 1.1
    rejects(H, a["bA"], a["HA"], a["bA"], RA, "camera block", r"H\[camera \d, camera \d\]")
    assert rel(H, a["HA"]) < 1e-5, "the gap this check closes: a whole-matrix ratio accepts a 10 % wrong camera block"
    # one affine-b entry of b_A doubled (the frame where that entry is largest on its scale)
    s = np.sqrt(np.diag(a["HA"]))
    ib = np.array([4 + 8 * f + 7 for f in range(nf)])
    i = ib[np.argmax(np.abs(a["bA"][ib]) / s[ib])]
    b = a["bA"].copy()
    b[i] *= 2
    rejects(a["HA"], b, a["HA"], a["bA"], RA, "affine b", rf"b\[frame {(i - 4) // 8} b\]")
    # one off-diagonal 8x8 frame-pair block transposed (and its mirror, so that H stays symmetric)
    f1, f2 = 0, nf - 1
    r1, r2 = slice(4 + 8 * f1, 12 + 8 * f1), slice(4 + 8 * f2, 12 + 8 * f2)
    H = a["HA"].copy()
    H[r1, r2] = a["HA"][r1, r2].T
    H[r2, r1] = a["HA"][r2, r1].T
    rejects(H, a["bA"], a["HA"], a["bA"], RA, "pair block", rf"H\[frame ({f1}|{f2}) .*, frame ({f1}|{f2}) ")
    # the Schur contribution of one frame pair dropped: the pair with the fewest IN residuals
    host = W["host"][W["res_point"]]
    inn = o["newState"] == RES_IN
    pairs = [(int(np.sum(inn & (host == h) & (W["res_target"] == t))), h, t) for h in range(nf) for t in range(nf) if h != t]
    n, h, t = min(p for p in pairs if p[0] > 0)
    st = o["newState"].copy()
    st[inn & (host == h) & (W["res_target"] == t)] = RES_OOB
    Hd, bd, _, _ = schur_reference(W, st, o["JpJdF"], po["Hcd"], po["HdiF"], po["bdSumF"], adH, adT)
    rejects(Hd, bd, a["Hsc"], a["bsc"], RS, f"Schur without pair {h}->{t}", rf"\[frame ({h}|{t}) ")
